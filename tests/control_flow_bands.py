"""Bands built to take one exit of the LM / outer loops of optimizeTEB deterministically, shared by
tests/test_reference_pin_edges.py (oracle against the reference's code) and tests/test_gpu_control_flow.py (device
against the oracle, and every launch schedule against every other).

Z  zero chi2: exactly representable, evenly spaced straight poses at y = 40 (far outside every obstacle threshold of
   the scenes here), dt = 0.25 inside autoResize's band [dt_ref - hyst, dt_ref + hyst], vel_start = vel_goal = the
   band's velocity 0.25 m/s. With weight_optimaltime = 0 every edge error is exactly 0. Every edge of the band is a
   penalty (flat where it is zero) or a norm taken at zero, so every Jacobian is 0 as well: H = 0, b = 0 and lambda =
   1e-5 max diag = 0. Every trial's factorisation fails (tempChi = DBL_MAX, rho < 0), so the first LM iteration of each
   outer iteration ends with ten rejections (nu = 2^11, lambda 0) and Terminate: lm_iters == outer, cost 0. In the
   latency regime's {8, 2} schedule the tenth rejection falls in round 1, on the retry side stream.
N  NaN: the Z band with x = NaN at one interior pose. H holds NaN and zeros, lambda = 0, the factorisation fails on
   every trial (tempChi = DBL_MAX, currentChi NaN, rho NaN): one trial per LM iteration, never Terminate, CHOL_FAILED.
   The reference asserts on a non-finite edge error (ROS_ASSERT in EdgeVelocity::computeError), so N is pinned against
   the oracle only.
S  shifting: a zero-chi2 straight band of exact, unevenly spaced poses (every speed <= 0.25 m/s) that autoResize
   changes in its first pass and again in its second, with chi2 and H still exactly 0 after the first. It takes Z's
   exit, so it is carried out of the first outer iteration, and the carried autoResize (on the side stream in the
   latency regime) is real work: the band after two outer iterations is the two-pass resize of the input.
P  rho == 0: the Z band under params(shortest_path=True). The shortest-path edges give H != 0 (lambda > 0) and, with
   evenly spaced poses, b = 0 exactly, so dx = 0, tempChi == currentChi and rho == 0: one rejected trial, Terminate
   with nu = 4, in every outer iteration.
D  disabled: max_vel_x < 0.01 (a parameter, so a batch of its own). autoResize runs once (dt = 0.75 > 2 dt_ref: poses
   are inserted), then optimizeGraph refuses: DISABLED, optimizeTEB returns false, cost stays HUGE_VAL.
"""
import numpy as np

from teb_local_planner_b200 import abi, scenes

Z_STEP, Z_DT, Z_Y = 0.0625, 0.25, 40.0
Z_VEL = Z_STEP / Z_DT           # 0.25 m/s, exactly


def params(autosize=True, shortest_path=False):
    """C3's parameters (inflated obstacles, turning radius) without the time-optimal and acceleration edges, which Z and
    S need, and without dynamic obstacles (the scenes here have none), so that autoResize runs its single fast-mode
    pass. shortest_path: weight_shortest_path = 1, which P needs."""
    p = scenes.config_params("C3")
    p.teb_autosize = int(autosize)
    p.include_dynamic_obstacles = 0
    p.weight_optimaltime = 0.0
    p.weight_acc_lim_x = p.weight_acc_lim_theta = 0.0
    p.weight_shortest_path = 1.0 if shortest_path else 0.0
    return p


def z_band(n, n_cap, x0=-2.0):
    rec = np.zeros((n_cap, 4))
    rec[:n, 0] = x0 + Z_STEP * np.arange(n)
    rec[:n, 1] = Z_Y
    rec[:n - 1, 3] = Z_DT
    return rec


def n_band(n, n_cap, at=None):
    rec = z_band(n, n_cap)
    rec[n // 2 if at is None else at, 0] = np.nan
    return rec


def d_band(n, n_cap):
    """an ordinary straight band whose dt are long enough for autoResize to insert poses"""
    rec = np.zeros((n_cap, 4))
    rec[:n, 0] = -2.0 + 0.3 * np.arange(n)
    rec[:n - 1, 3] = 0.75
    return rec


Z_VEL4 = np.array([Z_VEL, 0.0, 0.0, 1.0])


def resize_twice_band(p, auto_resize, seed=5):
    """the first seeded random band (n 10-50, dt 0.05-1.05 s) that a second fast-mode autoResize pass still changes:
    with autosize on and no inner iterations only the first outer iteration may resize it. auto_resize: the oracle's."""
    rng = np.random.default_rng(seed)
    while True:
        n = int(rng.integers(10, 51))
        rec = np.zeros((n, 4))
        rec[:, 0] = np.cumsum(rng.uniform(0.05, 0.4, n))
        rec[:, 1] = rng.uniform(-0.2, 0.2, n)
        rec[:-1, 3] = rng.uniform(0.05, 1.05, n - 1)
        a = auto_resize(rec, n, p.dt_ref, p.dt_hysteresis, p.min_samples, p.max_samples, 1)
        b = auto_resize(a, len(a), p.dt_ref, p.dt_hysteresis, p.min_samples, p.max_samples, 1)
        if len(a) != len(b) or not np.array_equal(a, b):
            return rec, n


def shifting_band(p, oracle, seed=1):
    """S: the first seeded band that satisfies its defining property (see the module docstring). oracle: the binding."""
    rng = np.random.default_rng(seed)
    kw = dict(obstacles=ordinary_batch().obstacles[0], vel_start=Z_VEL4, vel_goal=Z_VEL4)
    resize = lambda r: oracle.auto_resize(r, len(r), p.dt_ref, p.dt_hysteresis, p.min_samples, p.max_samples, 1)
    while True:
        n = 24
        dt = rng.choice([0.125, 0.1875, 0.25, 0.5, 0.75, 1.25], n - 1)
        rec = np.zeros((n, 4))
        rec[:, 0] = -2.0 + np.concatenate([[0.0], np.cumsum(dt * Z_VEL)])
        rec[:, 1] = Z_Y
        rec[:-1, 3] = dt
        once = resize(rec)
        twice = resize(once)
        if len(twice) == len(once) and np.array_equal(twice, once):
            continue
        if all(c == 0.0 and not H.any() for H, _, c in (oracle.build_system(p, r, len(r), **kw) for r in (rec, once))):
            return rec, n


def ordinary_batch(n=40, M=16, candidates=8, seed=3, n_cap=160):
    """ordinary C3-like bands (lateral sinusoids through inflated obstacles), scene 0"""
    return scenes.make_batch(n, M, candidates, 1, seed, inflated=True, n_cap=n_cap, amp=1.0)


def set_band(hb, b, rec, n, vel=None):
    hb.poses[b] = 0.0
    hb.poses[b, :len(rec)] = rec[:hb.n_cap]
    hb.n[b] = n
    hb.vel_start[b] = (0, 0, 0, 1) if vel is None else vel
    hb.vel_goal[b] = (0, 0, 0, 1) if vel is None else vel


def mixed_batch(kinds, n=40, n_cap=160, M=16, seed=3, s_band=None):
    """a batch whose band b is kinds[b]: 'Z' (also P's band), 'N', 'S' (s_band = shifting_band(...)), or any other
    letter for the next ordinary band of the seeded scene"""
    ob = ordinary_batch(n, M, max(1, sum(k not in "ZPNS" for k in kinds)), seed, n_cap)
    hb = scenes.make_batch(n, M, len(kinds), 1, seed, inflated=True, n_cap=n_cap, amp=1.0)
    hb.obstacles[:] = ob.obstacles
    k = 0
    for b, kind in enumerate(kinds):
        if kind in "ZP":
            set_band(hb, b, z_band(n, n_cap), n, Z_VEL4)
        elif kind == "S":
            set_band(hb, b, s_band[0], s_band[1], Z_VEL4)
        elif kind == "N":
            set_band(hb, b, n_band(n, n_cap), n, Z_VEL4)
        else:
            set_band(hb, b, ob.poses[k], int(ob.n[k]))
            k += 1
    return hb


def band_kwargs(hb, b):
    return dict(obstacles=hb.obstacles[0][:hb.obst_count[0]], vel_start=hb.vel_start[b], vel_goal=hb.vel_goal[b])


def args(inner, outer, cost=True, alt_time=False):
    return abi.make_args(inner, outer, cost, 2.0, 1.0, alt_time)


# (outer, inner) pairs at the argument edges of optimizeTEB and around them
EDGES = [(0, 5), (1, 0), (3, 0), (1, 1), (2, 1), (4, 5)]
