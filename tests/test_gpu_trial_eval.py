"""Every trial-evaluation kernel of the LM step, trial by trial, through tebgpu_eval_trials (TebGpu.eval_trials).

The end-to-end tests compare whole optimizeTEB runs, where a chi2 slightly wrong in one family shifts rho without
flipping a decision, and the rare branches of g2o's accept / reject chain never run. Here one round of trial
evaluation is pinned, for k_trial_eval2 (wide and one CTA per band, staged and global-table), the persistent
k_trial_eval2p (B > 2 x SMs), k_trial_eval3 and the first-generation k_trial_eval, all launched by launch_trial_eval as
in an optimize call (k_trial_eval2p with several bands per CTA: tests/test_gpu_trial_eval_persistent.py):
  a. each trial's chi2 by family (obstacles, via, time-optimal, other) against teb_oracle_trial_chi2 (long double, graph
     frozen at the linearisation point) within 1e-12 relative per family, every scenario at outer 0 and 3, on real LM
     steps, random steps of 1e-8 .. 1e-1 of the state, theta carried across +-pi, dt driven to 0 and below, dx = 0;
     computeScale() against a long-double sum dx (lambda dx + b), b from the oracle;
  b. at dx = 0 the trial chi2 per family equals kernel A's (29-pose tiles against 30-pose tiles) within 1e-13; the gap
     is reported in ulps;
  c. the decisions against teb_oracle_lm_decide fed the device's rows: trials consumed, need, Terminate, status bits
     and the committed state equal, lambda within 2 ulp (the device cubes by products, the oracle with pow); crafted
     rounds: failed factorisations, NaN trials, a band of chi2 exactly 0, lambda overflowing, retry rounds from trial
     4, 6, 8 and 9 (bands that reject every trial reach the 10-trial cap and terminate, or are queued again),
     iteration 0 against later ones. Fed the oracle's own chi2 (currentChi and tempChi), the decisions agree except
     where |currentChi - tempChi| lies within the chi2 bar (counted and reported);
  d. commit and hygiene, bit for bit: the accepted state is x [+] dx formed with teb_oracle_normalize_theta, on
     west-going bands whose accepted LM steps carry headings across +-pi (at least one such commit required); pose 0,
     the xyz of pose n-1, dt_{n-1}, records past n, rejected and inactive bands are untouched; res rows of trials that
     do not exist keep the all-ones pattern; NaN records past n change nothing;
  e. shapes: n from 3 to 512 around every 29 / 30-pose tile edge, n_cap = n and n_cap > n, K = 2 .. 8, ragged batches;
  f. every k_trial_eval2 / 2p launch and k_trial_eval3 give the same bits wherever a band sits (batch position among active
     neighbours with other trials, retry-list position), the global-table builds the bits of the staged ones;
     k_trial_eval agrees within 1e-13.
The worst errors per family go to the parity report that tests/test_gpu_parity.py writes, per kernel build (eval2 at
the scenario batch sizes, eval2_wide, eval2p, eval3, the global-table builds, v1), with the number of accepted
commits that crossed the theta cut."""
import os
import sys

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import banded_reference as R
from tests import oracle_binding as O
from tests import scenarios
from tests.param_cases import weight_multiplier
from tests.test_gpu_parity import _report as _write_report

pytestmark = pytest.mark.gpu

FAM_BAR = 1e-12       # per family, relative
LIN_BAR = 1e-13       # dx = 0 against kernel A, relative per family
SCALE_BAR = 1e-11     # computeScale() relative to sum |dx| (|lambda dx| + |b|)
ALL_ONES = np.uint64(0xFFFFFFFFFFFFFFFF)
TERMINATED = abi.TEB_STATUS_TERMINATED
DBL_MAX = sys.float_info.max
_worst = {}


def _report(key, value, kind=max):
    _worst[key] = kind(_worst.get(key, value), value)
    _write_report("trial_eval", dict(sorted(_worst.items())))


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ctx(hb, p, build="eval2", max_bands=None, max_obstacles=None):
    """a context whose trial evaluation is `build`: eval2 (the batch size picks wide / 512 / 256), eval3 or v1"""
    env = {"eval2": ("0", "0"), "eval3": ("1", "0"), "v1": ("0", "1")}[build]
    old = {k: os.environ.get(k) for k in ("TEBGPU_EVAL3", "TEBGPU_EVAL_V1")}
    os.environ["TEBGPU_EVAL3"], os.environ["TEBGPU_EVAL_V1"] = env
    try:
        g = T.TebGpu(max_bands or hb.B, hb.n_cap, hb.S, max_obstacles or max(hb.M_cap, 1), hb.V_cap,
                     max_obst_vertices=hb.PV_cap)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v
    g.set_params(p)
    return g


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _same_bits(a, b):
    return np.array_equal(_bits(a), _bits(b))


def _state(B, lam=0.0, nu=2.0, chi=0.0, parts_cur=0.0, parts_last=0.0, status=0, active=1):
    s = np.zeros((B, T.TebGpu.EVAL_STATE))
    s[:, 0], s[:, 1], s[:, 2] = lam, nu, chi
    s[:, 3:7] = np.broadcast_to(parts_cur, (B, 4)) if np.ndim(parts_cur) else parts_cur
    s[:, 7:11] = np.broadcast_to(parts_last, (B, 4)) if np.ndim(parts_last) else parts_last
    s[:, 11], s[:, 12] = status, active
    return s


def _real(n, n_cap):
    r = np.arange(4 * n_cap)
    return (R.row_is_real(r, n) & (r < 4 * n)).reshape(n_cap, 4)


def _oplus(rec, d, n):
    """x [+] dx on the host: VertexPose / VertexTimeDiff oplus with the oracle's normalize_theta, real rows only"""
    out = rec.copy()
    real = _real(n, rec.shape[0])
    v = rec + d.reshape(rec.shape)
    out[real] = v[real]
    nt = O.lib().teb_oracle_normalize_theta
    for i in np.flatnonzero(real[:, 2]):
        out[i, 2] = nt(float(v[i, 2]))
    return out


class Round:
    """one eval_trials call and everything its checks need"""

    def __init__(self, g, p, hb, K, dx, ok, lam, state, outer=0, iteration=1, qmax=None, order=None):
        self.p, self.hb, self.K, self.outer, self.iteration = p, hb, K, outer, iteration
        self.dx, self.ok, self.lam = (np.ascontiguousarray(np.broadcast_to(a, s), dtype=np.float64) for a, s in
                                      ((dx, (hb.B, K, 4 * hb.n_cap)), (ok, (hb.B, K)), (lam, (hb.B, K))))
        self.state_in, self.qmax_in, self.order = state.copy(), qmax, order
        self.Hb, _ = g.build_system(hb, outer)
        self.after = hb.copy()
        self.out = g.eval_trials(self.after, K, self.dx, self.ok, self.lam, state, outer_index=outer, iteration=iteration,
                                 qmax=qmax, order=order)
        self.retry = qmax is not None

    def bands(self):
        """bands that evaluated trials in this round"""
        listed = set(range(self.hb.B)) if not self.retry else set(int(b) for b in self.order)
        return [b for b in sorted(listed) if self.state_in[b, 12] != 0]

    def q0(self, b):
        return int(self.qmax_in[b]) if self.retry else 0

    def kact(self, b):
        return min(self.K, 10 - self.q0(b))

    def step(self, b, k):
        """the dx the device applies: the trial's, or b for a failed factorisation"""
        return self.dx[b, k] if self.ok[b, k] != 0 else self.Hb[b, :, 11]

    def trial_state(self, b, k):
        return _oplus(self.hb.poses[b], self.step(b, k), int(self.hb.n[b]))


def _fam_errors(got, ref):
    """relative error per family; non-finite values must match in kind"""
    got, ref = np.asarray(got), np.asarray(ref)
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(got), fin), f"finite pattern: {got} vs {ref}"
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(got[np.isinf(ref)], ref[np.isinf(ref)])
    err = np.zeros(got.shape)
    err[fin] = np.abs(got[fin] - ref[fin]) / np.maximum(ref[fin], 1e-300)
    err[fin & (ref == 0) & (got == 0)] = 0
    return err


def _oracle_b(p, hb, b, outer):
    """the oracle's b of band b at its graph state, in the device's row order (row = oracle row + 3)"""
    n = int(hb.n[b])
    _, bd, _ = O.build_system(p, hb.poses[b], n, weight_multiplier=weight_multiplier(p, outer), jac_mode=O.JAC_ANALYTIC,
                              **scenarios.band_kwargs(hb, b))
    full = np.zeros(4 * hb.n_cap)
    full[3:3 + bd.size] = bd
    return full


def check_chi2(rd, build, bands=None):
    """a. rows against the oracle, per family; scale against a long-double sum"""
    p, hb = rd.p, rd.hb
    for b in (rd.bands() if bands is None else bands):
        n, kact = int(hb.n[b]), rd.kact(b)
        trials = np.stack([rd.trial_state(b, k)[:n] for k in range(kact)])
        ref = O.trial_chi2(p, hb.poses[b], n, trials, weight_multiplier=weight_multiplier(p, rd.outer), **scenarios.band_kwargs(hb, b))
        got = rd.out["res"][b, :kact]
        err = _fam_errors(got[:, :4], ref)
        for f, nm in enumerate(("obst", "via", "time", "other")):
            _report(f"{build}/chi2_{nm}_rel", float(err[:, f].max()))
        assert (err <= FAM_BAR).all(), f"{build} band {b}: family errors {err.max(axis=0)} rows {got[:, :4]} oracle {ref}"
        bo = _oracle_b(p, hb, b, rd.outer)
        real = _real(n, hb.n_cap).ravel()
        for k in range(kact):
            d = rd.step(b, k)[real].astype(np.longdouble)
            lam = np.longdouble(rd.lam[b, k])
            ref_s = np.sum(d * (lam * d + bo[real].astype(np.longdouble)))
            bound = float(np.sum(np.abs(d) * (np.abs(lam * d) + np.abs(bo[real]))))
            if not np.isfinite(bound):
                continue
            e = abs(float(got[k, 4] - ref_s))
            _report(f"{build}/scale_rel", e / bound if bound > 0 else 0.0)
            assert e <= SCALE_BAR * bound + 1e-300, f"{build} band {b} trial {k}: scale {got[k, 4]} vs {float(ref_s)}"
        if np.isfinite(ref).all():
            yield b, got, ref


def check_zero_step(rd, build, k=0):
    """b. trial k has dx = 0: its chi2 per family is kernel A's"""
    for b in rd.bands():
        got, lin = rd.out["res"][b, k, :4], rd.out["chi_lin"][b]
        ulps = np.abs(got - lin) / np.spacing(np.maximum(np.abs(lin), np.finfo(float).tiny))
        _report(f"{build}/kernel_a_vs_eval_ulps", float(ulps.max()))
        assert (np.abs(got - lin) <= LIN_BAR * np.abs(lin)).all(), f"{build} band {b}: {got} vs kernel A {lin}"


def _ulps(a, b):
    if a == b:
        return 0.0
    return abs(a - b) / np.spacing(max(abs(a), abs(b)))


def check_decisions(rd, build, lam_ulps=2):
    """c. / d. the device's chain against teb_oracle_lm_decide, and the commit, band by band; lambda within lam_ulps.
    Returns {band: (decision, the committed trial carried a theta across the +-pi cut)}"""
    out, hb, st_in = rd.out, rd.hb, rd.state_in
    result = {}
    queued = set(int(b) for b in out["next_list"])
    assert len(queued) == out["next_list"].size
    active = set(rd.bands())
    for b in range(hb.B):
        if b not in active:   # untouched: poses, rows, state, no decision
            assert _same_bits(rd.after.poses[b], hb.poses[b]), f"{build}: band {b} (not in the round) moved"
            assert (_bits(out["res"][b]) == ALL_ONES).all()
            assert out["need"][b] == -1 and b not in queued
            continue
        n, q0, kact = int(hb.n[b]), rd.q0(b), rd.kact(b)
        rows = out["res"][b, :kact]
        assert (_bits(out["res"][b, kact:]) == ALL_ONES).all(), f"{build}: rows past kact written"
        tchi = [((r[0] + r[1]) + r[2]) + r[3] for r in rows]
        if rd.retry:
            cur, lam0, nu0 = st_in[b, 2], st_in[b, 0], st_in[b, 1]
            cur_parts = st_in[b, 3:7]
        else:
            cl = out["chi_lin"][b]
            cur, cur_parts = ((cl[0] + cl[1]) + cl[2]) + cl[3], cl
            # iteration 0: computeLambdaInit, 1e-5 max |H_rr| over the real rows of kernel A's system
            lam0, nu0 = ((1e-5 * R.max_real_diag(rd.Hb[b:b + 1], hb.n[b:b + 1])[0], 2.0) if rd.iteration == 0
                         else (st_in[b, 0], st_in[b, 1]))
        d = O.lm_decide(cur, lam0, nu0, q0, tchi, rows[:, 4], rd.ok[b, :kact] != 0)
        st = out["state"][b]
        assert out["qmax"][b] == d["q"], f"{build} band {b}: trials {out['qmax'][b]} vs {d}"
        assert out["need"][b] == int(d["need"]) and (b in queued) == d["need"]
        status = int(st_in[b, 11]) | d["status"]
        if not d["need"]:
            status = (status | TERMINATED) if d["terminate"] else (status & ~TERMINATED)
        assert int(st[11]) == status, f"{build} band {b}: status {int(st[11])} vs {status} ({d})"
        assert st[12] == (0 if (d["terminate"] and not d["need"]) else 1)
        assert st[13] == st_in[b, 13] + (0 if d["need"] else 1)
        assert st[1] == d["nu"] and st[2] == d["current_chi"]
        u = _ulps(st[0], d["lam"]) if np.isfinite(d["lam"]) else (0.0 if st[0] == d["lam"] else np.inf)
        _report(f"{build}/lambda_ulps", u)
        assert u <= lam_ulps, f"{build} band {b}: lambda {st[0]} vs {d['lam']}"
        acc = d["accepted"]
        want = rd.trial_state(b, acc) if acc >= 0 else hb.poses[b]
        assert _same_bits(rd.after.poses[b], want), f"{build} band {b}: committed state (trial {acc})"
        assert _same_bits(st[3:7], rows[acc, :4] if acc >= 0 else cur_parts)
        assert _same_bits(st[7:11], rows[d["used"] - 1, :4] if d["used"] else st_in[b, 7:11])
        wrapped = False
        if acc >= 0:
            raw = (hb.poses[b].ravel() + rd.step(b, acc))[2::4][_real(n, hb.n_cap)[:, 2]]
            wrapped = bool(((raw < -np.pi) | (raw >= np.pi)).any())
        result[b] = (d, wrapped)
    return result


def _steps(rd_hb, Hb, K, kind, rng):
    """trial steps [B][K][4 n_cap] of one kind (real rows only; fixed rows 0)"""
    B, n_cap = rd_hb.B, rd_hb.n_cap
    dx = np.zeros((B, K, 4 * n_cap))
    for b in range(B):
        n = int(rd_hb.n[b])
        real = _real(n, n_cap).ravel()
        rec = rd_hb.poses[b].ravel()
        mag = np.where(np.arange(4 * n_cap) % 4 == 2, np.pi, np.maximum(np.abs(rec), 0.1))
        for k in range(K):
            if kind == "random":      # 0, then 1e-8 .. 1e-1 of the magnitudes
                s = 0.0 if k == 0 else 10.0 ** (-8 + 7 * (k - 1) / max(K - 2, 1))
                dx[b, k] = s * mag * rng.standard_normal(4 * n_cap)
            elif kind == "wrap":      # theta of every free pose across +-pi, by 1e-9 .. 0.5 beyond
                th = np.arange(4 * n_cap) % 4 == 2
                sgn = np.where(rec[th] >= 0, 1.0, -1.0)
                dx[b, k, th] = sgn * (np.pi - np.abs(rec[th])) + sgn * 10.0 ** (-9 + 8.7 * k / max(K - 1, 1))
            elif kind == "dt":        # dt_i to exactly 0 (trial 1) and below (trial 2); small steps elsewhere
                dx[b, k] = 1e-4 * mag * rng.standard_normal(4 * n_cap)
                i = 1 + (k + b) % max(n - 2, 1)
                if k == 1:
                    dx[b, k, 4 * i + 3] = -rec[4 * i + 3]
                elif k == 2:
                    dx[b, k, 4 * i + 3] = -1.5 * rec[4 * i + 3]
            dx[b, k, ~real] = 0.0
    return dx


# ------------------------------------------------------------------ a. b. c. d. every scenario
@pytest.mark.parametrize("name", scenarios.ALL)
def test_trials_of_every_scenario_against_oracle(name):
    p, hb = scenarios.scenario(name)
    g = _ctx(hb, p)
    rng = np.random.default_rng(len(name))
    try:
        for outer in (0, 3):
            Hb, _ = g.build_system(hb, outer)
            n = hb.n.copy()
            # real LM steps, iteration 0 (lambda from kernel A), then later iterations from 1e-5 max diag upwards
            for K in (2, 8):
                dx, ok, lam = g.solve_system(n, K, n_cap=hb.n_cap)
                rd = Round(g, p, hb, K, dx, ok, lam, _state(hb.B), outer, iteration=0)
                list(check_chi2(rd, "eval2"))
                check_decisions(rd, "eval2")
            base = 1e-5 * R.max_real_diag(Hb, n)
            for mult in (1.0, 1e3):
                lam0 = base * mult
                dx, ok, lam = g.solve_system(n, 6, Hb=Hb, lam=lam0, nu=np.full(hb.B, 2.0))
                st = _state(hb.B, lam=lam0, nu=2.0)
                rd = Round(g, p, hb, 6, dx, ok, lam, st, outer, iteration=2)
                list(check_chi2(rd, "eval2"))
                check_decisions(rd, "eval2")
            lam = np.broadcast_to(base[:, None], (hb.B, 8))
            for kind in ("random", "wrap", "dt"):
                dx = _steps(hb, Hb, 8, kind, rng)
                rd = Round(g, p, hb, 8, dx, 1.0, lam, _state(hb.B, lam=base), outer, iteration=3)
                list(check_chi2(rd, "eval2"))
                check_decisions(rd, "eval2")
                if kind == "random":
                    check_zero_step(rd, "eval2")
    finally:
        g.close()


def _turned(hb):
    """the scene turned by pi about the origin: the bands run west, so their headings lie around the +-pi cut"""
    h = hb.copy()
    nt = O.lib().teb_oracle_normalize_theta
    for b in range(h.B):
        n = int(h.n[b])
        h.poses[b, :n, :2] *= -1.0
        h.poses[b, :n, 2] = [nt(float(t) + np.pi) for t in h.poses[b, :n, 2]]
    for f in ("x", "y", "vx", "vy"):
        h.obstacles[f] *= -1.0
    if h.PV_cap:
        h.obst_vertices *= -1.0
    if h.V_cap:
        h.via *= -1.0
    return h


@pytest.mark.parametrize("name", ["C2", "C3", "C4", "holonomic", "shapes_polygon"])
def test_commits_across_the_theta_cut(name):
    """d. west-going bands: accepted real LM steps carry headings across +-pi, and the committed state is
    x [+] dx with normalize_theta bit for bit; at least one accepted commit must have crossed the cut"""
    p, hb0 = scenarios.scenario(name)
    hb = _turned(hb0)
    g = _ctx(hb, p)
    crossed = 0
    try:
        for outer in (0, 2):
            Hb, _ = g.build_system(hb, outer)
            dx, ok, lam = g.solve_system(hb.n.copy(), 8, n_cap=hb.n_cap)
            rd = Round(g, p, hb, 8, dx, ok, lam, _state(hb.B), outer, iteration=0)
            list(check_chi2(rd, "eval2"))
            crossed += sum(w for _, w in check_decisions(rd, "eval2").values())
            base = 1e-5 * R.max_real_diag(Hb, hb.n)
            dx, ok, lam = g.solve_system(hb.n.copy(), 4, Hb=Hb, lam=base, nu=np.full(hb.B, 2.0))
            rd = Round(g, p, hb, 4, dx, ok, lam, _state(hb.B, lam=base), outer, iteration=1)
            list(check_chi2(rd, "eval2"))
            crossed += sum(w for _, w in check_decisions(rd, "eval2").values())
    finally:
        g.close()
    _report(f"theta_cut_commits/{name}", crossed)
    assert crossed >= 1, f"{name}: no accepted commit carried a heading across +-pi"


def test_decisions_with_oracle_chi2_agree_outside_ties():
    """c. second pass: teb_oracle_lm_decide fed the oracle's chi2 makes the device's decisions, except where
    |currentChi - tempChi| is within the chi2 bar"""
    ties = 0
    total = 0
    for name in ("C2", "C3", "C4", "all_edge_families", "vor", "holonomic"):
        p, hb = scenarios.scenario(name)
        g = _ctx(hb, p)
        try:
            for outer in (0, 3):
                dx, ok, lam = g.solve_system(hb.n.copy(), 8, n_cap=g.build_system(hb, outer)[0].shape[1] // 4)
                rd = Round(g, p, hb, 8, dx, ok, lam, _state(hb.B), outer, iteration=0)
                for b, got, ref in check_chi2(rd, "eval2"):
                    n = int(hb.n[b])
                    cl = rd.out["chi_lin"][b]
                    cur = ((cl[0] + cl[1]) + cl[2]) + cl[3]
                    # the oracle's chi2 at the linearisation point and at every trial
                    lin = O.trial_chi2(p, hb.poses[b], n, hb.poses[b:b + 1, :n], weight_multiplier=2.0 ** outer,
                                       **scenarios.band_kwargs(hb, b))[0]
                    cur_ref = float(np.sum(lin, dtype=np.longdouble))
                    tdev = [((r[0] + r[1]) + r[2]) + r[3] for r in got]
                    tref = [float(np.sum(r, dtype=np.longdouble)) for r in ref]
                    a = O.lm_decide(cur, lam[b, 0], 2.0, 0, tdev, got[:, 4], ok[b] != 0)
                    o = O.lm_decide(cur_ref, lam[b, 0], 2.0, 0, tref, got[:, 4], ok[b] != 0)
                    total += 1
                    if (a["accepted"], a["q"], a["terminate"]) != (o["accepted"], o["q"], o["terminate"]):
                        used = tref[:max(a["used"], o["used"])]
                        near = any(abs(cur_ref - t) <= FAM_BAR * 4 * max(cur_ref, t) for t in used)
                        assert near, f"{name} band {b}: decisions differ outside a tie: {a} vs {o}"
                        ties += 1
        finally:
            g.close()
    _report("decision_ties_with_oracle_chi2", ties)
    _report("decision_bands_compared", total)


# ------------------------------------------------------------------ c. crafted rounds
def _craft_batch():
    return scenarios.scenario("C3")


def test_failed_factorisations_and_nan_trials():
    """ok = 0: the trial is x + b, tempChi = DBL_MAX, CHOL_FAILED; a NaN in a trial step: NaN chi2 ends the iteration
    without Terminate"""
    p, hb = _craft_batch()
    g = _ctx(hb, p)
    try:
        Hb, _ = g.build_system(hb, 1)
        base = 1e-5 * R.max_real_diag(Hb, hb.n)
        dx, ok, lam = g.solve_system(hb.n.copy(), 4, Hb=Hb, lam=base, nu=np.full(hb.B, 2.0))
        ok = ok.copy()
        ok[0, :2] = 0      # band 0: two failed factorisations, then real steps
        ok[1, :] = 0       # band 1: all failed
        dx = dx.copy()
        dx[2, 0, 4 * 2] = np.nan   # band 2: NaN in trial 0
        rd = Round(g, p, hb, 4, dx, ok, lam, _state(hb.B, lam=base), 1, iteration=1)
        list(check_chi2(rd, "eval2"))
        check_decisions(rd, "eval2")
        assert int(rd.out["state"][0, 11]) & abi.TEB_STATUS_CHOL_FAILED
        assert rd.out["need"][1] == 1 and rd.out["qmax"][1] == 4
        assert np.isnan(rd.out["res"][2, 0, :4]).any() and rd.out["qmax"][2] == 1 and rd.out["need"][2] == 0
        assert not int(rd.out["state"][2, 11]) & TERMINATED and rd.out["state"][2, 12] == 1
    finally:
        g.close()


def test_lambda_overflow_and_retry_rounds_at_the_trial_cap():
    """lambda near DBL_MAX: NONFINITE and Terminate; retry rounds starting at trial 4, 6, 8, 9 consume at most 10 - q0
    trials and the rows of the rest stay all-ones; a band that rejects every trial terminates at the tenth rejection,
    or is queued again when the round ends before it (K = 4 from trial 4)"""
    p, hb = _craft_batch()
    g = _ctx(hb, p)
    try:
        Hb, _ = g.build_system(hb, 0)
        B = hb.B
        dx, ok, lam = g.solve_system(hb.n.copy(), 8, n_cap=hb.n_cap)
        lin = g.eval_trials(hb.copy(), 2, dx[:, :2], ok[:, :2], lam[:, :2], _state(B), iteration=0)["chi_lin"]
        cur = np.array([((c[0] + c[1]) + c[2]) + c[3] for c in lin])
        st = _state(B, lam=DBL_MAX / 3, nu=2.0, chi=cur, parts_cur=lin)
        rd = Round(g, p, hb, 4, dx[:, :4], 0.0, lam[:, :4], st, 0, iteration=1)
        check_decisions(rd, "eval2")
        assert (rd.out["state"][:, 11].astype(int) & abi.TEB_STATUS_NONFINITE).all()
        assert (rd.out["state"][:, 12] == 0).all()
        for K in (4, 8):
            for q0 in (4, 6, 8, 9):
                qmax = np.full(B, q0, np.int32)
                order = np.arange(B)[::-1].copy()
                lam0 = np.array([R.spec_lambda(1e-5 * R.max_real_diag(Hb, hb.n)[b], 2.0, q0) for b in range(B)])
                st = _state(B, lam=lam0, nu=2.0 ** (q0 + 1), chi=cur, parts_cur=lin)
                # trials that make chi2 worse, so that the chain runs to the cap
                bad = dx[:, :K] * 50.0
                rd = Round(g, p, hb, K, bad, 1.0, lam[:, :K], st, 0, iteration=1, qmax=qmax, order=order)
                list(check_chi2(rd, "eval2"))
                kact = min(K, 10 - q0)
                all_rejected = 0
                for b, (d, _) in check_decisions(rd, "eval2").items():
                    assert d["used"] <= kact and (_bits(rd.out["res"][b, kact:]) == ALL_ONES).all()
                    if d["accepted"] >= 0 or d["used"] < kact:
                        continue
                    all_rejected += 1   # every trial of the round rejected
                    st_out = rd.out["state"][b]
                    if q0 + K >= 10:    # the tenth rejection: Terminate, no further round
                        assert rd.out["qmax"][b] == 10 and rd.out["need"][b] == 0 and b not in rd.out["next_list"]
                        assert int(st_out[11]) & TERMINATED and st_out[12] == 0
                    else:               # queued for the next round with q0 + K trials used
                        assert rd.out["qmax"][b] == q0 + K and rd.out["need"][b] == 1 and b in rd.out["next_list"]
                        assert st_out[12] == 1
                assert all_rejected >= 1, f"K {K} q0 {q0}: no band rejected every trial of the round"
    finally:
        g.close()


def test_zero_chi2_band_terminates_after_one_trial():
    """a band whose every edge is inside its limits and far from the obstacles has chi2 exactly 0: dx = 0 gives
    rho == 0, which terminates after one trial"""
    p, hb = _craft_batch()
    p.weight_optimaltime = 0.0
    B, n_cap = hb.B, hb.n_cap
    hb.poses[:] = 0.0
    for b in range(B):
        n = int(hb.n[b])
        hb.poses[b, :n, 0] = 100.0 + 0.1 * np.arange(n)
        hb.poses[b, :n - 1, 3] = 0.5
    g = _ctx(hb, p)
    try:
        rd = Round(g, p, hb, 2, 0.0, 1.0, 1.0, _state(B), 0, iteration=0)
        assert (rd.out["chi_lin"] == 0).all()
        check_decisions(rd, "eval2")
        assert (rd.out["qmax"] == 1).all() and (rd.out["state"][:, 12] == 0).all()
        assert (rd.out["state"][:, 11].astype(int) & TERMINATED).all()
    finally:
        g.close()


# ------------------------------------------------------------------ d. hygiene
def test_nan_past_n_and_inactive_bands_change_nothing():
    p, hb = scenarios.scenario("C4")
    hb2 = abi.HostBatch(np.concatenate([hb.poses, np.zeros((hb.B, 7, 4))], axis=1), hb.n.copy(), hb.obstacles, hb.obst_count,
                        hb.scene_id, hb.via, hb.via_count, hb.vel_start, hb.vel_goal, hb.prefer_rotdir)
    g = _ctx(hb2, p)
    try:
        dx, ok, lam = g.solve_system(hb2.n.copy(), 6, n_cap=g.build_system(hb2, 1)[0].shape[1] // 4)
        act = np.ones(hb2.B)
        act[1] = 0
        st = _state(hb2.B, active=act)
        zero = Round(g, p, hb2, 6, dx, ok, lam, st, 1, iteration=0)
        check_decisions(zero, "eval2")
        nanb = hb2.copy()
        dxn = dx.copy()
        for b in range(hb2.B):
            nanb.poses[b, hb2.n[b]:] = np.nan
            dxn[b, :, 4 * hb2.n[b]:] = np.nan
        rd = Round(g, p, nanb, 6, dxn, ok, lam, st, 1, iteration=0)
        check_decisions(rd, "eval2")
        for key in ("res", "chi_lin", "state", "qmax", "need"):
            assert _same_bits(rd.out[key], zero.out[key]) if rd.out[key].dtype == np.float64 else \
                np.array_equal(rd.out[key], zero.out[key]), key
        for b in range(hb2.B):
            n = hb2.n[b]
            assert _same_bits(rd.after.poses[b, :n], zero.after.poses[b, :n])
            assert np.isnan(rd.after.poses[b, n:]).all()
    finally:
        g.close()


# ------------------------------------------------------------------ e. shapes
SHAPE_N = [3, 4, 29, 30, 31, 59, 60, 61, 119, 120, 121, 239, 240, 241, 269, 270, 271, 479, 480, 481, 510, 511, 512]


def _band_batch(ns, n_cap, seed=0, name="C3"):
    p = scenes.config_params(name)
    p.teb_autosize = 0
    B = len(ns)
    poses = np.zeros((B, n_cap, 4))
    for b, n in enumerate(ns):
        L = 0.4 * 0.3 * (n - 1)
        poses[b, :n] = scenes.make_band(n, np.random.default_rng(seed + b).uniform(-1.0, 1.0), 0.4, 0.3, length=max(L, 0.5))
    rng = np.random.default_rng(seed)
    Lmax = 0.4 * 0.3 * (max(ns) - 1)
    ob = scenes.make_obstacles(rng, 24, max(Lmax, 1.0), inflated=True, moving=True)[None]
    return p, abi.HostBatch(poses, np.array(ns, np.int32), ob, np.array([24], np.int32), np.zeros(B, np.int32))


@pytest.mark.parametrize("cap", ["n", "padded"])
def test_shapes_around_every_tile_edge(cap):
    """n at every 29 / 30-pose tile edge, 3 .. 512, with n_cap = n (one batch per n) or n_cap = 512 (one ragged batch)"""
    groups = [[n, max(n - 1, 3)] for n in SHAPE_N] if cap == "n" else [SHAPE_N]
    for gi, ns in enumerate(groups):
        n_cap = max(ns) if cap == "n" else 512
        K = (2, 4, 6, 8)[gi % 4]
        p, hb = _band_batch(ns, n_cap, seed=gi)
        g = _ctx(hb, p)
        try:
            Hb, _ = g.build_system(hb, 0)
            dx, ok, lam = g.solve_system(hb.n.copy(), K, n_cap=n_cap)
            rd = Round(g, p, hb, K, dx, ok, lam, _state(hb.B), 0, iteration=0)
            list(check_chi2(rd, "eval2"))
            check_decisions(rd, "eval2")
            dz = _steps(hb, Hb, K, "random", np.random.default_rng(gi))
            base = 1e-5 * R.max_real_diag(Hb, hb.n)
            rd = Round(g, p, hb, K, dz, 1.0, base[:, None], _state(hb.B, lam=base), 0, iteration=1)
            list(check_chi2(rd, "eval2"))
            check_zero_step(rd, "eval2")
            check_decisions(rd, "eval2")
        finally:
            g.close()


# ------------------------------------------------------------------ f. builds agree
def _placement_case(name):
    p, hb = scenarios.scenario(name, candidates=6)
    g = _ctx(hb, p)
    try:
        Hb, _ = g.build_system(hb, 1)
        dx, ok, lam = g.solve_system(hb.n.copy(), 8, n_cap=hb.n_cap)
    finally:
        g.close()
    return p, hb, Hb, dx, ok, lam


def _embed(hb, B, pos, filler_seed=0):
    """hb's bands at positions pos of a B-band batch, copies of them everywhere else"""
    rng = np.random.default_rng(filler_seed)
    src = rng.integers(0, hb.B, B)
    src[pos] = np.arange(hb.B)
    sel = lambda a: None if a is None else a[src].copy()
    out = abi.HostBatch(hb.poses[src].copy(), hb.n[src].copy(), hb.obstacles, hb.obst_count, hb.scene_id[src].copy(),
                        sel(hb.via) if hb.V_cap else None, sel(hb.via_count) if hb.V_cap else None, hb.vel_start[src].copy(),
                        hb.vel_goal[src].copy(), hb.prefer_rotdir[src].copy(), hb.obst_vertices if hb.PV_cap else None)
    return out, src


def _build_name(build, B, sms):
    """the launch launch_trial_eval picks for this build and batch size (TebGpu.last_trial_eval's names)"""
    if build != "eval2":
        return build
    return "eval2_wide" if 2 * B <= sms else ("eval2" if B <= 2 * sms else "eval2p")


def _run_placed(p, hb, dx, ok, lam, build, B, pos, K, sms, retry_q0=None, order_seed=0):
    """hb's bands at positions pos among B - hb.B active neighbours with trials of their own (their sources' steps,
    scaled); a retry round lists every band in a random order"""
    big, src = _embed(hb, B, pos, filler_seed=B)
    scale = np.random.default_rng(B + 1).uniform(0.5, 1.5, B)
    scale[pos] = 1.0
    g = _ctx(big, p, build, max_bands=B)
    try:
        Hb, _ = g.build_system(big, 1)
        base = 1e-5 * R.max_real_diag(Hb, big.n)
        st = _state(B, lam=base)
        qmax = order = None
        if retry_q0 is not None:
            qmax = np.full(B, retry_q0, np.int32)
            order = np.random.default_rng(order_seed).permutation(B).astype(np.int32)
        rd = Round(g, p, big, K, dx[src][:, :K] * scale[:, None, None], ok[src][:, :K], lam[src][:, :K], st, 1,
                   iteration=1, qmax=qmax, order=order)
        name, grid = g.last_trial_eval()
        assert name == _build_name(build, B, sms), (build, B, name)
        if name == "eval2p":
            _report(f"eval2p_grid/B{B}", grid)
        list(check_chi2(rd, name, bands=pos))
        check_decisions(rd, name)
    finally:
        g.close()
    return rd


@pytest.mark.parametrize("name", ["C2", "shapes_polygon", "holonomic", "vor"])
def test_every_build_gives_the_same_bits_wherever_the_band_sits(name):
    """k_trial_eval2 wide (2B <= SMs), k_trial_eval2 (B <= 2 SMs), k_trial_eval2p (above; the build each run took is
    read from the context) and k_trial_eval3: rows, decisions, state and poses bit-identical, at any batch position
    among active neighbours with other trials, in round 0 and at any position of a retry list that holds every band.
    At these sizes k_trial_eval2p's CTAs mostly take one slot each: tests/test_gpu_trial_eval_persistent.py runs it
    at several slots per CTA"""
    sms = _sms()
    p, hb, _, dx, ok, lam = _placement_case(name)
    nb = hb.B
    ref = {}
    runs = [("eval2", nb, None), ("eval2", 2 * sms, None), ("eval2", 2 * sms + 40, None), ("eval3", nb, None),
            ("eval3", sms, None), ("eval2", 2 * sms + 40, 4), ("eval2", nb, 4), ("eval3", sms, 4)]
    assert 2 * nb <= sms
    for i, (build, B, q0) in enumerate(runs):
        pos = np.sort(np.random.default_rng(i).choice(B, nb, replace=False))
        rd = _run_placed(p, hb, dx, ok, lam, build, B, pos, 8, sms, retry_q0=q0, order_seed=i)
        got = (rd.out["res"][pos], rd.out["state"][pos], rd.after.poses[pos], rd.out["qmax"][pos], rd.out["need"][pos])
        if q0 not in ref:   # round 0 and the retry round from trial 4 each have their reference
            ref[q0] = got
            continue
        for a, b2, what in zip(got, ref[q0], ("rows", "state", "poses", "qmax", "need")):
            assert _same_bits(a, b2) if a.dtype == np.float64 else np.array_equal(a, b2), f"{build} B {B}: {what} differ"


def test_global_table_builds_match_the_staged_builds():
    """a scene padded past 1024 rows (far points) runs the global-table k_trial_eval2 / k_trial_eval3: the bits of the
    staged run"""
    p, hb, _, dx, ok, lam = _placement_case("C3")
    M_cap = 1100
    ob = np.zeros((hb.S, M_cap), abi.OBST_DTYPE)
    ob["x"], ob["y"] = 1000.0, 1000.0
    for s in range(hb.S):
        ob[s, :hb.obst_count[s]] = hb.obstacles[s, :hb.obst_count[s]]
    big = abi.HostBatch(hb.poses.copy(), hb.n.copy(), ob, np.full(hb.S, M_cap, np.int32), hb.scene_id.copy(), None, None,
                        hb.vel_start.copy(), hb.vel_goal.copy(), hb.prefer_rotdir.copy())
    outs = {}
    for build in ("eval2", "eval3"):
        for nm, h in (("staged", hb), ("gt", big)):
            g = _ctx(h, p, build, max_obstacles=max(h.M_cap, 1))
            try:
                Hb, _ = g.build_system(h, 1)
                base = 1e-5 * R.max_real_diag(Hb, h.n)
                rd = Round(g, p, h, 8, dx, ok, lam, _state(h.B, lam=base), 1, iteration=1)
                if nm == "gt":
                    list(check_chi2(rd, f"{build}_gt"))
                    check_decisions(rd, f"{build}_gt")
                outs[build, nm] = (rd.out["res"], rd.out["state"], rd.after.poses)
            finally:
                g.close()
    for build in ("eval2", "eval3"):
        for a, b in zip(outs[build, "gt"], outs[build, "staged"]):
            assert _same_bits(a, b), build
        for a, b in zip(outs[build, "gt"], outs["eval2", "staged"]):
            assert _same_bits(a, b), build


@pytest.mark.parametrize("name", ["C2", "C4", "shapes_two_circles"])
def test_first_generation_kernel_agrees(name):
    """k_trial_eval (warp per trial, chunk per lane: another summation order) against the oracle and within 1e-13 of
    k_trial_eval2, with the same decisions outside ties"""
    p, hb, Hb, dx, ok, lam = _placement_case(name)
    outs = {}
    for build in ("v1", "eval2"):
        g = _ctx(hb, p, build)
        try:
            base = 1e-5 * R.max_real_diag(Hb, hb.n)
            rd = Round(g, p, hb, 8, dx, ok, lam, _state(hb.B, lam=base), 1, iteration=1)
            list(check_chi2(rd, build))
            check_decisions(rd, build)
            outs[build] = rd
        finally:
            g.close()
    a, b = outs["v1"].out["res"], outs["eval2"].out["res"]
    fin = np.isfinite(b)
    rel = np.abs(a[fin] - b[fin]) / np.maximum(np.abs(b[fin]), 1e-300)
    _report("v1_vs_eval2_rel", float(rel.max(initial=0.0)))
    assert (rel <= 1e-13).all()
    assert np.array_equal(outs["v1"].out["qmax"], outs["eval2"].out["qmax"]), "k_trial_eval and k_trial_eval2 decide differently"
