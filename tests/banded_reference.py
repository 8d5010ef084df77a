"""Plain extended-precision reference of the LM step's linear solve, CPU only (numpy).

The device solvers take the padded banded layout of kernel A: Hb[r] = (H[r][r-k] for k = 0 .. 10, b[r]), unknown
r = 4i + c is pose i (c = 0, 1, 2) or dt_i (c = 3), and they solve (H + lambda I_real) x = b, where I_real has ones
only on the real rows: rows 0 .. 2 (the fixed start pose) and the last four (the fixed goal pose, the non-existent
dt_{n-1}) are identity rows and take no lambda. This module restates that operation:

  * ldl_solve: banded LDL^T (half bandwidth 10) in np.longdouble, vectorised over systems;
  * residual / backward_error: b - A x of a double solution in longdouble, and the a-posteriori normwise bound
        ||b - A x||inf / (|| |L| |D| |L^T| ||inf ||x||inf + ||b||inf),
    which holds for any diagonal scaling of the system (obstacle rows grow with weight_adapt_factor^outer, the others
    stay near 1);
  * synthetic_systems: H = J^T W J from random edges with the widest real stencil (poses i .. i+2, dt_i, dt_{i+1})
    and weights spread over 1e-6 .. 1e6, right-hand side J^T W e;
  * make_indefinite: H minus a clearly negative rank-1 term on a narrow row window. By Sylvester's law of inertia every
    elimination order then meets a non-positive pivot, so every solver mapping must report the failure.
"""
import numpy as np

HB = 10                      # half bandwidth
U = 2.0 ** -53               # unit roundoff of double
LD = np.longdouble


def row_is_real(r, n):
    """teb_kernels.cuh row_is_real: rows of the free unknowns (numpy broadcasting over r and n)"""
    r = np.asarray(r)
    i, c = r >> 2, r & 3
    return np.where(c == 3, i <= n - 2, (i >= 1) & (i <= n - 2))


def _band(Hb, n, lam, dtype):
    """[S][N_max + HB][11] lower band of H + lambda I_real and [S][N_max + HB] rhs; identity rows from N on (what is
    stored there is never read, as on the device)"""
    Hb = np.asarray(Hb)
    n = np.asarray(n, dtype=np.int64)
    S = Hb.shape[0]
    Nmax = int(4 * n.max())
    r = np.arange(Nmax)
    live = r[None, :] < 4 * n[:, None]
    A = np.zeros((S, Nmax + HB, 11), dtype=dtype)
    y = np.zeros((S, Nmax + HB), dtype=dtype)
    A[:, :Nmax] = np.where(live[:, :, None], Hb[:, :Nmax, :11], 0).astype(dtype)
    y[:, :Nmax] = np.where(live, Hb[:, :Nmax, 11], 0).astype(dtype)
    A[:, Nmax:, 0] = 1
    A[:, :Nmax, 0] = np.where(live, A[:, :Nmax, 0], 1)
    real = live & row_is_real(r[None, :], n[:, None])
    A[:, :Nmax, 0] += np.where(real, np.asarray(lam, dtype=dtype).reshape(S, 1), 0)
    # entries that would reach above row 0
    for k in range(1, 11):
        A[:, :k, k] = 0
    return A, y, Nmax


def ldl_factor(Hb, n, lam, dtype=LD):
    """Right-looking banded LDL^T of H + lambda I_real, no pivoting. Returns (L, d, z, ok, Nmax): L[s][r][u] =
    L[r][r-u] (u = 1 .. 10), d the pivots, z = D^-1 L^-1 b, ok = every pivot positive and finite."""
    A, y, Nmax = _band(Hb, n, lam, dtype)
    S = A.shape[0]
    d = np.zeros((S, Nmax), dtype=dtype)
    ok = np.ones(S, dtype=bool)
    with np.errstate(all="ignore"):
        for j in range(Nmax):
            dj = A[:, j, 0].copy()
            ok &= (dj > 0) & np.isfinite(dj)
            d[:, j] = dj
            c = np.stack([A[:, j + u, u] for u in range(1, 11)], axis=1)   # column j below the diagonal: c_1 .. c_10
            lcol = c / dj[:, None]
            for u in range(1, 11):
                # A[j+u][j+q] -= l_u c_q for q = 1 .. u  ->  band offsets k = u - q = u-1 .. 0
                A[:, j + u, 0:u] -= lcol[:, u - 1:u] * c[:, u - 1::-1][:, :u]
                y[:, j + u] -= lcol[:, u - 1] * y[:, j]
                A[:, j + u, u] = lcol[:, u - 1]
        z = y[:, :Nmax] / d
    L = A
    return L, d, z, ok, Nmax


def ldl_solve(Hb, n, lam, dtype=LD):
    """x [S][N_max] (zero past each system's N) and ok [S]"""
    L, d, z, ok, Nmax = ldl_factor(Hb, n, lam, dtype)
    S = z.shape[0]
    x = np.zeros((S, Nmax + HB), dtype=dtype)
    u = np.arange(1, 11)
    with np.errstate(all="ignore"):
        for j in range(Nmax - 1, -1, -1):
            x[:, j] = z[:, j] - (L[:, j + u, u] * x[:, j + u]).sum(axis=1)
    x = x[:, :Nmax]
    live = np.arange(Nmax)[None, :] < 4 * np.asarray(n)[:, None]
    return np.where(live, x, 0), ok


def band_matvec(Hb, n, lam, x, dtype=LD):
    """(H + lambda I_real) x in `dtype`, x [S][>= N_max]; rows past N are zero"""
    A, y, Nmax = _band(Hb, n, lam, dtype)
    live = np.arange(Nmax)[None, :] < 4 * np.asarray(n)[:, None]
    x = np.where(live, np.asarray(x)[:, :Nmax], 0).astype(dtype)     # what lies past N (a NaN pattern) is not read
    xp =np.concatenate([np.zeros((x.shape[0], HB), dtype=dtype), x], axis=1)   # xp[:, r + HB] = x[r]
    out = A[:, :Nmax, 0] * x
    for k in range(1, 11):
        out += A[:, :Nmax, k] * xp[:, HB - k:HB - k + Nmax]                    # lower part: H[r][r-k] x[r-k]
        out[:, :Nmax - k] += A[:, k:Nmax, k] * x[:, k:]                         # upper part: H[r-k][r] = H[r][r-k]
    return np.where(live, out, 0), np.where(live, y[:, :Nmax], 0)


def residual(Hb, n, lam, x):
    """b - (H + lambda I_real) x in longdouble"""
    Ax, b = band_matvec(Hb, n, lam, x)
    return b - Ax


def ldl_norm(Hb, n, lam):
    """|| |L||D||L^T| ||inf per system, L D L^T the longdouble factor of H + lambda I_real. All of |L||D||L^T| is
    non-negative, so its inf-norm is the largest entry of |L| |D| |L^T| 1."""
    L, d, _, ok, Nmax = ldl_factor(Hb, n, lam)
    S = d.shape[0]
    live = np.arange(Nmax)[None, :] < 4 * np.asarray(n)[:, None]
    aL = np.abs(L[:, :Nmax + HB])
    u = np.arange(1, 11)
    # v = |L^T| 1: column sums of |L|, v_j = 1 + sum_u |L[j+u][j]|
    v = np.ones((S, Nmax), dtype=LD)
    for j in range(Nmax):
        v[:, j] += aL[:, j + u, u].sum(axis=1)
    w = np.abs(d) * np.where(live, v, 0)
    wp = np.concatenate([np.zeros((S, HB), dtype=LD), w], axis=1)
    m = w.copy()
    for k in range(1, 11):
        m += aL[:, :Nmax, k] * wp[:, HB - k:HB - k + Nmax]
    return np.where(live, m, 0).max(axis=1)


def backward_error(Hb, n, lam, x, norm=None):
    """||b - A x||inf / (|| |L||D||L^T| ||inf ||x||inf + ||b||inf) per system, A = H + lambda I_real (norm: the
    ldl_norm of these systems, if already known)"""
    if norm is None:
        norm = ldl_norm(Hb, n, lam)
    r = residual(Hb, n, lam, x)
    S, Nmax = r.shape
    _, b = band_matvec(Hb, n, lam, np.zeros((S, Nmax)))
    live = np.arange(Nmax)[None, :] < 4 * np.asarray(n)[:, None]
    xn = np.abs(np.where(live, np.asarray(x)[:, :Nmax], 0)).max(axis=1).astype(LD)
    den = norm * xn + np.abs(b).max(axis=1)
    return (np.abs(r).max(axis=1) / den).astype(np.float64)


def dense(Hb_band, n, lam):
    """dense float64 A = H + lambda I_real and b of one band (for condition numbers)"""
    N = 4 * int(n)
    A = np.zeros((N, N))
    for k in range(11):
        r = np.arange(k, N)
        A[r, r - k] = Hb_band[k:N, k]
        A[r - k, r] = Hb_band[k:N, k]
    real = row_is_real(np.arange(N), int(n))
    A[np.arange(N), np.arange(N)] += np.where(real, lam, 0.0)
    return A, Hb_band[:N, 11].copy()


def max_real_diag(Hb, n):
    """max |H_rr| over the real rows of each band: computeLambdaInit's tau is applied to this"""
    n = np.asarray(n)
    r = np.arange(Hb.shape[1])
    real = row_is_real(r[None, :], n[:, None]) & (r[None, :] < 4 * n[:, None])
    return np.where(real, np.abs(Hb[:, :, 0]), 0).max(axis=1)


def spec_lambda(lam, nu, k):
    """lambda of trial k after k rejections (teb_spec.cuh spec_lambda), in double like the device"""
    lam, nu = float(lam), float(nu)
    for _ in range(k):
        lam *= nu
        nu *= 2
    return lam


def synthetic_systems(rng, n, n_cap, w_lo=1e-6, w_hi=1e6, edges_per_anchor=2, rows_per_edge=3):
    """Hb [S][4 n_cap][12] of H = J^T W J, b = J^T W e for bands of n[s] poses. Every edge couples the widest real
    stencil, the 11 unknowns 4i .. 4i+10 (poses i .. i+2, dt_i, dt_{i+1}); its weight is log-uniform in
    [w_lo, w_hi]. Identity rows as kernel A writes them: H_rr = 1, no coupling, b_r = 0."""
    n = np.asarray(n, dtype=np.int64)
    S = n.size
    Hb = np.zeros((S, 4 * n_cap, 12))
    for s in range(S):
        N = 4 * int(n[s])
        real = row_is_real(np.arange(N), int(n[s]))
        H = np.zeros((N, N))
        g = np.zeros(N)
        for i in range(int(n[s]) - 2):
            cols = np.arange(4 * i, 4 * i + 11)
            for _ in range(edges_per_anchor):
                J = rng.normal(size=(rows_per_edge, 11)) * real[cols]
                w = np.exp(rng.uniform(np.log(w_lo), np.log(w_hi)))
                e = rng.normal(size=rows_per_edge)
                H[np.ix_(cols, cols)] += w * (J.T @ J)
                g[cols] += w * (J.T @ e)
        H[~real, :] = 0
        H[:, ~real] = 0
        H[~real, ~real] = 1.0
        g[~real] = 0
        for k in range(11):
            r = np.arange(k, N)
            Hb[s, r, k] = H[r, r - k]
        Hb[s, :N, 11] = g
    return Hb


def make_indefinite(Hb, n, lam, rows, rng, width=4):
    """Copy of the bands with a clearly negative rank-1 term: A - alpha v v^T, v a unit vector on `width` real rows
    starting at rows[s] (clipped into the real rows), alpha = 2 v^T A v + 1 with A = H + lambda I_real, so that
    v^T (A - alpha v v^T) v < 0. width <= 8 keeps v v^T inside the solver's profile."""
    Hb = np.array(Hb, copy=True)
    n = np.asarray(n)
    lam = np.broadcast_to(np.asarray(lam, dtype=np.float64), n.shape)
    for s in range(n.size):
        N = 4 * int(n[s])
        r0 = int(min(max(rows[s], 3), N - 4 - width))
        idx = np.arange(r0, r0 + width)
        assert row_is_real(idx, int(n[s])).all()
        v = rng.normal(size=width)
        v /= np.linalg.norm(v)
        A, _ = dense(Hb[s], n[s], lam[s])
        alpha = 2.0 * float(v @ A[np.ix_(idx, idx)] @ v) + 1.0
        for a in range(width):
            for c in range(a + 1):
                Hb[s, idx[a], a - c] -= alpha * v[a] * v[c]
    return Hb
