"""TEST-ONLY numpy/scipy statement of TrajSolver in its block-tridiagonal form.

The cost of segment i in the derivatives at its end waypoints is tau^(1-2h) S Hbar S (S = diag(tau^k),
h = N/2), so the system in all waypoint derivatives is banded with lower bandwidth 2h - 1.  Fixed
derivatives get a unit row and column; scipy's solveh_banded solves the rest.  Each segment's coefficients
then come from its own 2h x 2h end-point system.  It needs no dense (S N) x (S N) matrix, so it checks
paths far longer than the host's dense restatement can solve.
"""
from math import factorial

import numpy as np
from scipy.linalg import solveh_banded

VEL, ACC, JRK = 0x01, 0x03, 0x07
ORDER = {0x01: 1, 0x11: 1, 0x03: 2, 0x13: 2, 0x07: 3, 0x17: 3}


def _hbar(h):
    N = 2 * h
    A = np.zeros((N, N))
    Q = np.zeros((N, N))
    for k in range(h):
        A[k, k] = factorial(k)
        for n in range(k, N):
            A[h + k, n] = factorial(n) / factorial(n - k)
    for r in range(h, N):
        for n in range(h, N):
            Q[r, n] = factorial(r) / factorial(r - h) * factorial(n) / factorial(n - h) / (r + n - 2 * h + 1)
    Ai = np.linalg.inv(A)
    return Ai.T @ Q @ Ai


HBAR = {h: np.round(_hbar(h)) for h in (1, 2, 3)}  # integer matrices


def seg_matrix(h, tau):
    S = np.diag([tau ** k for k in range(h)] * 2)
    return tau ** (1 - 2 * h) * S @ HBAR[h] @ S


def solve_derivatives(h, taus, fixed, vals):
    """fixed: (W, h) bool; vals: (W, h, nc).  Returns D (W, h, nc): the minimiser's derivatives at every
    waypoint (fixed ones as given; with two waypoints the free ones are 0, as the reference leaves them)."""
    W, nc = len(fixed), vals.shape[2]
    D = np.where(fixed[:, :, None], vals, 0.0)
    if W <= 2:
        return D
    n = W * h
    ab = np.zeros((2 * h, n))  # lower band: ab[i - j, j] = K[i, j]
    b = np.zeros((n, nc))
    fx = fixed.reshape(-1)
    fv = vals.reshape(n, nc)
    for i, tau in enumerate(taus):
        Hi = seg_matrix(h, tau)
        g = np.arange(i * h, i * h + 2 * h)
        for a in range(2 * h):
            for c in range(2 * h):
                r, s = g[a], g[c]
                if fx[s] and not fx[r]:
                    b[r] -= Hi[a, c] * fv[s]
                if r >= s and not fx[r] and not fx[s]:
                    ab[r - s, s] += Hi[a, c]
    for r in np.nonzero(fx)[0]:
        ab[0, r] = 1.0
        b[r] = fv[r]
    x = solveh_banded(ab, b, lower=True)
    return np.where(fixed[:, :, None], vals, x.reshape(W, h, nc))


def seg_coeff(h, tau, d0, d1):
    """Primitive1D coefficients (6, highest order first) of the degree-(2h-1) polynomial with derivatives d0 at
    0 and d1 at tau."""
    N = 2 * h
    A = np.zeros((N, N))
    for k in range(h):
        A[k, k] = factorial(k)
        for m in range(k, N):
            A[h + k, m] = factorial(m) / factorial(m - k) * tau ** (m - k)
    p = np.linalg.solve(A, np.concatenate([d0, d1]))
    c = np.zeros(6)
    for k in range(N):
        c[5 - k] = p[k] * factorial(k)
    return c


def traj_solve(dim, control, pos=None, waypoints=None, wp_control=None, dts=None, v=1.0, yaw_control=VEL):
    """What TrajSolver<dim>(control, yaw_control) gives for one path (arguments as planner.run_traj_solve):
    dict(status, seg_t, coeff (S, dim + 1, 6))."""
    h, hy = ORDER[control], ORDER[yaw_control]
    if waypoints is None:
        p = np.asarray(pos, dtype=np.float64).reshape(-1, dim)
        W = len(p)
        vals = np.zeros((W, 3, dim))
        vals[:, 0] = p
        yaw = np.zeros(W)
        ctl = np.full(W, VEL)
        if W:
            ctl[0] = ctl[-1] = control
    else:
        W = len(waypoints)
        vals = np.stack([waypoints["pos"][:, :dim], waypoints["vel"][:, :dim], waypoints["acc"][:, :dim]], axis=1)
        yaw = np.asarray(waypoints["yaw"], dtype=np.float64)
        ctl = np.asarray(wp_control, dtype=np.int64)
        p = vals[:, 0]
    if dts is None:
        taus = np.abs(np.diff(p, axis=0)).max(axis=1) / v if W > 1 else np.zeros(0)
    else:
        taus = np.asarray(dts, dtype=np.float64)
    if W < 2:
        return dict(status=0, seg_t=taus, coeff=np.zeros((0, dim + 1, 6)))
    fixed = np.array([[(c >> k) & 1 for k in range(h)] for c in ctl], dtype=bool)
    D = solve_derivatives(h, taus, fixed, vals[:, :h])
    yc = np.full(W, VEL)
    yc[0] = yc[-1] = yaw_control
    yfixed = np.array([[(c >> k) & 1 for k in range(hy)] for c in yc], dtype=bool)
    yvals = np.zeros((W, hy, 1))
    yvals[:, 0, 0] = yaw
    Dy = solve_derivatives(hy, taus, yfixed, yvals)
    coeff = np.zeros((W - 1, dim + 1, 6))
    with np.errstate(all="ignore"):
        for i, tau in enumerate(taus):
            for a in range(dim):
                coeff[i, a] = seg_coeff(h, tau, D[i, :, a], D[i + 1, :, a])
            coeff[i, dim] = seg_coeff(hy, tau, Dy[i, :, 0], Dy[i + 1, :, 0])
    return dict(status=int(np.isfinite(coeff).all()), seg_t=taus, coeff=coeff)


def sample_columns(dim, ncols):
    """Column groups of a sample row {pos, vel, acc, jrk (dim each), yaw, yaw_dot, t} or a waypoint row
    {pos, vel, acc, jrk, yaw, t}, and the angle columns."""
    groups = [list(range(k * dim, (k + 1) * dim)) for k in range(4)] + [[c] for c in range(4 * dim, ncols)]
    return groups, ({4 * dim, 4 * dim + 1} if ncols == 4 * dim + 3 else {4 * dim})


def assert_close(got, ref, dim, rtol=1e-9, what=""):
    """|got - ref| <= rtol (1 + max |ref| over the column group) for every derivative group of sample rows
    (pos, vel, acc, jrk, yaw, yaw_dot, t) or waypoint rows (pos, vel, acc, jrk, yaw, t); angle columns compare
    modulo 2 pi (normalize_angle wraps them)."""
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert np.isfinite(got).all() and np.isfinite(ref).all(), what
    groups, angles = sample_columns(dim, got.shape[1])
    for g in groups:
        d = got[:, g] - ref[:, g]
        if g[0] in angles:
            d = (d + np.pi) % (2 * np.pi) - np.pi
        tol = rtol * (1 + np.abs(ref[:, g]).max())
        err = np.abs(d).max()
        assert err <= tol, (what, g, err, tol)
