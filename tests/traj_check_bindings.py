"""Trajectory-check bindings for the tests: the product's host restatement (planner.traj_check) and the
REFERENCE's own env_map::traverse_trajectory / is_free and validate_primitive (oracle/_ref/libmplref_traj_check.so,
built by oracle/traj_check.mk), with the same signature (mplh_traj_check in host/mpl_host_capi.cpp)."""
import numpy as np

from motion_primitive_library_b200 import planner as P
from motion_primitive_library_b200.planner import load_traj_check_fn, run_traj_check, traj_check  # noqa: F401
from reference_record import reference
from traj_bindings import ROOT

REF_CHECK = ROOT / "oracle" / "_ref" / "libmplref_traj_check.so"
VEL, ACC, JRK, YAW = 0x01, 0x03, 0x07, 0x10


def check_reference(dim, grid, mdim, origin, res, paths, control, **kw):
    """The reference's checks on a batch of trajectories (arguments as planner.run_traj_check)."""
    def live():
        lib, fn = load_traj_check_fn(REF_CHECK, "reft_traj_check")
        r = run_traj_check(fn, lib, dim, grid, mdim, origin, res, paths, control, **kw)
        r.pop("offset")
        return r

    return reference(REF_CHECK, live, max_bytes=None)


def solved_paths(dim, control, yaw, n_paths, seed, lo, hi, n_wp=(2, 12), v=(0.5, 2.0)):
    """Host TrajSolver outputs through random waypoints in the box [lo, hi): setPath without yaw, setWaypoints
    with yaws and control | YAW flags with yaw.  Returns (paths, per-path control flags)."""
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(lo, dtype=np.float64), np.asarray(hi, dtype=np.float64)
    paths, ctl = [], []
    for _ in range(n_paths):
        n = int(rng.integers(n_wp[0], n_wp[1] + 1))
        pos = lo + (hi - lo) * rng.random((n, dim))
        if not yaw:
            r = P.traj_solve(dim, control, pos=pos, v=float(rng.uniform(*v)), n_samples=1)
            ctl.append(control)
        else:
            w = np.zeros(n, dtype=P.WAYPOINT_DTYPE)
            w["pos"][:, :dim] = pos
            w["yaw"] = rng.uniform(-3, 3, n)
            r = P.traj_solve(dim, control | YAW, waypoints=w, wp_control=np.full(n, control | YAW, dtype=np.uint8),
                             dts=rng.uniform(0.5, 3, n - 1), yaw_control=int(rng.choice([VEL, ACC, JRK])), n_samples=1)
            ctl.append(control | YAW)
        paths.append(dict(seg_t=r["seg_t"], coeff=r["coeff"]))
    return paths, np.asarray(ctl, dtype=np.uint8)


def random_grid(mdim, seed, p_occ=0.04, p_unknown=0.05):
    """A random grid: occupied (100), unknown (-1) and free (0) cells."""
    rng = np.random.default_rng(seed)
    u = rng.random(int(np.prod(mdim)))
    return np.where(u < p_occ, 100, np.where(u < p_occ + p_unknown, -1, 0)).astype(np.int8)


def max_abs(coeff, t, order):
    """max |d^order p / dt^order| over [0, t] of one Primitive1D (coefficients highest first), from the ends and
    the critical points, in numpy's arithmetic (not the host's)."""
    c = np.asarray(coeff, dtype=np.float64)
    poly = np.array([c[0] / 120, c[1] / 24, c[2] / 6, c[3] / 2, c[4], c[5]])
    for _ in range(order):
        poly = np.polyder(poly)
    ts = [0.0, t] + [r.real for r in np.roots(np.polyder(poly)) if abs(r.imag) < 1e-12 and 0 < r.real < t] \
        if len(poly) > 1 else [0.0, t]
    return max(abs(np.polyval(poly, x)) for x in ts)


def wrapped_index_case():
    """A map whose far cells' getIndex wraps in 32 bits: 256 x 256 x 2 cells of 1 m at the origin, and a VEL path
    from (0.5, 0.5, 0.5) straight up to (0.5, 0.5, 65536.5) with segment time 65536.  The end's cell (0, 0, 65536)
    has the index 256 * 256 * 65536 = 2^32, which wraps to 0, the start's index.  Returns (grid, mdim, origin, res,
    paths); v_max = k / 65536 gives N = k samples after the first."""
    mdim, origin, res = (256, 256, 2), (0.0, 0.0, 0.0), 1.0
    grid = np.zeros(int(np.prod(mdim)), dtype=np.int8)
    p = P.traj_solve(3, VEL, pos=np.array([[0.5, 0.5, 0.5], [0.5, 0.5, 65536.5]]), v=1.0, n_samples=1)
    assert p["seg_t"][0] == 65536.0
    return grid, mdim, origin, res, [dict(seg_t=p["seg_t"], coeff=p["coeff"])]
