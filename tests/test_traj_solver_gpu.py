"""mplx_traj_solve (TrajSolverBatch): TrajSolver for batches of paths on the device.

Device coefficients are checked through what they evaluate to — the host Trajectory's sample(N) and
getWaypoints() — against the host's dense restatement (MPL::TrajSolver) for paths it solves in seconds and
against the block-tridiagonal statement (traj_restatement.py) for longer ones: |device - host| <=
1e-9 (1 + max |host| over the path) per derivative.  The device's own samples must equal the host Trajectory
built from the device's segment times and coefficients bit for bit."""
import ctypes as C

import numpy as np
import pytest

import traj_restatement as TR
from motion_primitive_library_b200 import TrajSolverBatch, abi
from motion_primitive_library_b200 import planner as P

pytestmark = pytest.mark.gpu

CONTROLS = [0x01, 0x03, 0x07, 0x11, 0x13, 0x17]
YAWS = [0x01, 0x03, 0x07]
NS = 40


@pytest.fixture(scope="module")
def solvers():
    s = {2: TrajSolverBatch(2), 3: TrajSolverBatch(3)}
    yield s
    for x in s.values():
        x.close()


def make_paths(rng, dim, n_paths, lo=2, hi=60, setwp=False):
    paths, ctls, dts = [], [], []
    for _ in range(n_paths):
        n = int(rng.integers(lo, hi + 1))
        pos = np.cumsum(rng.uniform(-2, 2, (n, dim)), axis=0)
        dts.append(rng.uniform(0.05, 5, n - 1))
        if setwp:
            w = np.zeros(n, dtype=P.WAYPOINT_DTYPE)
            w["pos"][:, :dim] = pos
            w["vel"][:, :dim] = rng.uniform(-1, 1, (n, dim))
            w["acc"][:, :dim] = rng.uniform(-1, 1, (n, dim))
            w["yaw"] = rng.uniform(-1, 1, n)
            c = rng.choice([0x01, 0x03, 0x07, 0x13], n).astype(np.uint8)
            c[[0, -1]] = rng.choice([0x03, 0x07], 2)
            paths.append(w)
            ctls.append(c)
        else:
            paths.append(pos)
    return paths, (ctls if setwp else None), dts


def host_kw(path, ctl, dts, v, yaw_control):
    kw = dict(yaw_control=yaw_control, v=v, dts=dts)
    if ctl is None:
        kw["pos"] = path
    else:
        kw.update(waypoints=path, wp_control=ctl)
    return kw


def check_path(dim, control, r, ref_samples, ref_waypoints, ctl0, what):
    """r: the device's result for one path; ref_*: the reference sampling of the same trajectory."""
    assert r["status"] == 1, what
    s, w = P.traj_sample(dim, r["seg_t"], r["coeff"], ctl0, NS)
    assert s.tobytes() == r["samples"].tobytes(), (what, "device samples differ from the host sampling")
    TR.assert_close(s, ref_samples, dim, what=what)
    TR.assert_close(w, ref_waypoints, dim, what=what)


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("yaw_control", YAWS)
@pytest.mark.parametrize("mode", ["path", "waypoints"])
@pytest.mark.parametrize("given_dts", [False, True])
def test_matches_host_restatement(solvers, dim, control, yaw_control, mode, given_dts):
    rng = np.random.default_rng([dim, control, yaw_control, mode == "path", given_dts])
    paths, ctls, dts = make_paths(rng, dim, 6, setwp=mode == "waypoints")
    if not given_dts:
        dts = None
    v = float(rng.uniform(0.5, 2.0))
    res, _ = solvers[dim].solve(paths, control, yaw_control, dts=dts, v=v, wp_control=ctls, n_samples=NS)
    for p in range(len(paths)):
        kw = host_kw(paths[p], None if ctls is None else ctls[p], None if dts is None else dts[p], v, yaw_control)
        host = P.traj_solve(dim, control, n_samples=NS, **kw)
        np.testing.assert_array_equal(res[p]["seg_t"], host["seg_t"])
        ctl0 = control if ctls is None else int(ctls[p][0])
        check_path(dim, control, res[p], host["samples"], host["waypoints"], ctl0, (p, len(paths[p])))


@pytest.mark.parametrize("control", [0x03, 0x07, 0x17])
def test_paths_of_200_waypoints(solvers, control):
    rng = np.random.default_rng(control)
    paths, _, dts = make_paths(rng, 3, 3, lo=150, hi=200)
    res, _ = solvers[3].solve(paths, control, 0x03, dts=dts, n_samples=NS)
    for p in range(3):
        host = P.traj_solve(3, control, pos=paths[p], dts=dts[p], yaw_control=0x03, n_samples=NS)
        check_path(3, control, res[p], host["samples"], host["waypoints"], control, p)


def test_reference_case():
    """The reference's test_traj_solver.cpp: path (0,0), (1,0), (2,1), (5,1), v = 1, VEL / ACC / JRK, against the
    reference's own TrajSolver (live where oracle/_ref is built, else its recording)."""
    import traj_bindings as TB

    path = np.array([(0, 0), (1, 0), (2, 1), (5, 1)], dtype=np.float64)
    refs = {c: TB.traj_reference(2, c, max_bytes=None, pos=path, v=1.0, n_samples=NS) for c in (0x01, 0x03, 0x07)}
    s = TrajSolverBatch(2)
    for control, ref in refs.items():
        res, _ = s.solve([path], control, v=1.0, n_samples=NS)
        np.testing.assert_array_equal(res[0]["seg_t"], ref["seg_t"])
        check_path(2, control, res[0], ref["samples"], ref["waypoints"], control, control)
    s.close()


def solve_alone(s, paths, control, yaw_control, dts, ctls, p):
    r, _ = s.solve([paths[p]], control, yaw_control, dts=None if dts is None else [dts[p]],
                   wp_control=None if ctls is None else [ctls[p]], n_samples=NS)
    return r[0]


def same_result(a, b, what):
    assert a["status"] == b["status"], what
    for k in ("seg_t", "coeff", "samples"):
        assert a[k].tobytes() == b[k].tobytes(), (what, k)


def test_batch_edge_cases(solvers):
    s = solvers[3]
    l0 = s.launch_count()
    res, sec = s.solve([], 0x07)
    assert res == [] and s.launch_count() == l0
    rng = np.random.default_rng(5)
    paths, _, dts = make_paths(rng, 3, 8, lo=2, hi=12)
    paths[1] = np.zeros((0, 3))
    dts[1] = np.zeros(0)
    paths[4] = paths[4][:1]
    dts[4] = np.zeros(0)
    bad = paths[6].copy()
    dts[6] = dts[6].copy()
    dts[6][len(dts[6]) // 2] = 0.0  # a zero-length segment
    paths[6] = bad
    res, _ = s.solve(paths, 0x07, dts=dts, n_samples=NS)
    assert [r["status"] for r in res] == [1, 0, 1, 1, 0, 1, 0, 1]
    assert not np.isfinite(res[6]["coeff"]).all()
    for p in (1, 4, 6):
        assert not res[p]["samples"].any()
    for p in range(len(paths)):
        same_result(res[p], solve_alone(s, paths, 0x07, 0x01, dts, None, p), p)
    one, _ = s.solve(paths[:1], 0x07, dts=dts[:1], n_samples=NS)
    same_result(one[0], res[0], "one path")
    # no path with a segment and no waypoint slot: the sweep and the samples run, the coefficient kernel does not
    l0 = s.launch_count()
    res, _ = s.solve([np.zeros((0, 3)), np.zeros((0, 3))], 0x07, n_samples=NS)
    assert s.launch_count() - l0 == 2
    assert [r["status"] for r in res] == [0, 0] and not any(r["samples"].any() for r in res)


def test_allocated_zero_length_segment(solvers):
    path = np.array([(0, 0), (1, 0), (1, 0), (2, 1)], dtype=np.float64)  # L-inf allocation gives a 0 s segment
    res, _ = solvers[2].solve([path], 0x03, v=1.0, n_samples=NS)
    host = P.traj_solve(2, 0x03, pos=path, v=1.0, n_samples=NS)
    assert res[0]["status"] == 0 and res[0]["seg_t"][1] == 0.0
    assert not np.isfinite(res[0]["coeff"]).all() and not np.isfinite(host["coeff"]).all()


@pytest.mark.parametrize("mode", ["path", "waypoints"])
def test_batch_of_4096_mixed_lengths(solvers, mode):
    rng = np.random.default_rng(4096 + (mode == "path"))
    paths, ctls, dts = [], [], []
    for _ in range(4096):
        n = int(rng.integers(0, 65))
        q, c, d = make_paths(rng, 3, 1, lo=max(n, 2), hi=max(n, 2), setwp=mode == "waypoints")
        paths.append(q[0][:n])
        dts.append(d[0][: max(n - 1, 0)])
        if c is not None:
            ctls.append(c[0][:n])
    ctls = ctls if mode == "waypoints" else None
    s = solvers[3]
    res, sec = s.solve(paths, 0x17, 0x07, dts=dts, wp_control=ctls, n_samples=NS)
    assert sec > 0
    for p in range(4096):
        assert res[p]["status"] == (1 if len(paths[p]) >= 2 else 0), p
        same_result(res[p], solve_alone(s, paths, 0x17, 0x07, dts, ctls, p), p)


def test_long_path(solvers):
    """5 000 waypoints, JRK, 3-D, against the block-tridiagonal statement; every waypoint's position is met."""
    rng = np.random.default_rng(5000)
    n = 5000
    pos = np.cumsum(rng.uniform(-1, 1, (n, 3)), axis=0)
    dts = rng.uniform(0.05, 5, n - 1)
    res, _ = solvers[3].solve([pos], 0x07, 0x07, dts=[dts], n_samples=2000)
    r = res[0]
    assert r["status"] == 1
    mine = TR.traj_solve(3, 0x07, pos=pos, dts=dts, yaw_control=0x07)
    s_dev, w_dev = P.traj_sample(3, r["seg_t"], r["coeff"], 0x07, 2000)
    s_ref, w_ref = P.traj_sample(3, mine["seg_t"], mine["coeff"], 0x07, 2000)
    assert s_dev.tobytes() == r["samples"].tobytes()
    TR.assert_close(s_dev, s_ref, 3)
    TR.assert_close(w_dev, w_ref, 3)
    # fixed derivatives: each segment starts at its waypoint exactly, ends there within the tolerance; the ends
    # also meet the zero velocity and acceleration of the JRK control
    np.testing.assert_array_equal(r["coeff"][:, :3, 5], pos[:-1])
    tol = 1e-9 * (1 + np.abs(pos).max())
    assert np.abs(w_dev[:, :3] - pos).max() <= tol
    assert np.abs(w_dev[[0, -1], 3:9]).max() <= tol


def test_refusals(solvers):
    s = solvers[2]
    lib = abi.load()
    wps = np.zeros(3, dtype=abi.WAYPOINT_DTYPE)
    wps["pos"][:, 0] = [0, 1, 2]
    off = np.array([0, 3], dtype=np.int64)
    status = np.full(1, 7, dtype=np.int32)
    seg_t = np.full(3, 7.0)
    coeff = np.full((3, 3, 6), 7.0)
    samples = np.full((1, 5, 11), 7.0)

    def call(n_paths=1, offset=off, w=wps, ctl=None, dts=None, v=1.0, control=0x03, yaw=0x01, n_samples=4,
             with_samples=True, out=True, status_p=True):
        o = abi.TrajOut(status.ctypes.data if status_p else None, seg_t.ctypes.data, coeff.ctypes.data,
                        samples.ctypes.data if with_samples else None, 0.0)
        return lib.mplx_traj_solve(s._h, n_paths, None if offset is None else offset.ctypes.data,
                                   None if w is None else w.ctypes.data, ctl, dts, v, control, yaw, n_samples,
                                   C.byref(o) if out else None)

    l0 = s.launch_count()
    cases = [dict(control=0x0F), dict(control=0x1F), dict(control=0x00), dict(yaw=0x0F), dict(yaw=0x13), dict(yaw=0),
             dict(v=0.0), dict(v=-1.0), dict(n_paths=-1), dict(offset=np.array([0, 3, 2], dtype=np.int64), n_paths=2),
             dict(offset=np.array([1, 3], dtype=np.int64)), dict(offset=None), dict(w=None), dict(out=False),
             dict(status_p=False), dict(n_samples=0), dict(n_samples=-3)]
    for kw in cases:
        assert call(**kw) == abi.MPLX_ERR_ARG, kw
    assert s.launch_count() == l0
    assert (status == 7).all() and (seg_t == 7.0).all() and (coeff == 7.0).all() and (samples == 7.0).all()
    assert call() == abi.MPLX_OK and status[0] == 1 and s.launch_count() == l0 + 3
