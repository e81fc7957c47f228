"""mplx_traj_scale (TrajSolverBatch.scale): Trajectory::scale / scale_down for batches of trajectories on the device,
against the host Trajectory (mpl_host.hpp) on the same segment times and coefficients.

Accuracy contract (DESIGN.md §8): VEL and ACC paths (extrema_v is linear or empty) and status-2 paths agree bit
for bit in the status, total time, segment times and lambda segments; so do the samples of scale with ri == rf
(lambda constant, getTau linear).  Otherwise every field is held to 1e-9 (1 + max |host value| over the path),
since the closed-form roots call CUDA's cbrt, acos and cos.  On those paths the two sides may disagree only about
the final row, where one finds the quartic root just past the last lambda segment (the start state) and the other
just inside it (the end state)."""
import ctypes as C

import numpy as np
import pytest

from motion_primitive_library_b200 import TrajSolverBatch, abi
from motion_primitive_library_b200 import planner as P

pytestmark = pytest.mark.gpu

VEL, ACC, JRK = 0x01, 0x03, 0x07
SCALE, SCALE_DOWN = 1, 2
NS = 40
FINAL_ROW_DISAGREEMENTS = []  # (case, path) where the sides disagree about the final row's getTau


@pytest.fixture(scope="module")
def solvers():
    s = {2: TrajSolverBatch(2), 3: TrajSolverBatch(3)}
    yield s
    for x in s.values():
        x.close()


def solved(s, dim, control, yaw_control, n_paths, seed, lo=2, hi=30, setwp=True):
    rng = np.random.default_rng(seed)
    paths, ctls = [], []
    for _ in range(n_paths):
        n = int(rng.integers(lo, hi + 1))
        if setwp:
            w = np.zeros(n, dtype=P.WAYPOINT_DTYPE)
            w["pos"][:, :dim] = np.cumsum(rng.uniform(-2, 2, (n, dim)), axis=0)
            w["yaw"] = rng.uniform(-3, 3, n)
            paths.append(w)
            ctls.append(np.full(n, control, dtype=np.uint8))
        else:
            paths.append(np.cumsum(rng.uniform(-2, 2, (n, dim)), axis=0))
    res, _ = s.solve(paths, control, yaw_control=yaw_control, v=float(rng.uniform(0.7, 1.5)),
                     wp_control=ctls if setwp else None, n_samples=NS)
    assert all(r["status"] == 1 for r in res)
    return res


def params(rng, n, mode):
    if mode == SCALE:
        ri = rng.choice([1.0, 0.5, 2.0], n)
        rf = np.where(rng.random(n) < 0.5, ri, rng.uniform(0.5, 2.0, n))
        return None, ri, rf
    return rng.uniform(0.3, 2.0, n), rng.uniform(0.5, 1.5, n), rng.uniform(0.5, 1.5, n)


def host(dim, r, mode, mv, ri, rf, control):
    return P.traj_scale(dim, r["seg_t"], r["coeff"], mode, mv=1.0 if mv is None else mv, ri=ri, rf=rf,
                        control=control, n_samples=NS)


def close(a, b, what, scale=None):
    """|a - b| <= 1e-9 (1 + max |scale|), scale defaulting to b"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, what
    # a lambda segment between knots an ulp apart is singular and not finite on both sides, as in the reference
    assert np.array_equal(np.isfinite(a), np.isfinite(b)), (what, a, b)
    f = np.isfinite(b)
    m = np.abs(b if scale is None else np.asarray(scale, dtype=np.float64))
    m = m[np.isfinite(m)]
    tol = 1e-9 * (1 + (m.max() if m.size else 0))
    assert np.all(np.abs(a[f] - b[f]) <= tol), (what, a, b, float(np.abs(a[f] - b[f]).max()), tol)


def compare(dim, d, h, exact, exact_samples, what):
    assert d["status"] == h["status"], what
    if exact:
        assert float(d["total_t"]).hex() == float(h["total_t"]).hex(), what
        assert d["seg_T"].tobytes() == h["seg_T"].tobytes(), what
        assert d["lambda"].tobytes() == h["lambda"].tobytes(), what
    else:
        close(d["total_t"], h["total_t"], what)
        close(d["seg_T"], h["seg_T"], what)
        assert d["lambda"].shape == h["lambda"].shape, what
        for k in range(7):
            close(d["lambda"][:, k], h["lambda"][:, k], (what, "lambda", k))
    ds, hs = d["samples"], h["samples"]
    if exact_samples:
        assert ds.tobytes() == hs.tobytes(), what
        return
    last = len(ds) - 1
    for f in range(ds.shape[1]):
        close(ds[:last, f], hs[:last, f], (what, "field", f))
    try:
        for f in range(ds.shape[1]):
            close(ds[last:, f], hs[:, f][last:], (what, "final row", f))
    except AssertionError:
        # one side found the last root an ulp past the final lambda segment: its row is the start state
        t, total = hs[last, -1], h["total_t"]
        assert abs(t - total) <= 1e-9 * (1 + total), what
        # (row 0 is getTau(0), a root within rounding of tau = 0, so the start state up to the tolerance)
        tol = 1e-9 * (1 + np.abs(hs[:, :dim]).max())
        d0 = bool(np.all(np.abs(ds[last, :dim] - hs[0, :dim]) <= tol))
        h0 = bool(np.all(np.abs(hs[last, :dim] - hs[0, :dim]) <= tol))
        assert d0 != h0, (what, ds[last], hs[last], ds[0])
        FINAL_ROW_DISAGREEMENTS.append(what)


@pytest.mark.parametrize("mode", [SCALE, SCALE_DOWN])
@pytest.mark.parametrize("yaw_control", [VEL, ACC, JRK])
@pytest.mark.parametrize("control", [VEL, ACC, JRK])
@pytest.mark.parametrize("dim", [2, 3])
def test_device_against_host(solvers, dim, control, yaw_control, mode):
    s = solvers[dim]
    seed = dim * 1000 + control * 100 + yaw_control * 10 + mode
    res = solved(s, dim, control | 0x10, yaw_control, 48, seed, setwp=yaw_control != VEL)
    rng = np.random.default_rng(seed)
    mv, ri, rf = params(rng, len(res), mode)
    out, sec = s.scale(res, mode, mv=mv, ri=ri, rf=rf, n_samples=NS, with_lambda=True)
    assert sec > 0
    counts = {0: 0, 1: 0, 2: 0}
    for p, (d, r) in enumerate(zip(out, res)):
        h = host(dim, r, mode, None if mv is None else mv[p], ri[p], rf[p], control | 0x10)
        counts[d["status"]] += 1
        exact = control != JRK or d["status"] == 2
        exact_samples = d["status"] == 2 or (mode == SCALE and ri[p] == rf[p])
        compare(dim, d, h, exact, exact_samples, (dim, control, yaw_control, mode, p))
    assert counts[0] == 0 and counts[1] > 0


@pytest.mark.parametrize("dim", [2, 3])
def test_unscaled_rows_equal_the_solver_samples(solvers, dim):
    """scale(1, 1) and status-2 paths: every row but the last is mplx_traj_solve's; the last is the host's."""
    s = solvers[dim]
    res = solved(s, dim, JRK, VEL, 32, 77 + dim, setwp=False)
    for mode, mv in ((SCALE, None), (SCALE_DOWN, 1e9)):
        out, _ = s.scale(res, mode, mv=mv, n_samples=NS)
        for d, r in zip(out, res):
            assert d["status"] == (1 if mode == SCALE else 2)
            assert d["samples"][:-1].tobytes() == r["samples"][:-1].tobytes()
            h = host(dim, r, mode, mv, 1.0, 1.0, JRK)
            assert d["samples"][-1].tobytes() == h["samples"][-1].tobytes()


def test_status_classes(solvers):
    s = solvers[3]
    res = solved(s, 3, ACC, VEL, 6, 5)
    bad_t = dict(res[1], seg_t=res[1]["seg_t"].copy())
    bad_t["seg_t"][0] = 0.0
    bad_c = dict(res[2], coeff=res[2]["coeff"].copy())
    bad_c["coeff"][-1, 3, 0] = np.inf
    empty = dict(seg_t=np.zeros(0), coeff=np.zeros((0, 4, 6)))
    batch = [res[0], bad_t, bad_c, empty, res[3], res[4], res[5]]
    mv = np.array([0.5, 0.5, 0.5, 0.5, 1e9, np.nan, 0.5])
    ri = np.array([1, 1, 1, 1, 1, 1, -1.0])
    out, _ = s.scale(batch, SCALE_DOWN, mv=mv, ri=ri, rf=1.0, n_samples=NS, with_lambda=True)
    assert [o["status"] for o in out] == [1, 0, 0, 0, 2, 0, 0]
    for o in out:
        if o["status"] == 0:
            assert o["total_t"] == 0 and not o["seg_T"].any() and not o["samples"].any() and len(o["lambda"]) == 0
    assert out[4]["total_t"] > 0 and out[4]["seg_T"].all() and len(out[4]["lambda"]) == 0
    # a batch in which no path has a segment has no waypoint slot: every kernel still runs, on one block
    for mode in (SCALE, SCALE_DOWN):
        for ns, with_lambda in ((0, False), (NS, True)):
            l0 = s.launch_count()
            out, _ = s.scale([empty, empty], mode, mv=0.5, ri=1.0, rf=1.0, n_samples=ns, with_lambda=with_lambda)
            assert s.launch_count() - l0 == 5 + (ns > 0)
            for o in out:
                assert o["status"] == 0 and o["total_t"] == 0 and not o["seg_T"].any()
                assert not o.get("samples", np.zeros(1)).any() and len(o.get("lambda", [])) == 0


def test_refusals(solvers):
    s = solvers[2]
    lib = s._lib
    res = solved(s, 2, ACC, VEL, 2, 9)
    n = np.array([len(r["seg_t"]) + 1 for r in res], dtype=np.int64)
    offset = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    seg_t = np.concatenate([np.append(r["seg_t"], 0) for r in res])
    coeff = np.concatenate([np.concatenate([r["coeff"], np.zeros((1, 3, 6))]) for r in res])
    one = np.ones(2)
    status = np.full(2, 7, dtype=np.int32)
    total, seg_T, samples = np.zeros(2), np.zeros(int(offset[-1])), np.zeros((2, NS + 1, 11))

    def out(**kw):
        f = dict(status=status.ctypes.data, total_t=total.ctypes.data, seg_T=seg_T.ctypes.data, n_lambda=None,
                 lambda_=None, samples=samples.ctypes.data, seconds=0.0)
        f.update(kw)
        return abi.TrajScaleOut(**f)

    def call(n_paths=2, off=offset.ctypes.data, st=seg_t.ctypes.data, co=coeff.ctypes.data, mode=SCALE_DOWN,
             mv=one.ctypes.data, ri=one.ctypes.data, rf=one.ctypes.data, ns=NS, o=None):
        o = o or out()
        return lib.mplx_traj_scale(s._h, n_paths, off, st, co, mode, mv, ri, rf, ns, C.byref(o))

    bad_off = offset.copy()
    bad_off[0] = 1
    dec = offset.copy()
    dec[1] = dec[2] + 1
    launches = s.launch_count()
    cases = [dict(mode=3), dict(mode=0), dict(mv=None), dict(ri=None), dict(rf=None), dict(n_paths=-1), dict(off=None),
             dict(off=bad_off.ctypes.data), dict(off=dec.ctypes.data), dict(st=None), dict(co=None), dict(ns=0),
             dict(o=out(status=None)), dict(o=out(total_t=None)), dict(o=out(seg_T=None))]
    for kw in cases:
        assert call(**kw) == 1, kw  # MPLX_ERR_ARG
    assert s.launch_count() == launches
    assert (status == 7).all()
    assert call(mode=SCALE, mv=None) == 0 and (status == 1).all()
    assert call(n_paths=0) == 0


def test_per_path_independence(solvers):
    """A 4 096-path mixed batch (controls, lengths, modes' parameters) against each path scaled on its own."""
    s = solvers[3]
    res = []
    for k, control in enumerate((VEL, ACC, JRK, ACC | 0x10)):
        res += solved(s, 3, control, VEL, 1024, 900 + k, lo=2, hi=40, setwp=bool(k % 2))
    rng = np.random.default_rng(4)
    order = rng.permutation(len(res))
    res = [res[i] for i in order]
    mv = rng.uniform(0.3, 3, len(res))
    ri = rng.uniform(0.5, 1.5, len(res))
    out, _ = s.scale(res, SCALE_DOWN, mv=mv, ri=ri, rf=1.0, n_samples=NS, with_lambda=True)
    assert {o["status"] for o in out} >= {1, 2}
    for p in rng.choice(len(res), 64, replace=False):
        one, _ = s.scale([res[p]], SCALE_DOWN, mv=mv[p], ri=ri[p], rf=1.0, n_samples=NS, with_lambda=True)
        for k in ("seg_T", "lambda", "samples"):
            assert one[0][k].tobytes() == out[p][k].tobytes(), (p, k)
        assert one[0]["status"] == out[p]["status"]
        assert float(one[0]["total_t"]).hex() == float(out[p]["total_t"]).hex()


def test_long_path(solvers):
    """A 5 000-waypoint JRK path: many knots per segment and the lambda slot bound."""
    s = solvers[3]
    res = solved(s, 3, JRK, VEL, 1, 31, lo=5000, hi=5000, setwp=False)
    out, _ = s.scale(res, SCALE_DOWN, mv=0.4, n_samples=2000, with_lambda=True)
    d = out[0]
    assert d["status"] == 1 and len(d["lambda"]) > 5000
    assert len(d["lambda"]) <= 5000 * 15
    h = P.traj_scale(3, res[0]["seg_t"], res[0]["coeff"], SCALE_DOWN, mv=0.4, control=JRK, n_samples=2000)
    assert len(h["lambda"]) == len(d["lambda"])
    close(d["total_t"], h["total_t"], "total")
    close(d["seg_T"], h["seg_T"], "seg_T")
    for f in range(d["samples"].shape[1]):
        close(d["samples"][:-1, f], h["samples"][:-1, f], ("field", f))


def test_acc_set_path_velocity_bound(solvers):
    """ACC setPath trajectories after scale_down(mv, 1, 1): every non-final sample whose tau lies in a
    constant-lambda segment has |vel| <= mv (1 + 1e-12)."""
    s = solvers[3]
    res = solved(s, 3, ACC, VEL, 256, 12, lo=2, hi=40, setwp=False)
    mv = 0.6
    out, _ = s.scale(res, SCALE_DOWN, mv=mv, n_samples=200, with_lambda=True)
    checked = 0
    for d in out:
        if d["status"] != 1:
            continue
        lam, t = d["lambda"], d["samples"][:-1, -1]
        T = np.zeros(len(lam) + 1)
        for k in range(len(lam)):
            T[k + 1] = T[k] + lam[k, 6]
        for k in range(len(lam)):
            if lam[k, 0] == 0 and lam[k, 1] == 0 and lam[k, 2] == 0:
                rows = (t > T[k]) & (t < T[k + 1])
                v = d["samples"][:-1][rows, 3:6]
                assert np.all(np.abs(v) <= mv * (1 + 1e-12)), (k, np.abs(v).max())
                checked += int(rows.sum())
    assert checked > 1000


def test_report_final_row_disagreements():
    print(f"final-row getTau disagreements: {len(FINAL_ROW_DISAGREEMENTS)} {FINAL_ROW_DISAGREEMENTS[:8]}")
