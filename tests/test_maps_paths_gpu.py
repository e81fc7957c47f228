"""mplx_update_potential_map and mplx_set_search_region_path (csrc/mplx_maps.cu) on every shape class, radius
class, source class, exponent, source range and refusal, bit for bit against the numpy restatement of
tests/test_maps_inputs_restatement_vs_ref.py — which that file pins, case by case, to the reference itself
(oracle/_ref or its recordings), so device = restatement = reference.  One larger map is compared with the
layer-wise statement scenarios.potential_from_map, pinned to the reference by digest in the same CPU file.

Also here: the device state the field call leaves behind (grid, occupancy words, occ2 pairs, weights) against
a fresh ctx given the field, repeated calls, the launches each call adds, and the region driving the expansion
and the stored-edge query."""
import ctypes as C

import numpy as np
import pytest

import oracle_bindings as ob
from parity import assert_expansion_equal
from test_maps_inputs_restatement_vs_ref import BIG, POTENTIAL, REGION, RN_MAX, big_grid, distinct_stencil_radii

pytestmark = pytest.mark.gpu
ACC = 0x03
WANT = ("succ", "cost", "action", "key", "lattice")
FIELD_LAUNCHES = 4   # source_bits_kernel, layer_rank_kernel, potential_combine_kernel + one for the re-pack of occ / occ2
REGION_LAUNCHES = 1  # region_stamp_kernel; none when the path yields no cell


def gpu_env(grid, dims, origin, res):
    from motion_primitive_library_b200 import MapUtil, env_map

    mu = MapUtil()
    mu.setMap(origin, dims, np.array(grid, dtype=np.int8), res)
    return env_map(mu)


def pad3(v):
    return None if v is None else tuple(v) + (0.0,) * (3 - len(v))


def run_field(env, case):
    return env.update_potential_map(pad3(case.radius), case.pow_, pad3(case.range_), pad3(case.pos))


def same_device_state(env, other):
    for a, b, what in zip(env.read_map(), other.read_map(), ("grid", "occupancy words", "occ2 pairs")):
        assert a.tobytes() == b.tobytes(), what


# ---- the potential field -------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(POTENTIAL))
def test_potential_field_matches_restatement(name):
    case = POTENTIAL[name]
    g = case.grid()
    env = gpu_env(g, case.dims, case.origin, case.res)
    before = env.launch_count()
    got = run_field(env, case)
    assert env.launch_count() - before == FIELD_LAUNCHES
    want = case.restate()
    assert got.tobytes() == want.tobytes(), (name, np.flatnonzero(got != want)[:8])
    # the call replaces the device grid by the field and re-packs both occupancy layouts
    same_device_state(env, gpu_env(want, case.dims, case.origin, case.res))


def test_rank_table_limit_and_refusals_leave_the_ctx_untouched():
    from motion_primitive_library_b200 import abi
    from scenarios import control_set

    case = POTENTIAL["3d_pow2.0"]
    env = gpu_env(case.grid(), case.dims, case.origin, case.res)
    env.set_control(ACC)
    env.set_u(control_set(1.0, 3, 3))
    env.set_v_max(2.0)
    env.set_potential_weight(0.7)
    run_field(env, case)
    rng = np.random.default_rng(1)
    nodes = np.zeros(300, dtype=ob.WAYPOINT_DTYPE)
    ext = np.asarray(case.dims) * case.res
    nodes["pos"][:, :3] = np.asarray(case.origin) + rng.random((300, 3)) * ext
    nodes["vel"][:, :3] = rng.integers(-2, 3, (300, 3)) * 0.5
    state, exp, launches = env.read_map(), env.expand(nodes, want=WANT), None
    launches = env.launch_count()
    res, r1 = case.res, case.res
    assert distinct_stencil_radii(RN_MAX + 1) >= 255
    refusals = (
        (dict(radius=(r1, r1, r1), pow_=0.0), "pow must be > 0"),
        (dict(radius=(r1, r1, r1), pow_=-1.0), "pow must be > 0"),
        (dict(radius=(r1, r1, r1), pow_=float("nan")), "pow must be > 0"),
        (dict(radius=(0.0, 0.0, r1), pow_=1.0), "smaller than one cell"),
        (dict(radius=(r1, r1, 0.0), pow_=1.0), "smaller than one cell"),
        (dict(radius=(-r1, r1, r1), pow_=1.0), "smaller than one cell"),
        (dict(radius=(r1, r1, r1), pow_=1.0, range_=(1.0, 1.0, 1.0)), "pos is required"),
        (dict(radius=((RN_MAX + 1) * res,) * 2 + (r1,), pow_=1.0), "too large (rank table)"),
    )
    for kw, msg in refusals:
        with pytest.raises(abi.MplxError) as e:
            env.update_potential_map(**kw)
        assert e.value.code == abi.MPLX_ERR_ARG and msg in str(e.value), (kw, str(e.value))
        assert env.launch_count() == launches
        for a, b in zip(env.read_map(), state):
            assert a.tobytes() == b.tobytes(), kw
        launches = env.launch_count()
    again = env.expand(nodes, want=WANT)
    assert again.count.tobytes() == exp.count.tobytes()
    emitted = (np.arange(exp.nU)[None, :] < exp.count[:, None]).reshape(-1)
    for f in ("succ", "cost", "action", "key"):
        assert getattr(again, f)[emitted].tobytes() == getattr(exp, f)[emitted].tobytes(), f
    # radius NULL and a ctx that never saw a map, through the raw ABI
    lib = env._lib
    rad = np.array([r1, r1, r1])
    assert lib.mplx_update_potential_map(env.handle, None, 1.0, None, None, 0.1, 0.0, None) == abi.MPLX_ERR_ARG
    h = C.c_void_p()
    abi.check(lib.mplx_create(3, 0, C.byref(h)))
    try:
        assert lib.mplx_update_potential_map(h, rad.ctypes.data, 1.0, None, None, 0.1, 0.0, None) == abi.MPLX_ERR_ARG
        assert b"mplx_set_map" in lib.mplx_last_error()
        path = np.zeros((2, 3))
        assert lib.mplx_set_search_region_path(h, path.ctypes.data, 2, rad.ctypes.data, 0, None) == abi.MPLX_ERR_ARG
        assert b"mplx_set_map" in lib.mplx_last_error()
    finally:
        lib.mplx_destroy(h)
    # the largest accepted radius is served on the same ctx right after the refusals
    big = dict(radius=(RN_MAX * res, RN_MAX * res, r1), pow_=1.0)
    from test_maps_inputs_restatement_vs_ref import restate_potential

    field = state[0]
    got = env.update_potential_map(**big)
    assert got.tobytes() == restate_potential(field, case.dims, case.origin, res, big["radius"], 1.0).tobytes()


def test_second_call_update_cells_and_null_output():
    """A second call takes the field's positive cells as sources (the reference's planner keeps the field as its
    map); a call after mplx_update_cells sees the new cells; out_map may be NULL."""
    from motion_primitive_library_b200 import abi

    for name in ("2d_pow2.0", "3d_pow0.5", "2d_int8"):
        case = POTENTIAL[name]
        env = gpu_env(case.grid(), case.dims, case.origin, case.res)
        once = run_field(env, case)
        assert once.tobytes() == case.restate().tobytes()
        twice = run_field(env, case)
        assert twice.tobytes() == case.restate(once).tobytes() and twice.tobytes() != once.tobytes(), name
        idx = np.array([0, 5, twice.size - 1, 5], dtype=np.int64)
        env.update_cells(idx, np.array([100, 0, 100, -1], dtype=np.int8))
        edited = twice.copy()
        edited[[0, twice.size - 1]] = 100
        edited[5] = -1
        np.testing.assert_array_equal(env.read_map()[0], edited)
        rad = np.ascontiguousarray(pad3(case.radius))
        abi.check(env._lib.mplx_update_potential_map(env.handle, rad.ctypes.data, case.pow_, None, None, 0.1, 0.0, None))
        want = case.restate(edited)
        assert env.read_map()[0].tobytes() == want.tobytes()
        same_device_state(env, gpu_env(want, case.dims, case.origin, case.res))


def test_big_map_matches_layerwise_statement():
    import scenarios as S

    g = big_grid()
    env = gpu_env(g, BIG["dims"], BIG["origin"], BIG["res"])
    got = env.update_potential_map(BIG["radius"])
    want = S.potential_from_map(g, BIG["dims"], BIG["res"], BIG["radius"])
    assert got.tobytes() == want.tobytes()
    assert (got > 0).sum() > 2 * (g > 0).sum()


def test_field_call_leaves_the_ctx_as_a_fresh_one_given_the_field():
    """After the call the ctx expands — through the auto rule, the register kernel and the fixed-point kernel — as
    a fresh ctx given the field as map and potential map, and both as the oracle with the weights that arrived."""
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 48)
    g = sc.grid().copy()
    g[::97] = -1
    rad, powv = (0.5, 0.5, 0.3), 2.0
    nodes = sc.frontier(1500, seed=4)
    for pw, gw in ((0.5, 0.0), (0.3, 0.4)):
        def make(grid):
            e = gpu_env(grid, sc.dim_cells, sc.origin, sc.res)
            e.set_control(sc.control)
            e.set_u(sc.U)
            e.set_v_max(sc.v_max)
            e.set_potential_weight(pw)
            e.set_gradient_weight(gw)
            return e

        env = make(g)
        field = env.update_potential_map(rad, powv)
        fresh = make(field)
        fresh.set_potential_map(field)
        same_device_state(env, fresh)
        orc = ob.OracleEnv(3, sc.control, sc.U, field, sc.dim_cells, sc.origin, sc.res, v_max=sc.v_max, potential=field,
                           potential_weight=pw, gradient_weight=gw).expand(nodes, nthreads=8)
        for k in (0, 2, 5):
            env.set_kernel(k)
            fresh.set_kernel(k)
            a, b = env.expand(nodes, want=WANT), fresh.expand(nodes, want=WANT)
            assert a.count.tobytes() == b.count.tobytes()
            emitted = (np.arange(a.nU)[None, :] < a.count[:, None]).reshape(-1)
            for f in ("succ", "cost", "action", "key", "lattice"):
                assert getattr(a, f)[emitted].tobytes() == getattr(b, f)[emitted].tobytes(), (k, f)
            st = assert_expansion_equal(a, orc)
            assert 0 < st["finite"] < st["successors"]


# ---- the search region ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(REGION))
def test_search_region_matches_restatement(name):
    case = REGION[name]
    env = gpu_env(np.zeros(int(np.prod(case.dims)), np.int8), case.dims, case.origin, case.res)
    before = env.launch_count()
    got = env.set_search_region_path(case.path, case.radius, case.dense)
    want = case.restate()
    assert got.tobytes() == want.tobytes(), (name, int(got.sum()), int(want.sum()))
    no_cells = not case.dense and len(case.path) < 2
    assert env.launch_count() - before == (0 if no_cells else REGION_LAUNCHES)
    if no_cells:
        assert got.sum() == 0  # everything is outside the region


def test_region_drives_expansion_and_stored_edges_in_3d():
    """The region installed by the path call gates the fixed-point expansion and mplx_edges_is_free exactly as
    the oracle given the returned bytes; a one-point sparse path (empty region) refuses every successor."""
    import scenarios as S
    from test_edges_oracle_vs_ref import edges_of

    sc = S.scaled(S.cfg_headline(), 48)
    nodes = sc.frontier(1500, seed=6)
    path = np.array([[-2.0, -2.0, -2.0], [0.0, 0.4, 0.2], [0.05, 0.45, 0.2], [2.0, 1.5, 2.2]])
    for pth, radius in ((path, (0.9, 0.7, 0.8)), (path[:1], (0.9, 0.7, 0.8))):
        env = gpu_env(sc.grid(), sc.dim_cells, sc.origin, sc.res)
        env.set_control(sc.control)
        env.set_u(sc.U)
        env.set_v_max(sc.v_max)
        region = env.set_search_region_path(pth, radius)
        oenv = ob.OracleEnv(3, sc.control, sc.U, sc.grid(), sc.dim_cells, sc.origin, sc.res, v_max=sc.v_max, region=region)
        orc = oenv.expand(nodes, nthreads=8)
        for k in (0, 5, 2):
            env.set_kernel(k)
            st = assert_expansion_equal(env.expand(nodes, want=WANT), orc, exact_cost=True)
        parents, actions, _ = edges_of(oenv, nodes, np.random.default_rng(2), extra=300)
        fo, co = oenv.edges_is_free(parents, actions)
        fg, cg = env.is_free_edges(parents, actions)
        np.testing.assert_array_equal(fg, fo)
        assert cg.tobytes() == co.tobytes()
        if len(pth) > 1:
            assert 0 < st["finite"] < st["successors"] and 0 < fo.sum() < fo.size and 0 < region.sum() < region.size
        else:
            assert st["finite"] == 0 and fo.sum() == 0 and region.sum() == 0
