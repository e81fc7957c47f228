"""Every refusal of the batched device searches (mplx_plan_batch, mplx_plan_batch_cost_terms, mplx_plan_batch_grow and
the two _fits calls): its return code, its message, no kernel launch and no output written.  Rows with two faults pin
which one each call reports."""
import ctypes as C

import numpy as np
import pytest

import fixtures
from motion_primitive_library_b200 import abi

pytestmark = pytest.mark.gpu
ACC, ACCxYAW = 0x03, 0x13
SENT = 7
NQ_ALLOC, MX_ALLOC = 4, 50
BOUNDED, GROW, FITS = ("batch", "cost"), ("grow",), ("fits", "cost_fits")
ALL = BOUNDED + GROW + FITS
FN = dict(batch="mplx_plan_batch", cost="mplx_plan_batch_cost_terms", grow="mplx_plan_batch_grow",
          fits="mplx_plan_batch_fits", cost_fits="mplx_plan_batch_cost_terms_fits")
ARG, ALLOC = abi.MPLX_ERR_ARG, abi.MPLX_ERR_ALLOC

# (case, calls, ctx kind, call arguments, code, message substring)
CASES = [
    ("null_ctx", ALL, None, {}, ARG, "null ctx"),
    ("no_map", ALL, "bare", {}, ARG, "map or params not set"),
    ("potential", ("batch", "grow", "fits"), "pot", {}, ARG, "a potential map is installed"),
    ("yaw", ("batch", "grow", "fits"), "yaw", {}, ARG, "yaw controls take mplx_plan_batch_cost_terms"),
    ("max_expand_0", BOUNDED + FITS, "occ", dict(mx=0), ARG, "max_expand must be > 0"),
    ("max_expand_neg", BOUNDED + FITS, "occ", dict(mx=-3), ARG, "max_expand must be > 0"),
    ("wide", ALL, "wide", {}, ARG, "nU > 256"),
    ("null_out", BOUNDED + GROW, "occ", dict(out=False), ARG, "null out"),
    ("n_q_neg", BOUNDED + GROW, "occ", dict(nq=-1), ARG, "bad query arrays"),
    ("n_q_neg", FITS, "occ", dict(nq=-1), ARG, "n_q < 0"),
    ("null_starts", BOUNDED + GROW, "occ", dict(starts=False), ARG, "bad query arrays"),
    ("no_valid", BOUNDED + GROW, "occ", dict(drop="valid"), ARG, "missing output array"),
    ("no_actions", BOUNDED, "occ", dict(drop="actions"), ARG, "missing output array"),
    ("no_searched", GROW, "occ", dict(drop="searched"), ARG, "missing output array"),
    ("no_closed_offset", BOUNDED, "occ", dict(drop="closed_offset"), ARG, "closed_offset missing"),
    ("small_capacity", BOUNDED, "occ", dict(cap=3 * MX_ALLOC - 1), ARG, "capacities below n_q*max_expand"),
    ("cost_terms_2", GROW, "occ", dict(ct=2), ARG, "cost_terms must be 0 or 1"),
    ("first_cap_neg", GROW, "occ", dict(first_cap=-1), ARG, "first_cap, max_cap and pool_bytes must be >= 0"),
    ("tunnels", ALL, "tun", {}, ARG, "mplx_set_batch_regions set 2 tunnels"),
    # a worst-case arena beyond any budget; the capacities are only read, never written to, before the refusal
    ("budget", BOUNDED + FITS, "occ", dict(mx=10 ** 9, cap=3 * 10 ** 9), ALLOC, "exceed the budget"),
    # two faults: the first one each call checks is reported
    ("no_map+null_out", BOUNDED + GROW, "bare", dict(out=False), ARG, "map or params not set"),
    ("null_out+n_q_neg", BOUNDED + GROW, "occ", dict(out=False, nq=-1), ARG, "null out"),
    ("n_q_neg+no_valid", BOUNDED + GROW, "occ", dict(nq=-1, drop="valid"), ARG, "bad query arrays"),
    ("no_valid+small_capacity", BOUNDED, "occ", dict(drop="valid", cap=1), ARG, "missing output array"),
    ("no_closed_offset+small_capacity", BOUNDED, "occ", dict(drop="closed_offset", cap=1), ARG,
     "closed_offset missing"),
    ("no_valid+first_cap_neg", GROW, "occ", dict(drop="valid", first_cap=-1), ARG, "missing output array"),
    ("cost_terms_2+no_map", GROW, "bare", dict(ct=2), ARG, "cost_terms must be 0 or 1"),
    ("max_expand_0+n_q_neg", BOUNDED + FITS, "occ", dict(mx=0, nq=-1), ARG, "max_expand must be > 0"),
    ("no_valid+tunnels", BOUNDED + GROW, "tun", dict(drop="valid"), ARG, "missing output array"),
    ("small_capacity+tunnels", BOUNDED, "tun", dict(cap=1), ARG, "capacities below n_q*max_expand"),
    ("first_cap_neg+tunnels", GROW, "tun", dict(first_cap=-1), ARG, "first_cap, max_cap and pool_bytes"),
    ("tunnels+budget", BOUNDED + FITS, "tun", dict(mx=10 ** 9, cap=3 * 10 ** 9), ARG, "set 2 tunnels"),
]
ROWS = [pytest.param(call, kind, kw, code, msg, id=f"{call}-{case}")
        for case, calls, kind, kw, code, msg in CASES for call in calls]


def make_ctx(kind):
    """A libmplx ctx of `kind`: bare (no map), occ (occupancy planning), pot (a potential map), yaw (a yaw
    control), wide (300 primitives) or tun (occupancy planning with 2 per-query tunnels).  Returns (handle, env)."""
    from motion_primitive_library_b200 import MapUtil, env_map

    if kind == "bare":
        h = C.c_void_p()
        assert abi.load().mplx_create(2, 0, C.byref(h)) == abi.MPLX_OK
        return h, None
    c = fixtures.corridor()
    mu = MapUtil()
    mu.setMap(c["origin"], c["dim"], c["grid"], c["res"])
    e = env_map(mu, device=0)
    if kind == "yaw":
        e.set_control(ACCxYAW)
        e.set_u(fixtures.U_2d_yaw())
    else:
        e.set_control(ACC)
        e.set_u(np.array([[0.01 * i, 0.0] for i in range(300)]) if kind == "wide" else fixtures.U_2d())
    e.set_dt(1.0)
    e.set_w(10.0)
    e.set_v_max(1.0)
    e.set_a_max(1.0)
    if kind == "pot":
        e.set_potential_map(np.zeros(c["grid"].size, np.int8))
    if kind == "tun":
        path = np.array([np.asarray(c["start"])[:2], np.asarray(c["goal"])[:2]])
        e.set_batch_regions([path, path], np.array([1.0, 1.0]))
    e._sync_params()
    return e.handle, e


def call_with_sentinels(lib, call, h, nq=3, mx=MX_ALLOC, starts=True, out=True, drop=None, cap=None, ct=0,
                        first_cap=0):
    """One call with every output filled with SENT: (rc, outputs)."""
    S = np.zeros(NQ_ALLOC, dtype=abi.WAYPOINT_DTYPE)
    sp = S.ctypes.data if starts else None
    n, m = NQ_ALLOC, NQ_ALLOC * MX_ALLOC
    if call in FITS:
        slots, nbytes = C.c_int32(SENT), C.c_int64(SENT)
        fn = lib.mplx_plan_batch_fits if call == "fits" else lib.mplx_plan_batch_cost_terms_fits
        rc = fn(h, nq, mx, 1, C.byref(slots), C.byref(nbytes))
        return rc, dict(meta=np.array([slots.value, nbytes.value]))
    o = dict(valid=np.full(n, SENT, np.int32), cost=np.full(n, float(SENT)), expanded=np.full(n, SENT, np.int32),
             n_closed=np.full(n, SENT, np.int32))
    p = lambda k: None if k == drop else o[k].ctypes.data  # noqa: E731
    if call in BOUNDED:
        o.update(action_offset=np.full(n + 1, SENT, np.int64), actions=np.full(m, SENT, np.int32),
                 closed_offset=np.full(n + 1, SENT, np.int64), closed_keys=np.full(m, SENT, np.uint64))
        bo = abi.BatchOut(p("valid"), p("cost"), p("expanded"), p("n_closed"), p("action_offset"), p("actions"),
                          m if cap is None else cap, p("closed_offset"), p("closed_keys"), m if cap is None else cap,
                          SENT, SENT, float(SENT))
        fn = lib.mplx_plan_batch if call == "batch" else lib.mplx_plan_batch_cost_terms
        rc = fn(h, sp, sp, None, nq, 1.0, mx, 0.5, -1.0, -1.0, -1.0, C.byref(bo) if out else None)
        o["meta"] = np.array([bo.slots, bo.arena_bytes, bo.seconds])
    else:
        o.update(n_actions=np.full(n, SENT, np.int32), searched=np.full(n, SENT, np.int32))
        go = abi.GrowOut(p("valid"), p("cost"), p("expanded"), p("n_closed"), p("n_actions"), p("searched"),
                         SENT, SENT, SENT, SENT, SENT, SENT, float(SENT))
        rc = lib.mplx_plan_batch_grow(h, ct, sp, sp, None, nq, 1.0, mx, 0.5, -1.0, -1.0, -1.0, 1, first_cap, 0, 0,
                                      C.byref(go) if out else None)
        o["meta"] = np.array([go.rounds, go.slots, go.first_cap, go.last_cap, go.arena_bytes, go.reruns, go.seconds])
    return rc, o


@pytest.mark.parametrize("call,kind,kw,code,msg", ROWS)
def test_refusal(call, kind, kw, code, msg):
    lib = abi.load()
    h, e = make_ctx(kind) if kind else (None, None)
    try:
        n0 = lib.mplx_launch_count(h) if h else 0
        rc, o = call_with_sentinels(lib, call, h, **kw)
        err = lib.mplx_last_error().decode()
        assert rc == code, err
        assert err.startswith(FN[call] + ":") and msg in err, err
        assert all((v == SENT).all() for v in o.values())
        if h:
            assert lib.mplx_launch_count(h) == n0
    finally:
        if e is not None:
            e.close()
        elif h:
            lib.mplx_destroy(h)
