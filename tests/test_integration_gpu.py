"""The drop-in boundary as compiled code: integration/env_map_b200.h (the subclass INTEGRATION.md §1 lists)
built against the UNMODIFIED reference planner (graph_search.h, planner_base.h, map_planner.h,
src/mpl_planner/map_planner.cpp: oracle/Makefile target _ref/libmplref_b200.so) and installed through the
reference's virtual MapPlanner::setMapUtil.  The reference's own A* then runs on the B200 env; validity, cost,
expansion count, closed set (lattice keys), open-set size and the action sequence must equal what the same
planner produces with its own env_map (oracle/_ref/libmplref_planner.so)."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb

ACC, JRK = 0x03, 0x07


def same(a, b):
    for k in ("valid", "expanded", "n_closed", "n_open", "n_actions"):
        assert a[k] == b[k], (k, a[k], b[k])
    assert a["cost"] == b["cost"]
    np.testing.assert_array_equal(a["closed"], b["closed"])
    np.testing.assert_array_equal(a["actions"], b["actions"])


needs_libs = pytest.mark.skipif(not (pb.ref_b200_available() and pb.ref_planner_available()),
                                reason="oracle/_ref not built (needs the reference sources at build time)")


@pytest.mark.gpu
@needs_libs
def test_reference_planner_on_b200_env_config1_corridor():
    """config 1: test/test_planner_2d.cpp on data/corridor.yaml."""
    c = fixtures.corridor()
    for eps in (1.0, 2.0):
        a = pb.make_args(2, ACC, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                         goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, eps=eps)
        ref = pb.plan_reference(a)
        assert ref["valid"] == 1 and ref["n_closed"] > 50
        same(pb.plan_reference_b200(a), ref)


@pytest.mark.gpu
@needs_libs
def test_reference_planner_on_b200_env_3d_voxel_maps():
    import scenarios as S

    for sc, max_num in ((S.scaled(S.cfg_headline(), 64), 3000), (S.scaled(S.cfg3(), 64), 400)):
        nodes = sc.frontier(16, seed=4, max_steps=0)
        for q in (0, 6):
            a = pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=nodes["pos"][q]),
                             goal=dict(pos=nodes["pos"][q + 1]), v_max=sc.v_max, a_max=sc.a_max, max_num=max_num)
            ref = pb.plan_reference(a)
            assert ref["n_closed"] > 10
            same(pb.plan_reference_b200(a), ref)


@needs_libs
def test_binding_refuses_without_gpu():
    """No CPU fallback behind the reference-side binding either: without a device the subclass's constructor
    throws (mplx_create fails) and the driver reports it."""
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    c = fixtures.corridor()
    a = pb.make_args(2, ACC, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                     goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pb.plan_reference_b200(a)
