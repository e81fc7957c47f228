"""End-to-end: MPL::MapPlanner::plan() with the GPU env (libmpl_host.so -> libmplx.so) must
expand exactly the nodes the same planner expands with the CPU oracle env: identical closed
sets (lattice keys), expansion counts, trajectory costs and action sequences — with and without
speculative batching (speculation must not change the expanded set)."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb
from reference_record import same_array

pytestmark = pytest.mark.gpu
ACC, JRK, ACCxYAW = 0x03, 0x07, 0x13


def check_same(args_factory, speculations=(1, 16)):
    ref = pb.plan_oracle(args_factory(1))
    # ... and the REFERENCE's own MapPlanner::plan() (oracle/_ref, unmodified sources, or its recorded results) agrees with both
    r0 = pb.plan_reference(args_factory(1))
    assert r0["valid"] == ref["valid"] and r0["n_closed"] == ref["n_closed"]
    same_array(r0["closed"], ref["closed"], "closed")
    same_array(r0["actions"], ref["actions"], "actions")
    for k in speculations:
        g = pb.plan_gpu(args_factory(k))
        assert g["valid"] == ref["valid"]
        assert g["expanded"] == ref["expanded"]
        assert g["n_closed"] == ref["n_closed"] and g["n_open"] == ref["n_open"]
        np.testing.assert_array_equal(g["closed"], ref["closed"])
        np.testing.assert_array_equal(g["actions"], ref["actions"])
        if ref["valid"]:
            assert g["cost"] == pytest.approx(ref["cost"], rel=1e-6)
        assert g["gpu_nodes"] >= g["expanded"] and g["gpu_launches"] >= 1
        if k > 1 and ref["expanded"] > 200:
            assert g["gpu_calls"] < g["expanded"], "speculation should batch several nodes per launch"
    return ref


def test_config1_test_planner_2d_corridor():
    """BASELINE.json configs[0]: test/test_planner_2d.cpp (ACC, 9 primitives) on data/corridor.yaml."""
    c = fixtures.corridor()

    def f(k):
        return pb.make_args(2, ACC, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(),
                            start=dict(pos=c["start"]), goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, speculate=k)

    ref = check_same(f)
    assert ref["valid"] == 1 and ref["expanded"] > 100


def test_corridor_with_yaw():
    """test/test_planner_2d_with_yaw.cpp: ACCxYAW, 27 primitives, yaw_max 0.7."""
    c = fixtures.corridor()

    def f(k):
        return pb.make_args(2, ACCxYAW, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d_yaw(),
                            start=dict(pos=c["start"]), goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, yaw_max=0.7,
                            speculate=k, max_num=4000)

    check_same(f, speculations=(8,))


def test_3d_acc_and_jrk_voxel_maps():
    import scenarios as S

    for sc, maxn in ((S.scaled(S.cfg_headline(), 96), 3000), (S.scaled(S.cfg3(), 64), 600)):
        grid = sc.grid()
        nodes = sc.frontier(64, seed=12, max_steps=0)  # free cell centres at rest
        d = np.abs(nodes["pos"][:, None, :] - nodes["pos"][None, :, :]).max(-1)
        i, j = np.unravel_index(np.argmax(d), d.shape)

        def f(k):
            return pb.make_args(3, sc.control, grid, sc.dim_cells, sc.origin, sc.res, sc.U,
                                start=dict(pos=nodes["pos"][i]), goal=dict(pos=nodes["pos"][j]), v_max=sc.v_max,
                                a_max=sc.a_max, T=sc.T, w=sc.w, speculate=k, max_num=maxn)

        ref = check_same(f, speculations=(1, 32))
        assert ref["expanded"] > 50
