"""Incremental (LPA*) sessions end to end on the GPU env: libmpl_host.so's MapPlanner with
setLPAstar(true) — get_succ, the getLinkedNodes voxel walk (mplx_edges_cells) and decreaseCost's
is_free(pr) re-validation (mplx_edges_is_free) all on the device — against the SAME host planner
driven by the CPU oracle env, which tests/test_lpastar_vs_ref.py pins to the reference's own LPA*.
After every step the whole search state (hash over key, g, rhs, flags of every state), the
voxel->edges table, validity, cost and the trajectory must be identical."""
import numpy as np
import pytest

import planner_bindings as pb
from test_lpastar_vs_ref import corridor_args, same_session, trajectory_cells, voxel_script, voxel_session_args, wall_at

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("idx,half,speculate", [(5, 0, 1), (10, 2, 8), (20, 0, 1), (30, 2, 16)])
def test_corridor_block_clear_sessions(idx, half, speculate):
    a, c = corridor_args(speculate=speculate)
    first = pb.lpa_oracle(a, [("plan",)])[0]
    cells = trajectory_cells(c, first, every=1)
    wall = wall_at(cells, idx, half)
    script = [("plan",), ("link",), ("block", wall), ("plan",), ("link",), ("clear", wall), ("plan",),
              ("subtree", 2), ("plan",), ("link",), ("block", cells[:3]), ("clear", cells[:3]), ("plan",)]
    orc = pb.lpa_oracle(a, script)
    assert orc[0]["valid"] == 1 and orc[1]["n_linked"] > 1000
    same_session(pb.lpa_session(a, script), orc)


@pytest.mark.parametrize("which,q,speculate", [("acc", 0, 1), ("acc", 4, 16), ("jrk", 2, 4)])
def test_voxel_map_sessions(which, q, speculate):
    import scenarios as S

    sc, maxn = (S.scaled(S.cfg_headline(), 64), 4000) if which == "acc" else (S.scaled(S.cfg3(), 48), 600)
    a = voxel_session_args(sc, q, maxn)
    a.speculate = speculate
    first = pb.lpa_oracle(a, [("plan",)])[0]
    assert first["valid"] == 1
    script = voxel_script(sc, a, first)
    orc = pb.lpa_oracle(a, script)
    assert orc[1]["n_linked"] > 100
    same_session(pb.lpa_session(a, script), orc)


def test_reference_session_if_available():
    """The GPU session against the reference's LPA* directly (or its recorded results)."""
    a, c = corridor_args()
    first = pb.lpa_reference(a, [("plan",)])[0]
    cells = trajectory_cells(c, first, every=1)
    wall = wall_at(cells, 10, 1)
    script = [("plan",), ("link",), ("block", wall), ("plan",), ("link",), ("clear", wall), ("plan",)]
    same_session(pb.lpa_session(a, script), pb.lpa_reference(a, script))
