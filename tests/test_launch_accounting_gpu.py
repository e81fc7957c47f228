"""mplx_launch_count after mplx_expand_packed: every chunk of the pipeline adds the launches of its expansion
(tests/test_fx_paths_gpu.py, launches_expected) and one for pack_kernel.  On occupancy planning a chunk of at
least 64*256 primitive slots runs expand_fxn_kernel + fx_resolve_kernel + pack_kernel, a smaller one
expand_fx_kernel + pack_kernel."""
from __future__ import annotations

import os

import pytest

import test_fx_paths_gpu as fx
from test_expand_parity_gpu import gpu_env

pytestmark = pytest.mark.gpu

CHUNK_LOG2 = 18  # MPLX_PACK_CHUNK_LOG2: chunks of 2^18 successor slots


def test_packed_launches_per_chunk():
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 96)
    nU = len(sc.U)
    chunk = (1 << CHUNK_LOG2) // nU
    # six full chunks and a last one below the fxn threshold
    tail = fx.FXN_MIN_SLOTS // nU // 2
    n = 6 * chunk + tail
    nodes = sc.frontier(n, seed=21)
    chunks = [min(chunk, n - off) for off in range(0, n, chunk)]
    assert len(chunks) == 7 and chunks[-1] == tail
    per_chunk = [fx.launches_expected(0, m, nU) + 1 for m in chunks]
    assert per_chunk == [3] * 6 + [2]
    env = gpu_env(sc)
    env.set_kernel(0)
    env._sync_params()
    os.environ["MPLX_PACK_CHUNK_LOG2"] = str(CHUNK_LOG2)
    try:
        for drop in (False, True):
            before = env.launch_count()
            p = env.expand_packed(nodes, drop_inf=drop)
            assert env.launch_count() - before == sum(per_chunk), drop
            assert p["total"] > 0
    finally:
        os.environ.pop("MPLX_PACK_CHUNK_LOG2", None)
