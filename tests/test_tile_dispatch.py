"""The Python restatement of the tile dispatch (tests/tile_dispatch.py) against the CUDA source it restates: the
GPU sweep chooses its cases from the restatement, so the two must not drift apart unnoticed."""
import numpy as np

from tests import tile_dispatch as td


def test_mirror_reaches_exactly_the_instances_in_the_source():
    src = td.source_instantiations()
    mirror = td.reachable_instantiations()
    assert len(src) > 250, f"parsed only {len(src)} instances from launch_tiles (line {td.tile_args_line()})"
    assert mirror == src, (f"only in the source: {sorted(map(str, src - mirror))[:8]}; "
                           f"only in the mirror: {sorted(map(str, mirror - src))[:8]}")


def test_dispatch_examples():
    # k = 128: 8 lanes x 4 float4, small tiles, round-1 kernel for the plain launch
    assert td.tile_instantiation(128) == td.Inst("v1", 8, 4, 64, td.OUT_IDENTITY, False, 1, False)
    # k = 20 (k4 = 5): big tiles, 8 lanes of one float4 of which three idle (not exact)
    assert td.tile_instantiation(20, td.OUT_ROWMAP, True) == td.Inst("v1", 8, 1, 128, td.OUT_ROWMAP, True, 1, False)
    assert td.tile_instantiation(20, big_tiles=0, tile_kernel=0) == td.Inst("gen", 8, 1, 64, td.OUT_IDENTITY, False, 1,
                                                                            False)
    assert td.tile_instantiation(16, rpg_req=2).RPG == 2
    assert td.tile_instantiation(16, td.OUT_ROWMAP, rpg_req=2).RPG == 1       # pairs exist for plain launches only
    assert td.spmm_kernels(10) == ["generic<ROWMAP=0,ACC=0>"]
    assert td.spmm_kernels(64, variant=2, rowmap=True) == ["tma<VPL=1,ROWMAP=1,ACC=0>"]
    assert td.spmm_kernels(256, variant=1, acc=True) == ["shfl<G=32,VPL=2,ROWMAP=0,ACC=1>"]
    assert td.spmm_kernels(64, variant=0, fused_operands=True, n_long_tasks=2)[1:] == ["long_partial",
                                                                                   "long_reduce<ROWMAP=0,ACC=0>"]


def test_build_tiles_caps():
    rng = np.random.default_rng(0)
    lens = rng.integers(250, 511, size=300)
    lens[17] = 513                                       # long: cut around, not tiled
    ip = np.concatenate([[0], np.cumsum(lens)])
    for rows_cap, nnz_cap in ((td.TILE_ROWS, td.TILE_NNZ), (td.TILE_ROWS_BIG, td.TILE_NNZ_BIG)):
        t = td.build_tiles(ip, rows_cap, nnz_cap)
        assert 17 not in np.concatenate([np.arange(a, b) for a, b, _, _ in t])
        assert (t[:, 3] - t[:, 2] <= nnz_cap - 4).all() and (t[:, 1] - t[:, 0] <= rows_cap).all()
        assert (t[:, 1] - t[:, 0]).max() <= nnz_cap // 250                 # the nnz cap binds, not the row cap
        assert set(np.unique(t[:, 2] % 4)) == {0, 1, 2, 3}                   # every alignment of the first entry
