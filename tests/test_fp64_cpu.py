"""CPU tests of float64 decompositions: loading and precision of the values, refusals, the byte accounting, and the
float64 tile shapes the GPU sweep reaches."""
import re

import numpy as np
import pytest
from scipy import sparse

from arrow_matrix_b200 import _lib, decomp, graphio, synth
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.engine import ArrowEngine, _LevelState
from tests import tile_dispatch as td
from tests.test_gpu_fp64 import KS as GPU_SWEEP_KS

W = 8


def _f64_decomposition(seed=3):
    """a two-level decomposition whose values are not representable in float32"""
    dec = synth.synth_decomposition(4, W, levels=2, perm_kind="random", seed=seed)
    rng = np.random.default_rng(seed)
    out = []
    for B, p in dec:
        B = sparse.csr_matrix(B, dtype=np.float64)
        B.data = rng.uniform(0.5, 1.5, B.nnz) / 3.0
        out.append((B, p))
    return out


def _values(blocks, dtype):
    return [decomp.arrow_rows(B, blocks.width, int(nb), True, 0, int(nb) * blocks.width, dtype=dtype)
            for (B, _), nb in zip(blocks.decomposition, blocks.n_blocks)]


def test_float64_values_are_kept(tmp_path):
    dec = _f64_decomposition()
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, W, True)
    blocks, n_blocks, _, _ = ArrowDecompositionMPI.load_decomposition_new(SelfComm(), base, W, True, np.float64)
    assert blocks.dtype == np.float64 and len(n_blocks) == 2
    for (B, _), (ip, idx, dat, dropped) in zip(dec, _values(blocks, np.float64)):
        assert dat.dtype == np.float64 and dropped == 0
        assert np.array_equal(dat, B.data) and np.array_equal(idx, B.indices)
        assert not np.array_equal(dat.astype(np.float32).astype(np.float64), dat)       # would not survive float32


def test_float32_files_are_upcast_exactly_and_missing_values_are_ones(tmp_path):
    dec = [(sparse.csr_matrix(B, dtype=np.float32), p) for B, p in _f64_decomposition(5)]
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, W, True)
    blocks, _, _, _ = ArrowDecompositionMPI.load_decomposition_new(SelfComm(), base, W, True, np.float64)
    for (B, _), (_, _, dat, _) in zip(dec, _values(blocks, np.float64)):
        assert dat.dtype == np.float64 and np.array_equal(dat, B.data.astype(np.float64))
    ones = str(tmp_path / "ones")
    graphio.save_decomposition_new(dec, ones, W, True, write_data=False)
    blocks, _, _, _ = ArrowDecompositionMPI.load_decomposition_new(SelfComm(), ones, W, True, np.float64)
    for (B, _), (_, _, dat, _) in zip(dec, _values(blocks, np.float64)):
        assert dat.dtype == np.float64 and dat.size == B.nnz and (dat == 1.0).all()
    # the float32 route is unchanged: the values stay float32
    blocks, _, _, _ = ArrowDecompositionMPI.load_decomposition_new(SelfComm(), base, W, True)
    assert blocks.dtype == np.float32
    assert all(v[2].dtype == np.float32 for v in _values(blocks, np.float32))


@pytest.mark.parametrize("datatype", [np.float16, np.int32])
def test_other_datatypes_are_rejected(tmp_path, datatype):
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(_f64_decomposition(), base, W, True)
    with pytest.raises(ValueError, match="float32 or float64"):
        ArrowDecompositionMPI.load_decomposition_new(SelfComm(), base, W, True, datatype)
    with pytest.raises(ValueError):
        _lib.element_type(datatype)


class _TwoRanks(SelfComm):
    def Get_size(self) -> int:
        return 2


def test_float64_on_two_ranks_is_refused_before_any_cuda_call(tmp_path, monkeypatch):
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(_f64_decomposition(), base, W, True)
    comm = _TwoRanks()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, W, True, np.float64)

    def no_cuda(*a, **k):
        raise AssertionError("a CUDA context was requested")
    monkeypatch.setattr(_lib.Context, "__init__", no_cuda)
    monkeypatch.setattr(_lib, "load_library", no_cuda)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, W, 4, 'gpu', True, True)
    with pytest.raises(ValueError, match="one GPU"):
        arrow.B.load_sparse_matrix_from_blocks(blocks)
    assert arrow._engine is None


def _accounting_engine(dtype, mode="exchange"):
    """an ArrowEngine shell with the state the accounting reads (no device)"""
    eng = object.__new__(ArrowEngine)
    eng.dtype, eng.k, eng.mode, eng.fused_style = np.dtype(dtype), 16, mode, "gather"
    rng = np.random.default_rng(1)
    eng.levels = []
    for j, (rows, nnz) in enumerate([(64, 700), (24, 130), (8, 31)]):
        st = _LevelState()
        st.rows, st.nnz = rows, nnz
        if j > 0:
            prev = eng.levels[-1].rows
            st.to_prev = np.where(rng.random(rows) < 0.7, rng.integers(0, prev, rows), 2 * prev)
        eng.levels.append(st)
    eng.L = len(eng.levels)
    return eng


def test_byte_accounting_uses_the_element_size():
    f32, f64 = _accounting_engine(np.float32), _accounting_engine(np.float64)
    k = f32.k
    # the float32 figures, written out the way they were before float64 existed: bit-identical
    old = 0.0
    for j, st in enumerate(f32.levels):
        old += st.nnz * 8 + (st.rows + 1) * 4 + 2.0 * st.rows * k * 4
        if j > 0:
            old += 5.0 * int(np.count_nonzero(st.to_prev < f32.levels[j - 1].rows)) * k * 4
    assert f32.algorithmic_bytes_per_step() == old
    # nnz*(4 + e) + (R+1)*4 + U*k*e + R*k*e, plus the exchanges, with e = 8
    new = 0.0
    for j, st in enumerate(f64.levels):
        new += st.nnz * 12 + (st.rows + 1) * 4 + 2.0 * st.rows * k * 8
        if j > 0:
            new += 5.0 * int(np.count_nonzero(st.to_prev < f64.levels[j - 1].rows)) * k * 8
    assert f64.algorithmic_bytes_per_step() == new
    for mode in ("exchange", "fused"):
        f32, f64 = _accounting_engine(np.float32, mode), _accounting_engine(np.float64, mode)
        st, nxt = f32.levels[0], f32.levels[1]
        routed = float(np.count_nonzero(nxt.to_prev < st.rows)) if mode == "fused" else 0.0
        assert f32.level_bytes(0) == st.nnz * 8 + (st.rows + 1) * 4 + 2.0 * st.rows * k * 4 + routed * k * 4
        assert f64.level_bytes(0) == st.nnz * 12 + (st.rows + 1) * 4 + 2.0 * st.rows * k * 8 + routed * k * 8


def f64_tile_shape(k: int):
    """(G, VPL) of the float64 tile kernel a launch with ``k`` columns runs (``launch_tiles_f64``): lanes per row and
    double2 per lane from k2 = k / 2"""
    assert k % 2 == 0 and 2 <= k <= 256
    k2 = k // 2
    vpl = 4 if k2 >= 32 else (2 if k2 >= 8 else 1)
    lanes = -(-k2 // vpl)
    g = 1
    while g < lanes:
        g <<= 1
    return g, vpl


def source_f64_shapes(path: str) -> set:
    """the TF(G, VPL) lines of ``launch_tiles_f64`` in the CUDA source"""
    with open(path) as f:
        src = f.read()
    body = src[src.index("int launch_tiles_f64(arrow_ctx *ctx"):]
    body = body[:body.index("#undef TF")]
    return {(int(m.group(1)), int(m.group(2))) for m in re.finditer(r"(?<![A-Z])TF\((\d+),\s*(\d+)\);", body)}


def test_float64_tile_shapes_are_all_reached_by_the_gpu_sweep():
    in_source = source_f64_shapes(td.SOURCE)
    reached = {f64_tile_shape(k) for k in GPU_SWEEP_KS if k % 2 == 0 and k <= 256}
    assert len(in_source) == 10 and reached == in_source, \
        f"unreached: {in_source - reached}, not in the source: {reached - in_source}"


def test_float64_tile_shape_restatement():
    """the widths either side of every shape boundary"""
    assert [f64_tile_shape(k) for k in (2, 4, 6, 8, 10, 16, 18, 32, 34, 62, 64, 66, 128, 130, 256)] == [
        (1, 1), (2, 1), (4, 1), (4, 1), (8, 1), (4, 2), (8, 2), (8, 2), (16, 2), (16, 2), (8, 4), (16, 4), (16, 4),
        (32, 4), (32, 4)]
