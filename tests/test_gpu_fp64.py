"""float64 decompositions on one GPU: every float64 kernel against the extended-precision bound of
tests/spmm_bound64.py, the refusals of mixed or multi-GPU launches, the engine in both modes and the reference surface.

Operands: X tiles are longer than the block's column count and every X row no entry reads is NaN, addend rows no row
adds are NaN, and C holds NaN (or, for accumulate, finite values) in rows the launch must not write, with extra rows
past the block: a stray read shows up as NaN in the output, a stray write as a changed unwritten row.
"""
import numpy as np
import pytest
from scipy import sparse

from arrow_matrix_b200 import _lib, graphio, synth
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.engine import ArrowEngine
from oracle import oracle
from tests import spmm_bound64 as sb
from tests import tile_dispatch as td
from tests.golden_util import GPU_CASES, GoldenCase
from tests.step_bound import abs_decomposition, bound_of, step_height
from tests.test_gpu_kernels import assert_close

pytestmark = pytest.mark.gpu

# every float64 tile shape (tests/test_fp64_cpu.py pins them to launch_tiles_f64), the generic kernel (k odd or > 256)
# and both sides of its boundary; 34 and 62 run TF(16, 2), at 62 with the last lane's second double2 as padding
KS = [1, 2, 3, 4, 6, 8, 10, 16, 30, 32, 34, 62, 64, 126, 128, 256, 258, 512]
GRIDS = {"1 CTA": (1, 1), "default": (0, 0)}          # (SPMM_SM_LIMIT, SPMM_CTAS_PER_SM)
ERR_ARG, ERR_UNSUPPORTED = -2, -6


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(cuda_device)
    yield c
    c.close()


def _grid(ctx, name):
    sm, per = GRIDS[name]
    ctx.set_option(_lib.Context.OPT_SPMM_SM_LIMIT, sm)
    ctx.set_option(_lib.Context.OPT_SPMM_CTAS_PER_SM, per)


def _nan_except(rows, k, keep, rng):
    out = np.full((rows, k), np.nan)
    keep = np.unique(keep)
    out[keep] = rng.uniform(-1, 1, (keep.size, k)) * 10.0 ** rng.uniform(-2, 2, (keep.size, 1))
    return out


def _ragged_block(rng):
    """20k rows: short ragged rows, empty rows, and hub rows above the long-row threshold (one and three segments)"""
    n = 20000
    lens = rng.integers(0, 24, n)
    lens[rng.integers(0, n, 300)] = 0
    lens[[7, 9000]] = [600, 5000]
    lens[15000:15004] = [513, 2048, 2049, 4100]
    return sb.ragged_csr64(lens, n, rng)


class Problem:
    """one float64 block and the operands of every epilogue at one k"""

    def __init__(self, ctx, A, k, seed, threshold=td.LONG_THRESHOLD, segment=td.LONG_SEGMENT):
        rng = np.random.default_rng(seed)
        self.ctx, self.A, self.k = ctx, A, k
        self.threshold, self.segment = threshold, segment          # the long-row tuning the block was uploaded under
        n, nc = A.shape
        self.n = n
        used = np.unique(A.indices)
        self.Xh = _nan_except(nc + 5, k, used, rng)
        self.Cold = rng.standard_normal((n + 3, k))
        self.Cnan = np.full((n + 3, k), np.nan)
        self.rm = rng.permutation(n + 3)[:n].astype(np.int64)
        self.rm[::9] = -1
        n_add = n // 2 + 4
        self.amap = np.where(rng.random(n) < 0.6, rng.integers(0, n_add, n), -1).astype(np.int64)
        self.addh = _nan_except(n_add, k, self.amap[self.amap >= 0], rng)
        self.cmap = rng.permutation(nc + 5)[:nc].astype(np.int64)
        self.cmap[::5] = -1                                    # entries whose image is invalid: skipped
        img = self.cmap[used]
        self.Xsh = _nan_except(nc + 7, k, img[img >= 0], rng)
        f64 = np.float64
        self.dA = ctx.csr_upload(n, nc, A.indptr, A.indices, A.data, dtype=f64)
        self.dAs = self.dA.remap_columns(ctx.map_upload(self.cmap, nc + 5), nc + 5)
        self.dm = ctx.map_upload(self.rm, n + 3)
        self.dam = ctx.map_upload(self.amap, n_add)
        self.dX = ctx.dense_from_host(self.Xh, f64)
        self.dXs = ctx.dense_from_host(self.Xsh, f64)
        self.dadd = ctx.dense_from_host(self.addh, f64)
        self.dC = ctx.dense_alloc(n + 3, k, f64)
        self.P = sb.products(A, self.Xh)
        self.Ps = sb.products(A, self.Xsh[: nc + 5], col_map=self.cmap)

    def run(self, epi):
        """launch one epilogue; returns (device result, expectation)"""
        ctx, P = self.ctx, self.P
        acc = epi in ("acc", "rowmap_acc", "skip")
        before = self.Cold if acc else self.Cnan
        self.dC.h2d(before)
        rowmap = self.rm if epi in ("rowmap", "rowmap_acc", "skip") else None
        tuning = dict(threshold=self.threshold, segment=self.segment)
        if epi == "add":
            ctx.spmm_add(self.dA, self.dX, self.dC, self.dadd, self.dam)
            e = sb.reference(P, before, add=self.addh, add_map=self.amap, label=f"k={self.k} {epi}", **tuning)
        elif epi == "skip":
            ctx.spmm(self.dAs, self.dXs, self.dC, rowmap=self.dm, accumulate=True)
            e = sb.reference(self.Ps, before, rowmap=rowmap, accumulate=True, label=f"k={self.k} {epi}", **tuning)
        else:
            ctx.spmm(self.dA, self.dX, self.dC, rowmap=self.dm if rowmap is not None else None, accumulate=acc)
            e = sb.reference(P, before, rowmap=rowmap, accumulate=acc, label=f"k={self.k} {epi}", **tuning)
        return self.dC.d2h(), e

    def free(self):
        for h in (self.dAs, self.dA, self.dm, self.dam, self.dX, self.dXs, self.dadd, self.dC):
            h.free()


EPILOGUES = ["plain", "acc", "rowmap", "rowmap_acc", "add", "skip"]


@pytest.fixture(scope="module")
def ragged():
    return _ragged_block(np.random.default_rng(64))


@pytest.mark.parametrize("k", KS)
def test_kernel_sweep_ragged_block(ctx, ragged, k):
    """every float64 kernel (tile for even k <= 256, generic otherwise, long rows) under every epilogue, at one CTA
    walking every tile and at the default grid; the tile path is bit-identical across grids"""
    pr = Problem(ctx, ragged, k, seed=k)
    assert pr.dA.info()["n_long_rows"] == 6
    try:
        for epi in EPILOGUES:
            results = {}
            for grid in GRIDS:
                _grid(ctx, grid)
                got, e = pr.run(epi)
                sb.assert_spmm64(got, e)
                results[grid] = got
            a, b = results.values()
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), f"k={k} {epi}: grids differ"
    finally:
        _grid(ctx, "default")
        pr.free()


def _boundary_blocks(rng):
    """tile-boundary shapes: no entry at all, 1..129 rows, and tiles whose first entry has every alignment mod 4"""
    yield "nnz=0", sparse.csr_matrix((50, 60), dtype=np.float64)
    for n in (1, 2, 63, 64, 65, 127, 128, 129):
        yield f"{n} rows", sb.ragged_csr64(rng.integers(0, 40, n), 300, rng)
    lens = rng.integers(250, 511, size=60)                  # ~2-4 rows per tile: first entries at every alignment
    yield "aligned", sb.ragged_csr64(lens, 4000, rng)


@pytest.mark.parametrize("k", [2, 6, 128, 5])
def test_tile_boundary_shapes(ctx, k):
    rng = np.random.default_rng(7 + k)
    for label, A in _boundary_blocks(rng):
        if label == "aligned":
            t = td.build_tiles(A.indptr, td.TILE_ROWS, td.TILE_NNZ)
            assert set(np.unique(t[:, 2] % 4)) == {0, 1, 2, 3}
        pr = Problem(ctx, A, k, seed=k)
        try:
            for epi in EPILOGUES:
                for grid in GRIDS:
                    _grid(ctx, grid)
                    got, e = pr.run(epi)
                    e.label = f"{label} {e.label} {grid}"
                    sb.assert_spmm64(got, e)
        finally:
            _grid(ctx, "default")
            pr.free()


@pytest.mark.parametrize("k", [3, 8, 128])
def test_gather_rows_float64_bit_exact(ctx, k):
    rng = np.random.default_rng(k)
    src = rng.standard_normal((300, k)) / 3.0
    dst0 = rng.standard_normal((250, k)) / 7.0
    m = np.where(rng.random(250) < 0.8, rng.permutation(300)[:250], -1).astype(np.int64)
    dS = ctx.dense_from_host(src, np.float64)
    dD = ctx.dense_from_host(dst0, np.float64)
    dm = ctx.map_upload(m, 300)
    ok = m >= 0
    for acc in (False, True):
        dD.h2d(dst0)
        ctx.gather_rows(dD, dS, dm, accumulate=acc)
        want = dst0.copy()
        want[ok] = (dst0[ok] + src[m[ok]]) if acc else src[m[ok]]
        got = dD.d2h()
        assert got.dtype == np.float64 and np.array_equal(got.view(np.uint64), want.view(np.uint64))
    for h in (dS, dD, dm):
        h.free()


def _code(fn):
    with pytest.raises(_lib.ArrowError) as e:
        fn()
    return e.value.code


def test_mixed_and_multi_gpu_launches_are_refused(ctx):
    rng = np.random.default_rng(0)
    A = sb.ragged_csr64(rng.integers(1, 9, 64), 64, rng)
    k = 8
    A64 = ctx.csr_upload(64, 64, A.indptr, A.indices, A.data, dtype=np.float64)
    A32 = ctx.csr_upload(64, 64, A.indptr, A.indices, A.data)
    X64, C64, S64 = (ctx.dense_alloc(64, k, np.float64) for _ in range(3))
    X32, C32, S32 = (ctx.dense_alloc(64, k) for _ in range(3))
    assert X64.device_dtype() == np.float64 and X32.device_dtype() == np.float32
    m = ctx.map_upload(np.arange(64), 64)
    assert _code(lambda: ctx.spmm(A64, X32, C64)) == ERR_ARG
    assert _code(lambda: ctx.spmm(A64, X64, C32)) == ERR_ARG
    assert _code(lambda: ctx.spmm(A32, X64, C64)) == ERR_ARG
    assert _code(lambda: ctx.spmm_add(A64, X64, C64, S32, m)) == ERR_ARG
    assert _code(lambda: ctx.spmm_add(A32, X32, C32, S64, m)) == ERR_ARG
    assert _code(lambda: ctx.gather_rows(C64, X32, m)) == ERR_ARG
    assert _code(lambda: ctx.gather_rows(C32, X64, m, accumulate=True)) == ERR_ARG
    assert _code(lambda: C64.copy_from(X32)) == ERR_ARG
    X2 = ctx.dense_alloc(64, k, np.float64)
    assert _code(lambda: ctx.spmm_ex(A64, X64, C64, X2=X2, x_split=32)) == ERR_UNSUPPORTED
    tab = ctx.ptrtable_upload([C32], np.zeros(64, np.int32), np.arange(64))
    assert _code(lambda: ctx.spmm_ex(A64, X64, None, out_table=tab)) == ERR_UNSUPPORTED
    assert _code(lambda: ctx.ptrtable_upload([C64], np.zeros(64, np.int32), np.arange(64))) == ERR_UNSUPPORTED
    for variant in (_lib.VARIANT_DIRECT, _lib.VARIANT_SHFL, _lib.VARIANT_TMA, _lib.VARIANT_TILES | (2 << 4)):
        assert _code(lambda: ctx.spmm(A64, X64, C64, variant=variant)) == ERR_UNSUPPORTED
    ctx.spmm(A64, X64, C64, variant=_lib.VARIANT_TILES)        # the default kernel named explicitly is fine
    ctx.sync()
    for h in (tab, m, X2, X64, C64, S64, X32, C32, S32, A64, A32):
        h.free()


# ---- the engine ----------------------------------------------------------------------------------------------------
def _bound64(mag, m):
    """tests/step_bound.py's per-element step bound at the float64 unit roundoff"""
    return bound_of(mag, m, u=sb.U64, eta=sb.ETA64, u_ref=sb.ULD)


def _check_engine_steps(eng, dec, width, k, block_diagonal, X0, steps=3):
    """``steps`` chained steps, each against the extended-precision oracle started from the device's state"""
    po = oracle.ReferenceProtocolOracle(dec, width, k, block_diagonal=block_diagonal, n_blocks=eng.n_blocks,
                                        dtype=np.longdouble)
    pa = oracle.ReferenceProtocolOracle(abs_decomposition(dec), width, k, block_diagonal=block_diagonal,
                                        n_blocks=eng.n_blocks, dtype=np.longdouble)
    m = step_height(po)
    eng.set_features(X0)
    for it in range(steps):
        x = eng.features(0).astype(np.longdouble) if it else X0.astype(np.longdouble)
        po.set_features(x)
        pa.set_features(np.abs(x))
        if eng.mode == "exchange":                     # rows behind the sentinel carry the device's previous results
            for j in range(1, eng.L):
                c = eng.result(j).astype(np.longdouble)
                po.C[j], pa.C[j] = c, np.abs(c)
        eng.step()
        got = eng.result()
        assert got.dtype == np.float64
        exact, mag = po.step(), pa.step()
        bound = _bound64(mag, m)
        err = np.abs(got.astype(np.longdouble) - exact).astype(np.float64)
        bad = ~(err <= bound)
        assert not bad.any(), (f"step {it} ({eng.mode}): {int(bad.sum())} elements outside the bound, worst ratio "
                               f"{float(np.max(err / np.where(bound > 0, bound, 1e-300))):.3g}")
    return got


@pytest.mark.parametrize("name", GPU_CASES)
def test_engine_float64_golden_decompositions(cuda_device, name):
    g = GoldenCase(name)
    rng = np.random.default_rng(11)
    for mode in ("auto", "exchange"):
        eng = ArrowEngine(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, device=cuda_device, mode=mode,
                          dtype=np.float64)
        X0 = g.X[0] if g.X[0] is not None else rng.uniform(-1, 1, (eng.n_rows, g.k))
        _check_engine_steps(eng, g.decomposition, g.width, g.k, g.block_diagonal, np.asarray(X0, np.float64))
        eng.close()
    # the float64 run of the reference's own schedule meets the float32 parity rule against its outputs
    eng = ArrowEngine(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, device=cuda_device, mode="exchange",
                      dtype=np.float64)
    for it in range(g.iterations):
        if g.X[it] is not None:
            eng.set_features(g.X[it])
        eng.step()
        for j in range(g.L):
            assert_close(eng.result(j), g.C[it][j])
    eng.close()


def _f32_valued_files(tmp_path, w=64, t0=10):
    """level files with float32 values (the reference's own files): a float64 load upcasts them exactly"""
    dec = synth.synth_decomposition(t0, w, levels=2, perm_kind="random", seed=5, hub_rows=2, hub_nnz=700)
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, w, True)
    return dec, base, w


def test_surface_float64_end_to_end(cuda_device, tmp_path):
    dec, base, w = _f32_valued_files(tmp_path)
    k = 12
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, w, True, np.float64,
                                                                                      slim=True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, w, k, 'gpu', True, True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    with pytest.raises(ValueError, match="float64"):
        arrow.B.zero_rhs(w, k, dtype=np.float32)
    arrow.B.zero_rhs(w, k, dtype=np.float64)
    eng = arrow._engine
    assert eng.dtype == np.float64
    X0 = np.random.default_rng(3).uniform(-1, 1, (eng.n_rows, k))
    arrow.B.set_features(X0)
    po = oracle.ReferenceProtocolOracle(dec, w, k, n_blocks=eng.n_blocks, dtype=np.longdouble)
    pa = oracle.ReferenceProtocolOracle(abs_decomposition(dec), w, k, n_blocks=eng.n_blocks, dtype=np.longdouble)
    po.set_features(X0.astype(np.longdouble))
    pa.set_features(np.abs(X0).astype(np.longdouble))
    arrow.step()
    got = arrow.B.result_tile()
    assert got.dtype == np.float64 and arrow.B.feature_tile().dtype == np.float64
    bound = _bound64(pa.step(), step_height(po))
    assert (np.abs(got.astype(np.longdouble) - po.step()).astype(np.float64) <= bound).all()
    full = np.empty_like(got)
    arrow.B.allgather_result(full)
    assert np.array_equal(full, got)
    with pytest.raises(ValueError):
        arrow.B.allgather_result(np.empty(got.shape, np.float32))
    # step_stream is bit-identical to set_features; step; result_tile
    X1 = np.random.default_rng(4).uniform(-1, 1, (eng.n_rows, k))
    arrow.B.set_features(X1)
    arrow.step()
    want = arrow.B.result_tile()
    pin_x = _lib.PinnedArray((eng.n_rows, k), np.float64)
    pin_o = _lib.PinnedArray((eng.n_rows, k), np.float64)
    pin_x.array[:] = X1
    arrow.step_stream(pin_x.array, pin_o.array)
    arrow.synchronize()
    assert np.array_equal(pin_o.array.view(np.uint64), want.view(np.uint64))
    pin_x.close()
    pin_o.close()
    eng.close()


def test_bench_spmm_float64(cuda_device, tmp_path, monkeypatch):
    from arrow_matrix_b200.arrow_bench import bench_spmm
    monkeypatch.chdir(tmp_path)
    _, base, w = _f32_valued_files(tmp_path)
    out = bench_spmm(base, w, 8, 2, True, 'gpu', datatype=np.float64, comm=SelfComm(), verbose=False)
    assert out is not None and len(out["times"]) == 2
    assert out["arrow"]._engine.dtype == np.float64
    out["arrow"]._engine.close()
