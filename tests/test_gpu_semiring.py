"""The (min, +) and (max, +) semirings on one GPU, held EXACTLY to the host restatement of tests/semiring_ref.py: every
term is rounded once and min / max are exact, so no tolerance applies to any kernel, grid, tile size, option or mode.

Canaries: X rows no entry reads, addend rows no row adds and the C rows past the block hold the finite value that would
win the ⊕ (∓3e38): a stray read shows up in the result, a stray write as a changed row past the block.
"""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200 import _lib, graphio
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from tests import semiring_ref as sr
from tests import tile_dispatch as td
from tests.golden_util import GPU_CASES, GoldenCase

pytestmark = pytest.mark.gpu

SEMIRINGS = {"min_plus": _lib.SR_MIN_PLUS, "max_plus": _lib.SR_MAX_PLUS}
ERR_ARG, ERR_UNSUPPORTED = -2, -6
Ctx = _lib.Context
# (option, value) pairs that change how a launch runs but never what it computes
OPTIONS = [("1 CTA", [(Ctx.OPT_SPMM_SM_LIMIT, 1), (Ctx.OPT_SPMM_CTAS_PER_SM, 1)]),
           ("default", []),
           ("no L2 hints", [(Ctx.OPT_L2_HINTS_PLAIN, 0)]),
           ("big tiles off", [(Ctx.OPT_BIG_TILES, 0)]),
           ("forced predicated path", [(Ctx.OPT_FORCE_PREDICATED, 1)])]
DEFAULTS = [(Ctx.OPT_SPMM_SM_LIMIT, 0), (Ctx.OPT_SPMM_CTAS_PER_SM, 0), (Ctx.OPT_L2_HINTS_PLAIN, 3),
            (Ctx.OPT_BIG_TILES, 1), (Ctx.OPT_FORCE_PREDICATED, 0)]


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(cuda_device)
    yield c
    c.close()


def _set(ctx, opts):
    for o, v in DEFAULTS + list(opts):
        ctx.set_option(o, v)


def _values(rng, n):
    return (rng.uniform(-1, 1, n) * 10.0 ** rng.uniform(-2, 2, n)).astype(np.float32)


def _ragged(lens, n_cols, rng):
    lens = np.asarray(lens, dtype=np.int64)
    ip = np.zeros(lens.size + 1, np.int64)
    ip[1:] = np.cumsum(lens)
    idx = rng.integers(0, n_cols, int(ip[-1]))
    return sparse.csr_matrix((_values(rng, idx.size), idx, ip), shape=(lens.size, n_cols))


def _ragged_block(rng):
    """20k rows: short ragged rows, empty rows, and hub rows of one to three long-row segments"""
    n = 20000
    lens = rng.integers(0, 24, n)
    lens[rng.integers(0, n, 300)] = 0
    lens[[7, 9000]] = [600, 5000]
    lens[15000:15004] = [513, 2048, 2049, 4100]
    return _ragged(lens, n, rng)


def _canaried(rows, k, keep, semiring, rng):
    out = np.full((rows, k), sr.WINNER[semiring], np.float32)
    keep = np.unique(keep)
    out[keep] = _values(rng, keep.size * k).reshape(keep.size, k)
    return out


class Problem:
    """one block and the operands of every epilogue at one k and semiring"""

    def __init__(self, ctx, A, k, semiring, seed):
        rng = np.random.default_rng(seed)
        self.ctx, self.A, self.k, self.semiring, self.code = ctx, A, k, semiring, SEMIRINGS[semiring]
        n, nc = A.shape
        self.n = n
        used = np.unique(A.indices)
        self.Xh = _canaried(nc + 5, k, used, semiring, rng)
        n_add = n // 2 + 4
        self.amap = np.where(rng.random(n) < 0.6, rng.integers(0, n_add, n), -1).astype(np.int64)
        self.addh = _canaried(n_add, k, self.amap[self.amap >= 0], semiring, rng)
        self.cmap = rng.permutation(nc + 5)[:nc].astype(np.int64)
        self.cmap[::5] = -1                                    # entries whose image is invalid: skipped
        img = self.cmap[used]
        self.Xsh = _canaried(nc + 7, k, img[img >= 0], semiring, rng)
        self.Cinit = np.full((n + 3, k), sr.WINNER[semiring], np.float32)
        self.dA = ctx.csr_upload(n, nc, A.indptr, A.indices, A.data)
        self.dAs = self.dA.remap_columns(ctx.map_upload(self.cmap, nc + 5), nc + 5)
        self.dam = ctx.map_upload(self.amap, n_add)
        self.dX = ctx.dense_from_host(self.Xh)
        self.dXs = ctx.dense_from_host(self.Xsh)
        self.dadd = ctx.dense_from_host(self.addh)
        self.dC = ctx.dense_alloc(n + 3, k)
        self.P = sr.spmm(A, self.Xh, semiring)
        self.Ps = sr.spmm(A, self.Xsh, semiring, col_map=self.cmap)

    def expect(self, epi):
        P = self.Ps if "skip" in epi else self.P
        if "add" in epi:
            ok = self.amap >= 0
            P = P.copy()
            P[ok] = sr.plus(self.semiring)(P[ok], self.addh[self.amap[ok]])
        return P

    def run(self, epi):
        self.dC.h2d(self.Cinit)
        A, X = (self.dAs, self.dXs) if "skip" in epi else (self.dA, self.dX)
        add, am = (self.dadd, self.dam) if "add" in epi else (None, None)
        self.ctx.spmm_sr(A, X, self.dC, add, am, self.code)
        got = self.dC.d2h()
        assert np.array_equal(got[self.n:].view(np.uint32), self.Cinit[self.n:].view(np.uint32)), "rows past the block written"
        return got[: self.n]

    def free(self):
        for h in (self.dAs, self.dA, self.dam, self.dX, self.dXs, self.dadd, self.dC):
            h.free()


EPILOGUES = ["plain", "add", "skip", "skip+add"]


def _check_all(ctx, pr, label):
    tile = pr.k % 4 == 0 and pr.k <= 256
    for epi in EPILOGUES:
        want = pr.expect(epi)
        for name, opts in (OPTIONS if tile else OPTIONS[:2]):       # the other options are switches of the tile kernel
            _set(ctx, opts)
            got = pr.run(epi)
            bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
            assert not bad.any(), f"{label} {pr.semiring} {epi} [{name}]: {int(bad.sum())} elements differ"


@pytest.fixture(scope="module")
def ragged():
    return _ragged_block(np.random.default_rng(64))


@pytest.mark.parametrize("k", sr.SWEEP_KS)
@pytest.mark.parametrize("semiring", list(SEMIRINGS))
def test_kernel_sweep_ragged_block(ctx, ragged, k, semiring):
    """tile kernels (k % 4 == 0, k <= 256), the generic kernel and the long-row kernels, every epilogue, every option"""
    pr = Problem(ctx, ragged, k, semiring, seed=k)
    assert pr.dA.info()["n_long_rows"] == 6
    try:
        _check_all(ctx, pr, f"k={k}")
    finally:
        _set(ctx, [])
        pr.free()


def test_long_row_tuning(ctx, ragged):
    """other long-row thresholds and segments (hub rows of more segments, more rows on the long-row path) give the same
    values"""
    try:
        for thr, seg in ((128, 256), (1016, 2048)):
            ctx.set_tuning(thr, seg)
            for k, semiring in ((16, "min_plus"), (36, "max_plus"), (5, "min_plus")):
                pr = Problem(ctx, ragged, k, semiring, seed=k)
                try:
                    for epi in EPILOGUES:
                        assert np.array_equal(pr.run(epi), pr.expect(epi)), f"threshold {thr} k={k} {epi}"
                finally:
                    pr.free()
    finally:
        ctx.set_tuning(td.LONG_THRESHOLD, td.LONG_SEGMENT)


def _boundary_blocks(rng):
    yield "nnz=0", sparse.csr_matrix((50, 60), dtype=np.float32)
    yield "no tiles", _ragged([600, 700, 900], 1000, rng)
    for n in (1, 2, 63, 64, 65, 127, 128, 129):
        yield f"{n} rows", _ragged(rng.integers(0, 40, n), 300, rng)
    yield "nnz cap", _ragged(rng.integers(250, 511, size=60), 4000, rng)


@pytest.mark.parametrize("k", [4, 12, 128, 5])
def test_tile_boundary_shapes(ctx, k):
    rng = np.random.default_rng(7 + k)
    for label, A in _boundary_blocks(rng):
        for semiring in SEMIRINGS:
            pr = Problem(ctx, A, k, semiring, seed=k)
            try:
                _check_all(ctx, pr, label)
            finally:
                _set(ctx, [])
                pr.free()


@pytest.mark.parametrize("k", [3, 8, 128])
def test_gather_rows_sr_and_count_diff(ctx, k):
    rng = np.random.default_rng(k)
    src = _values(rng, 300 * k).reshape(300, k)
    dst0 = _values(rng, 250 * k).reshape(250, k)
    m = np.where(rng.random(250) < 0.8, rng.permutation(300)[:250], -1).astype(np.int64)
    dS, dD = ctx.dense_from_host(src), ctx.dense_from_host(dst0)
    dm = ctx.map_upload(m, 300)
    ok = m >= 0
    for semiring, code in SEMIRINGS.items():
        dD.h2d(dst0)
        ctx.gather_rows_sr(dD, dS, dm, code)
        want = dst0.copy()
        want[ok] = sr.plus(semiring)(dst0[ok], src[m[ok]])
        got = dD.d2h()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        dB = ctx.dense_from_host(dst0)
        changed = int(np.count_nonzero(np.any(got != dst0, axis=1)))
        assert ctx.count_diff(dD, dB) == changed > 0
        assert ctx.count_diff(dB, dB) == 0
        dB.free()
    # by value: -0 == +0, NaN != NaN
    a = np.zeros((4, k), np.float32)
    b = a.copy()
    b[1, 0] = -0.0
    b[2, k - 1] = np.nan
    a[3, k // 2] = np.nan
    b[3, k // 2] = np.nan
    da, db = ctx.dense_from_host(a), ctx.dense_from_host(b)
    assert ctx.count_diff(da, db) == 2
    for h in (dS, dD, dm, da, db):
        h.free()


def _code(fn):
    with pytest.raises(_lib.ArrowError) as e:
        fn()
    return e.value.code


def test_plus_times_forwards_and_refusals(ctx):
    rng = np.random.default_rng(0)
    A = _ragged(rng.integers(1, 9, 64), 64, rng)
    k = 8
    dA = ctx.csr_upload(64, 64, A.indptr, A.indices, A.data)
    X = ctx.dense_from_host(_values(rng, 64 * k).reshape(64, k))
    S = ctx.dense_from_host(_values(rng, 64 * k).reshape(64, k))
    m = ctx.map_upload(np.where(rng.random(64) < 0.5, rng.permutation(64), -1), 64)
    C1, C2 = ctx.dense_alloc(64, k), ctx.dense_alloc(64, k)
    for add in (False, True):
        if add:
            ctx.spmm_add(dA, X, C1, S, m)
            ctx.spmm_sr(dA, X, C2, S, m, _lib.SR_PLUS_TIMES)
        else:
            ctx.spmm(dA, X, C1)
            ctx.spmm_sr(dA, X, C2, semiring=_lib.SR_PLUS_TIMES)
        assert np.array_equal(C1.d2h().view(np.uint32), C2.d2h().view(np.uint32))
    C1.copy_from(S)
    C2.copy_from(S)
    ctx.gather_rows(C1, X, m, accumulate=True)
    ctx.gather_rows_sr(C2, X, m, _lib.SR_PLUS_TIMES)
    assert np.array_equal(C1.d2h().view(np.uint32), C2.d2h().view(np.uint32))
    # refusals
    A64 = ctx.csr_upload(64, 64, A.indptr, A.indices, A.data, dtype=np.float64)
    X64, C64 = ctx.dense_alloc(64, k, np.float64), ctx.dense_alloc(64, k, np.float64)
    mp = _lib.SR_MIN_PLUS
    assert _code(lambda: ctx.spmm_sr(A64, X64, C64, semiring=mp)) == ERR_UNSUPPORTED
    assert _code(lambda: ctx.gather_rows_sr(C64, X64, m, mp)) == ERR_UNSUPPORTED
    assert _code(lambda: ctx.spmm_sr(dA, X64, C1, semiring=mp)) == ERR_ARG            # mixed
    assert _code(lambda: ctx.spmm_sr(dA, X, X, semiring=mp)) == ERR_ARG                # alias
    assert _code(lambda: ctx.spmm_sr(dA, X, C1, semiring=7)) == ERR_ARG                # unknown
    assert _code(lambda: ctx.gather_rows_sr(C1, X, m, 7)) == ERR_ARG
    assert _code(lambda: ctx.gather_rows_sr(C1, X64, m, mp)) == ERR_ARG
    Cn = ctx.dense_alloc(10, k)
    assert _code(lambda: ctx.spmm_sr(dA, X, Cn, semiring=mp)) == ERR_ARG              # shape
    assert _code(lambda: ctx.count_diff(C1, Cn)) == ERR_ARG
    assert _code(lambda: ctx.count_diff(C1, C64)) == ERR_ARG
    for h in (Cn, X64, C64, A64, C1, C2, m, S, X, dA):
        h.free()


# ---- the engine ----------------------------------------------------------------------------------------------------
def _features(rows, k, seed):
    rng = np.random.default_rng(seed)
    return _values(rng, rows * k).reshape(rows, k)


@pytest.mark.parametrize("name", GPU_CASES)
def test_engine_golden_decompositions(cuda_device, name):
    g = GoldenCase(name)
    for semiring in SEMIRINGS:
        results = {}
        for mode in ("auto", "exchange"):
            eng = ArrowEngine(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, device=cuda_device,
                              mode=mode, semiring=semiring)
            p = sr.SemiringProtocol(g.decomposition, g.width, g.k, semiring, block_diagonal=g.block_diagonal,
                                    n_blocks=eng.n_blocks)
            X0 = _features(eng.n_rows, g.k, 11)
            eng.set_features(X0)
            p.set_features(X0)
            out = []
            for it in range(3):
                eng.step()
                want = p.step()
                got = eng.result()
                assert np.array_equal(got, want), f"{name} {semiring} {eng.mode} step {it}"
                if eng.mode == "exchange":
                    for j in range(1, eng.L):
                        assert np.array_equal(eng.result(j), p.C[j]), f"{name} {semiring} level {j} step {it}"
                out.append(got)
            results[eng.mode] = out
            eng.close()
        if "fused" in results:
            for a, b in zip(results["fused"], results["exchange"]):
                assert np.array_equal(a, b)


def test_engine_stream_columns_and_zero_rhs(cuda_device):
    g = GoldenCase(GPU_CASES[0])
    dec, w = g.decomposition, g.width
    for semiring in SEMIRINGS:
        e128 = ArrowEngine(dec, w, 128, device=cuda_device, semiring=semiring, add_identity=True)
        n = e128.n_rows
        X = _features(n, 128, 5)
        e128.set_features(X)
        e128.step()
        e128.step()
        full = e128.result()
        for k, cols in ((1, [37]), (5, list(range(60, 65)))):
            e = ArrowEngine(dec, w, k, device=cuda_device, semiring=semiring, add_identity=True)
            e.set_features(np.ascontiguousarray(X[:, cols]))
            e.step()
            e.step()
            assert np.array_equal(e.result(), full[:, cols]), f"{semiring} k={k}"
            e.close()
        # step_stream == set_features; step; result
        e128.set_features(X)
        e128.step()
        want = e128.result()
        pin_x, pin_o = _lib.PinnedArray((n, 128)), _lib.PinnedArray((n, 128))
        pin_x.array[:] = X
        e128.stream_step(pin_x.array, pin_o.array)
        e128.stream_drain()
        assert np.array_equal(pin_o.array.view(np.uint32), want.view(np.uint32))
        pin_x.close()
        pin_o.close()
        e128.zero_rhs()
        ident = np.float32(sr.zero(semiring))
        assert (e128.features(0) == ident).all() and (e128.result() == ident).all()
        e128.close()


def test_end_to_end_sssp(cuda_device, tmp_path):
    """BA graph -> arrow_decomposition -> level files -> load -> min_plus with the identity, 32 sources, to the fixed
    point: equal to Dijkstra"""
    n, w = 200000, 20000
    A = sr.weighted_ba_graph(n, 3, seed=5)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, w, True)
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, w, True)
    sources = np.random.default_rng(8).choice(n, 32, replace=False)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, w, sources.size, 'gpu', True, True,
                                             semiring="min_plus", add_identity=True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    eng = arrow._engine
    perm0 = decomp_perm0(blocks, w)
    arrow.B.set_features(sr.source_features(perm0, eng.n_rows, n, sources))
    steps = eng.iterate_to_fixed_point(500)
    assert steps < 500 and eng.count_changed() == 0
    got = sr.distances(arrow.B.result_tile(), perm0, n)
    want = csgraph.shortest_path(A, method="D", indices=sources).astype(np.float32)
    assert np.array_equal(got, want), f"{int(np.sum(got != want))} distances differ after {steps} steps"
    eng.close()


def decomp_perm0(blocks, w):
    from arrow_matrix_b200 import decomp
    perms, _, _, _ = decomp.prepare_permutations([p for _, p in blocks.decomposition], blocks.n_blocks, w)
    return perms[0]
