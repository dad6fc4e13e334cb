"""The boolean semiring (or, and) on bit tiles, one GPU, held EXACTLY to the host restatement of tests/bool_ref.py: OR is
exact, so every kernel, grid, tile list, option and mode gives the same words, padding bits included.

Canaries: X rows no short row reads hold random bits, so a stray gather changes the result; output rows past the block
(and the block's rows before the launch) hold a fixed word pattern, so a stray store shows up as a changed row.  The rows of
more than 24 entries read all-zero rows except one marker per long-row segment, so every segment, warp share and addend of
the long-row path shows in the result (tests/test_bool_cpu.py checks that faulty long-row paths give other words).
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
from tests import bool_ref as br
from tests import semiring_ref as sr
from tests import tile_dispatch as td
from tests.golden_util import GPU_CASES, GoldenCase

pytestmark = pytest.mark.gpu

OR = _lib.SR_OR_AND
ERR_ARG, ERR_UNSUPPORTED = -2, -6
CANARY = np.uint32(0xA5C3_5A3C)
Ctx = _lib.Context
# (option, value) pairs that change how a launch runs but never what it computes
OPTIONS = [("1 CTA", [(Ctx.OPT_SPMM_SM_LIMIT, 1), (Ctx.OPT_SPMM_CTAS_PER_SM, 1)]),
           ("default", []),
           ("forced predicated path", [(Ctx.OPT_FORCE_PREDICATED, 1)]),
           ("big tiles off", [(Ctx.OPT_BIG_TILES, 0)])] + \
          [(f"{r}-row tiles", [(Ctx.OPT_TILE_ROWS, r)]) for r in (16, 32, 64, 128)]
DEFAULTS = [(Ctx.OPT_SPMM_SM_LIMIT, 0), (Ctx.OPT_SPMM_CTAS_PER_SM, 0), (Ctx.OPT_FORCE_PREDICATED, 0),
            (Ctx.OPT_BIG_TILES, 1), (Ctx.OPT_TILE_ROWS, 0)]
EPILOGUES = ["plain", "add", "skip", "skip+add"]


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(cuda_device)
    yield c
    c.close()


def _set(ctx, opts):
    for o, v in DEFAULTS + list(opts):
        ctx.set_option(o, v)


def _bits(ctx, X):
    d = ctx.dense_alloc(X.shape[0], X.shape[1], _lib.BITS)
    d.h2d(br.pack(X))
    return d


def _ragged(lens, n_cols, rng):
    lens = np.asarray(lens, dtype=np.int64)
    ip = np.zeros(lens.size + 1, np.int64)
    ip[1:] = np.cumsum(lens)
    idx = rng.integers(0, n_cols, int(ip[-1]))
    return sparse.csr_matrix((rng.uniform(-1, 1, idx.size).astype(np.float32), idx, ip), shape=(lens.size, n_cols))


class Problem:
    """one block and the operands of every epilogue at one k (``bool_ref.problem_inputs``: the rows of more than 24
    entries read markers that make every segment, warp share and addend of the long-row path visible)"""

    def __init__(self, ctx, A, k, seed, density=0.05):
        self.ctx, self.A, self.k = ctx, A, k
        n, nc = A.shape
        self.n = n
        self.Xh, self.addh, self.amap, self.cmap, self.Xsh = br.problem_inputs(A, k, seed, density)
        n_add = self.addh.shape[0]
        self.Cinit = np.full((n + 3, br.words(k)), CANARY, np.uint32)
        self.dA = ctx.csr_upload(n, nc, A.indptr, A.indices, A.data)
        self.dAs = self.dA.remap_columns(ctx.map_upload(self.cmap, nc + 5), nc + 5)
        self.dam = ctx.map_upload(self.amap, n_add)
        self.dX, self.dXs, self.dadd = _bits(ctx, self.Xh), _bits(ctx, self.Xsh), _bits(ctx, self.addh)
        self.dC = ctx.dense_alloc(n + 3, k, _lib.BITS)
        self.P = br.spmm(A, self.Xh)
        self.Ps = br.spmm(A, self.Xsh, col_map=self.cmap)

    def expect(self, epi):
        P = self.Ps if "skip" in epi else self.P
        if "add" in epi:
            ok = self.amap >= 0
            P = P.copy()
            P[ok] |= self.addh[self.amap[ok]]
        return br.pack(P)

    def run(self, epi):
        self.dC.h2d(self.Cinit)
        A, X = (self.dAs, self.dXs) if "skip" in epi else (self.dA, self.dX)
        add, am = (self.dadd, self.dam) if "add" in epi else (None, None)
        self.ctx.spmm_sr(A, X, self.dC, add, am, OR)
        got = self.dC.d2h()
        assert np.array_equal(got[self.n:], self.Cinit[self.n:]), "rows past the block written"
        return got[: self.n]

    def free(self):
        for h in (self.dAs, self.dA, self.dam, self.dX, self.dXs, self.dadd, self.dC):
            h.free()


def _check_all(ctx, pr, label, options=OPTIONS):
    for epi in EPILOGUES:
        want = pr.expect(epi)
        for name, opts in options:
            _set(ctx, opts)
            got = pr.run(epi)
            assert np.array_equal(got, want), \
                f"{label} {epi} [{name}]: {int(np.any(got != want, axis=1).sum())} rows differ"


@pytest.fixture(scope="module")
def ragged():
    return br.hub_block(np.random.default_rng(64))


@pytest.mark.parametrize("k", br.SWEEP_KS)
def test_kernel_sweep_ragged_block(ctx, ragged, k):
    """every bit tile shape and the long-row kernels, every epilogue, every option"""
    pr = Problem(ctx, ragged, k, seed=k)
    assert pr.dA.info()["n_long_rows"] == 6
    try:
        _check_all(ctx, pr, f"k={k}")
    finally:
        _set(ctx, [])
        pr.free()


@pytest.mark.parametrize("k", [1, 33, 128, 129, 512])
def test_many_tiles_per_cta(ctx, k):
    """600k rows: at least 8 CSR tiles per resident CTA on the default grid, on every tile list"""
    rng = np.random.default_rng(k)
    A = _ragged(rng.integers(0, 16, 600000), 600000, rng)
    pr = Problem(ctx, A, k, seed=k, density=0.02)
    try:
        _check_all(ctx, pr, f"600k rows k={k}", [o for o in OPTIONS if o[0] != "1 CTA"])
    finally:
        _set(ctx, [])
        pr.free()


def test_long_row_tuning(ctx, ragged):
    """other long-row thresholds and segments: threshold 128 moves the rows of 140 ... 500 entries onto the long-row path,
    segments of 256 cut the hub rows into up to 20 segments"""
    try:
        for thr, seg in ((128, 256), (1016, 2048)):
            ctx.set_tuning(thr, seg)
            for k in (16, 129, 2049):
                pr = Problem(ctx, ragged, k, seed=k)
                try:
                    for epi in EPILOGUES:
                        assert np.array_equal(pr.run(epi), pr.expect(epi)), f"threshold {thr} k={k} {epi}"
                finally:
                    pr.free()
    finally:
        ctx.set_tuning(td.LONG_THRESHOLD, td.LONG_SEGMENT)


def test_graph_capture(ctx, ragged):
    pr = Problem(ctx, ragged, 64, seed=3)
    try:
        pr.run("add")                                   # un-captured first: the long-row scratch is sized
        pr.dC.h2d(pr.Cinit)
        ctx.sync()
        ctx.graph_begin()
        ctx.spmm_sr(pr.dA, pr.dX, pr.dC, pr.dadd, pr.dam, OR)
        g = ctx.graph_end()
        ctx.graph_launch(g)
        ctx.sync()
        assert np.array_equal(pr.dC.d2h()[: pr.n], pr.expect("add"))
        ctx.graph_free(g)
    finally:
        pr.free()


@pytest.mark.parametrize("k", [1, 33, 128, 200, 300, 1100, 8192])
def test_gather_count_diff_and_mark_new(ctx, k):
    """every lane-group width of the OR gather (1, 2, 4 and 8 lanes, rows longer than the group) and of the forward move,
    count_diff with several words per lane"""
    rng = np.random.default_rng(k)
    src = rng.random((300, k)) < 0.3
    dst0 = rng.random((250, k)) < 0.3
    m = np.where(rng.random(250) < 0.8, rng.permutation(300)[:250], -1).astype(np.int64)
    ok = m >= 0
    dS, dD, dm = _bits(ctx, src), _bits(ctx, dst0), ctx.map_upload(m, 300)
    # forward exchange: rows move, unrouted rows stay
    ctx.gather_rows(dD, dS, dm)
    want = dst0.copy()
    want[ok] = src[m[ok]]
    assert np.array_equal(dD.d2h(), br.pack(want))
    # backward exchange: OR
    dD.h2d(br.pack(dst0))
    ctx.gather_rows_sr(dD, dS, dm, OR)
    want = dst0.copy()
    want[ok] |= src[m[ok]]
    got = dD.d2h()
    assert np.array_equal(got, br.pack(want))
    # count_diff over the k columns (padding bits do not count)
    dB = _bits(ctx, dst0)
    changed = int(np.count_nonzero(np.any(want != dst0, axis=1)))
    assert ctx.count_diff(dD, dB) == changed > 0 and ctx.count_diff(dB, dB) == 0
    noisy = br.pack(dst0)
    if k < noisy.shape[1] * 32:
        noisy[:, k // 32] |= np.uint32(1 << (k % 32))
        dN = ctx.dense_alloc(250, k, _lib.BITS)
        dN.h2d(noisy)
        assert ctx.count_diff(dN, dB) == 0
        dN.free()
    # the level record: fresh bits get the level, every other element keeps its value; the count is returned
    dist0 = rng.integers(-5, 50, (250, k)).astype(np.int32)
    dd = ctx.dense_alloc(250, k, np.int32)
    dd.h2d(dist0)
    n_new = ctx.bits_mark_new(dD, dB, dd, 7)
    fresh = want & ~dst0
    assert n_new == int(fresh.sum())
    assert np.array_equal(dd.d2h(), np.where(fresh, 7, dist0))
    assert ctx.bits_mark_new(dD, dD, dd, 9) == 0
    for h in (dS, dD, dm, dB, dd):
        h.free()


def _code(fn):
    with pytest.raises(_lib.ArrowError) as e:
        fn()
    return e.value.code


def test_bit_tiles_and_refusals(ctx):
    rng = np.random.default_rng(0)
    n, k = 64, 40
    A = _ragged(rng.integers(1, 9, n), n, rng)
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    dA64 = ctx.csr_upload(n, n, A.indptr, A.indices, A.data, dtype=np.float64)
    Xb = _bits(ctx, rng.random((n, k)) < 0.5)
    Cb, Cb2 = ctx.dense_alloc(n, k, _lib.BITS), ctx.dense_alloc(n, k, _lib.BITS)
    X, C = ctx.dense_alloc(n, k), ctx.dense_alloc(n, k)
    X64 = ctx.dense_alloc(n, k, np.float64)
    L = ctx.dense_alloc(n, k, np.int32)
    m = ctx.map_upload(np.where(rng.random(n) < 0.5, rng.permutation(n), -1), n)
    # the round trip: alloc (zero filled), h2d, copy, d2h, dtype, fill 0
    assert Cb.device_dtype() == _lib.BITS and not Cb.d2h().any() and Cb.d2h().shape == (n, br.words(k))
    Cb.copy_from(Xb)
    assert np.array_equal(Cb.d2h(), Xb.d2h())
    Cb.fill(0.0)
    assert not Cb.d2h().any()
    assert _code(lambda: Cb.fill(1.0)) == ERR_ARG
    assert _code(lambda: Cb.copy_from(X)) == ERR_ARG
    # the block's values are not read: a float64 block gives the same bits
    ctx.spmm_sr(dA, Xb, Cb, semiring=OR)
    ctx.spmm_sr(dA64, Xb, Cb2, semiring=OR)
    assert np.array_equal(Cb.d2h(), Cb2.d2h())
    # bit operands of the other launches
    mp = _lib.SR_MIN_PLUS
    assert _code(lambda: ctx.spmm(dA, Xb, C)) == ERR_ARG
    assert _code(lambda: ctx.spmm(dA, X, Cb)) == ERR_ARG
    assert _code(lambda: ctx.spmm_add(dA, X, C, Cb, m)) == ERR_ARG
    assert _code(lambda: ctx.spmm_ex(dA, Xb, Cb)) == ERR_ARG
    assert _code(lambda: ctx.spmm_sr(dA, Xb, Cb, semiring=mp)) == ERR_ARG
    assert _code(lambda: ctx.spmm_sr(dA, Xb, Cb, semiring=_lib.SR_MAX_PLUS)) == ERR_ARG
    assert _code(lambda: ctx.spmm_sr_witness(dA, Xb, L, Cb, semiring=mp)) == ERR_ARG
    assert _code(lambda: ctx.gather_rows_multi(Cb, [Xb], [0, n], m)) == ERR_ARG
    assert _code(lambda: ctx.push_rows([Cb], [0, n], Xb, m)) == ERR_ARG
    assert _code(lambda: ctx.reduce_rows([Xb], n, dst=Cb)) == ERR_ARG
    assert _code(lambda: ctx.ptrtable_upload([Cb], np.zeros(n, np.int32), np.arange(n))) == ERR_ARG
    assert _code(lambda: ctx.gather_rows(Cb, Xb, m, accumulate=True)) == ERR_ARG
    assert _code(lambda: ctx.gather_rows_sr(Cb, Xb, m, mp)) == ERR_ARG
    # OR_AND with float / int operands, mixed operands
    assert _code(lambda: ctx.spmm_sr(dA, X, C, semiring=OR)) == ERR_ARG
    assert _code(lambda: ctx.spmm_sr(dA64, X64, X64, semiring=OR)) == ERR_ARG
    assert _code(lambda: ctx.spmm_sr(dA, Xb, C, semiring=OR)) == ERR_ARG
    assert _code(lambda: ctx.spmm_sr(dA, X, Cb, semiring=OR)) == ERR_ARG
    assert _code(lambda: ctx.spmm_sr(dA, Xb, Cb, C, m, OR)) == ERR_ARG
    assert _code(lambda: ctx.spmm_sr(dA, Xb, Xb, semiring=OR)) == ERR_ARG             # alias
    assert _code(lambda: ctx.gather_rows_sr(C, X, m, OR)) == ERR_ARG
    assert _code(lambda: ctx.gather_rows_sr(Cb, X, m, OR)) == ERR_ARG
    assert _code(lambda: ctx.gather_rows_sr(L, L, m, OR)) == ERR_ARG
    assert _code(lambda: ctx.count_diff(Cb, C)) == ERR_ARG
    assert _code(lambda: ctx.bits_mark_new(Cb, X, L, 1)) == ERR_ARG
    assert _code(lambda: ctx.bits_mark_new(Cb, Cb2, C, 1)) == ERR_ARG
    # k > 8192
    wide, wide_c = ctx.dense_alloc(n, 8193, _lib.BITS), ctx.dense_alloc(n, 8193, _lib.BITS)
    assert _code(lambda: ctx.spmm_sr(dA, wide, wide_c, semiring=OR)) == ERR_UNSUPPORTED
    for h in (wide, wide_c, m, L, X64, C, X, Cb2, Cb, Xb, dA64, dA):
        h.free()


# ---- the engine ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", GPU_CASES)
def test_engine_golden_decompositions(cuda_device, name):
    g = GoldenCase(name)
    for add_identity in (False, True):
        results = {}
        for mode in ("auto", "exchange"):
            eng = ArrowEngine(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, device=cuda_device,
                              mode=mode, semiring="or_and", add_identity=add_identity)
            p = br.BoolProtocol(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, n_blocks=eng.n_blocks,
                                add_identity=add_identity)
            X0 = np.random.default_rng(11).random((eng.n_rows, g.k)) < 0.1
            eng.set_features(X0)
            p.set_features(X0)
            out = []
            for it in range(3):
                eng.step()
                want = p.step()
                got = eng.result()
                assert got.dtype == bool and np.array_equal(got, want), f"{name} {eng.mode} step {it}"
                if eng.mode == "exchange":
                    for j in range(1, eng.L):
                        assert np.array_equal(eng.result(j), p.C[j]), f"{name} level {j} step {it}"
                out.append(got)
            results[eng.mode] = out
            eng.close()
        if "fused" in results:
            for a, b in zip(results["fused"], results["exchange"]):
                assert np.array_equal(a, b)


def test_engine_columns_zero_rhs_and_fixed_point(cuda_device):
    g = GoldenCase(GPU_CASES[0])
    dec, w = g.decomposition, g.width
    e128 = ArrowEngine(dec, w, 128, device=cuda_device, semiring="or_and", add_identity=True)
    n = e128.n_rows
    X = np.random.default_rng(5).random((n, 128)) < 0.02
    e128.set_features(X)
    e128.step()
    e128.step()
    full = e128.result()
    for k, cols in ((1, [37]), (5, list(range(60, 65)))):
        e = ArrowEngine(dec, w, k, device=cuda_device, semiring="or_and", add_identity=True)
        e.set_features(np.ascontiguousarray(X[:, cols]))
        e.step()
        e.step()
        assert np.array_equal(e.result(), full[:, cols]), f"k={k}"
        e.close()
    e128.zero_rhs()
    assert not e128.features(0).any() and not e128.result().any()
    e128.close()
    # iterate_to_fixed_point / count_changed against the restatement
    e = ArrowEngine(dec, w, 128, device=cuda_device, semiring="or_and", add_identity=True)
    p = br.BoolProtocol(dec, w, 128, block_diagonal=g.block_diagonal, n_blocks=e.n_blocks, add_identity=True)
    p.set_features(X)
    e.set_features(X)
    steps = e.iterate_to_fixed_point(200)
    assert steps < 200 and e.count_changed() == 0
    for _ in range(steps):
        p.step()
    assert np.array_equal(e.result(), p.C[0])
    e.close()


def test_bfs_levels_through_the_level_files(cuda_device, tmp_path):
    """BA graph -> arrow_decomposition -> level files -> load -> or_and with the identity, 128 sources, bfs_levels: the
    scipy hop counts in vertex order, and the min_plus engine with unit values on the same files"""
    n, w = 200000, 20000
    A = sr.weighted_ba_graph(n, 3, seed=5, unit=True)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, w, True)
    sources = np.random.default_rng(8).choice(n, 128, replace=False)

    def load(semiring):
        comm = SelfComm()
        blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, w, True)
        arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, w, sources.size, 'gpu', True, True,
                                                 semiring=semiring, add_identity=True)
        arrow.B.load_sparse_matrix_from_blocks(blocks)
        return arrow, blocks

    arrow, blocks = load("or_and")
    from arrow_matrix_b200 import decomp
    perm0 = decomp.prepare_permutations([p for _, p in blocks.decomposition], blocks.n_blocks, w)[0][0]
    eng = arrow._engine
    arrow.B.set_features(br.source_bits(perm0, eng.n_rows, n, sources))
    levels = arrow.bfs_levels(500)
    assert eng.last_bfs_steps < 500 and levels.dtype == np.int32
    assert arrow.B.result_tile().dtype == bool
    hops = csgraph.shortest_path(A, unweighted=True, indices=sources)
    want = np.where(np.isinf(hops), -1, hops).astype(np.int32)
    got = br.vertex_order(levels, perm0, n, -1).T
    assert np.array_equal(got, want), f"{int(np.sum(got != want))} levels differ"
    # a second call from the same sources gives the same levels (the level tile is reused)
    arrow.B.set_features(br.source_bits(perm0, eng.n_rows, n, sources))
    assert np.array_equal(arrow.bfs_levels(500), levels)
    eng.close()
    mp, _ = load("min_plus")
    mp.B.set_features(sr.source_features(perm0, mp._engine.n_rows, n, sources))
    mp._engine.iterate_to_fixed_point(500)
    D = mp.B.result_tile()
    assert np.array_equal(levels, np.where(np.isinf(D), -1, D).astype(np.int32))
    mp._engine.close()


@pytest.mark.parametrize("name", [c for c in GPU_CASES if GoldenCase(c).L >= 2])
def test_bfs_levels_both_modes(cuda_device, name):
    """bfs_levels in the mode `auto` picks and in exchange mode (stale rows behind the sentinel kept) == the restated level
    record, twice on the same engine (the level tile is reused)"""
    g = GoldenCase(name)
    for mode in ("auto", "exchange"):
        eng = ArrowEngine(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, device=cuda_device, mode=mode,
                          semiring="or_and", add_identity=True)
        assert eng.last_bfs_steps == 0
        X0 = np.random.default_rng(2).random((eng.n_rows, g.k)) < 0.01
        for rep in range(2):
            p = br.BoolProtocol(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, n_blocks=eng.n_blocks,
                                add_identity=True)
            p.set_features(X0)
            if rep:
                eng.zero_rhs()                  # fresh level tiles, like the restatement's
            eng.set_features(X0)
            want, steps = p.bfs_levels(100)
            got = eng.bfs_levels(100)
            assert np.array_equal(got, want) and eng.last_bfs_steps == steps, f"{name} {eng.mode} call {rep}"
        eng.close()


def test_uint32_is_not_a_tile_type(ctx):
    with pytest.raises(ValueError):
        ctx.dense_alloc(4, 8, np.uint32)
