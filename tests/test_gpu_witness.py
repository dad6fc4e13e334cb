"""Predecessors of the (min, +) / (max, +) step on one GPU, held EXACTLY to the host restatement of tests/witness_ref.py:
the lexicographic ⊕ over (value, label) pairs is exact and order-free, so no tolerance applies to any kernel, grid,
option or mode.  Weights in {0..3} and features in {0..7} make most elements tie between several candidates, so the
smallest-label rule decides.

Canaries: X rows no entry reads and addend rows no row adds hold the value that would win the ⊕ (∓3e38, label 0); the
output rows past the block hold canary values and labels and must stay bit-identical.
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
from tests import witness_ref as wr
from tests.golden_util import GPU_CASES, GoldenCase
from tests.test_witness_cpu import _check_chains

pytestmark = pytest.mark.gpu

SEMIRINGS = {"min_plus": _lib.SR_MIN_PLUS, "max_plus": _lib.SR_MAX_PLUS}
ERR_ARG, ERR_UNSUPPORTED = -2, -6
LAB_CANARY = 0x7EADBEEF
Ctx = _lib.Context
OPTIONS = [("1 CTA", [(Ctx.OPT_SPMM_SM_LIMIT, 1), (Ctx.OPT_SPMM_CTAS_PER_SM, 1)]),
           ("default", []),
           ("big tiles off", [(Ctx.OPT_BIG_TILES, 0)]),
           ("forced predicated path", [(Ctx.OPT_FORCE_PREDICATED, 1)])]
DEFAULTS = [(Ctx.OPT_SPMM_SM_LIMIT, 0), (Ctx.OPT_SPMM_CTAS_PER_SM, 0), (Ctx.OPT_BIG_TILES, 1),
            (Ctx.OPT_FORCE_PREDICATED, 0)]


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(cuda_device)
    yield c
    c.close()


def _set(ctx, opts):
    for o, v in DEFAULTS + list(opts):
        ctx.set_option(o, v)


def _ragged_block(rng):
    """6000 rows of 0..23 entries with weights 0..3, diagonal entries on a third of them, and hub rows of one to three
    long-row segments"""
    n = 6000
    lens = rng.integers(0, 24, n)
    lens[rng.integers(0, n, 100)] = 0
    lens[[7, 3000, 4500, 4501, 5999]] = [600, 4100, 513, 2049, 2048]
    ip = np.zeros(n + 1, np.int64)
    ip[1:] = np.cumsum(lens)
    idx = rng.integers(0, n, int(ip[-1]))
    rows = np.repeat(np.arange(n), lens)
    diag = (rng.random(idx.size) < 0.05) & (rows % 3 == 0)
    idx[diag] = rows[diag]
    vals = rng.integers(0, 4, idx.size).astype(np.float32)
    return sparse.csr_matrix((vals, idx, ip), shape=(n, n))


def _features(rng, rows, k, semiring, used):
    """values 0..7 (5 % the ⊕ identity) on the rows entries read, the winning canary elsewhere"""
    X = np.full((rows, k), sr.WINNER[semiring], np.float32)
    used = np.unique(used)
    v = rng.integers(0, 8, (used.size, k)).astype(np.float32)
    v[rng.random(v.shape) < 0.05] = np.float32(sr.zero(semiring))
    X[used] = v
    return X


class Problem:
    """one block and the operands of every epilogue at one k and semiring"""

    def __init__(self, ctx, A, k, semiring, seed):
        rng = np.random.default_rng(seed)
        self.ctx, self.A, self.k, self.semiring, self.code = ctx, A, k, semiring, SEMIRINGS[semiring]
        n = A.shape[0]
        self.n = n
        self.Xh = _features(rng, n + 5, k, semiring, A.indices)
        # own labels: the row's first column on a third of the rows (excludes real entries), -1 or a random row elsewhere
        first = np.where(np.diff(A.indptr) > 0, A.indices[np.minimum(A.indptr[:-1], max(A.nnz - 1, 0))], -1)
        self.own = np.where(rng.random(n) < 0.33, first, np.where(rng.random(n) < 0.5, -1, rng.integers(0, n, n)))
        n_add = n // 2 + 4
        self.amap = np.where(rng.random(n) < 0.6, rng.integers(0, n_add, n), -1).astype(np.int64)
        self.add_v = _features(rng, n_add, k, semiring, self.amap[self.amap >= 0])
        self.add_l = np.where(self.add_v == sr.WINNER[semiring], 0, rng.integers(0, n, self.add_v.shape)).astype(np.int32)
        self.cmap = rng.permutation(n + 5)[:n].astype(np.int64)
        self.cmap[::5] = -1                                              # entries whose image is invalid: skipped
        img = self.cmap[A.indices]
        self.Xsh = _features(rng, n + 7, k, semiring, img[img >= 0])
        self.dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
        self.dAs = self.dA.remap_columns(ctx.map_upload(self.cmap, n + 5), n + 5)
        self.down = ctx.map_upload(self.own, n)
        self.dam = ctx.map_upload(self.amap, n_add)
        self.dX, self.dXs = ctx.dense_from_host(self.Xh), ctx.dense_from_host(self.Xsh)
        self.dav = ctx.dense_from_host(self.add_v)
        self.dal = ctx.dense_alloc(n_add, k, np.int32)
        self.dal.h2d(self.add_l)
        self.Vinit = np.full((n + 3, k), 1.5, np.float32)
        self.Linit = np.full((n + 3, k), LAB_CANARY, np.int32)
        self.dV, self.dL = ctx.dense_alloc(n + 3, k), ctx.dense_alloc(n + 3, k, np.int32)
        # expectations
        add = dict(add=(self.add_v, self.add_l), add_map=self.amap)
        self.want = {
            "pair": wr.witness_spmm(A, self.Xh, semiring),
            "pair+add": wr.witness_spmm(A, self.Xh, semiring, self_labels=self.own, **add),
            "skip+add": wr.witness_spmm(A, self.Xsh, semiring, col_map=self.cmap, self_labels=self.own, **add),
        }
        wv, wl = wr.witness_spmm(A, self.Xh, semiring, **add)
        # D: the witness value on 60 % of the elements (those get a parent), random values and identities elsewhere
        D = np.where(rng.random((n, k)) < 0.6, wv, rng.integers(0, 8, (n, k)).astype(np.float32)).astype(np.float32)
        D[rng.random(D.shape) < 0.05] = np.float32(sr.zero(semiring))
        self.Dh = np.vstack([D, np.full((2, k), 9.0, np.float32)])
        self.dD = ctx.dense_from_host(self.Dh)
        self.want["parent"] = (wv, wr.parents(semiring, D, wv, wl))
        assert (self.want["parent"][1] >= 0).sum() > D.size // 4

    def run(self, epi):
        self.dV.h2d(self.Vinit)
        self.dL.h2d(self.Linit)
        kw = dict(semiring=self.code, values=self.dV)
        if epi == "pair":
            self.ctx.spmm_sr_witness(self.dA, self.dX, self.dL, **kw)
        else:
            kw.update(add_values=self.dav, add_labels=self.dal, add_map=self.dam)
            if epi == "pair+add":
                self.ctx.spmm_sr_witness(self.dA, self.dX, self.dL, row_labels=self.down, **kw)
            elif epi == "skip+add":
                self.ctx.spmm_sr_witness(self.dAs, self.dXs, self.dL, row_labels=self.down, **kw)
            else:
                self.ctx.spmm_sr_witness(self.dA, self.dX, self.dL, dist=self.dD, **kw)
        V, L = self.dV.d2h(), self.dL.d2h()
        assert np.array_equal(V[self.n:].view(np.uint32), self.Vinit[self.n:].view(np.uint32)), "values past the block"
        assert np.array_equal(L[self.n:], self.Linit[self.n:]), "labels past the block"
        return V[: self.n], L[: self.n]

    def free(self):
        for h in (self.dAs, self.dA, self.down, self.dam, self.dX, self.dXs, self.dav, self.dal, self.dV, self.dL,
                  self.dD):
            h.free()


EPILOGUES = ["pair", "pair+add", "skip+add", "parent"]


def _check_all(ctx, pr, label):
    tile = pr.k % 4 == 0 and pr.k <= 256
    for epi in EPILOGUES:
        wv, wl = pr.want[epi]
        for name, opts in (OPTIONS if tile else OPTIONS[:2]):       # the other options are switches of the tile kernel
            _set(ctx, opts)
            V, L = pr.run(epi)
            assert np.array_equal(V, wv), f"{label} {pr.semiring} {epi} [{name}]: values differ"
            bad = L != wl
            assert not bad.any(), f"{label} {pr.semiring} {epi} [{name}]: {int(bad.sum())} labels differ"


@pytest.fixture(scope="module")
def ragged():
    return _ragged_block(np.random.default_rng(65))


@pytest.mark.parametrize("k", sr.SWEEP_KS)
@pytest.mark.parametrize("semiring", list(SEMIRINGS))
def test_kernel_sweep_ragged_block(ctx, ragged, k, semiring):
    """tile kernels (k % 4 == 0, k <= 256), the generic kernel and the long-row kernels, every epilogue, every option"""
    pr = Problem(ctx, ragged, k, semiring, seed=k)
    assert pr.dA.info()["n_long_rows"] == 5
    try:
        _check_all(ctx, pr, f"k={k}")
    finally:
        _set(ctx, [])
        pr.free()


# ---- the C ABI ------------------------------------------------------------------------------------------------------
def _code(fn):
    with pytest.raises(_lib.ArrowError) as e:
        fn()
    return e.value.code


def test_int32_tiles_and_refusals(ctx):
    rng = np.random.default_rng(0)
    n, k = 64, 8
    A = sparse.random(n, n, density=0.1, format="csr", random_state=1, dtype=np.float32)
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    X = ctx.dense_from_host(rng.integers(0, 8, (n, k)).astype(np.float32))
    V = ctx.dense_alloc(n, k)
    L, L2 = ctx.dense_alloc(n, k, np.int32), ctx.dense_alloc(n, k, np.int32)
    m = ctx.map_upload(np.where(rng.random(n) < 0.5, rng.permutation(n), -1), n)
    # the int32 round trip: alloc (zero filled), h2d, copy, d2h, dtype
    assert L.device_dtype() == np.int32 and L.d2h().dtype == np.int32 and not L.d2h().any()
    h = rng.integers(-2**31, 2**31 - 1, (n, k), dtype=np.int64).astype(np.int32)
    L.h2d(h)
    L2.copy_from(L)
    assert np.array_equal(L2.d2h(), h)
    assert _code(lambda: L2.copy_from(V)) == ERR_ARG                                       # int32 vs float32
    # int32 operands of the existing launches
    Xi = ctx.dense_alloc(n, k, np.int32)
    mp = _lib.SR_MIN_PLUS
    assert _code(lambda: ctx.spmm(dA, Xi, V)) == ERR_ARG
    assert _code(lambda: ctx.spmm(dA, X, L)) == ERR_ARG
    assert _code(lambda: ctx.spmm_add(dA, X, V, L, m)) == ERR_ARG
    assert _code(lambda: ctx.spmm_sr(dA, Xi, V, semiring=mp)) == ERR_ARG
    assert _code(lambda: ctx.spmm_sr(dA, X, L, semiring=mp)) == ERR_ARG
    assert _code(lambda: ctx.gather_rows(L, Xi, m)) == ERR_ARG
    assert _code(lambda: ctx.gather_rows(L, Xi, m, accumulate=True)) == ERR_ARG
    assert _code(lambda: ctx.gather_rows_sr(L, Xi, m, mp)) == ERR_ARG
    assert _code(lambda: ctx.count_diff(L, L2)) == ERR_ARG
    assert _code(lambda: L.fill(1.0)) == ERR_ARG
    assert _code(lambda: ctx.reduce_rows([L], n, dst=L2)) == ERR_ARG
    assert _code(lambda: ctx.ptrtable_upload([L], np.zeros(n, np.int32), np.arange(n))) == ERR_ARG
    # refusals of the witness launch
    A64 = ctx.csr_upload(n, n, A.indptr, A.indices, A.data, dtype=np.float64)
    X64, V64 = ctx.dense_alloc(n, k, np.float64), ctx.dense_alloc(n, k, np.float64)
    w = ctx.spmm_sr_witness
    assert _code(lambda: w(dA, X, L, V, semiring=_lib.SR_PLUS_TIMES)) == ERR_UNSUPPORTED
    assert _code(lambda: w(A64, X64, L, V64, semiring=mp)) == ERR_UNSUPPORTED
    assert _code(lambda: w(dA, X64, L, V, semiring=mp)) == ERR_ARG                       # mixed
    assert _code(lambda: w(dA, X, V, L, semiring=mp)) == ERR_ARG                         # labels must be int32
    assert _code(lambda: w(dA, X, L, X, semiring=mp)) == ERR_ARG                         # alias
    assert _code(lambda: w(dA, X, L, V, dist=V, semiring=mp)) == ERR_ARG                 # alias
    assert _code(lambda: w(dA, X, L, V, semiring=7)) == ERR_ARG                          # unknown
    assert _code(lambda: w(dA, X, L, semiring=mp)) == ERR_ARG                            # pair out without values
    Ln = ctx.dense_alloc(10, k, np.int32)
    assert _code(lambda: w(dA, X, Ln, V, semiring=mp)) == ERR_ARG                        # shape
    assert _code(lambda: w(dA, X, L, V, add_values=V64, add_labels=L2, add_map=m, semiring=mp)) == ERR_ARG
    assert _code(lambda: w(dA, X, L, V, add_values=X, add_labels=V, add_map=m, semiring=mp)) == ERR_ARG
    w(dA, X, L, V, dist=X, semiring=mp)                                                  # dist may be X
    for hh in (Ln, A64, X64, V64, Xi, m, L2, L, V, X, dA):
        hh.free()


# ---- the engine ----------------------------------------------------------------------------------------------------
def _int_features(rows, k, semiring, seed):
    rng = np.random.default_rng(seed)
    X = rng.integers(0, 8, (rows, k)).astype(np.float32)
    X[rng.random(X.shape) < 0.1] = np.float32(sr.zero(semiring))
    return X


@pytest.mark.parametrize("name", GPU_CASES)
def test_engine_golden_decompositions(cuda_device, name):
    g = GoldenCase(name)
    for semiring in SEMIRINGS:
        got = {}
        for mode in ("auto", "exchange"):
            eng = ArrowEngine(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, device=cuda_device,
                              mode=mode, semiring=semiring, add_identity=True)
            try:
                eng.set_features(_int_features(eng.n_rows, g.k, semiring, 3))
                eng.step()
                if not eng.fused_ok:
                    with pytest.raises(ValueError, match="sentinel"):
                        eng.predecessors()
                    continue
                D = eng.result()
                P = eng.predecessors()
                want = wr.predecessors(g.decomposition, g.width, D, semiring, block_diagonal=g.block_diagonal,
                                       n_blocks=eng.n_blocks)
                assert np.array_equal(P, want), f"{name} {semiring} {eng.mode}"
                assert np.array_equal(eng.result(), D) and np.array_equal(eng.predecessors(), P)    # repeatable
                got[eng.mode] = P
            finally:
                eng.close()
        if "fused" in got:
            assert np.array_equal(got["fused"], got["exchange"])


def _ba_decomposition(n, w, unit):
    A = sr.weighted_ba_graph(n, 3, seed=5, unit=unit)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    return A, dec


def _inv(perm0, rows0, n):
    inv = np.full(n, -1, np.int64)
    ok = perm0[:rows0] < n
    inv[perm0[:rows0][ok]] = np.flatnonzero(ok)
    return inv


def test_predecessors_leave_the_next_step_unchanged(cuda_device):
    """a twin engine that never calls predecessors() steps to the same bits, in fused and exchange mode"""
    n, w = 20000, 2000
    A, dec = _ba_decomposition(n, w, unit=False)
    for mode in ("auto", "exchange"):
        a = ArrowEngine(dec, w, 16, device=cuda_device, mode=mode, semiring="min_plus", add_identity=True)
        b = ArrowEngine(dec, w, 16, device=cuda_device, mode=mode, semiring="min_plus", add_identity=True)
        X = sr.source_features(decomp_perm0(dec, w, a), a.n_rows, n, np.arange(16) * 7)
        for e in (a, b):
            e.set_features(X)
            e.step()
        P1 = a.predecessors()
        for _ in range(3):
            a.step()
            b.step()
            assert np.array_equal(a.result().view(np.uint32), b.result().view(np.uint32)), mode
            assert np.array_equal(a.features().view(np.uint32), b.features().view(np.uint32)), mode
        assert (P1 >= 0).any()
        a.close()
        b.close()


def decomp_perm0(dec, w, eng):
    from arrow_matrix_b200 import decomp
    perms, _, _, _ = decomp.prepare_permutations([p for _, p in dec], eng.n_blocks, w)
    return perms[0]


def test_bfs_parents_are_one_level_closer(cuda_device):
    n, w = 30000, 3000
    A, dec = _ba_decomposition(n, w, unit=True)
    eng = ArrowEngine(dec, w, 8, device=cuda_device, semiring="min_plus", add_identity=True)
    perm0 = decomp_perm0(dec, w, eng)
    sources = np.random.default_rng(2).choice(n, 8, replace=False)
    eng.set_features(sr.source_features(perm0, eng.n_rows, n, sources))
    steps = eng.iterate_to_fixed_point(200)
    assert steps < 200
    D, P = eng.result(), eng.predecessors()
    vi, si = np.nonzero(P >= 0)
    assert np.array_equal(D[P[vi, si], si] + 1, D[vi, si])
    src = _inv(perm0, eng.n_rows, n)[sources]
    expect_none = ~np.isfinite(D)
    expect_none[src, np.arange(sources.size)] = True
    assert np.array_equal(P < 0, expect_none)
    hops = csgraph.shortest_path(A, method="D", unweighted=True, indices=sources).astype(np.float32)
    _check_chains(P, D, A, perm0, n, src, hops, "min_plus")
    eng.close()


def test_end_to_end_sssp_predecessors(cuda_device, tmp_path):
    """the 200k-vertex SSSP of test_gpu_semiring.test_end_to_end_sssp, then predecessors(): every parent is a tight edge
    and every chain reaches its source with the Dijkstra length"""
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
    from arrow_matrix_b200 import decomp
    perm0 = decomp.prepare_permutations([p for _, p in blocks.decomposition], blocks.n_blocks, w)[0][0]
    arrow.B.set_features(sr.source_features(perm0, eng.n_rows, n, sources))
    steps = eng.iterate_to_fixed_point(500)
    assert steps < 500
    D = arrow.B.result_tile()
    P = arrow.predecessors()
    assert P.dtype == np.int32 and P.shape == D.shape
    src = _inv(perm0, eng.n_rows, n)[sources]
    expect_none = ~np.isfinite(D)
    expect_none[src, np.arange(sources.size)] = True
    assert np.array_equal(P < 0, expect_none)
    dij = csgraph.shortest_path(A, method="D", indices=sources).astype(np.float32)
    _check_chains(P, D, A, perm0, n, src, dij, "min_plus")
    eng.close()


def test_refusals(cuda_device):
    g = GoldenCase(GPU_CASES[0])
    eng = ArrowEngine(g.decomposition, g.width, g.k, device=cuda_device)
    with pytest.raises(ValueError, match="min_plus / max_plus"):
        eng.predecessors()
    eng.close()
