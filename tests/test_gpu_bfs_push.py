"""The direction-optimising BFS on one GPU, held EXACTLY to the host restatement of tests/push_ref.py: the push adjacency
word for word, the frontier push at every feature width (padding words included), and bfs_levels under forced push,
forced pull and the automatic rule against each other, the restated arrow step and scipy."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200 import _lib, decomp, graphio
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from tests import bool_ref as br
from tests import push_ref as pr
from tests import semiring_ref as sr
from tests.golden_util import GPU_CASES, GoldenCase

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_HANDLE, ERR_RANGE, ERR_UNSUPPORTED = -2, -3, -4, -6
Ctx = _lib.Context
GRIDS = [("1 CTA", [(Ctx.OPT_SPMM_SM_LIMIT, 1), (Ctx.OPT_SPMM_CTAS_PER_SM, 1)]), ("default grid", [])]
DEFAULTS = [(Ctx.OPT_SPMM_SM_LIMIT, 0), (Ctx.OPT_SPMM_CTAS_PER_SM, 0)]
ALL_PUSH, ALL_PULL = 1 << 62, 0          # ArrowEngine._push_limit: push iff the frontier's edges are fewer


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(cuda_device)
    yield c
    c.close()


def _code(fn):
    with pytest.raises(_lib.ArrowError) as e:
        fn()
    return e.value.code


def _bits(ctx, X):
    d = ctx.dense_alloc(X.shape[0], X.shape[1], _lib.BITS)
    d.h2d(br.pack(X))
    return d


def _protocol(g, k, n_blocks=None):
    return br.BoolProtocol(g.decomposition, g.width, k, block_diagonal=g.block_diagonal,
                           n_blocks=g.n_blocks if n_blocks is None else n_blocks, add_identity=True)


def _engine(dec, width, k, cuda_device, mode="auto", block_diagonal=True, limit=None):
    eng = ArrowEngine(dec, width, k, block_diagonal=block_diagonal, device=cuda_device, mode=mode, semiring="or_and",
                      add_identity=True)
    eng._push_limit = limit
    return eng


def _assert_adj(got, want, label):
    assert np.array_equal(got[0], want[0]), f"{label}: row pointers differ"
    assert np.array_equal(got[1], want[1]), f"{label}: {int(np.sum(got[1] != want[1]))} destinations differ"


# ---- the adjacency ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", GPU_CASES)
def test_adjacency_of_golden_decompositions(cuda_device, name):
    g = GoldenCase(name)
    eng = _engine(g.decomposition, g.width, g.k, cuda_device, block_diagonal=g.block_diagonal)
    p = _protocol(g, g.k, eng.n_blocks)
    assert eng.fused_ok == pr.fused_ok(p)
    if eng.fused_ok:
        _assert_adj(eng._push_adjacency().d2h(), pr.adjacency(pr.protocol_parts(p), eng.n_rows), name)
    eng.close()


def test_adjacency_of_a_ba_decomposition_with_hubs(cuda_device):
    n, w = 30000, 1000
    A = sr.weighted_ba_graph(n, 3, seed=7, unit=True)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    eng = _engine(dec, w, 4, cuda_device)
    p = br.BoolProtocol(dec, w, 4, n_blocks=eng.n_blocks, add_identity=True)
    assert eng.fused_ok and eng.L == 3
    got = eng._push_adjacency().d2h()
    assert np.diff(got[0]).max() > 512, "no hub row"
    _assert_adj(got, pr.adjacency(pr.protocol_parts(p), eng.n_rows), "BA 30k")
    assert eng._adj.info() == {"n_vertices": eng.n_rows, "n_edges": got[1].size}
    eng.close()


def test_adjacency_of_a_random_block_and_a_remapped_copy(ctx):
    rng = np.random.default_rng(4)
    n = 5000
    A = sparse.random(n, n, density=0.002, format="csr", random_state=5, dtype=np.float32)
    A = (A + sparse.eye(n, dtype=np.float32, format="csr")).tocsr()            # the diagonal is dropped
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    adj = ctx.adj_build([(dA, None)], n)
    T = sparse.csr_matrix(A.T)
    T.setdiag(0)
    T.eliminate_zeros()
    T.sort_indices()
    _assert_adj(adj.d2h(), (T.indptr.astype(np.int32), T.indices.astype(np.int32)), "identity")
    adj.free()
    # a remapped copy: columns through a map with -1 entries (those entries are skipped)
    cmap = rng.permutation(n).astype(np.int64)
    cmap[::3] = -1
    dm = ctx.map_upload(cmap, n)
    dAs = dA.remap_columns(dm, n)
    As = A.copy()
    As.indices = cmap[A.indices].astype(np.int64)
    adj = ctx.adj_build([(dAs, None)], n)
    _assert_adj(adj.d2h(), pr.adjacency([(As, None)], n), "remapped")
    assert adj.info()["n_edges"] < T.nnz
    # a row map of both ends, and two parts
    rmap = rng.permutation(n + 100)[:n].astype(np.int64)
    rmap[::7] = -1
    dr = ctx.map_upload(rmap, n + 100)
    adj2 = ctx.adj_build([(dA, dr), (dA, None)], n + 100)
    _assert_adj(adj2.d2h(), pr.adjacency([(A, rmap), (A, None)], n + 100), "two parts")
    for h in (adj2, adj, dAs, dA, dm, dr):
        h.free()


def test_adjacency_refusals(ctx):
    n = 64
    A = sparse.random(n, n, density=0.1, format="csr", random_state=1, dtype=np.float32)
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    short = ctx.map_upload(np.arange(n - 1), n)
    wide = ctx.map_upload(np.arange(n), n + 10)
    assert _code(lambda: ctx.adj_build([(dA, short)], n)) == ERR_ARG           # a map shorter than the block
    assert _code(lambda: ctx.adj_build([(dA, wide)], n)) == ERR_ARG            # a map reaching past the vertices
    assert _code(lambda: ctx.adj_build([(dA, None)], n - 1)) == ERR_ARG        # an identity block past the vertices
    ctx.adj_build([(dA, wide)], n + 10).free()
    ctx.sync()
    ctx.graph_begin()
    code = _code(lambda: ctx.adj_build([(dA, None)], n))
    ctx.graph_free(ctx.graph_end())
    assert code == ERR_UNSUPPORTED
    # 2**31 edges or more: 33 parts of 2**26 - 2**12 edges each, refused after counting
    rows, per = 1 << 14, 1 << 12
    ip = np.arange(0, rows * per + 1, per, dtype=np.int64)
    big = ctx.csr_upload(rows, rows, ip, np.tile(np.arange(per, dtype=np.int32), rows), None)
    assert _code(lambda: ctx.adj_build([(big, None)] * 33, rows)) == ERR_RANGE
    adj = ctx.adj_build([(big, None)] * 2, rows)
    assert adj.info()["n_edges"] == 2 * (rows * per - per)
    for h in (adj, big, wide, short, dA):
        h.free()


# ---- the frontier record and the push --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hub_graph(ctx):
    """12 000 vertices, about 6 edges each, and a hub row of 10 500 destinations; (device adjacency, host adjacency)"""
    rng = np.random.default_rng(12)
    n = 12000
    r = rng.integers(0, n, 6 * n)
    c = rng.integers(0, n, 6 * n)
    hub = rng.choice(n, 10500, replace=False)
    # entry (r, c) is the edge c -> r: the hub is column 7 of 10 500 rows
    A = sparse.csr_matrix((np.ones(r.size + hub.size, np.float32), (np.r_[r, hub], np.r_[c, np.full(hub.size, 7)])),
                          shape=(n, n))
    A.sum_duplicates()
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    adj = ctx.adj_build([(dA, None)], n)
    host = pr.adjacency([(A, None)], n)
    _assert_adj(adj.d2h(), host, "hub graph")
    assert np.diff(host[0])[7] > 10000
    yield adj, host
    adj.free()
    dA.free()


def _frontiers(n, rng):
    return {"empty": np.zeros(0, np.int64), "hub": np.array([7]), "1 %": rng.choice(n, n // 100, replace=False),
            "all": np.arange(n)}


@pytest.mark.parametrize("k", br.SWEEP_KS)
def test_push_against_the_restatement(ctx, hub_graph, k):
    adj, host = hub_graph
    n = host[0].size - 1
    rng = np.random.default_rng(k)
    X = rng.random((n, k)) < min(0.05, 40.0 / k)
    dist0 = rng.integers(-3, 9, (n, k)).astype(np.int32)
    dX, dOld, dOut = _bits(ctx, X), ctx.dense_alloc(n, k, _lib.BITS), ctx.dense_alloc(n, k, _lib.BITS)
    dd, dd2 = ctx.dense_alloc(n, k, np.int32), ctx.dense_alloc(n, k, np.int32)
    try:
        for label, F in _frontiers(n, rng).items():
            Xf = X.copy()
            Xf[F, 0] = True                          # every frontier row holds a bit
            old = Xf.copy()
            old[F] = False
            dX.h2d(br.pack(Xf))
            dOld.h2d(br.pack(old))
            dd.h2d(dist0)
            dd2.h2d(dist0)
            n_new, rows, edges = ctx.bits_mark_frontier(adj, dX, dOld, dd, 5)
            assert (n_new, rows, edges) == (int((Xf & ~old).sum()), F.size, pr.frontier_edges(F, host)), label
            # the level record and the count are arrow_bits_mark_new's
            assert ctx.bits_mark_new(dX, dOld, dd2, 5) == n_new
            if label == "1 %" or k <= 128:
                assert np.array_equal(dd.d2h(), dd2.d2h()), label
            want = br.pack(pr.push(Xf, F, host))
            for grid, opts in GRIDS:
                for o, v in DEFAULTS + opts:
                    ctx.set_option(o, v)
                dOut.h2d(np.full((n, br.words(k)), 0xA5C35A3C, np.uint32))
                ctx.bits_push_frontier(adj, dX, dOut)
                got = dOut.d2h()
                assert np.array_equal(got, want), f"k={k} {label} [{grid}]: {int(np.any(got != want, axis=1).sum())} rows"
    finally:
        for o, v in DEFAULTS:
            ctx.set_option(o, v)
        for h in (dX, dOld, dOut, dd, dd2):
            h.free()


def test_push_refusals(ctx, hub_graph):
    adj, host = hub_graph
    n, k = host[0].size - 1, 40
    A_, B_ = ctx.dense_alloc(n, k, _lib.BITS), ctx.dense_alloc(n, k, _lib.BITS)
    C_, small = ctx.dense_alloc(n, k, _lib.BITS), ctx.dense_alloc(n - 1, k, _lib.BITS)
    narrow, F = ctx.dense_alloc(n, k - 8, _lib.BITS), ctx.dense_alloc(n, k)
    D, D_small = ctx.dense_alloc(n, k, np.int32), ctx.dense_alloc(n - 1, k, np.int32)
    fresh = ctx.adj_build([], n)
    assert fresh.info() == {"n_vertices": n, "n_edges": 0}
    assert _code(lambda: ctx.bits_push_frontier(fresh, A_, B_)) == ERR_ARG          # no record
    assert _code(lambda: ctx.bits_mark_frontier(adj, small, small, D_small, 1)) == ERR_ARG   # rows of another graph
    assert _code(lambda: ctx.bits_mark_frontier(adj, A_, F, D, 1)) == ERR_ARG       # a float tile
    ctx.bits_mark_frontier(adj, A_, C_, D, 1)
    assert _code(lambda: ctx.bits_push_frontier(adj, B_, C_)) == ERR_ARG            # a record tagged with another tile
    assert _code(lambda: ctx.bits_push_frontier(adj, A_, A_)) == ERR_ARG            # out == x
    assert _code(lambda: ctx.bits_push_frontier(adj, A_, small)) == ERR_ARG         # shape
    assert _code(lambda: ctx.bits_push_frontier(adj, A_, narrow)) == ERR_ARG        # k
    assert _code(lambda: ctx.bits_push_frontier(adj, A_, F)) == ERR_ARG            # a float tile
    ctx.bits_push_frontier(adj, A_, B_)
    ctx.bits_mark_frontier(adj, B_, C_, D, 1)                                         # the record moves to B
    assert _code(lambda: ctx.bits_push_frontier(adj, A_, C_)) == ERR_ARG
    ctx.bits_push_frontier(adj, B_, C_)
    W, Wo, Wd = ctx.dense_alloc(n, 8193, _lib.BITS), ctx.dense_alloc(n, 8193, _lib.BITS), ctx.dense_alloc(n, 8193, np.int32)
    ctx.bits_mark_frontier(adj, W, Wo, Wd, 1)
    assert _code(lambda: ctx.bits_push_frontier(adj, W, Wo)) == ERR_UNSUPPORTED
    fresh.free()
    assert _code(lambda: ctx.bits_push_frontier(fresh, A_, B_)) == ERR_HANDLE
    for h in (W, Wo, Wd, A_, B_, C_, small, narrow, F, D, D_small):
        h.free()


# ---- bfs_levels --------------------------------------------------------------------------------------------------------
DIRECTIONS = {"push": ALL_PUSH, "pull": ALL_PULL, "auto": None}


@pytest.mark.parametrize("name", GPU_CASES)
def test_bfs_levels_every_direction_on_golden_decompositions(cuda_device, name):
    """forced push, forced pull and the rule: the restated level record, the same steps and result(), twice per engine;
    one more step() after it gives the same result(j) at every level.  Decompositions with stale rows pull only."""
    g = GoldenCase(name)
    for mode in ("auto", "exchange"):
        runs = {}
        for label, limit in DIRECTIONS.items():
            eng = _engine(g.decomposition, g.width, g.k, cuda_device, mode=mode, block_diagonal=g.block_diagonal,
                          limit=limit)
            X0 = np.random.default_rng(2).random((eng.n_rows, g.k)) < 0.02
            for rep in range(2):
                p = _protocol(g, g.k, eng.n_blocks)
                p.set_features(X0)
                want, steps = p.bfs_levels(100)
                if rep:
                    eng.zero_rhs()
                eng.set_features(X0)
                got = eng.bfs_levels(100)
                tag = f"{name} {eng.mode} {label} call {rep}"
                assert np.array_equal(got, want) and eng.last_bfs_steps == steps, tag
                assert len(eng.last_bfs_directions) == steps, tag
                if not eng.fused_ok:
                    assert set(eng.last_bfs_directions) == {"pull"}, tag
                elif label != "auto":
                    assert set(eng.last_bfs_directions) == {label}, tag
            result = eng.result()
            assert np.array_equal(result, p.X[0]), f"{name} {eng.mode} {label}: result()"
            eng.step()
            runs[label] = [eng.result(j) for j in range(eng.L)]
            eng.close()
        for label in ("push", "auto"):
            for j in range(g.L):
                assert np.array_equal(runs[label][j], runs["pull"][j]), f"{name} {mode} {label}: result({j}) after step()"


@pytest.mark.parametrize("k", [128, 16])
def test_bfs_levels_through_the_level_files(cuda_device, tmp_path, k):
    """200k-vertex BA graph -> level files -> load: the scipy hop counts under the rule, forced push and forced pull; the
    rule takes both directions"""
    n, w = 200000, 20000
    A = sr.weighted_ba_graph(n, 3, seed=5, unit=True)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, w, True)
    sources = np.random.default_rng(8).choice(n, k, replace=False)
    hops = csgraph.shortest_path(A, unweighted=True, indices=sources)
    want = np.where(np.isinf(hops), -1, hops).astype(np.int32)
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, w, True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, w, k, 'gpu', True, True,
                                             semiring="or_and", add_identity=True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    eng = arrow._engine
    assert eng.fused_ok
    perm0 = decomp.prepare_permutations([p for _, p in blocks.decomposition], blocks.n_blocks, w)[0][0]
    X0 = br.source_bits(perm0, eng.n_rows, n, sources)
    runs = {}
    for label, limit in DIRECTIONS.items():
        eng._push_limit = limit
        eng.zero_rhs()
        arrow.B.set_features(X0)
        levels = arrow.bfs_levels(500)
        got = br.vertex_order(levels, perm0, n, -1).T
        assert np.array_equal(got, want), f"k={k} {label}: {int(np.sum(got != want))} levels differ"
        runs[label] = (eng.last_bfs_steps, list(eng.last_bfs_directions), eng.result())
    assert runs["push"][0] == runs["pull"][0] == runs["auto"][0]
    assert np.array_equal(runs["push"][2], runs["pull"][2]) and np.array_equal(runs["auto"][2], runs["pull"][2])
    assert set(runs["auto"][1]) == {"push", "pull"}, runs["auto"][1]
    eng.close()
