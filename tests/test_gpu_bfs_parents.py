"""BFS parents on one GPU, held EXACTLY to the host restatement of tests/parents_ref.py: the in-adjacency word for word,
the parent pass at every row shape (one-word rows, padded rows, k not a multiple of 32, k = 8192) on one CTA and the
default grid, a hub row split into segments, bfs_tree against bfs_levels in every direction, against the (min, +)
predecessors on unit weights, and a 200k-vertex BFS validated against scipy."""
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
from tests import parents_ref as par
from tests import push_ref as pr
from tests import semiring_ref as sr
from tests.golden_util import GPU_CASES, GoldenCase

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_HANDLE, ERR_RANGE, ERR_UNSUPPORTED = -2, -3, -4, -6
Ctx = _lib.Context
GRIDS = [("1 CTA", [(Ctx.OPT_SPMM_SM_LIMIT, 1), (Ctx.OPT_SPMM_CTAS_PER_SM, 1)]), ("default grid", [])]
DEFAULTS = [(Ctx.OPT_SPMM_SM_LIMIT, 0), (Ctx.OPT_SPMM_CTAS_PER_SM, 0)]
DIRECTIONS = {"push": 1 << 62, "pull": 0, "auto": None}      # ArrowEngine._push_limit
# one-word rows, then one uint4 and 2, 3, 5, 9, 17, 33 and 64 of them per row (every lanes-per-edge shape), with k not a
# multiple of 32 on both sides
KS = [1, 5, 31, 32, 33, 128, 129, 384, 513, 1025, 2049, 4097, 8192]
SENTINEL = 0x5A5A5A5A


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


def _unit(decomposition):
    out = []
    for B, p in decomposition:
        B = sparse.csr_matrix(B, copy=True)
        B.data = np.ones_like(B.data, dtype=np.float32)
        out.append((B, p))
    return out


def _engine(dec, width, k, cuda_device, mode="auto", block_diagonal=True, limit=None, semiring="or_and"):
    eng = ArrowEngine(dec, width, k, block_diagonal=block_diagonal, device=cuda_device, mode=mode, semiring=semiring,
                      add_identity=True)
    eng._push_limit = limit
    return eng


def _assert_adj(got, want, label):
    assert np.array_equal(got[0], want[0]), f"{label}: row pointers differ"
    assert np.array_equal(got[1], want[1]), f"{label}: {int(np.sum(got[1] != want[1]))} sources differ"


# ---- the in-adjacency ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", GPU_CASES)
def test_in_adjacency_of_golden_decompositions(cuda_device, name):
    g = GoldenCase(name)
    eng = _engine(g.decomposition, g.width, g.k, cuda_device, block_diagonal=g.block_diagonal)
    p = br.BoolProtocol(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, n_blocks=eng.n_blocks,
                        add_identity=True)
    parts = [(st.csr, st.cmap_dev) for st in eng.levels]
    adj = eng.ctx.adj_build(parts, eng.n_rows, direction="in")
    _assert_adj(adj.d2h(), par.in_adjacency(pr.protocol_parts(p), eng.n_rows), name)
    adj.free()
    eng.close()


def test_in_adjacency_of_a_ba_decomposition_with_hubs(cuda_device):
    n, w = 30000, 1000
    A = sr.weighted_ba_graph(n, 3, seed=7, unit=True)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    eng = _engine(dec, w, 4, cuda_device)
    p = br.BoolProtocol(dec, w, 4, n_blocks=eng.n_blocks, add_identity=True)
    eng.set_features(np.eye(eng.n_rows, 4, dtype=bool))
    eng.bfs_tree(3)                                            # builds the in-adjacency
    got = eng._in_adj.d2h()
    assert np.diff(got[0]).max() > 512, "no hub row"
    _assert_adj(got, par.in_adjacency(pr.protocol_parts(p), eng.n_rows), "BA 30k")
    assert eng._in_adj.info() == {"n_vertices": eng.n_rows, "n_edges": got[1].size}
    assert eng._in_adj.info() == eng._push_adjacency().info()
    eng.close()


def test_in_adjacency_of_a_remapped_copy(ctx):
    rng = np.random.default_rng(4)
    n = 5000
    A = sparse.random(n, n, density=0.002, format="csr", random_state=5, dtype=np.float32)
    A = (A + sparse.eye(n, dtype=np.float32, format="csr")).tocsr()            # the diagonal is dropped
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    cmap = rng.permutation(n).astype(np.int64)
    cmap[::3] = -1
    dm = ctx.map_upload(cmap, n)
    dAs = dA.remap_columns(dm, n)
    As = A.copy()
    As.indices = cmap[A.indices].astype(np.int64)
    adj = ctx.adj_build([(dAs, None)], n, direction="in")
    _assert_adj(adj.d2h(), par.in_adjacency([(As, None)], n), "remapped")
    rmap = rng.permutation(n + 100)[:n].astype(np.int64)
    rmap[::7] = -1
    dr = ctx.map_upload(rmap, n + 100)
    adj2 = ctx.adj_build([(dA, dr), (dA, None)], n + 100, direction="in")
    _assert_adj(adj2.d2h(), par.in_adjacency([(A, rmap), (A, None)], n + 100), "two parts")
    for h in (adj2, adj, dAs, dA, dm, dr):
        h.free()


# ---- the parent pass -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hub_graph(ctx):
    """12 000 vertices, about 6 edges each, a vertex with 10 500 sources (row 7 of the in-adjacency) and one with 10 500
    destinations; (device push adjacency, device in-adjacency, host in-adjacency)"""
    rng = np.random.default_rng(12)
    n = 12000
    r = rng.integers(0, n, 6 * n)
    c = rng.integers(0, n, 6 * n)
    hub = rng.choice(n, 10500, replace=False)
    # entry (r, c) is the edge c -> r: row 7 gathers from 10 500 columns, column 9 feeds 10 500 rows
    rows = np.r_[r, np.full(hub.size, 7), hub]
    cols = np.r_[c, hub, np.full(hub.size, 9)]
    A = sparse.csr_matrix((np.ones(rows.size, np.float32), (rows, cols)), shape=(n, n))
    A.sum_duplicates()
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    adj = ctx.adj_build([(dA, None)], n)
    in_adj = ctx.adj_build([(dA, None)], n, direction="in")
    host = par.in_adjacency([(A, None)], n)
    _assert_adj(in_adj.d2h(), host, "hub graph")
    assert np.diff(host[0])[7] > 10000
    yield adj, in_adj, host
    for h in (in_adj, adj, dA):
        h.free()


def _frontiers(n, rng):
    return {"hub": np.array([7]), "1 %": rng.choice(n, n // 100, replace=False), "all": np.arange(n)}


@pytest.mark.parametrize("k", KS)
def test_parents_against_the_restatement(ctx, hub_graph, k):
    """random X_old, X_new = X_old | (random bits on the frontier rows): parents where an in-neighbour holds the bit, -1
    where none does, everything else untouched"""
    adj, in_adj, host = hub_graph
    n = host[0].size - 1
    rng = np.random.default_rng(k)
    dNew, dOld = ctx.dense_alloc(n, k, _lib.BITS), ctx.dense_alloc(n, k, _lib.BITS)
    dP, dd = ctx.dense_alloc(n, k, np.int32), ctx.dense_alloc(n, k, np.int32)
    try:
        for label, F in _frontiers(n, rng).items():
            old = rng.random((n, k)) < min(0.05, 40.0 / k)
            new = old.copy()
            new[F] |= rng.random((F.size, k)) < 0.3
            new[F, k - 1] |= ~old[F, k - 1]                    # every frontier row holds a fresh bit, the last column too
            dNew.h2d(br.pack(new))
            dOld.h2d(br.pack(old))
            ctx.bits_mark_frontier(adj, dNew, dOld, dd, 1)
            want = par.level_parents(new, old, host, np.full((n, k), SENTINEL, np.int32))
            for grid, opts in GRIDS:
                for o, v in DEFAULTS + opts:
                    ctx.set_option(o, v)
                dP.h2d(np.full((n, k), SENTINEL, np.int32))
                scanned = ctx.bits_parents(in_adj, adj, dNew, dOld, dP, count=True)
                got = dP.d2h()
                assert np.array_equal(got, want), f"k={k} {label} [{grid}]: {int(np.sum(got != want))} elements differ"
                assert 0 < scanned <= int(np.sum(np.diff(host[0].astype(np.int64))[F]))
    finally:
        for o, v in DEFAULTS:
            ctx.set_option(o, v)
        for h in (dNew, dOld, dP, dd):
            h.free()


@pytest.mark.parametrize("k", [16, 128, 4097])
def test_a_split_hub_row_finds_its_parent_in_the_last_segment(ctx, hub_graph, k):
    """row 7 has 10 500 in-edges (21 segments); bit s of it is fresh and only its largest source holds s"""
    adj, in_adj, host = hub_graph
    n = host[0].size - 1
    ins = host[1][host[0][7]:host[0][8]]
    old = np.zeros((n, k), bool)
    new = np.zeros((n, k), bool)
    old[ins[-1], k - 1] = True
    old[ins[-2], 0] = True                                     # and one in the second to last position
    new[7, [0, k - 1]] = True
    dNew, dOld, dP, dd = _bits(ctx, new), _bits(ctx, old), ctx.dense_alloc(n, k, np.int32), ctx.dense_alloc(n, k, np.int32)
    for grid, opts in GRIDS:
        for o, v in DEFAULTS + opts:
            ctx.set_option(o, v)
        dP.h2d(np.full((n, k), SENTINEL, np.int32))
        ctx.bits_mark_frontier(adj, dNew, dOld, dd, 1)
        ctx.bits_parents(in_adj, adj, dNew, dOld, dP)
        got = dP.d2h()
        want = np.full((n, k), SENTINEL, np.int32)
        want[7, 0], want[7, k - 1] = ins[-2], ins[-1]
        assert np.array_equal(got, want), grid
    for o, v in DEFAULTS:
        ctx.set_option(o, v)
    for h in (dNew, dOld, dP, dd):
        h.free()


def test_abi_refusals(ctx, hub_graph):
    adj, in_adj, host = hub_graph
    n, k = host[0].size - 1, 40
    A_, B_ = ctx.dense_alloc(n, k, _lib.BITS), ctx.dense_alloc(n, k, _lib.BITS)
    P, D, F = ctx.dense_alloc(n, k, np.int32), ctx.dense_alloc(n, k, np.int32), ctx.dense_alloc(n, k)
    P_narrow, P_short = ctx.dense_alloc(n, k - 1, np.int32), ctx.dense_alloc(n - 1, k, np.int32)
    fresh = ctx.adj_build([], n)
    other = ctx.adj_build([], n + 1, direction="in")
    assert _code(lambda: ctx.bits_parents(in_adj, fresh, A_, B_, P)) == ERR_ARG      # no record
    ctx.bits_mark_frontier(adj, A_, B_, D, 1)
    ctx.bits_parents(in_adj, adj, A_, B_, P)
    assert _code(lambda: ctx.bits_parents(adj, in_adj, A_, B_, P)) == ERR_ARG        # swapped
    assert _code(lambda: ctx.bits_parents(in_adj, in_adj, A_, B_, P)) == ERR_ARG
    assert _code(lambda: ctx.bits_parents(adj, adj, A_, B_, P)) == ERR_ARG
    assert _code(lambda: ctx.bits_parents(other, adj, A_, B_, P)) == ERR_ARG         # other vertex count
    assert _code(lambda: ctx.bits_parents(in_adj, adj, B_, A_, P)) == ERR_ARG        # a record for another tile
    assert _code(lambda: ctx.bits_parents(in_adj, adj, A_, A_, P)) == ERR_ARG        # new == old
    assert _code(lambda: ctx.bits_parents(in_adj, adj, A_, F, P)) == ERR_ARG         # a float tile
    assert _code(lambda: ctx.bits_parents(in_adj, adj, A_, B_, B_)) == ERR_ARG       # a bit parent tile
    assert _code(lambda: ctx.bits_parents(in_adj, adj, A_, B_, F)) == ERR_ARG        # a float parent tile
    assert _code(lambda: ctx.bits_parents(in_adj, adj, A_, B_, P_narrow)) == ERR_ARG
    assert _code(lambda: ctx.bits_parents(in_adj, adj, A_, B_, P_short)) == ERR_ARG
    # every other call taking an adjacency refuses the in-adjacency
    assert _code(lambda: ctx.bits_mark_frontier(in_adj, A_, B_, D, 1)) == ERR_ARG
    assert _code(lambda: ctx.bits_push_frontier(in_adj, A_, B_)) == ERR_ARG
    assert _code(lambda: ctx.sr_mark_frontier(in_adj, F, F)) == ERR_ARG
    assert _code(lambda: ctx.sr_push_frontier(in_adj, F, F, _lib.SR_MIN_PLUS)) == ERR_ARG
    assert _code(lambda: in_adj.values_d2h()) == ERR_ARG
    with pytest.raises(ValueError):
        ctx.adj_build([], n, weighted=True, direction="in")
    W, Wo, Wd = ctx.dense_alloc(n, 8193, _lib.BITS), ctx.dense_alloc(n, 8193, _lib.BITS), ctx.dense_alloc(n, 8193, np.int32)
    ctx.bits_mark_frontier(adj, W, Wo, Wd, 1)
    assert _code(lambda: ctx.bits_parents(in_adj, adj, W, Wo, Wd)) == ERR_UNSUPPORTED
    fresh.free()
    assert _code(lambda: ctx.bits_parents(in_adj, fresh, A_, B_, P)) == ERR_HANDLE
    for h in (other, W, Wo, Wd, A_, B_, P, D, F, P_narrow, P_short):
        h.free()


def test_in_adjacency_refusals(ctx):
    n = 64
    A = sparse.random(n, n, density=0.1, format="csr", random_state=1, dtype=np.float32)
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    short = ctx.map_upload(np.arange(n - 1), n)
    wide = ctx.map_upload(np.arange(n), n + 10)
    assert _code(lambda: ctx.adj_build([(dA, short)], n, direction="in")) == ERR_ARG
    assert _code(lambda: ctx.adj_build([(dA, wide)], n, direction="in")) == ERR_ARG
    assert _code(lambda: ctx.adj_build([(dA, None)], n - 1, direction="in")) == ERR_ARG
    ctx.sync()
    ctx.graph_begin()
    code = _code(lambda: ctx.adj_build([(dA, None)], n, direction="in"))
    ctx.graph_free(ctx.graph_end())
    assert code == ERR_UNSUPPORTED
    rows, per = 1 << 14, 1 << 12                               # 2**31 edges or more, refused after counting
    ip = np.arange(0, rows * per + 1, per, dtype=np.int64)
    big = ctx.csr_upload(rows, rows, ip, np.tile(np.arange(per, dtype=np.int32), rows), None)
    assert _code(lambda: ctx.adj_build([(big, None)] * 33, rows, direction="in")) == ERR_RANGE
    for h in (big, wide, short, dA):
        h.free()


# ---- bfs_tree ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", GPU_CASES)
def test_bfs_tree_every_direction_and_the_min_plus_parents(cuda_device, name):
    """levels, steps and directions of bfs_levels under forced push, forced pull and the rule; P the same in every
    direction, the restatement's, and a min_plus engine's predecessors() on unit values, in auto and exchange mode"""
    g = GoldenCase(name)
    probe = _engine(g.decomposition, g.width, g.k, cuda_device, block_diagonal=g.block_diagonal)
    fused_ok, n, n_blocks = probe.fused_ok, probe.n_rows, probe.n_blocks
    probe.close()
    if not fused_ok:
        pytest.skip("a level reads rows behind the sentinel: no parents")
    X0 = np.random.default_rng(2).random((n, g.k)) < 0.02
    p = br.BoolProtocol(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, n_blocks=n_blocks,
                        add_identity=True)
    parts = pr.protocol_parts(p)
    want_L, want_P, _ = par.bfs_tree(par.in_adjacency(parts, n), pr.adjacency(parts, n), X0, 100)
    for mode in ("auto", "exchange"):
        mp = _engine(_unit(g.decomposition), g.width, g.k, cuda_device, mode=mode, block_diagonal=g.block_diagonal,
                     semiring="min_plus")
        mp.set_features(np.where(X0, 0.0, np.inf).astype(np.float32))
        mp.iterate_to_fixed_point(100)
        P_mp = mp.predecessors()
        mp.close()
        assert np.array_equal(P_mp, want_P), f"{name} {mode}: min_plus parents"
        for label, limit in DIRECTIONS.items():
            eng = _engine(g.decomposition, g.width, g.k, cuda_device, mode=mode, block_diagonal=g.block_diagonal,
                          limit=limit)
            eng.set_features(X0)
            L = eng.bfs_levels(100)
            steps, dirs = eng.last_bfs_steps, list(eng.last_bfs_directions)
            result = eng.result()
            eng.zero_rhs()
            eng.set_features(X0)
            L2, P = eng.bfs_tree(100)
            tag = f"{name} {eng.mode} {label}"
            assert np.array_equal(L2, L) and np.array_equal(L, want_L), tag
            assert eng.last_bfs_steps == steps and eng.last_bfs_directions == dirs, tag
            assert np.array_equal(eng.result(), result), tag
            assert np.array_equal(P, want_P), f"{tag}: {int(np.sum(P != want_P))} parents differ"
            if eng.mode == "exchange" and eng.L == 1:
                assert set(dirs) == {"pull"}, tag
            elif label != "auto":
                assert set(dirs) == {label}, tag
            eng.close()


def test_second_call_leaves_no_parents_behind(cuda_device):
    """two components; a BFS from the first, then one from the second with max_steps cutting it short: the second P
    is a fresh engine's"""
    n, w = 4000, 200
    A = sr.weighted_ba_graph(n // 2, 3, seed=3, unit=True)
    A = sparse.block_diag([A, A], format="csr")
    dec = arrow_decomposition(A, w, max_number_of_levels=2, block_diagonal=True, seed=1)
    k = 8
    eng = _engine(dec, w, k, cuda_device)
    rows = eng.n_rows
    rng = np.random.default_rng(1)
    X1, X2 = np.zeros((rows, k), bool), np.zeros((rows, k), bool)
    X1[rng.choice(rows, k), np.arange(k)] = True
    X2[rng.choice(rows, k), np.arange(k)] = True
    eng.set_features(X1)
    eng.bfs_tree(100)
    eng.zero_rhs()
    eng.set_features(X2)
    L, P = eng.bfs_tree(3)
    eng.close()
    fresh = _engine(dec, w, k, cuda_device)
    fresh.set_features(X2)
    L0, P0 = fresh.bfs_tree(3)
    fresh.close()
    assert np.array_equal(L, L0) and np.array_equal(P, P0)
    assert np.any(L == -1)


@pytest.mark.parametrize("k", [16, 128])
def test_bfs_tree_through_the_level_files_is_a_graph500_tree(cuda_device, tmp_path, k):
    """200k-vertex BA graph -> level files -> load -> bfs_tree, validated like Graph500: every source is its own root
    (-1), every reached vertex's parent is an edge one hop closer (scipy) and the smallest such level-0 row, unreached
    vertices have none"""
    n, w = 200000, 20000
    A = sr.weighted_ba_graph(n, 3, seed=5, unit=True)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, w, True)
    sources = np.random.default_rng(8).choice(n, k, replace=False)
    hops = csgraph.shortest_path(A, unweighted=True, indices=sources)               # [k x n]
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, w, True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, w, k, 'gpu', True, True,
                                             semiring="or_and", add_identity=True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    eng = arrow._engine
    perm0 = np.asarray(decomp.prepare_permutations([p for _, p in blocks.decomposition], blocks.n_blocks, w)[0][0],
                       dtype=np.int64)
    arrow.B.set_features(br.source_bits(perm0, eng.n_rows, n, sources))
    L, P = arrow.bfs_tree(500)
    eng.close()
    want = np.where(np.isinf(hops), -1, hops).astype(np.int32)
    assert np.array_equal(br.vertex_order(L, perm0, n, -1).T, want)
    Pv = br.vertex_order(P, perm0, n, -2).T
    assert not np.any(Pv == -2)
    m = min(eng.n_rows, perm0.size)
    label_vertex = np.full(eng.n_rows, -1, np.int64)
    label_vertex[:m] = np.where(perm0[:m] < n, perm0[:m], -1)
    inv = np.full(n, -1, np.int64)
    ok = label_vertex >= 0
    inv[label_vertex[ok]] = np.arange(eng.n_rows)[ok]
    A = sparse.csr_matrix(A)
    src = np.repeat(np.arange(n), np.diff(A.indptr))
    for s in range(k):
        h = hops[s]
        assert Pv[s, sources[s]] == -1
        assert np.all(Pv[s, np.isinf(h)] == -1)
        reached = np.isfinite(h) & (h > 0)
        assert np.all(Pv[s, reached] >= 0)
        u = label_vertex[Pv[s, reached]]                                           # parents as vertex ids
        v = np.flatnonzero(reached)
        assert np.all(u >= 0) and np.all(h[u] == h[v] - 1)
        assert np.all(np.asarray(A[v, u]).ravel() != 0), "a parent that is not an edge"
        # the smallest label among the in-neighbours one hop closer
        cols = A.indices
        closer = (h[cols] == h[src] - 1) & np.isfinite(h[src]) & (h[src] > 0)
        best = np.full(n, np.iinfo(np.int64).max)
        np.minimum.at(best, src[closer], inv[cols[closer]])
        assert np.array_equal(Pv[s, reached], best[reached])
