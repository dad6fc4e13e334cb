"""Betweenness on one GPU, held EXACTLY to the host restatement of tests/paths_ref.py: the path-count and dependency passes
driven level by level through the C ABI on hub graphs (in- and out-lists longer than a segment), remapped blocks and
duplicate entries at every width up to k = 8192 on one CTA and the default grid; bfs_path_counts / betweenness against
bfs_levels in every direction and mode on the golden decompositions and a BA graph with hubs; truncation, a second call,
the level-file path, and the refusals of the C ABI."""
import networkx as nx
import numpy as np
import pytest
from scipy import sparse

from arrow_matrix_b200 import _lib, decomp, graphio
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from tests import bool_ref as br
from tests import paths_ref as pa
from tests import push_ref as pr
from tests import semiring_ref as sr
from tests.golden_util import GPU_CASES, GoldenCase

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_HANDLE, ERR_UNSUPPORTED = -2, -3, -6
Ctx = _lib.Context
GRIDS = [("1 CTA", [(Ctx.OPT_SPMM_SM_LIMIT, 1), (Ctx.OPT_SPMM_CTAS_PER_SM, 1)]), ("default grid", [])]
DEFAULTS = [(Ctx.OPT_SPMM_SM_LIMIT, 0), (Ctx.OPT_SPMM_CTAS_PER_SM, 0)]
DIRECTIONS = {"push": 1 << 62, "pull": 0, "auto": None}      # ArrowEngine._push_limit
KS = [1, 5, 32, 33, 100, 128, 1000, 8192]
BIG = 10 ** 6


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


def _set_grid(ctx, opts):
    for o, v in DEFAULTS + opts:
        ctx.set_option(o, v)


def _assert_exact(got, want, what):
    for g, w, name in zip(got, want, ("levels", "sigma", "delta", "bc")):
        assert g.shape == w.shape, f"{what}: {name} shape"
        assert np.array_equal(g.view(np.uint64) if g.dtype == np.float64 else g,
                              w.view(np.uint64) if w.dtype == np.float64 else w), \
            f"{what}: {int(np.sum(g != w))} elements of {name} differ"


def _hub_matrix(n, seed, hub_deg=1500):
    """a sparse random graph with vertex 3 gathering from and vertex 5 feeding hub_deg others (lists of several
    segments); entry (r, c) is the edge c -> r"""
    rng = np.random.default_rng(seed)
    r, c = rng.integers(0, n, 4 * n), rng.integers(0, n, 4 * n)
    hub = rng.choice(n, hub_deg, replace=False)
    rows = np.r_[r, np.full(hub_deg, 3), hub]
    cols = np.r_[c, hub, np.full(hub_deg, 5)]
    A = sparse.csr_matrix((np.ones(rows.size, np.float32), (rows, cols)), shape=(n, n))
    A.sum_duplicates()
    return A


# ---- the C ABI driven level by level ---------------------------------------------------------------------------------
def _drive(ctx, adj, in_adj, L, counts=None, dep_counts=None):
    """levels L [n x k] -> (L, sigma, delta, bc) from the device passes: the bit tiles X_h = (0 <= L <= h) are marked level
    by level as a BFS would, sigma summed after each, every record kept, then the sweep and the row sum"""
    n, k = L.shape
    H = int(L.max(initial=0))
    tiles = [_bits(ctx, (L >= 0) & (L <= h)) for h in range(H + 1)]
    zero = _bits(ctx, np.zeros((n, k), bool))
    dist, sigma, delta = ctx.dense_alloc(n, k, np.int32), ctx.dense_alloc(n, k, np.float64), \
        ctx.dense_alloc(n, k, np.float64)
    bc = ctx.dense_alloc(n, 1, np.float64)
    try:
        sigma.fill(0.0)
        ctx.bits_fill_f64(tiles[0], zero, sigma, 1.0)
        ctx.bits_mark_frontier(adj, tiles[0], zero, dist, 0)
        ctx.adj_keep_record(adj, 0)
        for h in range(1, H + 1):
            ctx.bits_mark_frontier(adj, tiles[h], tiles[h - 1], dist, h)
            got = ctx.bits_path_counts(in_adj, adj, tiles[h], tiles[h - 1], sigma, count=True)
            if counts is not None:
                counts.append(got)
            ctx.adj_keep_record(adj, h)
        dist.h2d(L)
        delta.fill(0.0)
        for h in range(H, 0, -1):
            got = ctx.bits_dependencies(adj, h, dist, sigma, delta, count=True)
            if dep_counts is not None:
                dep_counts.insert(0, got)
        ctx.row_sum(delta, bc)
        return dist.d2h(), sigma.d2h(), delta.d2h(), bc.d2h().reshape(-1)
    finally:
        for t in tiles + [zero, dist, sigma, delta, bc]:
            t.free()


def _restated(parts, n, X0, max_steps=BIG):
    L, sigma, delta, bc, _ = pa.betweenness(parts, n, X0, max_steps)
    return L, sigma, delta, bc


@pytest.fixture(scope="module")
def hub_graph(ctx):
    n = 1200
    A = _hub_matrix(n, 12, hub_deg=1100)
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    adj = ctx.adj_build([(dA, None)], n)
    in_adj = ctx.adj_build([(dA, None)], n, direction="in")
    ip, _ = pa.adjacencies([(A, None)], n)[0]
    assert np.diff(ip).max() > 1024 and np.diff(pr.adjacency([(A, None)], n)[0]).max() > 1024
    yield A, adj, in_adj
    for h in (in_adj, adj, dA):
        h.free()


@pytest.mark.parametrize("k", KS)
def test_passes_on_a_hub_graph_against_the_restatement(ctx, hub_graph, k):
    A, adj, in_adj = hub_graph
    n = A.shape[0]
    rng = np.random.default_rng(k)
    X0 = rng.random((n, k)) < min(0.3, 2.0 / n + 1.0 / k)
    want = _restated([(A, None)], n, X0)
    L = want[0]
    in_deg = np.diff(pa.adjacencies([(A, None)], n)[0][0].astype(np.int64))
    out_deg = np.diff(pr.adjacency([(A, None)], n)[0].astype(np.int64))
    pad = np.full((n, -k % 32), -2, np.int32)
    words = np.concatenate([L, pad], axis=1).reshape(n, -1, 32)           # [n x words x 32]
    # every list entry of a (row, word) holding the level is read exactly once, whether one warp or its segments read it
    want_in = [int(np.sum(np.any(words == h, axis=2).sum(axis=1) * in_deg)) for h in range(1, L.max() + 1)]
    want_out = [int(np.sum(np.any(words == h, axis=2).sum(axis=1) * out_deg)) for h in range(1, L.max() + 1)]
    assert np.any(L[3] >= 1) and np.any(L[5] >= 1), "the hubs are not reached"
    try:
        for grid, opts in GRIDS:
            _set_grid(ctx, opts)
            counts, dep_counts = [], []
            got = _drive(ctx, adj, in_adj, L, counts, dep_counts)
            _assert_exact(got, want, f"k={k} [{grid}]")
            assert counts == want_in and dep_counts == want_out, f"k={k} [{grid}]"
    finally:
        _set_grid(ctx, [])


def test_passes_on_remapped_blocks_with_duplicate_entries(ctx):
    """a block with a partial column map, uploaded twice: every edge is listed twice and counts once"""
    rng = np.random.default_rng(4)
    n, k = 4000, 33
    A = _hub_matrix(n, 5, hub_deg=700)
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    cmap = rng.permutation(n).astype(np.int64)
    cmap[::11] = -1
    dm = ctx.map_upload(cmap, n)
    dAs = dA.remap_columns(dm, n)
    As = A.copy()
    As.indices = cmap[A.indices].astype(np.int64)
    parts = [(As, None), (As, None), (A, None)]
    adj = ctx.adj_build([(dAs, None), (dAs, None), (dA, None)], n)
    in_adj = ctx.adj_build([(dAs, None), (dAs, None), (dA, None)], n, direction="in")
    X0 = rng.random((n, k)) < 0.002
    want = _restated(parts, n, X0)
    assert np.array_equal(want[1], _restated(parts[1:], n, X0)[1])
    for grid, opts in GRIDS:
        _set_grid(ctx, opts)
        _assert_exact(_drive(ctx, adj, in_adj, want[0]), want, f"remapped [{grid}]")
    _set_grid(ctx, [])
    for h in (in_adj, adj, dAs, dA, dm):
        h.free()


def test_path_counts_round_past_2_53_as_restated(ctx):
    """40 chained three-way gadgets: sigma = 3^40 rounded on the way, bit for bit the ordered restatement"""
    m = 40
    us, vs = [], []
    for i in range(m):
        for b in (4 * i + 1, 4 * i + 2, 4 * i + 3):
            us += [4 * i, b]
            vs += [b, 4 * i + 4]
    n = 4 * m + 1
    A = sparse.csr_matrix((np.ones(len(us), np.float32), (vs, us)), shape=(n, n))
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    adj, in_adj = ctx.adj_build([(dA, None)], n), ctx.adj_build([(dA, None)], n, direction="in")
    X0 = np.zeros((n, 2), bool)
    X0[0, 0] = X0[4, 1] = True
    want = _restated([(A, None)], n, X0)
    assert int(want[1][n - 1, 0]) != 3 ** m
    _assert_exact(_drive(ctx, adj, in_adj, want[0]), want, "gadgets")
    for h in (in_adj, adj, dA):
        h.free()


# ---- the engine ------------------------------------------------------------------------------------------------------
def _engine(dec, width, k, cuda_device, mode="auto", block_diagonal=True, limit=None):
    eng = ArrowEngine(dec, width, k, block_diagonal=block_diagonal, device=cuda_device, mode=mode, semiring="or_and",
                      add_identity=True)
    eng._push_limit = limit
    return eng


def _run(eng, X0, max_steps):
    """(levels, sigma, delta, bc, steps, directions) from the engine's three calls, each from X0"""
    eng.zero_rhs()
    eng.set_features(X0)
    L, sigma = eng.bfs_path_counts(max_steps)
    steps, dirs = eng.last_bfs_steps, list(eng.last_bfs_directions)
    eng.zero_rhs()
    eng.set_features(X0)
    delta = np.full(sigma.shape, np.nan)
    bc = eng.betweenness(max_steps, dependencies_out=delta)
    assert eng.last_bfs_steps == steps and eng.last_bfs_directions == dirs
    return (L, sigma, delta, bc), steps, dirs


def _levels(eng, X0, max_steps):
    eng.zero_rhs()
    eng.set_features(X0)
    L = eng.bfs_levels(max_steps)
    return L, eng.last_bfs_steps, list(eng.last_bfs_directions)


@pytest.mark.parametrize("name", GPU_CASES)
def test_golden_decompositions_every_direction_and_mode(cuda_device, name):
    g = GoldenCase(name)
    probe = _engine(g.decomposition, g.width, g.k, cuda_device, block_diagonal=g.block_diagonal)
    fused_ok, n, n_blocks = probe.fused_ok, probe.n_rows, probe.n_blocks
    probe.close()
    if not fused_ok:
        pytest.skip("a level reads rows behind the sentinel: no vertex identity")
    X0 = np.random.default_rng(2).random((n, g.k)) < 0.02
    p = br.BoolProtocol(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, n_blocks=n_blocks,
                        add_identity=True)
    want = _restated(pr.protocol_parts(p), n, X0, 100)
    for mode in ("auto", "exchange"):
        for label, limit in DIRECTIONS.items():
            eng = _engine(g.decomposition, g.width, g.k, cuda_device, mode=mode, block_diagonal=g.block_diagonal,
                          limit=limit)
            L, steps, dirs = _levels(eng, X0, 100)
            got, steps2, dirs2 = _run(eng, X0, 100)
            tag = f"{name} {eng.mode} {label}"
            assert steps2 == steps and dirs2 == dirs, tag
            assert np.array_equal(L, got[0]), tag
            _assert_exact(got, want, tag)
            eng.close()


@pytest.fixture(scope="module")
def ba_hubs():
    """a BA graph with a vertex linked both ways to 1 200 others, decomposed in three levels"""
    n, w = 6000, 500
    A = sr.weighted_ba_graph(n, 3, seed=7, unit=True).tolil()
    hub = np.random.default_rng(3).choice(np.arange(1, n), 1200, replace=False)
    A[0, hub] = 1.0
    A[hub, 0] = 1.0
    A = sparse.csr_matrix(A)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    return dec, w


@pytest.mark.parametrize("k", [1, 33, 128, 1000])
def test_ba_with_hubs_every_direction_and_grid(cuda_device, ba_hubs, k):
    dec, w = ba_hubs
    eng = _engine(dec, w, k, cuda_device)
    n = eng.n_rows
    p = br.BoolProtocol(dec, w, k, n_blocks=eng.n_blocks, add_identity=True)
    parts = pr.protocol_parts(p)
    ip, op = pa.adjacencies(parts, n)[0][0], pr.adjacency(parts, n)[0]
    assert np.diff(ip).max() > 512 and np.diff(op).max() > 512, "no hub"
    rng = np.random.default_rng(k)
    X0 = np.zeros((n, k), bool)
    X0[rng.integers(0, n, k), np.arange(k)] = True
    want = _restated(parts, n, X0)
    try:
        for grid, opts in GRIDS:
            _set_grid(eng.ctx, opts)
            for label, limit in DIRECTIONS.items():
                eng._push_limit = limit
                L, steps, dirs = _levels(eng, X0, BIG)
                got, steps2, dirs2 = _run(eng, X0, BIG)
                tag = f"k={k} {label} [{grid}]"
                assert steps2 == steps and dirs2 == dirs and np.array_equal(L, got[0]), tag
                _assert_exact(got, want, tag)
    finally:
        _set_grid(eng.ctx, [])
        eng.close()


def test_truncation_and_a_second_call_leave_nothing_behind(cuda_device):
    """two components; a full run from the first, then one from the second cut short by max_steps: equal to a fresh
    engine's and to the truncated restatement"""
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
    _run(eng, X1, 100)
    got, steps, _ = _run(eng, X2, 3)
    n_blocks = eng.n_blocks
    eng.close()
    assert steps == 3 and np.any(got[0] == -1)
    fresh = _engine(dec, w, k, cuda_device)
    got0, _, _ = _run(fresh, X2, 3)
    fresh.close()
    _assert_exact(got, got0, "second call")
    p = br.BoolProtocol(dec, w, k, n_blocks=n_blocks, add_identity=True)
    _assert_exact(got, _restated(pr.protocol_parts(p), rows, X2, 3), "truncated")


def test_betweenness_through_the_level_files(cuda_device, tmp_path):
    """20k-vertex BA graph -> level files -> load -> betweenness of 16 one-hot columns: the restatement bit for bit, and
    networkx's Brandes betweenness (twice the undirected figure) in vertex order"""
    n, w, k = 20000, 2000, 16
    A = sr.weighted_ba_graph(n, 3, seed=5, unit=True)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, w, True)
    sources = np.random.default_rng(8).choice(n, k, replace=False)
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, w, True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, w, k, 'gpu', True, True,
                                             semiring="or_and", add_identity=True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    eng = arrow._engine
    perm0 = np.asarray(decomp.prepare_permutations([p for _, p in blocks.decomposition], blocks.n_blocks, w)[0][0],
                       dtype=np.int64)
    X0 = br.source_bits(perm0, eng.n_rows, n, sources)
    arrow.B.set_features(X0)
    L, sigma = arrow.bfs_path_counts(500)
    eng.zero_rhs()
    arrow.B.set_features(X0)
    delta = np.empty(sigma.shape)
    bc = arrow.betweenness(500, dependencies_out=delta)
    p = br.BoolProtocol(blocks.decomposition, w, k, n_blocks=eng.n_blocks, add_identity=True)
    want = _restated(pr.protocol_parts(p), eng.n_rows, X0, 500)
    eng.close()
    _assert_exact((L, sigma, delta, bc), want, "level files")
    G = nx.from_scipy_sparse_array(A)
    nxbc = nx.betweenness_centrality_subset(G, sources=[int(s) for s in sources], targets=list(range(n)),
                                            normalized=False)
    bcv = br.vertex_order(bc[:, None], perm0, n, np.nan)[:, 0]
    np.testing.assert_allclose(bcv, 2 * np.array([nxbc[v] for v in range(n)]), rtol=1e-10, atol=1e-9)


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_abi_refusals(ctx, hub_graph):
    A, adj, in_adj = hub_graph
    n, k = A.shape[0], 40
    X, Y = ctx.dense_alloc(n, k, _lib.BITS), ctx.dense_alloc(n, k, _lib.BITS)
    D, F32 = ctx.dense_alloc(n, k, np.int32), ctx.dense_alloc(n, k)
    S, T = ctx.dense_alloc(n, k, np.float64), ctx.dense_alloc(n, k, np.float64)
    S_narrow, S_short = ctx.dense_alloc(n, k - 1, np.float64), ctx.dense_alloc(n - 1, k, np.float64)
    bc, bc2 = ctx.dense_alloc(n, 1, np.float64), ctx.dense_alloc(n, 2, np.float64)
    fresh = ctx.adj_build([], n)
    other = ctx.adj_build([], n + 1, direction="in")
    try:
        # no record
        assert _code(lambda: ctx.bits_path_counts(in_adj, fresh, X, Y, S)) == ERR_ARG
        assert _code(lambda: ctx.adj_keep_record(fresh, 0)) == ERR_ARG
        ctx.bits_mark_frontier(adj, X, Y, D, 1)
        ctx.bits_path_counts(in_adj, adj, X, Y, S)
        # the adjacency kinds
        assert _code(lambda: ctx.bits_path_counts(adj, in_adj, X, Y, S)) == ERR_ARG
        assert _code(lambda: ctx.bits_path_counts(in_adj, in_adj, X, Y, S)) == ERR_ARG
        assert _code(lambda: ctx.bits_path_counts(adj, adj, X, Y, S)) == ERR_ARG
        assert _code(lambda: ctx.bits_path_counts(other, adj, X, Y, S)) == ERR_ARG
        assert _code(lambda: ctx.adj_keep_record(in_adj, 0)) == ERR_ARG
        assert _code(lambda: ctx.bits_dependencies(in_adj, 1, D, S, T)) == ERR_ARG
        weighted = ctx.adj_build([], n, weighted=True)
        assert _code(lambda: ctx.bits_dependencies(weighted, 1, D, S, T)) == ERR_ARG
        weighted.free()
        # the record of another tile, aliasing
        assert _code(lambda: ctx.bits_path_counts(in_adj, adj, Y, X, S)) == ERR_ARG
        assert _code(lambda: ctx.bits_path_counts(in_adj, adj, X, X, S)) == ERR_ARG
        # dtypes and shapes
        for bad in (D, F32, Y, S_narrow, S_short):
            assert _code(lambda: ctx.bits_path_counts(in_adj, adj, X, Y, bad)) == ERR_ARG
        assert _code(lambda: ctx.bits_path_counts(in_adj, adj, X, F32, S)) == ERR_ARG
        # the history: level 0 first, then in order; the sweep reads levels 1 .. kept - 1
        assert _code(lambda: ctx.adj_keep_record(adj, 1)) == ERR_ARG
        ctx.adj_keep_record(adj, 0)
        assert _code(lambda: ctx.adj_keep_record(adj, 2)) == ERR_ARG
        assert _code(lambda: ctx.bits_dependencies(adj, 1, D, S, T)) == ERR_ARG
        ctx.adj_keep_record(adj, 1)
        ctx.bits_dependencies(adj, 1, D, S, T)
        assert _code(lambda: ctx.bits_dependencies(adj, 0, D, S, T)) == ERR_ARG
        assert _code(lambda: ctx.bits_dependencies(adj, 2, D, S, T)) == ERR_ARG
        assert _code(lambda: ctx.bits_dependencies(adj, 1, D, S, S)) == ERR_ARG          # delta aliases sigma
        for d, s, t in ((S, S, T), (D, D, T), (D, S, D), (D, F32, T), (D, S_narrow, T), (D, S, S_short)):
            assert _code(lambda: ctx.bits_dependencies(adj, 1, d, s, t)) == ERR_ARG
        # the masked write and the row sum
        for bad in (D, F32, Y, S_narrow):
            assert _code(lambda: ctx.bits_fill_f64(X, Y, bad, 1.0)) == ERR_ARG
        assert _code(lambda: ctx.bits_fill_f64(S, Y, T, 1.0)) == ERR_ARG
        for x, out in ((S, bc2), (S, S), (F32, bc), (S, S_short), (D, bc)):
            assert _code(lambda: ctx.row_sum(x, out)) == ERR_ARG
        assert _code(lambda: ctx.row_sum(bc, bc)) == ERR_ARG                             # out aliases in
        W, Wo = ctx.dense_alloc(n, 8193, _lib.BITS), ctx.dense_alloc(n, 8193, _lib.BITS)
        Wd, Ws = ctx.dense_alloc(n, 8193, np.int32), ctx.dense_alloc(n, 8193, np.float64)
        ctx.bits_mark_frontier(adj, W, Wo, Wd, 1)
        assert _code(lambda: ctx.bits_path_counts(in_adj, adj, W, Wo, Ws)) == ERR_UNSUPPORTED
        for h in (W, Wo, Wd, Ws):
            h.free()
        fresh.free()
        assert _code(lambda: ctx.bits_path_counts(in_adj, fresh, X, Y, S)) == ERR_HANDLE
        assert _code(lambda: ctx.adj_keep_record(fresh, 0)) == ERR_HANDLE
    finally:
        for h in (other, X, Y, D, F32, S, T, S_narrow, S_short, bc, bc2):
            h.free()
