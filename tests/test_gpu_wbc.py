"""Weighted betweenness on one GPU, held EXACTLY to the host restatement of tests/wpaths_ref.py: shortest_path_counts /
weighted_betweenness on the golden decompositions and remapped multi-level BA graphs with hubs (in- and out-lists longer
than a segment) at several widths, on one CTA and the default grid; bit equality with the or_and betweenness on unit
weights; predecessors() as the smallest tight in-neighbour; a second call; the features after the call; networkx on a
2k-vertex graph; +inf weights and overflowing sums; a loop cut short by max_steps; the loop-free adjacencies; and the
refusals."""
import networkx as nx
import numpy as np
import pytest
from scipy import sparse

from arrow_matrix_b200 import _lib
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from tests import bool_ref as br
from tests import push_ref as pr
from tests import semiring_ref as sr
from tests import wpaths_ref as wp
from tests.golden_util import GPU_CASES, GoldenCase

pytestmark = pytest.mark.gpu

ERR_ARG = -2
Ctx = _lib.Context
GRIDS = [("1 CTA", [(Ctx.OPT_SPMM_SM_LIMIT, 1), (Ctx.OPT_SPMM_CTAS_PER_SM, 1)]), ("default grid", [])]
DEFAULTS = [(Ctx.OPT_SPMM_SM_LIMIT, 0), (Ctx.OPT_SPMM_CTAS_PER_SM, 0)]
BIG = 10 ** 6


def _set_grid(ctx, opts):
    for o, v in DEFAULTS + opts:
        ctx.set_option(o, v)


def _exact(got, want, what):
    for g, w, name in zip(got, want, ("D", "sigma", "delta", "bc")):
        assert g.shape == w.shape, f"{what}: {name} shape"
        assert np.array_equal(g.view(np.uint64 if g.dtype == np.float64 else np.uint32),
                              w.view(np.uint64 if w.dtype == np.float64 else np.uint32)), \
            f"{what}: {int(np.sum(g != w))} elements of {name} differ"


def _reweigh(dec, seed, unit=False):
    """the decomposition with seeded integer weights 1..16 (or 1) on every entry"""
    rng = np.random.default_rng(seed)
    out = []
    for B, perm in dec:
        B = sparse.csr_matrix(B, dtype=np.float32, copy=True)
        B.data = np.ones(B.nnz, np.float32) if unit else rng.integers(1, 17, B.nnz).astype(np.float32)
        out.append((B, perm))
    return out


def _engine(dec, width, k, cuda_device, semiring="min_plus", **kw):
    return ArrowEngine(dec, width, k, device=cuda_device, semiring=semiring, add_identity=True, **kw)


def _parts(eng, dec, width, block_diagonal=True):
    p = br.BoolProtocol(dec, width, eng.k, block_diagonal=block_diagonal, n_blocks=eng.n_blocks, add_identity=True)
    return pr.protocol_parts(p)


def _sources(n, k, seed, offsets=False):
    rng = np.random.default_rng(seed)
    X0 = np.full((n, k), np.inf, np.float32)
    X0[rng.integers(0, n, k), np.arange(k)] = 0.0
    if offsets:                                       # a second source with an offset in every other column
        X0[rng.integers(0, n, k)[::2], np.arange(0, k, 2)] = rng.integers(0, 5, (k + 1) // 2).astype(np.float32)
    return X0


def _run(eng, X0, max_steps=BIG):
    """(D, sigma, delta, bc) of the engine's two calls from X0; checks that they agree"""
    eng.set_features(X0)
    D, sigma = eng.shortest_path_counts(max_steps)
    rounds = eng.last_path_rounds
    eng.set_features(X0)
    delta = np.full(sigma.shape, np.nan)
    bc = eng.weighted_betweenness(max_steps, dependencies_out=delta)
    assert eng.last_path_rounds == rounds
    D2 = eng.result()
    assert np.array_equal(D, D2)
    return D, sigma, delta, bc


def _want(parts, n, X0, D, max_steps=BIG):
    assert np.array_equal(D.view(np.uint32), wp.fixed_point(parts, n, X0, max_steps).view(np.uint32)), "distances"
    return wp.betweenness(parts, n, X0, max_steps, D=D)


@pytest.mark.parametrize("name", GPU_CASES)
def test_golden_decompositions_against_the_restatement(cuda_device, name):
    g = GoldenCase(name)
    dec = _reweigh(g.decomposition, 3)
    eng = _engine(dec, g.width, g.k, cuda_device, block_diagonal=g.block_diagonal)
    if not eng.fused_ok:
        eng.close()
        pytest.skip("a level reads rows behind the sentinel: no vertex identity")
    n = eng.n_rows
    X0 = _sources(n, g.k, 2, offsets=True)
    got = _run(eng, X0)
    parts = _parts(eng, dec, g.width, g.block_diagonal)
    eng.close()
    _exact(got, _want(parts, n, X0, got[0]), name)


@pytest.fixture(scope="module")
def ba_hubs():
    """a weighted BA graph with a vertex linked both ways to 1 200 others, decomposed in three levels (remapped)"""
    n, w = 6000, 500
    A = sr.weighted_ba_graph(n, 3, seed=7).tolil()
    rng = np.random.default_rng(3)
    hub = rng.choice(np.arange(1, n), 1200, replace=False)
    A[0, hub] = rng.integers(1, 17, hub.size).astype(np.float32)
    A[hub, 0] = rng.integers(1, 17, hub.size).astype(np.float32)
    A = sparse.csr_matrix(A)
    return arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2), w


@pytest.mark.parametrize("k", [1, 31, 32, 33, 128, 300])
def test_ba_with_hubs_every_width_and_grid(cuda_device, ba_hubs, k):
    dec, w = ba_hubs
    eng = _engine(dec, w, k, cuda_device)
    n = eng.n_rows
    parts = _parts(eng, dec, w)
    (ip, _, _), (op, _, _) = wp.adjacencies(parts, n)
    assert np.diff(ip).max() > 512 and np.diff(op).max() > 512, "no hub"
    X0 = _sources(n, k, k, offsets=True)
    want = None
    try:
        for grid, opts in GRIDS:
            _set_grid(eng.ctx, opts)
            got = _run(eng, X0)
            if want is None:
                want = _want(parts, n, X0, got[0])
            _exact(got, want, f"k={k} [{grid}]")
    finally:
        _set_grid(eng.ctx, [])
        eng.close()


@pytest.mark.parametrize("k", [16, 33])
def test_unit_weights_are_the_or_and_betweenness_bit_for_bit(cuda_device, ba_hubs, k):
    dec, w = ba_hubs
    dec = _reweigh(dec, 0, unit=True)
    eng = _engine(dec, w, k, cuda_device)
    bits_eng = _engine(dec, w, k, cuda_device, semiring="or_and")
    n = eng.n_rows
    X0 = _sources(n, k, 5)
    D, sigma, delta, bc = _run(eng, X0)
    bits_eng.set_features(X0 == 0)
    L, s2 = bits_eng.bfs_path_counts(BIG)
    bits_eng.zero_rhs()
    bits_eng.set_features(X0 == 0)
    d2 = np.empty_like(delta)
    bc2 = bits_eng.betweenness(BIG, dependencies_out=d2)
    eng.close()
    bits_eng.close()
    assert np.array_equal(np.where(np.isfinite(D), D, -1).astype(np.int32), L)
    for a, b in ((sigma, s2), (delta, d2), (bc, bc2)):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


def test_predecessors_are_the_smallest_tight_in_neighbour(cuda_device, ba_hubs):
    dec, w = ba_hubs
    k = 8
    eng = _engine(dec, w, k, cuda_device)
    n = eng.n_rows
    X0 = _sources(n, k, 9)
    eng.set_features(X0)
    D, sigma = eng.shortest_path_counts(BIG)
    P = eng.predecessors()
    parts = _parts(eng, dec, w)
    eng.close()
    in_lists, _ = wp.adjacencies(parts, n)
    S = wp.sources(D, X0)
    for v in range(n):
        lst, T = wp._tight_pairs(D, v, *in_lists, True)
        for s in range(k):
            if sigma[v, s] > 0 and not S[v, s]:
                assert P[v, s] == lst[T[:, s]].min(), (v, s)


def test_two_calls_and_the_features_after_the_call(cuda_device, ba_hubs):
    dec, w = ba_hubs
    k = 20
    eng = _engine(dec, w, k, cuda_device)
    n = eng.n_rows
    X0 = _sources(n, k, 4, offsets=True)
    first = _run(eng, X0)
    X1 = _sources(n, k, 6)
    _run(eng, X1)
    second = _run(eng, X0)
    _exact(second, first, "second call")
    eng.set_features(X0)
    steps = eng.iterate_to_fixed_point(BIG)
    dirs = list(eng.last_fixed_point_directions)
    plain = eng.result()
    eng.set_features(X0)
    eng.shortest_path_counts(BIG)
    assert eng.last_fixed_point_directions == dirs and len(dirs) == steps
    assert np.array_equal(eng.result().view(np.uint32), plain.view(np.uint32))
    # cut short by max_steps: everything is defined on the distances reached
    cut = _run(eng, X0, 2)
    parts = _parts(eng, dec, w)
    eng.close()
    _exact(cut, _want(parts, n, X0, cut[0], 2), "max_steps = 2")


def test_a_2k_vertex_graph_against_networkx(cuda_device):
    n, w, k = 2000, 250, 12
    A = sr.weighted_ba_graph(n, 3, seed=11)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=1)
    eng = _engine(dec, w, k, cuda_device)
    rows = eng.n_rows
    X0 = np.full((rows, k), np.inf, np.float32)
    src = np.random.default_rng(2).choice(rows, k, replace=False)
    X0[src, np.arange(k)] = 0.0
    _, sigma, _, bc = _run(eng, X0)
    parts = _parts(eng, dec, w)
    eng.close()
    G = nx.DiGraph()
    G.add_nodes_from(range(rows))
    for u, v, wt in zip(*[a.tolist() for a in wp.edges(parts)]):
        G.add_edge(u, v, weight=wt)
    nxbc = nx.betweenness_centrality_subset(G, sources=[int(s) for s in src], targets=list(range(rows)),
                                            normalized=False, weight="weight")
    np.testing.assert_allclose(bc, [nxbc[v] for v in range(rows)], rtol=1e-9, atol=1e-9)


def test_loop_free_adjacencies_and_refusals(cuda_device):
    ctx = _lib.Context(cuda_device)
    n = 300
    A = sparse.random(n, n, density=0.03, format="csr", random_state=1, dtype=np.float32)
    A.setdiag(2.0)
    A = sparse.csr_matrix(A)
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    in_adj = ctx.adj_build_loopfree([(dA, None)], n, direction="in")
    out_adj = ctx.adj_build_loopfree([(dA, None)], n)
    plain_in, plain_out = ctx.adj_build([(dA, None)], n, direction="in"), ctx.adj_build([(dA, None)], n)
    (ip, iu, iw), (op, ov, ow) = wp.adjacencies([(A, None)], n)
    got_in, got_out = in_adj.d2h(), out_adj.d2h()
    assert np.array_equal(got_in[0], ip) and np.array_equal(got_in[1], iu)
    assert np.array_equal(got_out[0], op) and np.array_equal(got_out[1], ov)
    assert np.array_equal(got_in[1], plain_in.d2h()[1]) and np.array_equal(got_out[1], plain_out.d2h()[1])
    assert np.array_equal(np.sort(out_adj.values_d2h()), np.sort(ow))
    k = 5
    x0, D = ctx.dense_alloc(n, k), ctx.dense_alloc(n, k)
    st, sig, dl = ctx.dense_alloc(n, k, np.int32), ctx.dense_alloc(n, k, np.float64), ctx.dense_alloc(n, k, np.float64)
    narrow = ctx.dense_alloc(n, k - 1, np.float64)
    try:
        def code(fn):
            with pytest.raises(_lib.ArrowError) as e:
                fn()
            return e.value.code
        x0.fill(float("inf"))
        D.fill(float("inf"))
        assert code(lambda: ctx.wpaths_dependencies(out_adj, x0, D, st, sig, dl)) == ERR_ARG      # no rounds kept
        assert code(lambda: ctx.wpaths_counts(out_adj, in_adj, x0, D, st, sig)) == ERR_ARG
        assert code(lambda: ctx.wpaths_counts(plain_in, out_adj, x0, D, st, sig)) == ERR_ARG
        assert code(lambda: ctx.wpaths_counts(in_adj, out_adj, x0, x0, st, sig)) == ERR_ARG      # aliasing
        assert code(lambda: ctx.wpaths_counts(in_adj, out_adj, x0, D, sig, st)) == ERR_ARG      # types
        assert code(lambda: ctx.wpaths_counts(in_adj, out_adj, x0, D, st, narrow)) == ERR_ARG   # shapes
        rounds, _ = ctx.wpaths_counts(in_adj, out_adj, x0, D, st, sig)
        assert rounds == 0                          # nothing finite: no row listed
        ctx.wpaths_dependencies(out_adj, x0, D, st, sig, dl)
        assert code(lambda: ctx.wpaths_dependencies(in_adj, x0, D, st, sig, dl)) == ERR_ARG
    finally:
        for h in (x0, D, st, sig, dl, narrow, in_adj, out_adj, plain_in, plain_out, dA):
            h.free()
        ctx.close()


@pytest.mark.parametrize("bad", [0.0, -0.0, -1.0, float("nan")])
def test_a_weight_that_is_not_positive_is_refused(cuda_device, bad):
    n, w = 64, 32
    A = sparse.random(n, n, density=0.1, format="csr", random_state=3, dtype=np.float32)
    A.data[:] = 1.0
    A.setdiag(0.0)                                   # stored diagonal zeros are self-loops: dropped, not refused
    A = sparse.csr_matrix(A)
    eng = _engine([(A, np.arange(n))], w, 2, cuda_device)
    assert not eng._nonpos_weight
    eng.close()
    c = A[0].indices[A[0].indices != 0][0]           # row 0 lies in the arrow's head: the entry is kept
    A[0, c] = bad
    eng = _engine([(A, np.arange(n))], w, 2, cuda_device)
    with pytest.raises(ValueError, match="> 0"):
        eng.weighted_betweenness(5)
    eng.close()


@pytest.mark.parametrize("case", ["infinite weights", "cut short"])
def test_small_cases_against_the_restatement(cuda_device, case):
    """+inf weights and an overflowing sum never count into an element that is not reached, even where another column of
    its row is reached; a successor left without paths by a cut-off adds nothing (every dependency finite)"""
    if case == "infinite weights":
        (parts, X0), steps = wp.infinite_weight_case(), BIG
    else:
        parts, X0, steps = wp.cut_short_case()
    A = parts[0][0]
    n = A.shape[0]
    eng = _engine([(A, np.arange(n))], 8, X0.shape[1], cuda_device)
    rows = eng.n_rows
    X = np.full((rows, X0.shape[1]), np.inf, np.float32)
    X[:n] = X0
    got = _run(eng, X, steps)
    host = _parts(eng, [(A, np.arange(n))], 8)
    eng.close()
    want = _want(host, rows, X, got[0], steps)
    _exact(got, want, case)
    assert np.all(np.isfinite(got[2])) and np.all(np.isfinite(got[3]))
    if case == "infinite weights":
        assert got[1][3].tolist() == [0.0, 1.0, 0.0]
