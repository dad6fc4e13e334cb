"""CPU tests of the weighted betweenness of the min-plus engine: the host restatement (tests/wpaths_ref.py) against
networkx's weighted Brandes (per-column path counts and betweenness) on every golden decomposition and random graphs,
against the unweighted restatement on unit weights bit for bit, an absorbed weight, a multi-source column with offsets,
+inf weights and overflowing sums, a loop cut short by max_steps, the weight scan, and the refusals of shortest_path_counts / weighted_betweenness before any CUDA work."""
import networkx as nx
import numpy as np
import pytest
from networkx.algorithms.centrality.betweenness import _single_source_dijkstra_path_basic
from scipy import sparse

from arrow_matrix_b200 import _lib
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from tests import bool_ref as br
from tests import paths_ref as pa
from tests import push_ref as pr
from tests import semiring_ref as sr
from tests import wpaths_ref as wp
from tests.golden_util import CASES, GoldenCase

BIG = 10 ** 6


def _weighted(parts, seed):
    """the parts with seeded integer weights 1..16 on their entries"""
    rng = np.random.default_rng(seed)
    out = []
    for A, m in parts:
        A = sparse.csr_matrix(A, dtype=np.float32, copy=True)
        A.data = rng.integers(1, 17, A.nnz).astype(np.float32)
        out.append((A, m))
    return out


def _digraph(parts, n):
    """edge u -> v for every entry, of the smallest weight among its duplicates"""
    G = nx.DiGraph()
    G.add_nodes_from(range(n))
    for u, v, w in zip(*[a.tolist() for a in wp.edges(parts)]):
        if not G.has_edge(u, v) or G[u][v]["weight"] > w:
            G.add_edge(u, v, weight=w)
    return G


def _one_hot(n, k, seed):
    rows = np.random.default_rng(seed).choice(n, k, replace=False)
    X0 = np.full((n, k), np.inf, np.float32)
    X0[rows, np.arange(k)] = 0.0
    return X0, rows


def _check_networkx(parts, n, k, seed):
    X0, rows = _one_hot(n, k, seed)
    D, sigma, delta, bc = wp.betweenness(parts, n, X0, BIG)
    G = _digraph(parts, n)
    for s, src in enumerate(rows):
        _, _, nx_sigma, nx_dist = _single_source_dijkstra_path_basic(G, int(src), "weight")
        # networkx adds the source's count to itself (it is popped as its own predecessor): every count is doubled
        want_sigma = np.array([nx_sigma[v] / nx_sigma[int(src)] if v in nx_dist else 0.0 for v in range(n)])
        want_D = np.array([nx_dist.get(v, np.inf) for v in range(n)])
        assert np.array_equal(D[:, s], want_D.astype(np.float32))
        np.testing.assert_allclose(sigma[:, s], want_sigma, rtol=1e-9)
    nxbc = nx.betweenness_centrality_subset(G, sources=[int(r) for r in rows], targets=list(G.nodes), normalized=False,
                                            weight="weight")
    np.testing.assert_allclose(bc, [nxbc[v] for v in range(n)], rtol=1e-9, atol=1e-9)
    return D, sigma, delta


@pytest.mark.parametrize("name", CASES)
def test_restatement_is_networkx_weighted_brandes_on_golden_decompositions(name):
    g = GoldenCase(name)
    p = br.BoolProtocol(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, n_blocks=g.n_blocks,
                        add_identity=True)
    n = p.rows[0]
    _check_networkx(_weighted(pr.protocol_parts(p), 3), n, min(g.k, n), 4)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restatement_is_networkx_weighted_brandes_on_random_graphs(seed):
    n = 300
    A = sparse.random(n, n, density=0.02, format="csr", random_state=seed, dtype=np.float32)
    A.data = np.random.default_rng(seed).integers(1, 17, A.nnz).astype(np.float32)
    D, sigma, _ = _check_networkx([(A, None)], n, 8, seed)
    assert np.any(sigma > 1), "no ties: the counts are not exercised"


def test_restatement_is_networkx_on_a_weighted_ba_graph():
    A = sr.weighted_ba_graph(800, 3, seed=5)
    dec = arrow_decomposition(A, 100, max_number_of_levels=3, block_diagonal=True, seed=2)
    p = br.BoolProtocol(dec, 100, 4, add_identity=True)
    parts = [(p.mats[j].astype(np.float32), m) for j, (_, m) in enumerate(pr.protocol_parts(p))]
    # arrow_mask keeps the values of the weighted matrix
    assert np.any(parts[0][0].data > 1)
    _check_networkx(parts, p.rows[0], 6, 1)


@pytest.mark.parametrize("name", CASES)
def test_unit_weights_are_the_unweighted_betweenness_bit_for_bit(name):
    g = GoldenCase(name)
    p = br.BoolProtocol(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, n_blocks=g.n_blocks,
                        add_identity=True)
    n = p.rows[0]
    parts = [(sparse.csr_matrix((np.ones(A.nnz, np.float32), A.indices, A.indptr), shape=A.shape), m)
             for A, m in pr.protocol_parts(p)]
    bits = np.random.default_rng(2).random((n, g.k)) < 0.05
    X0 = np.where(bits, np.float32(0), np.float32(np.inf))
    D, sigma, delta, bc = wp.betweenness(parts, n, X0, BIG)
    L, s2, d2, bc2, _ = pa.betweenness(parts, n, bits, BIG)
    assert np.array_equal(np.where(np.isfinite(D), D, -1).astype(np.int64), L)
    for a, b in ((sigma, s2), (delta, d2), (bc, bc2)):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


def test_an_absorbed_weight_is_not_tight():
    """fl(1 + 2^25) == 2^25: the edge 1 -> 2 of weight 1 relaxes nothing and is not tight (equal distances)"""
    big = np.float32(2 ** 25)
    A = sparse.csr_matrix((np.array([big, 1.0, big], np.float32), (np.array([1, 2, 2]), np.array([0, 1, 0]))),
                          shape=(3, 3))
    X0 = np.array([[0.0], [np.inf], [np.inf]], np.float32)
    D, sigma, delta, _ = wp.betweenness([(A, None)], 3, X0, BIG)
    assert D[1, 0] == big and D[2, 0] == big and np.float32(1) + big == big
    assert sigma[:, 0].tolist() == [1.0, 1.0, 1.0]                 # 2 counts only 0 -> 2
    assert delta[:, 0].tolist() == [0.0, 0.0, 0.0]


def test_a_multi_source_column_with_offsets_is_one_super_source():
    """X0 holding offsets at several rows of a column == one source S* = row n with an edge of weight X0[v] to each of
    them: the distances, counts and the dependencies of every other row equal; the sources' own dependencies are 0"""
    n = 400
    A = sparse.random(n, n, density=0.02, format="csr", random_state=7, dtype=np.float32)
    A.data = np.random.default_rng(7).integers(1, 9, A.nnz).astype(np.float32)
    rng = np.random.default_rng(3)
    src = rng.choice(n, 5, replace=False)
    off = np.array([0, 2, 3, 3, 7], np.float32)
    X0 = np.full((n, 1), np.inf, np.float32)
    X0[src, 0] = off
    D, sigma, delta, _ = wp.betweenness([(A, None)], n, X0, BIG)
    S = wp.sources(D, X0)[:, 0]
    assert S.sum() >= 2
    # S* reaches src[i] at offset off[i]; an offset of 0 is the source itself in the super-source graph, so offsets get +1
    u, v, w = wp.edges([(A, None)])
    su = np.concatenate([u, np.full(src.size, n)])
    sv = np.concatenate([v, src])
    sw = np.concatenate([w, off + 1])
    B = sparse.csr_matrix((sw, (sv, su)), shape=(n + 1, n + 1))
    Xs = np.full((n + 1, 1), np.inf, np.float32)
    Xs[n, 0] = 0.0
    Ds, ss, ds, _ = wp.betweenness([(B, None)], n + 1, Xs, BIG)
    fin = np.isfinite(D[:, 0])
    assert np.array_equal(D[fin, 0] + 1, Ds[:n, 0][fin])
    assert np.array_equal(sigma[:, 0], ss[:n, 0])
    assert np.array_equal(delta[~S, 0], ds[:n, 0][~S]) and np.all(delta[S, 0] == 0)


def test_duplicate_entries_count_once():
    n = 300
    A = sparse.random(n, n, density=0.03, format="csr", random_state=4, dtype=np.float32)
    A.data = np.random.default_rng(4).integers(1, 5, A.nnz).astype(np.float32)
    heavier = A.copy()
    heavier.data = heavier.data + 3                            # never tight beside the lighter duplicate
    X0, _ = _one_hot(n, 6, 2)
    once = wp.betweenness([(A, None)], n, X0, BIG)
    twice = wp.betweenness([(heavier, None), (A, None), (A, None)], n, X0, BIG)
    for a, b in zip(once, twice):
        assert np.array_equal(a, b)


class _TwoRanks(SelfComm):
    def Get_size(self) -> int:
        return 2


class _NoCuda:
    pass


@pytest.fixture
def no_cuda(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a CUDA call was made")
    monkeypatch.setattr(_lib.Context, "__init__", refuse)
    monkeypatch.setattr(_lib, "load_library", refuse)


def _bare_engine(semiring, add_identity, fused_ok, nonpos=False):
    """an ArrowEngine without a device: only what the weighted path calls check before their first CUDA call"""
    eng = object.__new__(ArrowEngine)
    eng.sr, eng.semiring, eng.add_identity, eng.fused_ok = _lib.SEMIRINGS[semiring], semiring, add_identity, fused_ok
    eng._nonpos_weight = nonpos
    eng.k = 3

    class _Level:
        rows = 8
    eng.levels = [_Level()]
    return eng


@pytest.mark.parametrize("call", ["shortest_path_counts", "weighted_betweenness"])
def test_refusals_happen_before_any_cuda_call(no_cuda, call):
    for semiring in ("max_plus", "plus_times", "or_and"):
        with pytest.raises(ValueError, match="min_plus"):
            getattr(_bare_engine(semiring, True, True), call)(10)
    with pytest.raises(ValueError, match="add_identity"):
        getattr(_bare_engine("min_plus", False, True), call)(10)
    with pytest.raises(ValueError, match="sentinel"):
        getattr(_bare_engine("min_plus", True, False), call)(10)
    with pytest.raises(ValueError, match="> 0"):
        getattr(_bare_engine("min_plus", True, True, nonpos=True), call)(10)
    arrow = ArrowDecompositionMPI.initialize(_TwoRanks(), [4, 4], None, None, 8, 4, 'gpu', True, True,
                                             semiring="min_plus", add_identity=True)
    with pytest.raises(ValueError, match="one GPU"):
        getattr(arrow, call)(10)
    arrow = ArrowDecompositionMPI.initialize(SelfComm(), [4, 4], None, None, 8, 4, 'gpu', True, True,
                                             semiring="min_plus", add_identity=True)
    with pytest.raises(RuntimeError, match="not loaded"):
        getattr(arrow, call)(10)
    arrow._engine = _NoCuda()
    with pytest.raises(ValueError, match="one GPU"):
        getattr(arrow, call)(10)


def test_output_arrays_are_checked_before_any_cuda_call(no_cuda):
    eng = _bare_engine("min_plus", True, True)
    for out in (np.zeros(16)[::2], np.zeros(8, np.float32), np.zeros(7), np.zeros((8, 1))):
        with pytest.raises(ValueError, match="out must be"):
            eng.weighted_betweenness(10, out=out)
    for dep in (np.zeros((8, 6))[:, ::2], np.zeros((8, 3), np.float32), np.zeros((3, 8))):
        with pytest.raises(ValueError, match="dependencies_out must be"):
            eng.weighted_betweenness(10, dependencies_out=dep)


def test_the_unweighted_calls_keep_refusing_min_plus(no_cuda):
    with pytest.raises(ValueError, match="or_and"):
        _bare_engine("min_plus", True, True).betweenness(10)


def test_an_infinite_weight_or_an_overflowing_sum_is_never_tight():
    parts, X0 = wp.infinite_weight_case()
    D, sigma, delta, bc = wp.betweenness(parts, 6, X0, BIG)
    assert D[3].tolist() == [np.inf, 1.0, np.inf] and D[5].tolist() == [np.inf, 2.0, np.inf]
    assert sigma[3].tolist() == [0.0, 1.0, 0.0] and sigma[5].tolist() == [0.0, 1.0, 0.0]
    assert np.all(delta[:, [0, 2]] == 0) and delta[3, 1] == 1.0
    assert np.all(np.isfinite(bc))


def test_a_successor_without_paths_adds_nothing_after_a_cut():
    parts, X0, steps = wp.cut_short_case()
    D, sigma, delta, _ = wp.betweenness(parts, 7, X0, steps)
    assert D[[4, 5, 6], 0].tolist() == [3.0, 11.0, 12.0]
    assert sigma[[5, 6], 0].tolist() == [0.0, 0.0]
    assert np.all(np.isfinite(delta)) and delta[5, 0] == 0.0
    full = wp.betweenness(parts, 7, X0, BIG)
    assert full[0][[5, 6], 0].tolist() == [4.0, 5.0] and full[1][6, 0] == 1.0


def test_the_weight_scan_sees_only_edges_of_the_operator():
    from arrow_matrix_b200.engine import _nonpositive_edge
    ip, idx = np.array([0, 2, 4, 5]), np.array([0, 1, 0, 1, 2])
    ok = np.array([0.0, 3.0, 2.0, -1.0, 0.0], np.float32)              # zeros on the diagonal, -1 at (1, 1)
    assert not _nonpositive_edge(ip, idx, ok, np.arange(3))
    for bad in (0.0, -0.0, -1.0, np.nan):
        dat = ok.copy()
        dat[1] = bad                                                    # entry (0, 1): the edge 1 -> 0
        assert _nonpositive_edge(ip, idx, dat, np.arange(3))
        assert not _nonpositive_edge(ip, idx, dat, np.array([0, -1, 2]))   # an end at -1: no edge
        assert not _nonpositive_edge(ip, idx, dat, np.array([-1, 1, 2]))
    dat = ok.copy()
    dat[2] = np.inf                                                     # +inf is > 0: the "no edge" weight is accepted
    assert not _nonpositive_edge(ip, idx, dat, np.arange(3))
