"""CPU tests of the betweenness of the (or, and) engine: the host restatement (tests/paths_ref.py) against networkx's
Brandes betweenness on every golden decomposition and a BA graph, multi-source columns against a super-source graph, path
counts against counted walks, rounding past 2^53, duplicate entries, and the refusals of bfs_path_counts / betweenness
before any CUDA work."""
import networkx as nx
import numpy as np
import pytest
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
from tests.golden_util import CASES, GoldenCase

BIG = 10 ** 6       # max_steps that never truncates


def _golden(name):
    g = GoldenCase(name)
    p = br.BoolProtocol(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, n_blocks=g.n_blocks,
                        add_identity=True)
    return g, p


def _digraph(parts, n):
    G = nx.DiGraph()
    G.add_nodes_from(range(n))
    u, v = pr.edges(parts)
    G.add_edges_from(zip(u.tolist(), v.tolist()))
    return G


def _one_hot(n, k, seed):
    rows = np.random.default_rng(seed).choice(n, k, replace=False)
    X0 = np.zeros((n, k), bool)
    X0[rows, np.arange(k)] = True
    return X0, rows


def _nx_bc(G, sources):
    got = nx.betweenness_centrality_subset(G, sources=[int(s) for s in sources], targets=list(G.nodes), normalized=False)
    return np.array([got[v] for v in range(G.number_of_nodes())])


def _ba_parts(n=2000, w=100, seed=5):
    A = sr.weighted_ba_graph(n, 3, seed=seed, unit=True)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    p = br.BoolProtocol(dec, w, 4, add_identity=True)
    return pr.protocol_parts(p), p.rows[0]


@pytest.mark.parametrize("name", CASES)
def test_restatement_is_networkx_brandes_on_golden_decompositions(name):
    g, p = _golden(name)
    n = p.rows[0]
    parts = pr.protocol_parts(p)
    k = min(g.k, n)
    X0, rows = _one_hot(n, k, 4)
    L, sigma, delta, bc, steps = pa.betweenness(parts, n, X0, BIG)
    p.set_features(X0)
    want_L, want_steps = p.bfs_levels(BIG)
    assert np.array_equal(L, want_L) and steps == want_steps
    np.testing.assert_allclose(bc, _nx_bc(_digraph(parts, n), rows), rtol=1e-12, atol=1e-12)
    assert np.all(delta[L <= 0] == 0) and np.all(sigma[L == -1] == 0) and np.all(sigma[L == 0] == 1)
    assert np.all(sigma[L > 0] >= 1)


def test_restatement_is_networkx_brandes_on_a_ba_graph():
    parts, n = _ba_parts()
    X0, rows = _one_hot(n, 12, 7)
    _, _, delta, bc, _ = pa.betweenness(parts, n, X0, BIG)
    np.testing.assert_allclose(bc, _nx_bc(_digraph(parts, n), rows), rtol=1e-12, atol=1e-9)
    # per column: the dependencies of one source are networkx's betweenness from that source alone
    G = _digraph(parts, n)
    for s in (0, 5):
        np.testing.assert_allclose(delta[:, s], _nx_bc(G, [rows[s]]), rtol=1e-12, atol=1e-9)


def test_a_multi_source_column_is_one_super_source():
    """column of several sources == one source S* with an edge to each of them (S* = row n, the last): sigma and delta
    equal bit for bit at every row but the sources, whose delta is 0"""
    parts, n = _ba_parts(1500, 100, 8)
    rng = np.random.default_rng(3)
    X0 = np.zeros((n, 3), bool)
    for s in range(3):
        X0[rng.choice(n, 4 + s, replace=False), s] = True
    L, sigma, delta, bc, _ = pa.betweenness(parts, n, X0, BIG)
    u, v = pr.edges(parts)
    for s in range(3):
        src = np.flatnonzero(X0[:, s])
        su = np.concatenate([u, np.full(src.size, n)])
        sv = np.concatenate([v, src])
        A = sparse.csr_matrix((np.ones(su.size, np.float32), (sv, su)), shape=(n + 1, n + 1))
        Xs = np.zeros((n + 1, 1), bool)
        Xs[n, 0] = True
        Ls, ss, ds, _, _ = pa.betweenness([(A, None)], n + 1, Xs, BIG)
        assert np.array_equal(np.where(L[:, s] >= 0, L[:, s] + 1, -1), Ls[:n, 0])
        assert np.array_equal(sigma[:, s], ss[:n, 0])
        other = ~X0[:, s]
        assert np.array_equal(delta[other, s], ds[:n, 0][other])
        assert np.all(delta[src, s] == 0)
        G = _digraph([(A, None)], n + 1)
        np.testing.assert_allclose(delta[other, s], _nx_bc(G, [n])[:n][other], rtol=1e-12, atol=1e-9)


def test_path_counts_are_counted_shortest_walks():
    """sigma[v, s] = the walks of length L[v, s] from the sources of column s to v (each is a shortest path), counted
    in exact integers over M as a set"""
    rng = np.random.default_rng(11)
    for trial in range(4):
        n = 60
        A = sparse.random(n, n, density=0.06, format="csr", random_state=trial, dtype=np.float32)
        parts = [(A, None)]
        X0 = rng.random((n, 5)) < 0.04
        X0[trial, :] = True
        L, sigma, _, _, _ = pa.betweenness(parts, n, X0, BIG)
        u, v = pr.edges(parts)
        M = np.zeros((n, n), dtype=object)                      # M[v, u] = 1 for an edge u -> v
        M[v, u] = 1
        for s in range(5):
            walks = X0[:, s].astype(object)
            for h in range(int(L[:, s].max()) + 1):
                at = L[:, s] == h
                assert all(int(sigma[i, s]) == walks[i] for i in np.flatnonzero(at))
                walks = M.dot(walks)
        assert np.all(sigma[L == -1] == 0)


def _gadget_chain(m):
    """m three-way gadgets a -> {b1, b2, b3} -> a', chained: 3^m shortest paths from the first a to the last"""
    us, vs = [], []
    for i in range(m):
        a, nxt = 4 * i, 4 * (i + 1)
        for b in (a + 1, a + 2, a + 3):
            us += [a, b]
            vs += [b, nxt]
    n = 4 * m + 1
    A = sparse.csr_matrix((np.ones(len(us), np.float32), (vs, us)), shape=(n, n))
    return [(A, None)], n


def test_path_counts_round_past_2_53_in_the_fixed_order():
    m = 40
    parts, n = _gadget_chain(m)
    X0 = np.zeros((n, 1), bool)
    X0[0, 0] = True
    L, sigma, delta, bc, _ = pa.betweenness(parts, n, X0, BIG)
    x = 1.0
    for i in range(m):
        assert sigma[4 * i, 0] == x
        x = (x + x) + x                                        # three in-edges summed in ascending order
    assert sigma[n - 1, 0] == x and L[n - 1, 0] == 2 * m
    assert int(sigma[n - 1, 0]) != 3 ** m                      # not representable: rounded on the way
    assert np.all(np.isfinite(delta)) and np.all(np.isfinite(bc))


def test_duplicate_entries_count_once():
    parts, n = _ba_parts(800, 50, 9)
    X0, _ = _one_hot(n, 6, 2)
    once = pa.betweenness(parts, n, X0, BIG)
    twice = pa.betweenness(parts + parts, n, X0, BIG)
    for a, b in zip(once, twice):
        assert np.array_equal(a, b)


def test_truncated_levels_stop_the_sweep():
    parts, n = _ba_parts(800, 50, 9)
    X0, _ = _one_hot(n, 6, 2)
    L, sigma, delta, _, steps = pa.betweenness(parts, n, X0, 2)
    assert steps == 2 and L.max() == 2
    full_L, full_sigma, _, _, _ = pa.betweenness(parts, n, X0, BIG)
    assert np.array_equal(sigma[L >= 0], full_sigma[L >= 0])
    assert np.all(delta[L == 2] == 0)                          # no level 3 to depend on


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


def _bare_engine(semiring, add_identity, fused_ok):
    """an ArrowEngine without a device: only what bfs_path_counts() / betweenness() check before their first CUDA call"""
    eng = object.__new__(ArrowEngine)
    eng.sr, eng.semiring, eng.add_identity, eng.fused_ok = _lib.SEMIRINGS[semiring], semiring, add_identity, fused_ok
    return eng


@pytest.mark.parametrize("call", ["bfs_path_counts", "betweenness"])
def test_refusals_happen_before_any_cuda_call(no_cuda, call):
    for semiring in ("min_plus", "plus_times"):
        with pytest.raises(ValueError, match="or_and"):
            getattr(_bare_engine(semiring, True, True), call)(10)
    with pytest.raises(ValueError, match="add_identity"):
        getattr(_bare_engine("or_and", False, True), call)(10)
    with pytest.raises(ValueError, match="sentinel"):
        getattr(_bare_engine("or_and", True, False), call)(10)
    arrow = ArrowDecompositionMPI.initialize(_TwoRanks(), [4, 4], None, None, 8, 4, 'gpu', True, True,
                                             semiring="or_and", add_identity=True)
    with pytest.raises(ValueError, match="one GPU"):
        getattr(arrow, call)(10)
    arrow = ArrowDecompositionMPI.initialize(SelfComm(), [4, 4], None, None, 8, 4, 'gpu', True, True,
                                             semiring="or_and", add_identity=True)
    with pytest.raises(RuntimeError, match="not loaded"):
        getattr(arrow, call)(10)
    arrow._engine = _NoCuda()
    with pytest.raises(ValueError, match="one GPU"):
        getattr(arrow, call)(10)


def test_output_arrays_are_checked_before_any_cuda_call(no_cuda):
    """a strided or mistyped ``out`` / ``dependencies_out`` would not receive the rows: refused up front"""
    eng = _bare_engine("or_and", True, True)
    eng.k = 3

    class _Level:
        rows = 8
    eng.levels = [_Level()]
    for out in (np.zeros(16)[::2], np.zeros(8, np.float32), np.zeros(7), np.zeros((8, 1))):
        with pytest.raises(ValueError, match="out must be"):
            eng.betweenness(10, out=out)
    for dep in (np.zeros((8, 6))[:, ::2], np.zeros((8, 3), np.float32), np.zeros((3, 8))):
        with pytest.raises(ValueError, match="dependencies_out must be"):
            eng.betweenness(10, dependencies_out=dep)
