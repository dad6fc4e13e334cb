"""CPU tests of connected components: the host restatement of tests/cc_ref.py against networkx, its invariants on the
golden and Barabasi-Albert decompositions, entries of any value as edges, padding rows as singletons, the
ArrowDecompositionMPI view against csgraph on the original graph, and the refusals raised before any CUDA work."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200.engine import ArrowEngine
from tests import cc_ref
from tests import pagerank_ref as prr
from tests.golden_util import CASES, GoldenCase
from tests.test_pagerank_cpu import _decompose, directed_ba


def _random_digraph(n, m, seed):
    """a block whose entry (r, c) is the edge c -> r, with self-loops and duplicates"""
    rng = np.random.default_rng(seed)
    r, c = rng.integers(0, n, m), rng.integers(0, n, m)
    return sparse.csr_matrix((rng.random(m) + 0.5, (r, c)), shape=(n, n))


def _nx_labels(parts, n):
    import networkx as nx
    u, v, _, ok = prr.entries(parts)
    G = nx.DiGraph()
    G.add_nodes_from(range(n))
    G.add_edges_from(zip(u[ok].tolist(), v[ok].tolist()))
    labels = np.empty(n, np.int32)
    for comp in nx.weakly_connected_components(G):
        comp = list(comp)
        labels[comp] = min(comp)
    return labels


@pytest.mark.parametrize("seed", range(6))
def test_restatement_matches_networkx(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(1, 80))
    A = _random_digraph(n, int(rng.integers(0, 2 * n)), seed)
    parts = [(A, None)]
    if seed % 2:                                   # a second part through a partial row map (-1: not routed)
        m = rng.permutation(n).astype(np.int64)
        m[rng.random(n) < 0.2] = -1
        parts.append((_random_digraph(n, n // 2, seed + 50), m))
    labels, count, sizes = cc_ref.components(parts, n)
    assert np.array_equal(labels, _nx_labels(parts, n))
    assert count == len(np.unique(labels)) and sizes.sum() == n
    assert np.array_equal(sizes[labels], np.bincount(labels, minlength=n)[labels])
    assert np.all(sizes[np.setdiff1d(np.arange(n), labels)] == 0)


def _decompositions():
    for name in CASES:
        g = GoldenCase(name)
        yield name, g.decomposition, g.width, g.block_diagonal
    for seed in (1, 2):
        yield f"ba{seed}", _decompose(directed_ba(1536, 3, seed), 128, seed), 128, True


@pytest.mark.parametrize("add_identity", [False, True])
def test_invariants(add_identity):
    for name, dec, width, bd in _decompositions():
        parts, proto = prr.level_parts(dec, width, block_diagonal=bd, add_identity=add_identity)
        n = proto.rows[0]
        labels, count, sizes = cc_ref.components(parts, n)
        rows = np.arange(n)
        assert labels.dtype == np.int32 and np.all(labels <= rows), name
        assert np.array_equal(labels[labels], labels), name
        u, v, _, ok = prr.entries(parts)
        assert np.array_equal(labels[u[ok]], labels[v[ok]]), name
        assert count == np.count_nonzero(labels == rows) and int(sizes.sum()) == n, name
        assert np.array_equal(cc_ref.of(dec, width, bd, add_identity)[0], labels), name


def test_explicit_zero_and_nan_entries_are_edges():
    n = 6
    indptr = np.array([0, 1, 2, 2, 3, 3, 3])
    indices = np.array([1, 0, 4])                  # edges 1 -> 0, 0 -> 1 and 4 -> 3
    for data in ([0.0, np.nan, np.inf], [-0.0, 0.0, np.nan]):
        A = sparse.csr_matrix((np.array(data), indices, indptr), shape=(n, n))
        assert A.nnz == 3                          # the explicit zeros stay stored
        labels, count, sizes = cc_ref.components([(A, None)], n)
        assert labels.tolist() == [0, 0, 2, 3, 3, 5] and count == 4
        assert sizes.tolist() == [2, 0, 1, 2, 0, 1]


def test_padding_rows_are_singletons():
    A = directed_ba(1000, 3, 7)                    # 1000 vertices in blocks of 128: 24 padding rows
    dec = _decompose(A, 128, 7)
    parts, proto = prr.level_parts(dec, 128)
    n = proto.rows[0]
    assert n > 1000
    labels, _, sizes = cc_ref.components(parts, n)
    pad = np.flatnonzero(np.asarray(proto.perms[0]) >= 1000)
    assert pad.size == n - 1000
    assert np.array_equal(labels[pad], pad) and np.all(sizes[pad] == 1)


def pieces(n, seed):
    """many components: a BA graph cut into pieces, every 17th vertex isolated; symmetric, and the self-loops (no
    edges) keep every row in the decomposition's blocks"""
    rng = np.random.default_rng(seed)
    A = directed_ba(n, 2, seed).tocoo()
    keep = rng.random(A.nnz) < 0.35
    keep &= ~np.isin(A.row, np.arange(0, n, 17)) & ~np.isin(A.col, np.arange(0, n, 17))
    A = sparse.csr_matrix((A.data[keep] + 1, (A.row[keep], A.col[keep])), shape=(n, n))
    return sparse.csr_matrix(A + A.T + sparse.identity(n))


@pytest.mark.parametrize("seed", [3, 4])
def test_vertex_view_matches_csgraph_on_the_original_graph(seed):
    n = 1500
    A = pieces(n, seed)
    dec = _decompose(A, 128, seed)
    labels, count, _ = cc_ref.of(dec, 128)
    parts, proto = prr.level_parts(dec, 128)
    got = cc_ref.by_vertex(labels, proto.perms[0], n)
    n_ref, comp = csgraph.connected_components(A, directed=True, connection="weak")
    assert np.array_equal(got, cc_ref.smallest_labels(comp))
    assert count == n_ref + (proto.rows[0] - n) and n_ref > 50


# ---- refusals before any CUDA work -------------------------------------------------------------------------------------
def _shell(fused_ok=True, rows=8):
    e = ArrowEngine.__new__(ArrowEngine)
    e.fused_ok = fused_ok

    class L:
        pass
    st = L()
    st.rows = rows
    e.levels = [st]

    class NoCuda:
        def __getattr__(self, name):
            raise AssertionError("CUDA work before the refusal")
    e.ctx = NoCuda()
    e._cc_labels = e._cc_sizes = None
    return e


@pytest.mark.parametrize("kw, match", [
    (dict(fused_ok=False), "sentinel"),
    (dict(out=np.zeros(8, np.int64)), "out"), (dict(out=np.zeros(9, np.int32)), "out"),
    (dict(out=np.zeros(16, np.int32)[::2]), "out"), (dict(out=[0] * 8), "out"),
    (dict(sizes_out=np.zeros((8, 1), np.int32)), "sizes_out"), (dict(sizes_out=np.zeros(8, np.float32)), "sizes_out"),
])
def test_engine_refusals(kw, match):
    fused_ok = kw.pop("fused_ok", True)
    with pytest.raises(ValueError, match=match):
        _shell(fused_ok).connected_components(**kw)


def test_mpi_forwarding_refuses_several_ranks():
    from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI

    class Comm:
        def Get_size(self):
            return 2
    obj = ArrowDecompositionMPI.__new__(ArrowDecompositionMPI)
    obj.comm = Comm()
    with pytest.raises(ValueError, match="one GPU"):
        obj.connected_components()
