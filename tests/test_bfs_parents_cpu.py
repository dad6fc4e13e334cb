"""CPU tests of the BFS parents of the (or, and) engine: the host restatement (tests/parents_ref.py) against the definition
on every golden decomposition, against the (min, +) predecessor restatement on unit weights and against scipy's BFS, and
the refusals of bfs_tree before any CUDA work."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200 import _lib
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from tests import bool_ref as br
from tests import parents_ref as par
from tests import push_ref as pr
from tests import semiring_ref as sr
from tests import witness_ref as wr
from tests.golden_util import CASES, GoldenCase


def _unit(decomposition):
    out = []
    for B, p in decomposition:
        B = sparse.csr_matrix(B, copy=True)
        B.data = np.ones_like(B.data, dtype=np.float32)
        out.append((B, p))
    return out


def _golden(name):
    g = GoldenCase(name)
    p = br.BoolProtocol(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal, n_blocks=g.n_blocks,
                        add_identity=True)
    return g, p


def test_in_adjacency_is_the_transposed_push_adjacency():
    rng = np.random.default_rng(1)
    n = 300
    A = sparse.random(n, n, density=0.03, format="csr", random_state=2, dtype=np.float32)
    m = rng.permutation(n + 20)[:n].astype(np.int64)
    m[::9] = -1
    parts = [(A, None), (A, m)]                               # two parts: duplicate edges are kept
    ip, ix = par.in_adjacency(parts, n + 20)
    op, ox = pr.adjacency(parts, n + 20)
    assert ip[-1] == op[-1] == ix.size
    for v in range(n + 20):
        row = ix[ip[v]:ip[v + 1]]
        assert np.all(np.diff(row) >= 0)
    src = np.repeat(np.arange(n + 20), np.diff(op))
    T = sparse.csr_matrix((np.ones(ox.size), (ox, src)), shape=(n + 20, n + 20))
    got = sparse.csr_matrix((np.ones(ix.size), ix, ip), shape=(n + 20, n + 20))
    assert (T != got).nnz == 0


@pytest.mark.parametrize("name", CASES)
def test_restatement_is_the_definition_on_golden_decompositions(name):
    g, p = _golden(name)
    if not pr.fused_ok(p):
        pytest.skip("a level reads rows behind the sentinel: no parents")
    n = p.rows[0]
    parts = pr.protocol_parts(p)
    X0 = np.random.default_rng(4).random((n, g.k)) < 0.03
    p.set_features(X0)
    want_L, want_steps = p.bfs_levels(200)
    L, P, steps = par.bfs_tree(par.in_adjacency(parts, n), pr.adjacency(parts, n), X0, 200)
    assert np.array_equal(L, want_L) and steps == want_steps
    assert np.array_equal(P, par.definition(L, parts, n)), name
    # every reached non-source has a parent, the others none
    assert np.array_equal(P >= 0, L > 0)


@pytest.mark.parametrize("name", CASES)
def test_restatement_is_the_min_plus_witness_on_unit_weights(name):
    """P == the (min, +) predecessors of the hop distances: both take the lexicographic minimum of (hop, label), u != v"""
    g, p = _golden(name)
    if not pr.fused_ok(p):
        pytest.skip("a level reads rows behind the sentinel: no parents")
    n = p.rows[0]
    parts = pr.protocol_parts(p)
    X0 = np.random.default_rng(5).random((n, g.k)) < 0.03
    L, P, _ = par.bfs_tree(par.in_adjacency(parts, n), pr.adjacency(parts, n), X0, 200)
    D = np.where(L >= 0, L, np.inf).astype(np.float32)
    want = wr.predecessors(_unit(g.decomposition), g.width, D, "min_plus", block_diagonal=g.block_diagonal,
                           n_blocks=g.n_blocks)
    assert np.array_equal(P, want), f"{name}: {int(np.sum(P != want))} parents differ"


def test_restated_parents_are_scipy_bfs_trees():
    """a directed BA graph: every parent is an in-neighbour one hop closer (scipy), the smallest such level-0 row;
    sources and unreached vertices have none"""
    n, w = 3000, 100
    A = sr.weighted_ba_graph(n, 3, seed=5, unit=True)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    C = sparse.coo_matrix(A)
    keep = (C.row > C.col) | (np.random.default_rng(1).random(C.nnz) < 0.3)
    A = sparse.csr_matrix((C.data[keep], (C.row[keep], C.col[keep])), shape=A.shape)
    directed = []
    for B, perm in dec:
        Bc = sparse.coo_matrix(B)
        ok = np.asarray(A[perm[Bc.row], perm[Bc.col]]).ravel() != 0
        directed.append((sparse.csr_matrix((Bc.data[ok], (Bc.row[ok], Bc.col[ok])), shape=B.shape), perm))
    sources = np.random.default_rng(3).choice(n, 8, replace=False)
    p = br.BoolProtocol(directed, w, sources.size, add_identity=True)
    n0 = p.rows[0]
    parts = pr.protocol_parts(p)
    X0 = br.source_bits(p.perms[0], n0, n, sources)
    L, P, _ = par.bfs_tree(par.in_adjacency(parts, n0), pr.adjacency(parts, n0), X0, 500)
    perm0 = np.asarray(p.perms[0][:n0], dtype=np.int64)
    inv = np.full(n, -1, np.int64)
    ok = perm0 < n
    inv[perm0[ok]] = np.arange(n0)[ok]
    # a step computes X | A X: row v gathers from its columns u, the edge u -> v is A[v, u]
    hops = csgraph.shortest_path(A.T, unweighted=True, indices=sources)          # [k x n]
    Pv = br.vertex_order(P, perm0, n, -2).T                                        # [k x n], level-0 row labels
    assert not np.any(Pv == -2)
    At = A.tocsr()
    for s in range(sources.size):
        h = hops[s]
        assert Pv[s, sources[s]] == -1
        assert np.all(Pv[s, np.isinf(h)] == -1)
        for v in np.flatnonzero(np.isfinite(h) & (h > 0)):
            ins = At.indices[At.indptr[v]:At.indptr[v + 1]]
            closer = ins[h[ins] == h[v] - 1]
            assert closer.size and Pv[s, v] == inv[closer].min(), (s, v)


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
    """an ArrowEngine without a device: only what bfs_tree() checks before its first CUDA call"""
    eng = object.__new__(ArrowEngine)
    eng.sr, eng.semiring, eng.add_identity, eng.fused_ok = _lib.SEMIRINGS[semiring], semiring, add_identity, fused_ok
    return eng


def test_refusals_happen_before_any_cuda_call(no_cuda):
    with pytest.raises(ValueError, match="or_and"):
        _bare_engine("min_plus", True, True).bfs_tree(10)
    with pytest.raises(ValueError, match="or_and"):
        _bare_engine("plus_times", True, True).bfs_tree(10)
    with pytest.raises(ValueError, match="add_identity"):
        _bare_engine("or_and", False, True).bfs_tree(10)
    with pytest.raises(ValueError, match="sentinel"):
        _bare_engine("or_and", True, False).bfs_tree(10)
    arrow = ArrowDecompositionMPI.initialize(_TwoRanks(), [4, 4], None, None, 8, 4, 'gpu', True, True,
                                             semiring="or_and", add_identity=True)
    with pytest.raises(ValueError, match="one GPU"):
        arrow.bfs_tree(10)
    arrow = ArrowDecompositionMPI.initialize(SelfComm(), [4, 4], None, None, 8, 4, 'gpu', True, True,
                                             semiring="or_and", add_identity=True)
    with pytest.raises(RuntimeError, match="not loaded"):
        arrow.bfs_tree(10)
    arrow._engine = _NoCuda()
    with pytest.raises(ValueError, match="one GPU"):
        arrow.bfs_tree(10)
