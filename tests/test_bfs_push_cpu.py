"""CPU tests of the direction-optimising BFS: the host restatement of the push operator (tests/push_ref.py) against the
restated arrow step of tests/bool_ref.py and scipy's hop counts, the direction rule, and the push dispatch of the source
reached by the GPU sweep's feature widths."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import BFS_PUSH_ALPHA, bfs_direction
from tests import bool_ref as br
from tests import push_ref as pr
from tests import semiring_ref as sr
from tests import tile_dispatch as td
from tests.golden_util import CASES, GoldenCase


def _protocol(g: GoldenCase, k: int) -> br.BoolProtocol:
    return br.BoolProtocol(g.decomposition, g.width, k, block_diagonal=g.block_diagonal, n_blocks=g.n_blocks,
                           add_identity=True)


FUSED_CASES = [c for c in CASES if pr.fused_ok(_protocol(GoldenCase(c), 1))]


def test_some_golden_cases_are_fused_and_some_are_not():
    assert FUSED_CASES and len(FUSED_CASES) < len(CASES)


@pytest.mark.parametrize("k", [1, 5, 33, 128])
@pytest.mark.parametrize("name", FUSED_CASES)
def test_push_from_a_step_pair_is_the_next_step(name, k):
    """X_h = step(X_{h-1}) of the restated arrow step: push(X_h, frontier(X_h, X_{h-1})) == step(X_h), 3 chained levels;
    and M restates the step itself"""
    g = GoldenCase(name)
    p = _protocol(g, k)
    adj = pr.adjacency(pr.protocol_parts(p), p.rows[0])
    rng = np.random.default_rng(k)
    prev = rng.random((p.rows[0], k)) < 0.05
    p.set_features(prev)
    cur = p.step().copy()
    assert np.array_equal(cur, pr.step(prev, adj)), f"{name}: M is not the step"
    for level in range(3):
        want = p.step().copy()
        got = pr.push(cur, pr.frontier(cur, prev), adj)
        assert np.array_equal(got, want), f"{name} k={k} level {level}"
        prev, cur = cur, want


@pytest.mark.parametrize("name", FUSED_CASES)
def test_push_from_a_pair_that_is_not_a_step_differs(name):
    """the invariant matters: from an X_{h-1} whose step is not X_h, the frontier push misses bits of step(X_h) -- why the
    push runs inside bfs_levels only"""
    g = GoldenCase(name)
    p = _protocol(g, 4)
    adj = pr.adjacency(pr.protocol_parts(p), p.rows[0])
    X = np.random.default_rng(1).random((p.rows[0], 4)) < 0.3
    # the previous level claims every bit already: an empty frontier, so the push returns X unchanged
    assert pr.frontier(X, X).size == 0
    assert np.array_equal(pr.push(X, pr.frontier(X, X), adj), X)
    assert not np.array_equal(pr.step(X, adj), X), f"{name}: the step of X adds bits a push from X, X misses"


def test_adjacency_layout():
    """ascending destinations per row, duplicates kept, -1 columns and maps, u == v dropped"""
    A = sparse.csr_matrix(np.array([[1, 1, 0], [1, 1, 1], [0, 0, 0]], np.float32))
    B = sparse.csr_matrix(np.array([[0, 1], [1, 0]], np.float32))
    indptr, indices = pr.adjacency([(A, None), (B, np.array([2, 0]))], 3)
    # A: edges 1 -> 0, 0 -> 1, 2 -> 1; B through [2, 0]: 0 -> 2, 2 -> 0
    assert indptr.tolist() == [0, 2, 3, 5] and indices.tolist() == [1, 2, 0, 0, 1]
    dup = pr.adjacency([(A, None), (A, None)], 3)
    assert dup[0].tolist() == [0, 2, 4, 6] and dup[1].tolist() == [1, 1, 0, 0, 1, 1]
    C = sparse.csr_matrix((np.ones(3, np.float32), np.array([1, 0, 0]), np.array([0, 2, 3])), shape=(2, 2))
    C.indices[0] = -1                                        # a column remapped away
    u, v = pr.edges([(C, None)])
    assert u.tolist() == [0] and v.tolist() == [1]           # (0, -1) skipped, (0, 0) dropped, (1, 0) is 0 -> 1


def _ba_protocol(directed: bool, k: int):
    """the 3-level decomposition of a 3000-vertex BA graph (tests/test_bool_cpu.py), the directed variant keeping every
    downward edge and 30 % of the upward ones; (graph, protocol)"""
    n, w = 3000, 100
    A = sr.weighted_ba_graph(n, 3, seed=5, unit=True)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    if directed:
        C = sparse.coo_matrix(A)
        keep = (C.row > C.col) | (np.random.default_rng(1).random(C.nnz) < 0.3)
        A = sparse.csr_matrix((C.data[keep], (C.row[keep], C.col[keep])), shape=A.shape)
        out = []
        for B, perm in dec:
            Bc = sparse.coo_matrix(B)
            ok = np.asarray(A[perm[Bc.row], perm[Bc.col]]).ravel() != 0
            out.append((sparse.csr_matrix((Bc.data[ok], (Bc.row[ok], Bc.col[ok])), shape=B.shape), perm))
        dec = out
    p = br.BoolProtocol(dec, w, k, add_identity=True)
    assert p.L == 3 and pr.fused_ok(p)
    return A, p


@pytest.mark.parametrize("directed", [False, True], ids=["undirected", "directed"])
def test_restated_bfs_is_scipy_in_every_direction(directed):
    n = 3000
    A, p = _ba_protocol(directed, 8)
    sources = np.random.default_rng(3).choice(n, 8, replace=False)
    X0 = br.source_bits(p.perms[0], p.rows[0], n, sources)
    adj = pr.adjacency(pr.protocol_parts(p), p.rows[0])
    total_nnz = sum(M.nnz for M in p.mats) + p.rows[0]       # the engine's level blocks, level 0 with its diagonal
    hops = csgraph.shortest_path(A.T, unweighted=True, indices=sources)
    want = np.where(np.isinf(hops), -1, hops).astype(np.int32)
    runs = {"push": lambda e: "push", "pull": lambda e: "pull", "rule": lambda e: bfs_direction(e, total_nnz)}
    for label, rule in runs.items():
        levels, steps, dirs = pr.bfs(adj, X0, 500, rule)
        got = br.vertex_order(levels, p.perms[0], n, -1).T
        assert np.array_equal(got, want), f"{label}: {int(np.sum(got != want))} levels differ"
        assert steps == int(want.max()) + 1 and len(dirs) == steps
        if label == "rule":
            assert set(dirs) == {"push", "pull"}, dirs


def test_direction_rule():
    assert BFS_PUSH_ALPHA == 8
    assert bfs_direction(0, 1) == "push" and bfs_direction(0, 0) == "pull"
    assert bfs_direction(1, 8) == "pull" and bfs_direction(1, 9) == "push"
    assert bfs_direction(10, 140, alpha=14) == "pull" and bfs_direction(10, 141, alpha=14) == "push"
    assert bfs_direction(10, 1000, alpha=100) == "pull" and bfs_direction(9, 1000, alpha=100) == "push"


def test_push_dispatch_is_reached_by_the_gpu_sweep():
    in_source = pr.source_push_kinds(td.SOURCE)
    reached = {pr.push_kind(k) for k in br.SWEEP_KS}
    assert in_source == {"unsigned", "uint4"} and reached == in_source
