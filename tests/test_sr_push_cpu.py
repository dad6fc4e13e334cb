"""CPU tests of the direction-optimising min_plus / max_plus fixed point: the host restatement of the push
(tests/sr_push_ref.py) against the restated step and the restated arrow step, scipy's shortest paths and a DAG's longest
paths; why an engine with a -0 weight pulls; the refusals; and the push dispatch of the source reached by the GPU sweep's
feature widths."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200 import _lib, synth
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import SR_PUSH_ALPHA, ArrowEngine, bfs_direction
from tests import push_ref as pr
from tests import semiring_ref as sr
from tests import sr_push_ref as spr
from tests import tile_dispatch as td
from tests.golden_util import CASES, GoldenCase

SEMIRINGS = ["min_plus", "max_plus"]


def _protocol(g: GoldenCase, k: int, semiring: str, decomposition=None) -> sr.SemiringProtocol:
    return sr.SemiringProtocol(g.decomposition if decomposition is None else decomposition, g.width, k, semiring,
                               block_diagonal=g.block_diagonal, n_blocks=g.n_blocks, add_identity=True)


FUSED_CASES = [c for c in CASES if pr.fused_ok(_protocol(GoldenCase(c), 1, "min_plus"))]


def _bits(X):
    return np.asarray(X, np.float32).view(np.uint32)


def test_some_golden_cases_are_fused():
    assert FUSED_CASES and len(FUSED_CASES) < len(CASES)


@pytest.mark.parametrize("k", [1, 5, 33, 128])
@pytest.mark.parametrize("semiring", SEMIRINGS)
@pytest.mark.parametrize("name", FUSED_CASES)
def test_push_from_a_step_pair_is_the_next_step(name, semiring, k):
    """X_h = F(X_{h-1}), X_{-1} the ⊕ identity: push(X_h, frontier(X_h, X_{h-1})) == F(X_h) bit for bit over 3 chained
    levels, from features with ±inf, -0 and NaN, weights with 0, negatives and a negative self-loop; and F is the restated
    arrow step once the features are the step's own"""
    g = GoldenCase(name)
    rng = np.random.default_rng(k)
    dec = spr.with_weights(g.decomposition, rng)
    p = _protocol(g, k, semiring, dec)
    adj = spr.weighted_adjacency(pr.protocol_parts(p), p.rows[0])
    assert np.any((adj[1] == np.repeat(np.arange(p.rows[0]), np.diff(adj[0]))) & (adj[2] < 0)), "no negative self-loop"
    prev = np.full((p.rows[0], k), spr.ZERO[semiring], np.float32)
    cur = spr.special_features(p.rows[0], k, semiring, rng)
    for level in range(4):
        want = spr.step(cur, adj, semiring)
        got = spr.push(cur, spr.frontier(cur, prev), adj, semiring)
        assert np.array_equal(_bits(got), _bits(want)), f"{name} {semiring} k={k} level {level}"
        if level:                                   # the step's own features: no NaN, no -0
            p.set_features(cur)
            assert np.array_equal(p.step(), want), f"{name} {semiring} k={k} level {level}: F is not the arrow step"
        prev, cur = cur, want


@pytest.mark.parametrize("semiring", SEMIRINGS)
def test_a_negative_zero_weight_breaks_the_push(semiring):
    """u = 0 has a -0 self-loop and a -0 edge to v = 1.  F keeps u at -0, so u is not a frontier row at level 2, and the
    push loses the -0 that u's terms bring into both rows: equal by value, different in bits.  An engine with a -0 weight
    therefore pulls every level."""
    A = sparse.csr_matrix((np.array([-0.0, -0.0], np.float32), np.array([0, 0]), np.array([0, 1, 2])), shape=(2, 2))
    adj = spr.weighted_adjacency([(A, None)], 2)
    assert adj[0].tolist() == [0, 2, 2] and np.all(np.signbit(adj[2]))
    X0 = np.array([[-0.0], [5.0 if semiring == "min_plus" else -5.0]], np.float32)
    X1 = spr.step(X0, adj, semiring)
    assert np.all(np.signbit(X1)) and np.all(X1 == 0)
    assert spr.frontier(X1, X0).tolist() == [1]
    want = spr.step(X1, adj, semiring)
    got = spr.push(X1, spr.frontier(X1, X0), adj, semiring)
    assert np.array_equal(got, want) and not np.array_equal(_bits(got), _bits(want))


def test_weighted_adjacency_layout():
    """destinations by row, duplicates kept (ordered by weight bits), self-loops kept, -1 columns and maps dropped"""
    A = sparse.csr_matrix((np.array([3, -1, 2, 5, 4], np.float32), np.array([0, 1, 0, 1, 2]), np.array([0, 2, 5, 5])),
                          shape=(3, 3))
    B = sparse.csr_matrix(np.array([[0, 7], [9, 0]], np.float32))
    indptr, indices, values = spr.weighted_adjacency([(A, None), (B, np.array([2, 0]))], 3)
    # A: 0 -> 0 (3), 1 -> 0 (-1), 0 -> 1 (2), 1 -> 1 (5), 2 -> 1 (4); B through [2, 0]: 0 -> 2 (7), 2 -> 0 (9)
    assert indptr.tolist() == [0, 3, 5, 7]
    assert indices.tolist() == [0, 1, 2, 0, 1, 0, 1] and values.tolist() == [3, 2, 7, -1, 5, 9, 4]
    C = sparse.csr_matrix((np.array([1, 2, 3], np.float32), np.array([1, 0, 0]), np.array([0, 2, 3])), shape=(2, 2))
    C.indices[0] = -1                                        # a column remapped away
    u, v, w = spr.weighted_edges([(C, None)])
    assert u.tolist() == [0, 0] and v.tolist() == [0, 1] and w.tolist() == [2, 3]
    # the unweighted edges of the BFS are these without the self-loops
    assert np.array_equal(pr.edges([(A, None)])[0], spr.weighted_edges([(A, None)])[0][[1, 2, 4]])


def test_canon_and_the_frontier_by_bits():
    X = np.array([[np.nan, -0.0, 0.0, np.inf, -np.inf, 2.5]], np.float32)
    assert np.array_equal(_bits(spr.canon(X, "min_plus")), _bits(np.array([[np.inf, 0, 0, np.inf, -np.inf, 2.5]], np.float32)))
    assert np.array_equal(_bits(spr.canon(X, "max_plus")), _bits(np.array([[-np.inf, 0, 0, np.inf, -np.inf, 2.5]], np.float32)))
    a = np.array([[0.0], [np.nan], [1.0], [2.0]], np.float32)
    b = np.array([[-0.0], [np.nan], [1.0], [3.0]], np.float32)
    assert spr.frontier(a, b).tolist() == [0, 3]             # ±0 differ in bits, the same NaN does not
    assert spr.rows_changed(a, b) == 2                       # NaN != NaN and 2 != 3; -0 == +0


def _ba_protocol(directed: bool, k: int, semiring: str = "min_plus"):
    """the 3-level decomposition of a 3000-vertex weighted BA graph (weights 1-16), the directed variant keeping every
    downward edge and 30 % of the upward ones; (graph, protocol, decomposition)"""
    n, w = 3000, 100
    A = sr.weighted_ba_graph(n, 3, seed=5)
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
    p = sr.SemiringProtocol(dec, w, k, semiring, add_identity=True)
    assert p.L == 3 and pr.fused_ok(p)
    return A, p


def _runs(total_nnz):
    return {"push": lambda e: "push", "pull": lambda e: "pull",
            "rule": lambda e: bfs_direction(e, total_nnz, SR_PUSH_ALPHA)}


@pytest.mark.parametrize("directed", [False, True], ids=["undirected", "directed"])
def test_restated_fixed_point_is_scipy_in_every_direction(directed):
    n, k = 3000, 8
    A, p = _ba_protocol(directed, k)
    sources = np.random.default_rng(3).choice(n, k, replace=False)
    X0 = sr.source_features(p.perms[0], p.rows[0], n, sources)
    adj = spr.weighted_adjacency(pr.protocol_parts(p), p.rows[0])
    total_nnz = sum(M.nnz for M in p.mats) + p.rows[0]       # the engine's level blocks, level 0 with its diagonal
    want = csgraph.shortest_path(A.T, method="D", indices=sources).astype(np.float32)
    _, pull_steps = spr.protocol_fixed_point(p, X0, 500)
    for label, rule in _runs(total_nnz).items():
        X, steps, dirs = spr.fixed_point(adj, X0, 500, rule, "min_plus")
        got = sr.distances(X, p.perms[0], n)
        assert np.array_equal(got, want), f"{label}: {int(np.sum(got != want))} distances differ"
        assert steps == pull_steps and len(dirs) == steps, label
        if label == "rule":
            assert set(dirs) == {"push", "pull"}, dirs


def test_restated_max_plus_fixed_point_is_the_longest_dag_path():
    """the DAG orientation of tests/test_witness_cpu.py: the BA graph's edges from the smaller vertex id to the larger,
    the entries of the other direction -inf (a term that never wins a max)"""
    n, w = 3000, 100
    S = sr.weighted_ba_graph(n, 3, seed=5)
    A = sparse.csr_matrix(sparse.tril(S, k=-1))
    dec = []
    for B, perm in arrow_decomposition(S, w, max_number_of_levels=3, block_diagonal=True, seed=2):
        C = sparse.coo_matrix(B)
        data = np.where(perm[C.row] > perm[C.col], C.data, -np.inf).astype(np.float32)
        dec.append((sparse.csr_matrix((data, (C.row, C.col)), shape=B.shape), perm))
    p = sr.SemiringProtocol(dec, w, 4, "max_plus", add_identity=True)
    assert pr.fused_ok(p)
    sources = np.array([0, 3, 17, 200])
    X0 = np.where(np.isinf(sr.source_features(p.perms[0], p.rows[0], n, sources)), -np.inf, 0.0).astype(np.float32)
    Ac = sparse.csc_matrix(A.T)                              # column v of A^T: the in-edges of v
    want = np.full((sources.size, n), -np.inf)
    want[np.arange(sources.size), sources] = 0.0
    for vv in range(n):                                      # topological DP: every edge goes to a larger id
        lo, hi = Ac.indptr[vv], Ac.indptr[vv + 1]
        if hi > lo:
            want[:, vv] = np.maximum(want[:, vv], (want[:, Ac.indices[lo:hi]] + Ac.data[lo:hi]).max(axis=1))
    adj = spr.weighted_adjacency(pr.protocol_parts(p), p.rows[0])
    total_nnz = sum(M.nnz for M in p.mats) + p.rows[0]
    _, pull_steps = spr.protocol_fixed_point(p, X0, 3000)
    for label, rule in _runs(total_nnz).items():
        X, steps, _ = spr.fixed_point(adj, X0, 3000, rule, "max_plus")
        assert np.array_equal(sr.distances(X, p.perms[0], n), want.astype(np.float32)), label
        assert steps == pull_steps, label


class _NoCuda:
    pass


@pytest.fixture
def no_cuda(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a CUDA call was made")
    monkeypatch.setattr(_lib.Context, "__init__", refuse)
    monkeypatch.setattr(_lib, "load_library", refuse)


def _bare_engine(semiring, add_identity=True, fused_ok=True, neg_zero=False, mode="fused", L=2):
    """an ArrowEngine without a device: only what iterate_to_fixed_point() checks before it picks a loop"""
    eng = ArrowEngine.__new__(ArrowEngine)
    eng.sr = _lib.SEMIRINGS[semiring]
    eng.add_identity, eng.fused_ok, eng._neg_zero_weight, eng.mode, eng.L = add_identity, fused_ok, neg_zero, mode, L
    return eng


def test_which_engines_push_is_decided_before_any_cuda_call(no_cuda):
    assert _bare_engine("min_plus")._sr_push_ok() and _bare_engine("max_plus")._sr_push_ok()
    assert _bare_engine("min_plus", mode="exchange", L=2)._sr_push_ok()
    for eng in (_bare_engine("plus_times"), _bare_engine("or_and"), _bare_engine("min_plus", add_identity=False),
                _bare_engine("max_plus", fused_ok=False), _bare_engine("min_plus", neg_zero=True),
                _bare_engine("max_plus", mode="exchange", L=1)):
        assert not eng._sr_push_ok()
    arrow = ArrowDecompositionMPI.initialize(SelfComm(), [4, 4], None, None, 8, 4, 'gpu', True, True,
                                             semiring="min_plus", add_identity=True)
    with pytest.raises(RuntimeError, match="not loaded"):
        arrow.iterate_to_fixed_point(5)
    arrow._engine = _NoCuda()
    with pytest.raises(ValueError, match="one GPU"):
        arrow.iterate_to_fixed_point(5)


def test_direction_rule_constant():
    assert SR_PUSH_ALPHA > 0
    assert bfs_direction(0, 1, SR_PUSH_ALPHA) == "push" and bfs_direction(1, SR_PUSH_ALPHA, SR_PUSH_ALPHA) == "pull"


# feature widths of the GPU push sweep (tests/test_gpu_sr_push.py)
SWEEP_KS = sr.SWEEP_KS


def test_push_dispatch_is_reached_by_the_gpu_sweep():
    in_source = spr.source_push_kinds(td.SOURCE)
    assert in_source == {(s, e) for s in ("SrMinPlus", "SrMaxPlus") for e in ("float4", "float")}
    reached = {spr.push_kind(k) for k in SWEEP_KS}
    assert reached == {e for _, e in in_source}
