"""CPU tests of the bottleneck semirings (max_min, min_max): the host restatement of tests/bottleneck_ref.py against
independent oracles (spanning-forest paths, a heap-based Dijkstra), push against pull level by level, the path tree's
properties on tie-heavy inputs, the refusals before any CUDA call, and the kernel dispatch in the CUDA source."""
import heapq
import re

import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200 import _lib
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine, semiring_code
from tests import bottleneck_ref as bn
from tests import push_ref as pr
from tests import semiring_ref as sr
from tests import sr_push_ref as spr
from tests import tile_dispatch as td
from tests.golden_util import CASES, GoldenCase

PUSH, PULL = (lambda e: "push"), (lambda e: "pull")


def _bits(X):
    return np.asarray(X, np.float32).view(np.uint32)


def _source_features(perm0, rows0, n, sources, semiring):
    X = np.full((rows0, sources.size), bn.ZERO[semiring], np.float32)
    inv = np.full(n, -1, np.int64)
    m = min(rows0, perm0.size)
    ok = perm0[:m] < n
    inv[perm0[:m][ok]] = np.arange(m)[ok]
    X[inv[sources], np.arange(sources.size)] = bn.ONE[semiring]
    return X


def _tree_path_values(T: sparse.csr_matrix, s: int, semiring: str) -> np.ndarray:
    """the largest (min_max) or smallest (max_min) edge on the spanning-forest path from s to every vertex"""
    n = T.shape[0]
    out = np.full(n, bn.ZERO[semiring], np.float32)
    out[s] = bn.ONE[semiring]
    order, pred = csgraph.breadth_first_order(T, s, directed=False, return_predecessors=True)
    S = sparse.csr_matrix(T + T.T)
    for v in order[1:]:
        w = np.abs(S[pred[v], v])
        out[v] = bn.times(out[pred[v]], np.float32(w), semiring)
    return out


@pytest.mark.parametrize("semiring", bn.SEMIRINGS)
def test_spanning_forest_oracle_through_the_decomposition(semiring):
    """on a symmetric graph the minimax value is the largest edge on the minimum spanning forest's path, the widest
    value the smallest edge on the maximum spanning forest's path; restated arrow steps from one source per column
    reach them (positive weights: scipy drops explicit zeros)"""
    n, w = 600, 64
    rng = np.random.default_rng(3)
    A = sparse.random(n, n, density=0.006, format="csr", random_state=4, dtype=np.float32)
    A.data = rng.integers(1, 40, A.nnz).astype(np.float32)
    A = sparse.csr_matrix(sparse.triu(A, 1))
    A = sparse.csr_matrix(A + A.T)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    sources = rng.choice(n, 6, replace=False)
    p = bn.BottleneckProtocol(dec, w, sources.size, semiring, add_identity=True)
    perm0 = p.perms[0]
    X0 = _source_features(perm0, p.rows[0], n, sources, semiring)
    D, steps, _ = bn.protocol_fixed_point(p, X0, 200)
    assert steps < 200
    got = sr.distances(D, perm0, n)
    forest = csgraph.minimum_spanning_tree(A if semiring == "min_max" else sparse.csr_matrix((-A.data, A.indices, A.indptr),
                                                                                              shape=A.shape))
    forest = abs(forest)
    for i, s in enumerate(sources):
        want = _tree_path_values(sparse.csr_matrix(forest), s, semiring)
        assert np.array_equal(_bits(got[i]), _bits(want)), f"{semiring} source {s}"


def _dijkstra(n, u, v, a, s, semiring):
    """widest / minimax values from s along the edges u -> v of weight a (heap-based modified Dijkstra)"""
    larger = semiring == "max_min"
    best = np.full(n, bn.ZERO[semiring], np.float32)
    best[s] = bn.ONE[semiring]
    out = [[] for _ in range(n)]
    for x, y, w in zip(u, v, a):
        out[x].append((y, w))
    heap = [((-1 if larger else 1) * float(best[s]), s)]
    done = np.zeros(n, bool)
    while heap:
        _, x = heapq.heappop(heap)
        if done[x]:
            continue
        done[x] = True
        for y, w in out[x]:
            t = min(best[x], w) if larger else max(best[x], w)
            if (t > best[y]) if larger else (t < best[y]):
                best[y] = t
                heapq.heappush(heap, ((-1 if larger else 1) * float(t), y))
    return best


@pytest.mark.parametrize("semiring", bn.SEMIRINGS)
def test_directed_graph_against_dijkstra(semiring):
    rng = np.random.default_rng(7)
    n = 500
    r, c = rng.integers(0, n, 3000), rng.integers(0, n, 3000)
    A = sparse.csr_matrix((rng.integers(1, 30, r.size).astype(np.float32), (r, c)), shape=(n, n))
    A.sum_duplicates()
    adj = spr.weighted_adjacency([(A, None)], n)
    sources = rng.choice(n, 5, replace=False)
    X0 = np.full((n, sources.size), bn.ZERO[semiring], np.float32)
    X0[sources, np.arange(sources.size)] = bn.ONE[semiring]
    D, steps, _, _ = bn.fixed_point(adj, X0, 1000, PULL, semiring)
    assert steps < 1000
    rr = np.repeat(np.arange(n), np.diff(A.indptr))
    for i, s in enumerate(sources):
        want = _dijkstra(n, A.indices, rr, A.data, s, semiring)
        assert np.array_equal(_bits(D[:, i]), _bits(want)), f"{semiring} source {s}"


def _special_adjacency(n, rng):
    """edges with duplicates, self-loops and weights among integers, ±0, ±inf and NaN"""
    m = 6 * n
    r, c = rng.integers(0, n, m), rng.integers(0, n, m)
    r[:40], c[:40] = np.arange(40), np.arange(40)                     # self-loops
    r[40:80], c[40:80] = r[80:120], c[80:120]                         # duplicates
    w = rng.integers(-5, 20, m).astype(np.float32)
    pick = rng.random(m)
    w[pick < 0.05] = 0.0
    w[(pick >= 0.05) & (pick < 0.10)] = -0.0
    w[(pick >= 0.10) & (pick < 0.12)] = np.inf
    w[(pick >= 0.12) & (pick < 0.14)] = -np.inf
    w[(pick >= 0.14) & (pick < 0.16)] = np.nan
    order = np.lexsort((c, r))                                        # duplicates stay separate entries
    A = sparse.csr_matrix((w[order], c[order], np.r_[0, np.cumsum(np.bincount(r, minlength=n))]), shape=(n, n))
    return spr.weighted_adjacency([(A, None)], n)


def _special_features(n, k, semiring, rng):
    X = np.full((n, k), bn.ZERO[semiring], np.float32)
    pick = rng.random((n, k))
    X[pick < 0.10] = rng.integers(-5, 20, int(np.sum(pick < 0.10))).astype(np.float32)
    X[(pick >= 0.10) & (pick < 0.12)] = bn.ONE[semiring]
    X[(pick >= 0.12) & (pick < 0.15)] = np.float32(-0.0)
    X[(pick >= 0.15) & (pick < 0.18)] = np.float32(0.0)
    X[(pick >= 0.18) & (pick < 0.20)] = np.float32(np.nan)
    return X


@pytest.mark.parametrize("semiring", bn.SEMIRINGS)
def test_push_equals_pull_level_by_level(semiring):
    rng = np.random.default_rng(11)
    n, k = 700, 9
    adj = _special_adjacency(n, rng)
    X0 = _special_features(n, k, semiring, rng)
    pull = bn.fixed_point(adj, X0, 60, PULL, semiring)
    assert pull[1] < 60
    for h in range(1, pull[1] + 1):
        a = bn.fixed_point(adj, X0, h, PULL, semiring)
        b = bn.fixed_point(adj, X0, h, PUSH, semiring)
        alt = bn.fixed_point(adj, X0, h, lambda e, i=iter(range(10 ** 6)): "push" if next(i) % 2 else "pull", semiring)
        for other in (b, alt):
            assert other[1] == a[1] and np.array_equal(_bits(other[0]), _bits(a[0])), f"{semiring} level {h}"
            assert np.array_equal(other[3], a[3]), f"{semiring} level {h}: T"
    # -0 and +0 both occur in the fixed point, NaN does not
    D = pull[0]
    assert not np.isnan(D).any()
    assert np.any(_bits(D) == 0x80000000) and np.any(_bits(D) == 0)


def test_signed_zero_and_nan_rules():
    for semiring in bn.SEMIRINGS:
        z, nz = np.float32(0.0), np.float32(-0.0)
        larger = semiring == "max_min"
        assert _bits(bn.plus(z, nz, semiring)) == _bits(z if larger else nz)
        assert _bits(bn.plus(nz, z, semiring)) == _bits(z if larger else nz)
        assert _bits(bn.times(z, nz, semiring)) == _bits(nz if larger else z)
        assert bn.plus(np.float32(np.nan), np.float32(3), semiring) == 3
        assert bn.times(np.float32(np.nan), np.float32(3), semiring) == 3
        assert _bits(bn.canon(np.float32(np.nan), semiring)) == _bits(bn.ONE[semiring])
        assert _bits(bn.canon(nz, semiring)) == _bits(nz)


@pytest.mark.parametrize("name", CASES)
def test_protocol_equals_the_adjacency_fixed_point(name):
    """the restated arrow step with the identity (pull) and the weighted adjacency's fixed point agree on every golden
    decomposition that is fused-routable, with the step record and the tree"""
    g = GoldenCase(name)
    rng = np.random.default_rng(5)
    dec = spr.with_weights(g.decomposition, rng, self_loop=3.0)
    for semiring in bn.SEMIRINGS:
        p = bn.BottleneckProtocol(dec, g.width, g.k, semiring, block_diagonal=g.block_diagonal, add_identity=True)
        if not pr.fused_ok(p):
            continue
        n = p.rows[0]
        eye = sparse.csr_matrix((np.full(n, bn.ONE[semiring], np.float32), np.arange(n), np.arange(n + 1)), shape=(n, n))
        adj = spr.weighted_adjacency([(eye, None)] + pr.protocol_parts(p), n)
        X0 = _special_features(n, g.k, semiring, np.random.default_rng(2))
        Dp, sp, Tp = bn.protocol_fixed_point(p, X0, 50)
        Da, sa, _, Ta = bn.fixed_point(adj, X0, 50, PUSH, semiring)
        assert sp == sa and np.array_equal(_bits(Dp), _bits(Da)) and np.array_equal(Tp, Ta), f"{name} {semiring}"
        if sa < 50:
            bn.check_tree(adj, Da, Ta, bn.tree(adj, Da, Ta, semiring), semiring, X0=X0)


def test_tree_breaks_the_tie_cycle():
    """u = 0, v = 1 and v's real parent w = 2 all reach 5 from s = 3 (s -> w 5, w -> v 7, u <-> v 10).  The smallest
    in-neighbour with a ⊗ D[u] == D[v] is u for v and v for u: a cycle; the step record picks w for v."""
    n = 4
    r = np.array([2, 1, 0, 1])        # entry (r, c) is the edge c -> r
    c = np.array([3, 2, 1, 0])
    A = sparse.csr_matrix((np.array([5, 7, 10, 10], np.float32), (r, c)), shape=(n, n))
    adj = spr.weighted_adjacency([(A, None)], n)
    X0 = np.full((n, 1), -np.inf, np.float32)
    X0[3] = np.inf
    D, steps, _, T = bn.fixed_point(adj, X0, 10, PULL, "max_min")
    assert D[:3, 0].tolist() == [5, 5, 5] and T[:, 0].tolist() == [3, 2, 1, 0]
    P = bn.tree(adj, D, T, "max_min")
    assert P[:, 0].tolist() == [1, 2, 3, -1]
    bn.check_tree(adj, D, T, P, "max_min")


def _late_zero_case():
    """max_min, entry (r, c) the edge c -> r: s = 0 starts at +inf, the rest at -inf.  0 -> 1 (-0), 1 -> 2 (+inf),
    0 -> 3 -> 4 -> 5 (5 each), 5 -> 1 (+0).  Level 1 sets 1 to -0, level 2 sets 2 to -0, level 4 raises 1 to +0 and
    level 5 raises 2 to +0: levels 4 and 5 change no row by value, only in bits."""
    n = 6
    r = np.array([1, 2, 3, 4, 5, 1])
    c = np.array([0, 1, 0, 3, 4, 5])
    w = np.array([-0.0, np.inf, 5, 5, 5, 0.0], np.float32)
    order = np.lexsort((c, r))
    A = sparse.csr_matrix((w[order], c[order], np.r_[0, np.cumsum(np.bincount(r, minlength=n))]), shape=(n, n))
    X0 = np.full((n, 1), -np.inf, np.float32)
    X0[0] = np.inf
    return A, X0


def test_loop_stops_on_bits_not_values():
    """a level that only turns -0 into +0 is progress in the order with -0 below +0: the loop goes on, the widest value
    of 2 is +0 and its parent is 1"""
    A, X0 = _late_zero_case()
    n = A.shape[0]
    adj = spr.weighted_adjacency([(A, None)], n)
    for direction in (PULL, PUSH):
        D, steps, _, T = bn.fixed_point(adj, X0, 20, direction, "max_min")
        assert steps == 6 and T[:, 0].tolist() == [0, 4, 5, 1, 2, 3]
        assert _bits(D[:, 0]).tolist() == _bits(np.array([np.inf, 0, 0, 5, 5, 5], np.float32)).tolist()
        P = bn.tree(adj, D, T, "max_min")
        assert P[:, 0].tolist() == [-1, 5, 1, 0, 3, 4]
        bn.check_tree(adj, D, T, P, "max_min")


def test_nan_feature_reaching_through_the_identity_weight_has_no_parent():
    """0 is NaN, 0 -> 1 has weight +inf: level 1 gives both +inf with T = 1, so 1 has no parent; check_tree allows
    exactly this"""
    n = 3
    A = sparse.csr_matrix((np.array([np.inf, 4.0], np.float32), np.array([0, 1]), np.array([0, 0, 1, 2])), shape=(n, n))
    adj = spr.weighted_adjacency([(A, None)], n)
    X0 = np.array([[np.nan], [-np.inf], [-np.inf]], np.float32)
    D, steps, _, T = bn.fixed_point(adj, X0, 20, PULL, "max_min")
    assert D[:, 0].tolist() == [np.inf, np.inf, 4.0] and T[:, 0].tolist() == [1, 1, 2]
    P = bn.tree(adj, D, T, "max_min")
    assert P[:, 0].tolist() == [-1, -1, 1]
    bn.check_tree(adj, D, T, P, "max_min", X0=X0)
    with pytest.raises(AssertionError, match="no parent"):
        bn.check_tree(adj, D, T, P, "max_min")


@pytest.mark.parametrize("semiring", bn.SEMIRINGS)
def test_tree_with_all_weights_equal(semiring):
    rng = np.random.default_rng(9)
    n, k = 400, 6
    r, c = rng.integers(0, n, 2400), rng.integers(0, n, 2400)
    A = sparse.csr_matrix((np.full(r.size, 4.0, np.float32), (r, c)), shape=(n, n))
    adj = spr.weighted_adjacency([(A, None)], n)
    X0 = np.full((n, k), bn.ZERO[semiring], np.float32)
    X0[rng.choice(n, k), np.arange(k)] = bn.ONE[semiring]
    D, steps, _, T = bn.fixed_point(adj, X0, 100, PULL, semiring)
    assert steps < 100
    P = bn.tree(adj, D, T, semiring)
    bn.check_tree(adj, D, T, P, semiring)
    reached = (T > 0) & (D != bn.ZERO[semiring])
    assert reached.sum() > n and np.all(D[reached] == 4.0)
    assert np.all((P >= 0) == reached)


# ---- refusals before any CUDA call -------------------------------------------------------------------------------------
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


def _bare_engine(semiring, add_identity=True, fused_ok=True, mode="fused", L=2):
    eng = object.__new__(ArrowEngine)
    eng.sr, eng.semiring, eng.add_identity, eng.fused_ok = _lib.SEMIRINGS[semiring], semiring, add_identity, fused_ok
    eng._neg_zero_weight, eng.mode, eng.L = False, mode, L
    return eng


def test_refusals_happen_before_any_cuda_call(no_cuda):
    for other in ("min_plus", "max_plus", "plus_times", "or_and"):
        with pytest.raises(ValueError, match="max_min / min_max"):
            _bare_engine(other).bottleneck_tree(10)
    for semiring in bn.SEMIRINGS:
        with pytest.raises(ValueError, match="add_identity"):
            _bare_engine(semiring, add_identity=False).bottleneck_tree(10)
        with pytest.raises(ValueError, match="sentinel"):
            _bare_engine(semiring, fused_ok=False).bottleneck_tree(10)
        with pytest.raises(ValueError, match="bottleneck_tree"):
            _bare_engine(semiring).predecessors()
        assert _bare_engine(semiring)._sr_push_ok() and _bare_engine(semiring, mode="exchange", L=2)._sr_push_ok()
        for eng in (_bare_engine(semiring, add_identity=False), _bare_engine(semiring, fused_ok=False),
                    _bare_engine(semiring, mode="exchange", L=1)):
            assert not eng._sr_push_ok()
        assert semiring_code(semiring, np.float32) == _lib.SEMIRINGS[semiring]
        with pytest.raises(ValueError, match="float32"):
            semiring_code(semiring, np.float64)
        with pytest.raises(ValueError, match="gather"):
            semiring_code(semiring, np.float32, "scatter")
        arrow = ArrowDecompositionMPI.initialize(_TwoRanks(), [4, 4], None, None, 8, 4, 'gpu', True, True,
                                                 semiring=semiring, add_identity=True)
        with pytest.raises(ValueError, match="one GPU"):
            arrow.bottleneck_tree(10)
        arrow = ArrowDecompositionMPI.initialize(SelfComm(), [4, 4], None, None, 8, 4, 'gpu', True, True,
                                                 semiring=semiring, add_identity=True)
        with pytest.raises(RuntimeError, match="not loaded"):
            arrow.bottleneck_tree(10)
        arrow._engine = _NoCuda()
        with pytest.raises(ValueError, match="one GPU"):
            arrow.bottleneck_tree(10)
    assert (_lib.SR_MAX_MIN, _lib.SR_MIN_MAX) == (4, 5) and 7 not in _lib.SEMIRINGS.values()


# ---- the dispatch in the CUDA source -----------------------------------------------------------------------------------
def _source():
    with open(td.SOURCE) as f:
        return f.read()


def test_bottleneck_push_instances_are_reached_by_the_gpu_sweep():
    src = _source()
    body = src[src.index("void launch_bottleneck_push("):]
    body = body[:body.index("\n}\n")]
    kinds = set(re.findall(r"k_sr_push<SR, (\w+)>", body))
    assert kinds == {"float4", "float"}
    push = src[src.index("int arrow_sr_push_frontier(arrow_ctx *ctx"):]
    push = push[:push.index("\n}\n")]
    assert set(re.findall(r"launch_bottleneck_push<(\w+)>", push)) == {"SrMaxMin", "SrMinMax"}
    assert {spr.push_kind(k) for k in sr.SWEEP_KS} == kinds
    # the tropical launches inside arrow_sr_push_frontier stay exactly the four of before
    assert spr.source_push_kinds(td.SOURCE) == {(s, e) for s in ("SrMinPlus", "SrMaxPlus") for e in ("float4", "float")}


def test_semiring_tile_shapes_unchanged():
    shapes = {(1, 1, True), (2, 1, True), (4, 1, True), (8, 1, True), (4, 2, True),
              (1, 1, False), (2, 1, False), (4, 1, False), (8, 1, False), (4, 2, False), (8, 2, False), (16, 2, False),
              (8, 4, False), (16, 4, False)}
    assert sr.source_sr_shapes(td.SOURCE) == shapes
    reached = {sr.sr_tile_shape(k, big) for k in sr.SWEEP_KS if k % 4 == 0 and k <= 256 for big in (True, False)}
    assert reached == shapes
    src = _source()
    body = src[src.index("int launch_tiles_sr_shape(arrow_ctx *ctx"):]
    body = body[:body.index("#undef TSR")]
    assert "launch_tiles_sr_one<GG, VV, SR, TR, TN>" in body
