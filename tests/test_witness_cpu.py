"""CPU tests of the predecessor pass: the host restatement (tests/witness_ref.py) equals a brute-force scan, and at fixed
points of the step its parents form shortest-path trees (min_plus, Dijkstra lengths, BFS levels) and critical-path
chains (max_plus on a DAG, a topological DP); the refusals happen before any CUDA work; the GPU sweep reaches every
witness tile shape."""
import re

import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200 import _lib, graphio, synth
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition, reconstruct
from arrow_matrix_b200.engine import ArrowEngine
from tests import semiring_ref as sr
from tests import tile_dispatch as td
from tests import witness_ref as wr


def _small(seed, n=60, w=8, directed=False):
    rng = np.random.default_rng(seed)
    A = sparse.random(n, n, density=0.08, format="csr", random_state=seed, dtype=np.float32)
    A.data = rng.integers(0, 4, A.nnz).astype(np.float32)               # weights 0..3: many equal candidates
    if not directed:
        A = sparse.csr_matrix(A.maximum(A.T))
    A.setdiag(1.0)                                                         # self-loops are never candidates
    A = sparse.csr_matrix(A)
    return arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=seed), w


@pytest.mark.parametrize("semiring", ["min_plus", "max_plus"])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_restatement_equals_brute_force(semiring, seed):
    dec, w = _small(seed, directed=seed == 3)
    lv = wr.Levels(dec, w)
    assert lv.L >= 2 and lv.fused_ok()
    rng = np.random.default_rng(seed)
    D = rng.integers(0, 8, (lv.rows[0], 5)).astype(np.float32)
    D[rng.random(D.shape) < 0.1] = np.float32(sr.zero(semiring))
    D[rng.random(D.shape) < 0.05] = -np.float32(sr.zero(semiring))
    D[0, 0] = -0.0
    # half the rows take their witness value (as after one relaxation), so that many of them have a parent
    p = sr.SemiringProtocol(dec, w, D.shape[1], semiring)
    p.set_features(D)
    D = np.where(rng.random((D.shape[0], 1)) < 0.5, p.step(), D).astype(np.float32)
    got = wr.predecessors(dec, w, D, semiring, levels=lv)
    want = wr.brute_force(dec, w, D, semiring)
    assert np.array_equal(got, want)
    assert (got >= 0).sum() >= 20                                          # the test has teeth


def test_lex_plus_is_an_exact_monoid():
    """associative and commutative on ties, -0 == +0, and (identity, -1) is the identity"""
    rng = np.random.default_rng(0)
    for semiring in ("min_plus", "max_plus"):
        z = np.float32(sr.zero(semiring))
        v = rng.integers(0, 3, (3, 400)).astype(np.float32)
        v[rng.random(v.shape) < 0.2] = z
        v[0, :5] = -0.0
        lab = rng.integers(-1, 6, (3, 400)).astype(np.int32)
        lab[v != z] = np.abs(lab[v != z])
        ab = wr.lex_plus(semiring, v[0], lab[0], v[1], lab[1])
        ba = wr.lex_plus(semiring, v[1], lab[1], v[0], lab[0])
        assert np.array_equal(ab[0], ba[0]) and np.array_equal(ab[1], ba[1])
        l1 = wr.lex_plus(semiring, *ab, v[2], lab[2])
        r1 = wr.lex_plus(semiring, v[0], lab[0], *wr.lex_plus(semiring, v[1], lab[1], v[2], lab[2]))
        assert np.array_equal(l1[0], r1[0]) and np.array_equal(l1[1], r1[1])
        e = wr.lex_plus(semiring, v[0], lab[0], np.full(400, z), np.full(400, -1, np.int32))
        assert np.array_equal(e[0], v[0]) and np.array_equal(e[1], lab[0])


def _fixed_point(dec, w, X0, semiring):
    p = sr.SemiringProtocol(dec, w, X0.shape[1], semiring, add_identity=True)
    assert sum(p.dropped_nnz) == 0
    p.set_features(X0)
    for _ in range(1000):
        before = p.X[0].copy()
        p.step()
        if np.array_equal(p.C[0], before):
            return p
    raise AssertionError("no fixed point")


def _edges(A):
    """sorted (row * n + col) keys and values of A's entries"""
    A = sparse.csr_matrix(A)
    A.sort_indices()
    rows = np.repeat(np.arange(A.shape[0], dtype=np.int64), np.diff(A.indptr))
    return rows * A.shape[1] + A.indices, A.data.astype(np.float32), A.shape[1]


def _weights(E, perm0, rows_v, rows_u):
    """w(u -> v) = A[v, u] for level-0 rows (vertex ids through level 0's permutation); every pair must be an edge"""
    keys, data, nc = E
    q = perm0[rows_v].astype(np.int64) * nc + perm0[rows_u]
    i = np.minimum(np.searchsorted(keys, q), keys.size - 1)
    assert np.array_equal(keys[i], q), "a parent is not a neighbour"
    return data[i]


def _check_chains(P, D, A, perm0, n, sources_row, want_len, semiring):
    """every parent satisfies D[p] + w(p, v) == D[v]; every chain ends at its column's source after the expected length"""
    rows0, k = D.shape
    E = _edges(A)
    vi, si = np.nonzero(P >= 0)
    pu = P[vi, si]
    assert np.array_equal(D[pu, si] + _weights(E, perm0, vi, pu), D[vi, si])
    for s in range(k):
        reach = np.flatnonzero(np.isfinite(D[:, s]) & (perm0[:rows0] < n))
        length = np.zeros(reach.size, np.float64)
        cur = reach.copy()
        for _ in range(rows0 + 1):
            nxt = P[cur, s]
            live = nxt >= 0
            if not live.any():
                break
            length[live] += _weights(E, perm0, cur[live], nxt[live])
            cur = np.where(live, nxt, cur)
        else:
            raise AssertionError("a parent chain has a cycle")
        assert np.all(cur == sources_row[s]), f"column {s}: a chain ends away from its source"
        assert np.array_equal(length.astype(np.float32), want_len[s][perm0[reach]]), f"column {s}: chain lengths"


@pytest.mark.parametrize("unit", [False, True], ids=["weights 1-16", "unit weights (BFS)"])
def test_min_plus_fixed_point_parents_form_shortest_path_trees(unit):
    n, w = 3000, 100
    A = sr.weighted_ba_graph(n, 3, seed=5, unit=unit)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    sources = np.random.default_rng(3).choice(n, 8, replace=False)
    lv = wr.Levels(dec, w)
    assert lv.L == 3 and lv.fused_ok()
    perm0 = lv.perms[0]
    p = _fixed_point(dec, w, sr.source_features(perm0, lv.rows[0], n, sources), "min_plus")
    D = p.C[0]
    P = wr.predecessors(dec, w, D, "min_plus", levels=lv)
    inv = np.full(n, -1, np.int64)
    inv[perm0[: lv.rows[0]][perm0[: lv.rows[0]] < n]] = np.flatnonzero(perm0[: lv.rows[0]] < n)
    src_rows = inv[sources]
    # -1 exactly at the sources and the unreachable or padding rows
    expect_none = ~np.isfinite(D)
    expect_none[src_rows, np.arange(sources.size)] = True
    assert np.array_equal(P < 0, expect_none)
    dij = csgraph.shortest_path(A, method="D", indices=sources)
    _check_chains(P, D, A, perm0, n, src_rows, dij.astype(np.float32), "min_plus")
    if unit:                                                               # BFS: a parent is one level closer
        vi, si = np.nonzero(P >= 0)
        assert np.array_equal(D[P[vi, si], si] + 1, D[vi, si])


def test_max_plus_dag_chains_are_critical_paths():
    """longest paths of a weighted DAG (rows read their predecessors: A[v, u] = w(u -> v)) from a topological DP.  The DAG
    keeps the edges of the BA graph of the min_plus tests from the smaller vertex id to the larger; its decomposition is
    the BA graph's with -inf (a term that never wins a max) on the entries of the other direction."""
    n, w = 3000, 100
    S = sr.weighted_ba_graph(n, 3, seed=5)
    A = sparse.csr_matrix(sparse.tril(S, k=-1))
    dec = []
    for B, perm in arrow_decomposition(S, w, max_number_of_levels=3, block_diagonal=True, seed=2):
        C = sparse.coo_matrix(B)
        data = np.where(perm[C.row] > perm[C.col], C.data, -np.inf).astype(np.float32)
        dec.append((sparse.csr_matrix((data, (C.row, C.col)), shape=B.shape), perm))
    fin = [(sparse.csr_matrix(np.where(np.isfinite(B.toarray()), B.toarray(), 0)), p) for B, p in dec]
    assert abs(reconstruct(fin, n) - A).max() == 0
    lv = wr.Levels(dec, w)
    assert lv.fused_ok()
    perm0 = lv.perms[0]
    sources = np.array([0, 3, 17, 200])
    p = _fixed_point(dec, w, np.where(np.isinf(sr.source_features(perm0, lv.rows[0], n, sources)), -np.inf, 0.0)
                     .astype(np.float32), "max_plus")
    D = np.where(np.isneginf(p.C[0]), np.inf, p.C[0])                      # unreachable: same shape of test as min_plus
    P = wr.predecessors(dec, w, p.C[0], "max_plus", levels=lv)
    # topological DP in vertex order (every edge goes from a smaller to a larger id)
    Ac = sparse.csc_matrix(A.T)                                            # column v of A^T: the in-edges of v
    want = np.full((sources.size, n), -np.inf)
    want[np.arange(sources.size), sources] = 0.0
    for vv in range(n):
        lo, hi = Ac.indptr[vv], Ac.indptr[vv + 1]
        if hi > lo:
            cand = want[:, Ac.indices[lo:hi]] + Ac.data[lo:hi]
            want[:, vv] = np.maximum(want[:, vv], cand.max(axis=1))
    got = sr.distances(p.C[0], perm0, n)
    assert np.array_equal(got, want.astype(np.float32))
    inv = np.full(n, -1, np.int64)
    ok = perm0[: lv.rows[0]] < n
    inv[perm0[: lv.rows[0]][ok]] = np.flatnonzero(ok)
    want_len = np.where(np.isneginf(want), np.inf, want).astype(np.float32)
    _check_chains(P, D, A, perm0, n, inv[sources], want_len, "max_plus")


class _NoCuda:
    pass


@pytest.fixture
def no_cuda(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a CUDA call was made")
    monkeypatch.setattr(_lib.Context, "__init__", refuse)
    monkeypatch.setattr(_lib, "load_library", refuse)


def _bare_engine(dec, w, semiring, fused_ok):
    """an ArrowEngine without a device: only what predecessors() checks before its first CUDA call"""
    eng = ArrowEngine.__new__(ArrowEngine)
    eng.sr = _lib.SEMIRINGS[semiring]
    eng.fused_ok = fused_ok
    return eng


def test_refusals_happen_before_any_cuda_call(no_cuda):
    dec = synth.synth_decomposition(4, 8, levels=2, perm_kind="random", seed=3)
    with pytest.raises(ValueError, match="min_plus / max_plus"):
        _bare_engine(dec, 8, "plus_times", True).predecessors()
    with pytest.raises(ValueError, match="sentinel"):
        _bare_engine(dec, 8, "min_plus", False).predecessors()
    arrow = ArrowDecompositionMPI.initialize(SelfComm(), [4, 4], None, None, 8, 4, 'gpu', True, True,
                                             semiring="min_plus")
    with pytest.raises(RuntimeError, match="not loaded"):
        arrow.predecessors()
    arrow._engine = _NoCuda()
    with pytest.raises(ValueError, match="one GPU"):
        arrow.predecessors()


def test_restatement_refuses_rows_behind_the_sentinel():
    """a decomposition whose deeper levels read rows behind the sentinel has no label for those rows"""
    n, w = 3000, 100
    A = sparse.csr_matrix(sparse.tril(sr.weighted_ba_graph(n, 3, seed=5), k=-1))
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    lv = wr.Levels(dec, w)
    assert not lv.fused_ok()
    with pytest.raises(AssertionError, match="sentinel"):
        wr.predecessors(dec, w, np.zeros((lv.rows[0], 2), np.float32), "min_plus", levels=lv)


def wit_tile_shape(k: int, big_tiles: bool = True):
    """(G, VPL, big tiles) of the witness tile kernel a launch with ``k`` columns runs (``launch_tiles_wit_shape``): one
    float4 per lane up to 32 lanes, then two; the big tiles where launch_tiles would pick them (k <= 32)"""
    assert k % 4 == 0 and 4 <= k <= 256
    k4 = k // 4
    vpl = 2 if k4 > 32 else 1
    lanes = -(-k4 // vpl)
    g = 1
    while g < lanes:
        g <<= 1
    return g, vpl, bool(big_tiles) and k4 <= 8


def source_wit_shapes(path: str) -> set:
    """the WIB / WIS (G, VPL) lines of ``launch_tiles_wit_shape`` in the CUDA source"""
    with open(path) as f:
        src = f.read()
    body = src[src.index("int launch_tiles_wit_shape(arrow_ctx *ctx"):]
    body = body[:body.index("#undef WIS")]
    found = set()
    for macro, big in (("WIB", True), ("WIS", False)):
        for m in re.finditer(rf"(?<![A-Z]){macro}\((\d+),\s*(\d+)\);", body):
            found.add((int(m.group(1)), int(m.group(2)), big))
    return found


def test_witness_tile_shapes_are_all_reached_by_the_gpu_sweep():
    """tests/test_gpu_witness.py runs sr.SWEEP_KS with the big tiles on and off"""
    in_source = source_wit_shapes(td.SOURCE)
    reached = {wit_tile_shape(k, big) for k in sr.SWEEP_KS if k % 4 == 0 and k <= 256 for big in (True, False)}
    assert len(in_source) == 11 and reached == in_source, \
        f"unreached: {in_source - reached}, not in the source: {reached - in_source}"
