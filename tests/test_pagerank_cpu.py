"""CPU tests of personalized PageRank: the host restatement of tests/pagerank_ref.py against networkx.pagerank and a
direct solve of the fixed point, the stop rule's guarantee and mass conservation, the error bound against correct and
faulty simulated devices, and the refusals ArrowEngine.pagerank raises before any CUDA work."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse.linalg import spsolve

from arrow_matrix_b200 import _lib
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from tests import pagerank_ref as prr
from tests.golden_util import CASES, GoldenCase


def _seeds(n, k, seed):
    X = np.zeros((n, k), np.float32)
    X[np.random.default_rng(seed).integers(0, n, k), np.arange(k)] = 1.0
    return X


def directed_ba(n, m, seed, sinks=0.3):
    """a Barabasi-Albert pattern, symmetric so that the decomposition keeps every row, whose edges u -> v (entry (v, u))
    carry random positive integer weights, except that a ``sinks`` share of the vertices have weight 0 on every edge
    they leave: dangling once the operator has no identity diagonal"""
    rng = np.random.default_rng(seed)
    src, dst = [], []
    targets = list(range(m))
    pool = []
    for v in range(m, n):
        for t in set(targets):
            src.append(v), dst.append(t)
        pool.extend(targets)
        pool.extend([v] * m)
        targets = [pool[i] for i in rng.integers(0, len(pool), m)]
    u, v = np.r_[src, dst], np.r_[dst, src]
    w = rng.integers(1, 5, u.size).astype(np.float32)
    w[rng.random(n)[u] < sinks] = 0
    return sparse.csr_matrix((w, (v, u)), shape=(n, n))


def _decompose(A, width, seed=0):
    return arrow_decomposition(sparse.csr_matrix(A), width, max_number_of_levels=3, block_diagonal=True, seed=seed)


def _golden_walks(dtype):
    for name in CASES:
        g = GoldenCase(name)
        parts, proto = prr.level_parts([(abs(sparse.csr_matrix(B)), p) for B, p in g.decomposition], g.width,
                                       block_diagonal=g.block_diagonal, add_identity=True, dtype=dtype)
        yield name, prr.Walk(parts, proto.rows[0], dtype, proto.to_prev, g.width)


def _walks(dtype=np.float32):
    yield from _golden_walks(dtype)
    for seed in (1, 2):
        A = directed_ba(1536, 3, seed)
        yield f"ba{seed}", prr.Walk.of(_decompose(A, 128, seed), 128, dtype)          # no identity: dangling rows


def _fixed_point(walk, S, alpha):
    """p* = alpha M^ p* + (1 - alpha + alpha m(p*)) S, solved directly: (I - alpha M^ - alpha S d^T) p = (1 - alpha) S"""
    n = walk.n
    d = walk.dangling.astype(np.float64)
    out = np.zeros(S.shape)
    I = sparse.identity(n, format="csc")
    for s in range(S.shape[1]):
        A = I - alpha * walk.M.tocsc() - alpha * sparse.csc_matrix(np.outer(S[:, s], d))
        out[:, s] = spsolve(A.tocsc(), (1 - alpha) * S[:, s].astype(np.float64))
    return out


def test_restatement_matches_networkx_and_the_fixed_point():
    import networkx as nx
    alpha = 0.85
    for name, walk in _walks(np.float64):
        if walk.n > 2000:
            continue
        X0 = _seeds(walk.n, 2, 7)
        S, _, _ = walk.restart(X0)
        p, res, _ = walk.loop64(X0, alpha, 1e-14, 500)
        assert res[-1].max() <= 1e-14, name
        assert np.allclose(p, _fixed_point(walk, S, alpha), rtol=0, atol=1e-11), name
        G = prr.nx_graph(walk.parts, walk.n)
        for s in range(2):
            pers = {v: float(S[v, s]) for v in np.flatnonzero(S[:, s])}
            ref = nx.pagerank(G, alpha=alpha, personalization=pers, dangling=pers, tol=1e-15, max_iter=2000)
            got = np.array([ref[v] for v in range(walk.n)])
            assert np.allclose(p[:, s], got, rtol=0, atol=1e-10), name


def test_stop_rule_guarantee_and_mass():
    """||p - p*||_1 <= alpha / (1 - alpha) * r after the step whose residual is r; every iterate has mass 1"""
    for alpha in (0.5, 0.85, 0.95):
        for name, walk in _walks(np.float64):
            X0 = _seeds(walk.n, 3, 11) + (np.arange(walk.n)[:, None] % 5 == 0).astype(np.float32)
            S, _, _ = walk.restart(X0)
            pstar = _fixed_point(walk, S, alpha) if walk.n <= 2000 else walk.loop64(X0, alpha, 0.0, 3000)[0]
            for steps in (1, 3, 10):
                p, res, its = walk.loop64(X0, alpha, 0.0, steps)
                err = np.abs(p - pstar).sum(axis=0)
                assert np.all(err <= alpha / (1 - alpha) * res[-1] * (1 + 1e-9) + 1e-12), (name, alpha, steps)
                for q in its:
                    assert np.allclose(q.sum(axis=0), 1.0, rtol=0, atol=1e-12), name


def test_weights_restart_and_update_restatement():
    """w in the stated order (a sequential sum differs from a pairwise one), inv and the update's exact rounding"""
    rng = np.random.default_rng(5)
    A = directed_ba(1024, 4, 3)
    A.data = rng.random(A.data.size).astype(np.float32) * 1e3
    walk = prr.Walk.of(_decompose(A, 64, 3), 64, np.float32, add_identity=False)
    u, _, a, ok = prr.entries(walk.parts)
    for v in rng.integers(0, walk.n, 50):
        e = np.flatnonzero(ok & (u == v))
        acc = 0.0
        for x in a[e]:
            acc += float(x)
        assert walk.w[v] == acc
        assert walk.inv[v] == (np.float32(1.0 / acc) if acc else 0)
    X0 = rng.random((walk.n, 5)).astype(np.float32)
    S, sigma, m0 = walk.restart(X0)
    assert np.array_equal(sigma, prr.chunk_sums(X0.astype(np.float64)))
    Y = rng.random((walk.n, 5)).astype(np.float32)
    q, r, m = prr.update(Y, S, S, walk.dangling, 0.85, m0, np.float32)
    c = (1.0 - 0.85) + 0.85 * m0
    for v, s in zip(rng.integers(0, walk.n, 20), rng.integers(0, 5, 20)):
        assert q[v, s] == np.float32(0.85 * float(Y[v, s]) + c[s] * float(S[v, s]))


def test_chunk_sums_are_sequential_in_chunks():
    rng = np.random.default_rng(9)
    X = rng.random((1300, 3)) * 10.0 ** rng.integers(-8, 8, (1300, 3))
    got = prr.chunk_sums(X)
    for s in range(3):
        parts = []
        for b in range(0, 1300, 512):
            acc = 0.0
            for x in X[b:b + 512, s]:
                acc += x
            parts.append(acc)
        acc = 0.0
        for x in parts:
            acc += x
        assert got[s] == acc


def _simulate(walk, X0, alpha, steps, order="forward", fault=None, seed=0):
    """a float32 device: the step as sequential fp32 sums over every row's terms in the given order, then the update;
    ``fault`` plants one bug"""
    S, _, m = walk.restart(X0)
    if fault == "unnormalised":
        S = S.copy()
        S[:, 0] = X0[:, 0]
    M = walk.M.tocsr()
    rows = np.repeat(np.arange(walk.n), np.diff(M.indptr))
    cols, vals = M.indices, M.data.astype(np.float32)
    key = {"forward": np.arange(rows.size), "reverse": -np.arange(rows.size),
           "random": np.random.default_rng(seed).permutation(rows.size), "magnitude": vals}[order]
    perm = np.lexsort((key, rows))
    rows, cols, vals = rows[perm], cols[perm], vals[perm]
    counts = np.bincount(rows, minlength=walk.n)
    starts = np.r_[0, np.cumsum(counts)[:-1]]
    p = S.copy()
    for _ in range(steps):
        Y = np.zeros_like(p)
        for i in range(int(counts.max(initial=0))):
            sel = np.flatnonzero(counts > i)
            e = starts[sel] + i
            Y[sel] = Y[sel] + vals[e][:, None] * p[cols[e]]
        if fault == "neighbour":
            v = int(np.argmax(X0[:, 0]))
            Y[v] = Y[(v + 1) % walk.n]
        mm = np.zeros_like(m) if fault == "dangling" else m
        if fault == "alpha twice":
            Y = (alpha * Y.astype(np.float64)).astype(np.float32)
        p, _, m = prr.update(Y, p, S, walk.dangling, alpha, mm, np.float32)
    return p


def _ratio(walk, X0, alpha, steps, **kw):
    _, _, its = walk.loop64(X0, alpha, 0.0, steps)
    got = _simulate(walk, X0, alpha, steps, **kw)
    err = np.abs(got.astype(np.float64) - its[-1]).sum(axis=0)
    return float(np.max(err / walk.bound(its, alpha)))


@pytest.mark.parametrize("order", ["forward", "reverse", "random", "magnitude"])
def test_bound_has_no_false_alarm(order):
    for name, walk in _walks():
        X0 = _seeds(walk.n, 3, 4)
        assert _ratio(walk, X0, 0.85, 6, order=order) <= 1.0, name


@pytest.mark.parametrize("fault", ["dangling", "alpha twice", "unnormalised", "neighbour"])
def test_planted_faults_fail_the_bound(fault):
    A = directed_ba(1536, 3, 1)
    walk = prr.Walk.of(_decompose(A, 128, 1), 128, np.float32)
    X0 = _seeds(walk.n, 3, 4)
    if fault == "unnormalised":
        X0[:, 0] *= 2
    if fault == "dangling":
        X0 = np.zeros_like(X0)
        X0[np.flatnonzero(walk.dangling)[:3], np.arange(3)] = 1
    assert _ratio(walk, X0, 0.85, 6, fault=fault) > 1.0


# ---- refusals before any CUDA work -------------------------------------------------------------------------------------
class _Fake:
    """an ArrowEngine shell with no device: pagerank's checks run, any CUDA call fails the test"""


def _shell(sr=_lib.SR_PLUS_TIMES, fused_ok=True, rows=8, k=2, dtype=np.float32, refusal=None):
    e = ArrowEngine.__new__(ArrowEngine)
    e.sr, e.semiring, e.fused_ok, e.k, e.dtype = sr, {v: n for n, v in _lib.SEMIRINGS.items()}[sr], fused_ok, k, np.dtype(dtype)
    e._pr_refusal = refusal

    class L:
        pass
    st = L()
    st.rows = rows
    e.levels = [st]

    def no_cuda(*a, **kw):
        raise AssertionError("CUDA work before the refusal")
    e.sync = e._pagerank_prepare = no_cuda
    return e


@pytest.mark.parametrize("kw, match", [
    (dict(sr=_lib.SR_MIN_PLUS), "plus_times"),
    (dict(sr=_lib.SR_OR_AND), "plus_times"),
    (dict(fused_ok=False), "sentinel"),
    (dict(refusal="pagerank needs every edge weight"), "edge weight"),
])
def test_engine_refusals(kw, match):
    with pytest.raises(ValueError, match=match):
        _shell(**kw).pagerank(5)


@pytest.mark.parametrize("args, match", [
    (dict(alpha=1.0), "alpha"), (dict(alpha=-0.1), "alpha"), (dict(alpha=float("nan")), "alpha"),
    (dict(tol=-1e-9), "tol"), (dict(tol=float("nan")), "tol"), (dict(max_steps=-1), "max_steps"),
    (dict(out=np.zeros((8, 2), np.float64)), "out"), (dict(out=np.zeros((8, 3), np.float32)), "out"),
    (dict(out=np.zeros((2, 8), np.float32).T), "out"),
])
def test_argument_refusals(args, match):
    args = dict(dict(max_steps=5), **args)
    with pytest.raises(ValueError, match=match):
        _shell().pagerank(**args)


def test_mpi_forwarding_refuses_several_ranks():
    from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI

    class Comm:
        def Get_size(self):
            return 2
    obj = ArrowDecompositionMPI.__new__(ArrowDecompositionMPI)
    obj.comm = Comm()
    with pytest.raises(ValueError, match="one GPU"):
        obj.pagerank(3)
