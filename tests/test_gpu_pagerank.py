"""Personalized PageRank on one GPU: the out-weights, the scaled operands, the restart and the update pass bit for bit
against the host restatement of tests/pagerank_ref.py; the whole loop on every route within the restatement's error
bound; agreement with networkx; reproducibility, the stop rule, the state left behind and the refusals."""
import numpy as np
import pytest
from scipy import sparse

from arrow_matrix_b200 import _lib, synth
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.engine import ArrowEngine
from tests import pagerank_ref as prr
from tests.golden_util import GPU_CASES, GoldenCase
from tests.test_pagerank_cpu import _decompose, _seeds, directed_ba

pytestmark = pytest.mark.gpu

Ctx = _lib.Context
DTYPES = [np.float32, np.float64]
ROUTES = [("fused", "gather"), ("fused", "scatter"), ("exchange", "gather")]
ONE_CTA = [(Ctx.OPT_SPMM_SM_LIMIT, 1), (Ctx.OPT_SPMM_CTAS_PER_SM, 1)]
DEFAULT_GRID = [(Ctx.OPT_SPMM_SM_LIMIT, 0), (Ctx.OPT_SPMM_CTAS_PER_SM, 0)]


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(cuda_device)
    yield c
    c.close()


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _hub_graph(n=3072, seed=4):
    """directed_ba with two hubs whose out- and in-lists exceed 512 entries (several 512-row chunks, long rows)"""
    A = directed_ba(n, 3, seed).tolil()
    rng = np.random.default_rng(seed)
    for hub in (5, 1700):
        for v in rng.choice(n, 900, replace=False):
            if v != hub:
                A[v, hub] = float(rng.integers(1, 5))
                A[hub, v] = float(rng.integers(1, 5))
    return A.tocsr()


def _cases():
    """(label, decomposition, width, block_diagonal)"""
    for name in GPU_CASES:
        g = GoldenCase(name)
        yield name, [(abs(sparse.csr_matrix(B)), p) for B, p in g.decomposition], g.width, g.block_diagonal
    yield "hubs", _decompose(_hub_graph(), 256, 3), 256, True
    A = directed_ba(2048, 3, 8, sinks=1.0)                   # every edge weight 0: every vertex dangling
    yield "all zero", _decompose(A, 256, 1), 256, True


def _engine(dec, width, k, dtype, block_diagonal=True, add_identity=False, mode="auto", style="gather", device=0):
    return ArrowEngine(dec, width, k, block_diagonal=block_diagonal, dtype=dtype, add_identity=add_identity, mode=mode,
                       fused_style=style, device=device)


def _walk(dec, width, dtype, block_diagonal=True, add_identity=False):
    parts, proto = prr.level_parts(dec, width, block_diagonal=block_diagonal, add_identity=add_identity, dtype=dtype)
    return prr.Walk(parts, proto.rows[0], dtype, proto.to_prev, width)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("add_identity", [False, True])
def test_out_weights_bit_exact(cuda_device, dtype, add_identity):
    for label, dec, width, bd in _cases():
        eng = _engine(dec, width, 1, dtype, bd, add_identity, device=cuda_device)
        n = eng.n_rows
        w, inv = eng.ctx.dense_alloc(n, 1, np.float64), eng.ctx.dense_alloc(n, 1, dtype)
        bad, dangling, bad_inv = eng.ctx.out_weights([(st.csr, st.cmap_dev) for st in eng.levels], n, w, inv)
        walk = _walk(dec, width, dtype, bd, add_identity)
        assert _same(w.d2h()[:, 0], walk.w) and _same(inv.d2h()[:, 0], walk.inv), label
        assert (bad, dangling, bad_inv) == (walk.bad_edges, int(walk.dangling.sum()), walk.bad_inv), label
        if label == "all zero" and not add_identity:
            assert dangling == n
        w.free(), inv.free()
        eng.close()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode, style", ROUTES)
def test_scaled_operands_through_one_step(cuda_device, dtype, mode, style):
    """one scaled step on one-hot columns gives column u_s of M^: every pair (u, v) is one entry, so the sum is exact"""
    dec = _decompose(_hub_graph(), 256, 3)
    k = 16
    eng = _engine(dec, 256, k, dtype, mode=mode, style=style, device=cuda_device)
    walk = _walk(dec, 256, dtype)
    u = np.r_[5, 1700, np.random.default_rng(2).choice(np.flatnonzero(~walk.dangling), k - 2, replace=False)]
    X = np.zeros((eng.n_rows, k), dtype)
    X[u, np.arange(k)] = 1
    eng.set_features(X)
    eng._pagerank_prepare()
    eng._pagerank_step()
    got = eng.result()
    want = walk.M[:, u].toarray().astype(dtype)
    assert _same(got, want)
    eng.close()


def _restart_and_update(ctx, n, k, dtype, rng):
    X0 = (rng.random((n, k)) * 10.0 ** rng.integers(-3, 3, (n, k))).astype(dtype)
    if n > 1:
        X0[rng.random(n) < 0.1] = 0
    inv = (rng.random(n) + 0.5).astype(dtype)
    inv[rng.random(n) < 0.3] = 0
    dangling = inv == 0
    tiles = {name: ctx.dense_alloc(r, c, dt) for name, (r, c, dt) in dict(
        x=(n, k, dtype), inv=(n, 1, dtype), s=(n, k, dtype), y=(n, k, dtype), p=(n, k, dtype),
        scratch=((n + 511) // 512, 2 * k, np.float64), state=(4, k, np.float64)).items()}
    tiles["x"].h2d(X0), tiles["inv"].h2d(inv[:, None])
    sums, bad, first = ctx.pagerank_restart(tiles["x"], tiles["inv"], tiles["s"], tiles["scratch"], tiles["state"])
    S, sigma, m0 = prr.restart(X0, dangling, dtype)
    out = dict(restart=(bad, first, _same(sums, sigma), _same(tiles["s"].d2h(), S), _same(tiles["state"].d2h()[0], m0)))
    Y = rng.random((n, k)).astype(dtype) / n
    P = rng.random((n, k)).astype(dtype) / n
    tiles["y"].h2d(Y), tiles["p"].h2d(P)
    res = ctx.pagerank_update(tiles["y"], tiles["p"], tiles["s"], tiles["inv"], tiles["scratch"], tiles["state"], 0.85)
    q, r, m = prr.update(Y, P, S, dangling, 0.85, m0, dtype)
    out["update"] = (_same(tiles["y"].d2h(), q), _same(res, r), _same(tiles["state"].d2h()[0], m),
                     _same(tiles["state"].d2h()[1], r))
    out["bits"] = tiles["y"].d2h().tobytes() + res.tobytes()
    for t in tiles.values():
        t.free()
    return out


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("k", [1, 2, 3, 16, 32, 33, 128, 257])
def test_restart_and_update_bit_exact(ctx, dtype, k):
    seen = set()
    for n in (3000, 512, 1):
        for opts in (ONE_CTA, DEFAULT_GRID):
            for o, v in opts:
                ctx.set_option(o, v)
            got = _restart_and_update(ctx, n, k, dtype, np.random.default_rng(n + k))
            assert got["restart"] == (0, -1, True, True, True), (n, opts)
            assert got["update"] == (True, True, True, True), (n, opts)
            seen.add((n, got["bits"]))
    for o, v in DEFAULT_GRID:
        ctx.set_option(o, v)
    assert len(seen) == 3                      # one result per size: the grid changes no bit


def _check_loop(eng, walk, X0, alpha, steps, label):
    eng.set_features(X0)
    p = eng.pagerank(steps, alpha, tol=0.0)
    assert eng.last_pagerank_residuals.shape == (steps, X0.shape[1])
    _, res64, its = walk.loop64(X0, alpha, 0.0, steps)
    E = walk.bound(its, alpha)
    err = np.abs(p.astype(np.float64) - its[-1]).sum(axis=0)
    assert np.all(err <= E), (label, float(np.max(err / E)))
    assert np.all(p >= 0), label
    assert np.all(np.abs(p.astype(np.float64).sum(axis=0) - 1) <= E + prr.unit(eng.dtype)[0] * eng.n_rows), label
    return float(np.max(err / E))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode, style", ROUTES)
def test_whole_loop_within_the_bound(cuda_device, dtype, mode, style):
    dec = _decompose(_hub_graph(), 256, 3)
    walk = _walk(dec, 256, dtype)
    eng = _engine(dec, 256, 33, dtype, mode=mode, style=style, device=cuda_device)
    X0 = _seeds(eng.n_rows, 33, 5).astype(dtype)
    X0[:, 3] = 1.0                                              # a uniform column
    X0[np.flatnonzero(walk.dangling)[:4], 4] = 2.0              # dangling seeds
    _check_loop(eng, walk, X0, 0.85, 12, (mode, style))
    eng.close()
    ident = _engine(dec, 256, 33, dtype, add_identity=True, mode=mode, style=style, device=cuda_device)
    _check_loop(ident, _walk(dec, 256, dtype, add_identity=True), X0, 0.5, 6, (mode, style, "identity"))
    ident.close()


def test_g2_at_a_million_rows(cuda_device):
    """G2 of bench.py at 100 blocks of 10 000 rows, k = 128: the device loop within the bound (8 columns restated)"""
    dec = synth.synth_decomposition(100, 10000, levels=2, perm_kind="random", seed=503)
    dec = [(abs(sparse.csr_matrix(B)), p) for B, p in dec]
    eng = _engine(dec, 10000, 128, np.float32, device=cuda_device)
    n = eng.n_rows
    X0 = _seeds(n, 128, 6)
    eng.set_features(X0)
    p = eng.pagerank(5, 0.85, tol=0.0)
    eng.close()
    walk = _walk(dec, 10000, np.float32)
    cols = np.arange(0, 128, 16)
    _, _, its = walk.loop64(X0[:, cols], 0.85, 0.0, 5)
    err = np.abs(p[:, cols].astype(np.float64) - its[-1]).sum(axis=0)
    assert np.all(err <= walk.bound(its, 0.85))
    assert np.all(p >= 0)


def test_agrees_with_networkx(cuda_device):
    import networkx as nx
    dec = _decompose(directed_ba(2048, 3, 12), 256, 2)
    walk = _walk(dec, 256, np.float64)
    eng = _engine(dec, 256, 4, np.float64, device=cuda_device)
    X0 = _seeds(eng.n_rows, 4, 3)
    eng.set_features(X0)
    p = eng.pagerank(1000, 0.85, tol=1e-13)
    eng.close()
    G = prr.nx_graph(walk.parts, walk.n)
    for s in range(4):
        pers = {int(v): 1.0 for v in np.flatnonzero(X0[:, s])}
        ref = nx.pagerank(G, alpha=0.85, personalization=pers, dangling=pers, tol=1e-15, max_iter=3000)
        assert np.allclose(p[:, s], [ref[v] for v in range(walk.n)], rtol=0, atol=1e-10)


def test_reproducible_stop_rule_and_state(cuda_device):
    dec = _decompose(_hub_graph(), 256, 3)
    k = 16
    eng = _engine(dec, 256, k, np.float32, device=cuda_device)
    X0 = _seeds(eng.n_rows, k, 9)
    eng.set_features(X0)
    p1 = eng.pagerank(200, 0.85, 1e-6)
    res = eng.last_pagerank_residuals
    assert res.shape[0] < 200 and res[-1].max() <= 1e-6 and np.all(res[:-1].max(axis=1) > 1e-6)
    eng.set_features(X0)
    out = np.empty_like(p1)
    p2 = eng.pagerank(200, 0.85, 1e-6, out=out)
    assert p2 is out and _same(p1, p2) and _same(res, eng.last_pagerank_residuals)
    assert _same(eng.features(), p1) and _same(eng.result(), p1)
    eng.step()
    after = eng.result()
    fresh = _engine(dec, 256, k, np.float32, device=cuda_device)
    fresh.set_features(p1)
    fresh.step()
    assert _same(after, fresh.result())
    fresh.close()
    eng.set_features(X0)
    S = eng.pagerank(0)
    assert eng.last_pagerank_residuals.shape == (0, k) and _same(S, (X0 / X0.sum(axis=0)).astype(np.float32))
    eng.set_mode("exchange")                                    # frees the scaled operands first, then the fused copies
    eng.set_features(X0)
    assert np.allclose(eng.pagerank(200, 0.85, 1e-6), p1, rtol=0, atol=1e-5)
    eng.close()


def test_mpi_forwarding(cuda_device, tmp_path):
    from arrow_matrix_b200 import graphio
    n, w, k = 4096, 512, 8
    dec = _decompose(directed_ba(n, 3, 21), w, 2)
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, w, True)
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, w, True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, w, k, 'gpu', True, True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    eng = arrow._engine
    X0 = _seeds(eng.n_rows, k, 1)
    arrow.B.set_features(X0)
    p = arrow.pagerank(50, 0.85, 1e-7)
    eng.set_features(X0)
    assert _same(p, eng.pagerank(50, 0.85, 1e-7))
    eng.close()


@pytest.mark.parametrize("value", [-1.0, np.nan, np.inf, 1e-45])
def test_refused_weights_are_remembered(cuda_device, value):
    """a negative, NaN or infinite weight, or one whose inverse overflows float32, is refused after the out-weight pass;
    the next call refuses before any CUDA work"""
    A = directed_ba(2048, 3, 5, sinks=0.0)
    A.data[:] = 1.0
    u = 77
    col = A[:, u].tocoo()
    A = A.tolil()
    if value == 1e-45:
        for v in col.row:                        # every edge leaving u: w[u] is a subnormal, 1 / w overflows
            A[v, u] = 1e-45
    else:
        A[int(col.row[0]), u] = value
    dec = _decompose(A.tocsr(), 256, 1)
    eng = _engine(dec, 256, 2, np.float32, device=cuda_device)
    eng.set_features(_seeds(eng.n_rows, 2, 1))
    with pytest.raises(ValueError, match="pagerank needs"):
        eng.pagerank(5)
    launches = eng.ctx.launch_count()
    with pytest.raises(ValueError, match="pagerank needs"):
        eng.pagerank(5)
    assert eng.ctx.launch_count() == launches
    eng.close()


@pytest.mark.parametrize("bad", ["negative", "nan", "inf", "zero column"])
def test_refused_restart_column(cuda_device, bad):
    dec = _decompose(directed_ba(2048, 3, 5), 256, 1)
    eng = _engine(dec, 256, 4, np.float32, device=cuda_device)
    X0 = _seeds(eng.n_rows, 4, 2)
    X0[10, 2] = {"negative": -1.0, "nan": np.nan, "inf": np.inf, "zero column": 0.0}[bad]
    if bad == "zero column":
        X0[:, 2] = 0
    eng.set_features(X0)
    with pytest.raises(ValueError, match="column 2"):
        eng.pagerank(5)
    assert _same(eng.features(), X0)
    X0[:, 2] = X0[:, 1]
    eng.set_features(X0)
    assert eng.pagerank(5).shape == X0.shape                   # a good restart runs
    eng.close()
