"""The direction-optimising min_plus / max_plus fixed point on one GPU, held EXACTLY (bit for bit) to the host
restatement of tests/sr_push_ref.py: the weighted push adjacency, the frontier record, the push at every feature width,
and iterate_to_fixed_point under forced push, forced pull and the automatic rule against each other, the restated step
and Dijkstra."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200 import _lib, decomp, graphio
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from tests import push_ref as pr
from tests import semiring_ref as sr
from tests import sr_push_ref as spr
from tests.golden_util import GPU_CASES, GoldenCase

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_HANDLE, ERR_RANGE, ERR_UNSUPPORTED = -2, -3, -4, -6
Ctx = _lib.Context
GRIDS = [("1 CTA", [(Ctx.OPT_SPMM_SM_LIMIT, 1), (Ctx.OPT_SPMM_CTAS_PER_SM, 1)]), ("default grid", [])]
DEFAULTS = [(Ctx.OPT_SPMM_SM_LIMIT, 0), (Ctx.OPT_SPMM_CTAS_PER_SM, 0)]
ALL_PUSH, ALL_PULL = 1 << 62, 0          # ArrowEngine._push_limit: push iff the frontier's edges are fewer
SEMIRINGS = ["min_plus", "max_plus"]
CODE = {"min_plus": _lib.SR_MIN_PLUS, "max_plus": _lib.SR_MAX_PLUS}


def _bits(X):
    return np.asarray(X, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(cuda_device)
    yield c
    c.close()


def _code(fn):
    with pytest.raises(_lib.ArrowError) as e:
        fn()
    return e.value.code


def _tile(ctx, X):
    d = ctx.dense_alloc(X.shape[0], X.shape[1])
    d.h2d(np.ascontiguousarray(X, np.float32))
    return d


def _engine(dec, width, k, cuda_device, semiring, mode="auto", block_diagonal=True, limit=None):
    eng = ArrowEngine(dec, width, k, block_diagonal=block_diagonal, device=cuda_device, mode=mode, semiring=semiring,
                      add_identity=True)
    eng._push_limit = limit
    return eng


def _device_adj(adj):
    indptr, indices = adj.d2h()
    return (indptr,) + spr.sort_duplicates(indptr, indices, adj.values_d2h())


def _assert_adj(got, want, label):
    assert np.array_equal(got[0], want[0]), f"{label}: row pointers differ"
    assert np.array_equal(got[1], want[1]), f"{label}: {int(np.sum(got[1] != want[1]))} destinations differ"
    assert np.array_equal(_bits(got[2]), _bits(want[2])), f"{label}: {int(np.sum(_bits(got[2]) != _bits(want[2])))} weights"


def _engine_parts(eng, p):
    """the engine's blocks as the restatement sees them: the protocol's, level 0 with the identity diagonal"""
    parts = pr.protocol_parts(p)
    n = eng.n_rows
    eye = sparse.csr_matrix((np.zeros(n, np.float32), np.arange(n), np.arange(n + 1)), shape=(n, n))
    return [(eye, None)] + parts


# ---- the adjacency ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", GPU_CASES)
def test_weighted_adjacency_of_golden_decompositions(cuda_device, name):
    g = GoldenCase(name)
    dec = spr.with_weights(g.decomposition, np.random.default_rng(1))
    eng = _engine(dec, g.width, g.k, cuda_device, "min_plus", block_diagonal=g.block_diagonal)
    p = sr.SemiringProtocol(dec, g.width, g.k, "min_plus", block_diagonal=g.block_diagonal, n_blocks=eng.n_blocks,
                            add_identity=True)
    assert eng.fused_ok == pr.fused_ok(p)
    if eng.fused_ok:
        _assert_adj(_device_adj(eng._sr_push_adjacency()), spr.weighted_adjacency(_engine_parts(eng, p), eng.n_rows), name)
    eng.close()


def test_weighted_adjacency_of_a_ba_decomposition_with_hubs(cuda_device):
    n, w = 30000, 1000
    A = sr.weighted_ba_graph(n, 3, seed=7)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    eng = _engine(dec, w, 4, cuda_device, "min_plus")
    p = sr.SemiringProtocol(dec, w, 4, "min_plus", n_blocks=eng.n_blocks, add_identity=True)
    assert eng.fused_ok and eng.L == 3
    got = _device_adj(eng._sr_push_adjacency())
    assert np.diff(got[0]).max() > 512, "no hub row"
    _assert_adj(got, spr.weighted_adjacency(_engine_parts(eng, p), eng.n_rows), "BA 30k")
    assert eng._sr_adj.info() == {"n_vertices": eng.n_rows, "n_edges": got[1].size}
    eng.close()


def test_adjacency_refusals(ctx):
    n = 64
    A = sparse.random(n, n, density=0.1, format="csr", random_state=1, dtype=np.float32)
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    d64 = ctx.csr_upload(n, n, A.indptr, A.indices, A.data.astype(np.float64), dtype=np.float64)
    short = ctx.map_upload(np.arange(n - 1), n)
    wide = ctx.map_upload(np.arange(n), n + 10)
    build = lambda parts, nv: ctx.adj_build(parts, nv, weighted=True)
    assert _code(lambda: build([(dA, short)], n)) == ERR_ARG              # a map shorter than the block
    assert _code(lambda: build([(dA, wide)], n)) == ERR_ARG               # a map reaching past the vertices
    assert _code(lambda: build([(dA, None)], n - 1)) == ERR_ARG           # an identity block past the vertices
    assert _code(lambda: build([(d64, None)], n)) == ERR_UNSUPPORTED      # fp64 weights
    build([(dA, wide)], n + 10).free()
    ctx.sync()
    ctx.graph_begin()
    code = _code(lambda: build([(dA, None)], n))
    ctx.graph_free(ctx.graph_end())
    assert code == ERR_UNSUPPORTED
    plain = ctx.adj_build([(dA, None)], n)
    assert _code(plain.values_d2h) == ERR_ARG                            # no weights
    weighted = build([(dA, None)], n)
    _assert_adj(_device_adj(weighted), spr.weighted_adjacency([(A, None)], n), "random 64")
    for h in (weighted, plain, wide, short, d64, dA):
        h.free()


# ---- the frontier record and the push --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hub_graph(ctx):
    """12 000 vertices, about 6 edges each with weights in [-3, 8] (self-loops included), and a hub row of 10 500
    destinations; (device adjacency, host adjacency)"""
    rng = np.random.default_rng(12)
    n = 12000
    r = rng.integers(0, n, 6 * n)
    c = rng.integers(0, n, 6 * n)
    hub = rng.choice(n, 10500, replace=False)
    rows, cols = np.r_[r, hub, np.arange(0, n, 97)], np.r_[c, np.full(hub.size, 7), np.arange(0, n, 97)]
    # entry (r, c) is the edge c -> r: the hub is column 7 of 10 500 rows; duplicates stay separate entries
    order = np.lexsort((cols, rows))
    A = sparse.csr_matrix((rng.integers(-3, 9, rows.size).astype(np.float32), cols[order],
                           np.r_[0, np.cumsum(np.bincount(rows, minlength=n))]), shape=(n, n))
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    adj = ctx.adj_build([(dA, None)], n, weighted=True)
    host = spr.weighted_adjacency([(A, None)], n)
    _assert_adj(_device_adj(adj), host, "hub graph")
    assert np.diff(host[0])[7] > 10000
    yield adj, host
    adj.free()
    dA.free()


def _frontiers(n, rng):
    return {"empty": np.zeros(0, np.int64), "hub": np.array([7]), "1 %": rng.choice(n, n // 100, replace=False),
            "all": np.arange(n)}


@pytest.mark.parametrize("k", sr.SWEEP_KS)
def test_mark_and_push_against_the_restatement(ctx, hub_graph, k):
    adj, host = hub_graph
    n = host[0].size - 1
    rng = np.random.default_rng(k)
    dX, dOld, dOut = ctx.dense_alloc(n, k), ctx.dense_alloc(n, k), ctx.dense_alloc(n, k)
    try:
        for semiring in SEMIRINGS:
            X = spr.special_features(n, k, semiring, rng)
            for label, F in _frontiers(n, rng).items():
                old = X.copy()
                old[F, 0] = np.where(old[F, 0] == 7.0, 8.0, 7.0)      # every frontier row differs in column 0
                dX.h2d(X)
                dOld.h2d(old)
                changed, rows, edges = ctx.sr_mark_frontier(adj, dX, dOld)
                assert (rows, edges) == (F.size, spr.frontier_edges(np.sort(F), host)), f"{semiring} {label}"
                assert changed == spr.rows_changed(X, old) == ctx.count_diff(dX, dOld), f"{semiring} {label}"
                want = spr.push(X, F, host, semiring)
                for grid, opts in GRIDS:
                    for o, v in DEFAULTS + opts:
                        ctx.set_option(o, v)
                    dOut.h2d(np.full((n, k), 12345.0, np.float32))
                    ctx.sr_push_frontier(adj, dX, dOut, CODE[semiring])
                    got = dOut.d2h()
                    bad = int(np.any(_bits(got) != _bits(want), axis=1).sum())
                    assert bad == 0, f"k={k} {semiring} {label} [{grid}]: {bad} rows"
    finally:
        for o, v in DEFAULTS:
            ctx.set_option(o, v)
        for h in (dX, dOld, dOut):
            h.free()


def test_rows_changed_is_count_diff(ctx, hub_graph):
    """twin tiles that differ only in ±0 (frontier rows, no change by value), only in NaN (the same NaN: neither; NaN
    against a number: both), and in real values"""
    adj, host = hub_graph
    n, k = host[0].size - 1, 6
    rng = np.random.default_rng(3)
    base = rng.integers(-4, 9, (n, k)).astype(np.float32)
    zeros, nans, vals = rng.choice(n, 300, replace=False), rng.choice(n, 200, replace=False), rng.choice(n, 100, replace=False)
    a, b = base.copy(), base.copy()
    a[zeros, 1], b[zeros, 1] = 0.0, -0.0
    a[nans, 2], b[nans, 2] = np.nan, np.nan
    da, db = _tile(ctx, a), _tile(ctx, b)
    changed, rows, _ = ctx.sr_mark_frontier(adj, da, db)
    assert (changed, rows) == (ctx.count_diff(da, db), zeros.size) and changed == nans.size
    b[vals, 4] += 1.0
    b[vals[:50], 2] = 3.0
    db.h2d(b)
    changed, rows, _ = ctx.sr_mark_frontier(adj, da, db)
    assert changed == ctx.count_diff(da, db) == spr.rows_changed(a, b)
    assert rows == spr.frontier(a, b).size
    da.free()
    db.free()


def test_push_refusals(ctx, hub_graph):
    adj, host = hub_graph
    n, k = host[0].size - 1, 40
    A_, B_, C_ = ctx.dense_alloc(n, k), ctx.dense_alloc(n, k), ctx.dense_alloc(n, k)
    small, narrow = ctx.dense_alloc(n - 1, k), ctx.dense_alloc(n, k - 4)
    bits, f64 = ctx.dense_alloc(n, k, _lib.BITS), ctx.dense_alloc(n, k, np.float64)
    fresh = ctx.adj_build([], n, weighted=True)
    M = sparse.eye(n, dtype=np.float32, format="csr")
    dM = ctx.csr_upload(n, n, M.indptr, M.indices, M.data)
    plain = ctx.adj_build([(dM, None)], n)
    push = ctx.sr_push_frontier
    assert _code(lambda: push(fresh, A_, B_, _lib.SR_MIN_PLUS)) == ERR_ARG            # no record
    assert _code(lambda: ctx.sr_mark_frontier(adj, small, small)) == ERR_ARG         # rows of another graph
    assert _code(lambda: ctx.sr_mark_frontier(adj, A_, narrow)) == ERR_ARG           # k
    assert _code(lambda: ctx.sr_mark_frontier(adj, bits, bits)) == ERR_ARG           # bit tiles
    assert _code(lambda: ctx.sr_mark_frontier(adj, f64, f64)) == ERR_ARG             # fp64 tiles
    ctx.sr_mark_frontier(adj, A_, C_)
    assert _code(lambda: push(adj, B_, C_, _lib.SR_MIN_PLUS)) == ERR_ARG             # a record tagged with another tile
    assert _code(lambda: push(adj, A_, A_, _lib.SR_MIN_PLUS)) == ERR_ARG             # out == x
    assert _code(lambda: push(adj, A_, small, _lib.SR_MIN_PLUS)) == ERR_ARG          # shape
    assert _code(lambda: push(adj, A_, narrow, _lib.SR_MIN_PLUS)) == ERR_ARG         # k
    assert _code(lambda: push(adj, A_, bits, _lib.SR_MIN_PLUS)) == ERR_ARG           # a bit tile
    assert _code(lambda: push(adj, A_, f64, _lib.SR_MAX_PLUS)) == ERR_ARG            # a fp64 tile
    assert _code(lambda: push(adj, A_, B_, _lib.SR_PLUS_TIMES)) == ERR_UNSUPPORTED
    assert _code(lambda: push(adj, A_, B_, _lib.SR_OR_AND)) == ERR_UNSUPPORTED
    assert _code(lambda: push(adj, A_, B_, 17)) == ERR_ARG                           # an unknown code
    ctx.sr_mark_frontier(plain, A_, C_)
    assert _code(lambda: push(plain, A_, B_, _lib.SR_MIN_PLUS)) == ERR_ARG           # no weights
    push(adj, A_, B_, _lib.SR_MIN_PLUS)
    ctx.sr_mark_frontier(adj, B_, C_)                                                  # the record moves to B
    assert _code(lambda: push(adj, A_, C_, _lib.SR_MAX_PLUS)) == ERR_ARG
    push(adj, B_, C_, _lib.SR_MAX_PLUS)
    fresh.free()
    assert _code(lambda: push(fresh, A_, B_, _lib.SR_MIN_PLUS)) == ERR_HANDLE
    assert _code(lambda: ctx.sr_mark_frontier(fresh, A_, B_)) == ERR_HANDLE
    for h in (plain, dM, A_, B_, C_, small, narrow, bits, f64):
        h.free()


# ---- iterate_to_fixed_point ------------------------------------------------------------------------------------------
DIRECTIONS = {"push": ALL_PUSH, "pull": ALL_PULL, "auto": None}


@pytest.mark.parametrize("semiring", SEMIRINGS)
@pytest.mark.parametrize("name", GPU_CASES)
def test_fixed_point_every_direction_on_golden_decompositions(cuda_device, name, semiring):
    """forced push, forced pull and the rule: the features after every level bit for bit, the same step count, then
    predecessors() and one more step() (result(j) at every level) identical.  Decompositions with stale rows pull only.
    Weights have 0, negatives and a negative self-loop, so min_plus may not reach a fixed point: 6 levels at most."""
    g = GoldenCase(name)
    rng = np.random.default_rng(5)
    dec = spr.with_weights(g.decomposition, rng)
    for mode in ("auto", "exchange"):
        runs = {}
        for label, limit in DIRECTIONS.items():
            eng = _engine(dec, g.width, g.k, cuda_device, semiring, mode=mode, block_diagonal=g.block_diagonal,
                          limit=limit)
            X0 = spr.special_features(eng.n_rows, g.k, semiring, np.random.default_rng(2))
            levels, steps = [], 0
            for h in range(1, 7):                         # the features after every level: a run of h levels
                eng.set_features(X0)
                steps = eng.iterate_to_fixed_point(h)
                levels.append(eng.features())
                assert len(eng.last_fixed_point_directions) == steps
                if steps < h:
                    break
            tag = f"{name} {eng.mode} {semiring} {label}"
            if not eng._sr_push_ok():
                assert set(eng.last_fixed_point_directions) == {"pull"}, tag
            elif label != "auto":
                assert set(eng.last_fixed_point_directions) == {label}, tag
            eng.set_features(X0)
            total = eng.iterate_to_fixed_point(6)
            full = (total, list(eng.last_fixed_point_directions), eng.features())
            pred = eng.predecessors() if eng.fused_ok else None
            eng.step()
            after = [eng.result(j) for j in range(eng.L)]
            runs[label] = (levels, steps, full, pred, after, eng.fused_ok and eng._sr_push_ok())
            eng.close()
        pull = runs["pull"]
        for label in ("push", "auto"):
            levels, steps, full, pred, after, pushed = runs[label]
            tag = f"{name} {mode} {semiring} {label}"
            assert steps == pull[1] and len(levels) == len(pull[0]), tag
            for h, (a, b) in enumerate(zip(levels, pull[0])):
                assert np.array_equal(_bits(a), _bits(b)), f"{tag}: level {h + 1}"
            assert full[0] == pull[2][0] and np.array_equal(_bits(full[2]), _bits(pull[2][2])), f"{tag}: one call"
            if pushed and label == "push":
                assert set(full[1]) == {"push"}, tag
            if pred is not None:
                assert np.array_equal(pred, pull[3]), f"{tag}: predecessors()"
            for j in range(len(after)):
                assert np.array_equal(_bits(after[j]), _bits(pull[4][j])), f"{tag}: result({j}) after step()"


def test_negative_zero_weight_pulls_every_level(cuda_device):
    g = GoldenCase(GPU_CASES[0])
    dec = [(sparse.csr_matrix(B, dtype=np.float32, copy=True), p) for B, p in g.decomposition]
    dec[0][0].data[:] = -0.0                              # whichever entries level 0's arrow keeps
    eng = _engine(dec, g.width, 2, cuda_device, "min_plus", block_diagonal=g.block_diagonal, limit=ALL_PUSH)
    assert eng._neg_zero_weight and not eng._sr_push_ok()
    eng.set_features(np.zeros((eng.n_rows, 2), np.float32))
    n = eng.iterate_to_fixed_point(4)
    assert eng.last_fixed_point_directions == ["pull"] * n and eng._sr_adj is None
    eng.close()


@pytest.mark.parametrize("k", [32, 128])
def test_sssp_through_the_level_files(cuda_device, tmp_path, k):
    """200k-vertex BA graph with weights 1-16 -> level files -> load: Dijkstra's distances under the rule, forced push
    and forced pull, the same step count and features in all three; the rule takes both directions"""
    n, w = 200000, 20000
    A = sr.weighted_ba_graph(n, 3, seed=5)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, w, True)
    sources = np.random.default_rng(8).choice(n, k, replace=False)
    want = csgraph.shortest_path(A, method="D", indices=sources).astype(np.float32)
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, w, True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, w, k, 'gpu', True, True,
                                             semiring="min_plus", add_identity=True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    eng = arrow._engine
    assert eng.fused_ok and eng._sr_push_ok()
    perm0 = decomp.prepare_permutations([p for _, p in blocks.decomposition], blocks.n_blocks, w)[0][0]
    X0 = sr.source_features(perm0, eng.n_rows, n, sources)
    runs = {}
    for label, limit in DIRECTIONS.items():
        eng._push_limit = limit
        eng.zero_rhs()
        arrow.B.set_features(X0)
        steps = arrow.iterate_to_fixed_point(500)
        got = sr.distances(eng.result(), perm0, n)
        assert np.array_equal(got, want), f"k={k} {label}: {int(np.sum(got != want))} distances differ"
        runs[label] = (steps, list(eng.last_fixed_point_directions), eng.result())
    assert runs["push"][0] == runs["pull"][0] == runs["auto"][0] < 500
    assert np.array_equal(_bits(runs["push"][2]), _bits(runs["pull"][2]))
    assert np.array_equal(_bits(runs["auto"][2]), _bits(runs["pull"][2]))
    assert set(runs["auto"][1]) == {"push", "pull"}, runs["auto"][1]
    eng.close()
