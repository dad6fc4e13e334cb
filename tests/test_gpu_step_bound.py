"""Every float32 step route on the device against the per-element bound of tests/step_bound.py.

The whole-step tests elsewhere hold a step to ``1e-5 * max|C|`` of its level; here every element of level 0 is held to
``gamma_M * sum|terms|`` of its own row, on features whose scale varies by up to 2^-48 from element to element
(``step_bound.spread_features``): a row read from its neighbour, a level contribution dropped or added twice, a
precision loss on a small row or subnormals flushed to zero fail here while the normwise rule passes
(tests/test_step_bound_cpu.py plants each of them).  Three chained steps, each started from the device's own state.

Routes: ``ArrowEngine`` in exchange, fused/gather and fused/scatter mode at 1-4 levels and k from 1 to 256, the tile
options that change the schedule, ``stream_step``, the sharded engine with a world of one (two-part X operand,
row-pointer epilogues into staging and send tiles, head reduction, side lane, CUDA-graph replay), the public classes
from level files, and the benchmark's G2 decomposition at 1M rows (10M with ``ARROW_TEST_FULL_SIZE=1``) through the
rank-1 closed form.  Several ranks as threads of one process run with ``ARROW_TEST_RANK_THREADS=1`` (see
tests/test_gpu_ranks_one_gpu.py for why they are opt-in).

The worst ``err / bound`` of every route is printed at the end of the module (``pytest -s``).
"""
import os

import numpy as np
import pytest

from arrow_matrix_b200 import _lib, graphio, synth
from arrow_matrix_b200.engine import ArrowEngine
from tests import step_bound as stb
from tests.test_gpu_ranks_one_gpu import CASES, RANK_THREADS, run_ranks

pytestmark = pytest.mark.gpu

WORST = {}                      # route -> worst err / bound seen


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst err/bound per route:")
        for route in sorted(WORST):
            print(f"  {route:40s} {WORST[route]:.3g}")


def _note(route, worst):
    WORST[route] = max(WORST.get(route, 0.0), worst)


def _hub_dec(levels, seed=21, t0=12, w=64, hub_nnz=600):
    return synth.synth_decomposition(t0, w, levels=levels, perm_kind="random", seed=seed, hub_rows=2, hub_nnz=hub_nnz)


def _engine_route(route, dec, w, k, cuda_device):
    mode, _, style = route.partition("/")
    return ArrowEngine(dec, w, k, device=cuda_device, mode=mode, fused_style=style or "gather")


def _chain(eng, dec, w, k, X0, scale, route, steps=3):
    """``steps`` chained steps of an ``ArrowEngine``, each against the exact step from the device's own state; returns
    the level-0 results"""
    ex = stb.ExactStep(dec, w, k, n_blocks=eng.n_blocks)
    eng.set_features(X0)
    outs = []
    for it in range(steps):
        x = eng.features(0) if it else X0
        carried = [eng.result(j) for j in range(1, eng.L)] if eng.mode == "exchange" else None
        exact, mag = ex.run(x, carried)
        eng.step()
        got = eng.result()
        _note(route, stb.assert_step(got, exact, mag, ex.M, route=f"{route} step {it}", row_scale=scale))
        outs.append(got)
    return outs


def _features(dec, w, k, seed, **kw):
    """spread features over level 0's rows, the hub rows kept large"""
    from arrow_matrix_b200 import decomp
    n = decomp.number_of_blocks(dec[0][0], w) * w
    return stb.spread_features(n, k, w, np.random.default_rng(seed), large_rows=stb.hub_rows_of(dec), **kw)


# ---- ArrowEngine: routes x levels x k ----------------------------------------------------------------------------------
# every route at k <= 32, at 128 and at an odd k; 1-4 levels
ROUTES = [("exchange", 1, 1), ("exchange", 4, 8), ("exchange", 2, 33), ("exchange", 3, 128), ("exchange", 2, 256),
          ("fused/gather", 2, 3), ("fused/gather", 3, 16), ("fused/gather", 3, 32), ("fused/gather", 4, 64),
          ("fused/gather", 2, 128), ("fused/scatter", 3, 4), ("fused/scatter", 2, 32), ("fused/scatter", 2, 33),
          ("fused/scatter", 4, 128), ("fused/scatter", 1, 1)]


@pytest.mark.parametrize("route,levels,k", ROUTES)
def test_engine_routes(cuda_device, route, levels, k):
    dec = _hub_dec(levels, seed=levels * 100 + k)
    X0, scale = _features(dec, 64, k, seed=k)
    eng = _engine_route(route, dec, 64, k, cuda_device)
    _chain(eng, dec, 64, k, X0, scale, route)
    eng.close()


@pytest.mark.parametrize("route", ["exchange", "fused/gather", "fused/scatter"])
def test_engine_long_rows_rescaled_matrix_and_subnormal_band(cuda_device, route):
    """hub rows over one and two long-row segments, every matrix row's values rescaled by 2^-g, and a band of rows (the
    head except its hubs, and block-row 5) in the float32 subnormal range"""
    w = 64
    rng = np.random.default_rng(77)
    dec = stb.rescale_rows(_hub_dec(3, seed=5, t0=40, w=w, hub_nnz=2100), rng)
    for k in (8, 128):
        band = np.concatenate([np.arange(2, w), np.arange(5 * w, 6 * w)])
        X0, scale = _features(dec, w, k, seed=k, subnormal_rows=band)
        eng = _engine_route(route, dec, w, k, cuda_device)
        _chain(eng, dec, w, k, X0, scale, f"{route} rescaled+subnormal")
        eng.close()


@pytest.mark.parametrize("k", [16, 128])
def test_engine_barabasi_albert_decomposition(cuda_device, k):
    """a real decomposition: a Barabasi-Albert graph through this repository's arrow decomposition (hub rows, ragged last
    block, best-effort last level), in exchange mode and -- when its permutations allow it -- both fused styles"""
    from arrow_matrix_b200.decomposition import arrow_decomposition
    w = 128
    dec = arrow_decomposition(synth.barabasi_albert(6000, 5, seed=9), w, max_number_of_levels=3, block_diagonal=True,
                              seed=1)
    X0, scale = _features(dec, w, k, seed=3)
    probe = ArrowEngine(dec, w, k, device=cuda_device, mode="exchange")
    routes = ["exchange"] + (["fused/gather", "fused/scatter"] if probe.fused_ok else [])
    probe.close()
    for route in routes:
        eng = _engine_route(route, dec, w, k, cuda_device)
        _chain(eng, dec, w, k, X0, scale, f"{route} BA")
        eng.close()


def test_engine_non_nested_stale_rows(cuda_device):
    """non-nested permutations: rows behind the sentinel carry the previous step's level tiles (exchange mode)"""
    w, k = 32, 8
    dec = synth.synth_decomposition(8, w, levels=3, perm_kind="random", seed=4, nested=False, hub_rows=1, hub_nnz=200)
    X0, scale = _features(dec, w, k, seed=1)
    eng = ArrowEngine(dec, w, k, device=cuda_device, mode="auto")
    assert eng.mode == "exchange" and not eng.fused_ok
    _chain(eng, dec, w, k, X0, scale, "exchange stale", steps=4)
    eng.close()


# ---- tile options that change the schedule ------------------------------------------------------------------------------
C = _lib.Context
OPTIONS = [("ROWS_PER_GROUP", C.OPT_ROWS_PER_GROUP, 0, 0), ("ROWS_PER_GROUP", C.OPT_ROWS_PER_GROUP, 1, 0),
           ("ROWS_PER_GROUP", C.OPT_ROWS_PER_GROUP, 2, 0), ("TILE_ROWS", C.OPT_TILE_ROWS, 16, 0),
           ("TILE_ROWS", C.OPT_TILE_ROWS, 128, 0), ("BIG_TILES", C.OPT_BIG_TILES, 0, 1),
           ("TILE_KERNEL", C.OPT_TILE_KERNEL, 0, 1), ("PREFETCH", C.OPT_PREFETCH, 17, 0)]
BIT_IDENTICAL = {"TILE_ROWS"}           # include/arrow_b200.h: "Results are bit-identical for every value"


@pytest.mark.parametrize("route", ["exchange", "fused/gather", "fused/scatter"])
@pytest.mark.parametrize("k", [16, 128])
def test_tile_options_meet_the_bound(cuda_device, route, k):
    w = 64
    dec = _hub_dec(3, seed=9)
    X0, scale = _features(dec, w, k, seed=k + 1)
    eng = _engine_route(route, dec, w, k, cuda_device)
    default = _chain(eng, dec, w, k, X0, scale, f"{route} default options")
    try:
        for name, opt, value, restore in OPTIONS:
            eng.ctx.set_option(opt, value)
            try:
                outs = _chain(eng, dec, w, k, X0, scale, f"{route} {name}={value}")
            finally:
                eng.ctx.set_option(opt, restore)
            if name in BIT_IDENTICAL:
                for it, (a, b) in enumerate(zip(outs, default)):
                    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{route} k={k} {name}={value} step {it}"
    finally:
        eng.close()


# ---- streaming ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route", ["exchange", "fused/gather", "fused/scatter"])
def test_stream_step_bit_identical_and_within_the_bound(cuda_device, route):
    w, k = 64, 32
    dec = _hub_dec(3, seed=13)
    n = 12 * w
    rng = np.random.default_rng(4)
    Xs = [stb.spread_features(n, k, w, rng, large_rows=stb.hub_rows_of(dec)) for _ in range(4)]
    ex = stb.ExactStep(dec, w, k)
    eng = _engine_route(route, dec, w, k, cuda_device)
    want = []
    for i, (X, scale) in enumerate(Xs):                 # blocking calls; exchange mode carries its level tiles
        carried = [eng.result(j) for j in range(1, eng.L)] if eng.mode == "exchange" else None
        exact, mag = ex.run(X, carried)
        eng.set_features(X)
        eng.step()
        want.append(eng.result())
        _note(f"{route} blocking", stb.assert_step(want[-1], exact, mag, ex.M, route=f"{route} blocking {i}", row_scale=scale))
    eng.close()
    eng = _engine_route(route, dec, w, k, cuda_device)
    hx = [_lib.PinnedArray((n, k)) for _ in range(2)]
    hc = [_lib.PinnedArray((n, k)) for _ in range(2)]
    got = []
    for i, (X, _) in enumerate(Xs):
        if i >= 2:
            eng.stream_drain()
            got.append(hc[i % 2].array.copy())
        hx[i % 2].array[:] = X
        eng.stream_step(hx[i % 2].array, hc[i % 2].array)
    eng.stream_drain()
    got += [hc[(len(Xs) - 2) % 2].array.copy(), hc[(len(Xs) - 1) % 2].array.copy()]
    for i, (g, r) in enumerate(zip(got, want)):
        assert np.array_equal(g.view(np.uint32), r.view(np.uint32)), f"{route}: stream_step {i} differs from the blocking call"
    for h in hx + hc:
        h.close()
    eng.close()


# ---- the sharded engine, world of one -----------------------------------------------------------------------------------
def _case_dec(case):
    w, t0, k, levels, nested, banded = CASES[case]
    dec = synth.synth_decomposition(t0, w, levels=levels, perm_kind="random", seed=31, nested=nested, hub_rows=2, hub_nnz=600,
                                    band_nnz=4 if banded else 0, shrink=1 if banded else 2)
    return dec, w, k, not banded


def _sharded_chain(eng, dec, w, k, bd, X0, scale, route, world=1, gather=None, steps=3):
    """chained steps of a sharded engine (this rank's level-0 rows); ``gather`` collects every rank's rows"""
    ex = stb.ExactStep(dec, w, k, bd, world=world)
    sh0 = eng.plan.levels[0]
    r0, r1 = sh0.r0, sh0.r1
    eng.set_features(X0[r0:r1])
    x = X0
    outs = []
    for it in range(steps):
        exact, mag = ex.run(x)
        eng.step()
        got = eng.result(0)
        _note(route, stb.assert_step(got, exact[r0:r1], mag[r0:r1], ex.M[r0:r1], route=f"{route} step {it}",
                                     row_scale=scale[r0:r1], row0=r0))
        outs.append(got)
        x = gather(got) if gather is not None else got
    return outs


SCHEDULES = ["fused", "fused+side", "fused+side+graph"]


def _sharded_engine(dec, w, k, bd, schedule, comm, device, rank=0, world=1):
    from arrow_matrix_b200.sharded import CudaPeerBackend, ShardPlan, ShardedArrowEngine
    plan = ShardPlan(dec, w, rank, world, block_diagonal=bd)
    be = CudaPeerBackend(comm, device, w, plan=plan)
    eng = ShardedArrowEngine(plan, k, be, overlap="side" in schedule, mode="fused")
    assert eng.fp is not None and eng.mode.startswith("fused")
    eng.use_graphs = "graph" in schedule
    return eng


@pytest.mark.parametrize("schedule", SCHEDULES)
@pytest.mark.parametrize("case", [c for c in CASES if c != "L3stale_k6"])
def test_world_of_one_fused_engine(cuda_device, case, schedule):
    from arrow_matrix_b200.comm import SelfComm
    dec, w, k, bd = _case_dec(case)
    X0, scale = _features(dec, w, k, seed=2)
    eng = _sharded_engine(dec, w, k, bd, schedule, SelfComm(), cuda_device)
    _sharded_chain(eng, dec, w, k, bd, X0, scale, f"sharded {schedule} w=1")
    eng.close()


def _push_option_runs(eng, X_own, steps=2):
    """level-0 results of ``steps`` chained steps from ``X_own`` under the default push schedule, block-after-block
    pushes (``OPT_PUSH_INTERLEAVE`` 0) and a one-CTA push grid (``OPT_PUSH_CTAS`` 1)"""
    ctx = eng.ctx
    runs = {}
    eng.use_graphs = False                          # a replayed graph keeps the grid it was captured with
    for name, opt, value, restore in (("default", None, None, None), ("PUSH_INTERLEAVE=0", C.OPT_PUSH_INTERLEAVE, 0, 1),
                                      ("PUSH_CTAS=1", C.OPT_PUSH_CTAS, 1, 0)):
        if opt is not None:
            ctx.set_option(opt, value)
        try:
            eng.set_features(X_own)
            outs = []
            for _ in range(steps):
                eng.step()
                outs.append(eng.result(0))
            runs[name] = outs
        finally:
            if opt is not None:
                ctx.set_option(opt, restore)
    return runs


def _assert_push_runs_identical(runs, what):
    base = runs["default"]
    for name, outs in runs.items():
        for it, (a, b) in enumerate(zip(outs, base)):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{what}: {name} step {it} is not bit-identical"


@pytest.mark.parametrize("case", ["L2k128", "banded_k8"])
def test_world_of_one_push_options_bit_identical(cuda_device, case):
    from arrow_matrix_b200.comm import SelfComm
    dec, w, k, bd = _case_dec(case)
    X0, _ = _features(dec, w, k, seed=6)
    eng = _sharded_engine(dec, w, k, bd, "fused+side", SelfComm(), cuda_device)
    _assert_push_runs_identical(_push_option_runs(eng, X0), case)
    eng.close()


# ---- the public classes from level files --------------------------------------------------------------------------------
def test_public_classes_from_level_files(cuda_device, tmp_path):
    from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
    from arrow_matrix_b200.comm import SelfComm
    w, k = 64, 24
    dec = synth.synth_decomposition(10, w, levels=3, perm_kind="random", seed=5, hub_rows=2, hub_nnz=700)
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, w, True)
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, w, True, slim=True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, w, k, 'gpu', True, True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    arrow.B.zero_rhs(w, k)
    X0, scale = _features(dec, w, k, seed=8)
    ex = stb.ExactStep(dec, w, k, n_blocks=n_blocks)
    arrow.B.set_features(X0)
    x = X0
    for it in range(3):
        exact, mag = ex.run(x)
        arrow.step()
        got = arrow.B.result_tile()
        _note("ArrowDecompositionMPI", stb.assert_step(got, exact, mag, ex.M, route=f"ArrowDecompositionMPI step {it}",
                                                       row_scale=scale))
        x = got
    arrow._engine.close()


# ---- benchmark scale: the rank-1 closed form ----------------------------------------------------------------------------
@pytest.mark.parametrize("k", [128, 16])
def test_benchmark_scale_rank1(cuda_device, k):
    """G2 at width 10 000, random level-1 permutation (seed 503): 100 block-rows (1M rows), 1000 with
    ARROW_TEST_FULL_SIZE=1 -- the decomposition bench.py times"""
    full = os.environ.get("ARROW_TEST_FULL_SIZE") == "1"
    blocks, w = (1000 if full else 100), 10000
    n = blocks * w
    dec = synth.synth_decomposition(blocks, w, levels=2, perm_kind="random", seed=503)
    u, v = stb.rank1_vectors(n, k, w, np.random.default_rng(503))
    R = stb.Rank1Step.build(dec, w, u, v)
    eng = ArrowEngine(dec, w, k, device=cuda_device)
    hx, hc = _lib.PinnedArray((n, k)), _lib.PinnedArray((n, k))
    for a0 in range(0, n, 1 << 20):
        a1 = min(n, a0 + (1 << 20))
        hx.array[a0:a1] = stb.rank1_features(u, v, a0, a1)
    eng.set_features(hx.array)
    eng.step()
    got = eng.result(0, hc.array)
    worst, msg = R.check(got, route=f"{eng.mode} G2 {n} rows k={k}", row_scale=np.abs(u))
    _note(f"{eng.mode}/{eng.fused_style} G2 rank-1 k={k}", worst)
    eng.close()
    hx.close()
    hc.close()
    assert worst <= 1.0, msg


# ---- several ranks as threads of this process (opt-in) ------------------------------------------------------------------
RANK_MATRIX = [(2, "L2k128", "fused+side+graph"), (3, "L4k8", "fused"), (2, "banded_k8", "fused+side")]


@pytest.mark.skipif(not RANK_THREADS, reason="rank threads inside one CUDA context are timing sensitive on hardware "
                                             "(tests/test_gpu_ranks_one_gpu.py); set ARROW_TEST_RANK_THREADS=1")
@pytest.mark.parametrize("world,case,schedule", RANK_MATRIX)
def test_rank_threads(cuda_device, world, case, schedule):
    dec, w, k, bd = _case_dec(case)
    X0, scale = _features(dec, w, k, seed=2)

    def rank_body(rank, comm):
        eng = _sharded_engine(dec, w, k, bd, schedule, comm, cuda_device, rank, world)
        sh0 = eng.plan.levels[0]
        _sharded_chain(eng, dec, w, k, bd, X0, scale, f"sharded {schedule} w={world}", world=world,
                       gather=lambda rows: np.concatenate(comm.allgather(rows)))
        runs = _push_option_runs(eng, X0[sh0.r0:sh0.r1])
        eng.sync()
        comm.Barrier()
        eng.close()
        _assert_push_runs_identical(runs, f"{case} rank {rank}")

    run_ranks(world, rank_body)
