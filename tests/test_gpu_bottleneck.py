"""The bottleneck semirings (max_min, min_max) on one GPU, held EXACTLY (bit for bit) to the host restatement of
tests/bottleneck_ref.py: arrow_spmm_sr at every width (tile, generic and long-row kernels, hub rows, under every launch
option), arrow_gather_rows_sr, the engine step, the direction-optimising fixed point, the signed-zero order, and
bottleneck_tree with its entry points' refusals."""
import numpy as np
import pytest
from scipy import sparse

from arrow_matrix_b200 import _lib
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from tests import bottleneck_ref as bn
from tests import push_ref as pr
from tests import semiring_ref as sr
from tests import sr_push_ref as spr
from tests.golden_util import GPU_CASES, GoldenCase

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_HANDLE, ERR_UNSUPPORTED = -2, -3, -6
Ctx = _lib.Context
CODE = {"max_min": _lib.SR_MAX_MIN, "min_max": _lib.SR_MIN_MAX}
# (option, value) pairs that change how a launch runs but never what it computes (those of tests/test_gpu_semiring.py)
OPTIONS = [("1 CTA", [(Ctx.OPT_SPMM_SM_LIMIT, 1), (Ctx.OPT_SPMM_CTAS_PER_SM, 1)]),
           ("default", []),
           ("no L2 hints", [(Ctx.OPT_L2_HINTS_PLAIN, 0)]),
           ("big tiles off", [(Ctx.OPT_BIG_TILES, 0)]),
           ("forced predicated path", [(Ctx.OPT_FORCE_PREDICATED, 1)])]
DEFAULTS = [(Ctx.OPT_SPMM_SM_LIMIT, 0), (Ctx.OPT_SPMM_CTAS_PER_SM, 0), (Ctx.OPT_L2_HINTS_PLAIN, 3),
            (Ctx.OPT_BIG_TILES, 1), (Ctx.OPT_FORCE_PREDICATED, 0)]
GRIDS = OPTIONS[:2]
ALL_PUSH, ALL_PULL = 1 << 62, 0
DIRECTIONS = {"push": ALL_PUSH, "pull": ALL_PULL, "auto": None}


def _bits(X):
    return np.asarray(X, np.float32).view(np.uint32)


def _same(a, b):
    """bit for bit, any NaN equal to any NaN"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (_bits(a) == _bits(b)) | (np.isnan(a) & np.isnan(b))


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(cuda_device)
    yield c
    c.close()


def _set(ctx, opts):
    for o, v in DEFAULTS + list(opts):
        ctx.set_option(o, v)


def _code(fn):
    with pytest.raises(_lib.ArrowError) as e:
        fn()
    return e.value.code


def _values(rng, n, special=True):
    """integers in [-20, 20] (many ties) with ±0, ±inf and, when ``special``, NaN"""
    v = rng.integers(-20, 21, n).astype(np.float32)
    pick = rng.random(n)
    v[pick < 0.04] = 0.0
    v[(pick >= 0.04) & (pick < 0.08)] = -0.0
    v[(pick >= 0.08) & (pick < 0.10)] = np.inf
    v[(pick >= 0.10) & (pick < 0.12)] = -np.inf
    if special:
        v[(pick >= 0.12) & (pick < 0.14)] = np.nan
    return v


def _ragged_block(rng):
    """8000 rows: short ragged rows, empty rows, and hub rows of one to three long-row segments"""
    n = 8000
    lens = rng.integers(0, 24, n)
    lens[rng.integers(0, n, 120)] = 0
    lens[[7, 3000]] = [600, 5000]
    lens[6000:6004] = [513, 2048, 2049, 4100]
    ip = np.r_[0, np.cumsum(lens)]
    idx = rng.integers(0, n, int(ip[-1]))
    return sparse.csr_matrix((_values(rng, idx.size), idx, ip), shape=(n, n))


@pytest.fixture(scope="module")
def ragged():
    return _ragged_block(np.random.default_rng(64))


def _canaried(rows, k, keep, semiring, rng, special=True):
    out = np.full((rows, k), bn.WINNER[semiring], np.float32)
    keep = np.unique(keep)
    out[keep] = _values(rng, keep.size * k, special).reshape(keep.size, k)
    return out


@pytest.mark.parametrize("k", sr.SWEEP_KS)
@pytest.mark.parametrize("semiring", bn.SEMIRINGS)
def test_kernel_sweep_ragged_block(ctx, ragged, k, semiring):
    """every epilogue (plain, addend, skipped columns) under every option, against the restatement; the addend holds no
    NaN (an accumulator starting at NaN is outside the contract of the skipped slots)"""
    A = ragged
    rng = np.random.default_rng(k)
    n = A.shape[0]
    used = np.unique(A.indices)
    Xh = _canaried(n + 5, k, used, semiring, rng)
    n_add = n // 2 + 4
    amap = np.where(rng.random(n) < 0.6, rng.integers(0, n_add, n), -1).astype(np.int64)
    addh = _canaried(n_add, k, amap[amap >= 0], semiring, rng, special=False)
    cmap = rng.permutation(n + 5)[:n].astype(np.int64)
    cmap[::5] = -1
    img = cmap[used]
    Xsh = _canaried(n + 7, k, img[img >= 0], semiring, rng)
    Cinit = np.full((n + 3, k), bn.WINNER[semiring], np.float32)
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    assert dA.info()["n_long_rows"] == 6
    dmap = ctx.map_upload(cmap, n + 5)
    dAs = dA.remap_columns(dmap, n + 5)
    dam = ctx.map_upload(amap, n_add)
    dX, dXs, dadd, dC = ctx.dense_from_host(Xh), ctx.dense_from_host(Xsh), ctx.dense_from_host(addh), ctx.dense_alloc(n + 3, k)
    tile = k % 4 == 0 and k <= 256
    try:
        for epi in ("plain", "add", "skip", "skip+add"):
            skip = "skip" in epi
            want = bn.spmm(A, Xsh if skip else Xh, semiring, col_map=cmap if skip else None)
            if "add" in epi:
                ok = amap >= 0
                want[ok] = bn.plus(want[ok], addh[amap[ok]], semiring)
            for name, opts in (OPTIONS if tile else OPTIONS[:2]):
                _set(ctx, opts)
                dC.h2d(Cinit)
                ctx.spmm_sr(dAs if skip else dA, dXs if skip else dX, dC, dadd if "add" in epi else None,
                            dam if "add" in epi else None, CODE[semiring])
                got = dC.d2h()
                assert np.array_equal(_bits(got[n:]), _bits(Cinit[n:])), "rows past the block written"
                bad = ~_same(got[:n], want)
                assert not bad.any(), f"k={k} {semiring} {epi} [{name}]: {int(bad.sum())} elements differ"
    finally:
        _set(ctx, [])
        for h in (dAs, dmap, dA, dam, dX, dXs, dadd, dC):
            h.free()


@pytest.mark.parametrize("k", [1, 3, 4, 12, 64, 130])
def test_gather_rows_sr(ctx, k):
    rng = np.random.default_rng(k)
    n, m = 3000, 2000
    for semiring in bn.SEMIRINGS:
        D0 = _values(rng, n * k, special=False).reshape(n, k)
        S = _values(rng, m * k).reshape(m, k)
        mp = np.where(rng.random(n) < 0.7, rng.integers(0, m, n), -1).astype(np.int64)
        dD, dS, dm = ctx.dense_from_host(D0), ctx.dense_from_host(S), ctx.map_upload(mp, m)
        ctx.gather_rows_sr(dD, dS, dm, CODE[semiring])
        want = D0.copy()
        ok = mp >= 0
        want[ok] = bn.plus(D0[ok], S[mp[ok]], semiring)
        assert _same(dD.d2h(), want).all(), f"k={k} {semiring}"
        for h in (dD, dS, dm):
            h.free()


def test_signed_zero_order(ctx):
    """mixed-sign zeros in weights and features: ⊕ and ⊗ order -0 below +0 in the tile, generic and long-row kernels and
    in the push, bit for bit with the restatement"""
    n = 1200
    rng = np.random.default_rng(0)
    lens = np.full(n, 6)
    lens[5] = 700                                         # a long row
    ip = np.r_[0, np.cumsum(lens)]
    idx = rng.integers(0, n, int(ip[-1]))
    w = np.where(rng.random(idx.size) < 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32)
    A = sparse.csr_matrix((w, idx, ip), shape=(n, n))
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    for k in (3, 8, 128):
        X = np.where(rng.random((n, k)) < 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32)
        dX, dC = ctx.dense_from_host(X), ctx.dense_alloc(n, k)
        for semiring in bn.SEMIRINGS:
            ctx.spmm_sr(dA, dX, dC, None, None, CODE[semiring])
            got, want = dC.d2h(), bn.spmm(A, X, semiring)
            assert np.array_equal(_bits(got), _bits(want)), f"k={k} {semiring}"
            assert np.any(_bits(got) == 0) and np.any(_bits(got) == 0x80000000)
        dX.free()
        dC.free()
    adj = ctx.adj_build([(dA, None)], n, weighted=True)
    host = spr.weighted_adjacency([(A, None)], n)
    k = 8
    X = np.where(rng.random((n, k)) < 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32)
    old = X.copy()
    old[:, 0] = 5.0
    dX, dOld, dOut = ctx.dense_from_host(X), ctx.dense_from_host(old), ctx.dense_alloc(n, k)
    ctx.sr_mark_frontier(adj, dX, dOld)
    for semiring in bn.SEMIRINGS:
        ctx.sr_push_frontier(adj, dX, dOut, CODE[semiring])
        want = bn.push(X, np.arange(n), host, semiring)
        assert np.array_equal(_bits(dOut.d2h()), _bits(want)), semiring
        assert np.array_equal(_bits(want), _bits(bn.step(X, host, semiring)))
    for h in (adj, dX, dOld, dOut, dA):
        h.free()


# ---- the engine ------------------------------------------------------------------------------------------------------
def _engine(dec, width, k, cuda_device, semiring, mode="auto", block_diagonal=True, limit=None, add_identity=True):
    eng = ArrowEngine(dec, width, k, block_diagonal=block_diagonal, device=cuda_device, mode=mode, semiring=semiring,
                      add_identity=add_identity)
    eng._push_limit = limit
    return eng


def _features(rows, k, semiring, seed):
    rng = np.random.default_rng(seed)
    X = np.full((rows, k), bn.ZERO[semiring], np.float32)
    pick = rng.random((rows, k))
    X[pick < 0.3] = rng.integers(-5, 20, int(np.sum(pick < 0.3))).astype(np.float32)
    X[(pick >= 0.3) & (pick < 0.33)] = bn.ONE[semiring]
    X[(pick >= 0.33) & (pick < 0.36)] = np.float32(-0.0)
    X[(pick >= 0.36) & (pick < 0.39)] = np.float32(0.0)
    X[(pick >= 0.39) & (pick < 0.41)] = np.float32(np.nan)
    return X


@pytest.mark.parametrize("name", GPU_CASES)
def test_engine_step_golden_decompositions(cuda_device, name):
    """three steps in fused and exchange mode (stale rows included), every level's tile in exchange mode, then zero_rhs"""
    g = GoldenCase(name)
    dec = spr.with_weights(g.decomposition, np.random.default_rng(4), self_loop=3.0)
    for semiring in bn.SEMIRINGS:
        for add_identity in (False, True):
            results = {}
            for mode in ("auto", "exchange"):
                eng = _engine(dec, g.width, g.k, cuda_device, semiring, mode=mode, block_diagonal=g.block_diagonal,
                              add_identity=add_identity)
                p = bn.BottleneckProtocol(dec, g.width, g.k, semiring, block_diagonal=g.block_diagonal,
                                          n_blocks=eng.n_blocks, add_identity=add_identity)
                X0 = _features(eng.n_rows, g.k, semiring, 11)
                eng.set_features(X0)
                p.set_features(X0)
                out = []
                for it in range(3):
                    eng.step()
                    want = p.step()
                    got = eng.result()
                    tag = f"{name} {semiring} {eng.mode} identity={add_identity} step {it}"
                    assert _same(got, want).all(), tag
                    if eng.mode == "exchange":
                        for j in range(1, eng.L):
                            assert _same(eng.result(j), p.C[j]).all(), f"{tag} level {j}"
                    out.append(got)
                eng.zero_rhs()
                assert np.array_equal(_bits(eng.result()), _bits(np.full_like(X0, bn.ZERO[semiring]))), tag
                results[eng.mode] = out
                eng.close()
            if "fused" in results:
                for a, b in zip(results["fused"], results["exchange"]):
                    assert _same(a, b).all()


@pytest.mark.parametrize("semiring", bn.SEMIRINGS)
@pytest.mark.parametrize("name", GPU_CASES)
def test_fixed_point_every_direction(cuda_device, name, semiring):
    """forced push, forced pull and the rule: the features after every level bit for bit and the same step count; the
    restated protocol agrees; bottleneck_tree gives the same D and the restated tree, and a second call the same"""
    g = GoldenCase(name)
    dec = spr.with_weights(g.decomposition, np.random.default_rng(5), self_loop=3.0)
    for mode in ("auto", "exchange"):
        runs = {}
        for label, limit in DIRECTIONS.items():
            eng = _engine(dec, g.width, g.k, cuda_device, semiring, mode=mode, block_diagonal=g.block_diagonal,
                          limit=limit)
            X0 = _features(eng.n_rows, g.k, semiring, 2)
            levels, steps = [], 0
            for h in range(1, 40):
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
            tree = None
            if eng.fused_ok:
                eng.set_features(X0)
                D, P = eng.bottleneck_tree(60)
                dirs = list(eng.last_fixed_point_directions)
                eng.set_features(X0)
                D2, P2 = eng.bottleneck_tree(60)
                assert np.array_equal(_bits(D), _bits(D2)) and np.array_equal(P, P2), f"{tag}: second call"
                assert dirs == eng.last_fixed_point_directions
                p = bn.BottleneckProtocol(dec, g.width, g.k, semiring, block_diagonal=g.block_diagonal,
                                          n_blocks=eng.n_blocks, add_identity=True)
                n = eng.n_rows
                eye = sparse.csr_matrix((np.full(n, bn.ONE[semiring], np.float32), np.arange(n), np.arange(n + 1)),
                                        shape=(n, n))
                adj = spr.weighted_adjacency([(eye, None)] + pr.protocol_parts(p), n)
                Dr, sr_, _, Tr = bn.fixed_point(adj, X0, 60, lambda e: "pull", semiring)
                assert np.array_equal(_bits(D), _bits(Dr)), f"{tag}: D"
                want = bn.tree(adj, Dr, Tr, semiring)
                assert np.array_equal(P, want), f"{tag}: {int(np.sum(P != want))} parents differ"
                if sr_ < 60:
                    bn.check_tree(adj, Dr, Tr, P, semiring, X0=X0)
                tree = (D, P)
            runs[label] = (levels, steps, tree)
            eng.close()
        pull = runs["pull"]
        for label in ("push", "auto"):
            levels, steps, tree = runs[label]
            tag = f"{name} {mode} {semiring} {label}"
            assert steps == pull[1] and len(levels) == len(pull[0]), tag
            for h, (a, b) in enumerate(zip(levels, pull[0])):
                assert np.array_equal(_bits(a), _bits(b)), f"{tag}: level {h + 1}"
            if tree is not None:
                assert np.array_equal(_bits(tree[0]), _bits(pull[2][0])) and np.array_equal(tree[1], pull[2][1]), tag


BA_KS = [1, 5, 32, 33, 128, 260]


@pytest.fixture(scope="module")
def ba_case():
    """a BA graph whose in-lists exceed 512 entries, three levels, and per semiring the restated fixed point, T and tree
    at the widest k (the columns are independent: a narrower run is its first k columns)"""
    n, w, k = 30000, 1000, max(BA_KS)
    A = sr.weighted_ba_graph(n, 3, seed=7)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    ref = {}
    for semiring in bn.SEMIRINGS:
        p = bn.BottleneckProtocol(dec, w, k, semiring, add_identity=True)
        rows = p.rows[0]
        eye = sparse.csr_matrix((np.full(rows, bn.ONE[semiring], np.float32), np.arange(rows), np.arange(rows + 1)),
                                shape=(rows, rows))
        adj = spr.weighted_adjacency([(eye, None)] + pr.protocol_parts(p), rows)
        assert np.diff(adj[0]).max() > 512
        rng = np.random.default_rng(k)
        X0 = np.full((rows, k), bn.ZERO[semiring], np.float32)
        X0[rng.integers(0, rows, k), np.arange(k)] = bn.ONE[semiring]
        X0[rng.integers(0, rows, k), np.arange(k)] = 9.0
        Dr, steps, _, Tr = bn.fixed_point(adj, X0, 500, lambda e: "pull", semiring)
        assert steps < 500
        want = bn.tree(adj, Dr, Tr, semiring)
        bn.check_tree(adj, Dr, Tr, want, semiring)
        ref[semiring] = (X0, Dr, want)
    return dec, w, ref


@pytest.mark.parametrize("k", BA_KS)
def test_bottleneck_tree_ba_hubs(cuda_device, ba_case, k):
    dec, w, ref = ba_case
    for semiring in bn.SEMIRINGS:
        eng = _engine(dec, w, k, cuda_device, semiring)
        assert eng.fused_ok and eng.L == 3
        X0, Dr, want = (np.ascontiguousarray(a[:, :k]) for a in ref[semiring])
        for grid, opts in GRIDS:
            _set(eng.ctx, opts)
            eng.set_features(X0)
            D, P = eng.bottleneck_tree(500)
            tag = f"k={k} {semiring} [{grid}]"
            assert np.array_equal(_bits(D), _bits(Dr)), f"{tag}: D"
            assert np.array_equal(P, want), f"{tag}: {int(np.sum(P != want))} parents differ"
        _set(eng.ctx, [])
        assert eng._bt_in_adj is not None and eng._bt_tiles is not None
        eng.close()
        assert eng._bt_in_adj is None and eng._bt_tiles is None


def test_entry_point_refusals(ctx):
    n, k = 64, 8
    A = sparse.random(n, n, density=0.1, format="csr", random_state=1, dtype=np.float32)
    dA = ctx.csr_upload(n, n, A.indptr, A.indices, A.data)
    adj = ctx.adj_build([(dA, None)], n, weighted=True)
    lf_in = ctx.adj_build_loopfree([(dA, None)], n, direction="in")
    lf_out = ctx.adj_build_loopfree([(dA, None)], n)
    plain_in = ctx.adj_build([(dA, None)], n, direction="in")
    X, Y = ctx.dense_alloc(n, k), ctx.dense_alloc(n, k)
    T, P = ctx.dense_alloc(n, k, np.int32), ctx.dense_alloc(n, k, np.int32)
    T2 = ctx.dense_alloc(n, k - 1, np.int32)
    F = ctx.dense_alloc(n, k)
    mark = ctx.sr_mark_frontier_steps
    assert _code(lambda: mark(adj, X, Y, F, 0)) == ERR_ARG                 # steps not int32
    assert _code(lambda: mark(adj, X, Y, T2, 0)) == ERR_ARG                # steps of another k
    assert _code(lambda: mark(adj, X, Y, T, -1)) == ERR_ARG                # a negative level
    assert _code(lambda: mark(plain_in, X, Y, T, 0)) == ERR_ARG            # an in-adjacency
    mark(adj, X, Y, T, 0)
    assert np.all(T.d2h() == 0)
    tree = ctx.sr_tree_parents
    assert _code(lambda: tree(lf_out, X, T, P, _lib.SR_MAX_MIN)) == ERR_ARG          # the out-adjacency
    assert _code(lambda: tree(plain_in, X, T, P, _lib.SR_MAX_MIN)) == ERR_ARG        # not loop-free
    assert _code(lambda: tree(lf_in, X, F, P, _lib.SR_MAX_MIN)) == ERR_ARG           # steps not int32
    assert _code(lambda: tree(lf_in, X, T, F, _lib.SR_MAX_MIN)) == ERR_ARG           # parent not int32
    assert _code(lambda: tree(lf_in, X, T, T, _lib.SR_MAX_MIN)) == ERR_ARG           # parent aliases steps
    assert _code(lambda: tree(lf_in, X, T2, P, _lib.SR_MAX_MIN)) == ERR_ARG          # shape
    for code in (_lib.SR_PLUS_TIMES, _lib.SR_MIN_PLUS, _lib.SR_MAX_PLUS, _lib.SR_OR_AND):
        assert _code(lambda: tree(lf_in, X, T, P, code)) == ERR_UNSUPPORTED
    assert _code(lambda: tree(lf_in, X, T, P, 7)) == ERR_ARG
    tree(lf_in, X, T, P, _lib.SR_MIN_MAX)
    assert np.all(P.d2h() == -1)                                            # T == 0: every element a root
    # arrow_spmm_sr / gather / push accept 4 and 5; 7 stays unknown; the witness refuses the bottleneck codes
    for code in CODE.values():
        ctx.spmm_sr(dA, X, Y, None, None, code)
        assert _code(lambda: ctx.spmm_sr_witness(dA, X, P, dist=X, semiring=code)) == ERR_UNSUPPORTED
    assert _code(lambda: ctx.spmm_sr(dA, X, Y, None, None, 7)) == ERR_ARG
    ctx.sr_mark_frontier(adj, X, Y)
    for code in CODE.values():
        ctx.sr_push_frontier(adj, X, Y, code)
    d64, c64 = ctx.dense_alloc(n, k, np.float64), ctx.dense_alloc(n, k, np.float64)
    A64 = ctx.csr_upload(n, n, A.indptr, A.indices, A.data.astype(np.float64), dtype=np.float64)
    assert _code(lambda: ctx.spmm_sr(A64, d64, c64, None, None, _lib.SR_MAX_MIN)) == ERR_UNSUPPORTED
    # the bit-level row count of the bottleneck stop test: -0 against +0 counts, the same NaN does not
    a = np.zeros((n, k), np.float32)
    b = a.copy()
    b[3, 5], b[9, 0], b[20, 7] = -0.0, 1.0, -0.0
    a[30, 2] = b[30, 2] = np.nan
    da, db = ctx.dense_from_host(a), ctx.dense_from_host(b)
    assert ctx.count_diff_bits(da, db) == 3 and ctx.count_diff(da, db) == 2
    assert _code(lambda: ctx.count_diff_bits(da, T)) == ERR_ARG
    assert _code(lambda: ctx.count_diff_bits(d64, c64)) == ERR_ARG
    for h in (da, db, T2, F, P, T, Y, X, plain_in, lf_out, lf_in, adj, dA, d64, c64, A64):
        h.free()


def test_loop_stops_on_bits_not_values(cuda_device):
    """levels that only turn -0 into +0 (tests/test_bottleneck_cpu.py's six-vertex case) keep the loop going in every
    direction: the widest value of vertex 2 is +0 and its parent is 1"""
    from tests.test_bottleneck_cpu import _late_zero_case
    A, X6 = _late_zero_case()
    n, w = A.shape[0], 8
    eye = sparse.csr_matrix((np.full(w, np.inf, np.float32), np.arange(w), np.arange(w + 1)), shape=(w, w))
    Aw = sparse.csr_matrix((A.data, A.indices, np.r_[A.indptr, [A.indptr[-1]] * (w - n)]), shape=(w, w))
    adj = spr.weighted_adjacency([(eye, None), (Aw, None)], w)
    X0 = np.full((w, 1), -np.inf, np.float32)
    X0[:n] = X6
    Dr, steps_r, _, Tr = bn.fixed_point(adj, X0, 20, lambda e: "pull", "max_min")
    want = bn.tree(adj, Dr, Tr, "max_min")
    assert steps_r == 6 and want[:n, 0].tolist() == [-1, 5, 1, 0, 3, 4]
    for label, limit in DIRECTIONS.items():
        eng = _engine([(A, np.arange(n))], w, 1, cuda_device, "max_min", mode="fused", limit=limit)
        assert eng.n_rows == w and eng._sr_push_ok()
        eng.set_features(X0)
        assert eng.iterate_to_fixed_point(20) == steps_r, label
        assert np.array_equal(_bits(eng.result()), _bits(Dr)), label
        eng.set_features(X0)
        D, P = eng.bottleneck_tree(20)
        assert np.array_equal(_bits(D), _bits(Dr)) and np.array_equal(P, want), label
        eng.close()


def test_mpi_forwarding(cuda_device, tmp_path):
    from arrow_matrix_b200 import graphio
    n, w, k = 4000, 500, 8
    A = sr.weighted_ba_graph(n, 3, seed=9)
    dec = arrow_decomposition(A, w, max_number_of_levels=2, block_diagonal=True, seed=2)
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, w, True)
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, w, True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, w, k, 'gpu', True, True,
                                             semiring="max_min", add_identity=True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    eng = arrow._engine
    X0 = np.full((eng.n_rows, k), -np.inf, np.float32)
    X0[np.arange(k) * 7, np.arange(k)] = np.inf
    arrow.B.set_features(X0)
    D, P = arrow.bottleneck_tree(200)
    eng.set_features(X0)
    D2, P2 = eng.bottleneck_tree(200)
    assert np.array_equal(_bits(D), _bits(D2)) and np.array_equal(P, P2)
    assert np.all(np.isfinite(D[P >= 0]))
    eng.close()
