"""The per-element step bound of tests/step_bound.py, checked on the host.

* no false alarms: correct float32 evaluations of a step in other summation orders (SciPy, the C restatement of
  csr_matvecs, the reference's block algebra, entries in reverse order) meet the bound, on the golden decompositions and
  on synthetic ones with hub rows above the long-row threshold;
* planted faults: each of them fails the bound and passes the normwise rule of ``assert_close`` / ``close_rows``
  (``1e-5 * max|C|``) -- the gap the bound closes;
* the rank-1 closed form the benchmark-scale test uses agrees with the longdouble oracle.
"""
import numpy as np
import pytest

from arrow_matrix_b200 import synth
from oracle import oracle
from tests import step_bound as stb
from tests.golden_util import CASES, GoldenCase
from tests.spmm_bound import tree_height
from tests.test_gpu_kernels import assert_close
from tests.test_gpu_ranks_one_gpu import close_rows

HOWS = ["scipy", "c_kernel", "blockwise", "reversed"]


def _reversed_mm(A, X):
    """``A @ X`` in float32 with every row's entries summed last to first (rounded product, then rounded add)"""
    A = A.tocsr()
    X = np.asarray(X, dtype=np.float32)
    out = np.zeros((A.shape[0], X.shape[1]), dtype=np.float32)
    nnz = np.diff(A.indptr)
    data = A.data.astype(np.float32)
    for t in range(int(nnz.max(initial=0))):
        rows = np.flatnonzero(nnz > t)
        p = A.indptr[rows + 1] - 1 - t
        out[rows] = out[rows] + data[p][:, None] * X[A.indices[p]]
    return out


def _fp32_oracle(dec, w, k, block_diagonal, n_blocks, how):
    po = oracle.ReferenceProtocolOracle(dec, w, k, block_diagonal=block_diagonal, n_blocks=n_blocks,
                                        use_c_kernel=how == "c_kernel", blockwise=how == "blockwise")
    if how == "reversed":
        po._mm = _reversed_mm
    return po


def _chained(dec, w, k, block_diagonal, n_blocks, X0, how, steps=3):
    """``steps`` chained float32 steps; yields (got, exact, mag, M) with exact / mag from the evaluation's own state"""
    ex = stb.ExactStep(dec, w, k, block_diagonal, n_blocks)
    po = _fp32_oracle(dec, w, k, block_diagonal, n_blocks, how)
    x = X0.astype(np.float32)
    carried = [np.zeros_like(c) for c in po.C[1:]]
    for _ in range(steps):
        exact, mag = ex.run(x, carried)
        po.set_features(x.copy())
        for j in range(1, po.L):
            po.C[j] = carried[j - 1].copy()
        got = po.step().copy()
        yield got, exact, mag, ex.M
        x, carried = got, [c.copy() for c in po.C[1:]]


def _synthetic(name, perm_kind="random"):
    w, t0, k, levels, hub = {"hub600_L3k8": (64, 12, 8, 3, 600), "hub2100_L2k5": (64, 40, 5, 2, 2100),
                             "hub700_L4k3": (32, 24, 3, 4, 700)}[name]
    dec = synth.synth_decomposition(t0, w, levels=levels, perm_kind=perm_kind, seed=17, hub_rows=2, hub_nnz=hub)
    return dec, w, k, True, None


SYNTHETIC = ["hub600_L3k8", "hub2100_L2k5", "hub700_L4k3"]


@pytest.mark.parametrize("how", HOWS)
@pytest.mark.parametrize("name", CASES + SYNTHETIC)
def test_correct_fp32_orders_meet_the_bound(name, how):
    if name in SYNTHETIC:
        dec, w, k, bd, nb = _synthetic(name)
    else:
        g = GoldenCase(name)
        dec, w, k, bd, nb = g.decomposition, g.width, g.k, g.block_diagonal, g.n_blocks
    rng = np.random.default_rng(5)
    probe = oracle.ReferenceProtocolOracle(dec, w, k, block_diagonal=bd, n_blocks=nb)
    n = probe.rows[0]
    hubs = np.flatnonzero(np.diff(probe.mats[0].indptr) > stb.LONG_THRESHOLD)
    if name in SYNTHETIC:
        assert hubs.size > 0, "the long-row height must be exercised"
    X0, scale = stb.spread_features(n, k, w, rng, large_rows=hubs)
    worst = 0.0
    for it, (got, exact, mag, M) in enumerate(_chained(dec, w, k, bd, nb, X0, how)):
        worst = max(worst, stb.assert_step(got, exact, mag, M, route=f"{name} {how} step {it}", row_scale=scale))
    assert worst > 0.0


def test_matrix_row_scales_and_subnormal_band_meet_the_bound():
    dec, w, k, bd, nb = _synthetic("hub600_L3k8")
    rng = np.random.default_rng(8)
    dec = stb.rescale_rows(dec, rng)
    n = 12 * w
    band = np.concatenate([np.arange(2, w), np.arange(5 * w, 6 * w)])      # the head (hubs excluded) and block-row 5
    X0, scale = stb.spread_features(n, k, w, rng, large_rows=[0, 1], subnormal_rows=band)
    assert np.any((X0 != 0) & (np.abs(X0) < 2.0 ** -126))
    for how in ("scipy", "reversed"):
        for it, (got, exact, mag, M) in enumerate(_chained(dec, w, k, bd, nb, X0, how)):
            stb.assert_step(got, exact, mag, M, route=f"subnormal band {how} step {it}", row_scale=scale)


def test_tree_height_upto_is_the_prefix_maximum():
    n = np.arange(0, 5000)
    want = np.maximum.accumulate(tree_height(n))
    assert np.array_equal(stb.tree_height_upto(n), want)


def test_chain_heights_follow_the_level_maps():
    """the height of a level-0 row adds ``T + 1`` of every level whose row aggregates into it, nothing for the others"""
    dec, w, k, bd, nb = _synthetic("hub600_L3k8")
    po = oracle.ReferenceProtocolOracle(dec, w, k)
    M = stb.oracle_heights(po)
    maps = stb.chain_maps(po.to_prev, po.rows)
    want = tree_height(np.diff(po.mats[0].indptr)) + 1
    for j in range(1, po.L):
        h = tree_height(np.diff(po.mats[j].indptr)) + 1
        for s in range(po.rows[j]):
            if maps[j][s] >= 0:
                want[maps[j][s]] += h[s]
    assert np.array_equal(M, want)
    assert M[0] >= tree_height(600) + 1
    # the sharded rule: head rows pay the reduction of `world` partials, with the prefix-maximum height
    M4 = stb.chain_heights([np.diff(m.indptr) for m in po.mats], po.to_prev, w, world=4)
    assert np.all(M4 >= M) and M4[0] > M[0] and M4[w + 5] >= M[w + 5]


# ---- planted faults ---------------------------------------------------------------------------------------------------
class _Planted:
    """one correct float32 step on spread features, its exact value and the rows a fault is planted in.  Identity level
    permutations keep every level's chain row in its block-row, so a small block-row is small at every level."""

    def __init__(self, subnormal=False):
        dec, w, k, bd, nb = _synthetic("hub600_L3k8", perm_kind="identity")
        rng = np.random.default_rng(23)
        n = 12 * w
        band = np.concatenate([np.arange(2, w), np.arange(5 * w, 6 * w)]) if subnormal else None
        X0, self.scale = stb.spread_features(n, k, w, rng, large_rows=[0, 1], subnormal_rows=band)
        ex = stb.ExactStep(dec, w, k, bd, nb)
        self.exact, self.mag = ex.run(X0)
        self.M = ex.M
        po = oracle.ReferenceProtocolOracle(dec, w, k)
        po.set_features(X0.copy())
        self.got = po.step().copy()
        self.C1 = po.C[1]                                   # level 1 after the step: what it adds to level 0
        self.maps = stb.chain_maps(po.to_prev, po.rows)
        self.row_mag = self.mag.max(axis=1)
        assert stb.check(self.got, self.exact, self.mag, self.M)[0] <= 1.0

    def small_rows(self):
        """level-0 rows in increasing order of magnitude"""
        return np.argsort(self.row_mag)

    def assert_caught(self, bad, what):
        worst, msg = stb.check(bad, self.exact, self.mag, self.M, route=what, row_scale=self.scale)
        assert worst > 1.0, f"{what} was not caught: {msg}"
        # ... while the normwise rule of assert_close / close_rows lets it through
        exact64 = self.exact.astype(np.float64)
        assert_close(bad, self.got, exact=exact64)
        close_rows(bad, self.got, exact64, 0, bad.shape[0])
        return msg


@pytest.fixture(scope="module")
def planted():
    return _Planted()


def test_planted_row_swap(planted):
    order = planted.small_rows()
    tiny = planted.row_mag < 1e-7 * planted.row_mag.max()
    r = next(int(q) for q in order if q + 1 < tiny.size and tiny[q] and tiny[q + 1]
             and not np.array_equal(planted.got[q], planted.got[q + 1]))
    bad = planted.got.copy()
    bad[[r, r + 1]] = bad[[r + 1, r]]
    planted.assert_caught(bad, f"rows {r} and {r + 1} swapped")


def _row_with_level1(p):
    inv = np.full(p.got.shape[0], -1)
    ok = p.maps[1] >= 0
    inv[p.maps[1][ok]] = np.flatnonzero(ok)
    for q in p.small_rows():
        s = inv[q]
        if s >= 0 and p.row_mag[q] < 1e-7 * p.row_mag.max() and np.abs(p.C1[s]).max() > 1e-3 * p.row_mag[q]:
            return int(q), int(s)
    raise AssertionError("no small row with a level-1 contribution")


def test_planted_dropped_level_contribution(planted):
    r, s = _row_with_level1(planted)
    bad = planted.got.copy()
    bad[r] = bad[r] - planted.C1[s]
    planted.assert_caught(bad, f"level-1 row {s} dropped from row {r}")


def test_planted_doubled_level_contribution(planted):
    r, s = _row_with_level1(planted)
    bad = planted.got.copy()
    bad[r] = bad[r] + planted.C1[s]
    planted.assert_caught(bad, f"level-1 row {s} added twice to row {r}")


def test_planted_subnormals_flushed_to_zero():
    p = _Planted(subnormal=True)
    sub = (p.got != 0) & (np.abs(p.got) < 2.0 ** -126)
    assert sub.any()
    bad = np.where(sub, np.float32(0.0), p.got)
    p.assert_caught(bad, "float32 subnormal results flushed to zero")


def _bf16(x):
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000                        # round to nearest even on the top 16 bits
    return b.astype(np.uint32).view(np.float32)


def test_planted_bf16_row(planted):
    r = int(planted.small_rows()[0])
    bad = planted.got.copy()
    bad[r] = _bf16(bad[r])
    assert not np.array_equal(bad[r], planted.got[r])
    planted.assert_caught(bad, f"row {r} rounded to bfloat16")


def test_planted_column_swap(planted):
    r = int(planted.small_rows()[0])
    bad = planted.got.copy()
    bad[r, [0, 1]] = bad[r, [1, 0]]
    planted.assert_caught(bad, f"columns 0 and 1 swapped in row {r}")


# ---- the rank-1 form --------------------------------------------------------------------------------------------------
def test_rank1_form_agrees_with_the_oracle():
    dec, w, k, bd, nb = _synthetic("hub600_L3k8")
    n = 12 * w
    u, v = stb.rank1_vectors(n, k, w, np.random.default_rng(503), large_rows=[0, 1])
    R = stb.Rank1Step.build(dec, w, u, v)
    X = stb.rank1_features(u, v, 0, n)
    ex = stb.ExactStep(dec, w, k)
    exact, mag = ex.run(X)
    assert np.array_equal(R.M, ex.M[:, 0])
    want, _, mag1 = R.expect(0, n)
    # the closed form differs from the step of the rounded features by the input rounding pushed through |S|
    slack = (2.0 ** -24 + 4.0 * stb.gamma(R.M[:, None] + 1, stb.U64)) * mag1
    assert np.all(np.abs(want - exact.astype(np.float64)) <= slack)
    assert np.all(mag <= mag1 * (1.0 + 2.0 ** -23))
    # a correct float32 step passes, in one chunk or many; a swap of two small rows does not
    po = oracle.ReferenceProtocolOracle(dec, w, k)
    po.set_features(X.copy())
    got = po.step().copy()
    worst, msg = R.check(got, route="rank-1 scipy")
    assert 0.0 < worst <= 1.0, msg
    assert R.check(got, chunk=100)[0] == worst
    assert R.check(got[200:], r0=200)[0] <= worst
    r, r2 = (int(q) for q in np.argsort(np.abs(R.ya))[:2])
    assert abs(R.ya[r2]) < 1e-7 * np.abs(R.ya).max()
    bad = got.copy()
    bad[[r, r2]] = bad[[r2, r]]
    assert R.check(bad, route="swap")[0] > 1.0
    assert_close(bad, got)
