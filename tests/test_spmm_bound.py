"""CPU self-tests of the float64 SpMM reference and its error bound (tests/spmm_bound.py): a correct fp32 evaluation
passes, every simulated kernel fault fails.  No GPU: the faults are applied to CPU results."""
import numpy as np
import pytest
from scipy import sparse

from oracle import oracle
from tests import spmm_bound as sb
from tests import tile_dispatch as td
from tests.test_gpu_kernels import assert_close


def _hub_matrix(rng, n=5000, decades=0.0):
    lens = rng.integers(0, 12, size=n)
    lens[::97] = 0
    lens[5], lens[6], lens[4999], lens[10] = 3000, 4097, 513, 512
    return sb.ragged_csr(lens, n, rng, decades)


@pytest.fixture(scope="module")
def case():
    rng = np.random.default_rng(3)
    A = _hub_matrix(rng, decades=2.0)
    X = (rng.uniform(-1, 1, (A.shape[1], 16)) * 10.0 ** rng.uniform(-2, 2, (A.shape[1], 1))).astype(np.float32)
    return A, X


def test_tree_height_follows_the_kernels():
    assert sb.tree_height(0) == 2 and sb.tree_height(512) == 514
    # 513 entries, one segment: ceil(513 / 8) fmaf + 8 warp sums + 1 segment + addend + old
    assert sb.tree_height(513) == 65 + 8 + 1 + 2
    # 4097 entries in 2048-entry segments: 256 fmaf per warp, 3 segments
    assert sb.tree_height(4097) == 256 + 8 + 3 + 2
    assert sb.tree_height(100, threshold=8, segment=33) == 5 + 8 + 4 + 2


def test_oracle_passes(case):
    A, X = case
    C = np.full((A.shape[0], X.shape[1]), np.nan, np.float32)
    e = sb.reference(A, X, [C])
    got = oracle.csr_spmm_c(A, X)
    assert sb.assert_spmm([got], e) <= 1.0
    # accumulate, and a row map that drops rows and leaves the rest of C alone
    rng = np.random.default_rng(1)
    old = rng.standard_normal((A.shape[0] + 7, X.shape[1])).astype(np.float32)
    rm = rng.permutation(A.shape[0] + 7)[:A.shape[0]]
    rm[::13] = -1
    e = sb.reference(A, X, [old], rowmap=rm, accumulate=True)
    got = old.copy()
    ok = rm >= 0
    got[rm[ok]] = (old[rm[ok]] + oracle.csr_spmm_c(A, X)[ok]).astype(np.float32)
    sb.assert_spmm([got], e)


def _fails(got, e):
    worst, msg = sb.check_spmm([got], e)
    assert worst > 1.0, f"the simulated fault passed: {msg}"
    return msg


def _short_row(A, r):
    """the first row from r on with 3 .. 12 entries"""
    lens = np.diff(A.indptr)
    return r + int(np.flatnonzero((lens[r:] >= 3) & (lens[r:] <= 12))[0])


def _term_row(A, X, r):
    """the entry of row r with the largest contribution, and that contribution"""
    s, t = A.indptr[r], A.indptr[r + 1]
    contrib = np.abs(A.data[s:t, None].astype(np.float64) * X[A.indices[s:t]])
    p = s + int(np.argmax(contrib.max(axis=1)))
    return p, A.data[p].astype(np.float64) * X[A.indices[p]].astype(np.float64)


def test_dropped_term_fails(case):
    A, X = case
    e = sb.reference(A, X, [np.zeros((A.shape[0], X.shape[1]), np.float32)])
    got = oracle.csr_spmm_c(A, X)
    r = _short_row(A, 123)
    p, t = _term_row(A, X, r)
    got[r] = (got[r] - t).astype(np.float32)
    _fails(got, e)


def test_last_entry_of_a_tile_dropped_fails(case):
    A, X = case
    e = sb.reference(A, X, [np.zeros((A.shape[0], X.shape[1]), np.float32)])
    tiles = td.build_tiles(A.indptr, td.TILE_ROWS, td.TILE_NNZ)
    r0, r1, z0, z1 = tiles[17]
    last = z1 - 1
    r = int(np.searchsorted(A.indptr, last, side="right") - 1)
    assert r0 <= r < r1
    got = oracle.csr_spmm_c(A, X)
    got[r] = (got[r] - A.data[last].astype(np.float64) * X[A.indices[last]]).astype(np.float32)
    _fails(got, e)


def test_neighbour_value_fails(case):
    A, X = case
    e = sb.reference(A, X, [np.zeros((A.shape[0], X.shape[1]), np.float32)])
    got = oracle.csr_spmm_c(A, X)
    r = _short_row(A, 321)
    p, _ = _term_row(A, X, r)
    c = A.indices[p]
    got[r] = (got[r] + A.data[p].astype(np.float64) * (X[c + 1].astype(np.float64) - X[c])).astype(np.float32)
    _fails(got, e)


def test_swapped_rows_fail(case):
    A, X = case
    e = sb.reference(A, X, [np.zeros((A.shape[0], X.shape[1]), np.float32)])
    got = oracle.csr_spmm_c(A, X)
    got[[200, 201]] = got[[201, 200]]
    _fails(got, e)


def test_addend_from_wrong_row_fails(case):
    A, X = case
    rng = np.random.default_rng(2)
    n = A.shape[0]
    add = rng.standard_normal((n + 1, X.shape[1])).astype(np.float32)
    amap = rng.permutation(n)
    amap[::3] = -1
    C = np.full((n, X.shape[1]), np.nan, np.float32)
    e = sb.reference(A, X, [C], add=add, add_map=amap)
    prod = oracle.csr_spmm_c(A, X)
    ok = amap >= 0
    got = prod.copy()
    got[ok] = (prod[ok] + add[amap[ok]].astype(np.float64)).astype(np.float32)
    sb.assert_spmm([got], e)
    r = int(np.flatnonzero(ok)[5])
    got[r] = (prod[r] + add[amap[r] + 1].astype(np.float64)).astype(np.float32)
    _fails(got, e)


def test_unwritten_row_and_stray_nan_fail(case):
    A, X = case
    n = A.shape[0]
    rm = np.arange(n)
    rm[40] = -1
    C = np.full((n, X.shape[1]), np.nan, np.float32)
    e = sb.reference(A, X, [C], rowmap=rm)
    got = oracle.csr_spmm_c(A, X)
    got[40] = np.nan
    sb.assert_spmm([got], e)
    bad = got.copy()
    bad[40] = 0.0                               # a dropped row was written
    assert "outside the write set" in _fails(bad, e)
    bad = got.copy()
    bad[41, 3] = np.nan                         # a stray read of a canary
    _fails(bad, e)
    empty = int(np.flatnonzero(np.diff(A.indptr) == 0)[1])
    bad = got.copy()
    bad[empty, 0] = 1e-30                       # a row without terms must be exactly zero
    _fails(bad, e)


def test_scaled_short_row_next_to_hub_fails_where_assert_close_passes():
    """the old whole-tile tolerance lets a 1e-4 relative error through in a short row once a hub row sets the scale"""
    rng = np.random.default_rng(3)
    A = _hub_matrix(rng)
    X = rng.uniform(-1, 1, (A.shape[1], 16)).astype(np.float32)
    ref = oracle.csr_spmm_c(A, X)
    e = sb.reference(A, X, [np.zeros_like(ref)])
    sb.assert_spmm([ref], e)
    r = 7                                       # right after the 4097-entry row 6
    assert 2 <= A.indptr[r + 1] - A.indptr[r] <= 12
    got = ref.copy()
    got[r] = (got[r].astype(np.float64) * (1 + 1e-4)).astype(np.float32)
    assert_close(got, ref)                      # accepted by the scale-of-the-tile check
    assert_close(got, (A.astype(np.float64) @ X.astype(np.float64)).astype(np.float32))
    _fails(got, e)                              # rejected per element


def test_pointer_table_and_remapped_columns(case):
    A, X = case
    rng = np.random.default_rng(4)
    n, k = A.shape[0], X.shape[1]
    col_map = rng.permutation(A.shape[1] + 50)[:A.shape[1]]
    col_map[::11] = -1                          # skipped entries
    split = 1200
    Xn = np.full((A.shape[1] + 50, k), np.nan, np.float32)
    used = np.unique(col_map[A.indices][col_map[A.indices] >= 0])
    Xn[used] = rng.standard_normal((used.size, k))
    which = rng.integers(-1, 2, n)
    row = np.zeros(n, np.int64)
    for t in (0, 1):
        sel = np.flatnonzero(which == t)
        row[sel] = rng.permutation(n)[:sel.size]
    tiles = [np.full((n, k), np.nan, np.float32) for _ in range(2)]
    e = sb.reference(A, Xn[:split], tiles, X2=Xn[split:], x_split=split, col_map=col_map, table=(which, row))
    # a correct fp32 evaluation: the remapped block times the operand, routed through the table
    cm = col_map[A.indices]
    keep = cm >= 0
    rows_of = np.repeat(np.arange(n), np.diff(A.indptr))
    B = sparse.csr_matrix((A.data[keep], (rows_of[keep], cm[keep])), shape=(n, Xn.shape[0]))
    prod = oracle.csr_spmm_c(B, np.nan_to_num(Xn))
    got = [t.copy() for t in tiles]
    for t in (0, 1):
        sel = np.flatnonzero(which == t)
        got[t][row[sel]] = prod[sel]
    sb.assert_spmm(got, e)
    sel = np.flatnonzero((which == 1) & (np.diff(A.indptr) > 0))
    got[1][row[sel[0]]] = prod[sel[1]]          # a row delivered to the wrong slot
    assert sb.check_spmm(got, e)[0] > 1.0
