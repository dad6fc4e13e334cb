"""Float64 reference of every SpMM mode of the C ABI with a rigorous per-element fp32 error bound (test infrastructure).

``reference(...)`` evaluates ``arrow_spmm`` / ``arrow_spmm_add`` / ``arrow_spmm_ex`` exactly (float64 on the fp32
inputs) and returns, for every destination tile, the exact result, a bound on the error of ANY correct fp32
evaluation the kernels may use, and the rows the call may write.  ``assert_spmm`` checks a device result against it.

The bound
---------
Every output element is a sum of terms ``t_p = A[r, c_p] * X[c_p, j]`` plus, depending on the epilogue, the old
``C`` element and an addend element.  With unit roundoff ``u = 2^-24``, an evaluation in which every term passes
through at most ``m`` rounded operations (an FMA rounds once: its product is exact) satisfies

    |got - exact| <= gamma_m * (sum_p |t_p| + |C_old| + |add|),    gamma_m = m u / (1 - m u)

(Higham, *Accuracy and Stability of Numerical Algorithms*, 2nd ed., Lemma 3.1 and section 4.2: a summation tree of
height ``m``), plus ``m * 2^-150`` for gradual underflow.  ``m`` is the height of the deepest summation tree the
kernels in ``arrow_matrix_b200/csrc/arrow_b200.cu`` use for a row with ``n`` stored entries:

* ``k_spmm_tiles_v1`` / ``k_spmm_tiles``: ``acc = C_old`` (accumulate), ``acc += add`` (one f4_add), then one
  ``fmaf`` per entry in ascending order (``f4_fma`` in the batches and the predicated tail) -> ``n + 1``.
  Skipped entries (column -1) and padding lanes add ``fmaf(v, 0, acc) == acc``: no rounding.
* ``k_spmm_direct`` / ``k_spmm_shfl`` / ``k_spmm_tma``: ``n`` fmaf from zero, then ``acc + old`` -> ``n + 1``.
* ``k_spmm_generic<PlusTimes<float>>``: ``n`` fmaf from zero, ``*dst + acc`` (accumulate), ``r += add`` -> ``n + 2``.
* long rows (``n > threshold``), ``k_spmm_long_partial<PlusTimes<float>>``: a segment of at most
  ``s = min(segment, n)`` entries is split over 8 warps (256 threads), warp ``w`` chains the entries
  ``begin + w, begin + w + 8, ...`` -> at most ``ceil(s / 8)`` fmaf; the 8 warp partials are added in order from 0 ->
  7 more roundings (the first add is exact, count 8); ``k_spmm_long_reduce<PlusTimes<float>>`` adds the
  ``ceil(n / segment)`` segment partials in order from 0, then the addend, then ``*dst + sum`` ->
  ``ceil(s / 8) + 8 + ceil(n / segment) + 2``.

A row gets the largest ``m`` of the kernels that may evaluate it: ``n + 2`` for a row at or below the long-row
threshold, the long-row height above it.  The float64 reference itself is off by at most
``gamma_{n+2}(2^-53)`` of the same magnitude, which is added to the bound.  No constant in the bound is tuned.

Rows with no valid term are exact (0, the old row or the addend).  Rows outside the write set must be bit-identical to
what the destination held before the call.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np
from scipy import sparse

U32 = 2.0 ** -24
U64 = 2.0 ** -53
ETA32 = 2.0 ** -150          # half the smallest fp32 subnormal: the absolute error of a rounding in the subnormal range
WARPS_PER_LONG_CTA = 8       # k_spmm_long_partial<SR> runs 256 threads


def gamma(m, u=U32):
    m = np.asarray(m, dtype=np.float64)
    return m * u / (1.0 - m * u)


def tree_height(n, threshold: int = 512, segment: int = 2048):
    """``m`` of the module docstring for rows with ``n`` stored entries."""
    n = np.asarray(n, dtype=np.int64)
    s = np.minimum(n, segment)
    long_h = -(-s // WARPS_PER_LONG_CTA) + 8 + (-(-n // segment)) + 2
    return np.where(n > threshold, long_h, n + 2)


@dataclass
class Expect:
    """What one call must produce in each destination tile."""
    exact: List[np.ndarray]                 # float64 [rows, k] per tile
    bound: List[np.ndarray]                 # float64 [rows, k] per tile (0 = must be exact)
    written: List[np.ndarray]               # bool [rows] per tile
    before: List[np.ndarray]                # float32 tiles as they were before the call
    src_row: List[np.ndarray]               # int64 [rows] per tile: the block row written there (-1: none)
    row_nnz: np.ndarray                     # stored entries per block row
    label: str = ""
    notes: dict = field(default_factory=dict)


def reference(A: sparse.csr_matrix, X: np.ndarray, C_before: Sequence[np.ndarray], *, X2: Optional[np.ndarray] = None,
              x_split: int = 0, col_map: Optional[np.ndarray] = None, rowmap: Optional[np.ndarray] = None,
              accumulate: bool = False, add: Optional[np.ndarray] = None, add_map: Optional[np.ndarray] = None,
              table: Optional[Tuple[np.ndarray, np.ndarray]] = None, threshold: int = 512, segment: int = 2048,
              label: str = "") -> Expect:
    """Exact result, bound and write set of one SpMM call.

    ``A``: the block as uploaded (original columns).  ``col_map``: the column remap (``arrow_csr_remap_columns``) with
    -1 for an invalid image.  ``X`` / ``X2`` / ``x_split``: the operand (columns >= x_split read ``X2[c - x_split]``
    when ``X2`` is given).  ``rowmap`` (-1 = dropped) or ``table = (which, row)`` (which -1 = dropped) route the result
    rows; otherwise row r goes to row r of ``C_before[0]``.  ``add`` / ``add_map`` (-1 = none): the gather-add.
    ``C_before``: the destination tile(s) before the call (may hold NaN canaries)."""
    A = sparse.csr_matrix(A)
    n_rows = A.shape[0]
    indptr = A.indptr.astype(np.int64)
    row_nnz = np.diff(indptr)
    rows_of = np.repeat(np.arange(n_rows), row_nnz)
    cols = A.indices.astype(np.int64)
    if col_map is not None:
        cols = np.asarray(col_map, dtype=np.int64)[cols]
    valid = cols >= 0
    if X2 is not None:
        operand = np.concatenate([np.asarray(X[:x_split]), np.asarray(X2)])
    else:
        operand = np.asarray(X)
    n_op = operand.shape[0]
    assert not valid.any() or cols[valid].max() < n_op, "a valid column lies outside the operand"
    vals = A.data.astype(np.float64)
    S = sparse.csr_matrix((vals[valid], (rows_of[valid], cols[valid])), shape=(n_rows, n_op))
    Sabs = sparse.csr_matrix((np.abs(vals[valid]), (rows_of[valid], cols[valid])), shape=(n_rows, n_op))
    referenced = np.unique(cols[valid])
    op64 = np.zeros(operand.shape, dtype=np.float64)
    op64[referenced] = operand[referenced]
    assert np.isfinite(op64).all(), "the test put a NaN canary into a referenced operand row"
    prod = np.asarray(S @ op64)
    mag = np.asarray(Sabs @ np.abs(op64))
    n_terms = np.bincount(rows_of[valid], minlength=n_rows)
    has_add = np.zeros(n_rows, dtype=bool)
    if add_map is not None:
        am = np.asarray(add_map, dtype=np.int64)[:n_rows]
        has_add = am >= 0
        addv = np.asarray(add, dtype=np.float64)[am[has_add]]
        assert np.isfinite(addv).all(), "the test put a NaN canary into a referenced addend row"
        prod[has_add] += addv
        mag[has_add] += np.abs(addv)

    tiles = [np.asarray(c, dtype=np.float32) for c in C_before]
    if table is not None:
        which, trow = (np.asarray(t, dtype=np.int64)[:n_rows] for t in table)
        assert not accumulate and rowmap is None
        dest_t, dest_r = which, np.where(which >= 0, trow, -1)
    else:
        dest_t = np.zeros(n_rows, dtype=np.int64)
        dest_r = np.arange(n_rows) if rowmap is None else np.asarray(rowmap, dtype=np.int64)[:n_rows]
        dest_t = np.where(dest_r >= 0, 0, -1)
    m = tree_height(row_nnz, threshold, segment)
    exact, bound, written, src = [], [], [], []
    for t, before in enumerate(tiles):
        sel = np.flatnonzero(dest_t == t)
        q = dest_r[sel]
        assert np.unique(q).size == q.size, "destination rows must be injective"
        ex = np.asarray(before, dtype=np.float64).copy()
        bd = np.zeros(before.shape, dtype=np.float64)
        w = np.zeros(before.shape[0], dtype=bool)
        sr = np.full(before.shape[0], -1, dtype=np.int64)
        w[q] = True
        sr[q] = sel
        if accumulate:
            old = np.asarray(before[q], dtype=np.float64)
            assert np.isfinite(old).all(), "accumulating into a NaN canary"
            assert not has_add[sel].any(), "accumulate and gather-add do not meet in one call"
            ex[q] = old + prod[sel]
            mg = mag[sel] + np.abs(old)
        else:
            ex[q] = prod[sel]
            mg = mag[sel]
        mm = m[sel][:, None]
        bd[q] = (gamma(mm) + gamma(row_nnz[sel][:, None] + 2, U64)) * mg + mm * ETA32
        bd[q[n_terms[sel] == 0]] = 0.0                  # no term: the old row, the addend or zero, exactly
        exact.append(ex)
        bound.append(bd)
        written.append(w)
        src.append(sr)
    return Expect(exact, bound, written, tiles, src, row_nnz, label)


def ragged_csr(lens: Sequence[int], n_cols: int, rng: np.random.Generator, decades: float = 0.0,
               col_pool: Optional[np.ndarray] = None) -> sparse.csr_matrix:
    """fp32 block with the given row lengths: sorted distinct columns drawn from ``col_pool`` (default: all), values
    +-U(0.5, 1.5) times 10^U(-decades, decades) per row and per column (spread over 10^+-2*decades)."""
    lens = np.asarray(lens, dtype=np.int64)
    pool = np.arange(n_cols) if col_pool is None else np.asarray(col_pool)
    indptr = np.concatenate([[0], np.cumsum(lens)])
    cols = np.concatenate([np.sort(pool[rng.choice(pool.size, size=int(l), replace=False)]) for l in lens]
                          + [np.zeros(0, np.int64)]).astype(np.int32)
    vals = rng.uniform(0.5, 1.5, cols.size) * rng.choice([-1.0, 1.0], cols.size)
    if decades:
        rs = 10.0 ** rng.uniform(-decades, decades, lens.size)
        cs = 10.0 ** rng.uniform(-decades, decades, n_cols)
        vals = vals * np.repeat(rs, lens) * cs[cols]
    return sparse.csr_matrix((vals.astype(np.float32), cols, indptr), shape=(lens.size, n_cols))


def check_spmm(got_tiles: Sequence[np.ndarray], e: Expect):
    """(worst ratio to the bound, message describing the worst element); ratio inf = a NaN, a changed unwritten row
    or an inexact no-term row."""
    worst, msg = 0.0, "ok"
    for t, (got, ex, bd, w, before, sr) in enumerate(zip(got_tiles, e.exact, e.bound, e.written, e.before, e.src_row)):
        got = np.asarray(got, dtype=np.float32)
        assert got.shape == before.shape, f"tile {t}: shape {got.shape} != {before.shape}"
        untouched = ~w
        if untouched.any():
            diff = np.flatnonzero((got[untouched].view(np.uint32) != before[untouched].view(np.uint32)).any(axis=1))
            if diff.size:
                q = np.flatnonzero(untouched)[diff[0]]
                return float("inf"), (f"{e.label} tile {t}: row {q} is outside the write set but changed "
                                      f"({diff.size} such rows): got {got[q][:4]} before {before[q][:4]}")
        if not w.any():
            continue
        g = got[w].astype(np.float64)
        err = np.abs(g - ex[w])
        b = bd[w]
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err == 0, 0.0, np.inf))
        ratio = np.where(np.isnan(g), np.inf, ratio)
        i = int(np.argmax(ratio))
        r = float(ratio.flat[i])
        if r > worst:
            qi, j = divmod(i, got.shape[1])
            q = np.flatnonzero(w)[qi]
            s = int(sr[q])
            worst = r
            msg = (f"{e.label} tile {t} row {q} col {j} (block row {s}, nnz {int(e.row_nnz[s])}): got {got[q, j]!r} "
                   f"exact {ex[q, j]!r} |err| {err.flat[i]:.3e} bound {bd[q, j]:.3e} ratio {r:.3g}")
    return worst, msg


def assert_spmm(got_tiles: Sequence[np.ndarray], e: Expect) -> float:
    """Every written element within its bound (exact where there is no term), every other row bit-identical to
    before; returns the worst ratio |err| / bound."""
    worst, msg = check_spmm(got_tiles, e)
    assert worst <= 1.0, msg
    return worst
