"""Exact (``np.longdouble``) reference of the float64 SpMM modes with a rigorous per-element fp64 error bound.

The float64 sibling of ``tests/spmm_bound.py`` (whose fp32 rules stay as they are).  ``reference(...)`` evaluates an
``arrow_spmm`` / ``arrow_spmm_add`` call on float64 operands in extended precision and returns the exact result, the
bound and the rows the call may write (``products`` evaluates the product once for every epilogue of one operand);
``assert_spmm64`` checks a device result against it.

The bound
---------
Every output element is a sum of terms ``t_p = A[r, c_p] * X[c_p, j]`` plus the old ``C`` element (accumulate) or an
addend element (gather-add).  With unit roundoff ``u = 2^-53``, an evaluation in which every term passes through at
most ``m`` rounded operations (an FMA rounds once) satisfies

    |got - exact| <= gamma_m * (sum_p |t_p| + |C_old| + |add|) + m * 2^-1075,    gamma_m = m u / (1 - m u)

(Higham, *Accuracy and Stability of Numerical Algorithms*, 2nd ed., Lemma 3.1 and section 4.2; ``2^-1075`` is half the
smallest subnormal).  ``m`` for a row with ``n`` stored entries, from the float64 kernels of
``arrow_matrix_b200/csrc/arrow_b200.cu``:

* ``k_spmm_tiles_f64``: ``acc`` starts at zero, or at the addend (one exact add to zero), then one ``fma`` per entry
  in ascending order, then ``acc + C_old`` in accumulate mode -> ``n + 1``.  Skipped entries (column -1), predicated
  tail slots and padding lanes add ``fma(v, 0, acc) == acc``: no rounding.
* ``k_spmm_generic<PlusTimes<double>>``: ``n`` fma from zero, ``*dst + acc`` (accumulate), ``r += add`` -> ``n + 2``.
* long rows (``n > threshold``), ``k_spmm_long_partial`` / ``k_spmm_long_reduce`` on ``PlusTimes<double>``: the fp32
  structure -> ``ceil(s / 8) + 8 + ceil(n / segment) + 2`` with ``s = min(segment, n)``.

That is ``spmm_bound.tree_height``: a row gets ``n + 2`` at or below the threshold, the long-row height above it.  The
extended-precision reference (``u = 2^-64`` on x86-64) is off by at most ``gamma_{n+2}(2^-64)`` of the same magnitude,
which is added to the bound.  No constant is tuned.  Rows with no valid term are exact; rows outside the write set must
be bit-identical to what the destination held before the call.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
from scipy import sparse

from tests.spmm_bound import gamma, tree_height

U64 = 2.0 ** -53
ULD = float(np.finfo(np.longdouble).eps) / 2        # unit roundoff of the reference arithmetic
ETA64 = 2.0 ** -1075


@dataclass
class Expect64:
    exact: np.ndarray           # longdouble [rows, k]
    bound: np.ndarray           # float64 [rows, k] (0 = must be exact)
    written: np.ndarray         # bool [rows]
    before: np.ndarray          # float64 tile before the call
    row_nnz: np.ndarray
    label: str = ""


def _ld_spmm(rows_of, cols, vals, n_rows, operand, chunk=32):
    """sum_p vals[p] * operand[cols[p]] per row in np.longdouble (scipy has no longdouble SpMM); rows_of is sorted"""
    out = np.zeros((n_rows, operand.shape[1]), dtype=np.longdouble)
    if rows_of.size == 0:
        return out
    starts = np.flatnonzero(np.r_[True, rows_of[1:] != rows_of[:-1]])
    for j0 in range(0, operand.shape[1], chunk):
        terms = vals[:, None] * operand[cols, j0:j0 + chunk]
        out[rows_of[starts], j0:j0 + chunk] = np.add.reduceat(terms, starts, axis=0)
    return out


@dataclass
class Products:
    """the exact product of one (block, operand, column map) and its magnitude, shared by every epilogue"""
    prod: np.ndarray            # longdouble [rows, k]
    mag: np.ndarray             # longdouble [rows, k]: sum_p |A| |X|
    n_terms: np.ndarray         # valid terms per row
    row_nnz: np.ndarray         # stored entries per row


def products(A: sparse.csr_matrix, X: np.ndarray, col_map: Optional[np.ndarray] = None) -> Products:
    A = sparse.csr_matrix(A)
    n_rows = A.shape[0]
    row_nnz = np.diff(A.indptr.astype(np.int64))
    rows_of = np.repeat(np.arange(n_rows), row_nnz)
    cols = A.indices.astype(np.int64)
    if col_map is not None:
        cols = np.asarray(col_map, dtype=np.int64)[cols]
    valid = cols >= 0
    vals = A.data.astype(np.longdouble)[valid]
    r, c = rows_of[valid], cols[valid]
    op = np.asarray(X, dtype=np.longdouble)
    assert np.isfinite(op[np.unique(c)]).all(), "the test put a NaN canary into a referenced operand row"
    return Products(_ld_spmm(r, c, vals, n_rows, op), _ld_spmm(r, c, np.abs(vals), n_rows, np.abs(op)),
                    np.bincount(r, minlength=n_rows), row_nnz)


def reference(P: Products, C_before: np.ndarray, *, rowmap: Optional[np.ndarray] = None, accumulate: bool = False,
              add: Optional[np.ndarray] = None, add_map: Optional[np.ndarray] = None, threshold: int = 512,
              segment: int = 2048, label: str = "") -> Expect64:
    """Exact result, bound and write set of one float64 call on the products ``P`` (``rowmap`` -1 = dropped,
    ``add_map`` -1 = no addend; see ``spmm_bound.reference``)."""
    n_rows = P.prod.shape[0]
    prod, mag = P.prod.copy(), P.mag.copy()
    has_add = np.zeros(n_rows, dtype=bool)
    if add_map is not None:
        am = np.asarray(add_map, dtype=np.int64)[:n_rows]
        has_add = am >= 0
        addv = np.asarray(add, dtype=np.longdouble)[am[has_add]]
        assert np.isfinite(addv).all(), "the test put a NaN canary into a referenced addend row"
        prod[has_add] += addv
        mag[has_add] += np.abs(addv)
    before = np.asarray(C_before, dtype=np.float64)
    dest = np.arange(n_rows) if rowmap is None else np.asarray(rowmap, dtype=np.int64)[:n_rows]
    sel = np.flatnonzero(dest >= 0)
    q = dest[sel]
    assert np.unique(q).size == q.size, "destination rows must be injective"
    ex = before.astype(np.longdouble)
    bd = np.zeros(before.shape, dtype=np.float64)
    w = np.zeros(before.shape[0], dtype=bool)
    w[q] = True
    if accumulate:
        old = before[q].astype(np.longdouble)
        assert np.isfinite(old).all(), "accumulating into a NaN canary"
        assert not has_add[sel].any(), "accumulate and gather-add do not meet in one call"
        ex[q] = old + prod[sel]
        mg = mag[sel] + np.abs(old)
    else:
        ex[q] = prod[sel]
        mg = mag[sel]
    m = tree_height(P.row_nnz, threshold, segment)[sel][:, None]
    bd[q] = ((gamma(m, U64) + gamma(P.row_nnz[sel][:, None] + 2, ULD)) * mg.astype(np.float64)) + m * ETA64
    bd[q[P.n_terms[sel] == 0]] = 0.0                     # no term: the old row, the addend or zero, exactly
    return Expect64(ex, bd, w, before, P.row_nnz, label)


def check_spmm64(got: np.ndarray, e: Expect64):
    """(worst ratio |err| / bound, message); inf = a NaN, a changed unwritten row or an inexact no-term row"""
    got = np.asarray(got)
    assert got.dtype == np.float64 and got.shape == e.before.shape
    untouched = ~e.written
    if untouched.any():
        diff = np.flatnonzero((got[untouched].view(np.uint64) != e.before[untouched].view(np.uint64)).any(axis=1))
        if diff.size:
            q = np.flatnonzero(untouched)[diff[0]]
            return float("inf"), f"{e.label}: row {q} is outside the write set but changed ({diff.size} such rows)"
    if not e.written.any():
        return 0.0, "ok"
    g = got[e.written].astype(np.longdouble)
    err = np.abs(g - e.exact[e.written]).astype(np.float64)
    b = e.bound[e.written]
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err == 0, 0.0, np.inf))
    ratio = np.where(np.isnan(got[e.written]), np.inf, ratio)
    i = int(np.argmax(ratio))
    worst = float(ratio.flat[i])
    qi, j = divmod(i, got.shape[1])
    q = np.flatnonzero(e.written)[qi]
    return worst, (f"{e.label} row {q} col {j}: got {got[q, j]!r} exact {float(e.exact[q, j])!r} bound {e.bound[q, j]:.3e} "
                   f"ratio {worst:.3g}")


def assert_spmm64(got: np.ndarray, e: Expect64) -> float:
    worst, msg = check_spmm64(got, e)
    assert worst <= 1.0, msg
    return worst


def ragged_csr64(lens, n_cols: int, rng: np.random.Generator, col_pool: Optional[np.ndarray] = None,
                 decades: float = 2.0) -> sparse.csr_matrix:
    """float64 block with the given row lengths, values +-U(0.5, 1.5) * 10^U(-decades, decades) (not fp32 numbers)"""
    lens = np.asarray(lens, dtype=np.int64)
    pool = np.arange(n_cols) if col_pool is None else np.asarray(col_pool)
    indptr = np.concatenate([[0], np.cumsum(lens)])
    cols = np.concatenate([np.sort(pool[rng.choice(pool.size, size=int(l), replace=False)]) for l in lens]
                          + [np.zeros(0, np.int64)]).astype(np.int32)
    vals = rng.uniform(0.5, 1.5, cols.size) * rng.choice([-1.0, 1.0], cols.size) * 10.0 ** rng.uniform(-decades, decades, cols.size)
    return sparse.csr_matrix((vals, cols, indptr), shape=(lens.size, n_cols))
