"""Per-element error bound of one whole arrow step (test infrastructure, host only).

``tests/spmm_bound.py`` bounds one SpMM launch.  This module bounds what a chain of launches returns: one
``ArrowEngine.step()`` / ``ShardedArrowEngine.step()`` -- forward exchange, every level's product, backward aggregation
-- element by element, so that a wrong row map, a dropped or doubled level contribution or a precision loss shows up on
a row whose true value is far below the level's largest entry (the normwise rule ``1e-5 * max|C|`` of
``assert_close`` / ``close_rows`` cannot see those).

Exact result and magnitudes
---------------------------
``ExactStep`` runs ``oracle.ReferenceProtocolOracle`` at ``np.longdouble`` on the device's own starting state: the
level-0 features (``features(0)``) and, in exchange mode, the level tiles the rows behind the sentinel carry.  The same
oracle on the absolute decomposition and ``|X|`` gives ``mag``, the sum of ``|term|`` every element is made of.
``Rank1Step`` does the same for rank-1 features ``X = fp32(u v^T)`` with one float64 mat-vec per level
(``bench.expected_step_on_vector``), so a 10M-row step is checked in row chunks without a float64 tile.

The bound
---------
Every element of level 0 after one step is a sum of products ``A_j[s, c] * X_j[c, col]`` (exact inputs: the forward
exchange and the stale rows only copy) over the levels ``j`` whose chain row ``s`` maps onto it (``to_prev`` composed
down to level 0).  If every product passes through at most ``M`` rounded operations (an FMA rounds once)

    |got - exact| <= gamma_M(2^-24) * mag + M * 2^-150 * (1 + gamma_M(2^-24))

(Higham, *Accuracy and Stability of Numerical Algorithms*, 2nd ed., Lemma 3.1 and section 4.2; ``2^-150`` is the
absolute error of one rounding into the fp32 subnormal range, carried through at most ``M`` further roundings).  The
longdouble reference is off by at most ``gamma_M(u_ld) * mag`` and so is ``mag`` itself, hence ``2 gamma_M(u_ld) * mag``
on top.  Elements with ``mag == 0`` have no non-zero term and must be exact.  No constant is tuned.

``M`` is per level-0 row: ``sum_j (T_j + 1)`` over the levels whose chain row exists, ``T_j`` the tree height of that
row (``tree_height`` of ``spmm_bound.py``: ``n + 2`` at or below the long-row threshold, the long-row height above it;
``arrow_b200.cu:899-973`` ``k_spmm_tiles_v1``, ``:1110-1239`` ``k_spmm_tiles``, ``:1283-1331`` ``k_spmm_generic``,
``:1347-1409`` ``k_spmm_long_partial`` / ``k_spmm_long_reduce``).  The ``+ 1`` is the add that carries the row to the
level above.  Route by route (float32, ``ArrowEngine`` in ``arrow_matrix_b200/engine.py``):

* ``exchange`` (``engine.py:382-437``): ``gather_rows`` copies (``k_gather_rows``, ``arrow_b200.cu:1628-1672``: no
  arithmetic), one fresh product per level (``T_j``), then ``C_{j-1}[r] += C_j[s]``, one add per level
  (``k_gather_rows<.., ACC>``, ``:1657-1666``).  A level-``j`` product passes ``T_j + j`` roundings.
* ``fused/gather`` (``engine.py:397-411``): level ``j`` starts its accumulator at the deeper level's row (``acc += add``,
  ``arrow_b200.cu:1115-1125``, exact on a zero accumulator) and adds its own entries with one FMA each; the long-row pair
  adds the addend after the segment partials (``k_spmm_long_reduce``).  The deeper row therefore passes at most
  ``T_j`` more roundings: ``sum_{i<=j} T_i`` for a level-``j`` product.
* ``fused/scatter`` (``engine.py:412-416``): level 0's product, then each level ``j >= 1`` accumulates into level-0 rows
  (``acc = C_old``, ``:1112-1114``, then one FMA per entry).  Whatever is in the row passes ``T_j`` more roundings per
  later level: at most ``sum_j T_j``.
* two-part X operand and row-pointer epilogues (``k_spmm_tiles<.., OUT_ROWPTR, .., DUALX>``, ``:1011-1017, :1099-1101,
  :1231-1232``): they only change where an X row is read and where the result row is stored; ``T_j`` is unchanged.
* sharded engine (``arrow_matrix_b200/sharded.py:788-840``, fused with or without the side lane, and the CUDA graph that
  replays it): every rank multiplies its partial head rows (rows ``< min(width, rows_j)``) and GPU 0 adds the
  ``world`` partials in rank order (``k_reduce_rows``, ``arrow_b200.cu:1731-1756``: ``world - 1`` adds); a partial row
  holds at most ``n`` of the row's ``n`` entries, so its height is ``max_{m <= n} T(m)`` (``tree_height_upto``: the
  long-row height is not monotone across the threshold).  The staged level-1 rows reach level 0 with one gather-add
  (``final_add``).  Head rows get ``T_j + 1 + (world - 1)``.

All routes are covered by ``M = sum_j (T_j + 1) [+ world - 1 on head rows]``; the float64 engine runs the same
structure with ``u = 2^-53`` (``tests/test_gpu_fp64.py``).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
from scipy import sparse

from oracle import oracle
from tests.spmm_bound import ETA32, U32, U64, gamma, tree_height
from tests.spmm_bound64 import ULD

LONG_THRESHOLD, LONG_SEGMENT = 512, 2048          # arrow_set_tuning defaults (tests/tile_dispatch.py)


def abs_decomposition(dec):
    """the decomposition with every stored value replaced by its absolute value (the magnitudes' operator)"""
    return [(abs(sparse.csr_matrix(B)), p) for B, p in dec]


def tree_height_upto(n, threshold: int = LONG_THRESHOLD, segment: int = LONG_SEGMENT):
    """``max_{m <= n} tree_height(m)``: the height of any part of a row with ``n`` entries (a sharded partial head row)"""
    n = np.asarray(n, dtype=np.int64)
    return np.maximum(tree_height(n, threshold, segment), np.minimum(n, threshold) + 2)


def chain_maps(to_prev: Sequence[Optional[np.ndarray]], rows: Sequence[int]) -> List[np.ndarray]:
    """per level ``j``: the level-0 row each level-``j`` row is aggregated into (-1: none, the chain meets the
    sentinel).  Level 0 maps to itself."""
    maps = [np.arange(rows[0], dtype=np.int64)]
    for j in range(1, len(rows)):
        tp = np.asarray(to_prev[j][: rows[j]], dtype=np.int64)
        valid = tp < rows[j - 1]
        maps.append(np.where(valid, maps[j - 1][np.where(valid, tp, 0)], -1))
    return maps


def chain_heights(row_nnz: Sequence[np.ndarray], to_prev: Sequence[Optional[np.ndarray]], width: int,
                  world: int = 1) -> np.ndarray:
    """``M`` of the module docstring for every level-0 row (int64 [rows_0])"""
    rows = [int(n.size) for n in row_nnz]
    maps = chain_maps(to_prev, rows)
    M = np.zeros(rows[0], dtype=np.int64)
    for j, (nnz, cm) in enumerate(zip(row_nnz, maps)):
        h = (tree_height_upto(nnz) if world > 1 else tree_height(nnz)) + 1
        if world > 1:
            h[: min(width, rows[j])] += world - 1
        ok = cm >= 0
        M[cm[ok]] += h[ok]                        # the maps are injective
    return M


def oracle_heights(po: oracle.ReferenceProtocolOracle, world: int = 1) -> np.ndarray:
    return chain_heights([np.diff(M.indptr) for M in po.mats], po.to_prev, po.width, world)


def step_height(po: oracle.ReferenceProtocolOracle, world: int = 1) -> np.ndarray:
    """``M`` as a column [rows_0, 1], ready to broadcast over the feature columns"""
    return oracle_heights(po, world)[:, None]


def bound_of(mag: np.ndarray, M: np.ndarray, u: float = U32, eta: float = ETA32, u_ref: float = ULD) -> np.ndarray:
    """the bound of the module docstring (0 where ``mag == 0``: no non-zero term, the result must be exact)"""
    mag = np.asarray(mag, dtype=np.float64)
    g = gamma(M, u)
    b = (g + 2.0 * gamma(M, u_ref)) * mag + M * eta * (1.0 + g)
    return np.where(mag > 0, b, 0.0)


# ---- the exact step ------------------------------------------------------------------------------------------------
class ExactStep:
    """Exact (longdouble) step and magnitudes of one decomposition, started from a given device state."""

    def __init__(self, dec, width: int, k: int, block_diagonal: bool = True, n_blocks=None, world: int = 1):
        kw = dict(block_diagonal=block_diagonal, n_blocks=n_blocks, dtype=np.longdouble)
        self.po = oracle.ReferenceProtocolOracle(dec, width, k, **kw)
        self.pa = oracle.ReferenceProtocolOracle(abs_decomposition(dec), width, k, **kw)
        self.M = step_height(self.po, world)
        self.L = self.po.L

    def run(self, X0: np.ndarray, carried: Optional[Sequence[np.ndarray]] = None):
        """``(exact, mag)`` of level 0 after one step from features ``X0``; ``carried[j - 1]`` (exchange mode): level
        ``j``'s tile before the step, whose rows behind the sentinel stay in the product"""
        x = np.asarray(X0).astype(np.longdouble)
        self.po.set_features(x)
        self.pa.set_features(np.abs(x))
        for j in range(1, self.L):
            c = np.zeros_like(self.po.C[j]) if carried is None else np.asarray(carried[j - 1]).astype(np.longdouble)
            self.po.C[j], self.pa.C[j] = c, np.abs(c)
        exact = self.po.step().copy()
        mag = self.pa.step().astype(np.float64)
        return exact, mag


def check(got: np.ndarray, exact: np.ndarray, mag: np.ndarray, M: np.ndarray, *, route: str = "",
          row_scale: Optional[np.ndarray] = None, row0: int = 0, u: float = U32, eta: float = ETA32,
          u_ref: float = ULD):
    """(worst ``err / bound``, message naming its row, column, level-0 row scale and route); inf for a NaN or an
    inexact element without a term"""
    got = np.asarray(got)
    assert got.shape == exact.shape, f"{route}: shape {got.shape} != {exact.shape}"
    b = bound_of(mag, M, u, eta, u_ref)
    err = np.abs(got.astype(np.longdouble) - exact).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err == 0, 0.0, np.inf))
    ratio = np.where(np.isnan(err), np.inf, ratio)
    if ratio.size == 0:
        return 0.0, f"{route}: empty"
    i = int(np.argmax(ratio))
    r, c = divmod(i, got.shape[1])
    worst = float(ratio.flat[i])
    scale = float(row_scale[r]) if row_scale is not None else float("nan")
    Mr = int(np.broadcast_to(M, got.shape)[r, c])
    n_bad = int(np.count_nonzero(~(ratio <= 1.0)))
    msg = (f"{route}: worst err/bound {worst:.3g} at row {row0 + r} col {c} (level-0 row scale {scale:.3g}, height {Mr}): "
           f"got {got[r, c]!r} exact {float(exact[r, c])!r} |err| {err[r, c]:.3e} bound {b[r, c]:.3e} mag "
           f"{mag[r, c]:.3e}; {n_bad} elements outside the bound")
    return worst, msg


def assert_step(got, exact, mag, M, **kw) -> float:
    worst, msg = check(got, exact, mag, M, **kw)
    assert worst <= 1.0, msg
    return worst


# ---- features whose scale varies per element -------------------------------------------------------------------------
def row_exponents(n: int, width: int, rng: np.random.Generator, large_rows: Sequence[int] = ()) -> np.ndarray:
    """``e_r`` of the spread features: a block-row exponent in [0, 32] plus a row jitter in [0, 8], so whole block-rows
    are small; [24, 40] on the head block-row, which every block-row reads (a small block-row stays small); 0 on
    ``large_rows`` (hubs stay large)"""
    nb = -(-n // width)
    e = rng.integers(0, 33, nb)[np.arange(n) // width] + rng.integers(0, 9, n)
    e[: min(width, n)] = rng.integers(24, 41, min(width, n))
    e[np.asarray(large_rows, dtype=np.int64)] = 0
    return e


def spread_features(n: int, k: int, width: int, rng: np.random.Generator, large_rows: Sequence[int] = (),
                    subnormal_rows: Optional[np.ndarray] = None):
    """``X[r, c] = +-U[0.5, 1) * 2^-e_r * 2^-f_c`` (float32), ``e_r`` of ``row_exponents`` and ``f_c`` in [0, 8].
    ``subnormal_rows``: those rows get ``e_r`` in [130, 136], the float32 subnormal range.  Returns ``(X, 2^-e_r)``."""
    e = row_exponents(n, width, rng, large_rows)
    if subnormal_rows is not None:
        e[subnormal_rows] = rng.integers(130, 137, np.asarray(subnormal_rows).size)
    f = rng.integers(0, 9, k)
    mant = rng.uniform(0.5, 1.0, (n, k)) * rng.choice([-1.0, 1.0], (n, k))
    X = (mant * np.exp2(-e.astype(np.float64))[:, None] * np.exp2(-f.astype(np.float64))[None, :]).astype(np.float32)
    return X, np.exp2(-e.astype(np.float64))


def rescale_rows(dec, rng: np.random.Generator, spread: int = 24):
    """every matrix row's values times ``2^-g``, ``g`` in [0, spread] per row and level (exact in float32)"""
    out = []
    for B, p in dec:
        B = sparse.csr_matrix(B, copy=True)
        g = rng.integers(0, spread + 1, B.shape[0])
        B.data = (B.data * np.repeat(np.exp2(-g.astype(np.float64)), np.diff(B.indptr))).astype(B.dtype)
        out.append((B, p))
    return out


def hub_rows_of(dec, threshold: int = LONG_THRESHOLD) -> np.ndarray:
    """level-0 rows above the long-row threshold"""
    B = sparse.csr_matrix(dec[0][0])
    return np.flatnonzero(np.diff(B.indptr) > threshold)


# ---- rank-1 features at benchmark scale -------------------------------------------------------------------------------
def rank1_vectors(n: int, k: int, width: int, rng: np.random.Generator, large_rows: Sequence[int] = ()):
    """``u[r] = +-U[0.5, 1) * 2^-e_r`` (``e_r`` of ``row_exponents``, in [0, 40]) and ``v[c] = U[0.5, 1) * 2^-f_c`` with
    ``f_c`` in [0, 8]: ``X = fp32(u v^T)`` stays normal (no rounding below 2^-126)"""
    e = row_exponents(n, width, rng, large_rows)
    u = rng.uniform(0.5, 1.0, n) * rng.choice([-1.0, 1.0], n) * np.exp2(-e.astype(np.float64))
    v = rng.uniform(0.5, 1.0, k) * np.exp2(-rng.integers(0, 9, k).astype(np.float64))
    return u, v


def rank1_features(u: np.ndarray, v: np.ndarray, r0: int, r1: int) -> np.ndarray:
    return (u[r0:r1, None] * v[None, :]).astype(np.float32)


@dataclass
class Rank1Step:
    """Closed form of one step on ``X = fp32(u v^T)``: ``exact = (S u) v^T`` and ``mag = (|S| |u|) |v|^T`` with ``S``
    the step in float64 (``bench.expected_step_on_vector``).  Against the step of the rounded features the bound gains
    the input rounding ``|X - u v^T| <= 2^-24 |u| |v|^T`` pushed through ``|S|`` (``2^-24 mag``) and the float64
    arithmetic of ``S u``, ``|S| |u|`` and the product with ``v`` (``3 gamma_{M+1}(2^-53) mag``); the features are
    normal, so ``mag`` bounds the step of ``|X|`` up to ``(1 + 2^-24)``."""
    y: np.ndarray
    ya: np.ndarray
    v: np.ndarray
    M: np.ndarray

    @classmethod
    def build(cls, dec, width: int, u: np.ndarray, v: np.ndarray, block_diagonal: bool = True):
        import bench
        from arrow_matrix_b200 import decomp
        y, state_free = bench.expected_step_on_vector(dec, width, u, block_diagonal)
        assert state_free, "the rank-1 form needs a decomposition whose non-zeros never read a row behind the sentinel"
        ya, _ = bench.expected_step_on_vector(abs_decomposition(dec), width, np.abs(u), block_diagonal)
        n_blocks = [decomp.number_of_blocks(B, width) for B, _ in dec]
        _, to_prev, _, _ = decomp.prepare_permutations([p for _, p in dec], n_blocks, width)
        nnz = [np.diff(decomp.arrow_rows(B, width, nb, block_diagonal, 0, nb * width)[0]) for (B, _), nb in zip(dec, n_blocks)]
        return cls(y, ya, np.asarray(v, dtype=np.float64), chain_heights(nnz, to_prev, width))

    def expect(self, r0: int, r1: int):
        """``(exact, bound)`` of rows ``[r0, r1)`` in float64"""
        M = self.M[r0:r1, None]
        mag = np.abs(self.ya[r0:r1, None]) * np.abs(self.v)[None, :]
        g = gamma(M, U32)
        b = (g * (1.0 + U32) + U32 + 3.0 * gamma(M + 1, U64)) * mag + M * ETA32 * (1.0 + g)
        return self.y[r0:r1, None] * self.v[None, :], np.where(mag > 0, b, 0.0), mag

    def check(self, got: np.ndarray, r0: int = 0, route: str = "", row_scale: Optional[np.ndarray] = None,
              chunk: int = 1 << 16):
        """worst (ratio, message) over the rows ``got`` holds (``got[i]`` = row ``r0 + i``), in row chunks"""
        worst, msg, n_bad = -1.0, f"{route}: no rows", 0
        for a0 in range(0, got.shape[0], chunk):
            a1 = min(got.shape[0], a0 + chunk)
            exact, b, _ = self.expect(r0 + a0, r0 + a1)
            err = np.abs(got[a0:a1].astype(np.float64) - exact)
            with np.errstate(divide="ignore", invalid="ignore"):
                ratio = np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err == 0, 0.0, np.inf))
            ratio = np.where(np.isnan(err), np.inf, ratio)
            n_bad += int(np.count_nonzero(~(ratio <= 1.0)))
            i = int(np.argmax(ratio))
            if float(ratio.flat[i]) > worst:
                r, c = divmod(i, got.shape[1])
                worst = float(ratio.flat[i])
                q = r0 + a0 + r
                scale = float(row_scale[q]) if row_scale is not None else float("nan")
                msg = (f"{route}: worst err/bound {worst:.3g} at row {q} col {c} (level-0 row scale {scale:.3g}, height "
                       f"{int(self.M[q])}): got {got[a0 + r, c]!r} exact {exact[r, c]!r} |err| {err[r, c]:.3e} bound "
                       f"{b[r, c]:.3e}")
        return max(worst, 0.0), f"{msg}; {n_bad} elements outside the bound"
