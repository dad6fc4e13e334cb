"""Host restatement of the predecessor pass of the tropical semirings (test infrastructure only).

A candidate of a row is an entry whose (remapped) column ``u`` is valid and differs from the row's own label; its value
is ``fl32(a + X[u])`` (numpy float32, round to nearest like the device's FADD) and its label is ``u``.  The witness is
the lexicographic ⊕ of the candidates: the better value (min for ``min_plus``, max for ``max_plus``; NaN terms never
win, -0 == +0), ties to the smallest label; no candidate gives ``(⊕ identity, -1)``.  The ⊕ is exact and order-free, so
a device result must equal this restatement exactly.

``predecessors`` walks the levels like ``semiring_ref.SemiringProtocol``'s fused form: level ``j`` reads level-0 rows
through its composed map, each level's pair tile is ⊕-ed into the level above through ``to_prev``, and level 0 compares
the witness with ``D``: ``P[v] = label`` where ``D[v]`` is not the ⊕ identity and equals the witness value, else -1.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np
from scipy import sparse

from oracle.oracle import arrow_mask, number_of_blocks, prepare_permutations
from tests import semiring_ref as sr

_NONE = np.int64(1) << 32          # label -1 compared as unsigned: it loses every tie


def _key(lab: np.ndarray) -> np.ndarray:
    lab = np.asarray(lab, dtype=np.int64)
    return np.where(lab < 0, _NONE, lab)


def better(semiring: str, a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """a is strictly better than b (False where either is NaN)"""
    return (a < b) if semiring == "min_plus" else (a > b)


def lex_plus(semiring: str, av, al, bv, bl) -> Tuple[np.ndarray, np.ndarray]:
    """(av, al) ⊕ (bv, bl) element-wise"""
    take = better(semiring, bv, av) | ((bv == av) & (_key(bl) < _key(al)))
    return np.where(take, bv, av).astype(np.float32), np.where(take, bl, al).astype(np.int32)


def witness_spmm(A: sparse.csr_matrix, X: np.ndarray, semiring: str, col_map: Optional[np.ndarray] = None,
                 self_labels: Optional[np.ndarray] = None, add: Optional[Tuple[np.ndarray, np.ndarray]] = None,
                 add_map: Optional[np.ndarray] = None, max_terms: int = 1 << 23) -> Tuple[np.ndarray, np.ndarray]:
    """(values, labels) of ``arrow_spmm_sr_witness`` in the pair epilogue.  ``col_map`` sends column c to col_map[c]
    (-1: skipped); ``self_labels[r]`` is the label row r excludes (None: r itself, -1: none)."""
    A = sparse.csr_matrix(A)
    n, k = A.shape[0], X.shape[1]
    z = np.float32(sr.zero(semiring))
    X = np.asarray(X, dtype=np.float32)
    vals_out = np.full((n, k), z, dtype=np.float32)
    labs_out = np.full((n, k), -1, dtype=np.int32)
    ip = A.indptr.astype(np.int64)
    cols = A.indices.astype(np.int64)
    if col_map is not None:
        cols = np.asarray(col_map, dtype=np.int64)[cols]
    own = np.arange(n, dtype=np.int64) if self_labels is None else np.asarray(self_labels, dtype=np.int64)
    a_all = A.data.astype(np.float32)
    reduce_best = np.fmin if semiring == "min_plus" else np.fmax        # NaN terms are ignored
    per_chunk = max(max_terms // max(k, 1), 1)
    r = 0
    while r < n:
        r2 = int(np.searchsorted(ip, ip[r] + per_chunk, side="right")) - 1
        r2 = min(max(r2, r + 1), n)
        lo, hi = ip[r], ip[r2]
        rows = np.repeat(np.arange(r, r2), np.diff(ip[r:r2 + 1]))
        c = cols[lo:hi]
        keep = (c >= 0) & (c != own[rows])
        rows, c = rows[keep], c[keep]
        if rows.size:
            terms = a_all[lo:hi][keep][:, None] + X[c]                      # float32 + float32: one rounding
            starts = np.flatnonzero(np.r_[True, rows[1:] != rows[:-1]])
            best = reduce_best.reduceat(terms, starts, axis=0)
            seg = np.repeat(np.arange(starts.size), np.diff(np.r_[starts, rows.size]))
            hit = terms == best[seg]
            lab = np.where(hit, c[:, None], _NONE)
            lab = np.minimum.reduceat(lab, starts, axis=0)
            found = lab < _NONE
            ur = rows[starts]
            vals_out[ur] = np.where(found, best, z)
            labs_out[ur] = np.where(found, lab, -1)
        r = r2
    if add_map is not None:
        am = np.asarray(add_map)
        ok = am >= 0
        av, al = add
        vals_out[ok], labs_out[ok] = lex_plus(semiring, vals_out[ok], labs_out[ok], av[am[ok]], al[am[ok]])
    return vals_out, labs_out


def parents(semiring: str, D: np.ndarray, wv: np.ndarray, wl: np.ndarray) -> np.ndarray:
    """the parent epilogue: the witness label where D is not the ⊕ identity and equals the witness value"""
    D = np.asarray(D, dtype=np.float32)
    return np.where((D != np.float32(sr.zero(semiring))) & (wv == D), wl, -1).astype(np.int32)


class Levels:
    """the level matrices (arrow masks, as the engine uploads them) and the maps of the predecessor pass"""

    def __init__(self, decomposition: Sequence[Tuple[sparse.csr_matrix, np.ndarray]], width: int,
                 block_diagonal: bool = True, n_blocks: Optional[Sequence[int]] = None):
        self.L = len(decomposition)
        self.n_blocks = [number_of_blocks(B, width) for B, _ in decomposition] if n_blocks is None else list(n_blocks)
        self.perms, self.to_prev, _, _ = prepare_permutations([p for _, p in decomposition], self.n_blocks, width)
        self.rows = [nb * width for nb in self.n_blocks]
        self.mats = [arrow_mask(B, width, nb, block_diagonal) for (B, _), nb in zip(decomposition, self.n_blocks)]
        # cmap[j][r]: the level-0 row level j's row r reads (and lands on), -1 when it is not routed from level 0
        self.cmap = [np.arange(self.rows[0], dtype=np.int64)]
        self.tp = [None]
        for j in range(1, self.L):
            tp = np.asarray(self.to_prev[j][: self.rows[j]], dtype=np.int64)
            ok = tp < self.rows[j - 1]
            self.tp.append(np.where(ok, tp, -1))
            self.cmap.append(np.where(ok, self.cmap[j - 1][np.where(ok, tp, 0)], -1))

    def fused_ok(self) -> bool:
        return all(np.all(self.cmap[j][self.mats[j].indices] >= 0) for j in range(1, self.L))

    def to_next(self, j: int) -> np.ndarray:
        """level j-1 row -> the level j row that lands on it (-1: none)"""
        out = np.full(self.rows[j - 1], -1, dtype=np.int64)
        ok = self.tp[j] >= 0
        out[self.tp[j][ok]] = np.arange(self.rows[j])[ok]
        return out


def predecessors(decomposition, width: int, D: np.ndarray, semiring: str, block_diagonal: bool = True,
                 n_blocks: Optional[Sequence[int]] = None, levels: Optional[Levels] = None) -> np.ndarray:
    """P (int32, level-0 rows) of the level-0 features ``D``: deepest level first, level 0 last"""
    lv = levels if levels is not None else Levels(decomposition, width, block_diagonal, n_blocks)
    assert lv.fused_ok(), "a level reads rows behind the sentinel"
    pair = None
    for j in range(lv.L - 1, -1, -1):
        add = dict(add=pair, add_map=lv.to_next(j + 1)) if pair is not None else {}
        col_map = lv.cmap[j] if j > 0 else None
        pair = witness_spmm(lv.mats[j], D, semiring, col_map=col_map, self_labels=lv.cmap[j] if j > 0 else None, **add)
    return parents(semiring, D, *pair)


def brute_force(decomposition, width: int, D: np.ndarray, semiring: str, block_diagonal: bool = True) -> np.ndarray:
    """P by enumeration: every level-0 row collects its candidates from every level, sorts them and takes the first"""
    lv = Levels(decomposition, width, block_diagonal)
    n0, k = lv.rows[0], D.shape[1]
    D = np.asarray(D, dtype=np.float32)
    cands = [[] for _ in range(n0)]                   # (label, weight) per level-0 row
    for j in range(lv.L):
        M = lv.mats[j].tocoo()
        for r, c, a in zip(M.row, M.col, M.data):
            v, u = lv.cmap[j][r], lv.cmap[j][c]
            if v >= 0 and u >= 0 and u != v:
                cands[v].append((int(u), np.float32(a)))
    P = np.full((n0, k), -1, dtype=np.int32)
    sign = 1.0 if semiring == "min_plus" else -1.0
    for v in range(n0):
        for s in range(k):
            terms = [(np.float32(a + D[u, s]), u) for u, a in cands[v]]
            terms = [t for t in terms if not np.isnan(t[0])]
            if not terms or D[v, s] == np.float32(sr.zero(semiring)):
                continue
            val, lab = min(terms, key=lambda t: (sign * float(t[0]), t[1]))
            if val == D[v, s]:
                P[v, s] = lab
    return P
