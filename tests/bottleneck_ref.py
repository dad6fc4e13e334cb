"""Host restatement of the bottleneck semirings of the arrow engine (test infrastructure only).

``max_min`` (widest paths: ⊕ = max, ⊗ = min) and ``min_max`` (minimax paths: ⊕ = min, ⊗ = max) on float32.  Both
operations pick one of their operands, so a device result must equal this restatement bit for bit.  The order is the one
the device uses: a NaN operand is dropped (the other one is returned; two NaNs give NaN), and -0 is below +0.  numpy's
``fmin`` / ``fmax`` promise neither the zero order nor which NaN comes out, so the order here is on integer keys.

It restates the arrow step (through ``semiring_ref.SemiringProtocol``), the fixed point with a pull or a push per level
(the weighted adjacency of ``sr_push_ref``), the step record ``T`` (the level at which each element last changed its
bits) and the path tree of ``ArrowEngine.bottleneck_tree``.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np
from scipy import sparse

from tests import semiring_ref as sr
from tests import sr_push_ref as spr

SEMIRINGS = ("max_min", "min_max")
ZERO = {"max_min": np.float32(-np.inf), "min_max": np.float32(np.inf)}      # ⊕ identity
ONE = {"max_min": np.float32(np.inf), "min_max": np.float32(-np.inf)}       # ⊗ identity
# the tropical semiring with the same ⊕ (and so the same zero_rhs and fresh tiles)
_TWIN = {"max_min": "max_plus", "min_max": "min_plus"}
_PLUS_LARGER = {"max_min": True, "min_max": False}
# a finite value that wins every ⊕ it enters: the canary of rows a launch must not read
WINNER = {"max_min": np.float32(3e38), "min_max": np.float32(-3e38)}


def key(x) -> np.ndarray:
    """uint32 keys that order float32 values like the device's min / max: -0 below +0 (NaN keys are meaningless)"""
    b = np.asarray(x, np.float32).view(np.uint32)
    return np.where(b >= np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def unkey(k) -> np.ndarray:
    k = np.asarray(k, np.uint32)
    return np.where(k >= np.uint32(0x80000000), k & np.uint32(0x7FFFFFFF), ~k).astype(np.uint32).view(np.float32)


def _pick(a, b, larger: bool) -> np.ndarray:
    a, b = np.broadcast_arrays(np.asarray(a, np.float32), np.asarray(b, np.float32))
    ka, kb = key(a), key(b)
    r = np.where(ka > kb if larger else ka < kb, a, b)
    return np.where(np.isnan(a), b, np.where(np.isnan(b), a, r)).astype(np.float32)


def plus(a, b, semiring: str) -> np.ndarray:
    return _pick(a, b, _PLUS_LARGER[semiring])


def times(a, b, semiring: str) -> np.ndarray:
    return _pick(a, b, not _PLUS_LARGER[semiring])


def better(a, b, semiring: str) -> np.ndarray:
    """a is strictly better than b in the ⊕ order (neither NaN)"""
    return key(a) > key(b) if _PLUS_LARGER[semiring] else key(a) < key(b)


def canon(X, semiring: str) -> np.ndarray:
    """the identity diagonal's term: ONE ⊗ x ⊕ ZERO -- x itself, NaN -> the ⊗ identity"""
    return plus(times(ONE[semiring], X, semiring), ZERO[semiring], semiring)


def _fold_term_keys(out_k: np.ndarray, v: np.ndarray, tk: np.ndarray, semiring: str) -> None:
    """out_k[v] ⊕= tk (term keys) for every row of tk"""
    if v.size == 0:
        return
    op = np.maximum if _PLUS_LARGER[semiring] else np.minimum
    order = np.argsort(v, kind="stable")
    vs = v[order]
    starts = np.flatnonzero(np.r_[True, vs[1:] != vs[:-1]])
    red = op.reduceat(tk[order], starts, axis=0)
    out_k[vs[starts]] = op(out_k[vs[starts]], red)


def _term_keys(a: np.ndarray, x: np.ndarray, semiring: str) -> np.ndarray:
    """keys of a ⊗ x (a: [m, 1] weights, x: [m, k] features), a NaN term (both operands NaN) as the ⊕ identity"""
    one, zero = key(ONE[semiring]), key(ZERO[semiring])
    na, nx = np.isnan(a), np.isnan(x)
    ka, kx = np.where(na, one, key(a)), np.where(nx, one, key(x))
    t = np.minimum(ka, kx) if _PLUS_LARGER[semiring] else np.maximum(ka, kx)
    return np.where(na & nx, zero, t)


def _fold_keys(out_k: np.ndarray, v: np.ndarray, terms: np.ndarray, semiring: str) -> None:
    """out_k[v] ⊕= terms on keys, NaN terms dropped"""
    _fold_term_keys(out_k, v, np.where(np.isnan(terms), key(ZERO[semiring]), key(terms)), semiring)


def spmm(A: sparse.csr_matrix, X: np.ndarray, semiring: str, add: Optional[np.ndarray] = None,
         add_map: Optional[np.ndarray] = None, col_map: Optional[np.ndarray] = None) -> np.ndarray:
    """C[r] = (⊕_p A[r,p] ⊗ X[col_p]) ⊕ add[add_map[r]], ``col_map`` as in ``semiring_ref.spmm`` (-1: entry skipped).
    The product of a row never is NaN (it starts at the ⊕ identity and drops NaN terms)."""
    A = sparse.csr_matrix(A)
    n, k = A.shape[0], X.shape[1]
    X = np.asarray(X, np.float32)
    cols = A.indices.astype(np.int64)
    if col_map is not None:
        cols = np.asarray(col_map, np.int64)[cols]
    rows = np.repeat(np.arange(n), np.diff(A.indptr))
    keep = cols >= 0
    rows, cols, vals = rows[keep], cols[keep], A.data.astype(np.float32)[keep]
    out_k = np.full((n, k), key(ZERO[semiring]), np.uint32)
    step = max(1, (1 << 22) // max(k, 1))
    for e0 in range(0, rows.size, step):
        sl = slice(e0, e0 + step)
        _fold_term_keys(out_k, rows[sl], _term_keys(vals[sl, None], X[cols[sl]], semiring), semiring)
    out = unkey(out_k)
    if add_map is not None:
        am = np.asarray(add_map)
        ok = am >= 0
        out[ok] = plus(out[ok], np.asarray(add, np.float32)[am[ok]], semiring)
    return out


class BottleneckProtocol(sr.SemiringProtocol):
    """``semiring_ref.SemiringProtocol`` with the bottleneck ⊕ / ⊗ (the same exchanges, stale rows and zero_rhs)"""

    def __init__(self, decomposition, width: int, k: int, semiring: str, block_diagonal: bool = True,
                 n_blocks: Optional[Sequence[int]] = None, add_identity: bool = False):
        super().__init__(decomposition, width, k, _TWIN[semiring], block_diagonal=block_diagonal, n_blocks=n_blocks,
                         add_identity=add_identity)
        self.semiring = semiring
        self.plus = lambda a, b: plus(a, b, semiring)

    def spmm(self) -> None:
        for j in range(self.L):
            self.C[j] = spmm(self.mats[j], self.X[j], self.semiring)
        if self.add_identity:                             # the diagonal's term ONE ⊗ x: NaN -> the ⊗ identity
            self.C[0] = self.plus(self.C[0], canon(self.X[0], self.semiring))


# ---- the fixed point on the weighted adjacency (sr_push_ref's edges, self-loops included) ----------------------------
def step(X: np.ndarray, adj, semiring: str) -> np.ndarray:
    """F(X) = canon(X) ⊕ every edge's a ⊗ X[u]"""
    X = np.asarray(X, np.float32)
    out_k = key(canon(X, semiring))
    u, v, a = spr._edge_arrays(adj)
    step = max(1, (1 << 22) // max(X.shape[1], 1))
    for e0 in range(0, u.size, step):
        sl = slice(e0, e0 + step)
        _fold_term_keys(out_k, v[sl], _term_keys(a[sl, None], X[u[sl]], semiring), semiring)
    return unkey(out_k)


def push(X: np.ndarray, rows: np.ndarray, adj, semiring: str) -> np.ndarray:
    """out = canon(X), then t = a ⊗ X[u] folded into out[v] for every frontier row u and edge (u -> v, a) where t
    improves on canon(X[v]) in the key order (a NaN t never does)"""
    X = np.asarray(X, np.float32)
    c = canon(X, semiring)
    out_k = key(c)
    u, v, a = spr._edge_arrays(adj)
    sel = np.zeros(X.shape[0], bool)
    sel[np.asarray(rows, np.int64)] = True
    keep = sel[u]
    u, v, a = u[keep], v[keep], a[keep]
    t = times(a[:, None], X[u], semiring)
    ok = ~np.isnan(t) & better(t, c[v], semiring)
    _fold_keys(out_k, v, np.where(ok, t, ZERO[semiring]).astype(np.float32), semiring)
    return unkey(out_k)


def fixed_point(adj, X0: np.ndarray, max_steps: int, direction, semiring: str
                ) -> Tuple[np.ndarray, int, List[str], np.ndarray]:
    """iterate_to_fixed_point with the step record: (final features, steps, direction of each level, T).  The first
    frontier is every row of X0 that is not all ⊕ identity (bit for bit); ``direction(frontier_edges)`` picks "push" or
    "pull"; T[v, s] is the last level whose result differs from its input at (v, s) in bits (0 if none).  The loop stops
    after a level that changes no row in bits (-0 is below +0 in these semirings)."""
    X = np.asarray(X0, np.float32).copy()
    T = np.zeros(X.shape, np.int32)
    rows = spr.frontier(X, np.full_like(X, ZERO[semiring]))
    dirs = []
    for n in range(1, max_steps + 1):
        d = direction(spr.frontier_edges(rows, adj))
        new = push(X, rows, adj, semiring) if d == "push" else step(X, adj, semiring)
        dirs.append(d)
        T[new.view(np.uint32) != X.view(np.uint32)] = n
        rows = spr.frontier(new, X)
        X = new
        if rows.size == 0:
            return X, n, dirs, T
    return X, max_steps, dirs, T


def protocol_fixed_point(p: BottleneckProtocol, X0: np.ndarray, max_steps: int) -> Tuple[np.ndarray, int, np.ndarray]:
    """pull steps of the restated arrow step until one changes no row in bits: (level-0 result, steps, T)"""
    p.set_features(X0)
    prev = np.asarray(X0, np.float32).copy()
    T = np.zeros(prev.shape, np.int32)
    for n in range(1, max_steps + 1):
        cur = p.step().copy()
        T[cur.view(np.uint32) != prev.view(np.uint32)] = n
        if spr.frontier(cur, prev).size == 0:
            return cur, n, T
        prev = cur
    return prev, max_steps, T


# ---- the path tree ---------------------------------------------------------------------------------------------------
def tree_edges(adj) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(u, v, a) of the weighted adjacency without the edges u == v (arrow_adj_build_loopfree's entries)"""
    u, v, a = spr._edge_arrays(adj)
    keep = u != v
    return u[keep], v[keep], a[keep]


def edge_fits(a, du, dv, tu, tv, semiring: str) -> np.ndarray:
    """the tree rule for an edge u -> v of weight a: a ⊗ D[u] == D[v] in bits and D[u] strictly better than D[v], or
    equal in bits with T[u] < T[v]"""
    t = times(a, du, semiring)
    same = np.asarray(du, np.float32).view(np.uint32) == np.asarray(dv, np.float32).view(np.uint32)
    return (t.view(np.uint32) == np.asarray(dv, np.float32).view(np.uint32)) & (better(du, dv, semiring) | (same & (tu < tv)))


def tree(adj, D: np.ndarray, T: np.ndarray, semiring: str) -> np.ndarray:
    """P[v, s]: the smallest u of an edge u -> v (u != v) fitting the rule, where T[v, s] > 0 and D[v, s] is not the ⊕
    identity; -1 elsewhere and where no edge fits"""
    D = np.asarray(D, np.float32)
    n, k = D.shape
    u, v, a = tree_edges(adj)
    P = np.full((n, k), np.iinfo(np.int64).max, np.int64)
    fits = edge_fits(a[:, None], D[u], D[v], T[u], T[v], semiring)
    ee, cc = np.nonzero(fits)
    np.minimum.at(P, (v[ee], cc), u[ee])
    pending = (T > 0) & (D != ZERO[semiring])
    return np.where(pending & (P < np.iinfo(np.int64).max), P, -1).astype(np.int32)


def _bits_of(x) -> np.uint32:
    return np.asarray(x, np.float32).view(np.uint32)


def check_tree(adj, D: np.ndarray, T: np.ndarray, P: np.ndarray, semiring: str, fixed_point: bool = True,
               X0: Optional[np.ndarray] = None) -> None:
    """the tree properties, vectorised: every parent edge exists and fits the rule, only elements with T > 0 that are
    reached have parents, and the parents have no cycles (pointer jumping ends every chain at a root).  At a fixed point
    every element with T > 0 that is reached has a parent, with two exceptions that come from the NaN features of
    ``X0``: the NaN feature itself (the first level turns it into the ⊗ identity, a source with T == 1), and an element
    that the first level gives the ⊗ identity through an edge of weight ⊗ identity from such a feature (ONE ⊗ NaN = ONE:
    both ends then hold ONE with T == 1, so neither is strictly better nor earlier)."""
    D = np.asarray(D, np.float32)
    n, k = D.shape
    u, v, a = tree_edges(adj)
    has = P >= 0
    pending = (T > 0) & (D != ZERO[semiring])
    assert not np.any(has & ~pending), "a source or an element not reached has a parent"
    if fixed_point:
        if X0 is not None:
            X0 = np.asarray(X0, np.float32)
            pending &= ~np.isnan(X0)
            one = _bits_of(ONE[semiring])
            via = np.isnan(X0[u]) & (np.asarray(a, np.float32).view(np.uint32) == one)[:, None]
            ee, cc = np.nonzero(via)
            through_nan = np.zeros(D.shape, bool)
            through_nan[v[ee], cc] = True
            pending &= ~(through_nan & (T == 1) & (D.view(np.uint32) == one))
        assert np.all(has[pending]), f"{int(np.sum(pending & ~has))} elements reached at a level have no parent"
    # every parent edge exists and one of its duplicates fits the rule
    order = np.lexsort((v, u))
    pair = u[order] * n + v[order]
    ea = a[order]
    pv, pc = np.nonzero(has)
    pu = P[has].astype(np.int64)
    q = pu * n + pv
    j = np.searchsorted(pair, q)
    assert np.all(j < pair.size) and np.all(pair[np.minimum(j, pair.size - 1)] == q), "a parent edge does not exist"
    ok = np.zeros(pu.size, bool)
    while True:
        live = ~ok & (j < pair.size)
        live[live] = pair[j[live]] == q[live]
        if not live.any():
            break
        ok[live] = edge_fits(ea[j[live]], D[pu[live], pc[live]], D[pv[live], pc[live]], T[pu[live], pc[live]],
                             T[pv[live], pc[live]], semiring)
        j += 1
    assert ok.all(), f"{int((~ok).sum())} parent edges do not fit the rule"
    # no cycles: after log2(n) + 1 rounds of pointer jumping every chain sits at a root (P == -1); a cycle never does
    cols = np.broadcast_to(np.arange(k), (n, k))
    J = P.astype(np.int64)
    for _ in range(int(np.ceil(np.log2(max(n, 2)))) + 1):
        nxt = np.where(J >= 0, J[np.maximum(J, 0), cols], -1)
        J = np.where(nxt >= 0, nxt, J)
    assert np.all(np.where(J >= 0, P[np.maximum(J, 0), cols], -1) == -1), "the parents have a cycle"
