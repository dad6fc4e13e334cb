"""Host restatement of the weighted betweenness of the min-plus engine (test infrastructure only).

``M`` is the operator of ``tests/push_ref.py`` with a weight on every entry: entry ``(r, c)`` of value ``a`` of a part
is the edge ``map(c) -> map(r)`` of weight ``a``, ends at -1 and ``u == v`` dropped.  ``D`` is the min-plus fixed point
reached from the features ``X0`` (``fixed_point``, or the engine's).  Then, per column ``s``:

- an entry ``u -> v`` of weight ``a`` is tight when ``D[u, s] < D[v, s] < +inf`` and ``fl(a + D[u, s]) == D[v, s]``
  (float32: a ``+inf`` weight or an overflowing sum never reaches an element that is not reached);
  the pair ``(u, v)`` is tight when one of its entries is, and counts once, at its first entry of the sorted list;
- ``S_s = {v : D[v, s] finite and D[v, s] == X0[v, s]}``;
- ``sigma[v, s]`` is 0 where ``D[v, s]`` is not finite, else ``[v in S_s]`` plus the sum of ``sigma[u, s]`` over the
  tight pairs ``u -> v``;
- ``delta[v, s]`` is 0 where ``D[v, s]`` is not finite or ``v in S_s``, else ``sigma[v, s]`` times the sum of
  ``fl((1 + delta[w, s]) / sigma[w, s])`` over the tight pairs ``v -> w`` with ``sigma[w, s] != 0`` (a successor without
  paths, which a loop cut short by ``max_steps`` can leave, adds nothing);
- ``bc[v]`` is the sum of ``delta[v, s]`` over ``s`` in column order.

A tight pair strictly increases ``D``, so the elements are taken in ascending ``D`` (the counts) and descending ``D``
(the dependencies): an order that does not depend on how the device schedules them.  Every sum follows ``seg_sum`` of
``tests/paths_ref.py``, so the GPU results equal these bit for bit.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np
from scipy import sparse

from tests import paths_ref as pa


def edges(parts) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(u, v, weight) of every edge of M: entry (r, c) with c >= 0 gives map(c) -> map(r); ends at -1 and u == v dropped"""
    us, vs, ws = [], [], []
    for A, m in parts:
        A = sparse.csr_matrix(A)
        r = np.repeat(np.arange(A.shape[0], dtype=np.int64), np.diff(A.indptr))
        c = A.indices.astype(np.int64)
        w = np.asarray(A.data, np.float32)
        ok = c >= 0
        r, c, w = r[ok], c[ok], w[ok]
        if m is not None:
            m = np.asarray(m, dtype=np.int64)
            r, c = m[r], m[c]
        keep = (r >= 0) & (c >= 0) & (r != c)
        us.append(c[keep])
        vs.append(r[keep])
        ws.append(w[keep])
    if not us:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32)
    return np.concatenate(us), np.concatenate(vs), np.concatenate(ws)


def _csr(rows, cols, w, n):
    order = np.lexsort((cols, rows))
    indptr = np.zeros(n + 1, np.int64)
    np.add.at(indptr, rows + 1, 1)
    return np.cumsum(indptr), cols[order], w[order]


def adjacencies(parts, n: int):
    """(in-lists, out-lists), each (indptr, indices, weights): row v lists the u of its edges u -> v, row u the v of its
    edges u -> v, in ascending order, duplicates kept (their weights in any order)"""
    u, v, w = edges(parts)
    return _csr(v, u, w, n), _csr(u, v, w, n)


def fixed_point(parts, n: int, X0: np.ndarray, max_steps: int) -> np.ndarray:
    """the min-plus step with the identity, X' = min(canon(X), min over edges u -> v of fl(a + X[u])), from X0 until it
    changes nothing or max_steps steps (self-loops of positive weight never improve a value: they are left out; NaN terms
    are dropped, as in the step)"""
    u, v, w = edges(parts)
    D = np.where(np.isnan(X0), np.inf, X0 + np.float32(0)).astype(np.float32)
    for _ in range(max_steps):
        nxt = D.copy()
        with np.errstate(over="ignore", invalid="ignore"):
            t = (w[:, None] + D[u]).astype(np.float32)
        np.minimum.at(nxt, v, np.where(np.isnan(t), np.float32(np.inf), t))
        if np.array_equal(nxt, D):
            break
        D = nxt
    return D


def _tight_pairs(D: np.ndarray, row: int, ptr, idx, wts, incoming: bool) -> Tuple[np.ndarray, np.ndarray]:
    """(list, [entries x k] mask): the pairs of the row's list that are tight, marked at their first entry"""
    lst = idx[ptr[row]:ptr[row + 1]].astype(np.int64)
    a = wts[ptr[row]:ptr[row + 1]].astype(np.float32)[:, None]
    other, here = D[lst], D[row][None, :]
    with np.errstate(invalid="ignore", over="ignore"):
        if incoming:
            T = (other < here) & (here < np.inf) & ((a + other) == here)
        else:
            T = (here < other) & (other < np.inf) & ((a + here) == other)
    out = np.zeros_like(T)
    if lst.size:
        starts = np.flatnonzero(pa.distinct(lst))
        out[starts] = np.logical_or.reduceat(T, starts, axis=0)
    return lst, out


def sources(D: np.ndarray, X0: np.ndarray) -> np.ndarray:
    """[n x k] v in S_s"""
    return np.isfinite(D) & (D == X0)


def path_counts(D: np.ndarray, X0: np.ndarray, in_lists) -> np.ndarray:
    ptr, idx, wts = in_lists
    S = sources(D, X0)
    sigma = np.zeros(D.shape)
    fin = np.isfinite(D)
    for d in np.unique(D[fin]):
        for v in np.flatnonzero(np.any(D == d, axis=1)):
            lst, T = _tight_pairs(D, v, ptr, idx, wts, True)
            cols = D[v] == d
            total = pa.seg_sum(np.where(T, sigma[lst], 0.0))
            sigma[v, cols] = (np.where(S[v], 1.0, 0.0) + total)[cols]
    return sigma


def dependencies(D: np.ndarray, X0: np.ndarray, sigma: np.ndarray, out_lists) -> np.ndarray:
    ptr, idx, wts = out_lists
    S = sources(D, X0)
    delta = np.zeros(D.shape)
    fin = np.isfinite(D)
    for d in np.unique(D[fin])[::-1]:
        for v in np.flatnonzero(np.any(D == d, axis=1)):
            lst, T = _tight_pairs(D, v, ptr, idx, wts, False)
            cols = D[v] == d
            with np.errstate(divide="ignore", invalid="ignore"):
                terms = np.where(T & (sigma[lst] != 0), (1.0 + delta[lst]) / sigma[lst], 0.0)
                got = np.where(S[v], 0.0, sigma[v] * pa.seg_sum(terms))
            delta[v, cols] = got[cols]
    return delta


def betweenness(parts, n: int, X0: np.ndarray, max_steps: int, D: np.ndarray = None):
    """(D, sigma, delta, bc) from the features X0 [n x k] (float32); D is the host fixed point unless given"""
    X0 = np.asarray(X0, np.float32)
    if D is None:
        D = fixed_point(parts, n, X0, max_steps)
    in_lists, out_lists = adjacencies(parts, n)
    sigma = path_counts(D, X0, in_lists)
    delta = dependencies(D, X0, sigma, out_lists)
    return D, sigma, delta, pa.row_sum(delta)


# ---- small cases shared by the CPU and GPU tests ---------------------------------------------------------------------
def graph(n, entries):
    """entries (u, v, weight) as a one-part operator: entry (v, u) is the edge u -> v"""
    u, v, w = (np.array(x) for x in zip(*entries))
    return [(sparse.csr_matrix((w.astype(np.float32), (v, u)), shape=(n, n)), None)]


def infinite_weight_case():
    """(parts, X0): row 3 is reached in column 1 only; column 0 reaches it through two +inf weights and column 2 through a
    finite weight whose sum with the source's offset overflows to +inf"""
    big = np.float32(3e38)
    parts = graph(6, [(0, 3, np.inf), (1, 3, np.inf), (2, 3, 1.0), (4, 3, big), (3, 5, 1.0)])
    X0 = np.full((6, 3), np.inf, np.float32)
    X0[[0, 1], 0] = 0.0
    X0[2, 1] = 0.0
    X0[4, 2] = big
    return parts, X0


def cut_short_case():
    """(parts, X0, max_steps): after 3 steps D[4] = 3 came from 0 -> 1 -> 2 -> 4 while 5 = 11 and 6 = 12 still hold the
    relaxation through the first D[4] = 10, so 5 has no tight predecessor and no paths, and its tight successor 6 neither"""
    parts = graph(7, [(0, 4, 10.0), (0, 1, 1.0), (1, 2, 1.0), (2, 4, 1.0), (4, 5, 1.0), (5, 6, 1.0)])
    X0 = np.full((7, 1), np.inf, np.float32)
    X0[0, 0] = 0.0
    return parts, X0, 3

