"""Host restatement of the BFS parents of the (or, and) engine (test infrastructure only).

``M`` is the operator of ``tests/push_ref.py``.  The in-adjacency stores it by destination: row ``v`` lists every ``u``
of an edge ``u -> v`` in ascending order, duplicates kept.  Inside a BFS, ``X_h = X_{h-1} | M X_{h-1}``; a bit ``(v, s)``
fresh at level ``h`` takes as parent the first ``u`` of ``v``'s in-list whose bit ``s`` is set in ``X_{h-1}``.  Such a
``u`` has hop level ``h - 1``, so the parent tile is ``P[v, s] = min {u : u -> v in M, L[u, s] = L[v, s] - 1}`` where
``L[v, s] > 0`` and -1 elsewhere (``definition``).
"""
from __future__ import annotations

from typing import Tuple

import numpy as np

from tests import push_ref as pr


def in_adjacency(parts, n: int) -> Tuple[np.ndarray, np.ndarray]:
    """(indptr, indices) as int32: row v lists every u of an edge u -> v in ascending order, duplicates kept"""
    u, v = pr.edges(parts)
    order = np.lexsort((u, v))
    indptr = np.zeros(n + 1, np.int64)
    np.add.at(indptr, v + 1, 1)
    return np.cumsum(indptr).astype(np.int32), u[order].astype(np.int32)


def level_parents(X_new: np.ndarray, X_old: np.ndarray, in_adj, P: np.ndarray) -> np.ndarray:
    """``arrow_bits_parents``: for every bit set in X_new and clear in X_old, P = the first u of the row's in-list whose
    bit is set in X_old, -1 when none is; every other element of P is left alone.  Returns P (updated in place)."""
    indptr, indices = in_adj
    fresh = X_new & ~X_old
    for v in pr.frontier(X_new, X_old):
        ins = indices[indptr[v]:indptr[v + 1]]
        cols = np.flatnonzero(fresh[v])
        if ins.size == 0:
            P[v, cols] = -1
            continue
        hit = X_old[ins][:, cols]                         # [in-edges x fresh columns]
        P[v, cols] = np.where(hit.any(axis=0), ins[np.argmax(hit, axis=0)], -1)
    return P


def bfs_tree(in_adj, out_adj, X0: np.ndarray, max_steps: int) -> Tuple[np.ndarray, np.ndarray, int]:
    """(levels, parents, steps) of a BFS from X0: ``push_ref.bfs``'s levels (pull steps; the direction changes neither),
    the parents of each level's fresh bits from the two bit tiles of that level"""
    X = np.asarray(X0, bool).copy()
    dist = np.where(X, 0, -1).astype(np.int32)
    P = np.full(X.shape, -1, np.int32)
    steps = 0
    for level in range(1, max_steps + 1):
        new = pr.step(X, out_adj)
        steps = level
        fresh = new & ~X
        dist[fresh] = level
        level_parents(new, X, in_adj, P)
        X = new
        if not fresh.any():
            break
    return dist, P, steps


def definition(L: np.ndarray, parts, n: int) -> np.ndarray:
    """P[v, s] = min {u : u -> v in M, L[u, s] = L[v, s] - 1} where L[v, s] > 0, else -1 (by enumeration of the edges)"""
    u, v = pr.edges(parts)
    k = L.shape[1]
    big = np.iinfo(np.int64).max
    best = np.full((n, k), big, np.int64)
    ok = (L[v] > 0) & (L[u] == L[v] - 1)                  # [edges x k]
    e, s = np.nonzero(ok)
    np.minimum.at(best, (v[e], s), u[e])
    return np.where(best == big, -1, best).astype(np.int32)
