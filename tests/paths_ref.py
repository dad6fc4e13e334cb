"""Host restatement of the shortest-path counts and Brandes dependencies of the (or, and) engine (test infrastructure only).

``M`` is the operator of ``tests/push_ref.py``, taken as a set: its lists keep duplicate entries, and an entry equal to its
predecessor in the (sorted) list is skipped.  ``L`` is the level tile of a BFS (``push_ref.bfs``).  Then, float64:

- ``sigma[v, s]`` is 1 where ``L[v, s] = 0``, 0 where ``L[v, s] = -1``, else the sum of ``sigma[u, s]`` over the distinct
  ``u -> v`` with ``L[u, s] = L[v, s] - 1``;
- ``delta[v, s]`` is 0 where ``L[v, s] <= 0``, else ``sigma[v, s]`` times the sum of ``fl((1 + delta[w, s]) / sigma[w, s])``
  over the distinct ``v -> w`` with ``L[w, s] = L[v, s] + 1``;
- ``bc[v]`` is the sum of ``delta[v, s]`` over ``s`` in column order.

Every sum follows the kernels' order (``seg_sum``): the row's list in ascending order, ``SEG`` entries at a time from its
start, each segment summed left to right, the partials added in segment order.  So the GPU results equal these bit for bit.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np

from tests import parents_ref as par
from tests import push_ref as pr

SEG = 512           # list entries per partial sum (PATH_SEG)


def seg_sum(terms: np.ndarray) -> np.ndarray:
    """[entries x k] terms in list order -> [k]: left to right within each SEG-entry segment, then over the segments"""
    k = terms.shape[1]
    if terms.shape[0] == 0:
        return np.zeros(k)
    parts = np.stack([np.add.accumulate(terms[i:i + SEG], axis=0)[-1] for i in range(0, terms.shape[0], SEG)])
    return np.add.accumulate(parts, axis=0)[-1]


def distinct(row: np.ndarray) -> np.ndarray:
    """mask of the entries of a sorted list that differ from their predecessor"""
    keep = np.ones(row.size, bool)
    keep[1:] = row[1:] != row[:-1]
    return keep


def path_counts(L: np.ndarray, in_adj) -> np.ndarray:
    """sigma from the level tile, level after level along the in-lists"""
    indptr, indices = in_adj
    sigma = np.where(L == 0, 1.0, 0.0)
    for h in range(1, int(L.max(initial=0)) + 1):
        for v in np.flatnonzero(np.any(L == h, axis=1)):
            ins = indices[indptr[v]:indptr[v + 1]].astype(np.int64)
            hit = (L[ins] == h - 1) & (L[v] == h)[None, :] & distinct(ins)[:, None]
            cols = L[v] == h
            sigma[v, cols] = seg_sum(np.where(hit, sigma[ins], 0.0))[cols]
    return sigma


def dependencies(L: np.ndarray, sigma: np.ndarray, out_adj) -> np.ndarray:
    """delta from the levels and counts, from the deepest level down to 1 along the out-lists"""
    indptr, indices = out_adj
    delta = np.zeros(L.shape)
    for h in range(int(L.max(initial=0)), 0, -1):
        for u in np.flatnonzero(np.any(L == h, axis=1)):
            outs = indices[indptr[u]:indptr[u + 1]].astype(np.int64)
            hit = (L[outs] == h + 1) & (L[u] == h)[None, :] & distinct(outs)[:, None]
            terms = np.zeros((outs.size, L.shape[1]))
            terms[hit] = (1.0 + delta[outs][hit]) / sigma[outs][hit]
            cols = L[u] == h
            delta[u, cols] = sigma[u, cols] * seg_sum(terms)[cols]
    return delta


def row_sum(delta: np.ndarray) -> np.ndarray:
    """bc[v] = delta[v, 0] + delta[v, 1] + ..., left to right"""
    if delta.shape[1] == 0:
        return np.zeros(delta.shape[0])
    return np.add.accumulate(delta, axis=1)[:, -1].copy()


def adjacencies(parts, n: int):
    """(in-adjacency, push adjacency) of M"""
    return par.in_adjacency(parts, n), pr.adjacency(parts, n)


def betweenness(parts, n: int, X0: np.ndarray, max_steps: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, int]:
    """(levels, sigma, delta, bc, steps) of a BFS from the source bits X0 [n x k]"""
    in_adj, out_adj = adjacencies(parts, n)
    L, steps, _ = pr.bfs(out_adj, X0, max_steps, lambda edges: "pull")
    sigma = path_counts(L, in_adj)
    delta = dependencies(L, sigma, out_adj)
    return L, sigma, delta, row_sum(delta), steps
