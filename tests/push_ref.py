"""Host restatement of the direction-optimising BFS of the (or, and) engine (test infrastructure only).

With the identity, a fused (or, and) step is ``X' = X | M X``: ``M`` is the level-0 x level-0 union, over the levels ``j``,
of the edges ``cmap_j(c) -> cmap_j(r)`` for every entry ``(r, c)`` of level ``j`` (``cmap_0`` the identity, ``cmap_j`` the
level-j -> level-0 row map), without the edges that have an end at -1 or ``u == v``.  The push adjacency is ``M``
transposed as CSR: row ``u`` lists its destinations ``v`` in ascending order, duplicates kept.  Inside a BFS, where
``X_h = X_{h-1} | M X_{h-1}``, the next level is ``X_h | M F_h`` with ``F_h`` the rows holding a bit of ``X_h & ~X_{h-1}``:
a push of the frontier rows.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np
from scipy import sparse

from tests import bool_ref as br


def level_maps(p: br.BoolProtocol) -> List[np.ndarray]:
    """level-j row -> level-0 row (-1: not routed) of every level of a protocol; level 0 is the identity"""
    maps = [np.arange(p.rows[0], dtype=np.int64)]
    for j in range(1, p.L):
        tp = p.to_prev[j][: p.rows[j]]
        ok = tp < p.rows[j - 1]
        maps.append(np.where(ok, maps[-1][np.where(ok, tp, 0)], -1))
    return maps


def protocol_parts(p: br.BoolProtocol) -> List[Tuple[sparse.csr_matrix, Optional[np.ndarray]]]:
    """(level matrix, level-j -> level-0 map or None for the identity) of every level"""
    maps = level_maps(p)
    return [(p.mats[0], None)] + [(p.mats[j], maps[j]) for j in range(1, p.L)]


def fused_ok(p: br.BoolProtocol) -> bool:
    """every column a level > 0 reads is routed to a level-0 row (the engine's ``fused_ok``)"""
    maps = level_maps(p)
    return all(np.all(maps[j][p.mats[j].indices] >= 0) for j in range(1, p.L))


def edges(parts: Sequence[Tuple[sparse.csr_matrix, Optional[np.ndarray]]]) -> Tuple[np.ndarray, np.ndarray]:
    """(u, v) of every edge: entry (r, c) with c >= 0 of a part gives map(c) -> map(r); ends at -1 and u == v dropped"""
    us, vs = [], []
    for A, m in parts:
        A = sparse.csr_matrix(A)
        r = np.repeat(np.arange(A.shape[0], dtype=np.int64), np.diff(A.indptr))
        c = A.indices.astype(np.int64)
        ok = c >= 0
        r, c = r[ok], c[ok]
        if m is not None:
            m = np.asarray(m, dtype=np.int64)
            r, c = m[r], m[c]
        keep = (r >= 0) & (c >= 0) & (r != c)
        us.append(c[keep])
        vs.append(r[keep])
    return np.concatenate(us) if us else np.zeros(0, np.int64), np.concatenate(vs) if vs else np.zeros(0, np.int64)


def adjacency(parts, n: int) -> Tuple[np.ndarray, np.ndarray]:
    """(indptr, indices) as int32: row u lists every v of an edge u -> v in ascending order, duplicates kept"""
    u, v = edges(parts)
    order = np.lexsort((v, u))
    indptr = np.zeros(n + 1, np.int64)
    np.add.at(indptr, u + 1, 1)
    return np.cumsum(indptr).astype(np.int32), v[order].astype(np.int32)


def step(X: np.ndarray, adj) -> np.ndarray:
    """X | M X"""
    indptr, indices = adj
    src = np.repeat(np.arange(indptr.size - 1), np.diff(indptr))
    out = np.asarray(X, bool).copy()
    np.logical_or.at(out, indices, out[src].copy())
    return out


def frontier(X_new: np.ndarray, X_old: np.ndarray) -> np.ndarray:
    """rows holding a bit set in X_new and clear in X_old"""
    return np.flatnonzero(np.any(X_new & ~X_old, axis=1))


def frontier_edges(rows: np.ndarray, adj) -> int:
    indptr = adj[0].astype(np.int64)
    return int(np.sum(indptr[rows + 1] - indptr[rows]))


def push(X: np.ndarray, rows: np.ndarray, adj) -> np.ndarray:
    """out = X, then out[v] |= X[u] for every frontier row u and every v of adjacency row u"""
    indptr, indices = adj
    n = indptr.size - 1
    X = np.asarray(X, bool)
    sel = np.zeros(n, bool)
    sel[np.asarray(rows, dtype=np.int64)] = True
    src = np.repeat(np.arange(n), np.diff(indptr))
    keep = sel[src]
    S = sparse.csr_matrix((np.ones(int(keep.sum()), np.float32), (indices[keep], src[keep])), shape=(n, n))
    out = X.copy()
    for c0 in range(0, X.shape[1], 512):             # counts of set bits, exact below 2**24 per element
        out[:, c0:c0 + 512] |= (S @ X[:, c0:c0 + 512].astype(np.float32)) > 0
    return out


def bfs(adj, X0: np.ndarray, max_steps: int, direction) -> Tuple[np.ndarray, int, List[str]]:
    """hop levels (0 for the bits of X0, h where the h-th level sets the bit, -1 never), levels taken and the direction
    of each; ``direction(frontier_edges)`` picks ``"push"`` or ``"pull"``.  The first frontier is every row of X0 with a
    bit (the previous level is all zero)."""
    X = np.asarray(X0, bool).copy()
    dist = np.where(X, 0, -1).astype(np.int32)
    rows = frontier(X, np.zeros_like(X))
    steps, dirs = 0, []
    for level in range(1, max_steps + 1):
        d = direction(frontier_edges(rows, adj))
        new = push(X, rows, adj) if d == "push" else step(X, adj)
        dirs.append(d)
        steps = level
        fresh = new & ~X
        dist[fresh] = level
        rows = frontier(new, X)
        X = new
        if not fresh.any():
            break
    return dist, steps, dirs


# ---- the push dispatch of the source -----------------------------------------------------------------------------------
def push_kind(k: int) -> str:
    """the k_bits_push instance arrow_bits_push_frontier launches at k columns: uint32 one-word rows, else uint4 vectors"""
    return "unsigned" if br.words(k) == 1 else "uint4"


def source_push_kinds(path: str) -> set:
    """the ``k_bits_push<...>`` launches of ``arrow_bits_push_frontier`` in the CUDA source"""
    import re
    with open(path) as f:
        src = f.read()
    body = src[src.index("int arrow_bits_push_frontier(arrow_ctx *ctx"):]
    body = body[:body.index("\n}\n")]
    return set(re.findall(r"k_bits_push<(\w+)><<<", body))
