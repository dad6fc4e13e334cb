"""Host restatement of the direction-optimising fixed point of the min_plus / max_plus engine (test infrastructure only).

With the identity, a fused tropical step is ``F(X)[v] = canon(X[v]) ⊕ (⊕ over the edges (u -> v, a) of fl(a + X[u]))``,
NaN terms dropped, ``canon(x) = fl(0 + x)`` with NaN mapped to the ⊕ identity: the identity diagonal's term.  The edges
are those of ``tests/push_ref.py`` (entry (r, c) of level j is ``cmap_j(c) -> cmap_j(r)``), each carrying its entry's
value, self-loops included.  Inside a fixed-point loop (``X_h = F(X_{h-1})``, ``X_{-1}`` the ⊕ identity) the next level
is the push of the rows whose bits changed: ``canon(X_h) ⊕`` their relaxations, counted only where they improve on
``canon(X_h)``.  It equals ``F(X_h)`` bit for bit unless a weight is -0.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
from scipy import sparse

from tests import semiring_ref as sr

ZERO = {"min_plus": np.float32(np.inf), "max_plus": np.float32(-np.inf)}


def weighted_edges(parts) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(u, v, weight) of every edge: entry (r, c) with c >= 0 of a part gives map(c) -> map(r); ends at -1 dropped, u == v
    kept"""
    us, vs, ws = [], [], []
    for A, m in parts:
        A = sparse.csr_matrix(A)
        r = np.repeat(np.arange(A.shape[0], dtype=np.int64), np.diff(A.indptr))
        c = A.indices.astype(np.int64)
        w = A.data.astype(np.float32)
        ok = c >= 0
        r, c, w = r[ok], c[ok], w[ok]
        if m is not None:
            m = np.asarray(m, dtype=np.int64)
            r, c = m[r], m[c]
        keep = (r >= 0) & (c >= 0)
        us.append(c[keep])
        vs.append(r[keep])
        ws.append(w[keep])
    if not us:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32)
    return np.concatenate(us), np.concatenate(vs), np.concatenate(ws)


def sort_duplicates(indptr: np.ndarray, indices: np.ndarray, values: np.ndarray):
    """(indices, values) with every row's entries in (destination, weight bits) order: the layout a device build gives
    up to the order of the duplicates of (u, v)"""
    rows = np.repeat(np.arange(indptr.size - 1), np.diff(indptr.astype(np.int64)))
    bits = np.asarray(values, np.float32).view(np.uint32)
    order = np.lexsort((bits, indices, rows))
    return indices[order], values[order]


def weighted_adjacency(parts, n: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(indptr, indices, values): row u lists every (v, weight) of an edge u -> v by destination, duplicates kept"""
    u, v, w = weighted_edges(parts)
    indptr = np.zeros(n + 1, np.int64)
    np.add.at(indptr, u + 1, 1)
    indptr = np.cumsum(indptr).astype(np.int32)
    order = np.lexsort((w.view(np.uint32), v, u))
    return indptr, v[order].astype(np.int32), w[order]


def canon(X: np.ndarray, semiring: str) -> np.ndarray:
    """fl(0 + x), NaN -> the ⊕ identity"""
    out = np.float32(0) + np.asarray(X, np.float32)
    return np.where(np.isnan(out), ZERO[semiring], out).astype(np.float32)


def _fold(out: np.ndarray, v: np.ndarray, terms: np.ndarray, semiring: str) -> None:
    terms = np.where(np.isnan(terms), ZERO[semiring], terms)
    (np.minimum if semiring == "min_plus" else np.maximum).at(out, v, terms)


def _edge_arrays(adj):
    indptr, indices, values = adj
    src = np.repeat(np.arange(indptr.size - 1), np.diff(indptr.astype(np.int64)))
    return src, indices.astype(np.int64), np.asarray(values, np.float32)


def step(X: np.ndarray, adj, semiring: str) -> np.ndarray:
    """F(X): canon(X) ⊕ every edge's fl(a + X[u]), NaN terms dropped"""
    X = np.asarray(X, np.float32)
    out = canon(X, semiring)
    u, v, a = _edge_arrays(adj)
    for c0 in range(0, X.shape[1], 64):
        o = out[:, c0:c0 + 64]
        _fold(o, v, a[:, None] + X[u, c0:c0 + 64], semiring)
        out[:, c0:c0 + 64] = o
    return out


def frontier(X_new: np.ndarray, X_old: np.ndarray) -> np.ndarray:
    """rows in which some element differs in bits"""
    a = np.asarray(X_new, np.float32).view(np.uint32)
    b = np.asarray(X_old, np.float32).view(np.uint32)
    return np.flatnonzero(np.any(a != b, axis=1))


def rows_changed(X_new: np.ndarray, X_old: np.ndarray) -> int:
    """rows in which some element differs by value (-0 == +0, NaN != NaN): count_diff's figure"""
    return int(np.sum(np.any(np.asarray(X_new) != np.asarray(X_old), axis=1)))


def frontier_edges(rows: np.ndarray, adj) -> int:
    indptr = adj[0].astype(np.int64)
    return int(np.sum(indptr[rows + 1] - indptr[rows]))


def push(X: np.ndarray, rows: np.ndarray, adj, semiring: str) -> np.ndarray:
    """out = canon(X), then t = fl(a + X[u]) folded into out[v] for every frontier row u and edge (u -> v, a) where t
    improves on canon(X[v])"""
    X = np.asarray(X, np.float32)
    c = canon(X, semiring)
    out = c.copy()
    u, v, a = _edge_arrays(adj)
    sel = np.zeros(X.shape[0], bool)
    sel[np.asarray(rows, dtype=np.int64)] = True
    keep = sel[u]
    u, v, a = u[keep], v[keep], a[keep]
    for c0 in range(0, X.shape[1], 64):
        t = a[:, None] + X[u, c0:c0 + 64]
        better = t < c[v, c0:c0 + 64] if semiring == "min_plus" else t > c[v, c0:c0 + 64]
        o = out[:, c0:c0 + 64]
        _fold(o, v, np.where(better, t, ZERO[semiring]).astype(np.float32), semiring)
        out[:, c0:c0 + 64] = o
    return out


def fixed_point(adj, X0: np.ndarray, max_steps: int, direction, semiring: str) -> Tuple[np.ndarray, int, List[str]]:
    """iterate_to_fixed_point: (final features, steps, direction of each level); ``direction(frontier_edges)`` picks
    ``"push"`` or ``"pull"``.  The first frontier is every row of X0 that is not all ⊕ identity (bit for bit)."""
    X = np.asarray(X0, np.float32).copy()
    rows = frontier(X, np.full_like(X, ZERO[semiring]))
    dirs = []
    for n in range(1, max_steps + 1):
        d = direction(frontier_edges(rows, adj))
        new = push(X, rows, adj, semiring) if d == "push" else step(X, adj, semiring)
        dirs.append(d)
        changed = rows_changed(new, X)
        rows = frontier(new, X)
        X = new
        if changed == 0:
            return X, n, dirs
    return X, max_steps, dirs


def protocol_fixed_point(p: sr.SemiringProtocol, X0: np.ndarray, max_steps: int) -> Tuple[np.ndarray, int]:
    """pull steps of the restated arrow step until one changes no row (count_diff's test): (level-0 result, steps)"""
    p.set_features(X0)
    prev = np.asarray(X0, np.float32).copy()
    for n in range(1, max_steps + 1):
        cur = p.step().copy()
        if rows_changed(cur, prev) == 0:
            return cur, n
        prev = cur
    return prev, max_steps


def with_weights(decomposition: Sequence, rng: np.random.Generator, self_loop: float = -2.0):
    """the decomposition with integer weights in [-3, 8] (0 and negatives included) and, on level 0, a self-loop of weight
    ``self_loop`` on row 0 (the diagonal blocks are kept by every level's arrow mask)"""
    out = []
    for j, (B, perm) in enumerate(decomposition):
        B = sparse.csr_matrix(B, dtype=np.float32, copy=True)
        B.data = rng.integers(-3, 9, B.nnz).astype(np.float32)
        if j == 0:
            B = B.tolil()
            B[0, 0] = self_loop
            B = sparse.csr_matrix(B, dtype=np.float32)
        out.append((B, perm))
    return out


def special_features(rows: int, k: int, semiring: str, rng: np.random.Generator) -> np.ndarray:
    """features with finite values, both infinities, -0 and NaN; most elements the ⊕ identity"""
    X = np.full((rows, k), ZERO[semiring], np.float32)
    pick = rng.random((rows, k))
    X[pick < 0.10] = rng.integers(-5, 20, int(np.sum(pick < 0.10))).astype(np.float32)
    X[(pick >= 0.10) & (pick < 0.12)] = -ZERO[semiring]
    X[(pick >= 0.12) & (pick < 0.14)] = np.float32(-0.0)
    X[(pick >= 0.14) & (pick < 0.16)] = np.float32(np.nan)
    return X


# ---- the push dispatch of the source -----------------------------------------------------------------------------------
def push_kind(k: int) -> str:
    """the k_sr_push instance arrow_sr_push_frontier launches at k columns: float4 groups when k % 4 == 0, else floats"""
    return "float4" if k % 4 == 0 else "float"


def source_push_kinds(path: str) -> set:
    """the (semiring, element) instances of ``k_sr_push`` launched by ``arrow_sr_push_frontier`` in the CUDA source"""
    import re
    with open(path) as f:
        src = f.read()
    body = src[src.index("int arrow_sr_push_frontier(arrow_ctx *ctx"):]
    body = body[:body.index("\n}\n")]
    return set(re.findall(r"SRP\((SrM\w+), (\w+), ", body))
