"""Host restatement of ArrowEngine.connected_components (test infrastructure only).

The vertices are the level-0 rows ``0 .. n - 1``, padding rows included.  Every entry ``(r, c)`` of level ``j`` as the
step applies it (``pagerank_ref.level_parts``: the arrow pattern, with the identity diagonal when ``add_identity``) is the
edge ``cmap_j(c) -- cmap_j(r)`` whatever its value; an end at -1 and ``u == v`` give none, and direction is ignored.
``labels[v]`` is the smallest row of ``v``'s component, the count is the number of ``v`` with ``labels[v] == v`` and
``sizes[r]`` the member count of the component labelled ``r`` (0 where ``r`` is not a label).  The components come from
``scipy.sparse.csgraph.connected_components(directed=True, connection="weak")`` on the structural operator.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np
from scipy import sparse
from scipy.sparse import csgraph

from tests import pagerank_ref as prr


def structural(parts, n: int) -> sparse.csr_matrix:
    """the operator with every edge set to 1 (duplicates summed) and no diagonal: row v lists the sources u of u -> v"""
    u, v, _, ok = prr.entries(parts)
    keep = ok & (u != v)
    return sparse.csr_matrix((np.ones(int(keep.sum())), (v[keep], u[keep])), shape=(n, n))


def smallest_labels(comp: np.ndarray) -> np.ndarray:
    """component ids -> the smallest index of each component, per index (int32)"""
    comp = np.asarray(comp, np.int64)
    first = np.full(int(comp.max(initial=-1)) + 1, comp.size, np.int64)
    np.minimum.at(first, comp, np.arange(comp.size, dtype=np.int64))
    return first[comp].astype(np.int32)


def components(parts, n: int) -> Tuple[np.ndarray, int, np.ndarray]:
    """(labels int32 [n], component count, sizes int32 [n])"""
    _, comp = csgraph.connected_components(structural(parts, n), directed=True, connection="weak")
    labels = smallest_labels(comp)
    sizes = np.bincount(labels, minlength=n).astype(np.int32)
    return labels, int(np.count_nonzero(labels == np.arange(n))), sizes


def of(dec, width: int, block_diagonal: bool = True, add_identity: bool = False,
       n_blocks=None) -> Tuple[np.ndarray, int, np.ndarray]:
    """``components`` of the operator an engine on ``dec`` steps"""
    parts, proto = prr.level_parts(dec, width, n_blocks, block_diagonal=block_diagonal, add_identity=add_identity)
    return components(parts, proto.rows[0])


def by_vertex(labels: np.ndarray, perm0: np.ndarray, n_vertices: int) -> np.ndarray:
    """row-order labels (the ``ArrowDecompositionMPI`` view) -> per original vertex ``x < n_vertices``, the smallest vertex
    id of its component.  ``perm0[r]`` is the vertex at level-0 row ``r``; rows holding ids ``>= n_vertices`` are padding
    and must be singletons (asserted)."""
    perm0 = np.asarray(perm0, np.int64)
    labels = np.asarray(labels, np.int64)
    rows = np.arange(labels.size)
    pad = perm0 >= n_vertices
    assert np.all(labels[pad] == rows[pad]) and not np.any(np.isin(labels[~pad], rows[pad])), "a padding row is joined"
    first = np.full(labels.size, np.iinfo(np.int64).max)
    np.minimum.at(first, labels, perm0)
    out = np.empty(n_vertices, np.int64)
    out[perm0[~pad]] = first[labels[~pad]]
    return out
