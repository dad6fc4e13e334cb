"""Host-side preparation of a loaded decomposition for the device engine.

Product restatement of what the reference's root rank does between reading the files and sending
blocks (``arrow/arrow_dec_mpi.py:612-627, 679-749``; ``arrow/common/graphio.py:361-406``), written
for row *ranges* so that each GPU can prepare just its shard straight from memory-mapped files
instead of the reference's root-reads-everything + MPI scatter (SURVEY.md N1).
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
from scipy import sparse

Triplet = Tuple[Optional[np.ndarray], np.ndarray, np.ndarray]      # (data | None, indices, indptr)
Level = Union[sparse.csr_matrix, Triplet]


def level_triplet(level: Level) -> Triplet:
    if isinstance(level, tuple):
        return level
    m = sparse.csr_matrix(level)
    return (m.data, m.indices, m.indptr)


def number_of_blocks(level: Level, width: int) -> int:
    """Block-rows up to the last non-empty row (``ArrowDecompositionMPI.number_of_blocks``, :612-627)."""
    indptr = np.asarray(level_triplet(level)[2])
    nnz_total = int(indptr[-1] - indptr[0])
    if nnz_total == 0:
        raise ValueError("level has no non-zero row")
    # last row r with indptr[r+1] > indptr[r]  ==  first position where indptr reaches its final value
    last = int(np.searchsorted(indptr, indptr[-1], side="left")) - 1
    return -(-(last + 1) // width)


def prepare_permutations(perms: Sequence[np.ndarray], n_blocks: Sequence[int], width: int):
    """Padding, 1-based fix-up and level-to-level row maps (``arrow_dec_mpi.py:699-749``).

    Returns ``(perms, to_prev, to_next, sentinel)``: ``to_prev[j][r]`` is the row of level ``j-1``
    holding the same vertex as row ``r`` of level ``j`` (sentinel ``2*width*n_blocks[0]`` when that
    row lies outside level ``j-1``'s active block-rows); ``to_next`` likewise towards ``j+1``.
    """
    rows = int(n_blocks[0]) * width
    sentinel = 2 * width * int(n_blocks[0])
    fixed = []
    one_based = bool(np.min(perms[0]) > 0)
    for p in perms:
        p = np.array(p, dtype=np.int64)
        if one_based:
            p = p - 1
        if p.size < rows:
            p = np.concatenate([p, np.arange(p.size, rows, dtype=np.int64)])
        if p.size != rows:
            raise ValueError(f"permutation has {p.size} entries but level 0 has only {rows} rows "
                             f"({n_blocks[0]} blocks of {width}); the reference asserts here too")
        fixed.append(p)
    inv = []
    for p in fixed:
        q = np.empty(rows, dtype=np.int64)
        q[p] = np.arange(rows, dtype=np.int64)
        inv.append(q)
    L = len(fixed)
    to_prev: List[Optional[np.ndarray]] = [None] * L
    to_next: List[Optional[np.ndarray]] = [None] * L
    for j in range(L):
        if j > 0:
            t = inv[j - 1][fixed[j]]
            t[t >= width * int(n_blocks[j - 1])] = sentinel
            to_prev[j] = t
        if j < L - 1:
            t = inv[j + 1][fixed[j]]
            t[t >= width * int(n_blocks[j + 1])] = sentinel
            to_next[j] = t
    return fixed, to_prev, to_next, sentinel


def arrow_rows(level: Level, width: int, n_blocks: int, block_diagonal: bool, row_begin: int, row_end: int,
               chunk_rows: int = 1 << 21, dtype=np.float32):
    """CSR arrays of rows ``[row_begin, row_end)`` of a level, restricted to what the reference multiplies.

    The reference only ever materialises blocks (0,j), (i,0), (i,i) and, in banded mode, (i,i+-1)
    (``graphio.py:382-383``), truncated to ``n_blocks`` block-rows/columns (``arrow_dec_mpi.py:728-731``);
    rows at or beyond the end of the file are empty (the ``indptr`` edge padding of ``graphio.py:394-399``).
    Returns ``(indptr[int64, rebased], indices, data|None, dropped_nnz)``; ``data`` has element type ``dtype`` (float32
    values become float64 exactly when ``dtype`` is float64).
    """
    data, indices, indptr = level_triplet(level)
    n = n_blocks * width
    file_rows = indptr.shape[0] - 1
    row_end = min(row_end, n)
    assert 0 <= row_begin <= row_end
    have_end = min(row_end, file_rows)
    out_ptr = np.zeros(row_end - row_begin + 1, dtype=np.int64)
    idx_parts, dat_parts = [], []
    dropped = 0
    pos = 0
    r = row_begin
    while r < have_end:
        r2 = min(have_end, r + chunk_rows)
        ip = np.asarray(indptr[r:r2 + 1]).astype(np.int64)
        a, b = int(ip[0]), int(ip[-1])
        cols = np.asarray(indices[a:b])
        counts = np.diff(ip)
        rows = np.repeat(np.arange(r, r2, dtype=np.int64), counts)
        bi = rows // width
        bj = cols.astype(np.int64) // width
        keep = (cols < n) & ((bi == 0) | (bj == 0) | (bi == bj))
        if not block_diagonal:
            keep |= (cols < n) & (np.abs(bi - bj) == 1)
        vals = None if data is None else np.asarray(data[a:b])
        if keep.all():
            new_counts = counts
        else:
            dropped += int(keep.size - np.count_nonzero(keep))
            new_counts = np.bincount(rows[keep] - r, minlength=r2 - r)
            cols = cols[keep]
            if vals is not None:
                vals = vals[keep]
        out_ptr[r - row_begin + 1: r2 - row_begin + 1] = pos + np.cumsum(new_counts)
        pos += int(new_counts.sum())
        idx_parts.append(cols)
        if vals is not None:
            dat_parts.append(vals)
        r = r2
    if have_end < row_end:                       # rows past the end of the file: empty
        out_ptr[max(have_end - row_begin, 0) + 1:] = pos
    if not idx_parts:
        idx = np.zeros(0, dtype=np.int32)
    else:
        idx = np.concatenate(idx_parts) if len(idx_parts) != 1 else idx_parts[0]
    if data is None:
        dat = None
    elif not dat_parts:
        dat = np.zeros(0, dtype=dtype)
    else:
        dat = np.concatenate(dat_parts) if len(dat_parts) != 1 else dat_parts[0]
        dat = np.ascontiguousarray(dat, dtype=dtype)
    return out_ptr, np.ascontiguousarray(idx), dat, dropped


def with_diagonal(indptr: np.ndarray, indices: np.ndarray, data: Optional[np.ndarray], rows: int, value: float,
                  dtype=np.float32):
    """CSR arrays (as ``arrow_rows`` returns them) with an entry ``(r, r)`` of ``value`` in front of every row ``r <
    rows``, next to any entry the row already has there.  ``data`` None means ones.  In a semiring whose ⊗ identity is
    ``value`` the block then computes ``X ⊕ (A ⊗ X)`` on its rows; the diagonal lies in the blocks (i, i), which every
    arrow level keeps."""
    ip = np.asarray(indptr, dtype=np.int64)
    assert ip.size == rows + 1
    out_ptr = ip + np.arange(rows + 1, dtype=np.int64)
    nnz = int(out_ptr[-1])
    diag = out_ptr[:-1]
    rest = np.ones(nnz, dtype=bool)
    rest[diag] = False
    idx = np.empty(nnz, dtype=np.result_type(np.asarray(indices).dtype, np.int32))
    idx[diag] = np.arange(rows)
    idx[rest] = indices
    dat = np.empty(nnz, dtype=dtype)
    dat[diag] = value
    dat[rest] = 1 if data is None else data
    return out_ptr, idx, dat


def block_partition(n_blocks: int, parts: int) -> np.ndarray:
    """Contiguous, as-even-as-possible split of ``n_blocks`` block-rows over ``parts`` GPUs (bounds array).

    Ceil-based so the low ranks fill first: block-row 0 (the arrow head, which the sharded engine keeps on
    rank 0) always belongs to rank 0, and with fewer blocks than GPUs the trailing ranks own nothing."""
    g = np.arange(parts + 1, dtype=np.int64)
    return (g * n_blocks + parts - 1) // parts


def locality_partition(to_prev: np.ndarray, n_blocks: int, width: int, prev_bounds_rows: np.ndarray, parts: int,
                       min_local: float = 0.5, max_skew: float = 4.0) -> Optional[np.ndarray]:
    """Permutation-aware split of a level's block-rows (bounds array like ``block_partition``), or ``None``.

    ``to_prev[r]`` is the row of the level above that row ``r`` exchanges with; ``prev_bounds_rows`` says which GPU owns
    which rows there.  Every block-row votes for the GPU that owns most of its partners; if the votes are monotone
    (so the shards stay contiguous ranges), at least ``min_local`` of all routed rows then stay on their GPU and no shard
    exceeds ``max_skew`` times the even share, the level is cut where its rows map -- the exchange turns into local
    loads.  A uniformly random permutation fails the locality test and keeps the even split.  (The reference fixes
    one rank per block-row and always pays the all-to-all, arrow_dec_mpi.py:134-160.)"""
    rows = n_blocks * width
    if n_blocks < 1 or parts < 2:
        return None
    tp = np.asarray(to_prev[:rows])
    valid = tp < int(prev_bounds_rows[-1])
    owner = np.searchsorted(prev_bounds_rows, np.where(valid, tp, 0), side="right") - 1
    blk = np.arange(rows, dtype=np.int64) // width
    votes = np.zeros((n_blocks, parts), dtype=np.int64)
    np.add.at(votes, (blk[valid], owner[valid]), 1)
    routed = votes.sum(axis=1)
    choice = np.argmax(votes, axis=1)
    choice[0] = 0                                           # block-row 0 (the arrow head) lives on GPU 0
    choice = np.where(routed > 0, choice, -1)
    # blocks without any routed row follow their predecessor
    for b in range(1, n_blocks):
        if choice[b] < 0:
            choice[b] = choice[b - 1]
    if np.any(np.diff(choice) < 0):
        return None
    local = int(votes[np.arange(n_blocks), choice].sum())
    if routed.sum() == 0 or local < min_local * routed.sum():
        return None
    bounds = np.searchsorted(choice, np.arange(parts + 1), side="left").astype(np.int64)
    bounds[-1] = n_blocks
    if np.max(np.diff(bounds)) > max_skew * max(n_blocks / parts, 1.0):
        return None
    return bounds
