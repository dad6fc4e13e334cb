"""Host restatement of the arrow step in the boolean semiring (or, and) on bool arrays (test infrastructure only).

⊗ is "the entry exists" (the values of a block are never read) and ⊕ is OR.  OR is exact, so a device result must equal
this restatement bit for bit.  Bit tiles hold column c of a row in bit c % 32 of word c // 32, little-endian, and a row
of more than 32 columns is padded with zero words to a multiple of 4 words (a row of up to 32 is one word); ``pack`` /
``unpack`` restate that layout column by column.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np
from scipy import sparse

from oracle.oracle import arrow_mask, number_of_blocks, prepare_permutations


def words(k: int) -> int:
    """uint32 words per row of a bit tile of k columns: one for k <= 32, else a multiple of 4"""
    return 1 if k <= 32 else ((k + 31) // 32 + 3) // 4 * 4


def pack(X: np.ndarray) -> np.ndarray:
    n, k = X.shape
    out = np.zeros((n, words(k)), dtype=np.uint32)
    for c in range(k):
        out[:, c // 32] |= (X[:, c] != 0).astype(np.uint32) << np.uint32(c % 32)
    return out


def unpack(W: np.ndarray, k: int) -> np.ndarray:
    return np.stack([(W[:, c // 32] >> np.uint32(c % 32)) & np.uint32(1) for c in range(k)], axis=1).astype(bool) \
        if k else np.zeros((W.shape[0], 0), bool)


def spmm(A: sparse.csr_matrix, X: np.ndarray, add: Optional[np.ndarray] = None, add_map: Optional[np.ndarray] = None,
         col_map: Optional[np.ndarray] = None) -> np.ndarray:
    """C[r] = (OR_p X[col_p]) | add[add_map[r]] over the stored entries of A (structure only); ``col_map`` sends column c to
    col_map[c] (-1: entry skipped); a row without valid entries gets zeros"""
    A = sparse.csr_matrix(A)
    n = A.shape[0]
    X = np.asarray(X, dtype=bool)
    cols = A.indices.astype(np.int64)
    if col_map is not None:
        cols = np.asarray(col_map, dtype=np.int64)[cols]
    rows = np.repeat(np.arange(n), np.diff(A.indptr))
    keep = cols >= 0
    S = sparse.csr_matrix((np.ones(int(keep.sum()), np.float32), (rows[keep], cols[keep])), shape=(n, X.shape[0]))
    out = (S @ X.astype(np.float32)) > 0                  # counts of set bits: exact below 2**24 entries per row
    if add_map is not None:
        am = np.asarray(add_map)
        ok = am >= 0
        out[ok] |= np.asarray(add, dtype=bool)[am[ok]]
    return out


class BoolProtocol:
    """``semiring_ref.SemiringProtocol`` in (or, and): the forward exchange moves rows, each level's product is fresh,
    the backward aggregation ORs the routed rows in, and ``X`` aliases ``C`` after every exchange so that rows behind
    the sentinel keep the previous step's result.  ``add_identity`` ORs level 0's features into its product."""

    def __init__(self, decomposition: Sequence[Tuple[sparse.csr_matrix, np.ndarray]], width: int, k: int,
                 block_diagonal: bool = True, n_blocks: Optional[Sequence[int]] = None, add_identity: bool = False):
        self.k, self.L, self.add_identity = k, len(decomposition), add_identity
        self.n_blocks = [number_of_blocks(B, width) for B, _ in decomposition] if n_blocks is None else list(n_blocks)
        self.perms, self.to_prev, self.to_next, self.sentinel = prepare_permutations(
            [p for _, p in decomposition], self.n_blocks, width)
        self.rows = [nb * width for nb in self.n_blocks]
        self.mats = [arrow_mask(B, width, nb, block_diagonal) for (B, _), nb in zip(decomposition, self.n_blocks)]
        self.C = [np.zeros((r, k), bool) for r in self.rows]
        self.X = [np.zeros((r, k), bool) for r in self.rows]

    def set_features(self, X0: np.ndarray) -> None:
        assert X0.shape == (self.rows[0], self.k)
        self.X[0] = np.asarray(X0) != 0

    def step(self) -> np.ndarray:
        for j in range(1, self.L):
            tp = self.to_prev[j][: self.rows[j]]
            ok = tp < self.rows[j - 1]
            self.C[j][ok] = self.X[j - 1][tp[ok]]
            self.X[j] = self.C[j]
        for j in range(self.L):
            self.C[j] = spmm(self.mats[j], self.X[j])
        if self.add_identity:
            self.C[0] = self.C[0] | self.X[0]
        for j in range(self.L - 1, 0, -1):
            tp = self.to_prev[j][: self.rows[j]]
            ok = tp < self.rows[j - 1]
            self.C[j - 1][tp[ok]] |= self.C[j][ok]
            self.X[j - 1] = self.C[j - 1]
        return self.C[0]

    def bfs_levels(self, max_steps: int) -> Tuple[np.ndarray, int]:
        """hop levels from the current level-0 features (0 where set now, h where the h-th step first sets the bit, -1
        never) and the steps taken: stepping stops after the first step that sets no new bit"""
        dist = np.where(self.X[0], 0, -1).astype(np.int32)
        steps = 0
        for level in range(1, max_steps + 1):
            old = self.X[0].copy()
            new = self.step()
            steps = level
            fresh = new & ~old
            dist[fresh] = level
            if not fresh.any():
                break
        return dist, steps


def vertex_order(levels0: np.ndarray, perm0: np.ndarray, n: int, fill) -> np.ndarray:
    """[n x k] rows of level 0 in vertex order (row r of level 0 is vertex perm0[r])"""
    out = np.full((n, levels0.shape[1]), fill, dtype=levels0.dtype)
    m = min(n, perm0.size, levels0.shape[0])
    ok = perm0[:m] < n
    out[perm0[:m][ok]] = levels0[:m][ok]
    return out


def source_bits(perm0: np.ndarray, rows0: int, n: int, sources: np.ndarray) -> np.ndarray:
    """level-0 bool features of a multi-source BFS: column s is set at the row of vertex sources[s]"""
    X = np.zeros((rows0, sources.size), bool)
    inv = np.full(n, -1, dtype=np.int64)
    m = min(rows0, perm0.size)
    ok = perm0[:m] < n
    inv[perm0[:m][ok]] = np.arange(m)[ok]
    X[inv[sources], np.arange(sources.size)] = True
    return X


# ---- the tile dispatch of the (or, and) launch -------------------------------------------------------------------------
# feature widths of the GPU kernel sweep (tests/test_gpu_bool.py): both sides of the one-word boundary (32), of every
# 4-word row boundary (128) and of every (G, VPL) shape boundary of launch_tiles_bits_shape, up to the widest row (8192)
SWEEP_KS = [1, 5, 31, 32, 33, 127, 128, 129, 256, 257, 384, 512, 513, 896, 1024, 1025, 2048, 2049, 3968, 4096, 4097,
            8192]


def bits_tile_shape(k: int, big_tiles: bool = True) -> Tuple[int, int, bool]:
    """(G, VPL, big tiles) of the bit tile kernel at k columns: launch_tiles_sr_shape's choice for an fp32 row of
    words(k) columns, with at most 2 uint4 per lane; (0, 0, big) for the one-word rows of k <= 32 (a lane per row, one
    uint32 each, big tiles whenever they are on)"""
    assert 1 <= k <= 8192
    if k <= 32:
        return 0, 0, bool(big_tiles)
    k4 = words(k) // 4
    vpl = 2 if k4 >= 8 else 1
    lanes = -(-k4 // vpl)
    g = 1
    while g < lanes:
        g <<= 1
    return g, vpl, bool(big_tiles) and k4 <= 8


def source_bits_shapes(path: str) -> set:
    """the (G, VPL, big) lines of ``launch_tiles_bits_shape`` in the CUDA source"""
    import re
    with open(path) as f:
        src = f.read()
    body = src[src.index("int launch_tiles_bits_shape(arrow_ctx *ctx"):]
    body = body[:body.index("#undef BIS")]
    found = set()
    for macro, big in (("BIB", True), ("BIS", False)):
        for m in re.finditer(rf"(?<![A-Z]){macro}\((\d+),\s*(\d+)\);", body):
            found.add((int(m.group(1)), int(m.group(2)), big))
    for tr, big in (("TILE_ROWS_BIG", True), ("TILE_ROWS", False)):
        if re.search(rf"BIW\({tr},", body):
            found.add((0, 0, big))
    return found


# ---- a block whose long rows depend on every part of the long-row path ------------------------------------------------
LONG_SEGMENT = 2048      # arrow_ctx default segment of the long-row kernels (tests/tile_dispatch.py)
CTA_WARPS = 8            # warps of k_spmm_long_partial<OrAnd>: warp w takes the entries begin + w, begin + w + 8, ...


def hub_block(rng) -> sparse.csr_matrix:
    """20k rows: short ragged rows (0-23 entries), empty rows, hub rows of one to three long-row segments (513 ... 5000
    entries) and rows of 140 ... 500 entries that a lower long-row threshold moves onto the long-row path.  Every row of
    more than 24 entries reads a column range of its own, so ``problem_inputs`` can decide what each of its entries
    contributes."""
    n = 20000
    lens = rng.integers(0, 24, n)
    lens[rng.integers(0, n, 300)] = 0
    lens[[7, 9000]] = [600, 5000]
    lens[15000:15004] = [513, 2048, 2049, 4100]
    lens[[100, 3000, 6000, 12000, 18000]] = [140, 200, 300, 450, 500]
    ip = np.zeros(n + 1, np.int64)
    ip[1:] = np.cumsum(lens)
    idx = rng.integers(0, n, int(ip[-1]))
    perm, off = rng.permutation(n), 0
    for r in np.flatnonzero(lens > 24):
        idx[ip[r]:ip[r + 1]] = perm[off:off + lens[r]]
        off += lens[r]
    vals = rng.uniform(-1, 1, idx.size).astype(np.float32)
    return sparse.csr_matrix((vals, idx, ip), shape=(n, n))


def _markers(rng, s: int, e: int, img: np.ndarray) -> list:
    """one entry per long-row segment of the row [s, e) whose column image is valid: at an offset of 5 mod 8 into its
    segment (not warp 0's share) and, where the segment allows, past its first 128 entries"""
    picks = []
    for b in range(s, e, LONG_SEGMENT):
        L = min(b + LONG_SEGMENT, e) - b
        if L >= 134:
            offs = [8 * j + 5 for j in range(int(rng.integers(16, (L - 6) // 8 + 1)), -1, -1)]
        else:
            offs = list(range(L - 1, -1, -1))
        for o in offs:
            if img[b + o - s] >= 0:
                picks.append(b + o)
                break
    return picks


def problem_inputs(A: sparse.csr_matrix, k: int, seed: int, density: float = 0.05):
    """(X, addend, add_map, col_map, X for the remapped columns) of the GPU kernel tests.  Rows of more than 24 entries
    read all-zero X rows except one one-hot marker row per long-row segment (``_markers``); with k at least the number of
    markers they set distinct bits, so the last segment's bit comes from it alone; with fewer columns only the last
    segment's marker is set.  The first such row has no marker: its value is its addend row alone (forced valid and
    non-zero)."""
    rng = np.random.default_rng(seed)
    n, nc = A.shape
    X = rng.random((nc + 5, k)) < density
    n_add = n // 2 + 4
    amap = np.where(rng.random(n) < 0.6, rng.integers(0, n_add, n), -1).astype(np.int64)
    add = rng.random((n_add, k)) < density
    cmap = rng.permutation(nc + 5)[:nc].astype(np.int64)
    cmap[::5] = -1                                    # entries whose image is invalid: skipped
    Xs = rng.random((nc + 7, k)) < density
    long_rows = np.flatnonzero(np.diff(A.indptr) > 24)
    if long_rows.size:
        amap[long_rows] = rng.integers(0, n_add, long_rows.size)
        add[amap[long_rows[0]], rng.integers(k)] = True
    for Xm, cm in ((X, None), (Xs, cmap)):
        for i, r in enumerate(long_rows):
            s, e = int(A.indptr[r]), int(A.indptr[r + 1])
            img = A.indices[s:e].astype(np.int64) if cm is None else cm[A.indices[s:e]]
            Xm[img[img >= 0]] = False
            if i == 0:
                continue
            picks = _markers(rng, s, e, img)
            if k < len(picks):
                picks = picks[-1:]
            bits = rng.permutation(k)[:len(picks)]
            for q, bit in zip(picks, bits):
                Xm[img[q - s], bit] = True
    return X, add, amap, cmap, Xs


def long_row_mutants(A: sparse.csr_matrix, X: np.ndarray, add=None, add_map=None, col_map=None,
                     threshold: int = 512) -> dict:
    """rows of more than ``threshold`` entries as the correct long-row path computes them and as four faulty ones would:
    a reduce that reads only the first segment's slot, a partial that walks only warp 0's share of each segment, a reduce
    that drops the addend, a row cut after 128 entries"""
    rows = np.flatnonzero(np.diff(A.indptr) > threshold)
    X = np.asarray(X, bool)
    out = {name: np.zeros((rows.size, X.shape[1]), bool) for name in ("correct", "first slot", "warp 0", "no addend",
                                                                       "128 entries")}
    for i, r in enumerate(rows):
        s, e = int(A.indptr[r]), int(A.indptr[r + 1])
        cols = A.indices[s:e].astype(np.int64)
        if col_map is not None:
            cols = np.asarray(col_map)[cols]
        pos = np.arange(s, e)
        seg_off = (pos - s) % LONG_SEGMENT
        take = {"correct": np.ones(e - s, bool), "first slot": pos - s < LONG_SEGMENT,
                "warp 0": seg_off % CTA_WARPS == 0, "no addend": np.ones(e - s, bool), "128 entries": pos - s < 128}
        a = np.zeros(X.shape[1], bool)
        if add_map is not None and add_map[r] >= 0:
            a = np.asarray(add, bool)[add_map[r]]
        for name, t in take.items():
            c = cols[t & (cols >= 0)]
            v = X[c].any(axis=0) if c.size else np.zeros(X.shape[1], bool)
            out[name][i] = v if name == "no addend" else v | a
    return out
