"""Host restatement of the arrow step in a semiring, with ⊕ and ⊗ as parameters (test infrastructure only).

``plus_times`` computes in float64 (the exact-arithmetic yardstick of the (+, x) tests); ``min_plus`` / ``max_plus``
compute every term as ``fl32(a_p + x_p)`` in numpy float32 (round to nearest, like the device's FADD) and ⊕-reduce each
row with ``np.minimum/maximum.reduceat``.  Min and max are exact and do not depend on the order of the terms, so a
tropical device result must equal this restatement bit for bit (by value).
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np
from scipy import sparse

from oracle.oracle import arrow_mask, number_of_blocks, prepare_permutations

# name -> (⊕, ⊗, ⊕ identity, ⊗ identity, element type)
SEMIRINGS = {
    "plus_times": (np.add, np.multiply, 0.0, 1.0, np.float64),
    "min_plus": (np.minimum, np.add, np.inf, 0.0, np.float32),
    "max_plus": (np.maximum, np.add, -np.inf, 0.0, np.float32),
}
# a finite value that wins every ⊕ it enters: the canary of rows a launch must not read
WINNER = {"min_plus": np.float32(-3e38), "max_plus": np.float32(3e38)}


def plus(semiring: str):
    return SEMIRINGS[semiring][0]


def zero(semiring: str) -> float:
    return SEMIRINGS[semiring][2]


def spmm(A: sparse.csr_matrix, X: np.ndarray, semiring: str, add: Optional[np.ndarray] = None,
         add_map: Optional[np.ndarray] = None, col_map: Optional[np.ndarray] = None,
         max_terms: int = 1 << 23) -> np.ndarray:
    """C[r] = (⊕_p A[r,p] ⊗ X[col_p]) ⊕ add[add_map[r]]; ``col_map`` sends column c to col_map[c] (-1: entry skipped).
    Rows are processed in chunks of at most ``max_terms`` scalar terms (nnz x k)."""
    add_op, mul_op, z, _, dt = SEMIRINGS[semiring]
    A = sparse.csr_matrix(A)
    n, k = A.shape[0], X.shape[1]
    X = np.asarray(X, dtype=dt)
    out = np.full((n, k), z, dtype=dt)
    ip = A.indptr.astype(np.int64)
    cols = A.indices.astype(np.int64)
    if col_map is not None:
        cols = np.asarray(col_map, dtype=np.int64)[cols]
    vals = A.data.astype(dt)
    per_chunk = max(max_terms // max(k, 1), 1)
    r = 0
    while r < n:
        r2 = int(np.searchsorted(ip, ip[r] + per_chunk, side="right")) - 1
        r2 = min(max(r2, r + 1), n)
        a, b = ip[r], ip[r2]
        c = cols[a:b]
        keep = c >= 0
        rows = np.repeat(np.arange(r, r2), np.diff(ip[r:r2 + 1]))[keep]
        if rows.size:
            terms = mul_op(vals[a:b][keep][:, None], X[c[keep]])
            starts = np.flatnonzero(np.r_[True, rows[1:] != rows[:-1]])
            out[rows[starts]] = add_op.reduceat(terms, starts, axis=0)
        r = r2
    if add_map is not None:
        am = np.asarray(add_map)
        ok = am >= 0
        out[ok] = add_op(out[ok], np.asarray(add, dtype=dt)[am[ok]])
    return out


class SemiringProtocol:
    """``oracle.ReferenceProtocolOracle`` with ⊕ / ⊗ as parameters: the forward exchange moves rows, each level's
    product is fresh, the backward aggregation ⊕-adds the routed rows, and ``X`` aliases ``C`` after every exchange so
    that rows behind the sentinel keep the previous step's result.  ``zero_rhs`` fills the ⊕ identity.
    ``add_identity`` ⊕-adds level 0's features to its product (the ⊗ identity on its diagonal)."""

    def __init__(self, decomposition: Sequence[Tuple[sparse.csr_matrix, np.ndarray]], width: int, k: int, semiring: str,
                 block_diagonal: bool = True, n_blocks: Optional[Sequence[int]] = None, add_identity: bool = False):
        self.semiring, self.add_identity = semiring, add_identity
        self.plus = plus(semiring)
        dt = SEMIRINGS[semiring][4]
        self.k, self.L = k, len(decomposition)
        self.n_blocks = [number_of_blocks(B, width) for B, _ in decomposition] if n_blocks is None else list(n_blocks)
        self.perms, self.to_prev, self.to_next, self.sentinel = prepare_permutations(
            [p for _, p in decomposition], self.n_blocks, width)
        self.rows = [nb * width for nb in self.n_blocks]
        self.mats = [arrow_mask(B, width, nb, block_diagonal) for (B, _), nb in zip(decomposition, self.n_blocks)]
        self.dropped_nnz = [int(sparse.csr_matrix(B).nnz - M.nnz) for (B, _), M in zip(decomposition, self.mats)]
        self.C = [np.full((r, k), zero(semiring), dtype=dt) for r in self.rows]
        self.X = [np.full((r, k), zero(semiring), dtype=dt) for r in self.rows]

    def set_features(self, X0: np.ndarray) -> None:
        assert X0.shape == (self.rows[0], self.k)
        self.X[0] = np.array(X0, dtype=self.C[0].dtype)

    def propagate_features(self) -> None:
        for j in range(1, self.L):
            tp = self.to_prev[j][: self.rows[j]]
            ok = tp < self.rows[j - 1]
            self.C[j][ok] = self.X[j - 1][tp[ok]]
            self.X[j] = self.C[j]

    def spmm(self) -> None:
        for j in range(self.L):
            self.C[j] = spmm(self.mats[j], self.X[j], self.semiring)
        if self.add_identity:
            self.C[0] = self.plus(self.C[0], self.X[0])

    def aggregate(self) -> None:
        for j in range(self.L - 1, 0, -1):
            tp = self.to_prev[j][: self.rows[j]]
            ok = tp < self.rows[j - 1]
            self.C[j - 1][tp[ok]] = self.plus(self.C[j - 1][tp[ok]], self.C[j][ok])
            self.X[j - 1] = self.C[j - 1]

    def step(self) -> np.ndarray:
        self.propagate_features()
        self.spmm()
        self.aggregate()
        return self.C[0]


def weighted_ba_graph(n: int, m: int, seed: int, unit: bool = False) -> sparse.csr_matrix:
    """Barabasi-Albert graph with symmetric integer weights 1..16 (all 1 when ``unit``: BFS hop counts)"""
    from arrow_matrix_b200 import synth
    A = sparse.triu(synth.barabasi_albert(n, m, seed=seed), k=1).tocoo()
    w = np.ones(A.nnz, np.float32) if unit else np.random.default_rng(seed).integers(1, 17, A.nnz).astype(np.float32)
    U = sparse.coo_matrix((w, (A.row, A.col)), shape=(n, n))
    return sparse.csr_matrix(U + U.T)


def source_features(perm0: np.ndarray, rows0: int, n: int, sources: np.ndarray) -> np.ndarray:
    """level-0 features of a multi-source shortest-path run: column s is 0 at source ``sources[s]``, +inf elsewhere"""
    X = np.full((rows0, sources.size), np.inf, dtype=np.float32)
    inv = np.full(n, -1, dtype=np.int64)
    m = min(rows0, perm0.size)
    ok = perm0[:m] < n
    inv[perm0[:m][ok]] = np.arange(m)[ok]
    X[inv[sources], np.arange(sources.size)] = 0.0
    return X


def distances(C0: np.ndarray, perm0: np.ndarray, n: int) -> np.ndarray:
    """[n_sources, n] distances in vertex order from level-0 results (scipy.sparse.csgraph.shortest_path's layout)"""
    out = np.full((n, C0.shape[1]), np.inf, dtype=C0.dtype)
    m = min(n, perm0.size, C0.shape[0])
    ok = perm0[:m] < n
    out[perm0[:m][ok]] = C0[:m][ok]
    return out.T


# ---- the tile dispatch of arrow_spmm_sr ------------------------------------------------------------------------------
# feature widths of the GPU kernel sweep (tests/test_gpu_semiring.py): every tile shape, the generic kernel (k % 4 != 0,
# k > 256) and both sides of every boundary
SWEEP_KS = [1, 2, 3, 4, 5, 8, 12, 16, 20, 28, 32, 36, 64, 100, 128, 132, 256, 260, 512]


def sr_tile_shape(k: int, big_tiles: bool = True) -> Tuple[int, int, bool]:
    """(G, VPL, big tiles) of the semiring tile kernel a launch with ``k`` columns runs (``launch_tiles_sr_shape``):
    launch_tiles' choice for a plain launch with the default options"""
    assert k % 4 == 0 and 4 <= k <= 256
    k4 = k // 4
    vpl = 4 if k4 >= 32 else (2 if k4 >= 8 else 1)
    lanes = -(-k4 // vpl)
    g = 1
    while g < lanes:
        g <<= 1
    return g, vpl, bool(big_tiles) and k4 <= 8


def source_sr_shapes(path: str) -> set:
    """the (G, VPL, big) lines of ``launch_tiles_sr_shape`` in the CUDA source"""
    import re
    with open(path) as f:
        src = f.read()
    body = src[src.index("int launch_tiles_sr_shape(arrow_ctx *ctx"):]
    body = body[:body.index("#undef SRS")]
    found = set()
    for macro, big in (("SRB", True), ("SRS", False)):
        for m in re.finditer(rf"(?<![A-Z]){macro}\((\d+),\s*(\d+)\);", body):
            found.add((int(m.group(1)), int(m.group(2)), big))
    return found
