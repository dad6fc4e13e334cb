"""Single-GPU arrow SpMM engine: device-resident levels + the per-iteration step.

This is the GPU replacement for the body of ``ArrowDecompositionMPI.step()``
(``arrow/arrow_dec_mpi.py:283-307``) and ``ArrowSlimMPI._ad_spmm[_gpu]``
(``arrow/arrow_slim_mpi.py:78-244``) when one GPU holds every block-row of every level.  The
reference maps one MPI rank to one block-row and refuses to run with fewer ranks
(``arrow/arrow_bench.py:70-78``); here ranks and block-rows are decoupled.

Two execution modes, same results:

* ``exchange`` -- literal protocol: forward gather level by level, one SpMM per level, backward
  gather-add level by level.  Every level's tiles exist on the device exactly as the reference's
  ranks would hold them, including the ``X is C`` aliasing and the stale rows behind the
  sentinel (``arrow_dec_mpi.py:438, 544-545``).
* ``fused`` -- the forward permutation is folded into each level's column indices (they address
  level-0 rows directly) and the backward scatter-add into the SpMM epilogue
  (``C_0[map_j[r]] += ...``); no gather kernel runs and levels > 0 never materialise their tiles.
  Chosen automatically when no non-zero of a level reads a row behind the sentinel (then both
  modes are mathematically identical); otherwise the engine stays in ``exchange`` mode.

The precision (``dtype``, float32 or float64) is fixed at construction: the CSR values, every tile and the arithmetic
of every launch share it.

The semiring is fixed at construction too: ``plus_times`` (+, x), or the tropical ``min_plus`` / ``max_plus`` (float32),
where ⊗ is the float32 add and ⊕ is min / max.  The decomposition carries over unchanged (the operator is the ⊕ of its
levels in any semiring): the forward exchange only moves rows, the backward aggregation becomes a ⊕, and the stale rows
behind the sentinel are the same.  ``add_identity`` puts the ⊗ identity on level 0's diagonal, so that a step computes
``X ⊕ (A ⊗ X)``: the relaxation step of BFS and Bellman-Ford (``(I + A) X`` in ``plus_times``).

``or_and`` is the boolean semiring on bit tiles (one bit per element, 32 per word): ⊗ is "the entry exists" and ⊕ is
OR, so a step with ``add_identity`` is one hop of multi-source BFS / reachability.  Features go in as booleans (non-zero
is true) and come out as booleans; ``bfs_levels()`` steps to the fixed point and records the hop at which every element
was first reached.

``predecessors()`` returns, in the tropical semirings, the level-0 row each element's value came from (the parent array
of a BFS tree, the predecessor of a shortest or critical path): one more pass of the fused step over (value, label)
pairs, see DESIGN.md §4.

``max_min`` and ``min_max`` are the bottleneck semirings (float32): ⊕ and ⊗ are max and min (``max_min``, widest paths:
the largest capacity of a path, a path's capacity being its smallest edge) or min and max (``min_max``, minimax paths: the
smallest possible largest edge).  Every result is one of the operands, so no rounding enters.  ``bottleneck_tree()``
returns the fixed point with a path tree: ties are the rule in these semirings, so its parents follow the level at which
each value last changed rather than ``predecessors()``' witness rule.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from . import decomp


# the semiring's ⊕ identity (its "zero": what zero_rhs and fresh tiles hold) and ⊗ identity (what add_identity puts on
# level 0's diagonal)
_PLUS_ZERO = {_lib.SR_PLUS_TIMES: 0.0, _lib.SR_MIN_PLUS: float("inf"), _lib.SR_MAX_PLUS: float("-inf"), _lib.SR_OR_AND: 0.0,
              _lib.SR_MAX_MIN: float("-inf"), _lib.SR_MIN_MAX: float("inf")}
_TIMES_ONE = {_lib.SR_PLUS_TIMES: 1.0, _lib.SR_MIN_PLUS: 0.0, _lib.SR_MAX_PLUS: 0.0, _lib.SR_OR_AND: 1.0,
              _lib.SR_MAX_MIN: float("inf"), _lib.SR_MIN_MAX: float("-inf")}
_BOTTLENECK = (_lib.SR_MAX_MIN, _lib.SR_MIN_MAX)


# bfs_levels(): a level is a push when its frontier's edges times this are fewer than the non-zeros a pull step gathers.
# Beamer et al. (SC 2012) use 14.  Per level on an H100 80 GB HBM3 at 700 W (scripts/bfs_direction_bench.py, DESIGN.md §8)
# push and pull cross at total_nnz / frontier_edges of about 7.3 on G2 at k = 128 (pull 1.42 ms, push about 60 ps per edge
# plus the tile copy) and about 4 at k = 16; on the 10**6-vertex BA graph at k = 128 the push was faster at every level.
BFS_PUSH_ALPHA = 8


def bfs_direction(frontier_edges: int, total_nnz: int, alpha: float = BFS_PUSH_ALPHA) -> str:
    """``"push"`` when ``frontier_edges * alpha < total_nnz``, else ``"pull"``: the direction of the next BFS level"""
    return "push" if frontier_edges * alpha < total_nnz else "pull"


# iterate_to_fixed_point() in min_plus / max_plus (and max_min / min_max, whose push moves and compares as many values): a
# level is a push when its frontier's edges times this are fewer than the non-zeros a pull step gathers (bfs_direction with
# this alpha).  A tropical push moves k fp32 values per edge and
# compares each, so it costs more per edge than the bit push.  Per level on an H100 80 GB HBM3 at 700 W
# (scripts/sssp_direction_bench.py, DESIGN.md §8) push and pull cross at total_nnz / frontier_edges of about 9-10 on G2 at
# k = 128 (pull 10.8 ms, push 3.6 ms plus about 0.4 ns per edge), 7-9 at k = 16 and about 2 on the 10**6-vertex BA graph at
# k = 32.
SR_PUSH_ALPHA = 9


def semiring_code(semiring: str, dtype, fused_style: str = "gather") -> int:
    """``_lib.SR_*`` of a semiring name; raises ``ValueError`` (before any CUDA work) for an unknown name and for the
    combinations that do not exist: the tropical and boolean semirings need a float32 decomposition and run the gather
    style of the fused step."""
    if semiring not in _lib.SEMIRINGS:
        raise ValueError(f"unknown semiring {semiring!r}: expected one of {', '.join(_lib.SEMIRINGS)}")
    code = _lib.SEMIRINGS[semiring]
    if code != _lib.SR_PLUS_TIMES:
        if np.dtype(dtype) != np.float32:
            raise ValueError(f"the {semiring} semiring computes in float32, the decomposition is {np.dtype(dtype)}")
        if fused_style != "gather":
            raise ValueError(f"the {semiring} semiring runs the gather style of the fused step, not {fused_style!r}")
    return code


_SCAN_CHUNK = 1 << 24      # entries per chunk of the weight scan: bounds its host memory


def _nonpositive_edge(ip, idx, dat, cmap) -> bool:
    """some entry (r, c) of a level is an edge of the operator -- r != c (u != v: the row maps are injective) and both
    ends map to level-0 rows (``cmap``, -1 where not) -- whose weight is not > 0 (0, -0, negative or NaN).  Only the
    entries that are not > 0 get their row; the scan runs in chunks."""
    ip, idx, dat = np.asarray(ip), np.asarray(idx), np.asarray(dat)
    for e0 in range(0, dat.size, _SCAN_CHUNK):
        e = np.flatnonzero(~(dat[e0:e0 + _SCAN_CHUNK] > 0)) + e0
        if e.size == 0:
            continue
        r, c = np.searchsorted(ip, e, side="right") - 1, idx[e].astype(np.int64)
        ok = (r != c) & (c >= 0)
        if np.any(ok & (cmap[r] >= 0) & (cmap[np.where(ok, c, 0)] >= 0)):
            return True
    return False


class _LevelState:
    __slots__ = ("rows", "n_blocks", "csr", "csr_fused", "to_prev", "to_next_dev", "to_prev_dev", "cmap_dev",
                 "bufs", "xi", "ci", "nnz", "dropped", "cbuf")

    def __init__(self):
        self.csr = self.csr_fused = None
        self.to_prev = None
        self.to_prev_dev = self.to_next_dev = self.cmap_dev = None
        self.bufs = [None, None]
        self.xi = self.ci = 0
        self.cbuf = None


class ArrowEngine:
    """All levels of one decomposition resident on one GPU."""

    def __init__(self, decomposition: Sequence[Tuple[decomp.Level, np.ndarray]], width: int, k: int,
                 block_diagonal: bool = True, device: int = 0, mode: str = "auto", stream: Optional[int] = None,
                 variant: int = _lib.VARIANT_AUTO, n_blocks: Optional[Sequence[int]] = None,
                 ctx: Optional[_lib.Context] = None, fused_style: str = "gather", dtype=np.float32,
                 semiring: str = "plus_times", add_identity: bool = False):
        if mode not in ("auto", "fused", "exchange"):
            raise ValueError(f"mode must be auto|fused|exchange, got {mode!r}")
        self.dtype = _lib.element_type(dtype)
        self.sr = semiring_code(semiring, self.dtype, fused_style)
        self.semiring = semiring
        self.add_identity = bool(add_identity)
        self.ctx = ctx if ctx is not None else _lib.Context(device, stream)
        self.width, self.k, self.variant = int(width), int(k), variant
        if fused_style not in ("gather", "scatter"):
            raise ValueError("fused_style must be 'gather' or 'scatter'")
        self.fused_style = fused_style
        self.block_diagonal = block_diagonal
        self.L = len(decomposition)
        if self.L == 0:
            raise ValueError("empty decomposition")
        self.n_blocks = [decomp.number_of_blocks(B, width) for B, _ in decomposition] if n_blocks is None \
            else [int(b) for b in n_blocks]
        self.perms, self.to_prev, self.to_next, self.sentinel = decomp.prepare_permutations(
            [p for _, p in decomposition], self.n_blocks, width)
        self.levels: List[_LevelState] = []
        self._wit_labels: Optional[List[_lib.Dense]] = None     # predecessors(): int32 label tile per level (level 0: P)
        self._wit_values = {}                                    # predecessors(): value tiles of levels without a cbuf
        self._bfs_tiles: Optional[Tuple[_lib.Dense, ...]] = None   # bfs_levels(): (hop tile, all-zero and all-one bit tiles)
        self.last_bfs_steps = 0                                  # steps the last bfs_levels() call took
        self.last_bfs_directions: List[str] = []                 # "push" / "pull" per level of the last bfs_levels()
        self._adj: Optional[_lib.Adjacency] = None               # bfs_levels(): the push adjacency, built on first use
        self._in_adj: Optional[_lib.Adjacency] = None            # bfs_tree(): the in-adjacency, built on first use
        self._bfs_parents: Optional[_lib.Dense] = None           # bfs_tree(): the int32 parent tile
        self._bfs_sigma: Optional[_lib.Dense] = None            # bfs_path_counts(): the float64 path-count tile
        self._bfs_delta: Optional[Tuple[_lib.Dense, ...]] = None  # betweenness(): float64 dependencies and [n x 1] bc
        self._push_limit: Optional[int] = None                   # None: bfs_direction() decides; else push iff edges < it
        self.last_fixed_point_directions: List[str] = []         # "push" / "pull" per step of iterate_to_fixed_point()
        self._sr_adj: Optional[_lib.Adjacency] = None            # iterate_to_fixed_point(): weighted push adjacency
        self._neg_zero_weight = False                            # a -0 entry in some level: the tropical push is not exact
        self._nonpos_weight = False                              # an edge of weight not > 0: no weighted betweenness
        self._wp_adjs: Optional[Tuple[_lib.Adjacency, ...]] = None   # weighted betweenness: loop-free (in, out) lists
        self._wp_tiles: Optional[Tuple[_lib.Dense, ...]] = None      # weighted betweenness: X0, state, sigma tiles
        self._wp_delta: Optional[Tuple[_lib.Dense, ...]] = None      # weighted_betweenness(): delta and [n x 1] bc
        self.last_path_rounds = 0                                # tight-DAG rounds of the last weighted path call
        self._bt_in_adj: Optional[_lib.Adjacency] = None         # bottleneck_tree(): the loop-free in-adjacency
        self._bt_tiles: Optional[Tuple[_lib.Dense, ...]] = None  # bottleneck_tree(): int32 steps and parent tiles
        self._pr_weights: Optional[Tuple[_lib.Dense, _lib.Dense]] = None   # pagerank(): out-weights w and inverses inv
        self._pr_ops: Optional[List[_lib.Csr]] = None            # pagerank(): the scaled operand of every level (this mode)
        self._pr_work: Optional[Tuple[_lib.Dense, ...]] = None    # pagerank(): restart S, chunk scratch, state
        self._pr_refusal: Optional[str] = None                   # pagerank(): why the operator has no walk (bad weights)
        self.last_pagerank_residuals = np.zeros((0, int(k)), np.float64)   # [steps x k] of the last pagerank()
        self._cc_labels: Optional[_lib.Dense] = None             # connected_components(): int32 [n x 1] labels
        self._cc_sizes: Optional[_lib.Dense] = None              # connected_components(): int32 [n x 1] sizes
        self.last_component_count = 0                            # components found by the last connected_components()
        fused_ok = True
        cmap_prev = None                      # level j-1 row -> level-0 row (host, int64, -1 invalid)
        for j, (B, _) in enumerate(decomposition):
            st = _LevelState()
            st.n_blocks = self.n_blocks[j]
            st.rows = st.n_blocks * width
            ip, idx, dat, dropped = decomp.arrow_rows(B, width, st.n_blocks, block_diagonal, 0, st.rows, dtype=self.dtype)
            st.dropped = dropped
            entries = (ip, idx, dat)              # the level's own entries, before the identity diagonal
            if j == 0 and self.add_identity:
                ip, idx, dat = decomp.with_diagonal(ip, idx, dat, st.rows, _TIMES_ONE[self.sr], self.dtype)
            st.nnz = int(ip[-1])
            if self.sr in (_lib.SR_MIN_PLUS, _lib.SR_MAX_PLUS) and np.any((dat == 0) & np.signbit(dat)):
                self._neg_zero_weight = True
            st.csr = self.ctx.csr_upload(st.rows, st.rows, ip, idx, dat, dtype=self.dtype)
            if j > 0:
                tp = self.to_prev[j][: st.rows]
                prev_rows = self.levels[j - 1].rows
                st.to_prev = tp
                st.to_prev_dev = self.ctx.map_upload(tp, prev_rows)
                st.to_next_dev = st.to_prev_dev.invert(prev_rows)          # level j-1 row -> level j row
                valid = tp < prev_rows
                safe = np.where(valid, tp, 0)
                if j == 1:
                    cmap = np.where(valid, tp, -1)
                else:
                    cmap = np.where(valid, cmap_prev[safe], -1)
                cmap_prev = cmap
                # fused mode needs every referenced column to be routed all the way from level 0
                if np.any(cmap[idx] < 0):
                    fused_ok = False
                st.cmap_dev = self.ctx.map_upload(cmap, self.levels[0].rows)
            else:
                cmap_prev = np.arange(st.rows, dtype=np.int64)
            if self.sr == _lib.SR_MIN_PLUS and _nonpositive_edge(*entries, cmap_prev):
                self._nonpos_weight = True
            self.levels.append(st)
        if mode == "fused" and not fused_ok:
            raise ValueError("fused mode requested but a level reads rows behind the sentinel; use mode='exchange'")
        self.mode = ("fused" if fused_ok else "exchange") if mode == "auto" else mode
        self.fused_ok = fused_ok
        self._alloc_buffers()
        self.total_nnz = sum(st.nnz for st in self.levels)
        self.ctx.sync()

    # -- buffers ---------------------------------------------------------------------------------
    @property
    def bits(self) -> bool:
        """the tiles are bit tiles (``or_and``)"""
        return getattr(self, "sr", _lib.SR_PLUS_TIMES) == _lib.SR_OR_AND

    def _alloc(self, rows: int) -> _lib.Dense:
        """a feature tile holding the semiring's zero (the ⊕ identity): the engine's element type, bits in ``or_and``"""
        b = self.ctx.dense_alloc(rows, self.k, _lib.BITS if self.bits else self.dtype)
        if _PLUS_ZERO[self.sr] != 0.0:
            b.fill(_PLUS_ZERO[self.sr])
        return b

    def _alloc_buffers(self):
        for j, st in enumerate(self.levels):
            if j == 0 or self.mode == "exchange":
                st.bufs = [self._alloc(st.rows), self._alloc(st.rows)]
                st.xi, st.ci = 0, 0             # zero_rhs: X and C both zero (arrow_slim_mpi.py:354-394)
            if j > 0 and self.mode == "fused":
                st.csr_fused = st.csr.remap_columns(st.cmap_dev, self.levels[0].rows)
                if self.fused_style == "gather":
                    st.cbuf = self._alloc(st.rows)     # this level's result tile, written once per step

    def set_mode(self, mode: str):
        """Switch between 'fused' and 'exchange' (re-allocates level tiles; features are reset)."""
        if mode == self.mode:
            return
        if mode == "fused" and not self.fused_ok:
            raise ValueError("fused mode is not valid for this decomposition")
        if hasattr(self, "_slots"):                 # streaming slots hold level-0 tiles of the old mode
            self.stream_drain()
            for b in self._slots[1]:
                b.free()
            self.levels[0].bufs = list(self._slots[0])
            del self._slots
        self._free_pagerank_operands()              # they share the arrays of the blocks freed below
        for st in self.levels:
            for b in st.bufs:
                if b is not None:
                    b.free()
            st.bufs = [None, None]
            if st.csr_fused is not None:
                st.csr_fused.free()
                st.csr_fused = None
            if st.cbuf is not None:
                st.cbuf.free()
                st.cbuf = None
        self.mode = mode
        self._alloc_buffers()

    @property
    def n_rows(self) -> int:
        return self.levels[0].rows

    # -- features / results (level-0 row order, like the reference's per-rank tiles) -----------------
    def set_features(self, X: np.ndarray, sync: bool = True):
        """Level-0 feature tiles, concatenated (``B.set_features`` on every level-0 rank); in ``or_and`` non-zero is
        true."""
        st = self.levels[0]
        if X.shape != (st.rows, self.k):
            raise ValueError(f"expected features of shape {(st.rows, self.k)}, got {X.shape}")
        if st.xi == st.ci:                      # X aliases C: keep the result tile intact, like a rebind
            st.xi = 1 - st.ci
        st.bufs[st.xi].h2d(_lib.pack_bits(X) if self.bits else X)
        if sync:
            self.ctx.sync()

    def rewind_features(self):
        """Point level 0 back at the tile the last ``set_features`` filled (no copy), so the next ``step()``
        multiplies the same features again instead of chaining -- the benchmark's "fresh X every iteration"
        (``arrow_bench.py:113-116``) without a host round trip.  ``step()`` never writes that tile."""
        st = self.levels[0]
        if st.xi == st.ci:
            st.xi = 1 - st.ci

    def features_buffer(self) -> _lib.Dense:
        st = self.levels[0]
        return st.bufs[st.xi]

    def result_buffer(self, level: int = 0) -> _lib.Dense:
        st = self.levels[level]
        if st.bufs[0] is None:
            if st.cbuf is not None:             # fused/gather keeps every level's aggregated result tile
                return st.cbuf
            raise RuntimeError("level tiles are not materialised in fused/scatter mode; use mode='exchange'")
        return st.bufs[st.ci]

    def _host(self, tile: _lib.Dense, out: Optional[np.ndarray]) -> np.ndarray:
        """a feature tile on the host: as it is, or unpacked to bool [rows x k] in ``or_and``"""
        if not self.bits:
            return tile.d2h(out)
        got = _lib.unpack_bits(tile.d2h(), self.k)
        if out is None:
            return got
        out[...] = got
        return out

    def result(self, level: int = 0, out: Optional[np.ndarray] = None) -> np.ndarray:
        return self._host(self.result_buffer(level), out)

    # -- small uniform API shared with the sharded engine (used by the reference-facing classes) ----------
    def local_rows_of(self, level: int) -> int:
        return self.levels[level].rows

    def zero_rhs(self):
        """``zero_rhs`` on every rank of every level (arrow_slim_mpi.py:354-394): the semiring's zero (the ⊕ identity)."""
        for st in self.levels:
            for b in st.bufs:
                if b is not None:
                    b.fill(_PLUS_ZERO[self.sr])
            st.xi = st.ci = 0

    def features(self, level: int = 0, out: Optional[np.ndarray] = None) -> np.ndarray:
        st = self.levels[level]
        if st.bufs[st.xi] is None:
            raise RuntimeError("level tiles are not materialised in fused mode; use mode='exchange'")
        return self._host(st.bufs[st.xi], out)

    def spmm_level(self, level: int):
        """One level's arrow product on its current features (``B.spmm()`` of that level)."""
        self.ensure_level_tiles()
        st = self.levels[level]
        out = 1 - st.xi
        self._product(st.csr, st.bufs[st.xi], st.bufs[out])
        st.ci = out

    def ensure_level_tiles(self):
        """Materialise per-level tiles (exchange mode) keeping level 0's current tiles."""
        if self.mode == "exchange":
            return
        st0 = self.levels[0]
        keep = [b.d2h() for b in st0.bufs]                    # raw tiles (words in or_and)
        xi, ci = st0.xi, st0.ci
        self.set_mode("exchange")
        st0 = self.levels[0]
        for b, h in zip(st0.bufs, keep):
            b.h2d(h)
        st0.xi, st0.ci = xi, ci
        self.ctx.sync()

    def sync(self):
        if hasattr(self, "_slots"):
            self.stream_drain()
        self.ctx.sync()

    # -- the iteration ----------------------------------------------------------------------------------
    def _product(self, A: _lib.Csr, X: _lib.Dense, C: _lib.Dense, add: Optional[_lib.Dense] = None,
                 add_map: Optional[_lib.RowMap] = None):
        """C = A ⊗ X, ⊕ add[add_map] when given, in the engine's semiring ((+, x) honours the kernel variant)"""
        if self.sr != _lib.SR_PLUS_TIMES:
            self.ctx.spmm_sr(A, X, C, add, add_map, self.sr)
        elif add is None:
            self.ctx.spmm(A, X, C, variant=self.variant)
        else:
            self.ctx.spmm_add(A, X, C, add, add_map, variant=self.variant)

    def propagate_features(self):
        """Forward exchange (``_propagate_features_forwards``, arrow_dec_mpi.py:507-550)."""
        if self.mode == "fused":
            return
        for j in range(1, self.L):
            st, prev = self.levels[j], self.levels[j - 1]
            self.ctx.gather_rows(st.bufs[st.ci], prev.bufs[prev.xi], st.to_prev_dev)      # C_i[perm] = recvbuf (:544)
            st.xi = st.ci                                                                 # set_features(C_i) (:545)

    def spmm(self):
        """Every level's arrow product (``B.spmm``, arrow_slim_mpi.py:246-280 + :78-155)."""
        if self.mode == "fused":
            st0 = self.levels[0]
            x = st0.bufs[st0.xi]
            out = 1 - st0.xi
            if self.fused_style == "gather":
                # deepest level first; every level writes its tile once and ADDS the deeper level's rows that map onto
                # its own (C_j[r] += C_{j+1}[to_next_j[r]]): the reference's backward aggregation as an epilogue gather
                for j in range(self.L - 1, 0, -1):
                    st = self.levels[j]
                    if j == self.L - 1:
                        self._product(st.csr_fused, x, st.cbuf)
                    else:
                        nxt = self.levels[j + 1]
                        self._product(st.csr_fused, x, st.cbuf, nxt.cbuf, nxt.to_next_dev)
                if self.L > 1:
                    nxt = self.levels[1]
                    self._product(st0.csr, x, st0.bufs[out], nxt.cbuf, nxt.to_next_dev)
                else:
                    self._product(st0.csr, x, st0.bufs[out])
            else:
                self.ctx.spmm(st0.csr, x, st0.bufs[out], variant=self.variant)
                for st in self.levels[1:]:
                    self.ctx.spmm(st.csr_fused, x, st0.bufs[out], rowmap=st.cmap_dev, accumulate=True,
                                  variant=self.variant)
            st0.ci = out
            return
        for st in self.levels:
            out = 1 - st.xi
            self._product(st.csr, st.bufs[st.xi], st.bufs[out])                          # C_i = A @ X_i: fresh tile
            st.ci = out

    def aggregate(self):
        """Backward exchange (``_aggregate_features_backwards``, arrow_dec_mpi.py:404-440)."""
        if self.mode == "fused":
            st0 = self.levels[0]
            st0.xi = st0.ci                                                               # X := A X  (:289, :438)
            return
        for j in range(self.L - 1, 0, -1):
            st, prev = self.levels[j], self.levels[j - 1]
            # C_{j-1}[to_prev[r]] += C_j[r], written as a gather-add over level j-1 rows (to_prev is injective)
            if self.sr == _lib.SR_PLUS_TIMES:
                self.ctx.gather_rows(prev.bufs[prev.ci], st.bufs[st.ci], st.to_next_dev, accumulate=True)
            else:
                self.ctx.gather_rows_sr(prev.bufs[prev.ci], st.bufs[st.ci], st.to_next_dev, self.sr)
            prev.xi = prev.ci                                                             # set_features(C_i) (:438)

    def step(self):
        """One ``ArrowDecompositionMPI.step()``; stream-ordered, does not synchronise."""
        self.propagate_features()
        self.spmm()
        self.aggregate()

    def count_changed(self) -> int:
        """Level-0 rows in which the last ``step()`` changed the features (synchronises).  A step reads one level-0 tile
        and leaves the result in the other, in both modes, so the two tiles are compared on the device."""
        st = self.levels[0]
        return self.ctx.count_diff(st.bufs[0], st.bufs[1])

    def iterate_to_fixed_point(self, max_steps: int) -> int:
        """``step()`` until a step changes no level-0 row (BFS levels, shortest paths, reachability), at most
        ``max_steps`` times; returns the number of steps taken (the last one changed nothing unless it hit the limit).

        Direction-optimising in ``min_plus`` / ``max_plus`` with ``add_identity`` when ``fused_ok`` holds (DESIGN.md §4):
        a level is either a ``step()`` (pull) or a push of the rows whose bits changed in the previous level along the
        weighted transposed operator (built on the first call, kept until ``close()``), whichever :func:`bfs_direction`
        picks with ``SR_PUSH_ALPHA`` from the frontier's edges; ``last_fixed_point_directions`` lists the choice per
        level.  The step count and, after every level, the level-0 features (so ``result()``, ``features()``,
        ``count_changed()``, ``predecessors()`` and the next ``step()``) are bit-identical to pull steps only.  After a
        push level the tiles of the levels ``j >= 1`` (``result(j)``) are not that level's product; the next ``step()``
        rewrites them.  The same holds in ``max_min`` / ``min_max``, -0 weights included; there the loop stops when a step
        changes no level-0 row in bits, since their order puts -0 below +0 (a step that only turns -0 into +0 is
        progress).  Every other engine, and a tropical one with a -0 weight, pulls every level."""
        adj = self._sr_push_adjacency() if self._sr_push_ok() and int(max_steps) >= 1 else None
        if adj is None:
            st0 = self.levels[0]
            for n in range(1, int(max_steps) + 1):
                self.step()
                changed = self.ctx.count_diff_bits(st0.bufs[0], st0.bufs[1]) if self.sr in _BOTTLENECK \
                    else self.count_changed()
                if changed == 0:
                    self.last_fixed_point_directions = ["pull"] * n
                    return n
            self.last_fixed_point_directions = ["pull"] * max(int(max_steps), 0)
            return int(max_steps)
        return self._marked_fixed_point(max_steps, adj, True)

    def _marked_fixed_point(self, max_steps: int, adj: _lib.Adjacency, pushes: bool,
                            steps: Optional[_lib.Dense] = None) -> int:
        """the direction-optimising loop of ``iterate_to_fixed_point`` on the weighted push adjacency ``adj``; every level
        is a pull unless ``pushes``.  With ``steps`` (int32) the mark pass after level h also writes h where the level
        changed an element's bits (0 everywhere after level 0): T of ``bottleneck_tree``."""
        st0 = self.levels[0]
        limit = self._push_limit

        def mark(new, old, level):
            """(rows changed, push next): the stop test -- rows changed by value, in bits in the bottleneck semirings --
            and the direction of the next level"""
            if steps is None:
                changed, rows, edges = self.ctx.sr_mark_frontier(adj, new, old)
            else:
                changed, rows, edges = self.ctx.sr_mark_frontier_steps(adj, new, old, steps, level)
            if self.sr in _BOTTLENECK:
                changed = rows
            if not pushes:
                return changed, False
            push = edges < limit if limit is not None else bfs_direction(edges, self.total_nnz, SR_PUSH_ALPHA) == "push"
            return changed, push

        # X_{-1} is the ⊕ identity: the first frontier is every row holding something else.  The tile that the first level
        # writes holds it meanwhile.
        xi = st0.xi
        st0.bufs[1 - xi].fill(_PLUS_ZERO[self.sr])
        _, push = mark(st0.bufs[xi], st0.bufs[1 - xi], 0)
        directions = []
        for n in range(1, int(max_steps) + 1):
            xi = st0.xi
            if push:                             # canon(X_h) ⊕ the frontier rows' relaxations
                self.ctx.sr_push_frontier(adj, st0.bufs[xi], st0.bufs[1 - xi], self.sr)
                st0.xi = st0.ci = 1 - xi
            else:
                self.step()                      # reads bufs[xi], leaves the result in bufs[1 - xi]
            directions.append("push" if push else "pull")
            changed, push = mark(st0.bufs[1 - xi], st0.bufs[xi], n)
            if changed == 0:
                self.last_fixed_point_directions = directions
                return n
        self.last_fixed_point_directions = directions
        return int(max_steps)

    def _sr_push_ok(self) -> bool:
        """iterate_to_fixed_point() may push: a tropical engine without a -0 weight or a bottleneck engine, with the
        identity, every non-zero behind a level-0 row, and a step that advances level 0's features (an exchange-mode step
        of one level does not)"""
        return ((self.sr in (_lib.SR_MIN_PLUS, _lib.SR_MAX_PLUS) and not self._neg_zero_weight or self.sr in _BOTTLENECK)
                and self.add_identity and self.fused_ok and (self.mode == "fused" or self.L > 1))

    def _sr_push_adjacency(self) -> _lib.Adjacency:
        """the weighted transposed operator of the fused step with the identity (built on the first call): every level's
        own block with its level-j -> level-0 row map (level 0: the identity, its diagonal included)"""
        if self._sr_adj is None:
            parts = [(st.csr, st.cmap_dev) for st in self.levels]
            self._sr_adj = self.ctx.adj_build(parts, self.levels[0].rows, weighted=True)
        return self._sr_adj

    # -- predecessors (min_plus / max_plus) ----------------------------------------------------------------------
    def predecessors(self, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Parents of the current level-0 features ``D`` (int32 [n x k], level-0 row order like ``result()``): ``P[v, s]``
        is the level-0 row ``u`` of the witness of ``(v, s)`` -- the lexicographic ⊕ of the terms ``fl(a + D[u, s])`` the
        fused step reduces into row ``v`` at any level, with ``u != v``, ties to the smallest ``u`` -- where ``D[v, s]``
        is not the ⊕ identity and equals the witness value; ``-1`` elsewhere (sources, unreachable vertices).  At a fixed
        point of the step with ``add_identity`` every vertex whose value came from an edge has a parent.  Synchronises.

        One pass over the levels, deepest first, on the column-remapped level matrices of the fused step (built on the
        first call and kept in exchange mode); value tiles are the levels' ``cbuf`` in fused mode (so ``result(j)`` for
        ``j >= 1`` is overwritten there), label tiles are allocated on the first call.  Features, results of level 0,
        the exchange-mode level tiles and the streaming slots are not touched: the next ``step()`` is the same.
        Raises ``ValueError`` in ``plus_times`` and when a level reads rows behind the sentinel (``fused_ok`` is false:
        such a row has no vertex identity)."""
        if self.sr == _lib.SR_PLUS_TIMES:
            raise ValueError("predecessors exist in the min_plus / max_plus semirings only, the engine runs plus_times")
        if self.sr == _lib.SR_OR_AND:
            raise ValueError("predecessors exist in the min_plus / max_plus semirings only, the engine runs or_and")
        if self.sr in _BOTTLENECK:
            raise ValueError(f"predecessors' witness rule makes cycles in the {self.semiring} semiring, where ties are the "
                             "rule: use bottleneck_tree()")
        if not self.fused_ok:
            raise ValueError("predecessors need a level-0 row behind every non-zero, but a level reads rows behind the "
                             "sentinel")
        self.sync()
        return self._predecessor_pass().d2h(out)

    def _predecessor_pass(self) -> _lib.Dense:
        """enqueue the launches of ``predecessors()`` (stream-ordered); returns the level-0 label tile holding P"""
        st0 = self.levels[0]
        x = st0.bufs[st0.xi]
        if self._wit_labels is None:
            self._wit_labels = [self.ctx.dense_alloc(st.rows, self.k, np.int32) for st in self.levels]
        values = {}
        for j in range(self.L - 1, 0, -1):
            st = self.levels[j]
            if st.csr_fused is None:                  # exchange mode: the remapped copy of the fused step, kept
                st.csr_fused = st.csr.remap_columns(st.cmap_dev, st0.rows)
            if st.cbuf is not None:
                values[j] = st.cbuf
            else:
                if j not in self._wit_values:
                    self._wit_values[j] = self.ctx.dense_alloc(st.rows, self.k)
                values[j] = self._wit_values[j]
            add = {}
            if j + 1 < self.L:
                nxt = self.levels[j + 1]
                add = dict(add_values=values[j + 1], add_labels=self._wit_labels[j + 1], add_map=nxt.to_next_dev)
            self.ctx.spmm_sr_witness(st.csr_fused, x, self._wit_labels[j], values[j], row_labels=st.cmap_dev,
                                     semiring=self.sr, **add)
        add = {}
        if self.L > 1:
            nxt = self.levels[1]
            add = dict(add_values=values[1], add_labels=self._wit_labels[1], add_map=nxt.to_next_dev)
        self.ctx.spmm_sr_witness(st0.csr, x, self._wit_labels[0], dist=x, semiring=self.sr, **add)
        return self._wit_labels[0]

    # -- bottleneck path trees (max_min / min_max) ------------------------------------------------------------------
    def bottleneck_tree(self, max_steps: int, distances_out: Optional[np.ndarray] = None,
                        parents_out: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
        """``iterate_to_fixed_point(max_steps)`` that also returns a path tree of the fixed point reached (``D`` float32
        and ``P`` int32, both [n x k] in level-0 row order like ``result()``).  ``D[v, s]`` is the widest (``max_min``)
        or minimax (``min_max``) value from the sources of column ``s``.  Let ``T[v, s]`` be the level at which the loop
        last changed the element's bits (0 if never).  ``P[v, s]`` is -1 where ``T[v, s] == 0`` (the sources) or
        ``D[v, s]`` is the ⊕ identity (not reached).  Otherwise it is the smallest level-0 row ``u != v`` with an entry
        ``u -> v`` of weight ``a`` of the fused step's operator such that ``a ⊗ D[u, s] == D[v, s]`` in bits and either
        ``D[u, s]`` is strictly better than ``D[v, s]`` in the ⊕ order or the two are equal and ``T[u, s] < T[v, s]``;
        -1 when there is none.  Along every parent edge ``D`` strictly improves or ``T`` strictly drops, so ``P`` has no
        cycles, and at a fixed point every element with ``T > 0`` that is reached has a parent (DESIGN.md §4), with the
        NaN exceptions below.  The loop stops after a level that changes no row in bits.  ``max_steps`` may stop it
        early, which can leave such elements at -1.  ⊕ and ⊗ drop a NaN operand: a NaN weight passes the feature
        through, and a NaN feature becomes the ⊗ identity at the first level (a source whose ``T`` is 1); an element that
        the first level gives the ⊗ identity through an edge of weight ⊗ identity from a NaN feature has no parent either.
        -0 orders below +0 everywhere.

        The step count, ``last_fixed_point_directions`` and the features are those of ``iterate_to_fixed_point``; the
        mark pass after each level also writes ``T``, and one pass over the in-lists then finds the parents.  An engine
        that does not push (exchange mode with one level) still builds the weighted push adjacency for the frontier record
        and pulls every level.  The loop-free in-adjacency (8 bytes per edge) and the int32 ``T`` and parent tiles (4
        bytes per element each: 5.1 GB apiece at 10M rows and k = 128, beside the two feature tiles and the weighted push
        adjacency) are made on the first call and kept until ``close()``.  Raises ``ValueError`` before any CUDA work for
        another semiring, ``add_identity=False``, and when a level reads rows behind the sentinel (``fused_ok`` is false:
        such a row has no vertex identity).  Synchronises."""
        D, P = self._bottleneck_tree_run(max_steps)
        return D.d2h(distances_out), P.d2h(parents_out)

    def _bottleneck_tree_run(self, max_steps: int) -> Tuple[_lib.Dense, _lib.Dense]:
        """the device part of ``bottleneck_tree``: the level-0 feature tile holding D and the int32 parent tile"""
        self._bottleneck_checks("bottleneck_tree")
        self.sync()
        st0 = self.levels[0]
        if self._bt_in_adj is None:
            parts = [(st.csr, st.cmap_dev) for st in self.levels]
            self._bt_in_adj = self.ctx.adj_build_loopfree(parts, st0.rows, direction="in")
        if self._bt_tiles is None:
            self._bt_tiles = (self.ctx.dense_alloc(st0.rows, self.k, np.int32),
                              self.ctx.dense_alloc(st0.rows, self.k, np.int32))
        steps, parents = self._bt_tiles
        self._marked_fixed_point(max_steps, self._sr_push_adjacency(), self._sr_push_ok(), steps)
        D = self.result_buffer(0)
        self.ctx.sr_tree_parents(self._bt_in_adj, D, steps, parents, self.sr)
        return D, parents

    def _bottleneck_checks(self, what: str):
        if self.sr not in _BOTTLENECK:
            raise ValueError(f"{what} runs the max_min / min_max semirings, the engine runs {self.semiring}")
        if not self.add_identity:
            raise ValueError(f"{what} needs add_identity=True: a step must keep the values it already has")
        if not self.fused_ok:
            raise ValueError(f"{what} needs a level-0 row behind every non-zero, but a level reads rows behind the "
                             "sentinel")

    # -- personalized PageRank (plus_times) --------------------------------------------------------------------------
    def pagerank(self, max_steps: int, alpha: float = 0.85, tol: float = 1e-6, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Personalized PageRank (random walk with restart) from the current level-0 features, one restart distribution
        per column; returns ``p`` (the engine's dtype ``T``, [n x k] in level-0 row order like ``result()``).

        ``M`` is the operator ``step()`` applies (with the identity diagonal when ``add_identity``): entry ``(r, c)`` of
        level ``j`` with value ``a`` is the edge ``cmap_j(c) -> cmap_j(r)``, duplicates counted separately.  ``w[u]`` is
        the float64 sum of the values of the edges leaving ``u`` (levels ascending, then entry order), ``u`` is dangling
        when ``w[u] == 0`` and ``inv[u] = fl_T(1 / w[u])`` (0 when dangling).  The walk steps on ``M^``, ``M`` with each
        entry ``fl_T(a * inv[u])``.  The restart is ``S[:, s] = fl_T(X0[:, s] / sigma_s)``, ``sigma_s`` the column sum of
        the features.  From ``p_0 = S`` every step computes ``Y = M^ p_t`` through the engine's own route, the dangling
        mass ``m_t[s]``, ``c_t[s] = fl(fl(1 - alpha) + fl(alpha * m_t[s]))`` and ``p_{t+1} = fl_T(fl(fl(alpha * Y) +
        fl(c_t * S)))``: dangling mass returns through the restart.  The loop stops after the first step whose largest
        residual ``r[s] = sum_v |p_{t+1}[v, s] - p_t[v, s]|`` is ``<= tol``, or after ``max_steps`` steps
        (``max_steps = 0`` returns ``S``); ``last_pagerank_residuals`` (float64 [steps x k]) holds every step's
        residuals.  Every column reduction runs in float64 over fixed 512-row chunks (DESIGN.md §4), so two calls give
        the same bits.  At the fixed point ``||p - p*||_1 <= alpha / (1 - alpha) * r`` per column.

        The out-weights (12 or 16 bytes per row) and the scaled values of every level's operand (4 or 8 bytes per entry)
        are built on the first call and kept until ``close()`` or a mode change; ``S`` (one tile), the chunk scratch (16 k
        bytes per 512 rows) and the state are allocated on first use.  Afterwards the level-0 features are ``p``:
        ``result()`` and ``features()`` return it and the next ``step()`` multiplies it by ``M``; the tiles of the levels
        ``j >= 1`` are unspecified.  Raises ``ValueError`` before any CUDA work outside ``plus_times``, when a level reads
        rows behind the sentinel, for ``alpha`` outside ``[0, 1)``, a negative or NaN ``tol``, a negative ``max_steps``
        and an ``out`` that is not a C-contiguous ``T`` array of shape [n x k]; after the out-weight pass for an edge
        whose weight is negative, NaN or +-inf, or a non-dangling vertex whose inverse is not finite (remembered: later
        calls refuse at once); after the restart pass, with the features unchanged, for a column holding a negative,
        NaN or +-inf value or summing to 0.  Synchronises."""
        max_steps = self._pagerank_checks(max_steps, alpha, tol, out)
        S, scratch, state = self._pagerank_prepare()
        st0 = self.levels[0]
        x = st0.bufs[st0.xi]
        inv = self._pr_weights[1]
        sums, bad, first = self.ctx.pagerank_restart(x, inv, S, scratch, state)
        if bad:
            raise ValueError(f"pagerank needs every restart column non-negative and finite with a positive sum: column "
                             f"{first} is not ({bad} such column(s)); sum {sums[first]!r}")
        x.copy_from(S)
        residuals = []
        for _ in range(max_steps):
            p_tile = self._pagerank_step()
            res = self.ctx.pagerank_update(st0.bufs[st0.xi], p_tile, S, inv, scratch, state, alpha)
            residuals.append(res)
            if res.max(initial=0.0) <= tol:
                break
        self.last_pagerank_residuals = np.array(residuals, np.float64).reshape(len(residuals), self.k)
        return st0.bufs[st0.xi].d2h(out)

    def _pagerank_checks(self, max_steps, alpha, tol, out) -> int:
        if self.sr != _lib.SR_PLUS_TIMES:
            raise ValueError(f"pagerank runs the plus_times semiring, the engine runs {self.semiring}")
        if not self.fused_ok:
            raise ValueError("pagerank needs a level-0 row behind every non-zero, but a level reads rows behind the sentinel")
        alpha, tol = float(alpha), float(tol)
        if not (0.0 <= alpha < 1.0):
            raise ValueError(f"alpha must lie in [0, 1), got {alpha!r}")
        if not (tol >= 0.0):
            raise ValueError(f"tol must be >= 0, got {tol!r}")
        if int(max_steps) != max_steps or int(max_steps) < 0:
            raise ValueError(f"max_steps must be a non-negative integer, got {max_steps!r}")
        shape = (self.levels[0].rows, self.k)
        if out is not None and (not isinstance(out, np.ndarray) or out.dtype != self.dtype or out.shape != shape
                                or not out.flags.c_contiguous):
            raise ValueError(f"out must be a C-contiguous {self.dtype} array of shape {shape}")
        if self._pr_refusal is not None:
            raise ValueError(self._pr_refusal)
        return int(max_steps)

    def _pagerank_prepare(self) -> Tuple[_lib.Dense, _lib.Dense, _lib.Dense]:
        """the out-weights, the scaled operands of the current mode and the work tiles, made where missing"""
        self.sync()
        st0 = self.levels[0]
        n = st0.rows
        if self._pr_weights is None:
            w, inv = self.ctx.dense_alloc(n, 1, np.float64), self.ctx.dense_alloc(n, 1, self.dtype)
            self._pr_weights = (w, inv)
            bad, _, bad_inv = self.ctx.out_weights([(st.csr, st.cmap_dev) for st in self.levels], n, w, inv)
            if bad:
                self._pr_refusal = (f"pagerank needs every edge weight non-negative and finite: {bad} edge(s) of the operator "
                                    "have a negative, NaN or infinite weight")
            elif bad_inv:
                self._pr_refusal = (f"pagerank needs a finite non-zero 1 / w for every vertex with out-weight w != 0: "
                                    f"{bad_inv} vertex(es) have none in {self.dtype}")
            if self._pr_refusal is not None:
                raise ValueError(self._pr_refusal)
        inv = self._pr_weights[1]
        if self._pr_ops is None:
            ops = [st0.csr.scale_columns(inv)]
            for st in self.levels[1:]:
                ops.append(st.csr_fused.scale_columns(inv) if self.mode == "fused" else st.csr.scale_columns(inv, st.cmap_dev))
            self._pr_ops = ops
        if self._pr_work is None:
            chunks = (n + 511) // 512
            self._pr_work = (self.ctx.dense_alloc(n, self.k, self.dtype), self.ctx.dense_alloc(chunks, 2 * self.k, np.float64),
                             self.ctx.dense_alloc(4, self.k, np.float64))
        return self._pr_work

    def _pagerank_step(self) -> _lib.Dense:
        """one ``step()`` on the scaled operands; returns the tile it read (p_t), level 0's features then being Y"""
        st0 = self.levels[0]
        p_tile = st0.bufs[st0.xi]
        attr = "csr_fused" if self.mode == "fused" else "csr"
        kept = [st0.csr] + [getattr(st, attr) for st in self.levels[1:]]
        try:
            st0.csr = self._pr_ops[0]
            for st, op in zip(self.levels[1:], self._pr_ops[1:]):
                setattr(st, attr, op)
            self.step()
        finally:
            st0.csr = kept[0]
            for st, op in zip(self.levels[1:], kept[1:]):
                setattr(st, attr, op)
        st0.xi = st0.ci                      # an exchange-mode step of one level leaves xi where it was
        return p_tile

    def _free_pagerank_operands(self):
        for op in self._pr_ops or ():
            op.free()
        self._pr_ops = None

    # -- connected components (any semiring) ------------------------------------------------------------------------
    def connected_components(self, out: Optional[np.ndarray] = None,
                             sizes_out: Optional[np.ndarray] = None) -> np.ndarray:
        """Weakly connected components of the operator ``step()`` applies: int32 ``labels[v]`` (``[n]``, level-0 row
        order like ``result()``) is the smallest level-0 row in ``v``'s component; ``last_component_count`` receives the
        number of components (the ``v`` with ``labels[v] == v``) and ``sizes_out`` (int32 ``[n]``), when given, the
        member count of the component labelled ``r`` at row ``r`` and 0 at the rows that are not labels.

        The vertices are the level-0 rows, padding rows included (they are singletons unless an entry names them).
        Every entry ``(r, c)`` of level ``j`` as the step applies it (the arrow pattern, and the identity diagonal when
        ``add_identity``) gives the undirected edge ``cmap_j(c) -- cmap_j(r)`` whatever its value (0, NaN and +-inf
        included); ``u == v`` gives none.  The answer is unique, so it is bit-identical on every route, semiring, dtype,
        ``k`` and grid.  One device pass of a lock-free union-find over the level blocks and the row maps the engine
        keeps (DESIGN.md §4): no adjacency is built and nothing is sorted.

        The label tile (4 bytes per row; another 4 with ``sizes_out``) is allocated on the first call and kept until
        ``close()``.  Features, results and the next ``step()`` are untouched.  Raises ``ValueError`` before any CUDA
        work when a level reads rows behind the sentinel (``fused_ok`` is false: such a row has no vertex identity) and
        for an ``out`` or ``sizes_out`` that is not a C-contiguous int32 array of shape ``[n]``.  Synchronises."""
        if not self.fused_ok:
            raise ValueError("connected_components needs a level-0 row behind every non-zero, but a level reads rows "
                             "behind the sentinel")
        n = self.levels[0].rows
        for name, arr in (("out", out), ("sizes_out", sizes_out)):
            if arr is not None and (not isinstance(arr, np.ndarray) or arr.dtype != np.int32 or arr.shape != (n,)
                                    or not arr.flags.c_contiguous):
                raise ValueError(f"{name} must be a C-contiguous int32 array of shape {(n,)}")
        if self._cc_labels is None:
            self._cc_labels = self.ctx.dense_alloc(n, 1, np.int32)
        if sizes_out is not None and self._cc_sizes is None:
            self._cc_sizes = self.ctx.dense_alloc(n, 1, np.int32)
        sizes = self._cc_sizes if sizes_out is not None else None
        self.last_component_count = self.ctx.connected_components([(st.csr, st.cmap_dev) for st in self.levels], n,
                                                                  self._cc_labels, sizes)
        if sizes is not None:
            sizes.d2h(sizes_out[:, None])           # a view of sizes_out: the rows land in it
        if out is None:
            return self._cc_labels.d2h().reshape(-1)
        self._cc_labels.d2h(out[:, None])
        return out

    # -- multi-source BFS (or_and) ----------------------------------------------------------------------------------
    def bfs_levels(self, max_steps: int, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Hop levels of a multi-source BFS from the current level-0 features (int32 [n x k], level-0 row order like
        ``result()``): ``0`` where a feature bit is set now (the sources), ``h`` where the bit was first set by the
        ``h``-th level, ``-1`` where it is never set.  Takes levels until one sets no new bit, at most ``max_steps``;
        ``last_bfs_steps`` holds the number taken.  After every level one device pass records the fresh bits and counts
        them: the level record and the fixed-point test at once.  Needs ``or_and`` with ``add_identity`` (bits then only
        grow); raises ``ValueError`` before any CUDA work otherwise.  The features end at the fixed point (``result()``);
        synchronises.

        Direction-optimising (DESIGN.md §4): when ``fused_ok`` holds, a level is either a ``step()`` (pull) or a push of
        the rows that gained a bit in the previous level along the transposed operator (built on the first call, kept
        until ``close()``), whichever :func:`bfs_direction` picks from the frontier's edges; ``last_bfs_directions`` lists
        the choice per level.  The levels, ``last_bfs_steps``, ``result()`` / ``features()`` of level 0 and the next
        ``step()``'s level-0 result are bit-identical to a run of pull steps only.  After a push level the tiles of the
        levels ``j >= 1`` (``result(j)``) are not that level's product; the next ``step()`` rewrites them."""
        return self._bfs_run(max_steps).d2h(out)

    def bfs_tree(self, max_steps: int, levels_out: Optional[np.ndarray] = None,
                 parents_out: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
        """``bfs_levels`` that also returns the BFS parents (both int32 [n x k], level-0 row order like ``result()``):
        ``P[v, s]`` is the smallest level-0 row ``u`` with an edge ``u -> v`` of the fused step's operator (``u != v``)
        whose level is ``L[v, s] - 1``, where ``L[v, s] > 0``; ``-1`` for the sources and for elements not reached
        (within ``max_steps``).  On unit weights this is what ``predecessors()`` gives after ``iterate_to_fixed_point()``
        on a ``min_plus`` engine with ``add_identity``.  The levels, ``last_bfs_steps``, ``last_bfs_directions`` and the
        features are those of ``bfs_levels``.

        After each level's record one more device pass searches the in-lists of the rows that gained a bit, in ascending
        ``u``, for the first source row holding the bit one level earlier (DESIGN.md §4).  The in-adjacency is built on
        the first call and kept until ``close()``; an engine that does not push (exchange mode with one level) builds the
        push adjacency for the frontier record and still pulls every level.  Raises ``ValueError`` before any CUDA work
        outside ``or_and`` with ``add_identity``, and when a level reads rows behind the sentinel (``fused_ok`` is false:
        such a row has no vertex identity).  Synchronises."""
        self._bfs_checks("bfs_tree")
        if not self.fused_ok:
            raise ValueError("bfs_tree needs a level-0 row behind every non-zero, but a level reads rows behind the "
                             "sentinel")
        dist, parents = self._bfs_tree_run(max_steps)
        return dist.d2h(levels_out), parents.d2h(parents_out)

    def _bfs_tree_run(self, max_steps: int) -> Tuple[_lib.Dense, _lib.Dense]:
        """the device part of ``bfs_tree``: the int32 level and parent tiles, left on the device"""
        if self._in_adj is None:
            parts = [(st.csr, st.cmap_dev) for st in self.levels]
            self._in_adj = self.ctx.adj_build(parts, self.levels[0].rows, direction="in")
        if self._bfs_parents is None:
            self._bfs_parents = self.ctx.dense_alloc(self.levels[0].rows, self.k, np.int32)
        return self._bfs_run(max_steps, self._bfs_parents), self._bfs_parents

    def bfs_path_counts(self, max_steps: int, levels_out: Optional[np.ndarray] = None,
                        counts_out: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
        """``bfs_levels`` that also returns the shortest-path counts (levels int32, counts float64, both [n x k] in
        level-0 row order like ``result()``): ``sigma[v, s]`` is 1 where ``L[v, s] = 0``, 0 where ``L[v, s] = -1``, and
        otherwise the sum of ``sigma[u, s]`` over the distinct edges ``u -> v`` of the fused step's operator (``u != v``)
        with ``L[u, s] = L[v, s] - 1``.  A column with several sources counts paths from any of them.  The sums run in
        ascending ``u``, 512 in-list entries at a time, the partials added in order (DESIGN.md §4): the counts are exact
        below 2^53 and bit-reproducible beyond.  The levels, ``last_bfs_steps``, ``last_bfs_directions`` and the features
        are those of ``bfs_levels``.

        After each level's record one more device pass sums the in-lists of the rows that gained a bit.  The in-adjacency
        and the float64 count tile (8 bytes per element: 10.2 GB at 10M rows and k = 128, beside the 5.1 GB level tile)
        are made on the first call and kept until ``close()``.  Raises ``ValueError`` before any CUDA work where
        ``bfs_tree`` does.  Synchronises."""
        dist, sigma = self._bfs_paths_run(max_steps, "bfs_path_counts")
        return dist.d2h(levels_out), sigma.d2h(counts_out)

    def betweenness(self, max_steps: int, out: Optional[np.ndarray] = None,
                    dependencies_out: Optional[np.ndarray] = None) -> np.ndarray:
        """Brandes betweenness over the engine's ``k`` source columns: float64 ``bc[v] = sum over s < k of delta[v, s]``,
        in level-0 row order like ``result()``, summed in column order.  ``delta[v, s]`` is 0 where ``L[v, s] <= 0``, and
        otherwise ``sigma[v, s]`` (``bfs_path_counts``) times the sum of ``fl((1 + delta[w, s]) / sigma[w, s])`` over the
        distinct edges ``v -> w`` with ``L[w, s] = L[v, s] + 1`` (0 at the last level and at ``max_steps``), summed in
        ascending ``w`` like the counts.  With one source per column this is the unnormalised betweenness restricted to
        those sources, counting ordered pairs ``(s, t)``: twice networkx's undirected figure on a symmetric operator.
        ``dependencies_out`` (float64 [n x k]) receives ``delta``.  Levels run as in ``bfs_levels``
        (``last_bfs_steps``, ``last_bfs_directions``).

        The forward part is ``bfs_path_counts`` keeping each level's frontier rows (4 bytes per row and level in which
        it gained a bit); the backward sweep then visits, from the deepest level to 1, only that level's rows along the
        push adjacency's out-lists, and one pass sums each row.  The dependency tile (8 bytes per element, as the count
        tile) is allocated on the first call and kept until ``close()``.  Raises ``ValueError`` before any CUDA work where
        ``bfs_tree`` does.  Synchronises."""
        self._paths_checks("betweenness")
        self._check_bc_outputs(out, dependencies_out)
        delta, bc = self._betweenness_run(max_steps)
        if dependencies_out is not None:
            delta.d2h(dependencies_out)
        if out is None:
            return bc.d2h().reshape(-1)
        bc.d2h(out[:, None])                    # a view of out: the rows land in it
        return out

    def _betweenness_run(self, max_steps: int) -> Tuple[_lib.Dense, _lib.Dense]:
        """the device part of ``betweenness``: the float64 dependency and [n x 1] betweenness tiles, left on the device"""
        dist, sigma = self._bfs_paths_run(max_steps, "betweenness")
        if self._bfs_delta is None:
            n = self.levels[0].rows
            self._bfs_delta = (self.ctx.dense_alloc(n, self.k, np.float64), self.ctx.dense_alloc(n, 1, np.float64))
        delta, bc = self._bfs_delta
        delta.fill(0.0)
        for level in range(self.last_bfs_steps, 0, -1):
            self.ctx.bits_dependencies(self._adj, level, dist, sigma, delta)
        self.ctx.row_sum(delta, bc)
        return delta, bc

    def _bfs_paths_run(self, max_steps: int, what: str) -> Tuple[_lib.Dense, _lib.Dense]:
        """the device part of ``bfs_path_counts``: the int32 level and float64 count tiles, left on the device, with the
        frontier rows of levels 0 .. ``last_bfs_steps`` kept in the push adjacency's history"""
        self._paths_checks(what)
        if self._in_adj is None:
            parts = [(st.csr, st.cmap_dev) for st in self.levels]
            self._in_adj = self.ctx.adj_build(parts, self.levels[0].rows, direction="in")
        if self._bfs_sigma is None:
            self._bfs_sigma = self.ctx.dense_alloc(self.levels[0].rows, self.k, np.float64)
        return self._bfs_run(max_steps, sigma=self._bfs_sigma), self._bfs_sigma

    # -- weighted betweenness (min_plus) ---------------------------------------------------------------------------
    def shortest_path_counts(self, max_steps: int, distances_out: Optional[np.ndarray] = None,
                             counts_out: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
        """``iterate_to_fixed_point(max_steps)`` that also returns the number of shortest paths to every element (``D``
        float32 and ``sigma`` float64, both [n x k] in level-0 row order like ``result()``).  An entry ``u -> v`` of weight
        ``a`` of the fused step's operator (``u != v``) is *tight* in column ``s`` when ``D[u, s] < D[v, s] < +inf`` and
        ``fl(a + D[u, s]) == D[v, s]`` (so a ``+inf`` weight or an overflowing sum never counts); a pair ``(u, v)`` is tight when one of its entries is.  The sources ``S_s`` are the
        ``v`` with ``D[v, s]`` finite and equal to the features the call started from (the 0 / +inf start, or any offsets:
        a column with several sources acts as one super-source).  ``sigma[v, s]`` is 0 where ``D[v, s]`` is not finite,
        otherwise ``[v in S_s]`` plus the sum of ``sigma[u, s]`` over the distinct tight pairs ``u -> v``, in ascending
        ``u``, 512 in-list entries at a time, the partials added in order (DESIGN.md §4): exact below 2^53 and
        bit-reproducible beyond.  On unit weights from 0 / +inf features this is ``bfs_path_counts`` bit for bit.  When
        ``max_steps`` stops the loop before the fixed point, everything is defined on the ``D`` reached.  The step count
        and ``last_fixed_point_directions`` are those of ``iterate_to_fixed_point``, the features end at ``D``, and
        ``last_path_rounds`` holds the rounds of the tight-pair DAG.

        The loop-free weighted in- and out-adjacencies (8 bytes per edge each) and the tiles (the starting features 4,
        the round state 4 and the counts 8 bytes per element: 20.5 GB at 10M rows and k = 128, beside the two 5.1 GB
        feature tiles) are made on the first call and kept until ``close()``.  Needs ``min_plus`` with ``add_identity``,
        a level-0 row behind every non-zero and every edge's weight ``> 0`` (an edge: an off-diagonal entry with both
        ends routed; ``+inf`` is allowed); raises ``ValueError`` before any CUDA work otherwise.  Synchronises."""
        D, sigma = self._wpaths_run(max_steps, "shortest_path_counts")
        return D.d2h(distances_out), sigma.d2h(counts_out)

    def weighted_betweenness(self, max_steps: int, out: Optional[np.ndarray] = None,
                             dependencies_out: Optional[np.ndarray] = None) -> np.ndarray:
        """Brandes betweenness over the weighted shortest paths from the engine's ``k`` source columns: float64
        ``bc[v] = sum over s < k of delta[v, s]`` in level-0 row order, summed in column order.  ``delta[v, s]`` is 0
        where ``D[v, s]`` is not finite and for ``v`` in ``S_s``, otherwise ``sigma[v, s]`` (``shortest_path_counts``)
        times the sum of ``fl((1 + delta[w, s]) / sigma[w, s])`` over the distinct tight pairs ``v -> w`` with
        ``sigma[w, s] != 0``, summed in ascending ``w`` like the counts.  (A finite element outside ``S_s`` with no tight
        predecessor has no paths, ``sigma = 0``: a loop cut short by ``max_steps`` can leave such elements, and their
        successors add nothing, so every dependency stays finite.)  With one source per column this is the unnormalised weighted betweenness
        restricted to those sources, counting ordered pairs; on unit weights it is ``betweenness`` bit for bit.
        ``dependencies_out`` (float64 [n x k]) receives ``delta``.  The loop, features and ``last_path_rounds`` are those
        of ``shortest_path_counts``.

        The backward sweep visits the rounds of the tight-pair DAG from the deepest to 0 along the out-lists; the
        round rows take 4 bytes per row and round in which the row has an element.  The dependency tile (8 bytes per
        element) is allocated on the first call and kept until ``close()``.  Raises ``ValueError`` before any CUDA work
        where ``shortest_path_counts`` does, and for an ``out`` or ``dependencies_out`` that is not a C-contiguous float64
        array of the right shape.  Synchronises."""
        self._wpaths_checks("weighted_betweenness")
        self._check_bc_outputs(out, dependencies_out)
        delta, bc = self._wbc_run(max_steps)
        if dependencies_out is not None:
            delta.d2h(dependencies_out)
        if out is None:
            return bc.d2h().reshape(-1)
        bc.d2h(out[:, None])
        return out

    def _wbc_run(self, max_steps: int) -> Tuple[_lib.Dense, _lib.Dense]:
        """the device part of ``weighted_betweenness``: the float64 dependency and [n x 1] betweenness tiles"""
        D, sigma = self._wpaths_run(max_steps, "weighted_betweenness")
        if self._wp_delta is None:
            n = self.levels[0].rows
            self._wp_delta = (self.ctx.dense_alloc(n, self.k, np.float64), self.ctx.dense_alloc(n, 1, np.float64))
        delta, bc = self._wp_delta
        x0, state, _ = self._wp_tiles
        delta.fill(0.0)
        self.ctx.wpaths_dependencies(self._wp_adjs[1], x0, D, state, sigma, delta)
        self.ctx.row_sum(delta, bc)
        return delta, bc

    def _wpaths_run(self, max_steps: int, what: str) -> Tuple[_lib.Dense, _lib.Dense]:
        """the device part of ``shortest_path_counts``: the fixed point (the level-0 features tile) and the float64 count
        tile, with the rounds kept in the loop-free out-adjacency's history"""
        self._wpaths_checks(what)
        self.sync()
        st0 = self.levels[0]
        if self._wp_adjs is None:
            parts = [(st.csr, st.cmap_dev) for st in self.levels]
            self._wp_adjs = (self.ctx.adj_build_loopfree(parts, st0.rows, direction="in"),
                             self.ctx.adj_build_loopfree(parts, st0.rows))
        if self._wp_tiles is None:
            self._wp_tiles = (self.ctx.dense_alloc(st0.rows, self.k), self.ctx.dense_alloc(st0.rows, self.k, np.int32),
                              self.ctx.dense_alloc(st0.rows, self.k, np.float64))
        x0, state, sigma = self._wp_tiles
        x0.copy_from(st0.bufs[st0.xi])          # the loop overwrites both level-0 tiles
        self.iterate_to_fixed_point(max_steps)
        D = st0.bufs[st0.xi]
        self.last_path_rounds, _ = self.ctx.wpaths_counts(self._wp_adjs[0], self._wp_adjs[1], x0, D, state, sigma)
        return D, sigma

    def _wpaths_checks(self, what: str):
        if self.sr != _lib.SR_MIN_PLUS:
            raise ValueError(f"{what} runs the min_plus semiring, the engine runs {self.semiring}")
        if not self.add_identity:
            raise ValueError(f"{what} needs add_identity=True: a step must keep the distances it already has")
        if not self.fused_ok:
            raise ValueError(f"{what} needs a level-0 row behind every non-zero, but a level reads rows behind the "
                             "sentinel")
        if self._nonpos_weight:
            raise ValueError(f"{what} needs every off-diagonal weight > 0: a zero, negative or NaN weight lets ties "
                             "close cycles of tight pairs")

    def _check_bc_outputs(self, out: Optional[np.ndarray], dependencies_out: Optional[np.ndarray]):
        n = self.levels[0].rows
        for name, arr, shape in (("out", out, (n,)), ("dependencies_out", dependencies_out, (n, self.k))):
            if arr is not None and (arr.dtype != np.float64 or arr.shape != shape or not arr.flags.c_contiguous):
                raise ValueError(f"{name} must be a C-contiguous float64 array of shape {shape}, got {arr.dtype} "
                                 f"{arr.shape}{'' if arr.flags.c_contiguous else ' (not contiguous)'}")

    def _paths_checks(self, what: str):
        self._bfs_checks(what)
        if not self.fused_ok:
            raise ValueError(f"{what} needs a level-0 row behind every non-zero, but a level reads rows behind the "
                             "sentinel")

    def _bfs_checks(self, what: str):
        if not self.bits:
            raise ValueError(f"{what} runs the or_and semiring, the engine runs {self.semiring}")
        if not self.add_identity:
            raise ValueError(f"{what} needs add_identity=True: a step must keep the bits it already has")

    def _bfs_run(self, max_steps: int, parents: Optional[_lib.Dense] = None,
                 sigma: Optional[_lib.Dense] = None) -> _lib.Dense:
        """the device part of ``bfs_levels``: runs the levels and returns the int32 level tile, left on the device.  With
        ``parents`` (``bfs_tree``) also writes the parent of every element into that int32 tile; with ``sigma``
        (``bfs_path_counts``) the path count of every element into that float64 tile, and keeps every level's frontier
        rows in the push adjacency's history."""
        self._bfs_checks("bfs_levels")
        self.sync()
        st0 = self.levels[0]
        if self._bfs_tiles is None:
            ones = self._alloc(st0.rows)
            ones.h2d(np.repeat(_lib.pack_bits(np.ones((1, self.k), bool)), st0.rows, axis=0))
            self._bfs_tiles = (self.ctx.dense_alloc(st0.rows, self.k, np.int32), self._alloc(st0.rows), ones)
        dist, zero, ones = self._bfs_tiles
        # an exchange-mode step of one level has no backward exchange and leaves level 0's features where they are, so a
        # push (which advances them like a fused step) would not match it: that engine pulls every level
        pushes = self.fused_ok and (self.mode == "fused" or self.L > 1)
        # the parent and path-count passes read the frontier record, so they keep one even on an engine that only pulls
        adj = self._push_adjacency() if pushes or parents is not None or sigma is not None else None
        limit = self._push_limit

        def mark(new, old, level):
            """(fresh bits, push next): the level record, and the direction of the next level"""
            if adj is None:
                return self.ctx.bits_mark_new(new, old, dist, level), False
            n_new, _, edges = self.ctx.bits_mark_frontier(adj, new, old, dist, level)
            if parents is not None and level > 0:        # old is X_{h-1} until the next level writes its tile
                self.ctx.bits_parents(self._in_adj, adj, new, old, parents)
            if sigma is not None:
                if level > 0:
                    self.ctx.bits_path_counts(self._in_adj, adj, new, old, sigma)
                self.ctx.adj_keep_record(adj, level)
            if not pushes:
                return n_new, False
            push = edges < limit if limit is not None else bfs_direction(edges, self.total_nnz) == "push"
            return n_new, push

        if parents is not None:                          # the sources have no parent
            self.ctx.bits_mark_new(st0.bufs[st0.xi], zero, parents, -1)
        if sigma is not None:                            # one path to each source, none to an element never reached
            sigma.fill(0.0)
            self.ctx.bits_fill_f64(st0.bufs[st0.xi], zero, sigma, 1.0)
        _, push = mark(st0.bufs[st0.xi], zero, 0)
        steps, directions = 0, []
        for level in range(1, int(max_steps) + 1):
            xi = st0.xi
            if push:                             # X_h | M F_h, F_h the rows marked by the previous pass
                self.ctx.bits_push_frontier(adj, st0.bufs[xi], st0.bufs[1 - xi])
                st0.xi = st0.ci = 1 - xi
            else:
                self.step()                      # reads bufs[xi], leaves the result in bufs[1 - xi]
            directions.append("push" if push else "pull")
            steps = level
            n_new, push = mark(st0.bufs[1 - xi], st0.bufs[xi], level)
            if n_new == 0:
                break
        self.last_bfs_steps = steps
        self.last_bfs_directions = directions
        # every element reached in this call was written by it; the others (clear in the final bits) become -1
        self.ctx.bits_mark_new(ones, st0.bufs[st0.xi], dist, -1)
        if parents is not None:
            self.ctx.bits_mark_new(ones, st0.bufs[st0.xi], parents, -1)
        return dist

    def _push_adjacency(self) -> _lib.Adjacency:
        """the transposed operator of the fused step with the identity (built on the first call): every level's own block
        with its level-j -> level-0 row map (level 0: the identity)"""
        if self._adj is None:
            parts = [(st.csr, st.cmap_dev) for st in self.levels]
            self._adj = self.ctx.adj_build(parts, self.levels[0].rows)
        return self._adj

    # -- streaming iteration for host-resident features ------------------------------------------------------
    def stream_step(self, X_host: np.ndarray, out_host: np.ndarray):
        """Enqueue one full iteration on host data: upload ``X_host`` -> ``step()`` -> download level-0 result
        into ``out_host``.  Returns immediately; uploads, compute and downloads of consecutive calls overlap
        (side copy streams ordered with events, two device slots).  Both arrays must be pinned
        (``_lib.PinnedArray``) of the engine's dtype and must stay untouched until ``stream_drain()``; use at least two
        (X, out) pairs in rotation.  Results are identical to ``set_features(X); step(); result()``."""
        if self.bits:
            raise ValueError("stream_step moves float tiles; the or_and engine steps on device-resident bits only")
        st = self.levels[0]
        if X_host.shape != (st.rows, self.k) or out_host.shape != (st.rows, self.k):
            raise ValueError(f"expected host arrays of shape {(st.rows, self.k)}")
        if X_host.dtype != self.dtype or out_host.dtype != self.dtype:
            raise ValueError(f"expected {self.dtype} host arrays, got {X_host.dtype} / {out_host.dtype}")
        ctx = self.ctx
        if not hasattr(self, "_slots"):
            # slot 0 re-uses the engine's own level-0 tiles, slot 1 gets two more
            self._slots = [list(st.bufs), [self._alloc(st.rows), self._alloc(st.rows)]]
            self._slot_i = 0
        s = self._slot_i % 2
        slot = self._slots[s]
        self._slot_i += 1
        EV_H2D, EV_MAIN, EV_D2H = 3 * s, 3 * s + 1, 3 * s + 2      # per-slot events
        ctx.event_wait(EV_MAIN, ctx.LANE_H2D)      # the compute two calls ago has finished reading slot[0]
        ctx.h2d_lane(ctx.LANE_H2D, slot[0], X_host)
        ctx.event_record(EV_H2D, ctx.LANE_H2D)
        ctx.event_wait(EV_H2D, ctx.LANE_MAIN)      # features are on the device
        ctx.event_wait(EV_D2H, ctx.LANE_MAIN)      # slot[1]'s previous result has been downloaded
        st.bufs = slot
        st.xi, st.ci = 0, 1                        # X = uploaded tile, C = the slot's second tile
        self.step()
        ctx.event_record(EV_MAIN, ctx.LANE_MAIN)
        ctx.event_wait(EV_MAIN, ctx.LANE_D2H)
        ctx.d2h_lane(ctx.LANE_D2H, st.bufs[st.ci], out_host)
        ctx.event_record(EV_D2H, ctx.LANE_D2H)

    def stream_drain(self):
        ctx = self.ctx
        ctx.lane_sync(ctx.LANE_H2D)
        ctx.sync()
        ctx.lane_sync(ctx.LANE_D2H)

    # -- accounting (SURVEY.md 8d) ------------------------------------------------------------------------
    def flops_per_step(self) -> float:
        """one ⊗ and one ⊕ per term, in every semiring"""
        return 2.0 * self.total_nnz * self.k

    def _entry_and_row_bytes(self) -> Tuple[int, float]:
        """bytes per non-zero (index + value; index only in or_and) and per feature row (k*e; the row's words in or_and)"""
        if self.bits:
            return 4, 4.0 * _lib.b1_words(self.k)
        e = self.dtype.itemsize
        return 4 + e, float(self.k * e)

    def algorithmic_bytes_per_step(self) -> float:
        """Per level nnz*(4+e) + (R+1)*4 + U*k*e + R*k*e (U = R = active rows, e = 4 or 8 bytes per element), plus the
        exchanges (forward 2 passes, backward 3 passes over the routed rows) -- the figure a fused implementation still
        reports against.  In ``or_and`` a non-zero is its 4-byte index and a row its words."""
        nz, row = self._entry_and_row_bytes()
        total = 0.0
        for j, st in enumerate(self.levels):
            total += st.nnz * nz + (st.rows + 1) * 4 + 2.0 * st.rows * row
            if j > 0:
                m = int(np.count_nonzero(st.to_prev < self.levels[j - 1].rows))
                total += 5.0 * m * row
        return total

    def _launch_level_as_in_step(self, j: int, src, dst):
        st = self.levels[j]
        if self.mode == "fused" and self.fused_style == "gather" and j + 1 < self.L:
            nxt = self.levels[j + 1]
            self._product(st.csr, src, dst, nxt.cbuf, nxt.to_next_dev)
        else:
            self._product(st.csr, src, dst)

    def time_level_spmm(self, j: int, iters: int, warmup: int = 3) -> float:
        """Average duration (ms) of level ``j``'s launch exactly as ``step()`` issues it (level 0 of the fused/gather
        path includes the epilogue gather-add of level 1's tile), CUDA events on the engine's stream."""
        st = self.levels[j]
        if j > 0 and self.mode == "fused":
            raise ValueError("levels > 0 are timed through step() in fused mode")
        src = st.bufs[st.xi]
        scratch = self._alloc(st.rows)
        for _ in range(warmup):
            self._launch_level_as_in_step(j, src, scratch)
        self.ctx.timer_start(5)
        for _ in range(iters):
            self._launch_level_as_in_step(j, src, scratch)
        self.ctx.timer_stop(5)
        ms = self.ctx.timer_ms(5) / iters
        scratch.free()
        return ms

    def level_bytes(self, j: int) -> float:
        """algorithmic bytes of level ``j``'s launch: nnz*(4+e) + (R+1)*4 + R*k*e (X) + R*k*e (C) with e = 4 or 8 bytes
        per element, plus -- when the launch carries the epilogue gather-add -- one read of the routed rows of the deeper
        level's tile (the other two passes of the reference's backward exchange do not exist in this launch).  In
        ``or_and`` a non-zero is its 4-byte index and a row its words."""
        nz, row = self._entry_and_row_bytes()
        st = self.levels[j]
        b = st.nnz * nz + (st.rows + 1) * 4 + 2.0 * st.rows * row
        if self.mode == "fused" and self.fused_style == "gather" and j + 1 < self.L:
            nxt = self.levels[j + 1]
            b += float(np.count_nonzero(nxt.to_prev < st.rows)) * row
        return b

    def close(self):
        for b in (self._wit_labels or []) + list(self._wit_values.values()) + list(self._bfs_tiles or ()):
            b.free()
        for a in (self._adj, self._sr_adj, self._in_adj, self._bfs_parents):
            if a is not None:
                a.free()
        self._wit_labels, self._wit_values, self._bfs_tiles, self._adj, self._sr_adj = None, {}, None, None, None
        for b in (self._bfs_sigma,) + (self._bfs_delta or ()) + (self._wp_adjs or ()) + (self._wp_tiles or ()) + \
                (self._wp_delta or ()):
            if b is not None:
                b.free()
        self._in_adj = self._bfs_parents = self._bfs_sigma = self._bfs_delta = None
        self._wp_adjs = self._wp_tiles = self._wp_delta = None
        for b in (self._bt_in_adj,) + (self._bt_tiles or ()):
            if b is not None:
                b.free()
        self._bt_in_adj = self._bt_tiles = None
        self._free_pagerank_operands()
        for b in (self._pr_weights or ()) + (self._pr_work or ()):
            b.free()
        self._pr_weights = self._pr_work = None
        for b in (self._cc_labels, self._cc_sizes):
            if b is not None:
                b.free()
        self._cc_labels = self._cc_sizes = None
        self.ctx.close()
