"""``ArrowDecompositionMPI`` on the GPU -- the upper drop-in boundary of the hot path.

Same class surface as the reference (``arrow/arrow_dec_mpi.py:21-930``): ``load_decomposition_new``,
``initialize``, ``step``, ``_propagate_features``, ``_aggregate``, ``_all_to_all_tables``,
``number_of_blocks`` and the attributes ``B, matrix_index, decomposition_length, comm, device``; the
benchmark driver and the tests call exactly these.  Differences that follow from the hardware
mapping (one process per GPU, every level resident on every GPU):

* ``blocks`` returned by ``load_decomposition_new`` is an opaque handle on the memory-mapped level
  files (each process slices its own rows; no root scatter, ``:695-887``);
* every process takes part in every level, so ``matrix_index`` is 0 and ``B`` is the level-0
  operator; ``levels[j]`` gives the operator of level ``j``;
* ``step()`` runs the fused path when that is exactly equivalent (see ``engine.py``).
"""
from __future__ import annotations

import time
from typing import List, Optional

import numpy as np

from . import decomp, graphio, wb_logging
from .arrow_mpi import ArrowMPI
from .arrow_slim_mpi import ArrowSlimMPI, _require_gpu
from .engine import ArrowEngine, semiring_code


class DecompositionBlocks:
    """What ``load_decomposition_new`` hands to ``load_sparse_matrix_from_blocks``."""

    def __init__(self, decomposition, width, block_diagonal, n_blocks, dtype=np.float32):
        self.decomposition = decomposition
        self.width = width
        self.block_diagonal = block_diagonal
        self.n_blocks = n_blocks
        self.dtype = np.dtype(dtype)          # precision of the values, the tiles and the arithmetic


class ArrowDecompositionMPI:
    B: ArrowSlimMPI
    matrix_index: int
    decomposition_length: int
    device: str

    def __init__(self, comm, B: ArrowSlimMPI, matrix_index: int, number_of_rows_per_rank: int,
                 number_of_feature_columns: int, groups, to_previous_permutation, to_next_mapping,
                 device='gpu', slim=True, block_diagonal=True, n_blocks=None, mode="auto", exchange="p2p", overlap=1,
                 semiring: str = "plus_times", add_identity: bool = False):
        _require_gpu(device)
        self.comm = comm
        self.B = B
        self.matrix_index = matrix_index
        self.decomposition_length = len(groups) if groups is not None else (len(n_blocks) if n_blocks is not None else 1)
        self._n_rows_per_rank = number_of_rows_per_rank
        self._n_feature_columns = number_of_feature_columns
        self.device = device
        self.slim = slim
        self.block_diagonal = block_diagonal
        self.n_blocks = n_blocks
        self._to_prev = to_previous_permutation
        self._to_next = to_next_mapping
        self._mode = mode
        self._exchange = exchange
        self._overlap = overlap
        self._semiring = semiring
        self._add_identity = bool(add_identity)
        self._engine = None
        self.levels: List[ArrowSlimMPI] = [B]
        B._owner = self

    # -- factory -----------------------------------------------------------------------------------------
    @staticmethod
    def initialize(comm, n_blocks: np.ndarray, to_prev_permutation, to_next_permutation, rows_per_rank: int,
                   feature_columns: int, device='gpu', block_diagonal: bool = True, slim: bool = False, mode: str = "auto",
                   exchange: str = "p2p", overlap: int = 1, semiring: str = "plus_times", add_identity: bool = False):
        """Same arguments as the reference (``:106-115``).  ``slim`` only selects the reference's rank
        layout; on a GPU both layouts are the same row-partitioned kernels, so it is accepted and ignored.
        Extensions (one GPU): ``semiring`` -- ``"plus_times"`` (the reference's product), ``"min_plus"`` or
        ``"max_plus"`` (float32), ``"max_min"`` or ``"min_max"`` (float32 bottleneck semirings: widest and minimax paths,
        see ``bottleneck_tree``), or ``"or_and"`` (bit features: ``set_features`` takes booleans, non-zero is true, and
        ``result_tile()`` returns booleans; with ``add_identity`` a step is one hop of multi-source BFS, see
        ``bfs_levels``) -- and ``add_identity``, which makes a step compute ``X ⊕ (A ⊗ X)`` (see ``engine.py``)."""
        assert not slim or block_diagonal
        assert np.sum(n_blocks) > 0
        def level_operator(owner, j):           # the reference hands out ArrowSlimMPI or ArrowMPI (``:166-197``)
            return ArrowSlimMPI(comm, owner, j) if slim else ArrowMPI(comm, block_diagonal, owner, j)
        B = level_operator(None, 0)
        arrow = ArrowDecompositionMPI(comm, B, 0, rows_per_rank, feature_columns, None, to_prev_permutation,
                                      to_next_permutation, device=device, slim=slim, block_diagonal=block_diagonal,
                                      n_blocks=[int(b) for b in n_blocks], mode=mode, exchange=exchange, overlap=overlap,
                                      semiring=semiring, add_identity=add_identity)
        arrow.levels = [B] + [level_operator(arrow, j) for j in range(1, len(n_blocks))]
        return arrow

    def _build_engine(self, blocks: DecompositionBlocks):
        if not isinstance(blocks, DecompositionBlocks):
            raise TypeError("blocks must come from ArrowDecompositionMPI.load_decomposition_new")
        if blocks.width != self._n_rows_per_rank:
            raise ValueError(f"decomposition was loaded for width {blocks.width}, initialised for {self._n_rows_per_rank}")
        dtype = getattr(blocks, "dtype", np.dtype(np.float32))
        if self.comm.Get_size() > 1 and dtype != np.float32:
            raise ValueError(f"a {dtype} decomposition runs on one GPU only: the multi-GPU engine computes in float32; "
                             "load it with datatype=np.float32 or run a single process")
        fused_style = getattr(self, "_fused_style", "gather")
        semiring_code(self._semiring, dtype, fused_style)
        if self.comm.Get_size() > 1 and (self._semiring != "plus_times" or self._add_identity):
            raise ValueError(f"semiring={self._semiring!r} / add_identity={self._add_identity} run on one GPU only: the "
                             "multi-GPU engine computes (+, x) without the identity; run a single process")
        if self._engine is not None:
            self._engine.close()
        if self.comm.Get_size() > 1:
            # one process per GPU: this rank's block-rows of every level, straight from the memory maps
            import os
            from .sharded import CudaPeerBackend, NcclBackend, ShardPlan, ShardedArrowEngine
            dev = getattr(self.comm, "device", None)
            if dev is None:
                dev = int(os.environ.get("LOCAL_RANK", self.comm.Get_rank()))
            plan = ShardPlan(blocks.decomposition, blocks.width, self.comm.Get_rank(), self.comm.Get_size(),
                             block_diagonal=blocks.block_diagonal, n_blocks=self.n_blocks)
            be = NcclBackend(self.comm, dev, blocks.width, plan) if self._exchange == "nccl" \
                else CudaPeerBackend(self.comm, dev, blocks.width, plan=None if self._exchange == "p2p-direct" else plan)
            be.layout_plan = plan
            self._engine = ShardedArrowEngine(plan, self._n_feature_columns, be, overlap=self._overlap, mode=self._mode)
        else:
            self._engine = ArrowEngine(blocks.decomposition, blocks.width, self._n_feature_columns,
                                       block_diagonal=blocks.block_diagonal, mode=self._mode, n_blocks=self.n_blocks,
                                       fused_style=fused_style, dtype=dtype, semiring=self._semiring,
                                       add_identity=self._add_identity)
        self.decomposition_length = self._engine.L

    def load_data_from_blocks(self, blocked: DecompositionBlocks):
        self.B.load_sparse_matrix_from_blocks(blocked)

    # -- iteration (arrow_dec_mpi.py:283-307) ---------------------------------------------------------------
    def step(self):
        """One SpMM iteration: X := A X on level 0 (postcondition of ``:289``)."""
        eng = self._require_engine()
        tic = time.perf_counter()
        eng.step()
        toc = time.perf_counter()
        wb_logging.log({'spmm_arrow_time': toc - tic})

    def _propagate_features(self):
        eng = self._require_engine()
        eng.ensure_level_tiles()
        tic = time.perf_counter()
        eng.propagate_features()
        wb_logging.log({"spmm_bcast_time": time.perf_counter() - tic})
        return None

    def _aggregate(self):
        eng = self._require_engine()
        tic = time.perf_counter()
        eng.aggregate()
        wb_logging.log({"spmm_reduce_time": time.perf_counter() - tic})

    def step_stream(self, X_host: np.ndarray, out_host: np.ndarray):
        """Extension for host-resident features: enqueue ``set_features(X); step(); result_tile(out)`` so that
        uploads, compute and downloads of consecutive iterations overlap (see ``ArrowEngine.stream_step``).
        Call ``synchronize()`` before reading ``out_host``.  On N GPUs every rank passes its own rows."""
        self._require_engine().stream_step(X_host, out_host)

    def predecessors(self, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Extension (one GPU, ``min_plus`` / ``max_plus``): the parent of every element of the level-0 features, int32
        in ``result_tile()`` row order, ``-1`` for sources and unreachable vertices (see ``ArrowEngine.predecessors``).
        Entries are level-0 rows; level 0's permutation maps them to vertex ids like the distances."""
        eng = self._require_engine()
        if not isinstance(eng, ArrowEngine):
            raise ValueError("predecessors run on one GPU only")
        return eng.predecessors(out)

    def bfs_levels(self, max_steps: int, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Extension (one GPU, ``or_and`` with ``add_identity``): hop levels of a multi-source BFS from the current
        level-0 features, int32 in ``result_tile()`` row order, ``-1`` where never reached (see
        ``ArrowEngine.bfs_levels``)."""
        eng = self._require_engine()
        if not isinstance(eng, ArrowEngine):
            raise ValueError("bfs_levels runs on one GPU only")
        return eng.bfs_levels(max_steps, out)

    def bfs_tree(self, max_steps: int, levels_out: Optional[np.ndarray] = None,
                 parents_out: Optional[np.ndarray] = None):
        """Extension (one GPU, ``or_and`` with ``add_identity``): ``bfs_levels`` and the BFS parents, both int32 in
        ``result_tile()`` row order; a parent is a level-0 row, ``-1`` for sources and elements never reached (see
        ``ArrowEngine.bfs_tree``).  Level 0's permutation maps the parents to vertex ids like the rows."""
        if self.comm.Get_size() > 1:
            raise ValueError("bfs_tree runs on one GPU only")
        eng = self._require_engine()
        if not isinstance(eng, ArrowEngine):
            raise ValueError("bfs_tree runs on one GPU only")
        return eng.bfs_tree(max_steps, levels_out, parents_out)

    def bfs_path_counts(self, max_steps: int, levels_out: Optional[np.ndarray] = None,
                        counts_out: Optional[np.ndarray] = None):
        """Extension (one GPU, ``or_and`` with ``add_identity``): ``bfs_levels`` and the shortest-path counts, int32 and
        float64 in ``result_tile()`` row order (see ``ArrowEngine.bfs_path_counts``)."""
        return self._bfs_engine("bfs_path_counts").bfs_path_counts(max_steps, levels_out, counts_out)

    def betweenness(self, max_steps: int, out: Optional[np.ndarray] = None,
                    dependencies_out: Optional[np.ndarray] = None) -> np.ndarray:
        """Extension (one GPU, ``or_and`` with ``add_identity``): Brandes betweenness over the feature columns as
        sources, float64 [n] in ``result_tile()`` row order (see ``ArrowEngine.betweenness``).  Level 0's permutation
        maps the rows to vertex ids."""
        return self._bfs_engine("betweenness").betweenness(max_steps, out, dependencies_out)

    def shortest_path_counts(self, max_steps: int, distances_out: Optional[np.ndarray] = None,
                             counts_out: Optional[np.ndarray] = None):
        """Extension (one GPU, ``min_plus`` with ``add_identity``): ``iterate_to_fixed_point`` and the number of tight
        shortest paths to every element, float32 distances and float64 counts in ``result_tile()`` row order (see
        ``ArrowEngine.shortest_path_counts``)."""
        return self._bfs_engine("shortest_path_counts").shortest_path_counts(max_steps, distances_out, counts_out)

    def weighted_betweenness(self, max_steps: int, out: Optional[np.ndarray] = None,
                             dependencies_out: Optional[np.ndarray] = None) -> np.ndarray:
        """Extension (one GPU, ``min_plus`` with ``add_identity``): Brandes betweenness over the weighted shortest paths
        from the feature columns, float64 [n] in ``result_tile()`` row order (see ``ArrowEngine.weighted_betweenness``).
        Level 0's permutation maps the rows to vertex ids."""
        return self._bfs_engine("weighted_betweenness").weighted_betweenness(max_steps, out, dependencies_out)

    def bottleneck_tree(self, max_steps: int, distances_out: Optional[np.ndarray] = None,
                        parents_out: Optional[np.ndarray] = None):
        """Extension (one GPU, ``max_min`` / ``min_max`` with ``add_identity``): ``iterate_to_fixed_point`` and a path tree
        of the widest or minimax values, float32 values and int32 parents in ``result_tile()`` row order; a parent is a
        level-0 row, ``-1`` for sources and elements not reached (see ``ArrowEngine.bottleneck_tree``).  Level 0's
        permutation maps the parents to vertex ids like the rows."""
        return self._bfs_engine("bottleneck_tree").bottleneck_tree(max_steps, distances_out, parents_out)

    def pagerank(self, max_steps: int, alpha: float = 0.85, tol: float = 1e-6, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Extension (one GPU, ``plus_times``): personalized PageRank with one restart distribution per feature column,
        in ``result_tile()`` row order (see ``ArrowEngine.pagerank``).  Level 0's permutation maps the rows to vertex
        ids."""
        return self._bfs_engine("pagerank").pagerank(max_steps, alpha, tol, out)

    def connected_components(self, out: Optional[np.ndarray] = None, sizes_out: Optional[np.ndarray] = None) -> np.ndarray:
        """Extension (one GPU, any semiring): weakly connected components of the operator, int32 labels (the smallest row
        of each row's component) in ``result_tile()`` row order (see ``ArrowEngine.connected_components``).  Level 0's
        permutation maps the rows, and so the labels, to vertex ids."""
        return self._bfs_engine("connected_components").connected_components(out, sizes_out)

    def _bfs_engine(self, what: str) -> ArrowEngine:
        if self.comm.Get_size() > 1:
            raise ValueError(f"{what} runs on one GPU only")
        eng = self._require_engine()
        if not isinstance(eng, ArrowEngine):
            raise ValueError(f"{what} runs on one GPU only")
        return eng

    def iterate_to_fixed_point(self, max_steps: int) -> int:
        """Extension (one GPU): ``step()`` until a step changes no level-0 row, at most ``max_steps`` times; returns the
        number of steps taken.  Direction-optimising in ``min_plus`` / ``max_plus`` / ``max_min`` / ``min_max`` with
        ``add_identity`` (multi-source shortest, critical, widest and minimax paths; see
        ``ArrowEngine.iterate_to_fixed_point``)."""
        eng = self._require_engine()
        if not isinstance(eng, ArrowEngine):
            raise ValueError("iterate_to_fixed_point runs on one GPU only")
        return eng.iterate_to_fixed_point(max_steps)

    def synchronize(self):
        self._require_engine().sync()

    def _require_engine(self):
        if self._engine is None:
            raise RuntimeError("sparse blocks not loaded yet: call B.load_sparse_matrix_from_blocks(blocks)")
        return self._engine

    # -- static helpers kept for drop-in parity ---------------------------------------------------------------
    @staticmethod
    def _all_to_all_tables(out_permutation: np.ndarray, rows_per_rank: int, n_columns: int, total_ranks: int,
                           put_offset: int = 0):
        """Routing tables of the reference's alltoallv (``:325-384``): counts, displacements, pack order and
        unpack order.  The device path routes with global row maps instead; this stays for callers and tests
        that use the reference's static helper."""
        out_permutation = np.asarray(out_permutation)
        assert out_permutation.size == rows_per_rank
        assert put_offset < total_ranks and n_columns > 0 and total_ranks > 0
        dest = np.floor_divide(out_permutation, rows_per_rank).astype(np.intp)
        counted = dest[dest + put_offset < total_ranks] + put_offset
        counts = np.bincount(counted, minlength=total_ranks).astype(np.int64) * n_columns
        displs = np.zeros(total_ranks, dtype=np.int64)
        displs[1:] = np.cumsum(counts)[:-1]
        send_perm = np.argsort(dest, kind='stable')
        routed = np.flatnonzero(dest < total_ranks)
        recv_perm = routed[np.lexsort((out_permutation[routed], dest[routed]))].astype(np.intp)
        return list(counts), list(displs), send_perm, recv_perm

    @staticmethod
    def number_of_blocks(adjacency, width: int) -> int:
        return decomp.number_of_blocks(adjacency, width)

    @staticmethod
    def load_decomposition_new(comm, filename: str, width: int, is_block_diagonal: bool, datatype=np.float32,
                               slim=False, use_npy=True, use_mmap=True):
        """Open the level files (``:629-887``).  Returns ``(blocks, n_blocks, to_prev, to_next)`` like the
        reference; ``blocks`` is ``None`` (and ``n_blocks`` empty) when nothing was found.  Files are memory
        mapped -- every process slices its own rows, nothing is scattered from a root.  ``datatype`` (float32, the
        reference's default, or float64) is the precision of the values, the tiles and the arithmetic of every step;
        float32 values in the files become float64 exactly, missing value files mean ones.  float64 runs on one GPU."""
        assert not slim or is_block_diagonal
        if np.dtype(datatype) not in (np.float32, np.float64):
            raise ValueError(f"datatype must be float32 or float64 (numpy.random.Generator.random's types), got "
                             f"{np.dtype(datatype)}")
        if use_npy:
            dec = graphio.load_decomposition_new(filename, width, block_diagonal=is_block_diagonal, mem_map=True)
        else:                                  # SciPy .npz per level (``:641-648``): read whole, then sliced per rank
            dec = graphio.load_decomposition(filename, width, block_diagonal=is_block_diagonal)
        if len(dec) == 0:
            print("ERROR: decomposition with name ", filename, " and width ", width, "not found", flush=True)
            return None, np.zeros(0, dtype=np.int32), None, None
        n_blocks = np.array([decomp.number_of_blocks(B, width) for B, _ in dec], dtype=np.int32)
        _, to_prev, to_next, _ = decomp.prepare_permutations([p for _, p in dec], n_blocks, width)
        blocks = DecompositionBlocks(dec, width, is_block_diagonal, n_blocks, datatype)
        return blocks, n_blocks, to_prev, to_next
