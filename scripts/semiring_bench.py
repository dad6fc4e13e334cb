"""Semiring step timings on one GPU: (+, x) vs (min, +) vs (max, +) on the G2 workload of bench.py, in one process.

G2 (10M rows, width 10 000, two levels, ~10 nnz/row, random level-1 permutation, seed 503) goes through the level files
(save_decomposition_new -> load_decomposition_new -> initialize(semiring=...)), like bench.py.  For k = 128 and k = 16 and
every semiring it times the whole step and the level-0 launch as the step issues it (CUDA events on the engine's
stream).  It then runs a single-source-shortest-path batch on a Barabasi-Albert graph (min_plus with the identity, 32
sources, weights 1..16) to its fixed point and reports the steps and the time per step.  One JSON line, with the card
and its power limit; the files go to a temporary directory.

    python scripts/semiring_bench.py [--blocks 1000] [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (gpu_info)
from arrow_matrix_b200 import graphio, synth  # noqa: E402
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI  # noqa: E402
from arrow_matrix_b200.comm import SelfComm  # noqa: E402

SEMIRINGS = ["plus_times", "min_plus", "max_plus"]


def engine(base, width, k, semiring, add_identity=False):
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, width, True, slim=True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, width, k, 'gpu', True, True,
                                             semiring=semiring, add_identity=add_identity)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    arrow.B.zero_rhs(width, k)
    return arrow, arrow._engine


def time_step(eng, steps, warmup):
    for _ in range(warmup):
        eng.step()
    eng.ctx.timer_start(6)
    for _ in range(steps):
        eng.step()
    eng.ctx.timer_stop(6)
    return eng.ctx.timer_ms(6) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sssp-vertices", type=int, default=1000000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("semiring_bench.py: no CUDA device")
    out = {"workload": f"G2: {a.blocks * a.width} rows, width {a.width}, 2 levels, random permutation (seed 503)",
           "steps": a.steps, **bench.gpu_info(0)}
    work = tempfile.mkdtemp(prefix="arrow_semiring_")
    try:
        base = os.path.join(work, "g2")
        graphio.save_decomposition_new(synth.synth_decomposition(a.blocks, a.width, levels=2, perm_kind="random",
                                                                 seed=503), base, a.width, block_diagonal=True)
        rng = np.random.default_rng(42)
        for k in (128, 16):
            X = (2 * rng.random((a.blocks * a.width, k), dtype=np.float32) - 1)
            for semiring in SEMIRINGS:
                arrow, eng = engine(base, a.width, k, semiring)
                eng.set_features(X)
                step_ms = time_step(eng, a.steps, a.warmup)
                eng.rewind_features()
                l0_ms = eng.time_level_spmm(0, a.steps, a.warmup)
                out[f"{semiring}_k{k}"] = {"mode": eng.mode, "step_ms": round(step_ms, 4), "level0_ms": round(l0_ms, 4),
                                           "level0_gbs": round(eng.level_bytes(0) / l0_ms / 1e6, 1)}
                eng.close()
        for k in (128, 16):
            out[f"min_plus_over_plus_times_k{k}"] = round(out[f"min_plus_k{k}"]["step_ms"] /
                                                          out[f"plus_times_k{k}"]["step_ms"], 3)
        # multi-source shortest paths to the fixed point
        n, w, n_src = a.sssp_vertices, 20000, 32
        from arrow_matrix_b200.decomposition import arrow_decomposition
        from scipy import sparse
        A = sparse.triu(synth.barabasi_albert(n, 3, seed=503), k=1).tocoo()
        wts = np.random.default_rng(5).integers(1, 17, A.nnz).astype(np.float32)
        U = sparse.coo_matrix((wts, (A.row, A.col)), shape=(n, n))
        dec = arrow_decomposition(sparse.csr_matrix(U + U.T), w, max_number_of_levels=3, block_diagonal=True, seed=2)
        sbase = os.path.join(work, "ba")
        graphio.save_decomposition_new(dec, sbase, w, block_diagonal=True)
        arrow, eng = engine(sbase, w, n_src, "min_plus", add_identity=True)
        from arrow_matrix_b200 import decomp
        perm0 = decomp.prepare_permutations([p for _, p in dec], eng.n_blocks, w)[0][0]
        inv = np.full(n, -1, np.int64)
        ok = perm0 < n
        inv[perm0[ok]] = np.flatnonzero(ok)
        X = np.full((eng.n_rows, n_src), np.inf, np.float32)
        X[inv[np.random.default_rng(8).choice(n, n_src, replace=False)], np.arange(n_src)] = 0.0
        eng.set_features(X)
        eng.sync()
        t = time.perf_counter()
        steps = eng.iterate_to_fixed_point(1000)
        ms = (time.perf_counter() - t) * 1e3
        out["sssp"] = {"graph": f"Barabasi-Albert {n} vertices, m=3, weights 1..16, width {w}, {eng.L} levels",
                       "sources": n_src, "mode": eng.mode, "steps": steps,
                       "ms_per_step_incl_count": round(ms / steps, 4)}
        eng.close()
    finally:
        shutil.rmtree(work, True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
