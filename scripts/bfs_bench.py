"""Boolean-semiring (or, and) timings on one GPU against (min, +), in one process.

1. G2 of bench.py (10M rows, width 10 000, two levels, ~10 nnz/row, random level-1 permutation, seed 503) through the
   level files (save_decomposition_new -> load_decomposition_new -> initialize(semiring=...)).  For k = 128 and k = 16 and
   both semirings: the whole step and the level-0 launch as the step issues it (CUDA events on the engine's stream, after
   warm-up), their algorithmic GB/s (the engine's byte accounting: 4 B per non-zero and the row's words in or_and), and
   the or_and / min_plus ratios.
2. Multi-source BFS to the fixed point on the 10**6-vertex Barabasi-Albert graph of semiring_bench.py (m = 3, width
   20 000, 3 levels) from 128 sources: ``bfs_levels`` (bit tiles, one level-record pass per step) against min_plus with
   unit weights and ``iterate_to_fixed_point``, each call timed whole (host clock, it ends in a synchronising download of
   the n x 128 levels / distances into a touched host buffer) and the download on its own (best of 3); the per-step figure
   leaves the download out.
   ``verified``: the hop levels equal the min_plus distances cast to int, -1 where those are inf.

One JSON line with the card and its power limit; the level files go to a temporary directory.

    python scripts/bfs_bench.py [--blocks 1000] [--steps 20] [--warmup 5]
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
from arrow_matrix_b200 import decomp, graphio, synth  # noqa: E402
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI  # noqa: E402
from arrow_matrix_b200.comm import SelfComm  # noqa: E402

SEMIRINGS = ["or_and", "min_plus"]


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
    ap.add_argument("--bfs-vertices", type=int, default=1000000)
    ap.add_argument("--sources", type=int, default=128)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bfs_bench.py: no CUDA device")
    out = {"workload": f"G2: {a.blocks * a.width} rows, width {a.width}, 2 levels, random permutation (seed 503)",
           "steps": a.steps, **bench.gpu_info(0)}
    work = tempfile.mkdtemp(prefix="arrow_bfs_")
    try:
        base = os.path.join(work, "g2")
        graphio.save_decomposition_new(synth.synth_decomposition(a.blocks, a.width, levels=2, perm_kind="random",
                                                                 seed=503), base, a.width, block_diagonal=True)
        rng = np.random.default_rng(42)
        rows = a.blocks * a.width
        for k in (128, 16):
            for semiring in SEMIRINGS:
                X = rng.random((rows, k)) < 0.5 if semiring == "or_and" else \
                    (2 * rng.random((rows, k), dtype=np.float32) - 1)
                arrow, eng = engine(base, a.width, k, semiring)
                eng.set_features(X)
                step_ms = time_step(eng, a.steps, a.warmup)
                eng.rewind_features()
                l0_ms = eng.time_level_spmm(0, a.steps, a.warmup)
                out[f"{semiring}_k{k}"] = {
                    "mode": eng.mode, "step_ms": round(step_ms, 4), "level0_ms": round(l0_ms, 4),
                    "step_gbs": round(eng.algorithmic_bytes_per_step() / step_ms / 1e6, 1),
                    "level0_gbs": round(eng.level_bytes(0) / l0_ms / 1e6, 1),
                    "step_algorithmic_gb": round(eng.algorithmic_bytes_per_step() / 1e9, 3)}
                eng.close()
            for key in ("step_ms", "level0_ms"):
                out[f"or_and_over_min_plus_k{k}_{key}"] = round(out[f"or_and_k{k}"][key] / out[f"min_plus_k{k}"][key], 3)
        # multi-source BFS to the fixed point
        n, w, n_src = a.bfs_vertices, 20000, a.sources
        from arrow_matrix_b200.decomposition import arrow_decomposition
        from scipy import sparse
        A = sparse.triu(synth.barabasi_albert(n, 3, seed=503), k=1).tocoo()
        U = sparse.coo_matrix((np.ones(A.nnz, np.float32), (A.row, A.col)), shape=(n, n))
        dec = arrow_decomposition(sparse.csr_matrix(U + U.T), w, max_number_of_levels=3, block_diagonal=True, seed=2)
        sbase = os.path.join(work, "ba")
        graphio.save_decomposition_new(dec, sbase, w, block_diagonal=True)
        sources = np.random.default_rng(8).choice(n, n_src, replace=False)
        res = {}
        for semiring in SEMIRINGS:
            arrow, eng = engine(sbase, w, n_src, semiring, add_identity=True)
            perm0 = decomp.prepare_permutations([p for _, p in dec], eng.n_blocks, w)[0][0]
            inv = np.full(n, -1, np.int64)
            ok = perm0 < n
            inv[perm0[ok]] = np.flatnonzero(ok)
            hit = (inv[sources], np.arange(n_src))
            if semiring == "or_and":
                X = np.zeros((eng.n_rows, n_src), bool)
                X[hit] = True
            else:
                X = np.full((eng.n_rows, n_src), np.inf, np.float32)
                X[hit] = 0.0
            # a host buffer touched beforehand receives the n x 128 levels / distances, so that no call pays for first-touch
            # page faults; the download into it is timed on its own (best of 3, host clock around a synchronising d2h)
            buf = np.zeros((eng.n_rows, n_src), np.int32 if semiring == "or_and" else np.float32)
            for warm in (True, False):          # the first run loads the kernels and allocates the level tile
                eng.set_features(X)
                eng.sync()
                t = time.perf_counter()
                if semiring == "or_and":
                    eng.bfs_levels(1000, out=buf)
                    steps = eng.last_bfs_steps
                else:
                    steps = eng.iterate_to_fixed_point(1000)
                    eng.result(out=buf)
                ms = (time.perf_counter() - t) * 1e3
            res[semiring] = buf.copy()
            tile = eng._bfs_tiles[0] if semiring == "or_and" else eng.result_buffer()
            dl = float("inf")
            for _ in range(3):
                t = time.perf_counter()
                tile.d2h(buf)
                dl = min(dl, (time.perf_counter() - t) * 1e3)
            key = "bfs_levels" if semiring == "or_and" else "min_plus_fixed_point"
            out[key] = {"mode": eng.mode, "steps": steps, "total_ms": round(ms, 3), "download_ms": round(dl, 3),
                        "ms_per_step_without_download": round((ms - dl) / steps, 4)}
            eng.close()
        D = res["min_plus"]
        out["bfs"] = {"graph": f"Barabasi-Albert {n} vertices, m=3, unit weights, width {w}, {len(dec)} levels",
                      "sources": n_src,
                      "verified": bool(np.array_equal(res["or_and"], np.where(np.isinf(D), -1, D).astype(np.int32))),
                      "total_ratio": round(out["bfs_levels"]["total_ms"] / out["min_plus_fixed_point"]["total_ms"], 3),
                      "per_step_ratio": round(out["bfs_levels"]["ms_per_step_without_download"] /
                                              out["min_plus_fixed_point"]["ms_per_step_without_download"], 3)}
    finally:
        shutil.rmtree(work, True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
