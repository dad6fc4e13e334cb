"""Predecessor pass timings on one GPU: ``ArrowEngine.predecessors()`` next to one ``min_plus`` step, in one process.

Workloads:
* the 10^6-vertex Barabasi-Albert shortest-path batch of scripts/semiring_bench.py (weights 1..16, width 20 000, 3
  levels, 32 sources, min_plus with the identity), timed at its fixed point;
* G2 of bench.py (10M rows, width 10 000, two levels, random level-1 permutation, seed 503) at k = 16 and k = 128,
  min_plus on random features in {0..7}.

For each it reports the step and the device pass of ``predecessors()`` (every launch, no download; CUDA events on the
engine's stream, mean of ``--steps`` after ``--warmup``), their ratio, and the wall time of one whole
``predecessors()`` call (synchronise + pass + download of the int32 tile).  ``--runs`` repeats every measurement and
reports each run, so the spread is visible.  One JSON line, with the card and its power limit; the level files go to a
temporary directory.

    python scripts/witness_bench.py [--blocks 1000] [--steps 20] [--warmup 5] [--runs 3]
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


def engine(base, width, k, add_identity=False):
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, width, True, slim=True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, width, k, 'gpu', True, True,
                                             semiring="min_plus", add_identity=add_identity)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    return arrow, arrow._engine


def _events(eng, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    eng.ctx.timer_start(7)
    for _ in range(steps):
        fn()
    eng.ctx.timer_stop(7)
    return eng.ctx.timer_ms(7) / steps


def measure(eng, X, steps, warmup, runs):
    """per run: step (rewound to the same features each time) and pass, both on X"""
    out = {"mode": eng.mode, "levels": eng.L, "step_ms": [], "pass_ms": [], "call_ms": []}

    def step():
        eng.rewind_features()
        eng.step()

    for _ in range(runs):
        eng.set_features(X)
        out["step_ms"].append(round(_events(eng, step, steps, warmup), 4))
        eng.set_features(X)
        out["pass_ms"].append(round(_events(eng, eng._predecessor_pass, steps, warmup), 4))
        eng.sync()
        t = time.perf_counter()
        P = eng.predecessors()
        out["call_ms"].append(round((time.perf_counter() - t) * 1e3, 2))
    out["parents"] = int(np.count_nonzero(P >= 0))
    out["pass_over_step"] = round(float(np.median(out["pass_ms"]) / np.median(out["step_ms"])), 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--sssp-vertices", type=int, default=1000000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("witness_bench.py: no CUDA device")
    out = {"steps": a.steps, "runs": a.runs, **bench.gpu_info(0)}
    work = tempfile.mkdtemp(prefix="arrow_witness_")
    try:
        # shortest paths at the fixed point (the batch of semiring_bench.py)
        n, w, n_src = a.sssp_vertices, 20000, 32
        from arrow_matrix_b200.decomposition import arrow_decomposition
        from scipy import sparse
        A = sparse.triu(synth.barabasi_albert(n, 3, seed=503), k=1).tocoo()
        wts = np.random.default_rng(5).integers(1, 17, A.nnz).astype(np.float32)
        U = sparse.coo_matrix((wts, (A.row, A.col)), shape=(n, n))
        dec = arrow_decomposition(sparse.csr_matrix(U + U.T), w, max_number_of_levels=3, block_diagonal=True, seed=2)
        sbase = os.path.join(work, "ba")
        graphio.save_decomposition_new(dec, sbase, w, block_diagonal=True)
        arrow, eng = engine(sbase, w, n_src, add_identity=True)
        perm0 = decomp.prepare_permutations([p for _, p in dec], eng.n_blocks, w)[0][0]
        inv = np.full(n, -1, np.int64)
        ok = perm0 < n
        inv[perm0[ok]] = np.flatnonzero(ok)
        X = np.full((eng.n_rows, n_src), np.inf, np.float32)
        X[inv[np.random.default_rng(8).choice(n, n_src, replace=False)], np.arange(n_src)] = 0.0
        eng.set_features(X)
        fixed = eng.iterate_to_fixed_point(1000)
        D = eng.result()
        out["sssp"] = {"graph": f"Barabasi-Albert {n} vertices, m=3, weights 1..16, width {w}", "sources": n_src,
                       "steps_to_fixed_point": fixed, **measure(eng, D, a.steps, a.warmup, a.runs)}
        eng.close()
        # G2
        base = os.path.join(work, "g2")
        graphio.save_decomposition_new(synth.synth_decomposition(a.blocks, a.width, levels=2, perm_kind="random",
                                                                 seed=503), base, a.width, block_diagonal=True)
        rng = np.random.default_rng(42)
        for k in (16, 128):
            X = rng.integers(0, 8, (a.blocks * a.width, k)).astype(np.float32)
            arrow, eng = engine(base, a.width, k)
            out[f"g2_k{k}"] = {"rows": a.blocks * a.width, **measure(eng, X, a.steps, a.warmup, a.runs)}
            eng.close()
            del X
    finally:
        shutil.rmtree(work, True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
