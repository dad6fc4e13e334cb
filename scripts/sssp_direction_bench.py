"""Direction-optimising min_plus fixed point on one GPU: pull-only, push-only and the automatic rule of
``iterate_to_fixed_point``, in one process.

Workloads (level files in a temporary directory, loaded like scripts/semiring_bench.py):
  * the SSSP batch of scripts/semiring_bench.py: Barabasi-Albert graph of 10**6 vertices (m = 3, weights 1..16, width
    20 000, 3 levels), 32 random sources;
  * G2 of bench.py (10M rows, width 10 000, two levels, ~10 nnz/row, random level-1 permutation, seed 503; its values are
    rng.random, non-negative, so a fixed point exists) at k = 16 and k = 128, each column's source a random row.

For each workload, 3 rounds, the three directions alternating within a round:
  * ``stepping_ms``: host clock around ``iterate_to_fixed_point`` (every level and its mark pass; it ends in the mark
    pass's synchronising read-back);
  * ``pull_with_count_diff``: the previous loop (a step and an arrow_dense_count_diff pass per level), same clock;
  * a per-level table from a further run that issues the same launches as ``iterate_to_fixed_point`` with CUDA events
    around each level's push or step and around its mark pass: direction, frontier rows and edges before the level, ms,
    mark_ms.
``verified``: the step counts and the final features (bit for bit) of the three directions and of the previous loop are
identical in every round.  One JSON line with the card and its power limit.

    python scripts/sssp_direction_bench.py [--rounds 3] [--sssp-vertices 1000000]
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
from arrow_matrix_b200.engine import _PLUS_ZERO, SR_PUSH_ALPHA, bfs_direction  # noqa: E402

LIMITS = {"pull": 0, "push": 1 << 62, "auto": None}      # ArrowEngine._push_limit of each direction
MAX_STEPS = 1000


def engine(base, width, k):
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, width, True, slim=True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, width, k, 'gpu', True, True,
                                             semiring="min_plus", add_identity=True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    return arrow._engine


def per_level(eng, X0, limit):
    """the launches of ``iterate_to_fixed_point`` with the direction rule or a forced limit, a CUDA event pair around each
    level's push or step and one around the mark pass that follows it"""
    eng.zero_rhs()
    eng.set_features(X0)
    ctx, st0 = eng.ctx, eng.levels[0]
    adj = eng._sr_push_adjacency()
    xi = st0.xi
    st0.bufs[1 - xi].fill(_PLUS_ZERO[eng.sr])
    _, rows, edges = ctx.sr_mark_frontier(adj, st0.bufs[xi], st0.bufs[1 - xi])
    table = []
    for level in range(1, MAX_STEPS + 1):
        push = edges < limit if limit is not None else bfs_direction(edges, eng.total_nnz, SR_PUSH_ALPHA) == "push"
        xi = st0.xi
        ctx.timer_start(7)
        if push:
            ctx.sr_push_frontier(adj, st0.bufs[xi], st0.bufs[1 - xi], eng.sr)
            st0.xi = st0.ci = 1 - xi
        else:
            eng.step()
        ctx.timer_stop(7)
        entry = {"level": level, "dir": "push" if push else "pull", "frontier_rows": rows, "frontier_edges": edges,
                 "ms": round(ctx.timer_ms(7), 4)}
        ctx.timer_start(7)
        changed, rows, edges = ctx.sr_mark_frontier(adj, st0.bufs[1 - xi], st0.bufs[xi])
        ctx.timer_stop(7)
        entry["mark_ms"] = round(ctx.timer_ms(7), 4)
        table.append(entry)
        if changed == 0:
            break
    return table


def count_diff_loop(eng, X0):
    """the previous iterate_to_fixed_point loop: a step and an arrow_dense_count_diff pass per level (host clock)"""
    eng.zero_rhs()
    eng.set_features(X0)
    eng.sync()
    t = time.perf_counter()
    steps = MAX_STEPS
    for n in range(1, MAX_STEPS + 1):
        eng.step()
        if eng.count_changed() == 0:
            steps = n
            break
    return (time.perf_counter() - t) * 1e3, steps


def run_workload(eng, X0, rounds):
    out = {"rows": eng.n_rows, "k": eng.k, "L": eng.L, "total_nnz": eng.total_nnz, "mode": eng.mode,
           "fused_ok": eng.fused_ok, "push_ok": eng._sr_push_ok()}
    ref, verified = None, True
    times = {d: [] for d in list(LIMITS) + ["pull_with_count_diff"]}
    dirs = {}
    buf = np.zeros((eng.n_rows, eng.k), np.float32)
    for d, limit in LIMITS.items():                     # warm-up: kernels loaded, adjacency built
        eng._push_limit = limit
        eng.zero_rhs()
        eng.set_features(X0)
        eng.iterate_to_fixed_point(MAX_STEPS)
    out["adjacency_edges"] = eng._sr_adj.info()["n_edges"]

    def check(steps):
        nonlocal ref, verified
        eng.result(out=buf)
        if ref is None:
            ref = (steps, buf.view(np.uint32).copy())
        else:
            verified &= steps == ref[0] and bool(np.array_equal(buf.view(np.uint32), ref[1]))

    for _ in range(rounds):
        for d, limit in LIMITS.items():
            eng._push_limit = limit
            eng.zero_rhs()
            eng.set_features(X0)
            eng.sync()
            t = time.perf_counter()
            steps = eng.iterate_to_fixed_point(MAX_STEPS)
            times[d].append((time.perf_counter() - t) * 1e3)
            dirs[d] = list(eng.last_fixed_point_directions)
            check(steps)
        ms, steps = count_diff_loop(eng, X0)
        times["pull_with_count_diff"].append(ms)
        check(steps)
    out["steps"] = ref[0]
    out["stepping_ms"] = {d: [round(x, 3) for x in v] for d, v in times.items()}
    out["directions_auto"] = dirs["auto"]
    out["levels"] = {d: per_level(eng, X0, limit) for d, limit in LIMITS.items() if d != "auto"}
    out["verified"] = verified
    best = {d: min(v) for d, v in times.items()}
    out["auto_over_pull"] = round(best["auto"] / best["pull"], 3)
    out["auto_not_slower"] = min(times["auto"]) <= max(times["pull"])         # within the spread of the pull runs
    return out


def random_sources(rows, k, rng):
    X = np.full((rows, k), np.inf, np.float32)
    X[rng.choice(rows, k, replace=False), np.arange(k)] = 0.0
    return X


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--sssp-vertices", type=int, default=1000000)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("sssp_direction_bench.py: no CUDA device")
    out = {"alpha": SR_PUSH_ALPHA, "rounds": a.rounds, **bench.gpu_info(0)}
    work = tempfile.mkdtemp(prefix="arrow_sssp_dir_")
    rng = np.random.default_rng(42)
    try:
        from arrow_matrix_b200.decomposition import arrow_decomposition
        from scipy import sparse
        n, w = a.sssp_vertices, 20000
        A = sparse.triu(synth.barabasi_albert(n, 3, seed=503), k=1).tocoo()
        wts = np.random.default_rng(5).integers(1, 17, A.nnz).astype(np.float32)
        U = sparse.coo_matrix((wts, (A.row, A.col)), shape=(n, n))
        dec = arrow_decomposition(sparse.csr_matrix(U + U.T), w, max_number_of_levels=3, block_diagonal=True, seed=2)
        sbase = os.path.join(work, "ba")
        graphio.save_decomposition_new(dec, sbase, w, block_diagonal=True)
        eng = engine(sbase, w, 32)
        out["ba_k32"] = run_workload(eng, random_sources(eng.n_rows, 32, rng), a.rounds)
        eng.close()
        base = os.path.join(work, "g2")
        graphio.save_decomposition_new(synth.synth_decomposition(a.blocks, a.width, levels=2, perm_kind="random",
                                                                 seed=503), base, a.width, block_diagonal=True)
        for k in (16, 128):
            eng = engine(base, a.width, k)
            out[f"g2_k{k}"] = run_workload(eng, random_sources(eng.n_rows, k, rng), a.rounds)
            eng.close()
    finally:
        shutil.rmtree(work, True)
    out["verified"] = all(out[w]["verified"] for w in ("ba_k32", "g2_k16", "g2_k128"))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
