"""Direction-optimising BFS on one GPU: pull-only, push-only and the automatic rule of ``bfs_levels``, in one process.

Workloads (level files in a temporary directory, loaded like scripts/bfs_bench.py):
  * G2 of bench.py (10M rows, width 10 000, two levels, ~10 nnz/row, random level-1 permutation, seed 503) at k = 16 and
    k = 128, each column's source a random row;
  * the 10**6-vertex Barabasi-Albert graph of scripts/bfs_bench.py (m = 3, width 20 000, 3 levels), 128 random sources.

For each workload, 3 rounds, the three directions alternating within a round:
  * ``stepping_ms``: host clock around ``ArrowEngine._bfs_run`` (every level and its record pass; it ends in a synchronising
    count read-back), the hop levels left on the device; ``download_ms``: the levels' download on its own;
  * ``pull_with_mark_new``: the previous bfs_levels loop (a step and an arrow_bits_mark_new pass per level), same clock;
  * a per-level table from a second run that issues the same launches as ``_bfs_run`` with CUDA events around each
    level's push or step and around its record pass: direction, frontier rows and edges before the level, ms, mark_ms.
``verified``: the hop levels of the three directions and of the previous loop are identical in every round.  One JSON line with the card and its
power limit.

    python scripts/bfs_direction_bench.py [--rounds 3] [--bfs-vertices 1000000]
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
from arrow_matrix_b200.engine import BFS_PUSH_ALPHA, bfs_direction  # noqa: E402

LIMITS = {"pull": 0, "push": 1 << 62, "auto": None}      # ArrowEngine._push_limit of each direction


def engine(base, width, k):
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, width, True, slim=True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, width, k, 'gpu', True, True,
                                             semiring="or_and", add_identity=True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    return arrow._engine


def per_level(eng, X0, limit, max_steps=1000):
    """the launches of ``_bfs_run`` with the direction rule or a forced limit, a CUDA event pair around each level's push
    or step (the record pass that follows it is not in the time)"""
    eng.zero_rhs()
    eng.set_features(X0)
    ctx, st0 = eng.ctx, eng.levels[0]
    eng._bfs_run(1)                                     # allocates the tiles, builds the adjacency
    eng.zero_rhs()
    eng.set_features(X0)
    dist, zero, _ = eng._bfs_tiles
    adj = eng._adj
    _, rows, edges = ctx.bits_mark_frontier(adj, st0.bufs[st0.xi], zero, dist, 0)
    table = []
    for level in range(1, max_steps + 1):
        push = edges < limit if limit is not None else bfs_direction(edges, eng.total_nnz) == "push"
        xi = st0.xi
        ctx.timer_start(7)
        if push:
            ctx.bits_push_frontier(adj, st0.bufs[xi], st0.bufs[1 - xi])
            st0.xi = st0.ci = 1 - xi
        else:
            eng.step()
        ctx.timer_stop(7)
        ms = ctx.timer_ms(7)
        entry = {"level": level, "dir": "push" if push else "pull", "frontier_rows": rows, "frontier_edges": edges,
                 "ms": round(ms, 4)}
        ctx.timer_start(7)
        n_new, rows, edges = ctx.bits_mark_frontier(adj, st0.bufs[1 - xi], st0.bufs[xi], dist, level)
        ctx.timer_stop(7)
        entry["mark_ms"] = round(ctx.timer_ms(7), 4)          # the record pass (ends in its synchronising read-back)
        table.append(entry)
        if n_new == 0:
            break
    return table


def pull_loop(eng, X0, dist, zero, ones, max_steps=1000):
    """the previous bfs_levels loop: a step and an arrow_bits_mark_new pass per level, no adjacency (host clock)"""
    st0 = eng.levels[0]
    eng.zero_rhs()
    eng.set_features(X0)
    eng.sync()
    t = time.perf_counter()
    eng.ctx.bits_mark_new(st0.bufs[st0.xi], zero, dist, 0)
    for level in range(1, max_steps + 1):
        xi = st0.xi
        eng.step()
        if eng.ctx.bits_mark_new(st0.bufs[1 - xi], st0.bufs[xi], dist, level) == 0:
            break
    eng.ctx.bits_mark_new(ones, st0.bufs[st0.xi], dist, -1)
    eng.sync()
    return (time.perf_counter() - t) * 1e3


def run_workload(eng, X0, rounds):
    out = {"rows": eng.n_rows, "k": eng.k, "total_nnz": eng.total_nnz, "mode": eng.mode, "fused_ok": eng.fused_ok}
    levels_ref, verified = None, True
    times = {d: [] for d in list(LIMITS) + ["pull_with_mark_new"]}
    downloads, dirs = [], {}
    buf = np.zeros((eng.n_rows, eng.k), np.int32)       # touched beforehand: no first-touch faults in the download
    for d, limit in LIMITS.items():                     # warm-up: kernels loaded, tiles and adjacency allocated
        eng._push_limit = limit
        eng.zero_rhs()
        eng.set_features(X0)
        eng._bfs_run(1000)
    for _ in range(rounds):
        for d, limit in LIMITS.items():
            eng._push_limit = limit
            eng.zero_rhs()
            eng.set_features(X0)
            eng.sync()
            t = time.perf_counter()
            dist = eng._bfs_run(1000)
            times[d].append((time.perf_counter() - t) * 1e3)
            dirs[d] = list(eng.last_bfs_directions)
            t = time.perf_counter()
            dist.d2h(buf)
            downloads.append((time.perf_counter() - t) * 1e3)
            if levels_ref is None:
                levels_ref = buf.copy()
            else:
                verified &= bool(np.array_equal(buf, levels_ref))
        times["pull_with_mark_new"].append(pull_loop(eng, X0, *eng._bfs_tiles))
        verified &= bool(np.array_equal(eng._bfs_tiles[0].d2h(buf), levels_ref))
    out["steps"] = eng.last_bfs_steps
    out["stepping_ms"] = {d: [round(x, 3) for x in v] for d, v in times.items()}
    out["directions_auto"] = dirs["auto"]
    out["download_ms"] = [round(min(downloads), 3), round(max(downloads), 3)]
    out["levels"] = {d: per_level(eng, X0, limit) for d, limit in LIMITS.items() if d != "auto"}
    out["verified"] = verified
    best = {d: min(v) for d, v in times.items()}
    out["auto_over_pull"] = round(best["auto"] / best["pull"], 3)
    out["auto_not_slower"] = min(times["auto"]) <= max(times["pull"])         # within the spread of the pull runs
    return out


def random_sources(rows, k, rng):
    X = np.zeros((rows, k), bool)
    X[rng.choice(rows, k, replace=False), np.arange(k)] = True
    return X


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--bfs-vertices", type=int, default=1000000)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bfs_direction_bench.py: no CUDA device")
    out = {"alpha": BFS_PUSH_ALPHA, "rounds": a.rounds, **bench.gpu_info(0)}
    work = tempfile.mkdtemp(prefix="arrow_bfs_dir_")
    rng = np.random.default_rng(42)
    try:
        base = os.path.join(work, "g2")
        graphio.save_decomposition_new(synth.synth_decomposition(a.blocks, a.width, levels=2, perm_kind="random",
                                                                 seed=503), base, a.width, block_diagonal=True)
        for k in (16, 128):
            eng = engine(base, a.width, k)
            out[f"g2_k{k}"] = run_workload(eng, random_sources(eng.n_rows, k, rng), a.rounds)
            eng.close()
        from arrow_matrix_b200.decomposition import arrow_decomposition
        from scipy import sparse
        n, w = a.bfs_vertices, 20000
        A = sparse.triu(synth.barabasi_albert(n, 3, seed=503), k=1).tocoo()
        U = sparse.coo_matrix((np.ones(A.nnz, np.float32), (A.row, A.col)), shape=(n, n))
        dec = arrow_decomposition(sparse.csr_matrix(U + U.T), w, max_number_of_levels=3, block_diagonal=True, seed=2)
        sbase = os.path.join(work, "ba")
        graphio.save_decomposition_new(dec, sbase, w, block_diagonal=True)
        eng = engine(sbase, w, 128)
        out["ba_k128"] = run_workload(eng, random_sources(eng.n_rows, 128, rng), a.rounds)
        eng.close()
    finally:
        shutil.rmtree(work, True)
    out["verified"] = all(out[w]["verified"] for w in ("g2_k16", "g2_k128", "ba_k128"))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
