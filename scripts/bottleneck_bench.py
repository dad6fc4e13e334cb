"""Bottleneck semiring timings on one GPU (max_min: widest paths, min_max: minimax paths), in one process.

* G2 of bench.py (10M rows, width 10 000, two levels, ~10 nnz/row, random level-1 permutation, seed 503) through the
  level files: the step time of max_min, min_max and min_plus at k = 16 and 128, the semirings alternating within each
  of the rounds (CUDA events on the engine's stream).
* A 10**6-vertex Barabasi-Albert graph (m = 3, symmetric integer weights 1..16, three levels) at k = 32 and 128, one
  source per column: ``iterate_to_fixed_point`` pulling every level against the direction-optimising loop (with its
  per-level directions), and ``bottleneck_tree`` against ``iterate_to_fixed_point``, alternating within each round.
  ``bottleneck_tree`` is timed on the device (the loop with its T-writing mark passes and the tree pass, up to a
  synchronise) apart from the download of D and P; the tree pass alone is timed with CUDA events over repeated launches.

``verified``: the pull and push features are identical in every round, and every parent satisfies the tree rule
(checked vectorised on the host: the parent edge exists with a weight a such that a ⊗ D[u] == D[v] in bits, and D[u] is
strictly better than D[v] or equal with T[u] < T[v], T being the device's step record).  One JSON line with
the card and its power limit; the level files go to a temporary directory.

    python scripts/bottleneck_bench.py [--blocks 1000] [--rounds 3] [--steps 20] [--warmup 5]
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

ALL_PULL = 0


def engine(base, width, k, semiring, add_identity=False):
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, width, True, slim=True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, width, k, 'gpu', True, True,
                                             semiring=semiring, add_identity=add_identity)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    arrow.B.zero_rhs(width, k)
    return arrow._engine


def time_step(eng, steps, warmup):
    for _ in range(warmup):
        eng.step()
    eng.ctx.timer_start(6)
    for _ in range(steps):
        eng.step()
    eng.ctx.timer_stop(6)
    return eng.ctx.timer_ms(6) / steps


def progress(msg):
    print(f"[bottleneck_bench] {msg}", file=sys.stderr, flush=True)


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return r, (time.perf_counter() - t0) * 1e3


def tree_ok(eng, D, P, T, chunk=16):
    """every parent edge exists in the weighted push adjacency (u != v) and satisfies the tree rule (column chunks)"""
    return all(_tree_ok(eng, D[:, c:c + chunk], P[:, c:c + chunk], T[:, c:c + chunk]) for c in range(0, D.shape[1], chunk))


def _tree_ok(eng, D, P, T):
    indptr, indices = eng._sr_adj.d2h()
    vals = eng._sr_adj.values_d2h()
    n = indptr.size - 1
    u = np.repeat(np.arange(n, dtype=np.int64), np.diff(indptr.astype(np.int64)))
    v = indices.astype(np.int64)
    keep = u != v
    u, v, a = u[keep], v[keep], vals[keep]
    larger = eng.semiring == "max_min"
    zero = np.float32(-np.inf if larger else np.inf)
    pending = (T > 0) & (D != zero)
    has = P >= 0
    if np.any(has & ~pending) or not np.all(has[pending]):
        return False
    pv, pc = np.nonzero(has)
    pu = P[has].astype(np.int64)
    pair = u * n + v
    order = np.argsort(pair, kind="stable")
    pair, a = pair[order], a[order]
    q = pu * n + pv
    lo, hi = np.searchsorted(pair, q, "left"), np.searchsorted(pair, q, "right")
    if np.any(lo == hi):
        return False

    def key(x):
        b = np.asarray(x, np.float32).view(np.uint32)
        return np.where(b >= np.uint32(0x80000000), ~b, b | np.uint32(0x80000000))

    du, dv, tu, tv = D[pu, pc], D[pv, pc], T[pu, pc], T[pv, pc]
    ok = np.zeros(q.size, bool)
    j = lo.copy()
    while True:                                      # every duplicate of (u, v) until one fits
        live = ~ok & (j < hi)
        if not live.any():
            break
        w = a[j[live]]
        kw, kd = key(w), key(du[live])
        t = np.where(np.isnan(w), du[live], np.where((kw < kd) if larger else (kw > kd), w, du[live]))
        same_v = t.view(np.uint32) == dv[live].view(np.uint32)
        better = (key(du[live]) > key(dv[live])) if larger else (key(du[live]) < key(dv[live]))
        eq = du[live].view(np.uint32) == dv[live].view(np.uint32)
        ok[live] = same_v & (better | (eq & (tu[live] < tv[live])))
        j += 1
    return bool(ok.all())


def tree_pass_ms(eng, reps=5):
    """the tree pass alone (arrow_sr_tree_parents on the last fixed point and T), CUDA events over ``reps`` launches"""
    steps, parents = eng._bt_tiles
    D = eng.result_buffer(0)
    eng.ctx.sr_tree_parents(eng._bt_in_adj, D, steps, parents, eng.sr)
    eng.ctx.timer_start(7)
    for _ in range(reps):
        eng.ctx.sr_tree_parents(eng._bt_in_adj, D, steps, parents, eng.sr)
    eng.ctx.timer_stop(7)
    return eng.ctx.timer_ms(7) / reps


def run_ba(eng, X0, rounds, max_steps=500):
    times = {"pull": [], "auto": [], "tree": [], "tree_download": []}
    verified, dirs, steps = True, None, None
    D_pull = None
    for d in ("pull", "auto", "tree"):                 # warm-up: kernels loaded, adjacencies and tiles built
        eng._push_limit = ALL_PULL if d == "pull" else None
        eng.set_features(X0)
        eng.bottleneck_tree(max_steps) if d == "tree" else eng.iterate_to_fixed_point(max_steps)
    for r in range(rounds):
        progress(f"{eng.semiring} k={eng.k} round {r}")
        for d in ("pull", "auto", "tree"):
            eng._push_limit = ALL_PULL if d == "pull" else None
            eng.set_features(X0)
            if d == "tree":                        # the device part up to a synchronise, then the download
                (dD, dP), ms = timed(lambda: (eng._bottleneck_tree_run(max_steps), eng.sync())[0])
                (D, P), ms_d2h = timed(lambda: (dD.d2h(), dP.d2h()))
                times["tree_download"].append(round(ms_d2h, 3))
            else:
                n, ms = timed(lambda: (eng.iterate_to_fixed_point(max_steps), eng.sync())[0])
                D = eng.result()
                if d == "pull":
                    D_pull, steps = D, n
                else:
                    dirs = list(eng.last_fixed_point_directions)
                    verified &= n == steps
            times[d].append(round(ms, 3))
            verified &= np.array_equal(D.view(np.uint32), D_pull.view(np.uint32))
    eng._push_limit = None
    eng.set_features(X0)
    D, P = eng.bottleneck_tree(max_steps)
    verified &= tree_ok(eng, D, P, eng._bt_tiles[0].d2h())
    return {"steps": steps, "directions_auto": dirs, "ms": times, "tree_pass_ms": round(tree_pass_ms(eng), 3),
            "auto_over_pull": round(min(times["auto"]) / min(times["pull"]), 3),
            "tree_over_fixed_point": round(min(times["tree"]) / min(times["auto"]), 3), "verified": bool(verified)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--vertices", type=int, default=1000000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bottleneck_bench.py: no CUDA device")
    out = {"rounds": a.rounds, **bench.gpu_info(0)}
    work = tempfile.mkdtemp(prefix="arrow_bottleneck_")
    rng = np.random.default_rng(42)
    try:
        from arrow_matrix_b200.decomposition import arrow_decomposition
        from scipy import sparse
        n, w = a.vertices, 20000
        A = sparse.triu(synth.barabasi_albert(n, 3, seed=503), k=1).tocoo()
        wts = np.random.default_rng(5).integers(1, 17, A.nnz).astype(np.float32)
        U = sparse.coo_matrix((wts, (A.row, A.col)), shape=(n, n))
        progress("decomposing the BA graph")
        dec = arrow_decomposition(sparse.csr_matrix(U + U.T), w, max_number_of_levels=3, block_diagonal=True, seed=2)
        sbase = os.path.join(work, "ba")
        graphio.save_decomposition_new(dec, sbase, w, block_diagonal=True)
        for k in (32, 128):
            for semiring in ("max_min", "min_max"):
                eng = engine(sbase, w, k, semiring, add_identity=True)
                X0 = np.full((eng.n_rows, k), -np.inf if semiring == "max_min" else np.inf, np.float32)
                X0[rng.choice(eng.n_rows, k, replace=False), np.arange(k)] = np.inf if semiring == "max_min" else -np.inf
                out[f"ba_{semiring}_k{k}"] = run_ba(eng, X0, a.rounds)
                eng.close()
        base = os.path.join(work, "g2")
        progress("writing G2")
        graphio.save_decomposition_new(synth.synth_decomposition(a.blocks, a.width, levels=2, perm_kind="random",
                                                                 seed=503), base, a.width, block_diagonal=True)
        for k in (16, 128):
            X = (2 * rng.random((a.blocks * a.width, k), dtype=np.float32) - 1)
            engines = {s: engine(base, a.width, k, s) for s in ("max_min", "min_max", "min_plus")}
            times = {s: [] for s in engines}
            for s, eng in engines.items():
                eng.set_features(X)
            for r in range(a.rounds):
                progress(f"G2 k={k} round {r}")
                for s, eng in engines.items():
                    eng.rewind_features()
                    times[s].append(round(time_step(eng, a.steps, a.warmup), 4))
            out[f"g2_k{k}_step_ms"] = times
            for eng in engines.values():
                eng.close()
    finally:
        shutil.rmtree(work, True)
    out["verified"] = all(v["verified"] for key, v in out.items() if key.startswith("ba_"))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
