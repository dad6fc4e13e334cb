"""BFS parents on one GPU: ``bfs_levels`` (hop levels only), ``bfs_tree`` (levels and parents from the bit tiles) and the
(min, +) route (``iterate_to_fixed_point`` then ``predecessors()`` on unit weights), in one process.

Workloads (the decompositions of scripts/bfs_direction_bench.py, held in memory, sources random rows):
  * G2 of bench.py (10M rows, width 10 000, two levels, ~10 nnz/row, random level-1 permutation, seed 503) at k = 16 and
    k = 128;
  * the 10**6-vertex Barabasi-Albert graph (m = 3, width 20 000, 3 levels) at k = 128.

For each workload, 3 rounds, the three routes alternating within a round on the same sources, host clock around work
that ends in a synchronise, results left on the device:
  * ``bfs_levels_ms``: ``ArrowEngine._bfs_run`` (the device part of ``bfs_levels``);
  * ``bfs_tree_ms``: ``ArrowEngine._bfs_tree_run`` (the device part of ``bfs_tree``);
  * ``min_plus_ms``: ``iterate_to_fixed_point`` + the predecessor pass of ``predecessors()`` on a ``min_plus`` engine with
    ``add_identity`` over the same decomposition with every value 1.
Also the in-adjacency's build time and bytes, and a per-level table from one more run issuing ``_bfs_tree_run``'s
launches with CUDA events around each level's parent pass: direction, frontier rows, in-edges gathered, ms.
``verified``: the hop levels of the three routes are identical and the parents equal the (min, +) parents in every
round.  One JSON line per workload as it ends, then one with them all, each with the card and its power limit.

    python scripts/bfs_parents_bench.py [--rounds 3] [--bfs-vertices 1000000]
"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np
from scipy import sparse

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (gpu_info)
from arrow_matrix_b200 import synth  # noqa: E402
from arrow_matrix_b200.engine import ArrowEngine, bfs_direction  # noqa: E402


def unit(decomposition):
    out = []
    for B, p in decomposition:
        B = sparse.csr_matrix(B, copy=True)
        B.data = np.ones_like(B.data, dtype=np.float32)
        out.append((B, p))
    return out


def digest(tile, conv=None, chunk=1 << 20):
    """SHA-1 of a device tile's rows (after ``conv``), downloaded in chunks: 10M x 128 tiles are compared without holding
    several of them on the host"""
    h = hashlib.sha1()
    for r0 in range(0, tile.rows, chunk):
        x = tile.d2h(row0=r0, rows=min(chunk, tile.rows - r0))
        h.update(np.ascontiguousarray(conv(x) if conv else x).tobytes())
    return h.hexdigest()


def hops(D):
    return np.where(np.isfinite(D), D, -1).astype(np.int32)


def clock(fn):
    t = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t) * 1e3, r


def per_level(eng, X0, max_steps=1000):
    """the launches of ``_bfs_tree_run`` (automatic direction) with a CUDA event pair around each parent pass"""
    eng.zero_rhs()
    eng.set_features(X0)
    ctx, st0 = eng.ctx, eng.levels[0]
    dist, zero, ones = eng._bfs_tiles
    adj, in_adj, P = eng._adj, eng._in_adj, eng._bfs_parents
    ctx.bits_mark_new(st0.bufs[st0.xi], zero, P, -1)
    _, rows, edges = ctx.bits_mark_frontier(adj, st0.bufs[st0.xi], zero, dist, 0)
    table = []
    for level in range(1, max_steps + 1):
        push = bfs_direction(edges, eng.total_nnz) == "push"
        xi = st0.xi
        if push:
            ctx.bits_push_frontier(adj, st0.bufs[xi], st0.bufs[1 - xi])
            st0.xi = st0.ci = 1 - xi
        else:
            eng.step()
        n_new, rows, edges = ctx.bits_mark_frontier(adj, st0.bufs[1 - xi], st0.bufs[xi], dist, level)
        ctx.timer_start(7)
        scanned = ctx.bits_parents(in_adj, adj, st0.bufs[1 - xi], st0.bufs[xi], P, count=True)
        ctx.timer_stop(7)
        table.append({"level": level, "dir": "push" if push else "pull", "fresh_bits": n_new, "frontier_rows": rows,
                      "in_edges_scanned": scanned, "parents_ms": round(ctx.timer_ms(7), 4)})
        if n_new == 0:
            break
    return table


def run_workload(dec, width, k, rng, rounds):
    eng = ArrowEngine(dec, width, k, semiring="or_and", add_identity=True)
    mp = ArrowEngine(unit(dec), width, k, semiring="min_plus", add_identity=True)
    n = eng.n_rows
    X0 = np.zeros((n, k), bool)
    X0[rng.choice(n, k, replace=False), np.arange(k)] = True
    D0 = np.where(X0, 0.0, np.inf).astype(np.float32)
    out = {"rows": n, "k": k, "total_nnz": eng.total_nnz, "mode": eng.mode}
    parts = [(st.csr, st.cmap_dev) for st in eng.levels]
    build_ms, in_adj = clock(lambda: eng.ctx.adj_build(parts, n, direction="in"))
    ip, _ = in_adj.d2h()
    deg = np.diff(ip.astype(np.int64))
    segs = int(np.sum(np.where(deg > 512, (deg + 511) // 512, 0)))
    out["in_adjacency"] = {"build_ms": round(build_ms, 3), "edges": int(ip[-1]), "long_rows": int(np.sum(deg > 512)),
                           "segments": segs, "bytes": 4 * (n + 1) + 4 * int(ip[-1]) + 16 * segs}
    in_adj.free()

    def levels_run():
        eng.zero_rhs()
        eng.set_features(X0)
        eng.sync()
        return clock(lambda: eng._bfs_run(1000))

    def tree_run():
        eng.zero_rhs()
        eng.set_features(X0)
        eng.sync()
        return clock(lambda: eng._bfs_tree_run(1000))

    def min_plus_run():
        mp.zero_rhs()
        mp.set_features(D0)
        mp.sync()

        def go():
            steps = mp.iterate_to_fixed_point(1000)
            P = mp._predecessor_pass()
            mp.sync()
            return steps, P
        return clock(go)

    levels_run(), tree_run(), min_plus_run()              # warm-up: kernels, tiles and adjacencies
    times = {"bfs_levels_ms": [], "bfs_tree_ms": [], "min_plus_ms": []}
    verified = True
    for _ in range(rounds):
        ms, dist = levels_run()
        times["bfs_levels_ms"].append(ms)
        L1 = digest(dist)
        steps, dirs = eng.last_bfs_steps, list(eng.last_bfs_directions)
        ms, (dist, P) = tree_run()
        times["bfs_tree_ms"].append(ms)
        L2, P2 = digest(dist), digest(P)
        verified &= eng.last_bfs_steps == steps and eng.last_bfs_directions == dirs
        ms, (_, Pm) = min_plus_run()
        times["min_plus_ms"].append(ms)
        st0 = mp.levels[0]
        L3, Pm = digest(st0.bufs[st0.xi], hops), digest(Pm)
        verified &= L1 == L2 == L3 and P2 == Pm
    out["steps"] = eng.last_bfs_steps
    out["min_plus_steps"] = len(mp.last_fixed_point_directions)
    out["directions"] = list(eng.last_bfs_directions)
    out.update({key: [round(x, 3) for x in v] for key, v in times.items()})
    best = {key: min(v) for key, v in times.items()}
    out["tree_over_levels"] = round(best["bfs_tree_ms"] / best["bfs_levels_ms"], 3)
    out["min_plus_over_tree"] = round(best["min_plus_ms"] / best["bfs_tree_ms"], 3)
    out["per_level"] = per_level(eng, X0)
    out["verified"] = verified
    eng.close()
    mp.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--bfs-vertices", type=int, default=1000000)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bfs_parents_bench.py: no CUDA device")
    out = {"rounds": a.rounds, **bench.gpu_info(0)}
    rng = np.random.default_rng(42)
    g2 = synth.synth_decomposition(a.blocks, a.width, levels=2, perm_kind="random", seed=503)
    for k in (16, 128):
        out[f"g2_k{k}"] = run_workload(g2, a.width, k, rng, a.rounds)
        print(json.dumps({f"g2_k{k}": out[f"g2_k{k}"], **bench.gpu_info(0)}), flush=True)   # each workload as it ends
    del g2
    from arrow_matrix_b200.decomposition import arrow_decomposition
    n, w = a.bfs_vertices, 20000
    A = sparse.triu(synth.barabasi_albert(n, 3, seed=503), k=1).tocoo()
    U = sparse.coo_matrix((np.ones(A.nnz, np.float32), (A.row, A.col)), shape=(n, n))
    dec = arrow_decomposition(sparse.csr_matrix(U + U.T), w, max_number_of_levels=3, block_diagonal=True, seed=2)
    out["ba_k128"] = run_workload(dec, w, 128, rng, a.rounds)
    print(json.dumps({"ba_k128": out["ba_k128"], **bench.gpu_info(0)}), flush=True)
    out["verified"] = all(out[x]["verified"] for x in ("g2_k16", "g2_k128", "ba_k128"))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
