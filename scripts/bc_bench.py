"""Betweenness on one GPU: ``bfs_levels`` (hop levels only), ``bfs_path_counts`` (levels and shortest-path counts) and
``betweenness`` (counts, the backward dependency sweep and the row sum), in one process.

Workloads (those of scripts/bfs_parents_bench.py, held in memory, one source per column at random rows):
  * G2 of bench.py (10M rows, width 10 000, two levels, ~10 nnz/row, random level-1 permutation, seed 503) at k = 16 and
    k = 128;
  * the 10**6-vertex Barabasi-Albert graph (m = 3, width 20 000, 3 levels) at k = 128.

For each workload, 3 rounds, the three routes alternating within a round on the same sources, host clock around work
that ends in a synchronise, results left on the device:
  * ``bfs_levels_ms``: ``ArrowEngine._bfs_run`` (the device part of ``bfs_levels``);
  * ``path_counts_ms``: ``ArrowEngine._bfs_paths_run`` (the device part of ``bfs_path_counts``);
  * ``betweenness_ms``: ``ArrowEngine._betweenness_run`` (the device part of ``betweenness``).
Also a per-level table from one more run issuing the same launches with CUDA events around each level's path-count pass
(forward) and dependency pass (backward): direction, frontier rows, list entries read, ms.  ``verified``: the levels of
the three routes are identical and the counts and betweenness the same bits in every round; and, at a reduced size (a
20 000-vertex BA graph, k = 32), levels, counts, dependencies and betweenness equal tests/paths_ref.py bit for bit.  One
JSON line per workload as it ends, then one with them all, each with the card and its power limit.

    python scripts/bc_bench.py [--rounds 3] [--bfs-vertices 1000000]
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
from arrow_matrix_b200.decomposition import arrow_decomposition  # noqa: E402
from arrow_matrix_b200.engine import ArrowEngine, bfs_direction  # noqa: E402


def digest(tile, chunk=1 << 20):
    """SHA-1 of a device tile's rows, downloaded in chunks: 10M x 128 tiles are compared without holding several of them
    on the host"""
    h = hashlib.sha1()
    for r0 in range(0, tile.rows, chunk):
        h.update(np.ascontiguousarray(tile.d2h(row0=r0, rows=min(chunk, tile.rows - r0))).tobytes())
    return h.hexdigest()


def clock(fn):
    t = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t) * 1e3, r


def ba_decomposition(n, w, seed=503):
    A = sparse.triu(synth.barabasi_albert(n, 3, seed=seed), k=1).tocoo()
    U = sparse.coo_matrix((np.ones(A.nnz, np.float32), (A.row, A.col)), shape=(n, n))
    return arrow_decomposition(sparse.csr_matrix(U + U.T), w, max_number_of_levels=3, block_diagonal=True, seed=2)


def sources(n, k, rng):
    X0 = np.zeros((n, k), bool)
    X0[rng.choice(n, k, replace=False), np.arange(k)] = True
    return X0


def per_level(eng, X0, max_steps=1000):
    """the launches of ``_betweenness_run`` (automatic direction) with a CUDA event pair around each path-count and each
    dependency pass"""
    eng.zero_rhs()
    eng.set_features(X0)
    ctx, st0 = eng.ctx, eng.levels[0]
    dist, zero, ones = eng._bfs_tiles
    adj, in_adj = eng._adj, eng._in_adj
    sigma, (delta, _) = eng._bfs_sigma, eng._bfs_delta
    sigma.fill(0.0)
    ctx.bits_fill_f64(st0.bufs[st0.xi], zero, sigma, 1.0)
    _, rows, edges = ctx.bits_mark_frontier(adj, st0.bufs[st0.xi], zero, dist, 0)
    ctx.adj_keep_record(adj, 0)
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
        scanned = ctx.bits_path_counts(in_adj, adj, st0.bufs[1 - xi], st0.bufs[xi], sigma, count=True)
        ctx.timer_stop(7)
        ctx.adj_keep_record(adj, level)
        table.append({"level": level, "dir": "push" if push else "pull", "fresh_bits": n_new, "frontier_rows": rows,
                      "in_entries_read": scanned, "path_counts_ms": round(ctx.timer_ms(7), 4)})
        if n_new == 0:
            break
    ctx.bits_mark_new(ones, st0.bufs[st0.xi], dist, -1)
    delta.fill(0.0)
    for row in reversed(table):
        ctx.timer_start(7)
        row["out_entries_read"] = ctx.bits_dependencies(adj, row["level"], dist, sigma, delta, count=True)
        ctx.timer_stop(7)
        row["dependencies_ms"] = round(ctx.timer_ms(7), 4)
    return table


def run_workload(dec, width, k, rng, rounds):
    eng = ArrowEngine(dec, width, k, semiring="or_and", add_identity=True)
    n = eng.n_rows
    X0 = sources(n, k, rng)
    out = {"rows": n, "k": k, "total_nnz": eng.total_nnz, "mode": eng.mode}

    def run(fn):
        eng.zero_rhs()
        eng.set_features(X0)
        eng.sync()
        return clock(lambda: (fn(), eng.sync())[0])

    routes = {"bfs_levels_ms": lambda: eng._bfs_run(1000),
              "path_counts_ms": lambda: eng._bfs_paths_run(1000, "bfs_path_counts"),
              "betweenness_ms": lambda: eng._betweenness_run(1000)}
    for fn in routes.values():                            # warm-up: kernels, tiles, adjacencies and the history
        run(fn)
    times = {key: [] for key in routes}
    seen = set()
    verified = True
    for _ in range(rounds):
        ms, dist = run(routes["bfs_levels_ms"])
        times["bfs_levels_ms"].append(ms)
        L1 = digest(dist)
        steps, dirs = eng.last_bfs_steps, list(eng.last_bfs_directions)
        ms, (dist, sigma) = run(routes["path_counts_ms"])
        times["path_counts_ms"].append(ms)
        L2, S2 = digest(dist), digest(sigma)
        verified &= eng.last_bfs_steps == steps and eng.last_bfs_directions == dirs
        ms, (_, bc) = run(routes["betweenness_ms"])
        times["betweenness_ms"].append(ms)
        L3, S3, B3 = digest(eng._bfs_tiles[0]), digest(eng._bfs_sigma), digest(bc)
        verified &= L1 == L2 == L3 and S2 == S3
        seen.add((L1, S2, B3))
    verified &= len(seen) == 1
    out["steps"] = eng.last_bfs_steps
    out["directions"] = list(eng.last_bfs_directions)
    out.update({key: [round(x, 3) for x in v] for key, v in times.items()})
    best = {key: min(v) for key, v in times.items()}
    out["path_counts_over_levels"] = round(best["path_counts_ms"] / best["bfs_levels_ms"], 3)
    out["betweenness_over_levels"] = round(best["betweenness_ms"] / best["bfs_levels_ms"], 3)
    out["per_level"] = per_level(eng, X0)
    out["history_rows"] = sum(r["frontier_rows"] for r in out["per_level"])
    out["sigma_bytes"] = out["delta_bytes"] = 8 * n * k
    out["verified"] = verified
    eng.close()
    return out


def verify_small(rng):
    """a 20 000-vertex BA graph at k = 32: every result of betweenness() bit for bit the host restatement"""
    from tests import bool_ref as br
    from tests import paths_ref as pa
    from tests import push_ref as pr
    n, w, k = 20000, 2000, 32
    dec = ba_decomposition(n, w, seed=11)
    eng = ArrowEngine(dec, w, k, semiring="or_and", add_identity=True)
    X0 = sources(eng.n_rows, k, rng)
    eng.set_features(X0)
    L, sigma = eng.bfs_path_counts(1000)
    eng.zero_rhs()
    eng.set_features(X0)
    delta = np.empty(sigma.shape)
    bc = eng.betweenness(1000, dependencies_out=delta)
    p = br.BoolProtocol(dec, w, k, n_blocks=eng.n_blocks, add_identity=True)
    want = pa.betweenness(pr.protocol_parts(p), eng.n_rows, X0, 1000)
    eng.close()
    return all(np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
               for a, b in zip((L, sigma, delta, bc), want[:4]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--bfs-vertices", type=int, default=1000000)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bc_bench.py: no CUDA device")
    out = {"rounds": a.rounds, **bench.gpu_info(0)}
    rng = np.random.default_rng(42)
    out["verified_small"] = verify_small(rng)
    print(json.dumps({"verified_small": out["verified_small"], **bench.gpu_info(0)}), flush=True)
    g2 = synth.synth_decomposition(a.blocks, a.width, levels=2, perm_kind="random", seed=503)
    for k in (16, 128):
        out[f"g2_k{k}"] = run_workload(g2, a.width, k, rng, a.rounds)
        print(json.dumps({f"g2_k{k}": out[f"g2_k{k}"], **bench.gpu_info(0)}), flush=True)   # each workload as it ends
    del g2
    out["ba_k128"] = run_workload(ba_decomposition(a.bfs_vertices, 20000), 20000, 128, rng, a.rounds)
    print(json.dumps({"ba_k128": out["ba_k128"], **bench.gpu_info(0)}), flush=True)
    out["verified"] = out["verified_small"] and all(out[x]["verified"] for x in ("g2_k16", "g2_k128", "ba_k128"))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
