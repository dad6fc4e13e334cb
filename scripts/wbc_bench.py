"""Weighted betweenness on one GPU: ``iterate_to_fixed_point`` (distances only), ``shortest_path_counts`` (distances and
tight shortest-path counts) and ``weighted_betweenness`` (counts, the backward sweep over the tight-pair rounds and the
row sum) of a ``min_plus`` engine with the identity, in one process.

Workloads (those of scripts/bc_bench.py, one source per column at random rows):
  * G2 of bench.py (10M rows, width 10 000, two levels, ~10 nnz/row, random level-1 permutation, seed 503) at k = 16 and
    k = 128;
  * the 10**6-vertex Barabasi-Albert graph (m = 3, width 20 000, 3 levels) at k = 128;
each with seeded integer weights 1..16 on every entry (exact sums, many ties) and with unit weights.

For each, 3 rounds, the routes alternating within a round on the same sources, host clock around work that ends in a
synchronise, results left on the device; on unit weights also the ``or_and`` engine's ``betweenness`` on the same
decomposition (run after the ``min_plus`` engine is closed, so the two never share the card).  Per round: the routes' ms,
the tight-pair rounds and the list entries read by the passes of one more call.  ``verified``: the three routes give the
same distances, every round the same bits, the unit-weight distances, counts, dependencies and betweenness equal the
``or_and`` levels and results bit for bit; and, at a reduced size (a 20 000-vertex weighted BA graph, k = 32), every
result equals tests/wpaths_ref.py bit for bit.  One JSON line per workload as it ends, then one with them all, each with
the card and its power limit.

    python scripts/wbc_bench.py [--rounds 3] [--blocks 1000] [--bfs-vertices 1000000] [--workloads g2_k16_w16,...]
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
from arrow_matrix_b200.engine import ArrowEngine  # noqa: E402


def digest(tile, as_levels=False, chunk=1 << 20):
    """SHA-1 of a device tile's rows, downloaded in chunks; ``as_levels`` hashes float distances as int32 hop levels
    (-1 where not finite), the layout of ``bfs_levels``"""
    h = hashlib.sha1()
    for r0 in range(0, tile.rows, chunk):
        x = tile.d2h(row0=r0, rows=min(chunk, tile.rows - r0))
        if as_levels:
            x = np.where(np.isfinite(x), x, -1).astype(np.int32)
        h.update(np.ascontiguousarray(x).tobytes())
    return h.hexdigest()


def clock(fn):
    t = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t) * 1e3, r


def weighted(dec, unit, seed=7):
    """the decomposition with seeded integer weights 1..16 (or 1) on every entry"""
    rng = np.random.default_rng(seed)
    out = []
    for B, perm in dec:
        B = sparse.csr_matrix(B, dtype=np.float32, copy=True)
        B.data = np.ones(B.nnz, np.float32) if unit else rng.integers(1, 17, B.nnz).astype(np.float32)
        out.append((B, perm))
    return out


def ba_decomposition(n, w, seed=503):
    A = sparse.triu(synth.barabasi_albert(n, 3, seed=seed), k=1).tocoo()
    U = sparse.coo_matrix((np.ones(A.nnz, np.float32), (A.row, A.col)), shape=(n, n))
    return arrow_decomposition(sparse.csr_matrix(U + U.T), w, max_number_of_levels=3, block_diagonal=True, seed=2)


def sources(n, k, seed):
    X0 = np.full((n, k), np.inf, np.float32)
    X0[np.random.default_rng(seed).choice(n, k, replace=False), np.arange(k)] = 0.0
    return X0


def entries_read(eng):
    """list entries read by the passes of the last weighted call, re-run on its tiles (the rounds' rows are kept)"""
    ctx = eng.ctx
    x0, state, sigma = eng._wp_tiles
    D = eng.features_buffer()
    _, fwd = ctx.wpaths_counts(eng._wp_adjs[0], eng._wp_adjs[1], x0, D, state, sigma, count=True)
    bwd = ctx.wpaths_dependencies(eng._wp_adjs[1], x0, D, state, sigma, eng._wp_delta[0], count=True)
    return fwd, bwd


def run_workload(dec, width, k, unit, rounds, seed):
    eng = ArrowEngine(dec, width, k, semiring="min_plus", add_identity=True)
    n = eng.n_rows
    X0 = sources(n, k, seed)
    out = {"rows": n, "k": k, "weights": "1" if unit else "1..16", "total_nnz": eng.total_nnz, "mode": eng.mode}

    def run(fn):
        eng.set_features(X0)
        eng.sync()
        return clock(lambda: (fn(), eng.sync())[0])

    routes = {"fixed_point_ms": lambda: eng.iterate_to_fixed_point(10000),
              "path_counts_ms": lambda: eng._wpaths_run(10000, "shortest_path_counts"),
              "weighted_betweenness_ms": lambda: eng._wbc_run(10000)}
    for fn in routes.values():                            # warm-up: kernels, tiles and adjacencies
        run(fn)
    table, seen, verified = [], set(), True
    for r in range(rounds):
        row = {"round": r}
        row["fixed_point_ms"], _ = run(routes["fixed_point_ms"])
        dirs = list(eng.last_fixed_point_directions)
        steps = len(dirs)
        D1 = digest(eng.features_buffer())
        row["path_counts_ms"], (D, sigma) = run(routes["path_counts_ms"])
        D2, S2 = digest(D), digest(sigma)
        verified &= list(eng.last_fixed_point_directions) == dirs
        row["weighted_betweenness_ms"], _ = run(routes["weighted_betweenness_ms"])
        D3, S3 = digest(eng.features_buffer()), digest(eng._wp_tiles[2])
        B3, T3 = digest(eng._wp_delta[1]), digest(eng._wp_delta[0])
        verified &= D1 == D2 == D3 and S2 == S3
        seen.add((D1, S2, T3, B3))
        row["dag_rounds"] = eng.last_path_rounds
        table.append(row)
    verified &= len(seen) == 1
    out["steps"] = steps
    out["directions"] = dirs
    out["forward_entries_read"], out["backward_entries_read"] = entries_read(eng)
    for row in table:
        row["rows"] = n
        row["entries_read"] = out["forward_entries_read"] + out["backward_entries_read"]
    out["per_round"] = table
    best = {key: min(r[key] for r in table) for key in routes}
    out["path_counts_over_fixed_point"] = round(best["path_counts_ms"] / best["fixed_point_ms"], 3)
    out["betweenness_over_fixed_point"] = round(best["weighted_betweenness_ms"] / best["fixed_point_ms"], 3)
    levels, sig, dep, bc = D1, S2, T3, B3
    if unit:
        levels = digest(eng.features_buffer(), as_levels=True)
    eng.close()
    if unit:                                              # the or_and engine on the same decomposition and sources
        bits = ArrowEngine(dec, width, k, semiring="or_and", add_identity=True)
        Xb = X0 == 0
        ms = []
        for _ in range(rounds + 1):
            bits.zero_rhs()
            bits.set_features(Xb)
            bits.sync()
            t, _ = clock(lambda: (bits._betweenness_run(10000), bits.sync()))
            ms.append(t)
        for row, t in zip(table, ms[1:]):
            row["or_and_betweenness_ms"] = t
        same = [levels == digest(bits._bfs_tiles[0]), sig == digest(bits._bfs_sigma),
                dep == digest(bits._bfs_delta[0]), bc == digest(bits._bfs_delta[1])]
        out["equals_or_and"] = all(same)
        verified &= all(same)
        bits.close()
    for row in table:
        for key in list(row):
            if key.endswith("_ms"):
                row[key] = round(row[key], 3)
    out["verified"] = bool(verified)
    return out


def verify_small():
    """a 20 000-vertex weighted BA graph at k = 32: every result bit for bit the host restatement"""
    from tests import bool_ref as br
    from tests import push_ref as pr
    from tests import wpaths_ref as wp
    n, w, k = 20000, 2000, 32
    dec = weighted(ba_decomposition(n, w, seed=11), False, seed=3)
    eng = ArrowEngine(dec, w, k, semiring="min_plus", add_identity=True)
    X0 = sources(eng.n_rows, k, 1)
    eng.set_features(X0)
    D, sigma = eng.shortest_path_counts(10000)
    eng.set_features(X0)
    delta = np.empty(sigma.shape)
    bc = eng.weighted_betweenness(10000, dependencies_out=delta)
    p = br.BoolProtocol(dec, w, k, n_blocks=eng.n_blocks, add_identity=True)
    parts = pr.protocol_parts(p)
    want = wp.betweenness(parts, eng.n_rows, X0, 10000)
    eng.close()
    return all(np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
               for a, b in zip((D, sigma, delta, bc), want))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--bfs-vertices", type=int, default=1000000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="g2_k16_w16,g2_k16_unit,g2_k128_w16,g2_k128_unit,ba_k128_w16,ba_k128_unit",
                    help="comma-separated subset of the workloads to run")
    a = ap.parse_args()
    chosen = a.workloads.split(",")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("wbc_bench.py: no CUDA device")
    out = {"rounds": a.rounds, **bench.gpu_info(0)}
    out["verified_small"] = verify_small()
    print(json.dumps({"verified_small": out["verified_small"], **bench.gpu_info(0)}), flush=True)
    names = []
    if any(x.startswith("g2") for x in chosen):
        g2 = synth.synth_decomposition(a.blocks, a.width, levels=2, perm_kind="random", seed=503)
        for k in (16, 128):
            for unit in (False, True):
                name = f"g2_k{k}_{'unit' if unit else 'w16'}"
                if name in chosen:
                    out[name] = run_workload(weighted(g2, unit), a.width, k, unit, a.rounds, k)
                    names.append(name)
                    print(json.dumps({name: out[name], **bench.gpu_info(0)}), flush=True)   # each workload as it ends
        del g2
    if any(x.startswith("ba") for x in chosen):
        ba = ba_decomposition(a.bfs_vertices, 20000)
        for unit in (False, True):
            name = f"ba_k128_{'unit' if unit else 'w16'}"
            if name in chosen:
                out[name] = run_workload(weighted(ba, unit), 20000, 128, unit, a.rounds, 128)
                names.append(name)
                print(json.dumps({name: out[name], **bench.gpu_info(0)}), flush=True)
    out["verified"] = out["verified_small"] and all(out[x]["verified"] for x in names)
    print(json.dumps({"verified": out["verified"], **bench.gpu_info(0)}))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
