"""Personalized PageRank on one GPU (ArrowEngine.pagerank): cost per step beside a plain step, the update pass alone,
the one-time set-up and the steps to tol.

Workloads, one random seed vertex per column, alpha = 0.85, tol = 1e-6:
  * G2 of bench.py (10M rows, width 10 000, two levels, seed 503; absolute values) at k = 16 and 128 in float32 and at
    k = 16 in float64;
  * the 10**6-vertex Barabasi-Albert graph of scripts/bc_bench.py at k = 128.

Each workload prints one JSON line with the card and its power limit.  Within each of the rounds the routes alternate:
``step_ms`` is a plain ``step()`` on the rewound features, ``pagerank_step_ms`` one scaled step plus its update, both
over ``--steps`` steps after a synchronise; ``update_ms`` is the update pass alone (CUDA events over ``--steps``
launches on the same tiles, its chunk-sum kernel and the residual copy included) with its rate over 4 tile passes
(read Y, p, S; write p).  ``setup_ms`` is the out-weight pass plus the scaled operands, ``steps_to_tol`` and
``to_tol_ms`` one full call.  ``verified`` holds when every column of p sums to 1 within the mass bound below, p >= 0,
two calls give the same bits and, on a 100 000-row G2, the loop stays within tests/pagerank_ref.py's error bound.

Mass bound: each iterate adds at most eps = gamma_{h + 5}(u_T) + gamma_cm(u_64) relative error per element (h the
largest per-row step height, tests/step_bound.py; cm = 512 + chunks + 2) and Phi keeps the mass within eta =
gamma_2(u_T) + gamma_{d + 1}(u_64) (d the largest row length of any level, an upper bound of the out-degree over one
level times the levels), so after T steps |sum p - 1| <= ((1 + eps)(1 + eta))^T (1 + gamma_1(u_T) + gamma_cm(u_64)) - 1
plus the float64 summation of the check itself.
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
from tests.spmm_bound import U32, U64, gamma, tree_height  # noqa: E402

ALPHA, TOL = 0.85, 1e-6


def digest(a) -> str:
    return hashlib.sha1(np.ascontiguousarray(a).view(np.uint8)).hexdigest()


def g2(blocks, width):
    dec = synth.synth_decomposition(blocks, width, levels=2, perm_kind="random", seed=503)
    return [(abs(sparse.csr_matrix(B)), p) for B, p in dec]


def ba_decomposition(n, w, seed=503):
    A = sparse.triu(synth.barabasi_albert(n, 3, seed=seed), k=1).tocoo()
    U = sparse.coo_matrix((np.ones(A.nnz, np.float32), (A.row, A.col)), shape=(n, n))
    return arrow_decomposition(sparse.csr_matrix(U + U.T), w, max_number_of_levels=3, block_diagonal=True, seed=2)


def seeds(n, k, rng, dtype):
    X0 = np.zeros((n, k), dtype)
    X0[rng.integers(0, n, k), np.arange(k)] = 1
    return X0


def mass_bound(eng, steps) -> float:
    u = U32 if eng.dtype == np.float32 else U64
    info = [st.csr.info() for st in eng.levels]
    h = sum(int(tree_height(i["max_row_nnz"])) + 1 for i in info)
    d = sum(i["max_row_nnz"] for i in info)
    cm = 512 + (eng.n_rows + 511) // 512 + 2
    eps = gamma(h + 5, u) + gamma(cm, U64)
    eta = gamma(2, u) + gamma(d + 1, U64)
    return float(((1 + eps) * (1 + eta)) ** steps * (1 + gamma(1, u) + gamma(cm, U64)) - 1 + gamma(eng.n_rows, U64))


def run_workload(dec, width, k, dtype, rng, rounds, steps):
    eng = ArrowEngine(dec, width, k, dtype=dtype)
    n = eng.n_rows
    X0 = seeds(n, k, rng, dtype)
    ctx = eng.ctx
    out = {"rows": n, "k": k, "dtype": np.dtype(dtype).name, "total_nnz": eng.total_nnz, "mode": eng.mode}
    eng.set_features(X0)
    eng.sync()
    t = time.perf_counter()
    eng._pagerank_prepare()
    out["setup_ms"] = round((time.perf_counter() - t) * 1e3, 3)
    S, scratch, state = eng._pr_work
    inv = eng._pr_weights[1]
    st0 = eng.levels[0]

    def plain():
        eng.set_features(X0)
        eng.sync()
        t = time.perf_counter()
        for _ in range(steps):
            eng.rewind_features()
            eng.step()
        eng.sync()
        return (time.perf_counter() - t) * 1e3 / steps

    def scaled():
        eng.features_buffer().copy_from(S)                    # p_0 = S (the restart of the first call below)
        eng.sync()
        t = time.perf_counter()
        for _ in range(steps):
            p_tile = eng._pagerank_step()
            ctx.pagerank_update(st0.bufs[st0.xi], p_tile, S, inv, scratch, state, ALPHA)
        return (time.perf_counter() - t) * 1e3 / steps

    def update():
        eng.features_buffer().copy_from(S)
        p = eng._pagerank_step()
        y = st0.bufs[st0.xi]
        ctx.timer_start(6)
        for _ in range(steps):
            ctx.pagerank_update(y, p, S, inv, scratch, state, ALPHA)
        ctx.timer_stop(6)
        return ctx.timer_ms(6) / steps

    p = np.empty((n, k), dtype)
    eng.pagerank(0, out=p)                                    # the restart: S and m_0
    plain(), scaled(), update()                               # warm-up
    times = {"step_ms": [], "pagerank_step_ms": [], "update_ms": []}
    for _ in range(rounds):
        times["step_ms"].append(plain())
        times["pagerank_step_ms"].append(scaled())
        times["update_ms"].append(update())
    out.update({key: [round(x, 4) for x in v] for key, v in times.items()})
    tile_bytes = n * k * np.dtype(dtype).itemsize
    out["update_bytes"] = 4 * tile_bytes
    out["update_gb_per_s"] = round(4 * tile_bytes / (min(times["update_ms"]) * 1e-3) / 1e9, 1)
    out["pagerank_over_step"] = round(min(times["pagerank_step_ms"]) / min(times["step_ms"]), 3)
    digests, verified = set(), True
    for _ in range(2):
        eng.set_features(X0)
        eng.sync()
        t = time.perf_counter()
        eng.pagerank(1000, ALPHA, TOL, out=p)
        out["to_tol_ms"] = round((time.perf_counter() - t) * 1e3, 3)       # the download of p included
        digests.add(digest(p) + digest(eng.last_pagerank_residuals))
        sums = np.zeros(k)
        for r0 in range(0, n, 1 << 20):
            blk = p[r0:r0 + (1 << 20)]
            verified &= bool(np.all(blk >= 0))
            sums += blk.sum(axis=0, dtype=np.float64)
        err = float(np.max(np.abs(sums - 1)))
        out["mass_error"], out["mass_bound"] = err, mass_bound(eng, len(eng.last_pagerank_residuals))
        verified &= err <= out["mass_bound"]
    out["steps_to_tol"] = int(len(eng.last_pagerank_residuals))
    out["verified"] = bool(verified and len(digests) == 1)
    out["memory_bytes"] = {"S": tile_bytes, "w_inv": n * (8 + np.dtype(dtype).itemsize),
                           "scaled_values": eng.total_nnz * np.dtype(dtype).itemsize, "scratch": 16 * k * ((n + 511) // 512)}
    eng.close()
    return out


def verify_small(rng) -> float:
    """worst err / bound of the loop on a 100 000-row G2 at k = 16 (float32, 8 steps): <= 1 holds the bound"""
    from tests import pagerank_ref as prr
    dec = g2(10, 10000)
    eng = ArrowEngine(dec, 10000, 16)
    X0 = seeds(eng.n_rows, 16, rng, np.float32)
    eng.set_features(X0)
    p = eng.pagerank(8, ALPHA, 0.0)
    eng.close()
    parts, proto = prr.level_parts(dec, 10000)
    walk = prr.Walk(parts, proto.rows[0], np.float32, proto.to_prev, 10000)
    _, _, its = walk.loop64(X0, ALPHA, 0.0, 8)
    err = np.abs(p.astype(np.float64) - its[-1]).sum(axis=0)
    return float(np.max(err / walk.bound(its, ALPHA)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--ba-vertices", type=int, default=1000000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("pagerank_bench.py: no CUDA device")
    info = bench.gpu_info(0)
    rng = np.random.default_rng(42)
    out = {"rounds": a.rounds, "steps": a.steps, **info}
    out["small_err_over_bound"] = verify_small(rng)
    print(json.dumps({"small_err_over_bound": out["small_err_over_bound"], **info}), flush=True)
    dec = g2(a.blocks, a.width)
    for name, k, dtype in (("g2_k16", 16, np.float32), ("g2_k128", 128, np.float32), ("g2_k16_f64", 16, np.float64)):
        out[name] = run_workload(dec, a.width, k, dtype, rng, a.rounds, a.steps)
        print(json.dumps({name: out[name], **info}), flush=True)
    del dec
    out["ba_k128"] = run_workload(ba_decomposition(a.ba_vertices, 20000), 20000, 128, np.float32, rng, a.rounds, a.steps)
    print(json.dumps({"ba_k128": out["ba_k128"], **info}), flush=True)
    out["verified"] = out["small_err_over_bound"] <= 1.0 and all(
        out[x]["verified"] for x in ("g2_k16", "g2_k128", "g2_k16_f64", "ba_k128"))
    print(json.dumps(out))
    print(f"verified: {str(out['verified']).lower()}")


if __name__ == "__main__":
    main()
