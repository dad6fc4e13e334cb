"""Connected components on one GPU (ArrowEngine.connected_components): the whole call, the hook pass alone, a plain step
for scale and scipy on the host.

Workloads:
  * G2 of bench.py (10M rows, width 10 000, two levels, seed 503);
  * the 10**6-vertex Barabasi-Albert graph of scripts/bc_bench.py (m = 3, width 20 000, at most three levels).

Each workload prints one JSON line with the card and its power limit, read in the same run.  Fields:
  * ``cc_ms``: the whole call, warm (host clock around ``connected_components()``, which ends in a device synchronise and
    includes the download of the labels), every repetition listed;
  * ``hook_ms``: the hook pass alone (the ``k_cc_hook`` launches of one call, one per level), CUDA kernel time from
    ``torch.profiler``'s activity records over the repetitions of a separate profiled run, per call; ``init_ms`` and
    ``label_ms`` likewise for the other two passes, ``download_ms`` the host clock around the labels' download alone;
  * ``hook_bytes`` / ``hook_gb_per_s``: the algorithmic bytes of the hook pass over ``hook_ms``.  Per level j, every
    entry reads its column index (4 B), the parents of its two ends (8 B) and, for j >= 1, the row map of both ends
    (8 B); the row pointers are read once (4 (rows_j + 1) B).  Root walks beyond the first parent, the CASes and the
    row searches are not counted: the figure is a lower bound of the traffic;
  * ``step_ms_k16``: a plain ``step()`` of the same engine (plus_times, float32, k = 16), CUDA events over ``--steps``
    steps on rewound features; ``cc_over_step`` the median call over it;
  * ``scipy_ms``: ``scipy.sparse.csgraph.connected_components(directed=True, connection="weak")`` on the host, one
    thread (it has no parallel path), on the structural operator of tests/cc_ref.py (its construction not timed);
  * ``verified``: labels, count and sizes equal tests/cc_ref.py bit for bit and two calls give the same bits.  The host
    restatement of the full G2 (150M entries) needs more host memory than the device run, so G2 is verified, and timed
    on the host, at 100 000 rows (``small``); the BA graph at full size.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (gpu_info)
from arrow_matrix_b200 import synth  # noqa: E402
from arrow_matrix_b200.engine import ArrowEngine  # noqa: E402
from scripts.bc_bench import ba_decomposition  # noqa: E402
from tests import cc_ref  # noqa: E402
from tests import pagerank_ref as prr  # noqa: E402


def g2(blocks, width):
    return synth.synth_decomposition(blocks, width, levels=2, perm_kind="random", seed=503)


def hook_bytes(eng) -> int:
    return sum(st.nnz * (12 + (8 if j > 0 else 0)) + 4 * (st.rows + 1) for j, st in enumerate(eng.levels))


def pass_kernel_ms(eng, reps):
    """CUDA time per call of the init, hook and label launches, from torch.profiler's kernel records (None for a pass it
    recorded no launch of)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            eng.connected_components()
    us = {}
    for ev in prof.key_averages():
        for name in ("k_cc_init", "k_cc_hook", "k_cc_label"):
            if name in ev.key:
                us[name] = us.get(name, 0.0) + (getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0))
    return {name: round(us[name] / 1e3 / reps, 4) if name in us else None for name in ("k_cc_init", "k_cc_hook", "k_cc_label")}


def step_ms(eng, steps):
    X = np.zeros((eng.n_rows, eng.k), np.float32)
    X[np.random.default_rng(1).integers(0, eng.n_rows, eng.k), np.arange(eng.k)] = 1
    eng.set_features(X)
    for _ in range(3):
        eng.rewind_features()
        eng.step()
    eng.sync()
    eng.ctx.timer_start(6)
    for _ in range(steps):
        eng.rewind_features()
        eng.step()
    eng.ctx.timer_stop(6)
    return round(eng.ctx.timer_ms(6) / steps, 4)


def host(dec, width):
    """(labels, count, sizes) of tests/cc_ref.py and the csgraph time alone"""
    from scipy.sparse import csgraph
    parts, proto = prr.level_parts(dec, width)
    S = cc_ref.structural(parts, proto.rows[0])
    t = time.perf_counter()
    csgraph.connected_components(S, directed=True, connection="weak")
    ms = (time.perf_counter() - t) * 1e3
    return cc_ref.components(parts, proto.rows[0]), round(ms, 3)


def device(dec, width, reps, steps, verify):
    eng = ArrowEngine(dec, width, 16)
    n = eng.n_rows
    out = {"rows": n, "levels": eng.L, "total_nnz": eng.total_nnz, "mode": eng.mode}
    sizes = np.empty(n, np.int32)
    first = eng.connected_components(sizes_out=sizes)                # allocates the tiles, loads the kernels
    eng.connected_components()
    times = []
    for _ in range(reps):
        t = time.perf_counter()
        labels = eng.connected_components()
        times.append((time.perf_counter() - t) * 1e3)
    out["cc_ms"] = [round(x, 4) for x in times]
    out["cc_ms_median"] = round(statistics.median(times), 4)
    out["components"] = eng.last_component_count
    passes = pass_kernel_ms(eng, reps)
    out["hook_ms"], out["init_ms"], out["label_ms"] = passes["k_cc_hook"], passes["k_cc_init"], passes["k_cc_label"]
    t = time.perf_counter()
    eng._cc_labels.d2h()
    out["download_ms"] = round((time.perf_counter() - t) * 1e3, 4)
    out["hook_bytes"] = hook_bytes(eng)
    if out["hook_ms"]:
        out["hook_gb_per_s"] = round(out["hook_bytes"] / (out["hook_ms"] * 1e-3) / 1e9, 1)
    out["step_ms_k16"] = step_ms(eng, steps)
    out["cc_over_step"] = round(out["cc_ms_median"] / out["step_ms_k16"], 3)
    out["memory_bytes"] = 8 * n
    same = bool(np.array_equal(first, labels))
    count = eng.last_component_count
    eng.close()
    if verify:
        (want, want_count, want_sizes), out["scipy_ms"] = host(dec, width)
        out["scipy_threads"] = 1
        out["verified"] = bool(same and np.array_equal(labels, want) and count == want_count
                               and np.array_equal(sizes, want_sizes))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--ba-vertices", type=int, default=1000000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("cc_bench.py: no CUDA device")
    torch.cuda.init()
    info = bench.gpu_info(0)
    out = {"reps": a.reps, **info}
    g = device(g2(a.blocks, a.width), a.width, a.reps, a.steps, verify=False)
    g["small"] = device(g2(10, a.width), a.width, a.reps, a.steps, verify=True)
    g["verified"] = g["small"]["verified"]
    out["g2"] = g
    print(json.dumps({"g2": g, **info}), flush=True)
    out["ba"] = device(ba_decomposition(a.ba_vertices, 20000), 20000, a.reps, a.steps, verify=True)
    print(json.dumps({"ba": out["ba"], **info}), flush=True)
    out["verified"] = bool(out["g2"]["verified"] and out["ba"]["verified"])
    print(json.dumps(out))
    print(f"verified: {str(out['verified']).lower()}")


if __name__ == "__main__":
    main()
