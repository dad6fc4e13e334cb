"""float32 vs float64 step on the benchmark workload, one GPU; prints one JSON line.

The workload of ``bench.py``: the synthetic arrow decomposition with 10M rows (1000 blocks of width 10 000), 2 levels and
a random level-1 permutation (seed 503), written as level files to a temporary directory and loaded through
``ArrowDecompositionMPI`` with ``datatype`` float32 and float64, at k = 128 and k = 16.  Each engine is closed before
the next one is built (float64 at k = 128 holds about 38 GB).

Per (k, dtype): the device-resident step time (CUDA events, warm-up first, the features rewound before every step as
``bench.py`` does), the level-0 launch alone (``time_level_spmm``), the algorithmic bytes with the element size and
their fraction of the H100 SXM data-sheet bandwidth (3.35 TB/s).  The features are rank-1, ``X = u v^T``; for float64 the
last timed step must equal ``(S u) v^T`` within ``1e-12 * max|(S u) v^T|``, with the step ``S`` applied to ``u`` in
``np.longdouble`` on the host (``verified``).
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from arrow_matrix_b200 import decomp, graphio, synth                  # noqa: E402
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI      # noqa: E402
from arrow_matrix_b200.comm import SelfComm                            # noqa: E402

PEAK_GBS = 3350.0              # H100 SXM data sheet
CHUNK = 1 << 20                # host rows per transfer: the full float64 feature matrix never exists on the host


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return out[0].strip(), float(out[1])
    except Exception:
        return None, None


def rank1(n, k):
    u = 2.0 * np.random.default_rng(9001).random(n) - 1.0
    v = 0.5 + np.random.default_rng(9002).random(k)
    return u, v


def step_on_vector(dec, width, u):
    """one step applied to ``u`` (level-0 order) in np.longdouble: forward maps, every level's arrow blocks, backward
    scatter-add.  Only valid when no non-zero reads a row behind the sentinel (checked)."""
    from scipy import sparse
    n_blocks = [decomp.number_of_blocks(B, width) for B, _ in dec]
    _, to_prev, _, _ = decomp.prepare_permutations([p for _, p in dec], n_blocks, width)
    rows = [int(b) * width for b in n_blocks]
    x = [np.asarray(u, dtype=np.longdouble)]
    fed = [np.ones(rows[0], dtype=bool)]
    for j in range(1, len(dec)):
        tp = to_prev[j][: rows[j]]
        valid = tp < rows[j - 1]
        safe = np.where(valid, tp, 0)
        fed.append(valid & fed[j - 1][safe])
        x.append(np.where(fed[j], x[j - 1][safe], 0).astype(np.longdouble))
    c = []
    for j, (B, _) in enumerate(dec):
        ip, idx, dat, _ = decomp.arrow_rows(B, width, n_blocks[j], True, 0, rows[j], dtype=np.float64)
        assert not idx.size or bool(fed[j][idx].all()), "a non-zero reads a row behind the sentinel"
        vals = np.ones(idx.size) if dat is None else dat
        c.append(sparse.csr_matrix((vals.astype(np.longdouble), idx, ip), shape=(rows[j], rows[j])) @ x[j])
    for j in range(len(dec) - 1, 0, -1):
        tp = to_prev[j][: rows[j]]
        valid = tp < rows[j - 1]
        c[j - 1][tp[valid]] += c[j][valid]
    return c[0]


def run_one(base, width, k, dtype, steps, warmup, u, v, expected):
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, width, True, dtype,
                                                                                      slim=True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, width, k, 'gpu', True, True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    arrow.B.zero_rhs(width, k, dtype=dtype)
    eng = arrow._engine
    ctx = eng.ctx
    n = eng.n_rows
    eng.rewind_features()
    xbuf = eng.features_buffer()
    for r0 in range(0, n, CHUNK):
        xbuf.h2d(np.outer(u[r0:r0 + CHUNK], v).astype(dtype), r0)
        ctx.sync()
    for _ in range(warmup):
        eng.rewind_features()
        eng.step()
    ctx.sync()
    ctx.timer_start(0)
    for _ in range(steps):
        eng.rewind_features()
        eng.step()
    ctx.timer_stop(0)
    ms = ctx.timer_ms(0) / steps
    out = {"k": k, "dtype": np.dtype(dtype).name, "mode": eng.mode, "step_ms": ms,
           "algorithmic_bytes_per_step": eng.algorithmic_bytes_per_step(),
           "step_frac_of_3350_GBs": eng.algorithmic_bytes_per_step() / ms / 1e6 / PEAK_GBS}
    if expected is not None:
        res = eng.result_buffer(0)
        scale = float(np.max(np.abs(expected))) * float(np.max(np.abs(v)))
        worst = 0.0
        host = np.empty((CHUNK, k), dtype=np.float64)
        for r0 in range(0, n, CHUNK):
            rows = min(CHUNK, n - r0)
            got = res.d2h(host[:rows], r0, rows)
            want = np.outer(expected[r0:r0 + rows], v.astype(np.longdouble))
            worst = max(worst, float(np.max(np.abs(got.astype(np.longdouble) - want))))
        out["rank1_max_abs_err"] = worst
        out["rank1_scale"] = scale
        out["verified"] = bool(worst <= 1e-12 * scale)
    level_ms = eng.time_level_spmm(0, steps)
    out["level0_ms"] = level_ms
    out["level0_bytes"] = eng.level_bytes(0)
    out["level0_frac_of_3350_GBs"] = eng.level_bytes(0) / level_ms / 1e6 / PEAK_GBS
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--ks", type=str, default="128,16")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    workdir = tempfile.mkdtemp(prefix="arrow_fp64_bench_")
    try:
        base = os.path.join(workdir, "bench")
        dec = synth.synth_decomposition(a.blocks, a.width, levels=2, perm_kind="random", seed=503)
        graphio.save_decomposition_new(dec, base, a.width, block_diagonal=True)
        del dec
        mapped = graphio.load_decomposition_new(base, a.width, block_diagonal=True, mem_map=True)
        u, v = rank1(a.blocks * a.width, max(int(k) for k in a.ks.split(",")))
        expected = step_on_vector(mapped, a.width, u)
        runs = []
        for k in (int(x) for x in a.ks.split(",")):
            for dtype in (np.float32, np.float64):
                runs.append(run_one(base, a.width, k, dtype, a.steps, a.warmup, u, v[:k],
                                    expected if dtype == np.float64 else None))
        ratios = {}
        for r in runs:
            if r["dtype"] == "float64":
                f32 = next(x for x in runs if x["k"] == r["k"] and x["dtype"] == "float32")
                ratios[f"k{r['k']}"] = {"step": r["step_ms"] / f32["step_ms"], "level0": r["level0_ms"] / f32["level0_ms"]}
        name, power = gpu_info()
        print(json.dumps({"workload": f"{a.blocks * a.width} rows, width {a.width}, 2 levels, random level-1 permutation "
                                      f"(seed 503)", "gpu": name, "power_limit_w": power, "peak_gbs": PEAK_GBS,
                          "runs": runs, "fp64_over_fp32": ratios,
                          "verified": all(r.get("verified", True) for r in runs)}))
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


if __name__ == "__main__":
    main()
