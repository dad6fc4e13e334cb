"""How much does the window of rows in flight cost the tile kernels?  One process, one GPU, JSON lines.

The persistent tile CTAs take row tiles from one atomic ticket, so the rows in flight are about
``resident CTAs x rows per tile``.  At width 10 000 and k = 128 that window touches 3-4 block-rows, whose X panels
(``w * k * elem`` bytes each, plus the head panel every row reads) must stay in L2 for the gathers to hit it.  This script
changes the window without touching the kernels and times the result:

1. the L2 -> SM gather probes of ``scripts/probe_gather.py`` (the gather roof of the card);
2. G2 of ``bench.py`` (10M rows, width 10 000, 2 levels, random level-1 permutation, seed 503) written as level files
   and loaded through ``ArrowDecompositionMPI``; for float32 k = 128, float32 k = 16 and float64 k = 128 the
   device-resident step and the level-0 launch (``time_level_spmm(0)``) under every combination of
   ``ARROW_OPT_SPMM_CTAS_PER_SM`` (``--ctas``), ``ARROW_OPT_SPMM_SM_LIMIT`` (``--sm-limits``) and
   ``ARROW_OPT_TILE_ROWS`` (``--tile-rows``), the combinations repeated ``--reps`` times in alternation.

Every line carries the GPU name, its power limit and the SM clock read right after the measurement.
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
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

from arrow_matrix_b200 import graphio, synth                            # noqa: E402
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI      # noqa: E402
from arrow_matrix_b200.comm import SelfComm                            # noqa: E402

CHUNK = 1 << 20


def gpu_state():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1]), "sm_mhz": float(out[2]),
                "sm_mhz_max": float(out[3])}
    except Exception:
        return {"gpu": None}


def load(base, width, k, dtype):
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, width, True, dtype,
                                                                                      slim=True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, width, k, 'gpu', True, True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    arrow.B.zero_rhs(width, k, dtype=dtype)
    eng = arrow._engine
    rng = np.random.default_rng(9001)
    v = 0.5 + rng.random(k)
    xbuf = eng.features_buffer()
    for r0 in range(0, eng.n_rows, CHUNK):
        u = 2.0 * rng.random(min(CHUNK, eng.n_rows - r0)) - 1.0
        xbuf.h2d(np.outer(u, v).astype(dtype), r0)
        eng.ctx.sync()
    return eng


def time_step(eng, steps, warmup):
    for _ in range(warmup):
        eng.rewind_features()
        eng.step()
    eng.ctx.sync()
    eng.ctx.timer_start(0)
    for _ in range(steps):
        eng.rewind_features()
        eng.step()
    eng.ctx.timer_stop(0)
    return eng.ctx.timer_ms(0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--width", type=int, default=10000)
    ap.add_argument("--cases", type=str, default="float32:128,float32:16,float64:128")
    ap.add_argument("--ctas", type=str, default="4,3,2")
    ap.add_argument("--sm-limits", type=str, default="0,66")
    ap.add_argument("--tile-rows", type=str, default="", help="ARROW_OPT_TILE_ROWS values to sweep (empty: not set)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-gather-probe", action="store_true")
    a = ap.parse_args()

    if not a.no_gather_probe:
        import probe_gather
        probe_gather.main()

    tile_rows = [int(x) for x in a.tile_rows.split(",")] if a.tile_rows else [None]
    configs = [(c, s, t) for t in tile_rows for s in (int(x) for x in a.sm_limits.split(","))
               for c in (int(x) for x in a.ctas.split(","))]
    workdir = tempfile.mkdtemp(prefix="arrow_window_probe_")
    try:
        base = os.path.join(workdir, "g2")
        dec = synth.synth_decomposition(a.blocks, a.width, levels=2, perm_kind="random", seed=503)
        graphio.save_decomposition_new(dec, base, a.width, block_diagonal=True)
        del dec
        for case in a.cases.split(","):
            dname, k = case.split(":")
            k = int(k)
            eng = load(base, a.width, k, np.dtype(dname).type)
            ctx = eng.ctx
            for rep in range(a.reps):
                for ctas, sms, tr in configs:
                    ctx.set_option(ctx.OPT_SPMM_CTAS_PER_SM, ctas)
                    ctx.set_option(ctx.OPT_SPMM_SM_LIMIT, sms)
                    if tr is not None:
                        ctx.set_option(ctx.OPT_TILE_ROWS, tr)
                    step_ms = time_step(eng, a.steps, a.warmup)
                    level0_ms = eng.time_level_spmm(0, a.steps)
                    line = {"dtype": dname, "k": k, "ctas_per_sm": ctas, "sm_limit": sms, "rep": rep,
                            "step_ms": round(step_ms, 4), "level0_ms": round(level0_ms, 4),
                            "level0_frac_of_3350_GBs": round(eng.level_bytes(0) / level0_ms / 1e6 / 3350.0, 3)}
                    if tr is not None:
                        line["tile_rows"] = tr
                    line.update(gpu_state())
                    print(json.dumps(line), flush=True)
            ctx.set_option(ctx.OPT_SPMM_CTAS_PER_SM, 0)
            ctx.set_option(ctx.OPT_SPMM_SM_LIMIT, 0)
            eng.close()
    finally:
        shutil.rmtree(workdir, ignore_errors=True)


if __name__ == "__main__":
    main()
