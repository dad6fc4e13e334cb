"""Multi-GPU parity (needs >= 2 GPUs on the box): one process per GPU, NVLink peer memory through CUDA IPC."""
import os
import socket
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, case, exchange, q):
    try:
        sys.path.insert(0, ROOT)
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world,
                                device_id=torch.device("cuda", rank))
        from arrow_matrix_b200 import synth
        from arrow_matrix_b200.comm import world_comm
        from arrow_matrix_b200.sharded import ShardedArrowDecomposition
        from oracle import oracle
        w, t0, k, levels, nested = {"L2k128": (128, 9, 128, 2, True), "L3k16": (64, 11, 16, 3, True),
                                    "L3stale_k6": (32, 6, 6, 3, False), "banded_k8": (32, 9, 8, 2, True)}[case]
        banded = case.startswith("banded")
        dec = synth.synth_decomposition(t0, w, levels=levels, perm_kind="random", seed=31, nested=nested, hub_rows=2, hub_nnz=600,
                                        band_nnz=4 if banded else 0, shrink=1 if banded else 2)
        from tests.test_gpu_ranks_one_gpu import close_rows
        fused = exchange.startswith("fused")
        arrow = ShardedArrowDecomposition(world_comm(), dec, w, k, device=rank, exchange="p2p" if fused else exchange.split("+")[0],
                                          overlap=2 if exchange.endswith("+overlap2") else ("+overlap" in exchange or "+side" in exchange),
                                          block_diagonal=not banded, mode="auto" if fused else "exchange")
        eng = arrow.engine
        if fused and nested:
            assert eng.fp is not None, eng.mode
        if exchange.endswith("+graph"):
            eng.use_graphs = True
        from tests import step_bound as stb
        from tests.test_gpu_step_bound import _assert_push_runs_identical, _push_option_runs
        po = oracle.ReferenceProtocolOracle(dec, w, k, block_diagonal=not banded)
        po64 = oracle.ReferenceProtocolOracle(dec, w, k, block_diagonal=not banded, dtype=np.float64)
        # the fused step (no state behind the sentinel) is also held to the per-element bound of tests/step_bound.py,
        # every step started from the device's own level-0 rows of all ranks
        ex = stb.ExactStep(dec, w, k, block_diagonal=not banded, world=world) if eng.fp is not None else None
        comm = world_comm()
        rng = np.random.default_rng(2)
        sh0 = eng.plan.levels[0]
        x_dev = None
        for it in range(3):
            X = synth.generate_dense_matrix(t0 * w, k, np.float32, rng)
            if it != 1:                                     # iteration 1 is chained (X := A X)
                arrow.B.set_features(X[sh0.r0:sh0.r1])
                po.set_features(X.copy())
                po64.set_features(X)
                x_dev = X
            if ex is not None:
                exact, mag = ex.run(x_dev)
            arrow.step()
            po.step()
            po64.step()
            for j in range(1 if eng.fp is not None else eng.L):
                sh = eng.plan.levels[j]
                close_rows(eng.result(j), po.C[j], po64.C[j], sh.r0, sh.r1)
            po64.C[0][:] = po.C[0]                          # the chained product starts from the same point in both
            if ex is not None:
                got = eng.result(0)
                r0, r1 = sh0.r0, sh0.r1
                stb.assert_step(got, exact[r0:r1], mag[r0:r1], ex.M[r0:r1], route=f"{case} {exchange} world {world} step {it}",
                                row0=r0)
                x_dev = np.concatenate(comm.allgather(got))
        if eng.fp is not None:                              # the push schedule options move the same rows: same bits
            _assert_push_runs_identical(_push_option_runs(eng, X[sh0.r0:sh0.r1]), f"{case} {exchange} rank {rank}")
        arrow.synchronize()
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except BaseException:     # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + traceback.format_exc()))


@pytest.mark.skipif(_n_gpus() < 2, reason="needs at least 2 GPUs (the same engine runs on one GPU in test_gpu_ranks_one_gpu.py)")
@pytest.mark.parametrize("case,exchange",
                         [("L2k128", e) for e in ("fused", "fused+side", "fused+side+graph", "p2p", "p2p+overlap", "p2p+overlap2",
                                                  "p2p-direct", "nccl")] +
                         [("L3k16", "fused+side+graph"), ("L3k16", "p2p+overlap"), ("L3stale_k6", "fused"), ("L3stale_k6", "nccl"),
                          ("L3stale_k6", "p2p-direct"), ("banded_k8", "fused+side"), ("banded_k8", "p2p"), ("banded_k8", "p2p+overlap2")])
def test_sharded_engine_on_gpus(case, exchange):
    import torch.multiprocessing as mp
    world = min(_n_gpus(), 4)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, case, exchange, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(60)
    bad = [f"rank {r}: {m}" for r, m in sorted(results) if m != "ok"]
    assert not bad, "\n".join(bad)


def _stream_worker(rank, world, port, q):
    try:
        sys.path.insert(0, ROOT)
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world,
                                device_id=torch.device("cuda", rank))
        from arrow_matrix_b200 import _lib, synth
        from arrow_matrix_b200.comm import world_comm
        from arrow_matrix_b200.sharded import ShardedArrowDecomposition
        w, t0, k = 64, 10, 32
        dec = synth.synth_decomposition(t0, w, levels=2, perm_kind="random", seed=12)
        rng = np.random.default_rng(3)
        Xs = [synth.generate_dense_matrix(t0 * w, k, np.float32, rng) for _ in range(5)]
        arrow = ShardedArrowDecomposition(world_comm(), dec, w, k, device=rank, overlap=True)
        sh0 = arrow.engine.plan.levels[0]
        ref = []
        for X in Xs:
            arrow.set_features(X[sh0.r0:sh0.r1])
            arrow.step()
            ref.append(arrow.result_tile())
        n = sh0.own_rows
        hx = [_lib.PinnedArray((n, k)) for _ in range(2)]
        hc = [_lib.PinnedArray((n, k)) for _ in range(2)]
        got = []
        for i, X in enumerate(Xs):
            if i >= 2:
                arrow.synchronize()
                got.append(hc[i % 2].array.copy())
            hx[i % 2].array[:] = X[sh0.r0:sh0.r1]
            arrow.step_stream(hx[i % 2].array, hc[i % 2].array)
        arrow.synchronize()
        got += [hc[(len(Xs) - 2) % 2].array.copy(), hc[(len(Xs) - 1) % 2].array.copy()]
        for g, r in zip(got, ref):
            assert np.array_equal(g, r)
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except BaseException:     # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + traceback.format_exc()))


@pytest.mark.skipif(_n_gpus() < 2, reason="needs at least 2 GPUs")
def test_sharded_stream_step():
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_stream_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(60)
    bad = [f"rank {r}: {m}" for r, m in sorted(results) if m != "ok"]
    assert not bad, "\n".join(bad)
