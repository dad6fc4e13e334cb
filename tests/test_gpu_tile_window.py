"""Every row-tile list (``ARROW_OPT_TILE_ROWS`` = 16 / 32 / 64 / 128 / automatic) gives the bits of the 64-row list.

The lists only change which rows are in flight at once: each element is still one FMA (or ⊕) chain in entry order, so the
float32 product under every epilogue, float64, min-plus and the witness launch must be bit-identical to the 64-row list,
under one CTA walking every tile and at the default grid, on the sweep's 20k-row ragged block with hub rows and on a block
with >= 8 tiles per resident CTA in every list.  The first float32 result per epilogue is also held to the float64 bound
(tests/spmm_bound.py).  Last, the automatic choice on this device is checked against the rule restated here.
"""
import numpy as np
import pytest
from scipy import sparse

from arrow_matrix_b200 import _lib
from tests import tile_dispatch as td
from tests.test_gpu_spmm_sweep import EPILOGUES, Problem, pipeline_block, set_options

pytestmark = pytest.mark.gpu

Ctx = _lib.Context
TILE_ROWS = (64, 16, 32, 128, 0)          # 64 first: the reference of every other list
GRIDS = {"1 CTA": (1, 1), "default": (0, 0)}      # (SPMM_SM_LIMIT, SPMM_CTAS_PER_SM)


@pytest.fixture(scope="module")
def torch_cuda(cuda_device):
    import torch
    torch.cuda.init()
    return torch


@pytest.fixture(scope="module")
def ctx(torch_cuda, cuda_device):
    c = Ctx(cuda_device)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def defaults(ctx):
    yield
    set_options(ctx)
    ctx.set_option(Ctx.OPT_TILE_ROWS, 0)


def configure(ctx, tile_rows, grid):
    set_options(ctx, sm_limit=GRIDS[grid][0], ctas_per_sm=GRIDS[grid][1])
    ctx.set_option(Ctx.OPT_TILE_ROWS, tile_rows)


def many_tiles_block(ctx):
    """>= 8 tiles per resident CTA at the default grid in every list (the 128-row one needs the most rows)"""
    rng = np.random.default_rng(77)
    n = td.TILE_ROWS_BIG * 8 * td.RESIDENT_CTAS_PER_SM * ctx.device_info()[0] + 1000
    lens = rng.integers(0, 5, size=n)
    rows = np.repeat(np.arange(n), lens)
    cols = rng.integers(0, n, rows.size)
    order = np.lexsort((cols, rows))
    vals = rng.uniform(0.5, 1.5, rows.size) * 10.0 ** rng.uniform(-2, 2, rows.size)
    return sparse.csr_matrix((vals[order].astype(np.float32), cols[order], np.concatenate([[0], np.cumsum(lens)])),
                             shape=(n, n))


@pytest.fixture(scope="module")
def blocks(ctx):
    return {"20k ragged": pipeline_block(np.random.default_rng(2024)), "many tiles": many_tiles_block(ctx)}


def assert_same_bits(got, ref, what):
    for a, b in zip(got, ref):
        if a.dtype.kind == "f":
            a, b = a + a.dtype.type(0), b + b.dtype.type(0)                 # +0 == -0
        ba, bb = a.view(np.uint8).reshape(a.shape[0], -1), b.view(np.uint8).reshape(b.shape[0], -1)
        if not np.array_equal(ba, bb):
            r = int(np.argwhere((ba != bb).any(axis=1))[0][0])
            pytest.fail(f"{what}: row {r} differs from the 64-row list ({int((ba != bb).any(axis=1).sum())} rows)")


@pytest.mark.parametrize("block,k", [("20k ragged", 8), ("20k ragged", 32), ("20k ragged", 128), ("20k ragged", 256),
                                     ("many tiles", 8)])
def test_float32_every_epilogue(ctx, torch_cuda, blocks, block, k):
    P = Problem(torch_cuda, ctx, blocks[block], k, seed=k)
    for tr in TILE_ROWS:
        for grid in GRIDS:
            for ep, (out_mode, acc, dualx) in EPILOGUES.items():
                configure(ctx, tr, grid)
                P.run_tile(ep, td.tile_instantiation(k, out_mode, acc, dualx), f"tile_rows={tr} grid={grid}")
    P.free()


class Operands:
    """float64 / min-plus / witness launches on one block, every output downloaded"""

    def __init__(self, ctx, A, k, seed):
        rng = np.random.default_rng(seed)
        self.ctx, self.k = ctx, k
        n, nc = A.shape
        self.n = n
        self.A64 = ctx.csr_upload(n, nc, A.indptr, A.indices, A.data.astype(np.float64), dtype=np.float64)
        self.A32 = ctx.csr_from_scipy(sparse.csr_matrix((np.round(np.abs(A.data) % 4).astype(np.float32), A.indices,
                                                         A.indptr), shape=A.shape))
        cmap = rng.permutation(nc + 3)[:nc].astype(np.int64)
        cmap[::5] = -1                                                   # skipped entries
        self.cm = ctx.map_upload(cmap, nc + 3)
        self.A64s = self.A64.remap_columns(self.cm, nc + 3)
        self.A32s = self.A32.remap_columns(self.cm, nc + 3)
        self.rm = ctx.map_upload(np.where(rng.random(n) < 0.9, rng.permutation(n), -1), n)
        n_add = n // 2 + 4
        self.am = ctx.map_upload(np.where(rng.random(n) < 0.6, rng.integers(0, n_add, n), -1), n_add)
        self.X64 = ctx.dense_from_host(rng.uniform(-1, 1, (nc + 3, k)), np.float64)
        self.add64 = ctx.dense_from_host(rng.uniform(-1, 1, (n_add, k)), np.float64)
        self.C64 = ctx.dense_alloc(n, k, np.float64)
        self.X32 = ctx.dense_from_host(rng.integers(0, 8, (nc + 3, k)).astype(np.float32))
        self.add32 = ctx.dense_from_host(rng.integers(0, 8, (n_add, k)).astype(np.float32))
        self.C32 = ctx.dense_alloc(n, k)
        self.lab = ctx.dense_alloc(n, k, np.int32)
        self.Cold = rng.uniform(-1, 1, (n, k))

    def run(self, what):
        ctx = self.ctx
        if what.startswith("f64"):
            self.C64.h2d(self.Cold)
            ctx.sync()
            if what == "f64 plain":
                ctx.spmm(self.A64, self.X64, self.C64)
            elif what == "f64 accumulate":
                ctx.spmm(self.A64, self.X64, self.C64, accumulate=True)
            elif what == "f64 row map":
                ctx.spmm(self.A64, self.X64, self.C64, rowmap=self.rm)
            elif what == "f64 gather-add":
                ctx.spmm_add(self.A64, self.X64, self.C64, self.add64, self.am)
            else:
                ctx.spmm(self.A64s, self.X64, self.C64, rowmap=self.rm, accumulate=True)
            return [self.C64.d2h()]
        if what == "min_plus":
            ctx.spmm_sr(self.A32, self.X32, self.C32, semiring=_lib.SR_MIN_PLUS)
        elif what == "min_plus addend, skipped":
            ctx.spmm_sr(self.A32s, self.X32, self.C32, self.add32, self.am, semiring=_lib.SR_MIN_PLUS)
        else:
            ctx.spmm_sr_witness(self.A32s if "skipped" in what else self.A32, self.X32, self.lab, values=self.C32,
                                semiring=_lib.SR_MIN_PLUS)
            return [self.C32.d2h(), self.lab.d2h()]
        return [self.C32.d2h()]

    def free(self):
        for h in (self.A64s, self.A32s, self.A64, self.A32, self.cm, self.rm, self.am, self.X64, self.add64, self.C64,
                  self.X32, self.add32, self.C32, self.lab):
            h.free()


LAUNCHES = ["f64 plain", "f64 accumulate", "f64 row map", "f64 gather-add", "f64 skipped", "min_plus",
            "min_plus addend, skipped", "witness", "witness skipped"]


@pytest.mark.parametrize("block,k", [("20k ragged", 16), ("20k ragged", 128), ("many tiles", 16)])
def test_float64_min_plus_witness(ctx, torch_cuda, blocks, block, k):
    ops = Operands(ctx, blocks[block], k, seed=k + 1)
    for what in LAUNCHES:
        configure(ctx, 64, "default")
        ref = ops.run(what)
        assert all(np.isfinite(r).all() for r in ref if r.dtype.kind == "f" and "f64" in what)
        for tr in TILE_ROWS:
            for grid in GRIDS:
                configure(ctx, tr, grid)
                assert_same_bits(ops.run(what), ref, f"{block} k={k} {what} tile_rows={tr} grid={grid}")
    ops.free()


def restated_rule(k, elem, l2_bytes, resident_ctas, big_ok):
    """the largest list whose window (resident CTAs x rows x k x element bytes) fits a quarter of the L2, else 16"""
    for rows in ((128,) if big_ok else ()) + (64, 32):
        if resident_ctas * rows * k * elem <= l2_bytes // 4:
            return rows
    return 16


def test_automatic_choice_on_this_device(ctx, torch_cuda):
    props = torch_cuda.cuda.get_device_properties(0)
    sms = ctx.device_info()[0]
    for sm_limit, per_sm in ((0, 0), (66, 0), (0, 2), (1, 1)):
        set_options(ctx, sm_limit=sm_limit, ctas_per_sm=per_sm)
        resident = (min(sm_limit, sms) if sm_limit else sms) * (min(per_sm, 4) if per_sm else 4)
        for k in range(4, 260, 4):
            for dtype, elem in ((np.float32, 4), (np.float64, 8)):
                want = restated_rule(k, elem, props.L2_cache_size, resident, elem == 4 and k <= 32)
                assert ctx.tile_rows(k, dtype) == want, (k, dtype, sm_limit, per_sm)
    set_options(ctx, big_tiles=0)
    assert ctx.tile_rows(16) == restated_rule(16, 4, props.L2_cache_size, 4 * sms, False)
    set_options(ctx)
    for forced in (16, 32, 64, 128):
        ctx.set_option(Ctx.OPT_TILE_ROWS, forced)
        assert ctx.tile_rows(16) == forced
        assert ctx.tile_rows(128) == min(forced, 64) and ctx.tile_rows(16, np.float64) == min(forced, 64)
    with pytest.raises(_lib.ArrowError):
        ctx.set_option(Ctx.OPT_TILE_ROWS, 48)
    if "H100" in props.name:
        ctx.set_option(Ctx.OPT_TILE_ROWS, 0)
        assert [ctx.tile_rows(k) for k in (16, 32, 64, 128)] == [128, 128, 64, 32]
        assert ctx.tile_rows(128, np.float64) == 16
