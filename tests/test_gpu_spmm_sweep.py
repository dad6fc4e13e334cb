"""Every SpMM kernel instance against the float64 bound of tests/spmm_bound.py, with CTAs walking many tiles.

* Every tile kernel instance the dispatch can reach (tests/tile_dispatch.py, pinned to the source) runs under every
  epilogue it serves on a 20k-row block (>= 150 tiles in both tile sizes) at three grids: one CTA walking every tile
  (every mbarrier phase flip and stage reuse), 3 CTAs (interleaved tickets) and the default grid.
* The tile kernels evaluate each element as one FMA chain in ascending entry order from (old C) + addend, so every
  instance, override, grid and measurement switch must give BIT-IDENTICAL results for one (block, X, epilogue); the
  first result is held to the bound, the others to it.  The direct / shfl / TMA / generic / long-row kernels are held
  to the bound.
* Every operand sits between NaN guard rows (``dense_wrap`` of a torch tensor's interior); X rows no entry reads,
  addend rows no row adds and C before a non-accumulating launch are NaN too: a stray read shows up as NaN in the
  output, a stray write as a changed guard or unwritten row.  Nothing can fault the device.
"""
import time

import numpy as np
import pytest
from scipy import sparse

from arrow_matrix_b200 import _lib
from tests import spmm_bound as sb
from tests import tile_dispatch as td

pytestmark = pytest.mark.gpu

GUARD = 2
START = []                        # wall clock at the module's first test
LAUNCHED = set()                  # tile kernel instances run by this module
WORST = {}                        # kernel family -> worst ratio to the bound
REGIMES = []                      # printed at the end
# epilogue -> (output mode, accumulate, two-part X) as the tile dispatch sees it
EPILOGUES = {
    "plain": (td.OUT_IDENTITY, False, False), "acc": (td.OUT_IDENTITY, True, False),
    "rowmap": (td.OUT_ROWMAP, False, False), "rowmap_acc": (td.OUT_ROWMAP, True, False),
    "add": (td.OUT_IDENTITY, False, False), "skip": (td.OUT_ROWMAP, True, False),
    "dual": (td.OUT_IDENTITY, False, True), "ptr": (td.OUT_ROWPTR, False, False),
    "ptr_dual": (td.OUT_ROWPTR, False, True),
}
VEC_EPILOGUES = ["plain", "acc", "rowmap", "rowmap_acc", "skip"]      # what direct / shfl / TMA serve
DEFAULTS = [(_lib.Context.OPT_L2_HINTS_PLAIN, 3), (_lib.Context.OPT_L2_HINTS_FUSED, 0), (_lib.Context.OPT_BIG_TILES, 1),
            (_lib.Context.OPT_SPMM_CTAS_PER_SM, 0), (_lib.Context.OPT_PREFETCH, 0),
            (_lib.Context.OPT_ROWS_PER_GROUP, 0), (_lib.Context.OPT_SPMM_SM_LIMIT, 0),
            (_lib.Context.OPT_SMEM_CARVEOUT, -1), (_lib.Context.OPT_FORCE_PREDICATED, 0),
            (_lib.Context.OPT_TILE_KERNEL, 1)]
GRIDS = {"1 CTA": (1, 1), "3 CTAs": (3, 1), "default": (0, 0)}       # (SPMM_SM_LIMIT, SPMM_CTAS_PER_SM)


@pytest.fixture(scope="module")
def torch_cuda(cuda_device):
    START.append(time.time())
    import torch
    torch.cuda.init()
    return torch


@pytest.fixture(scope="module")
def ctx(torch_cuda, cuda_device):
    c = _lib.Context(cuda_device)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def defaults(ctx):
    yield
    for opt, v in DEFAULTS:
        ctx.set_option(opt, v)
    ctx.set_tuning(td.LONG_THRESHOLD, td.LONG_SEGMENT)


def set_options(ctx, **opts):
    for opt, v in DEFAULTS:
        ctx.set_option(opt, v)
    names = {"big_tiles": _lib.Context.OPT_BIG_TILES, "rows_per_group": _lib.Context.OPT_ROWS_PER_GROUP,
             "tile_kernel": _lib.Context.OPT_TILE_KERNEL, "sm_limit": _lib.Context.OPT_SPMM_SM_LIMIT,
             "ctas_per_sm": _lib.Context.OPT_SPMM_CTAS_PER_SM, "hints_plain": _lib.Context.OPT_L2_HINTS_PLAIN,
             "hints_fused": _lib.Context.OPT_L2_HINTS_FUSED, "prefetch": _lib.Context.OPT_PREFETCH,
             "carveout": _lib.Context.OPT_SMEM_CARVEOUT, "force_predicated": _lib.Context.OPT_FORCE_PREDICATED}
    for name, v in opts.items():
        ctx.set_option(names[name], v)


class Canary:
    """a [rows, k] operand between NaN guard rows of one torch tensor, handed to the library with dense_wrap"""

    def __init__(self, torch, ctx, host):
        self.torch, self.ctx = torch, ctx
        self.rows, self.k = host.shape
        self.t = torch.full((self.rows + 2 * GUARD, self.k), float("nan"), dtype=torch.float32, device="cuda")
        self.d = ctx.dense_wrap(self.t[GUARD:].data_ptr(), self.rows, self.k)
        self.set(host)

    def set(self, host):
        self.t[GUARD:GUARD + self.rows].copy_(self.torch.from_numpy(np.ascontiguousarray(host, dtype=np.float32)))
        self.torch.cuda.synchronize()

    def get(self):
        self.ctx.sync()
        full = self.t.cpu().numpy()
        guards = np.concatenate([full[:GUARD], full[GUARD + self.rows:]])
        assert np.isnan(guards).all(), "a guard row next to a tile was written"
        return full[GUARD:GUARD + self.rows]


def _nan_except(rows, k, keep, rng, scale_decades=2.0):
    out = np.full((rows, k), np.nan, np.float32)
    keep = np.unique(keep)
    out[keep] = rng.uniform(-1, 1, (keep.size, k)) * 10.0 ** rng.uniform(-scale_decades, scale_decades, (keep.size, 1))
    return out


class Problem:
    """One uploaded block and every operand its epilogues need, at one k, with the float64 references cached."""

    def __init__(self, torch, ctx, A, k, seed, threshold=td.LONG_THRESHOLD, segment=td.LONG_SEGMENT):
        rng = np.random.default_rng(seed)
        self.ctx, self.A, self.k = ctx, A, k
        self.threshold, self.segment = threshold, segment
        n, nc = A.shape
        self.n = n
        used = np.unique(A.indices)
        self.Xh = _nan_except(nc + 5, k, used, rng)                        # X longer than n_cols, unread rows NaN
        self.Cold = rng.standard_normal((n + 3, k)).astype(np.float32)     # C longer than n_rows
        self.Cnan = np.full((n + 3, k), np.nan, np.float32)
        self.rm = rng.permutation(n + 3)[:n].astype(np.int64)
        self.rm[::9] = -1
        n_add = n // 2 + 4
        self.amap = np.where(rng.random(n) < 0.6, rng.integers(0, n_add, n), -1).astype(np.int64)
        self.addh = _nan_except(n_add, k, self.amap[self.amap >= 0], rng)
        new_nc = nc + 5
        self.cmap = rng.permutation(new_nc)[:nc].astype(np.int64)
        self.cmap[::5] = -1                                                # entries whose image is invalid: skipped
        img = self.cmap[used]
        self.Xsh = _nan_except(new_nc + 2, k, img[img >= 0], rng)
        self.split = nc // 3
        self.X1h = np.concatenate([self.Xh[:self.split], np.full((4, k), np.nan, np.float32)])
        self.X2h = np.concatenate([self.Xh[self.split:nc], np.full((2, k), np.nan, np.float32)])
        self.which = rng.integers(-1, 2, n).astype(np.int32)
        self.trow = np.zeros(n, np.int64)
        for t in (0, 1):
            sel = np.flatnonzero(self.which == t)
            self.trow[sel] = rng.permutation(n + 5)[:sel.size]
        self.Tnan = np.full((n + 5, k), np.nan, np.float32)
        # device side
        self.dA = ctx.csr_from_scipy(A)
        self.info = self.dA.info()
        self.dm = ctx.map_upload(self.rm, n + 3)
        self.dam = ctx.map_upload(self.amap, n_add)
        self.dcm = ctx.map_upload(self.cmap, new_nc)
        self.dAs = self.dA.remap_columns(self.dcm, new_nc)
        self.X = Canary(torch, ctx, self.Xh)
        self.Xs = Canary(torch, ctx, self.Xsh)
        self.X1 = Canary(torch, ctx, self.X1h)
        self.X2 = Canary(torch, ctx, self.X2h)
        self.add = Canary(torch, ctx, self.addh)
        self.C = Canary(torch, ctx, self.Cnan)
        self.T = [Canary(torch, ctx, self.Tnan) for _ in range(2)]
        self.tab = ctx.ptrtable_upload([t.d for t in self.T], self.which, self.trow)
        self.refs, self.first = {}, {}
        self.tiles = {tr: td.build_tiles(A.indptr, tr, nnz, threshold) for tr, nnz in
                      ((td.TILE_ROWS, td.TILE_NNZ), (td.TILE_ROWS_BIG, td.TILE_NNZ_BIG))}
        self.n_long_tasks = td.long_tasks(A.indptr, threshold, segment)

    def before(self, ep):
        if ep in ("ptr", "ptr_dual"):
            return [self.Tnan, self.Tnan]
        return [self.Cold if EPILOGUES[ep][1] else self.Cnan]

    def reference(self, ep):
        if ep not in self.refs:
            kw = dict(threshold=self.threshold, segment=self.segment, label=f"k={self.k} {ep}")
            X = self.Xh
            if ep in ("rowmap", "rowmap_acc", "skip"):
                kw["rowmap"] = self.rm
            if ep in ("acc", "rowmap_acc", "skip"):
                kw["accumulate"] = True
            if ep in ("add", "ptr"):
                kw.update(add=self.addh, add_map=self.amap)
            if ep == "skip":
                X, kw["col_map"] = self.Xsh, self.cmap
            if ep in ("dual", "ptr_dual"):
                X, kw["X2"], kw["x_split"] = self.X1h, self.X2h, self.split
            if ep in ("ptr", "ptr_dual"):
                kw["table"] = (self.which, self.trow)
            self.refs[ep] = sb.reference(self.A, X, self.before(ep), **kw)
        return self.refs[ep]

    def launch(self, ep, variant=_lib.VARIANT_AUTO):
        ctx, dests = self.ctx, (self.T if ep in ("ptr", "ptr_dual") else [self.C])
        for d, b in zip(dests, self.before(ep)):
            d.set(b)
        A, X, C = self.dA, self.X.d, self.C.d
        if ep in ("plain", "acc", "rowmap", "rowmap_acc"):
            ctx.spmm(A, X, C, rowmap=self.dm if "rowmap" in ep else None, accumulate=ep.endswith("acc"), variant=variant)
        elif ep == "skip":
            ctx.spmm(self.dAs, self.Xs.d, C, rowmap=self.dm, accumulate=True, variant=variant)
        elif ep == "add":
            ctx.spmm_add(A, X, C, self.add.d, self.dam, variant=variant)
        elif ep == "dual":
            ctx.spmm_ex(A, self.X1.d, C=C, X2=self.X2.d, x_split=self.split, variant=variant)
        elif ep == "ptr":
            ctx.spmm_ex(A, X, out_table=self.tab, add=self.add.d, add_map=self.dam, variant=variant)
        else:
            ctx.spmm_ex(A, self.X1.d, X2=self.X2.d, x_split=self.split, out_table=self.tab, variant=variant)
        return [d.get() for d in dests]

    def run_tile(self, ep, inst, label, variant=_lib.VARIANT_TILES):
        """a tile kernel launch: the first result per epilogue is held to the bound, every other one to that result"""
        got = self.launch(ep, variant)
        LAUNCHED.add(inst)
        if ep not in self.first:
            family = f"tile {inst.kernel} TR={inst.TR}" + (" + long rows" if self.n_long_tasks else "")
            r = sb.assert_spmm(got, self.reference(ep))
            WORST[family] = max(WORST.get(family, 0.0), r)
            self.first[ep] = (got, f"{inst} {label}")
            return
        ref, ref_label = self.first[ep]
        for t, (a, b) in enumerate(zip(got, ref)):
            ba, bb = (a + np.float32(0)).view(np.uint32), (b + np.float32(0)).view(np.uint32)    # +0 == -0
            if not np.array_equal(ba, bb):
                r, c = np.argwhere(ba != bb)[0]
                pytest.fail(f"k={self.k} {ep}: {inst} {label} differs from {ref_label} (tile {t} row {r} col {c}: "
                            f"{a[r, c]!r} vs {b[r, c]!r}, {int((ba != bb).any(axis=1).sum())} rows)")

    def run_bound(self, ep, family, variant=_lib.VARIANT_AUTO):
        r = sb.assert_spmm(self.launch(ep, variant), self.reference(ep))
        WORST[family] = max(WORST.get(family, 0.0), r)

    def free(self):
        for h in (self.tab, self.dAs, self.dA, self.dm, self.dam, self.dcm):
            h.free()


def pipeline_block(rng, n=20000):
    """20k rows of 0..8 entries, a band of 250..510-entry rows (the nnz cap of a tile binds), rows at the long-row
    threshold and one above, a 3000-entry hub, empty rows; a seventh of the columns is never read; values spread
    over 10^+-4"""
    lens = rng.integers(0, 9, size=n)
    lens[::97] = 0
    lens[5000:5040] = rng.integers(250, 511, size=40)
    lens[7000], lens[7001], lens[9000] = 512, 513, 3000
    pool = np.flatnonzero(np.arange(n) % 7 != 3)
    return sb.ragged_csr(lens, n, rng, decades=2.0, col_pool=pool)


TILE_KS = [4, 8, 12, 16, 20, 32, 36, 64, 68, 128, 132, 256]


def tile_cases(k):
    """(epilogue, instance, variant, options) for every distinct instance reachable at k, default first"""
    seen, out = set(), []
    big_opts = (1, 0) if k <= 32 else (1,)
    for tk in (1, 0):
        for big in big_opts:
            for vpl in (0, 1, 2, 4):
                for rpg_var, rpg_opt in ((0, 0), (2, 0), (0, 2)):
                    opts = dict(tile_kernel=tk, big_tiles=big, rows_per_group=rpg_opt)
                    for ep, (out_mode, acc, dualx) in EPILOGUES.items():
                        inst = td.tile_instantiation(k, out_mode, acc, dualx, vpl, rpg_var, big, rpg_opt, tk)
                        if (ep, inst) not in seen:
                            seen.add((ep, inst))
                            out.append((ep, inst, _lib.VARIANT_TILES | (vpl << 4) | (rpg_var << 8), opts))
    return out


@pytest.fixture(scope="module")
def pipeline_A():
    A = pipeline_block(np.random.default_rng(2024))
    for tr, nnz in ((td.TILE_ROWS, td.TILE_NNZ), (td.TILE_ROWS_BIG, td.TILE_NNZ_BIG)):
        assert len(td.build_tiles(A.indptr, tr, nnz)) >= 150
    return A


@pytest.mark.parametrize("k", TILE_KS)
def test_every_tile_instance_at_three_grids(ctx, torch_cuda, pipeline_A, k):
    P = Problem(torch_cuda, ctx, pipeline_A, k, seed=k)
    sms = ctx.device_info()[0]
    for grid, (sm_limit, per_sm) in GRIDS.items():
        for ep, inst, variant, opts in tile_cases(k):
            set_options(ctx, sm_limit=sm_limit, ctas_per_sm=per_sm, **opts)
            P.run_tile(ep, inst, f"grid={grid} variant={variant:#x} {opts}", variant)
        for tr in (td.TILE_ROWS, td.TILE_ROWS_BIG) if k == TILE_KS[0] else ():
            nt = len(P.tiles[tr])
            g = {"1 CTA": 1, "3 CTAs": 3}.get(grid)
            REGIMES.append(f"20k rows, TR={tr}, grid={grid}: {nt} tiles, "
                           + (f"{nt / g:.0f} tiles per CTA" if g else
                              f"grid <= {min(nt, td.RESIDENT_CTAS_PER_SM * sms)} CTAs"))
    P.free()


def test_measurement_switches_are_bit_identical(ctx, torch_cuda, pipeline_A):
    """L2 hints, bulk L2 prefetch, shared-memory carve-out and the forced predicated path change no bit"""
    for k in (16, 128):
        P = Problem(torch_cuda, ctx, pipeline_A, k, seed=k)
        switches = [dict(hints_plain=h, hints_fused=h) for h in range(4)] + [dict(prefetch=0x01), dict(prefetch=0x10),
                    dict(prefetch=0x11)] + [dict(carveout=c) for c in (0, 50, 100)] + [dict(force_predicated=1)]
        for tk in (1, 0):
            for sw in [{}] + switches:
                for ep, (out_mode, acc, dualx) in EPILOGUES.items():
                    set_options(ctx, tile_kernel=tk, **sw)
                    P.run_tile(ep, td.tile_instantiation(k, out_mode, acc, dualx, tile_kernel=tk), f"{sw}")
        P.free()


def test_many_tiles_per_resident_cta(ctx, torch_cuda):
    """a block with >= 8 tiles per resident CTA at the default grid: both tile sizes, both kernels, every epilogue"""
    rng = np.random.default_rng(77)
    sms = ctx.device_info()[0]
    n = td.TILE_ROWS_BIG * 8 * td.RESIDENT_CTAS_PER_SM * sms + 1000
    lens = rng.integers(0, 5, size=n)
    rows = np.repeat(np.arange(n), lens)
    cols = rng.integers(0, n, rows.size)                 # duplicates allowed: the block sums them like the kernels
    order = np.lexsort((cols, rows))
    vals = rng.uniform(0.5, 1.5, rows.size) * 10.0 ** rng.uniform(-2, 2, rows.size)
    A = sparse.csr_matrix((vals[order].astype(np.float32), cols[order], np.concatenate([[0], np.cumsum(lens)])),
                          shape=(n, n))
    k = 8
    P = Problem(torch_cuda, ctx, A, k, seed=5)
    for tk in (1, 0):
        for big in (1, 0):
            for ep, (out_mode, acc, dualx) in EPILOGUES.items():
                set_options(ctx, tile_kernel=tk, big_tiles=big)
                P.run_tile(ep, td.tile_instantiation(k, out_mode, acc, dualx, big_tiles=big, tile_kernel=tk),
                           f"big={big}")
    for tr in (td.TILE_ROWS, td.TILE_ROWS_BIG):
        nt = len(P.tiles[tr])
        REGIMES.append(f"k={k} TR={tr} grid=default ({n} rows): {nt} tiles, >= "
                       f"{nt / (td.RESIDENT_CTAS_PER_SM * sms):.1f} tiles per CTA")
    P.free()


def boundary_blocks(rng):
    out = {}
    for n in (1, 2, 3, 5, 63, 64, 65, 127, 128, 129):
        out[f"rows={n}"] = sb.ragged_csr(rng.integers(0, 7, size=n), 200, rng, decades=2.0)
    out["nnz=0"] = sb.ragged_csr(np.zeros(70, np.int64), 50, rng)
    out["all long"] = sb.ragged_csr(rng.integers(513, 900, size=4), 2000, rng, decades=2.0)
    lens = rng.integers(0, 6, size=600)
    lens[100:110] = rng.integers(250, 511, size=10)
    lens[200:203] = [512, 513, 1]
    lens[300:305] = [511, 510, 509, 508, 507]       # first entries of the following tiles at every residue mod 4
    out["tile edges"] = sb.ragged_csr(lens, 3000, rng, decades=2.0)
    return out


@pytest.mark.parametrize("k", [12, 64, 10])
def test_tile_boundary_shapes(ctx, torch_cuda, k):
    rng = np.random.default_rng(k)
    blocks = boundary_blocks(np.random.default_rng(0))
    edges = td.build_tiles(blocks["tile edges"].indptr, td.TILE_ROWS, td.TILE_NNZ)
    assert set(edges[:, 2] % 4) == {0, 1, 2, 3}
    for name, A in blocks.items():
        P = Problem(torch_cuda, ctx, A, k, seed=int(rng.integers(1 << 30)))
        for ep, (out_mode, acc, dualx) in EPILOGUES.items():
            for grid in ("1 CTA", "default"):
                set_options(ctx, sm_limit=GRIDS[grid][0], ctas_per_sm=GRIDS[grid][1])
                if k % 4:
                    P.run_bound(ep, "generic + long rows")
                elif P.info["n_rows"] > P.info["n_long_rows"]:
                    P.run_tile(ep, td.tile_instantiation(k, out_mode, acc, dualx), f"{name} grid={grid}")
                else:
                    P.run_bound(ep, "long rows only")
        P.free()


@pytest.mark.parametrize("threshold", [1, 8, 100, 1016])
def test_long_row_tuning(ctx, torch_cuda, threshold):
    rng = np.random.default_rng(threshold)
    for segment in (32, 33, 2048):
        lens = rng.integers(0, 12, size=400)
        lens[[10, 11, 12, 13, 14, 15]] = [segment, 2 * segment, segment + 1, threshold, threshold + 1, 1016]
        lens[16:20] = [4096, 2048, 66, 64]
        A = sb.ragged_csr(lens, 6000, rng, decades=2.0)
        ctx.set_tuning(threshold, segment)
        for k in (16, 10):
            P = Problem(torch_cuda, ctx, A, k, seed=segment + k, threshold=threshold, segment=segment)
            assert P.info["n_long_rows"] == int((lens > threshold).sum())
            for ep, (out_mode, acc, dualx) in EPILOGUES.items():
                if k % 4:
                    P.run_bound(ep, "generic + long rows")
                else:
                    P.run_tile(ep, td.tile_instantiation(k, out_mode, acc, dualx), f"threshold={threshold} "
                                                                                   f"segment={segment}")
            P.free()


@pytest.fixture(scope="module")
def ragged_A():
    rng = np.random.default_rng(3)
    lens = rng.integers(0, 12, size=3000)
    lens[::97] = 0
    lens[5], lens[6], lens[2999], lens[10] = 3000, 4097, 513, 512
    return sb.ragged_csr(lens, 6000, rng, decades=2.0, col_pool=np.flatnonzero(np.arange(6000) % 7 != 3))


@pytest.mark.parametrize("k", [4, 8, 16, 32, 64, 128, 256])
def test_direct_shfl_tma_kernels(ctx, torch_cuda, ragged_A, k):
    P = Problem(torch_cuda, ctx, ragged_A, k, seed=k)
    variants = [(_lib.VARIANT_DIRECT, "direct"), (_lib.VARIANT_SHFL, "shfl")]
    if 32 <= k <= 128:
        variants.append((_lib.VARIANT_TMA, "tma"))
    for v, name in variants:
        for ep in VEC_EPILOGUES:
            P.run_bound(ep, f"{name} + long rows", v)
    for ep in EPILOGUES:                            # fused operands always run the tile kernel
        P.run_bound(ep, "tile (ragged, hubs) + long rows", _lib.VARIANT_DIRECT if ep not in VEC_EPILOGUES else 3)
    P.free()


@pytest.mark.parametrize("k", [1, 3, 6, 10, 130, 260, 300])
def test_generic_kernel(ctx, torch_cuda, ragged_A, k):
    P = Problem(torch_cuda, ctx, ragged_A, k, seed=k)
    for ep in EPILOGUES:
        P.run_bound(ep, "generic + long rows")
    P.free()


def test_graph_replay_resets_the_scheduler(ctx, torch_cuda, pipeline_A):
    """two tile launches (row map, gather-add) on one lane at grid 1, captured once and replayed on changing X: every
    replay equals an un-captured run bit for bit"""
    k = 32
    P = Problem(torch_cuda, ctx, pipeline_A, k, seed=9)
    set_options(ctx, sm_limit=1, ctas_per_sm=1)
    C2 = Canary(torch_cuda, ctx, P.Cnan)
    rng = np.random.default_rng(1)

    def sequence():
        ctx.spmm(P.dA, P.X.d, P.C.d, rowmap=P.dm)
        ctx.spmm_add(P.dA, P.X.d, C2.d, P.add.d, P.dam)

    def fresh_x():
        x = P.Xh.copy()
        ok = ~np.isnan(x[:, 0])
        x[ok] = rng.standard_normal((int(ok.sum()), k))
        return x

    xs = [fresh_x() for _ in range(3)]
    expect = []
    for x in xs:
        P.X.set(x)
        P.C.set(P.Cnan)
        C2.set(P.Cnan)
        sequence()
        expect.append((P.C.get(), C2.get()))
    P.C.set(P.Cnan)
    C2.set(P.Cnan)
    ctx.graph_begin()
    sequence()
    g = ctx.graph_end()
    for x, (e1, e2) in zip(xs, expect):
        P.X.set(x)
        ctx.graph_launch(g)
        got1, got2 = P.C.get(), C2.get()
        assert np.array_equal(got1.view(np.uint32), e1.view(np.uint32))
        assert np.array_equal(got2.view(np.uint32), e2.view(np.uint32))
    ctx.graph_free(g)
    P.free()


def test_every_instance_was_launched(capsys):
    """last in the module: the sweep ran every tile kernel instance the source contains"""
    src = td.source_instantiations()
    missing = src - LAUNCHED
    with capsys.disabled():
        print(f"\n[spmm sweep] tile kernel instances launched: {len(LAUNCHED & src)} of {len(src)} in the source")
        for line in REGIMES:
            print(f"[spmm sweep] {line}")
        for fam in sorted(WORST):
            print(f"[spmm sweep] worst |err| / bound, {fam}: {WORST[fam]:.3g}")
        print(f"[spmm sweep] module wall time {time.time() - START[0]:.1f} s")
    assert not missing, f"never launched: {sorted(map(str, missing))[:10]}"
    assert LAUNCHED <= src
