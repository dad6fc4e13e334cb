"""Python restatement of the SpMM dispatch of ``arrow_matrix_b200/csrc/arrow_b200.cu`` (test infrastructure only).

``tile_instantiation`` restates ``launch_tiles`` / ``launch_tiles_gv``: which ``k_spmm_tiles_v1`` / ``k_spmm_tiles``
template instance a launch runs.  ``spmm_kernels`` restates ``spmm_impl``'s choice between the generic, direct, shfl,
TMA, tile and long-row kernels.  ``build_tiles`` restates the row tiles ``build_long_rows`` cuts at upload.
``source_instantiations`` parses the tile dispatch out of the CUDA source, so that ``tests/test_tile_dispatch.py`` can
check that the restatement reaches exactly the template instances the library contains.
"""
from __future__ import annotations

import itertools
import os
import re
from typing import List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

SOURCE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "arrow_matrix_b200", "csrc",
                      "arrow_b200.cu")

TILE_ROWS, TILE_NNZ = 64, 1024               # small tiles
TILE_ROWS_BIG, TILE_NNZ_BIG = 128, 2048      # k <= 32
TILE_THREADS = 256
# resident tile-kernel CTAs per SM on H100: __launch_bounds__(256, 4) holds every instance at <= 64 registers (56..64 in
# `cuobjdump --dump-resource-usage`), 256 x 64 registers of the SM's 65536 -> 4 CTAs; shared memory (<= 34 KB) fits 4
RESIDENT_CTAS_PER_SM = 4
LONG_THRESHOLD, LONG_SEGMENT = 512, 2048     # arrow_ctx defaults (arrow_set_tuning)

# epilogues a tile launch can have through the C ABI: (output mode, accumulate, two-part X operand)
OUT_IDENTITY, OUT_ROWMAP, OUT_ROWPTR = "identity", "rowmap", "rowptr"
EPILOGUES = [(OUT_IDENTITY, False, False), (OUT_IDENTITY, True, False), (OUT_ROWMAP, False, False),
             (OUT_ROWMAP, True, False), (OUT_IDENTITY, False, True), (OUT_ROWPTR, False, False),
             (OUT_ROWPTR, False, True)]


class Inst(NamedTuple):
    """one template instance of a tile kernel"""
    kernel: str          # "v1" (k_spmm_tiles_v1) or "gen" (k_spmm_tiles)
    G: int
    VPL: int
    TR: int
    OUT: str
    ACC: bool
    RPG: int
    DUALX: bool

    def __str__(self):
        return (f"{self.kernel}<G={self.G},VPL={self.VPL},TR={self.TR},{self.OUT},ACC={int(self.ACC)},RPG={self.RPG},"
                f"DUALX={int(self.DUALX)}>")


def tile_shape(k: int, vpl_req: int = 0, rpg_req: int = 0, big_tiles: int = 1, rows_per_group: int = 0,
               has_tiles: bool = True) -> Tuple[int, int, int, int]:
    """(G, VPL, TR, RPG) that ``launch_tiles`` picks for ``k`` (a multiple of 4, <= 256)."""
    assert k % 4 == 0 and 4 <= k <= 256
    k4 = k // 4
    vpl = vpl_req if vpl_req in (1, 2, 4) else (4 if k4 >= 32 else (2 if k4 >= 8 else 1))
    while vpl > 1 and k4 < vpl:
        vpl >>= 1
    lanes = -(-k4 // vpl)
    if lanes > 32:
        vpl = 2 if -(-k4 // 32) <= 2 else 4
        lanes = -(-k4 // vpl)
    g = 1
    while g < lanes:
        g <<= 1
    big = k4 <= 8 and bool(big_tiles) and has_tiles
    rpg = rpg_req if rpg_req else (rows_per_group if rows_per_group else 1)
    if not big or rpg != 2:
        rpg = 1
    if big and rpg == 2 and (g, vpl) in ((4, 1), (8, 1), (2, 2), (4, 2)):            # TLP(...)
        return g, vpl, TILE_ROWS_BIG, 2
    if big and (g, vpl) in ((1, 1), (2, 1), (4, 1), (8, 1), (1, 2), (2, 2), (4, 2), (1, 4), (2, 4)):   # TLB(...)
        return g, vpl, TILE_ROWS_BIG, 1
    if (g, vpl) in {(gg, 1) for gg in (1, 2, 4, 8, 16, 32)} | {(gg, 2) for gg in (1, 2, 4, 8, 16, 32)} | \
            {(gg, 4) for gg in (1, 2, 4, 8, 16)}:                                        # TL(...)
        return g, vpl, TILE_ROWS, 1
    raise ValueError(f"no tile kernel for k4={k4} vpl={vpl}")


def tile_instantiation(k: int, out: str = OUT_IDENTITY, acc: bool = False, dualx: bool = False, vpl_req: int = 0,
                       rpg_req: int = 0, big_tiles: int = 1, rows_per_group: int = 0, tile_kernel: int = 1) -> Inst:
    """The tile kernel instance a launch with these options runs (``launch_tiles`` + ``launch_tiles_gv``)."""
    g, vpl, tr, rpg = tile_shape(k, vpl_req, rpg_req, big_tiles, rows_per_group)
    if out == OUT_ROWPTR:
        if acc:
            raise ValueError("row-pointer epilogue does not accumulate")
        return Inst("gen", g, vpl, tr, OUT_ROWPTR, False, rpg, dualx)
    if dualx:
        if out != OUT_IDENTITY or acc:
            raise ValueError("dual X base needs a plain or row-pointer epilogue")
        return Inst("gen", g, vpl, tr, OUT_IDENTITY, False, rpg, True)
    if rpg == 2 and out == OUT_IDENTITY and not acc:
        return Inst("gen", g, vpl, tr, OUT_IDENTITY, False, 2, False)
    if tile_kernel == 1:
        return Inst("v1", g, vpl, tr, out, acc, 1, False)
    return Inst("gen", g, vpl, tr, out, acc, 1, False)


def reachable_instantiations():
    """every tile kernel instance some launch reaches: k over the vector widths, every override, every epilogue"""
    found = set()
    for k in range(4, 257, 4):
        for vpl_req, rpg_req, big, rpg_opt, tk in itertools.product((0, 1, 2, 4), (0, 1, 2), (0, 1), (0, 1, 2), (0, 1)):
            for out, acc, dualx in EPILOGUES:
                found.add(tile_instantiation(k, out, acc, dualx, vpl_req, rpg_req, big, rpg_opt, tk))
    return found


def spmm_kernels(k: int, variant: int = -1, rowmap: bool = False, acc: bool = False, fused_operands: bool = False,
                 n_tiles: int = 1, n_long_tasks: int = 0, **tile_opts) -> List[str]:
    """Kernels ``spmm_impl`` launches.  ``fused_operands``: the call has an addend, a second X base or a pointer table
    (those live in the tile / generic / long kernels only).  ``tile_opts`` go to ``tile_instantiation``."""
    v = 3 if variant == -1 else variant
    tile_opts.setdefault("vpl_req", (v >> 4) & 0xF)
    tile_opts.setdefault("rpg_req", (v >> 8) & 0x3)
    v &= 0xF
    if fused_operands:
        v = 3
    tags = f"ROWMAP={int(rowmap)},ACC={int(acc)}"
    out: List[str] = []
    if k % 4 != 0 or k > 256:
        out.append(f"generic<{tags}>")
    elif v == 3:
        if n_tiles > 0:
            out.append(str(tile_instantiation(k, **tile_opts)))
    elif v == 2 and 32 <= k <= 128:
        out.append(f"tma<VPL={1 if k // 4 <= 32 else 2},{tags}>")
    else:
        k4 = k // 4
        g, vpl = next((gg, 1) for gg in (1, 2, 4, 8, 16, 32) if k4 <= gg) if k4 <= 32 else (32, 2)
        out.append(f"{'shfl' if v in (1, 2) else 'direct'}<G={g},VPL={vpl},{tags}>")
    if n_long_tasks > 0:
        out += ["long_partial", f"long_reduce<{tags}>"]
    return out


def build_tiles(indptr: Sequence[int], rows_cap: int, nnz_cap: int, threshold: int = LONG_THRESHOLD) -> np.ndarray:
    """[n_tiles, 4] = (row_begin, row_end, nnz_begin, nnz_end) as ``build_long_rows`` cuts them (rebased indptr)."""
    ip = np.asarray(indptr, dtype=np.int64)
    ip = ip - ip[0]
    lens = np.diff(ip)
    n = lens.size
    tiles = []
    r = 0
    while r < n:
        if lens[r] > threshold:
            r += 1
            continue
        e = r
        while e < n and e - r < rows_cap:
            if lens[e] > threshold:
                break
            if ip[e + 1] - ip[r] > nnz_cap - 4 and e > r:
                break
            e += 1
        if e == r:
            e += 1
        tiles.append((r, e, ip[r], ip[e]))
        r = e
    return np.array(tiles, dtype=np.int64).reshape(-1, 4)


def long_tasks(indptr: Sequence[int], threshold: int = LONG_THRESHOLD, segment: int = LONG_SEGMENT) -> int:
    lens = np.diff(np.asarray(indptr, dtype=np.int64))
    return int(sum(-(-int(l) // segment) for l in lens if l > threshold))


# ---- the dispatch as written in the source ----------------------------------------------------------------------
def _template_args(text: str, name: str) -> List[List[str]]:
    return [[a.strip() for a in m.group(1).split(",")] for m in re.finditer(rf"{name}<([^<>]*)>\(ctx", text)]


def source_instantiations(path: str = SOURCE) -> set:
    """The tile kernel instances the source can launch: every TL / TLB / TLP shape of ``launch_tiles`` combined with
    every ``launch_tiles_one`` / ``launch_tiles_v1`` call of ``launch_tiles_gv``.  A call whose RPG argument is a
    literal applies to the shapes of that RPG (the ``if constexpr (RPG == 2)`` branch and the RPG = 1 recursion)."""
    with open(path) as f:
        src = f.read()
    body = src[src.index("int launch_tiles(arrow_ctx *ctx"):]
    body = body[:body.index("#undef TL")]
    shapes = set()
    for macro, tr, rpg in (("TL", TILE_ROWS, 1), ("TLB", TILE_ROWS_BIG, 1), ("TLP", TILE_ROWS_BIG, 2)):
        for m in re.finditer(rf"(?<![A-Z]){macro}\((\d+),\s*(\d+)\);", body):
            shapes.add((int(m.group(1)), int(m.group(2)), tr, rpg))
    gv = src[src.index("int launch_tiles_gv(arrow_ctx *ctx"):]
    gv = gv[:gv.index("\n}\n")]
    one = _template_args(gv, "launch_tiles_one")
    v1 = _template_args(gv, "launch_tiles_v1")
    outs = {"OUT_IDENTITY": OUT_IDENTITY, "OUT_ROWMAP": OUT_ROWMAP, "OUT_ROWPTR": OUT_ROWPTR}
    boolean = {"true": True, "false": False}
    found = set()
    for g, vpl, tr, rpg in shapes:
        for a in one:       # <G, VPL, OUT, ACC, TR, TN, RPG, MINB, DUALX>
            if a[6] != "RPG" and int(a[6]) != rpg and not (rpg == 2 and a[6] == "1"):
                continue
            eff_rpg = rpg if a[6] == "RPG" else int(a[6])
            found.add(Inst("gen", g, vpl, tr, outs[a[2]], boolean[a[3]], eff_rpg, boolean[a[8]]))
        for a in v1:        # <G, VPL, ROWMAP, ACC, TR, TN>
            found.add(Inst("v1", g, vpl, tr, OUT_ROWMAP if boolean[a[2]] else OUT_IDENTITY, boolean[a[3]], 1, False))
    return found


def tile_args_line(path: str = SOURCE) -> Optional[int]:
    """line of ``launch_tiles`` in the source (for messages)"""
    with open(path) as f:
        for i, line in enumerate(f, 1):
            if line.startswith("int launch_tiles(arrow_ctx *ctx"):
                return i
    return None
