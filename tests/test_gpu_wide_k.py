"""Hub rows at wide feature widths: the long-row kernels of every float family against the host references.

Rows with more entries than the long-row threshold go to a partial kernel (one CTA per segment) and a reduce kernel
(one CTA per row).  The partial kernels reduce each 128-column chunk through a fixed shared array, so a width needs no
more shared memory than any other; these tests run the widths either side of where a [8 warps][k] array would pass
48 KB (the opt-in limit) and 227 KB (the H100's per-block limit), and k % 4 != 0.  Every width is > 256, so the short
rows run the generic kernels and the grid options do not matter.

* float32: every epilogue of tests/test_gpu_spmm_sweep.py (NaN guard rows) against the float64 bound of
  tests/spmm_bound.py.
* float64: every epilogue of tests/test_gpu_fp64.py against the extended-precision bound of tests/spmm_bound64.py.
* (min, +) / (max, +) and the witness: exact, as in tests/test_gpu_semiring.py and tests/test_gpu_witness.py.

Each width runs at the default long-row tuning and at (threshold 128, segment 256), which puts more rows and more
segments on the long-row path.
"""
import numpy as np
import pytest
from scipy import sparse

from tests import spmm_bound64 as sb64
from tests import test_gpu_fp64 as fp64
from tests import test_gpu_semiring as semiring
from tests import test_gpu_spmm_sweep as sweep
from tests import test_gpu_witness as witness
from tests import tile_dispatch as td

pytestmark = pytest.mark.gpu

HUBS = (513, 600, 2048, 2049, 4100, 5000)        # 1 to 3 segments at the default tuning
MIDS = (129, 300, 511, 512)                      # short at the default tuning, long at the second
TUNINGS = ((td.LONG_THRESHOLD, td.LONG_SEGMENT), (128, 256))
# 32 k bytes for a float [8][k] array, 64 k for a double or a (value, label) one: 48 KB at k = 1537 / 769, 227 KB
# (232448 bytes) at k = 7265 / 3633
KS_4BYTE = [257, 1536, 1537, 2049, 7264, 7265, 8192, 8195]
KS_8BYTE = [257, 768, 769, 3632, 3633, 4096, 4099]


@pytest.fixture(scope="module")
def torch_cuda(cuda_device):
    import torch
    torch.cuda.init()
    return torch


@pytest.fixture(scope="module")
def ctx(torch_cuda, cuda_device):
    from arrow_matrix_b200 import _lib
    c = _lib.Context(cuda_device)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def default_tuning(ctx):
    yield
    ctx.set_tuning(td.LONG_THRESHOLD, td.LONG_SEGMENT)


@pytest.fixture(scope="module")
def structure():
    """1000 rows of 0..24 entries with empty rows, rows of 129..512 entries (long rows under the second tuning only) and
    the hub rows; columns c % 7 == 3 are never read.  A hub has more entries than there are columns, so columns repeat
    within a row (every reference sums or ⊕-reduces repeats).  The block is small because the host references at
    k ~ 8192 are what the module's run time is made of."""
    rng = np.random.default_rng(8192)
    n = 1000
    lens = rng.integers(0, 25, n)
    lens[rng.integers(0, n, 40)] = 0
    lens[rng.choice(n, len(MIDS) + len(HUBS), replace=False)] = MIDS + HUBS
    pool = np.flatnonzero(np.arange(n) % 7 != 3)
    indptr = np.concatenate([[0], np.cumsum(lens)])
    indices = np.concatenate([np.sort(rng.choice(pool, int(l))) for l in lens]).astype(np.int32)
    return n, indptr, indices


def _block(structure, values):
    n, indptr, indices = structure
    return sparse.csr_matrix((values, indices, indptr), shape=(n, n))


def _spread(rng, size):
    """+-U(0.5, 1.5) * 10^U(-2, 2)"""
    return rng.uniform(0.5, 1.5, size) * rng.choice([-1.0, 1.0], size) * 10.0 ** rng.uniform(-2, 2, size)


def _long_rows(A, threshold):
    return int((np.diff(A.indptr) > threshold).sum())


def _retune(ctx, pr, threshold, segment):
    """upload the block of a float64 / semiring / witness Problem again under another long-row tuning (the tuning is
    fixed at upload); its expectations do not depend on it"""
    ctx.set_tuning(threshold, segment)
    n, nc = pr.A.shape
    dtype = np.float64 if pr.A.dtype == np.float64 else np.float32
    dA = ctx.csr_upload(n, nc, pr.A.indptr, pr.A.indices, pr.A.data, dtype=dtype)
    cm = ctx.map_upload(pr.cmap, nc + 5)
    dAs = dA.remap_columns(cm, nc + 5)
    ctx.sync()
    cm.free()
    pr.dAs.free()                     # the remapped copy shares its source's row pointers and long-row tasks
    pr.dA.free()
    pr.dA, pr.dAs = dA, dAs
    pr.threshold, pr.segment = threshold, segment
    assert dA.info()["n_long_rows"] == _long_rows(pr.A, threshold)


@pytest.mark.parametrize("k", KS_4BYTE)
def test_float32_every_epilogue(ctx, torch_cuda, structure, k):
    A = _block(structure, _spread(np.random.default_rng(1), structure[2].size).astype(np.float32))
    for threshold, segment in TUNINGS:
        ctx.set_tuning(threshold, segment)
        P = sweep.Problem(torch_cuda, ctx, A, k, seed=k, threshold=threshold, segment=segment)
        try:
            assert P.info["n_long_rows"] == _long_rows(A, threshold)
            for ep in sweep.EPILOGUES:
                P.run_bound(ep, "generic + long rows, k > 256")
                del P.refs[ep]
        finally:
            P.free()
            del P


@pytest.mark.parametrize("k", KS_8BYTE)
def test_float64_every_epilogue(ctx, structure, k):
    A = _block(structure, _spread(np.random.default_rng(2), structure[2].size))
    pr = fp64.Problem(ctx, A, k, seed=k)
    try:
        for threshold, segment in TUNINGS:
            _retune(ctx, pr, threshold, segment)
            for epi in fp64.EPILOGUES:
                got, e = pr.run(epi)
                e.label = f"{e.label} threshold={threshold} segment={segment}"
                sb64.assert_spmm64(got, e)
    finally:
        pr.free()


@pytest.mark.parametrize("k", KS_4BYTE)
@pytest.mark.parametrize("sr_name", list(semiring.SEMIRINGS))
def test_tropical_every_epilogue(ctx, structure, k, sr_name):
    A = _block(structure, _spread(np.random.default_rng(3), structure[2].size).astype(np.float32))
    pr = semiring.Problem(ctx, A, k, sr_name, seed=k)
    try:
        for threshold, segment in TUNINGS:
            _retune(ctx, pr, threshold, segment)
            for epi in semiring.EPILOGUES:
                got, want = pr.run(epi), pr.expect(epi)
                bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
                assert not bad.any(), f"k={k} {sr_name} {epi} threshold={threshold}: {int(bad.sum())} elements differ"
    finally:
        pr.free()


@pytest.mark.parametrize("k", KS_8BYTE)
@pytest.mark.parametrize("sr_name", list(witness.SEMIRINGS))
def test_witness_every_epilogue(ctx, structure, k, sr_name):
    """weights 0..3 and features 0..7 (tests/test_gpu_witness.py): most elements tie, so the smallest label decides"""
    A = _block(structure, np.random.default_rng(4).integers(0, 4, structure[2].size).astype(np.float32))
    pr = witness.Problem(ctx, A, k, sr_name, seed=k)
    try:
        for threshold, segment in TUNINGS:
            _retune(ctx, pr, threshold, segment)
            for epi in witness.EPILOGUES:
                wv, wl = pr.want[epi]
                V, L = pr.run(epi)
                assert np.array_equal(V, wv), f"k={k} {sr_name} {epi} threshold={threshold}: values differ"
                bad = L != wl
                assert not bad.any(), f"k={k} {sr_name} {epi} threshold={threshold}: {int(bad.sum())} labels differ"
    finally:
        pr.free()


@pytest.mark.parametrize("k", [7265, 8192])
def test_preload_kernels_at_wide_k(ctx, k):
    """the preload's block has a 600-entry row, so it launches the long-row kernels at k"""
    ctx.preload_kernels(k)
    ctx.sync()
