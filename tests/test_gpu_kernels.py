"""GPU parity tests: the CUDA path (through the C ABI) against the oracle on identical inputs.

Every SpMM result is held element by element to the float64 bound of tests/spmm_bound.py (``assert_spmm``); the
comparisons with the oracle stay as a second check with the parity tolerance: max |err| <= 1e-5 * max |ref|
(BASELINE.json: "within 1e-5 relative") and np.allclose(rtol=1e-5, atol=1e-5*scale) element-wise -- the reference
tests use np.allclose defaults (tests/test_arrowmpi.py:304, 329, 396).
"""
import numpy as np
import pytest
from scipy import sparse

pytestmark = pytest.mark.gpu

from oracle import oracle
from arrow_matrix_b200 import _lib, synth
from tests.spmm_bound import assert_spmm, ragged_csr, reference


# kernel kinds; for the CSR-streaming tile kernel also force 1 / 2 / 4 float4 per lane (bits 4..7)
ALL_VARIANTS = [_lib.VARIANT_DIRECT, _lib.VARIANT_SHFL, _lib.VARIANT_TMA, _lib.VARIANT_TILES,
                _lib.VARIANT_TILES | (1 << 4), _lib.VARIANT_TILES | (2 << 4), _lib.VARIANT_TILES | (4 << 4),
                # bits 8..9: rows a lane group works on at once (the paired kernels exist for k <= 32; else ignored)
                _lib.VARIANT_TILES | (1 << 8), _lib.VARIANT_TILES | (2 << 8), _lib.VARIANT_TILES | (2 << 8) | (2 << 4)]


def assert_close(got, ref, tol=1e-5, exact=None):
    """north_star parity: max|got - ref| <= 1e-5 * max|ref| (and element-wise np.allclose like the reference's tests).

    ``exact`` (optional): the same quantity in float64.  Two fp32 evaluations of one sum differ by rounding that grows
    with the number and the cancellation of the terms (hub rows of several hundred entries, the third chained
    product); when the direct comparison exceeds the tolerance, the device result passes iff it is within ``tol`` of
    the EXACT value or no farther from it than twice the reference arithmetic's own rounding -- never by a
    loosened constant."""
    got, ref = np.asarray(got), np.asarray(ref)
    scale = max(float(np.max(np.abs(ref))) if ref.size else 0.0, 1e-30)
    err = float(np.max(np.abs(got.astype(np.float64) - ref.astype(np.float64)))) if ref.size else 0.0
    if err <= tol * scale and np.allclose(got, ref, rtol=1e-5, atol=tol * scale):
        return
    assert exact is not None, f"max err {err:.3e} vs scale {scale:.3e} (rel {err / scale:.3e})"
    exact = np.asarray(exact, dtype=np.float64)
    e_got = float(np.max(np.abs(got.astype(np.float64) - exact)))
    e_ref = float(np.max(np.abs(ref.astype(np.float64) - exact)))
    assert e_got <= max(tol * scale, 2.0 * e_ref), \
        f"device vs exact {e_got:.3e}, reference arithmetic vs exact {e_ref:.3e}, scale {scale:.3e} (rel {e_got / scale:.3e})"


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(cuda_device)
    yield c
    c.close()


def ref_spmm64(A, X):
    return (A.astype(np.float64) @ X.astype(np.float64)).astype(np.float32)


@pytest.mark.parametrize("variant", ALL_VARIANTS)
@pytest.mark.parametrize("k", [4, 8, 16, 32, 64, 128, 256, 48])
def test_spmm_vector_k(ctx, variant, k):
    rng = np.random.default_rng(42)
    n = 3000
    A = synth.generate_sparse_matrix(n, n, 10 * n, np.float32, rng)
    X = synth.generate_dense_matrix(n, k, np.float32, rng)
    dA, dX, dC = ctx.csr_from_scipy(A), ctx.dense_from_host(X), ctx.dense_alloc(n, k)
    ctx.spmm(dA, dX, dC, variant=variant)
    got = dC.d2h()
    assert_spmm([got], reference(A, X, [np.zeros((n, k), np.float32)]))
    assert_close(got, oracle.csr_spmm_c(A, X))
    assert_close(got, A @ X)
    assert_close(got, ref_spmm64(A, X))
    # accumulate: C += A X   (arrow_slim_mpi.py:142-144)
    ctx.spmm(dA, dX, dC, accumulate=True, variant=variant)
    got2 = dC.d2h()
    assert_spmm([got2], reference(A, X, [got], accumulate=True))
    assert_close(got2, 2 * ref_spmm64(A, X))
    for h in (dA, dX, dC):
        h.free()


@pytest.mark.parametrize("k", [1, 2, 3, 5, 10, 130, 300])
def test_spmm_generic_k(ctx, k):
    # the reference's own tests use k=1 (test_spmm), 4, 10 (test_decomposition), 2 and 5 (test_larger_ranks)
    rng = np.random.default_rng(7)
    n = 700
    A = synth.generate_sparse_matrix(n, n, 6 * n, np.float32, rng)
    X = synth.generate_dense_matrix(n, k, np.float32, rng)
    dA, dX, dC = ctx.csr_from_scipy(A), ctx.dense_from_host(X), ctx.dense_alloc(n, k)
    ctx.spmm(dA, dX, dC)
    got = dC.d2h()
    assert_spmm([got], reference(A, X, [np.zeros((n, k), np.float32)]))
    assert_close(got, oracle.csr_spmm_c(A, X))
    ctx.spmm(dA, dX, dC, accumulate=True)
    got2 = dC.d2h()
    assert_spmm([got2], reference(A, X, [got], accumulate=True))
    assert_close(got2, 2 * ref_spmm64(A, X))


@pytest.mark.parametrize("variant", ALL_VARIANTS)
@pytest.mark.parametrize("k", [16, 128, 10])
def test_spmm_ragged_and_long_rows(ctx, variant, k):
    """empty rows, 1-entry rows, rows above the long-row threshold (hub rows of the arrow head)."""
    _ragged_and_long_rows(ctx, variant, k, decades=0)


@pytest.mark.parametrize("variant", ALL_VARIANTS)
@pytest.mark.parametrize("k", [16, 128, 10])
def test_spmm_ragged_and_long_rows_dynamic_range(ctx, variant, k):
    """the same rows with values scaled per row and per column over 10^+-2 each (products spread over 10^+-4) and X
    rows over 10^+-2: a small-magnitude row is held to its own bound, not to the scale of the hub rows"""
    _ragged_and_long_rows(ctx, variant, k, decades=2)


def _ragged_and_long_rows(ctx, variant, k, decades):
    rng = np.random.default_rng(3)
    n = 5000
    lens = rng.integers(0, 12, size=n)
    lens[::97] = 0
    lens[5] = 3000          # > threshold 512: segmented path, 2 segments
    lens[6] = 4097          # 3 segments
    lens[4999] = 513
    lens[10] = 512          # exactly at the threshold: regular path
    indptr = np.concatenate([[0], np.cumsum(lens)])
    if decades:
        A = ragged_csr(lens, n, rng, decades)
        X = (synth.generate_dense_matrix(n, k, np.float32, rng) * 10.0 ** rng.uniform(-2, 2, (n, 1))).astype(np.float32)
    else:
        cols = np.concatenate([np.sort(rng.choice(n, size=l, replace=False)) for l in lens]).astype(np.int32)
        vals = rng.random(cols.size, dtype=np.float32)
        A = sparse.csr_matrix((vals, cols, indptr), shape=(n, n))
        X = synth.generate_dense_matrix(n, k, np.float32, rng)
    dA, dX, dC = ctx.csr_from_scipy(A), ctx.dense_from_host(X), ctx.dense_alloc(n, k)
    info = dA.info()
    assert info["n_long_rows"] == 3 and info["max_row_nnz"] == 4097
    dC.fill(7.0)            # must be overwritten everywhere, also for empty rows
    ctx.spmm(dA, dX, dC, variant=variant)
    got = dC.d2h()
    assert_spmm([got], reference(A, X, [np.full((n, k), 7.0, np.float32)]))
    assert_close(got, ref_spmm64(A, X))
    ctx.spmm(dA, dX, dC, accumulate=True, variant=variant)
    got2 = dC.d2h()
    assert_spmm([got2], reference(A, X, [got], accumulate=True))
    assert_close(got2, 2 * ref_spmm64(A, X))


def test_spmm_int64_inputs_missing_data_and_row_slice(ctx):
    rng = np.random.default_rng(11)
    n, k = 2000, 32
    A = synth.generate_sparse_matrix(n, n, 8 * n, np.float32, rng)
    X = synth.generate_dense_matrix(n, k, np.float32, rng)
    # int64 index arrays (Julia converter), no data file -> ones
    d64 = ctx.csr_upload(n, n, A.indptr.astype(np.int64), A.indices.astype(np.int64), None)
    dX, dC = ctx.dense_from_host(X), ctx.dense_alloc(n, k)
    ctx.spmm(d64, dX, dC)
    ones = sparse.csr_matrix((np.ones_like(A.data), A.indices, A.indptr), shape=A.shape)
    got = dC.d2h()
    assert_spmm([got], reference(ones, X, [np.zeros((n, k), np.float32)]))
    assert_close(got, ref_spmm64(ones, X))
    # a row slice with un-rebased indptr (what a sharded loader hands over)
    r0, r1 = 300, 1700
    a, b = A.indptr[r0], A.indptr[r1]
    dS = ctx.csr_upload(r1 - r0, n, A.indptr[r0:r1 + 1], A.indices[a:b], A.data[a:b])
    dCs = ctx.dense_alloc(r1 - r0, k)
    ctx.spmm(dS, dX, dCs)
    got = dCs.d2h()
    assert_spmm([got], reference(A[r0:r1], X, [np.zeros((r1 - r0, k), np.float32)]))
    assert_close(got, ref_spmm64(A[r0:r1], X))


@pytest.mark.parametrize("variant", ALL_VARIANTS)
@pytest.mark.parametrize("k", [16, 128, 6])
def test_spmm_fused_permutations(ctx, variant, k):
    """column remap (forward gather folded in) + rowmap epilogue (backward scatter-add folded in)."""
    rng = np.random.default_rng(5)
    n1, n0 = 1500, 4000
    A = synth.generate_sparse_matrix(n1, n1, 9 * n1, np.float32, rng)
    A[7, :] = 0
    A = sparse.csr_matrix(A)
    A.eliminate_zeros()
    to_prev = rng.permutation(n0)[:n1].astype(np.int64)
    to_prev[::50] = 2 * n0                      # sentinel rows (arrow_dec_mpi.py:740-741)
    X0 = synth.generate_dense_matrix(n0, k, np.float32, rng)
    C0 = synth.generate_dense_matrix(n0, k, np.float32, rng)
    valid = to_prev < n0
    # oracle: X1 = gather (stale rows = 0 here), C1 = A X1, C0[to_prev] += C1
    X1 = np.zeros((n1, k), np.float32)
    X1[valid] = X0[to_prev[valid]]
    C1 = ref_spmm64(A, X1)
    ref = C0.copy()
    ref[to_prev[valid]] += C1[valid]
    m = ctx.map_upload(to_prev, n0)
    dA = ctx.csr_from_scipy(A)
    dAf = dA.remap_columns(m, n0)
    dX0, dC0 = ctx.dense_from_host(X0), ctx.dense_from_host(C0)
    ctx.spmm(dAf, dX0, dC0, rowmap=m, accumulate=True, variant=variant)
    got = dC0.d2h()
    col_map = np.where(valid, to_prev, -1)
    rowmap = np.where(valid, to_prev, -1)
    assert_spmm([got], reference(A, X0, [C0], col_map=col_map, rowmap=rowmap, accumulate=True))
    assert_close(got, ref)
    # without accumulate only routed rows are written
    dC0.h2d(C0)
    ctx.spmm(dAf, dX0, dC0, rowmap=m, accumulate=False, variant=variant)
    ref2 = C0.copy()
    ref2[to_prev[valid]] = C1[valid]
    got = dC0.d2h()
    assert_spmm([got], reference(A, X0, [C0], col_map=col_map, rowmap=rowmap))
    assert_close(got, ref2)


@pytest.mark.parametrize("k", [1, 4, 10, 16, 128])
def test_gather_rows_forward_backward(ctx, k):
    rng = np.random.default_rng(9)
    n0, n1 = 3000, 1200
    to_prev = rng.permutation(n0)[:n1].astype(np.int64)
    to_prev[3] = 2 * n0
    to_prev[77] = 2 * n0
    X0 = synth.generate_dense_matrix(n0, k, np.float32, rng)
    stale = synth.generate_dense_matrix(n1, k, np.float32, rng)
    m = ctx.map_upload(to_prev, n0)
    d0, d1 = ctx.dense_from_host(X0), ctx.dense_from_host(stale)
    ctx.gather_rows(d1, d0, m)                          # forward: X1[r] = X0[to_prev[r]], stale rows kept
    ref = stale.copy()
    oracle._lib().oracle_gather_rows_f32                # (symbol exists)
    valid = to_prev < n0
    ref[valid] = X0[to_prev[valid]]
    assert np.array_equal(d1.d2h(), ref)                # pure data movement: bit exact
    # backward as gather-add with the inverted map: C0[to_prev[r]] += C1[r]
    inv = m.invert(n0)
    h = inv.to_host()
    exp_inv = np.full(n0, -1, np.int32)
    exp_inv[to_prev[valid]] = np.flatnonzero(valid)
    assert np.array_equal(h, exp_inv)
    C1 = synth.generate_dense_matrix(n1, k, np.float32, rng)
    C0 = synth.generate_dense_matrix(n0, k, np.float32, rng)
    dc1, dc0 = ctx.dense_from_host(C1), ctx.dense_from_host(C0)
    ctx.gather_rows(dc0, dc1, inv, accumulate=True)
    refc = C0.copy()
    refc[to_prev[valid]] += C1[valid]
    assert np.array_equal(dc0.d2h(), refc)              # one add per element: bit exact


def test_gather_rows_multi_source(ctx):
    rng = np.random.default_rng(13)
    k = 16
    bounds = [0, 500, 500, 1300, 2000]                  # one empty source
    tiles = [synth.generate_dense_matrix(bounds[i + 1] - bounds[i], k, np.float32, rng) for i in range(4)]
    full = np.concatenate(tiles)
    m_host = rng.integers(0, 2000, size=900).astype(np.int64)
    m_host[::10] = -1
    m = ctx.map_upload(m_host, 2000)
    srcs = [ctx.dense_from_host(t) if t.shape[0] else ctx.dense_alloc(0, k) for t in tiles]
    dst = ctx.dense_alloc(900, k)
    dst.fill(3.0)
    ctx.gather_rows_multi(dst, srcs, bounds, m)
    ref = np.full((900, k), 3.0, np.float32)
    ok = m_host >= 0
    ref[ok] = full[m_host[ok]]
    assert np.array_equal(dst.d2h(), ref)


def test_errors_are_reported(ctx):
    with pytest.raises(_lib.ArrowError):
        ctx.spmm(_lib.Csr(ctx, 999, 1, 1, 0), ctx.dense_alloc(1, 4), ctx.dense_alloc(1, 4))
    A = ctx.csr_from_scipy(sparse.identity(8, format="csr", dtype=np.float32))
    x = ctx.dense_alloc(8, 4)
    with pytest.raises(_lib.ArrowError):
        ctx.spmm(A, x, x)                                # aliasing
    with pytest.raises(_lib.ArrowError):
        ctx.spmm(A, x, ctx.dense_alloc(8, 8))            # k mismatch
    with pytest.raises(_lib.ArrowError):
        ctx.spmm(A, ctx.dense_alloc(4, 4), ctx.dense_alloc(8, 4))   # X too short
    with pytest.raises(_lib.ArrowError):
        ctx.csr_upload(2, 2, np.array([0, 2, 1]), np.array([0]), None)      # decreasing indptr
    for dt in (np.int32, np.int64):
        with pytest.raises(_lib.ArrowError):
            ctx.csr_upload(2, 2, np.array([0, 1, 2]), np.array([0, 5], dtype=dt), None)   # column outside the block
    remapped = A.remap_columns(ctx.map_upload(np.arange(8, dtype=np.int64), 8), 8)
    with pytest.raises(_lib.ArrowError):
        A.free()                                         # its arrays still back the remapped copy
    remapped.free()
    A.free()


@pytest.mark.parametrize("k", [16, 128, 6, 256])
def test_spmm_add_epilogue_gather(ctx, k):
    """C[r] = (A X)[r] + add[add_map[r]]: the backward exchange folded into the receiving level (incl. long rows)"""
    rng = np.random.default_rng(17)
    n, m = 3000, 1300
    lens = rng.integers(0, 12, size=n)
    lens[4] = 2000                      # long row: segmented path must apply the addend too
    indptr = np.concatenate([[0], np.cumsum(lens)])
    cols = np.concatenate([np.sort(rng.choice(n, size=l, replace=False)) for l in lens]).astype(np.int32)
    A = sparse.csr_matrix((rng.random(cols.size, dtype=np.float32), cols, indptr), shape=(n, n))
    X = synth.generate_dense_matrix(n, k, np.float32, rng)
    add = synth.generate_dense_matrix(m, k, np.float32, rng)
    amap = np.full(n, -1, dtype=np.int64)
    pick = rng.permutation(n)[:m]
    amap[pick] = rng.permutation(m)
    amap[4] = 7
    dA, dX, dC, dAdd = ctx.csr_from_scipy(A), ctx.dense_from_host(X), ctx.dense_alloc(n, k), ctx.dense_from_host(add)
    dmap = ctx.map_upload(amap, m)
    dC.fill(5.0)
    ctx.spmm_add(dA, dX, dC, dAdd, dmap)
    ref = ref_spmm64(A, X)
    ok = amap >= 0
    ref[ok] += add[amap[ok]]
    got = dC.d2h()
    assert_spmm([got], reference(A, X, [np.full((n, k), 5.0, np.float32)], add=add, add_map=amap))
    assert_close(got, ref)


# ---- round 2: the fused multi-GPU step's building blocks, each against plain numpy ------------------------------
@pytest.mark.parametrize("k", [16, 32, 128, 20, 5])
def test_spmm_ex_dual_operand_row_pointers_and_gather_add(ctx, k):
    """C-ABI ``arrow_spmm_ex``: columns below the split read X, the others X2; every result row goes where its pointer
    says (two destination tiles, dropped rows), plus the epilogue gather-add; long rows and generic k included"""
    rng = np.random.default_rng(k)
    n, split, n2 = 700, 300, 450
    A = sparse.random(n, split + n2, density=0.02, format="csr", dtype=np.float32, random_state=3)
    A = sparse.csr_matrix(A)
    hub = sparse.csr_matrix((rng.random(600, dtype=np.float32), (np.zeros(600, dtype=np.int64), rng.choice(split + n2, 600, replace=False))),
                            shape=A.shape)
    A = sparse.csr_matrix(A + hub)                          # row 0: a long row (> 512 entries)
    A.sort_indices()
    X1 = synth.generate_dense_matrix(split + 40, k, np.float32, rng)      # X may be longer than the split
    X2 = synth.generate_dense_matrix(n2, k, np.float32, rng)
    add = synth.generate_dense_matrix(200, k, np.float32, rng)
    add_map = np.where(rng.random(n) < 0.3, rng.integers(0, 200, n), -1).astype(np.int64)
    which = rng.integers(-1, 2, n).astype(np.int32)         # -1 dropped, 0 / 1 = two destination tiles
    row = np.zeros(n, dtype=np.int64)
    for t in (0, 1):
        sel = np.flatnonzero(which == t)
        row[sel] = rng.permutation(900)[: sel.size]         # injective inside a tile
    dA = ctx.csr_from_scipy(A)
    dX1, dX2, dadd = ctx.dense_from_host(X1), ctx.dense_from_host(X2), ctx.dense_from_host(add)
    t0, t1 = ctx.dense_alloc(900, k), ctx.dense_alloc(900, k)
    tab = ctx.ptrtable_upload([t0, t1], which, row)
    dmap = ctx.map_upload(add_map, 200)
    ctx.spmm_ex(dA, dX1, X2=dX2, x_split=split, out_table=tab, add=dadd, add_map=dmap)
    ref = ref_spmm64(A, np.concatenate([X1[:split], X2]))
    sel = add_map >= 0
    ref[sel] += add[add_map[sel]]
    outs = [t0.d2h(), t1.d2h()]
    zeros = np.zeros((900, k), np.float32)
    assert_spmm(outs, reference(A, X1, [zeros, zeros], X2=X2, x_split=split, add=add, add_map=add_map,
                                table=(which, row)))
    for t in (0, 1):
        s2 = np.flatnonzero(which == t)
        expect = np.zeros((900, k))
        expect[row[s2]] = ref[s2]
        assert_close(outs[t], expect.astype(np.float32))
        untouched = np.setdiff1d(np.arange(900), row[s2])
        assert not outs[t][untouched].any()                 # nothing but the routed rows is written
    # plain destination with a dual operand (no table)
    dC = ctx.dense_alloc(n, k)
    ctx.spmm_ex(dA, dX1, C=dC, X2=dX2, x_split=split)
    got = dC.d2h()
    assert_spmm([got], reference(A, X1, [np.zeros((n, k), np.float32)], X2=X2, x_split=split))
    assert_close(got, ref_spmm64(A, np.concatenate([X1[:split], X2])).astype(np.float32))
    for h in (tab, dmap, dA, dX1, dX2, dadd, t0, t1, dC):
        h.free()


@pytest.mark.parametrize("k", [16, 128, 6])
def test_push_rows_and_reduce_rows(ctx, k):
    """``arrow_push_rows`` (forward exchange as one pass: item i of destination d lands in slot i - bound[d]) and
    ``arrow_reduce_rows`` (sum of the partial head tiles in source order, optionally delivered through a pointer table):
    pure data movement is compared bit for bit, the reduction against the same order in numpy"""
    rng = np.random.default_rng(k)
    src = synth.generate_dense_matrix(500, k, np.float32, rng)
    dsrc = ctx.dense_from_host(src)
    counts = [120, 0, 75, 300]
    bounds = np.concatenate([[0], np.cumsum(counts)])
    m = rng.integers(0, 500, bounds[-1]).astype(np.int64)
    dsts = [ctx.dense_alloc(max(c, 1) + 3, k) if c else None for c in counts]
    dm = ctx.map_upload(m, 500)
    ctx.push_rows(dsts, bounds, dsrc, dm)
    for d, c in enumerate(counts):
        if c:
            got = dsts[d].d2h()
            assert np.array_equal(got[:c], src[m[bounds[d]:bounds[d + 1]]])
            assert not got[c:].any()
    parts = [synth.generate_dense_matrix(64, k, np.float32, rng) for _ in range(5)]
    dparts = [ctx.dense_from_host(p) for p in parts]
    expect = parts[0].copy()
    for p in parts[1:]:
        expect += p                                         # rank order, fp32: bit-identical to the kernel's order
    out = ctx.dense_alloc(64, k)
    ctx.reduce_rows(dparts, 64, dst=out)
    assert np.array_equal(out.d2h(), expect)
    ctx.reduce_rows(dparts, 64, dst=dparts[0])              # in place on the first source (GPU 0 reduces into its own tile)
    assert np.array_equal(dparts[0].d2h(), expect)
    dparts[0].h2d(parts[0]); ctx.sync()
    which = np.where(np.arange(64) % 3 == 0, -1, np.arange(64) % 2).astype(np.int32)
    row = rng.permutation(100)[:64].astype(np.int64)
    ta, tb = ctx.dense_alloc(100, k), ctx.dense_alloc(100, k)
    tab = ctx.ptrtable_upload([ta, tb], which, row)
    ctx.reduce_rows(dparts, 64, out_table=tab)
    for t, tile in enumerate((ta, tb)):
        sel = np.flatnonzero(which == t)
        got = tile.d2h()
        assert np.array_equal(got[row[sel]], expect[sel])
        assert not got[np.setdiff1d(np.arange(100), row[sel])].any()
    with pytest.raises(_lib.ArrowError):
        ctx.push_rows(dsts, bounds[:-1].tolist() + [int(bounds[-1]) + 1], dsrc, dm)      # bounds must span the map
    with pytest.raises(_lib.ArrowError):
        ctx.ptrtable_upload([ta, tb], np.array([2], dtype=np.int32), np.array([0], dtype=np.int64))   # tile index out of range
    with pytest.raises(_lib.ArrowError):
        ctx.ptrtable_upload([ta, tb], np.array([0], dtype=np.int32), np.array([100], dtype=np.int64))  # row outside the tile


def test_graph_capture_replays_a_two_lane_sequence(ctx):
    """``arrow_graph_begin/end/launch``: a fork to the side lane, two SpMMs (per-lane tile schedulers re-arm themselves
    on the device), a join and a gather-add are recorded once and replayed on changing inputs"""
    rng = np.random.default_rng(0)
    n, k = 3000, 64
    A = synth.arrow_csr(n, 100, 30, rng)
    dA = ctx.csr_from_scipy(A)
    X = [synth.generate_dense_matrix(n, k, np.float32, rng) for _ in range(3)]
    dX, c1, c2 = ctx.dense_alloc(n, k), ctx.dense_alloc(n, k), ctx.dense_alloc(n, k)
    ident = ctx.map_upload(np.arange(n, dtype=np.int64), n)

    def sequence():
        ctx.lane_wait(3, 0)
        ctx.set_lane(3)
        ctx.spmm(dA, dX, c2)                # side lane
        ctx.set_lane(0)
        ctx.spmm(dA, dX, c1)                # main lane, concurrently
        ctx.lane_wait(0, 3)
        ctx.gather_rows(c1, c2, ident, accumulate=True)

    dX.h2d(X[0]); ctx.sync()
    sequence()                              # plain run first (lazy allocations)
    ctx.sync()
    ctx.graph_begin()
    sequence()
    g = ctx.graph_end()
    for x in X:
        dX.h2d(x); ctx.sync()
        ctx.graph_launch(g)
        ctx.sync()
        assert_close(c1.d2h(), (2 * ref_spmm64(A, x)).astype(np.float32))
    ctx.graph_free(g)
    with pytest.raises(_lib.ArrowError):
        ctx.graph_launch(g)


def test_dense_wrap_rejects_misaligned_pointers(ctx):
    """the vector kernels move float4 rows: a wrapped tile must start 16-byte aligned when k % 4 == 0, else 4-byte
    aligned (nothing is launched)"""
    import torch
    t = torch.zeros(64, device="cuda")
    base = t.data_ptr()
    assert base % 16 == 0
    for k, ptr in ((4, base + 4), (8, base + 8), (3, base + 2)):
        with pytest.raises(_lib.ArrowError) as e:
            ctx.dense_wrap(ptr, 2, k)
        assert e.value.code == -2
    ctx.dense_wrap(base + 16, 2, 4).free()
    ctx.dense_wrap(base + 4, 2, 3).free()
