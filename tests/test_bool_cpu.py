"""CPU tests of the (or, and) step: the bit layout of the host helpers, the host restatement (tests/bool_ref.py) anchored to
the (min, +) restatement and to scipy's BFS, the refusals before any CUDA work, and the tile dispatch of the bit kernels
covered by the feature widths of the GPU sweep."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200 import _lib, graphio, synth
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from tests import bool_ref as br
from tests import semiring_ref as sr
from tests import tile_dispatch as td
from tests.golden_util import CASES, GoldenCase


@pytest.mark.parametrize("k", [1, 31, 32, 33, 127, 128, 129, 8192])
def test_pack_unpack_round_trip(k):
    rng = np.random.default_rng(k)
    X = rng.random((37, k)) < 0.3
    W = _lib.pack_bits(X)
    assert W.dtype == np.uint32 and W.shape == (37, br.words(k)) and (k <= 32) == (W.shape[1] == 1)
    assert W.shape[1] % 4 == 0 or k <= 32
    assert np.array_equal(W, br.pack(X)), "bit c of a row is bit c % 32 of word c // 32"
    assert np.array_equal(_lib.unpack_bits(W, k), X)
    assert np.array_equal(br.unpack(W, k), X)
    # padding bits are zero; non-zero is true; unpack ignores padding bits
    full = br.unpack(W, W.shape[1] * 32)
    assert not full[:, k:].any()
    assert np.array_equal(_lib.pack_bits(X.astype(np.float32) * 3.5), W)
    if k < W.shape[1] * 32:                    # the first padding bit
        noisy = W.copy()
        noisy[:, k // 32] |= np.uint32(1 << (k % 32))
        assert np.array_equal(_lib.unpack_bits(noisy, k), X)


def _unit(decomposition):
    """the decomposition with every stored value 1 (same structure)"""
    out = []
    for B, p in decomposition:
        B = sparse.csr_matrix(B, copy=True)
        B.data = np.ones_like(B.data, dtype=np.float32)
        out.append((B, p))
    return out


@pytest.mark.parametrize("add_identity", [False, True])
@pytest.mark.parametrize("name", CASES)
def test_restatement_is_min_plus_with_unit_values(name, add_identity):
    """(or, and) == (min, +) on unit values with finiteness as the boolean: 3 chained steps on every golden fixture,
    every level (maps, truncation, stale rows behind the sentinel)"""
    g = GoldenCase(name)
    dec = _unit(g.decomposition)
    pb = br.BoolProtocol(dec, g.width, g.k, block_diagonal=g.block_diagonal, n_blocks=g.n_blocks,
                         add_identity=add_identity)
    pm = sr.SemiringProtocol(dec, g.width, g.k, "min_plus", block_diagonal=g.block_diagonal, n_blocks=g.n_blocks,
                             add_identity=add_identity)
    X0 = np.random.default_rng(3).random((pb.rows[0], g.k)) < 0.2
    pb.set_features(X0)
    pm.set_features(np.where(X0, 0.0, np.inf).astype(np.float32))
    for it in range(3):
        pb.step()
        pm.step()
        for j in range(pb.L):
            assert np.array_equal(pb.C[j], np.isfinite(pm.C[j])), f"{name} step {it} level {j}"


def test_restated_product_with_maps():
    rng = np.random.default_rng(0)
    A = sparse.random(200, 150, density=0.05, format="csr", random_state=1)
    X = rng.random((150, 40)) < 0.1
    add = rng.random((30, 40)) < 0.5
    amap = np.where(rng.random(200) < 0.5, rng.integers(0, 30, 200), -1)
    cmap = rng.permutation(150)
    cmap[::4] = -1
    Xs = np.zeros((150, 40), bool)
    Xs[cmap[cmap >= 0]] = X[cmap >= 0]
    got = br.spmm(A, Xs, add, amap, col_map=cmap)
    D = A.toarray() != 0
    want = np.zeros((200, 40), bool)
    for r in range(200):
        for c in np.flatnonzero(D[r]):
            if cmap[c] >= 0:
                want[r] |= Xs[cmap[c]]
        if amap[r] >= 0:
            want[r] |= add[amap[r]]
    assert np.array_equal(got, want)


@pytest.mark.parametrize("directed", [False, True], ids=["undirected", "directed"])
def test_restated_bfs_levels_are_scipy_hop_counts(directed):
    n, w = 3000, 100
    A = sr.weighted_ba_graph(n, 3, seed=5, unit=True)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    if directed:
        # every downward edge, 30 % of the upward ones; the levels of the undirected decomposition keep the entries of
        # the directed edges (the decomposition itself is built for a symmetric pattern)
        C = sparse.coo_matrix(A)
        keep = (C.row > C.col) | (np.random.default_rng(1).random(C.nnz) < 0.3)
        A = sparse.csr_matrix((C.data[keep], (C.row[keep], C.col[keep])), shape=A.shape)
        directed_dec = []
        for B, perm in dec:
            Bc = sparse.coo_matrix(B)
            ok = np.asarray(A[perm[Bc.row], perm[Bc.col]]).ravel() != 0
            directed_dec.append((sparse.csr_matrix((Bc.data[ok], (Bc.row[ok], Bc.col[ok])), shape=B.shape), perm))
        dec = directed_dec
        assert sum(B.nnz for B, _ in dec) == A.nnz
    sources = np.random.default_rng(3).choice(n, 8, replace=False)
    p = br.BoolProtocol(dec, w, sources.size, add_identity=True)
    assert p.L == 3
    p.set_features(br.source_bits(p.perms[0], p.rows[0], n, sources))
    levels, steps = p.bfs_levels(500)
    got = br.vertex_order(levels, p.perms[0], n, -1).T
    # a step computes X | A X: row v gathers from its columns, so hops follow the edges v -> u of A backwards
    hops = csgraph.shortest_path(A.T, unweighted=True, indices=sources)
    want = np.where(np.isinf(hops), -1, hops).astype(np.int32)
    assert np.array_equal(got, want), f"{int(np.sum(got != want))} levels differ"
    assert steps == int(want.max()) + 1


class _TwoRanks(SelfComm):
    def Get_size(self) -> int:
        return 2


@pytest.fixture
def no_cuda(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a CUDA context was requested")
    monkeypatch.setattr(_lib.Context, "__init__", refuse)
    monkeypatch.setattr(_lib, "load_library", refuse)


def _bare_engine(semiring, add_identity):
    """an engine object in the given semiring without a device (the refusals must come before any CUDA call)"""
    eng = object.__new__(ArrowEngine)
    eng.sr, eng.semiring, eng.add_identity = _lib.SEMIRINGS[semiring], semiring, add_identity
    eng.fused_ok = True
    return eng


def test_refusals_happen_before_any_cuda_call(tmp_path, no_cuda):
    dec = synth.synth_decomposition(4, 8, levels=2, perm_kind="random", seed=3)
    with pytest.raises(ValueError, match="float32"):
        ArrowEngine(dec, 8, 4, semiring="or_and", dtype=np.float64)
    with pytest.raises(ValueError, match="gather"):
        ArrowEngine(dec, 8, 4, semiring="or_and", fused_style="scatter")
    with pytest.raises(ValueError, match="min_plus / max_plus"):
        _bare_engine("or_and", True).predecessors()
    with pytest.raises(ValueError, match="stream_step"):
        _bare_engine("or_and", True).stream_step(np.zeros((1, 1), bool), np.zeros((1, 1), bool))
    with pytest.raises(ValueError, match="add_identity"):
        _bare_engine("or_and", False).bfs_levels(10)
    with pytest.raises(ValueError, match="or_and"):
        _bare_engine("min_plus", True).bfs_levels(10)
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, 8, True)
    for comm, dtype, add_identity, match in ((_TwoRanks(), np.float32, True, "one GPU"),
                                             (_TwoRanks(), np.float32, False, "one GPU"),
                                             (SelfComm(), np.float64, True, "float32")):
        blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, 8, True, dtype)
        arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, 8, 4, 'gpu', True, True,
                                                 semiring="or_and", add_identity=add_identity)
        with pytest.raises(ValueError, match=match):
            arrow.B.load_sparse_matrix_from_blocks(blocks)
        assert arrow._engine is None


def test_bit_tile_shapes_are_all_reached_by_the_gpu_sweep():
    in_source = br.source_bits_shapes(td.SOURCE)
    reached = {br.bits_tile_shape(k, big) for k in br.SWEEP_KS for big in (True, False)}
    assert in_source and reached == in_source, f"unreached: {in_source - reached}, not in the source: {reached - in_source}"


def test_gpu_fixture_exposes_faulty_long_row_paths():
    """the hub rows of the GPU kernel sweep's block (same seeds) give other words under a long-row reduce that reads only
    the first segment's slot, a partial that walks only warp 0's share, a reduce that drops the addend (with an addend)
    and a row cut after 128 entries -- at every sweep width and epilogue, and at the thresholds of the tuning test"""
    A = br.hub_block(np.random.default_rng(64))
    lens = np.diff(A.indptr)
    assert np.count_nonzero(lens > 512) == 6 and np.count_nonzero((lens > 128) & (lens <= 512)) >= 5
    for k in br.SWEEP_KS:
        X, add, amap, cmap, Xs = br.problem_inputs(A, k, k)
        for label, args in (("plain", (X,)), ("add", (X, add, amap)), ("skip", (Xs, None, None, cmap)),
                            ("skip+add", (Xs, add, amap, cmap))):
            for thr in ((512, 128) if k in (16, 129, 2049) else (512,)):
                m = br.long_row_mutants(A, *args, threshold=thr)
                rows = np.flatnonzero(lens > thr)
                amap = args[2][rows] if len(args) > 2 and args[2] is not None else None
                assert np.array_equal(m["correct"], br.spmm(A[rows], args[0], args[1] if len(args) > 1 else None, amap,
                                                            col_map=args[3] if len(args) > 3 else None))
                for name in ("first slot", "warp 0", "128 entries") + (("no addend",) if "add" in label else ()):
                    assert (m[name] != m["correct"]).any(), f"k={k} {label} threshold {thr}: {name} not detected"
