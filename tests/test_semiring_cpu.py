"""CPU tests of the semiring step: the host restatement (tests/semiring_ref.py) is anchored to the reference's golden
runs in (+, x) and to Dijkstra in (min, +); the refusals happen before any CUDA work; the tile dispatch of the semiring
kernels is covered by the feature widths of the GPU sweep."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200 import _lib, graphio, synth
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from oracle import oracle
from tests import semiring_ref as sr
from tests import tile_dispatch as td
from tests.golden_util import CASES, GoldenCase
from tests.test_gpu_kernels import assert_close


@pytest.mark.parametrize("name", CASES)
def test_plus_times_restatement_matches_the_protocol_oracle(name):
    """(+, x) restated with ⊕ / ⊗ as parameters == the protocol oracle for 3 chained steps (maps, truncation, stale rows),
    and == the reference's own outputs on the golden schedule"""
    g = GoldenCase(name)
    po = oracle.ReferenceProtocolOracle(g.decomposition, g.width, g.k, block_diagonal=g.block_diagonal,
                                        n_blocks=g.n_blocks, dtype=np.float64)
    ps = sr.SemiringProtocol(g.decomposition, g.width, g.k, "plus_times", block_diagonal=g.block_diagonal,
                             n_blocks=g.n_blocks)
    X0 = g.X[0] if g.X[0] is not None else np.random.default_rng(1).uniform(-1, 1, (ps.rows[0], g.k))
    po.set_features(np.asarray(X0, np.float64))
    ps.set_features(X0)
    for _ in range(3):
        po.step()
        ps.step()
        for j in range(ps.L):
            assert_close(ps.C[j], po.C[j])
    ps = sr.SemiringProtocol(g.decomposition, g.width, g.k, "plus_times", block_diagonal=g.block_diagonal,
                             n_blocks=g.n_blocks)
    for it in range(g.iterations):
        if g.X[it] is not None:
            ps.set_features(g.X[it])
        ps.step()
        for j in range(ps.L):
            assert_close(ps.C[j], g.C[it][j])


def _decomposed(unit, n=3000, w=100):
    A = sr.weighted_ba_graph(n, 3, seed=5, unit=unit)
    dec = arrow_decomposition(A, w, max_number_of_levels=3, block_diagonal=True, seed=2)
    return A, dec, w


@pytest.mark.parametrize("unit", [False, True], ids=["weights 1-16", "unit weights (BFS)"])
def test_min_plus_reaches_dijkstra_exactly(unit):
    A, dec, w = _decomposed(unit)
    n = A.shape[0]
    sources = np.random.default_rng(3).choice(n, 8, replace=False)
    p = sr.SemiringProtocol(dec, w, sources.size, "min_plus", add_identity=True)
    assert p.L == 3 and sum(p.dropped_nnz) == 0
    p.set_features(sr.source_features(p.perms[0], p.rows[0], n, sources))
    for steps in range(1, 500):
        before = p.X[0].copy()
        p.step()
        if np.array_equal(p.C[0], before):
            break
    got = sr.distances(p.C[0], p.perms[0], n)
    want = csgraph.shortest_path(A, method="D", indices=sources)
    assert np.array_equal(got, want.astype(np.float32)), f"{int(np.sum(got != want))} distances differ"
    if unit:
        assert np.array_equal(got, csgraph.shortest_path(A, method="D", unweighted=True, indices=sources))


def test_max_plus_is_negated_min_plus():
    """max_plus(A, X) == -min_plus(-A, -X) bit for bit: round to nearest is symmetric under negation"""
    rng = np.random.default_rng(4)
    A = sparse.random(300, 200, density=0.05, format="csr", random_state=5, dtype=np.float32)
    A.data = (rng.standard_normal(A.nnz) * 10.0 ** rng.uniform(-3, 3, A.nnz)).astype(np.float32)
    X = (rng.standard_normal((200, 7)) * 10.0 ** rng.uniform(-3, 3, (200, 1))).astype(np.float32)
    add = rng.standard_normal((50, 7)).astype(np.float32)
    amap = np.where(rng.random(300) < 0.5, rng.integers(0, 50, 300), -1)
    mx = sr.spmm(A, X, "max_plus", add, amap)
    mn = sr.spmm(-A, -X, "min_plus", -add, amap)
    assert np.array_equal((-mn).view(np.uint32), mx.view(np.uint32))
    A2, dec, w = _decomposed(False, n=1000, w=64)
    negdec = [(-sparse.csr_matrix(B), perm) for B, perm in dec]
    X0 = rng.uniform(-50, 50, (1024, 3)).astype(np.float32)
    pmax = sr.SemiringProtocol(dec, w, 3, "max_plus", add_identity=True)
    pmin = sr.SemiringProtocol(negdec, w, 3, "min_plus", add_identity=True)
    pmax.set_features(X0)
    pmin.set_features(-X0)
    for _ in range(3):
        assert np.array_equal((-pmin.step()).view(np.uint32), pmax.step().view(np.uint32))


class _TwoRanks(SelfComm):
    def Get_size(self) -> int:
        return 2


@pytest.fixture
def no_cuda(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a CUDA context was requested")
    monkeypatch.setattr(_lib.Context, "__init__", refuse)
    monkeypatch.setattr(_lib, "load_library", refuse)


def test_refusals_happen_before_any_cuda_call(tmp_path, no_cuda):
    dec = synth.synth_decomposition(4, 8, levels=2, perm_kind="random", seed=3)
    with pytest.raises(ValueError, match="float32"):
        ArrowEngine(dec, 8, 4, semiring="min_plus", dtype=np.float64)
    with pytest.raises(ValueError, match="gather"):
        ArrowEngine(dec, 8, 4, semiring="max_plus", fused_style="scatter")
    with pytest.raises(ValueError, match="unknown semiring"):
        ArrowEngine(dec, 8, 4, semiring="max_times")
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, 8, True)
    cases = [(_TwoRanks(), np.float32, "min_plus", False, "one GPU"),
             (_TwoRanks(), np.float32, "plus_times", True, "one GPU"),
             (SelfComm(), np.float64, "max_plus", False, "float32"),
             (SelfComm(), np.float32, "tropical", False, "unknown semiring")]
    for comm, dtype, semiring, add_identity, match in cases:
        blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, 8, True, dtype)
        arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, 8, 4, 'gpu', True, True,
                                                 semiring=semiring, add_identity=add_identity)
        with pytest.raises(ValueError, match=match):
            arrow.B.load_sparse_matrix_from_blocks(blocks)
        assert arrow._engine is None


def test_semiring_tile_shapes_are_all_reached_by_the_gpu_sweep():
    in_source = sr.source_sr_shapes(td.SOURCE)
    reached = {sr.sr_tile_shape(k, big) for k in sr.SWEEP_KS if k % 4 == 0 and k <= 256 for big in (True, False)}
    assert in_source and reached == in_source, f"unreached: {in_source - reached}, not in the source: {reached - in_source}"
