"""Connected components on one GPU: labels, count and sizes bit for bit against the host restatement of tests/cc_ref.py on
every route, semiring, dtype, k and grid; hub rows, one-way edges, many small components, deep union trees on long
paths and cycles, an operator of the identity alone; reproducibility, the engine state left untouched, the refusals and
the ArrowDecompositionMPI view."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from arrow_matrix_b200 import _lib, decomp
from arrow_matrix_b200.arrow_dec_mpi import ArrowDecompositionMPI
from arrow_matrix_b200.comm import SelfComm
from arrow_matrix_b200.decomposition import arrow_decomposition
from arrow_matrix_b200.engine import ArrowEngine
from tests import cc_ref
from tests.golden_util import GPU_CASES, GoldenCase
from tests.test_cc_cpu import pieces
from tests.test_gpu_pagerank import DEFAULT_GRID, ONE_CTA, ROUTES, _hub_graph, _same
from tests.test_pagerank_cpu import _decompose, directed_ba

pytestmark = pytest.mark.gpu

# (semiring, dtype, mode, fused_style, k, add_identity): every route, semiring and dtype the engine runs, k = 1, 16, 128
CONFIGS = [
    ("plus_times", np.float32, "fused", "gather", 16, False),
    ("plus_times", np.float32, "fused", "scatter", 1, True),
    ("plus_times", np.float64, "exchange", "gather", 128, False),
    ("plus_times", np.float64, "fused", "scatter", 16, True),
    ("min_plus", np.float32, "fused", "gather", 1, True),
    ("or_and", np.float32, "exchange", "gather", 128, True),
    ("or_and", np.float32, "fused", "gather", 16, False),
    ("max_min", np.float32, "fused", "gather", 16, True),
]


def _engine(dec, width, config, block_diagonal=True, device=0, n_blocks=None):
    semiring, dtype, mode, style, k, ident = config
    return ArrowEngine(dec, width, k, block_diagonal=block_diagonal, dtype=dtype, semiring=semiring, add_identity=ident,
                       mode=mode, fused_style=style, device=device, n_blocks=n_blocks)


def _grid(eng, opts):
    for o, v in opts:
        eng.ctx.set_option(o, v)


def _check(eng, want, label):
    """labels, count and sizes bit for bit, twice, into fresh and caller-given arrays"""
    labels, count, sizes = want
    n = eng.n_rows
    got = eng.connected_components()
    assert _same(got, labels), (label, int(np.count_nonzero(got != labels)))
    assert eng.last_component_count == count, label
    out, sizes_out = np.full(n, -7, np.int32), np.full(n, -7, np.int32)
    assert eng.connected_components(out, sizes_out) is out
    assert _same(out, labels) and _same(sizes_out, sizes) and eng.last_component_count == count, label


def _golden(name):
    g = GoldenCase(name)
    return g.decomposition, g.width, g.block_diagonal


@pytest.mark.parametrize("config", CONFIGS, ids=lambda c: f"{c[0]}-{np.dtype(c[1]).name}-{c[2]}-{c[3]}-k{c[4]}-{c[5]}")
def test_golden_cases(cuda_device, config):
    for name in GPU_CASES:
        dec, width, bd = _golden(name)
        cfg = config if config[2] == "exchange" else config[:2] + ("auto",) + config[3:]
        eng = _engine(dec, width, cfg, bd, cuda_device)
        if not eng.fused_ok:                                     # rows behind the sentinel: refused before any launch
            launches = eng.ctx.launch_count()
            with pytest.raises(ValueError, match="sentinel"):
                eng.connected_components()
            assert eng.ctx.launch_count() == launches
        else:
            _check(eng, cc_ref.of(dec, width, bd, config[5]), (name, config))
        eng.close()


@pytest.mark.parametrize("k", [1, 16, 128])
@pytest.mark.parametrize("mode, style", ROUTES)
def test_hub_graph_on_both_grids(cuda_device, mode, style, k):
    """lists longer than 512 entries; on one CTA the grid-stride loops of every pass wrap many times"""
    dec = _decompose(_hub_graph(), 256, 3)
    want = cc_ref.of(dec, 256)
    eng = _engine(dec, 256, ("plus_times", np.float32, mode, style, k, False), device=cuda_device)
    assert max(st.csr.info()["max_row_nnz"] for st in eng.levels) > 512
    assert eng.total_nnz > 8 * 2048 and eng.n_rows > 8 * 256
    for opts in (ONE_CTA, DEFAULT_GRID):
        _grid(eng, opts)
        _check(eng, want, (mode, style, k, opts))
    eng.close()


@pytest.mark.parametrize("semiring, dtype", [("plus_times", np.float32), ("plus_times", np.float64), ("min_plus", np.float32),
                                             ("or_and", np.float32), ("max_min", np.float32)])
@pytest.mark.parametrize("mode, style", ROUTES)
def test_engine_state_untouched(cuda_device, semiring, dtype, mode, style):
    if semiring != "plus_times" and style == "scatter":
        pytest.skip("the semirings other than plus_times run the gather style")
    dec = _decompose(_hub_graph(), 256, 3)
    config = (semiring, dtype, mode, style, 16, True)
    X = (np.random.default_rng(5).random((3072 + 256, 16)) < 0.01).astype(dtype)
    runs = []
    for with_cc in (True, False):
        eng = _engine(dec, 256, config, device=cuda_device)
        X0 = X[: eng.n_rows]
        eng.set_features(X0)
        eng.step()
        before = (eng.features(), eng.result())
        if with_cc:
            eng.connected_components()
            assert _same(eng.features(), before[0]) and _same(eng.result(), before[1])
        eng.step()
        runs.append(eng.result())
        eng.close()
    assert _same(runs[0], runs[1])


def test_one_way_edges_join(cuda_device):
    """a directed BA decomposition keeping only the entries u -> v with u < v (original ids): every edge is one-way"""
    n, w = 4096, 256
    dec = _decompose(directed_ba(n, 3, 11), w, 11)
    n_blocks = [decomp.number_of_blocks(B, w) for B, _ in dec]
    fixed, _, _, _ = decomp.prepare_permutations([p for _, p in dec], n_blocks, w)
    one_way = []
    for (B, _), p in zip(dec, fixed):
        B = sparse.coo_matrix(B)
        keep = p[B.col] < p[B.row]
        one_way.append((sparse.csr_matrix((B.data[keep], (B.row[keep], B.col[keep])), shape=B.shape), p))
    want = cc_ref.of(one_way, w, n_blocks=n_blocks)
    S = cc_ref.structural(*_parts(one_way, w, n_blocks))
    assert (S != S.T).nnz > 0 and S.multiply(S.T).nnz == 0
    for config in (("min_plus", np.float32, "fused", "gather", 16, True), ("or_and", np.float32, "exchange", "gather", 1, False)):
        eng = _engine(one_way, w, config, device=cuda_device, n_blocks=n_blocks)
        _check(eng, want, config)
        eng.close()
    assert want[1] < n // 4                                      # one-way edges join as much as two-way ones
    assert want[1] == cc_ref.of(dec, w)[1]


def _parts(dec, width, n_blocks=None, block_diagonal=True):
    from tests import pagerank_ref as prr
    parts, proto = prr.level_parts(dec, width, n_blocks, block_diagonal=block_diagonal)
    return parts, proto.rows[0]


def test_many_components_and_the_mpi_view(cuda_device, tmp_path):
    from arrow_matrix_b200 import graphio
    n, w = 6000, 512
    A = pieces(n, 8)
    dec = _decompose(A, w, 8)
    want = cc_ref.of(dec, w)
    assert want[1] > 500
    eng = _engine(dec, w, ("max_min", np.float32, "fused", "gather", 1, False), device=cuda_device)
    _check(eng, want, "pieces")
    eng.close()
    base = str(tmp_path / "g")
    graphio.save_decomposition_new(dec, base, w, True)
    comm = SelfComm()
    blocks, n_blocks, to_prev, to_next = ArrowDecompositionMPI.load_decomposition_new(comm, base, w, True)
    arrow = ArrowDecompositionMPI.initialize(comm, n_blocks, to_prev, to_next, w, 4, 'gpu', True, True)
    arrow.B.load_sparse_matrix_from_blocks(blocks)
    sizes = np.zeros(arrow._engine.n_rows, np.int32)
    labels = arrow.connected_components(sizes_out=sizes)
    assert _same(labels, want[0]) and _same(sizes, want[2])
    perm0 = decomp.prepare_permutations([p for _, p in dec], list(n_blocks), w)[0][0]
    n_ref, comp = csgraph.connected_components(A, directed=True, connection="weak")
    assert np.array_equal(cc_ref.by_vertex(labels, perm0, n), cc_ref.smallest_labels(comp))
    assert arrow._engine.last_component_count == n_ref + arrow._engine.n_rows - n
    arrow._engine.close()


def _path(n, cycle):
    i = np.arange(n - 1)
    P = sparse.coo_matrix((np.ones(n - 1, np.float32), (i, i + 1)), shape=(n, n)).tolil()
    if cycle:
        P[n - 1, 0] = 1
    P = sparse.csr_matrix(P)
    return sparse.csr_matrix(P + P.T)


def _banded(n, width, cycle, seed):
    """two levels: level 0 the diagonal alone (self-loops: no edges), level 1 the path (cycle) r -- r + 1 in its own row
    order, banded (blocks (i, i +- 1); the closing entries lie in block row / column 0), its rows random level-0 rows"""
    P = _path(n, cycle)
    B0 = sparse.identity(n, np.float32, format="csr")
    perm1 = np.random.default_rng(seed).permutation(n)
    return [(B0, np.arange(n)), (P, perm1)]


@pytest.mark.parametrize("cycle", [False, True])
def test_long_path_and_cycle(cuda_device, cycle):
    n, w = 131072, 4096
    cases = [("arrow_decomposition", arrow_decomposition(_path(n, cycle), w, max_number_of_levels=3, block_diagonal=True,
                                                         seed=1), True),
             ("banded", _banded(n, w, cycle, 9), False)]
    for label, dec, bd in cases:
        want = cc_ref.of(dec, w, bd)
        assert want[1] == 1 + (decomp.number_of_blocks(dec[0][0], w) * w - n), label
        for config in (("plus_times", np.float32, "fused", "gather", 1, False), ("or_and", np.float32, "exchange", "gather", 16, True)):
            eng = _engine(dec, w, config, bd, cuda_device)
            assert eng.fused_ok and eng.L == len(dec), label
            for opts in (ONE_CTA, DEFAULT_GRID):
                _grid(eng, opts)
                _check(eng, want, (label, config, opts))
            eng.close()


@pytest.mark.parametrize("semiring", ["plus_times", "or_and"])
def test_identity_alone(cuda_device, semiring):
    """add_identity on a level without entries: the diagonal gives no edge, every row is its own component"""
    w, nb = 256, 12
    n = w * nb
    dec = [(sparse.csr_matrix((n, n), dtype=np.float32), np.arange(n))]
    eng = _engine(dec, w, (semiring, np.float32, "fused", "gather", 16, True), device=cuda_device, n_blocks=[nb])
    assert eng.total_nnz == n
    rows = np.arange(n, dtype=np.int32)
    _check(eng, (rows, n, np.ones(n, np.int32)), semiring)
    eng.close()


def test_bad_out_refused_before_any_launch(cuda_device):
    dec, width, bd = _golden(GPU_CASES[0])
    eng = _engine(dec, width, CONFIGS[0], bd, cuda_device)
    launches = eng.ctx.launch_count()
    for kw in (dict(out=np.zeros(eng.n_rows, np.int64)), dict(sizes_out=np.zeros(eng.n_rows + 1, np.int32))):
        with pytest.raises(ValueError, match="C-contiguous int32"):
            eng.connected_components(**kw)
    assert eng.ctx.launch_count() == launches
    eng.close()
