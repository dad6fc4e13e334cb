"""Host restatement of personalized PageRank on the arrow engine (test infrastructure only).

Operator, weights and restart
-----------------------------
``M`` is what the engine's step applies: entry ``(r, c)`` of level ``j`` with value ``a`` is the edge
``cmap_j(c) -> cmap_j(r)`` (level 0: the identity map, with the identity diagonal in front of every row when
``add_identity``); an entry with an end at -1 is not part of ``M`` and duplicates count separately.  ``level_parts``
restates the blocks as the engine uploads them (``decomp.arrow_rows``: file order, the reference's block pattern) and
takes the maps from the protocol (``push_ref.level_maps``).  ``w[u]`` is the float64 sum from +0 of the values of the
edges leaving ``u``, levels ascending then entry order; ``inv[u] = fl_T(1 / w[u])`` (0 when ``w[u] == 0``: dangling);
``M^`` holds ``fl_T(a * inv[u])``.  ``S[:, s] = fl_T(X0[:, s] / sigma_s)``.

Iteration
---------
``p_{t+1} = fl_T(fl(fl(alpha * Y) + fl(c_t * S)))`` with ``Y = M^ p_t``, ``c_t = fl(fl(1 - alpha) + fl(alpha * m_t))`` and
``m_t`` the dangling mass of ``p_t``; ``r_{t+1} = sum_v |fl(p_{t+1} - p_t)|``.  Every column sum runs in float64 over
512-row chunks from row 0, sequential inside a chunk (``np.cumsum`` is a sequential loop), the partials added in order.
``update`` restates one iterate bit for bit given ``Y``; ``loop64`` runs the whole iteration in float64 (``Y`` and ``p``
never rounded to ``T``): the yardstick of the error bound.

Error bound
-----------
All data are non-negative.  Let ``Phi(p) = alpha M^ p + c(p) S`` be the exact map.  One device iterate is
``Phi(p~)_v (1 + theta_v)`` with ``|theta_v| <= eps_v``: the step's row ``v`` passes at most ``M_v`` roundings in ``T``
(``step_bound.chain_heights`` of the blocks with their diagonal, every route), and the iterate adds the scaled entry
``fl_T(a * inv)``, the two float64 products, the add and the final rounding to ``T`` (``h_v = M_v + 5``, all counted at
``u_T >= u_64``); ``c`` carries the float64 chunked sum of ``m`` and two more roundings (``cm = 512 + chunks + 2`` at
``u_64``).  So ``eps_v = gamma_{h_v}(u_T) + gamma_cm(u_64) + their product`` (Higham, Lemma 3.1), plus an absolute
``h_v * eta_T`` per element for roundings in the subnormal range.  ``loop64``'s own iterate has
``eps_ref_v = gamma_{h_v + cm}(u_64)``.

``Phi(p) - Phi(q) = alpha M^ (p - q) + alpha (m(p) - m(q)) S``: a column of ``M^`` sums to ``1 + eta`` with ``|eta| <=
gamma_2(u_T) + gamma_{d + 1}(u_64)`` (``d`` the largest out-degree: ``w`` is a float64 sum, ``1 / w`` one divide,
``inv`` and the product one rounding each) and ``S`` to ``1 + gamma_1(u_T) + gamma_cm(u_64)``.  So ``Phi`` is an L1
contraction by ``rho = alpha (1 + eta)``.  With ``E_t`` the L1 distance of a column of the device iterate from
``loop64``'s and ``q_{t+1}`` the latter's next iterate,

    E_{t+1} <= rho (1 + eps_max) E_t + sum_v (eps_v + eps_ref_v) q_{t+1, v} / (1 - eps_ref_v) + sum_v h_v eta_T,

``E_0 = 0`` (both start from the same ``S``): a geometric sum of per-step terms.  No constant is tuned.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np
from scipy import sparse

from tests import bool_ref as br
from tests import push_ref as pr
from tests.spmm_bound import ETA32, U32, U64, gamma
from tests.spmm_bound64 import ETA64
from tests.step_bound import chain_heights

CHUNK = 512


def unit(dtype) -> Tuple[float, float]:
    """(unit roundoff, subnormal rounding error) of T"""
    return (U32, ETA32) if np.dtype(dtype) == np.float32 else (U64, ETA64)


# ---- operator -----------------------------------------------------------------------------------------------------------
def _arrow_block(B, width: int, n_blocks: int, block_diagonal: bool, dtype) -> sparse.csr_matrix:
    """the entries of a level the engine uploads, in file order: rows and columns below n_blocks * width, blocks (0, j),
    (i, 0), (i, i) and, banded, (i, i +- 1)"""
    B = sparse.csr_matrix(B)
    n = n_blocks * width
    ip = B.indptr.astype(np.int64)
    rows_have = min(B.shape[0], n)
    r = np.repeat(np.arange(rows_have, dtype=np.int64), np.diff(ip[: rows_have + 1]))
    c = B.indices[: ip[rows_have]].astype(np.int64)
    a = B.data[: ip[rows_have]]
    bi, bj = r // width, c // width
    keep = (c < n) & ((bi == 0) | (bj == 0) | (bi == bj))
    if not block_diagonal:
        keep |= (c < n) & (np.abs(bi - bj) == 1)
    r, c, a = r[keep], c[keep], a[keep].astype(dtype)
    indptr = np.zeros(n + 1, np.int64)
    np.add.at(indptr, r + 1, 1)
    return sparse.csr_matrix((a, c, np.cumsum(indptr)), shape=(n, n))


def _with_diagonal(A: sparse.csr_matrix) -> sparse.csr_matrix:
    """an entry (r, r) of 1 in front of every row"""
    n = A.shape[0]
    ip = A.indptr.astype(np.int64)
    out_ptr = ip + np.arange(n + 1)
    nnz = int(out_ptr[-1])
    diag = out_ptr[:-1]
    rest = np.ones(nnz, bool)
    rest[diag] = False
    idx = np.empty(nnz, np.int64)
    dat = np.empty(nnz, A.dtype)
    idx[diag], dat[diag] = np.arange(n), 1
    idx[rest], dat[rest] = A.indices, A.data
    return sparse.csr_matrix((dat, idx, out_ptr), shape=A.shape)


def level_parts(dec, width: int, n_blocks: Optional[Sequence[int]] = None, block_diagonal: bool = True,
                add_identity: bool = False, dtype=np.float32):
    """([(block, level-j -> level-0 map or None)], protocol) as the engine steps them"""
    proto = br.BoolProtocol(dec, width, 1, block_diagonal, n_blocks)
    maps = pr.level_maps(proto)
    parts = []
    for j, ((B, _), nb) in enumerate(zip(dec, proto.n_blocks)):
        A = _arrow_block(B, width, nb, block_diagonal, dtype)
        if j == 0 and add_identity:
            A = _with_diagonal(A)
        parts.append((A, None if j == 0 else maps[j]))
    return parts, proto


def entries(parts) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """(u, v, value, is an edge of M) of every entry, in (part, entry) order"""
    us, vs, vals, ok = [], [], [], []
    for A, m in parts:
        r = np.repeat(np.arange(A.shape[0], dtype=np.int64), np.diff(A.indptr))
        c = A.indices.astype(np.int64)
        u, v = c, r
        if m is not None:
            m = np.asarray(m, np.int64)
            u, v = np.where(c >= 0, m[np.maximum(c, 0)], -1), m[r]
        us.append(u), vs.append(v), vals.append(A.data), ok.append((c >= 0) & (u >= 0) & (v >= 0))
    cat = lambda x, dt: np.concatenate(x) if x else np.zeros(0, dt)
    return cat(us, np.int64), cat(vs, np.int64), cat(vals, np.float64), cat(ok, bool)


def seq_group_sums(groups: np.ndarray, values: np.ndarray, n: int) -> np.ndarray:
    """per group, the float64 sum from +0 of its values in the given order (sequential)"""
    order = np.argsort(groups, kind="stable")
    g, v = groups[order], np.asarray(values, np.float64)[order]
    counts = np.bincount(g, minlength=n)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    acc = np.zeros(n)
    for i in range(int(counts.max(initial=0))):
        sel = np.flatnonzero(counts > i)
        acc[sel] = acc[sel] + v[starts[sel] + i]
    return acc


def out_weights(parts, n: int, dtype) -> Tuple[np.ndarray, np.ndarray, int, int]:
    """(w float64, inv T, edges with a negative / NaN / +-inf value, non-dangling vertices whose inverse is not finite or 0)"""
    u, _, a, ok = entries(parts)
    a = a.astype(np.float64)
    bad = int(np.count_nonzero(ok & ~((a >= 0) & np.isfinite(a))))
    w = seq_group_sums(u[ok], a[ok], n)
    with np.errstate(divide="ignore", over="ignore"):
        inv = np.where(w == 0, 0.0, 1.0 / np.where(w == 0, 1.0, w)).astype(dtype)
    bad_inv = int(np.count_nonzero((w != 0) & (~np.isfinite(inv) | (inv == 0))))
    return w, inv, bad, bad_inv


def scale_parts(parts, inv: np.ndarray):
    """every block with entry (r, c) holding fl_T(a * inv[map(c)]) (0 where the column is not routed)"""
    out = []
    for A, m in parts:
        c = A.indices.astype(np.int64)
        u = c if m is None else np.asarray(m, np.int64)[c]
        s = np.where(u >= 0, inv[np.maximum(u, 0)], 0).astype(A.dtype)
        out.append((sparse.csr_matrix((A.data * s, A.indices, A.indptr), shape=A.shape), m))
    return out


def operator(parts, n: int) -> sparse.csr_matrix:
    """M (or M^ of scaled parts) as a float64 level-0 matrix, rows v = destinations (duplicates summed)"""
    u, v, a, ok = entries(parts)
    return sparse.csr_matrix((a[ok], (v[ok], u[ok])), shape=(n, n))


def out_degrees(parts, n: int) -> np.ndarray:
    u, _, _, ok = entries(parts)
    return np.bincount(u[ok], minlength=n)


# ---- reductions, restart and update -------------------------------------------------------------------------------------
def chunk_sums(A: np.ndarray) -> np.ndarray:
    """float64 column sums over 512-row chunks: sequential from +0 inside a chunk, the partials added in order from +0"""
    A = np.asarray(A)
    n, k = A.shape
    nch = -(-n // CHUNK)
    out = np.zeros(k)
    for c0 in range(0, k, 32):
        blk = np.zeros((nch * CHUNK, min(32, k - c0)))
        blk[:n] = A[:, c0:c0 + 32]
        P = np.concatenate([np.zeros((nch, 1, blk.shape[1])), blk.reshape(nch, CHUNK, -1)], axis=1)
        part = np.cumsum(P, axis=1)[:, -1, :]
        out[c0:c0 + 32] = np.cumsum(np.concatenate([np.zeros((1, part.shape[1])), part]), axis=0)[-1]
    return out


def bad_columns(X0: np.ndarray) -> np.ndarray:
    """the columns the restart refuses: a negative, NaN or +-inf value, or a sum that is not positive and finite"""
    X = np.asarray(X0, np.float64)
    sigma = chunk_sums(X)
    return np.flatnonzero(np.any(~((X >= 0) & np.isfinite(X)), axis=0) | ~(sigma > 0) | ~np.isfinite(sigma))


def restart(X0: np.ndarray, dangling: np.ndarray, dtype) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(S, sigma, m_0)"""
    X = np.asarray(X0).astype(np.float64)
    sigma = chunk_sums(X)
    S = (X / sigma).astype(dtype)
    return S, sigma, chunk_sums(np.where(dangling[:, None], S.astype(np.float64), 0.0))


def update(Y: np.ndarray, P: np.ndarray, S: np.ndarray, dangling: np.ndarray, alpha: float, m: np.ndarray, dtype):
    """(p_{t+1}, r_{t+1}, m_{t+1}) of one iterate given the step Y, bit for bit"""
    alpha = float(alpha)
    beta = 1.0 - alpha
    c = beta + alpha * np.asarray(m, np.float64)
    q = (alpha * np.asarray(Y, np.float64) + c * np.asarray(S, np.float64)).astype(dtype)
    q64 = q.astype(np.float64)
    r = chunk_sums(np.abs(q64 - np.asarray(P, np.float64)))
    return q, r, chunk_sums(np.where(dangling[:, None], q64, 0.0))


class Walk:
    """the operator of one decomposition: w, inv, M^ (float64 of its T values), dangling rows and the per-row bound terms"""

    def __init__(self, parts, n: int, dtype, to_prev, width: int):
        self.parts, self.n, self.dtype = parts, n, np.dtype(dtype)
        self.w, self.inv, self.bad_edges, self.bad_inv = out_weights(parts, n, dtype)
        self.dangling = self.w == 0
        self.scaled = scale_parts(parts, self.inv)
        self.M = operator(self.scaled, n)
        self.max_degree = int(out_degrees(parts, n).max(initial=0))
        self.heights = chain_heights([np.diff(A.indptr) for A, _ in parts], to_prev, width)

    @classmethod
    def of(cls, dec, width: int, dtype=np.float32, add_identity: bool = False, block_diagonal: bool = True):
        parts, proto = level_parts(dec, width, block_diagonal=block_diagonal, add_identity=add_identity, dtype=dtype)
        return cls(parts, proto.rows[0], dtype, proto.to_prev, width)

    def restart(self, X0):
        return restart(X0, self.dangling, self.dtype)

    def loop64(self, X0, alpha: float, tol: float, max_steps: int):
        """the iteration in float64 from S: (p float64, residuals [steps x k], every iterate p_1 .. p_T)"""
        S, _, _ = self.restart(X0)
        S64 = S.astype(np.float64)
        p = S64.copy()
        beta = 1.0 - alpha
        res, its = [], []
        for _ in range(max_steps):
            m = chunk_sums(np.where(self.dangling[:, None], p, 0.0))
            q = alpha * (self.M @ p) + (beta + alpha * m) * S64
            r = chunk_sums(np.abs(q - p))
            res.append(r), its.append(q)
            p = q
            if r.max(initial=0.0) <= tol:
                break
        return p, np.array(res).reshape(len(res), S.shape[1]), its

    def bound(self, iterates: List[np.ndarray], alpha: float) -> np.ndarray:
        """E_T per column after len(iterates) steps (module docstring)"""
        u, eta_abs = unit(self.dtype)
        nch = -(-self.n // CHUNK)
        cm = CHUNK + nch + 2
        h = self.heights.astype(np.float64) + 5
        gc = gamma(cm, U64)
        eps = gamma(h, u) + gc + gamma(h, u) * gc
        eps_ref = gamma(h + cm, U64)
        g2, gd = gamma(2, u), gamma(self.max_degree + 1, U64)
        g1 = gamma(1, u)
        eta = max(g2 + gd + g2 * gd, g1 + gc + g1 * gc)
        rho = alpha * (1 + eta)
        absolute = float(np.sum(h)) * eta_abs * 2
        wgt = ((eps + eps_ref) / (1 - eps_ref))[:, None]
        E = np.zeros(iterates[0].shape[1] if iterates else 0)
        for q in iterates:
            E = rho * (1 + eps.max(initial=0.0)) * E + np.sum(wgt * q, axis=0) + absolute
        return E


def nx_graph(parts, n: int):
    """the weighted MultiDiGraph of M (duplicates as parallel edges): networkx.pagerank's input"""
    import networkx as nx
    u, v, a, ok = entries(parts)
    G = nx.MultiDiGraph()
    G.add_nodes_from(range(n))
    G.add_weighted_edges_from(zip(u[ok].tolist(), v[ok].tolist(), a[ok].tolist()))
    return G
