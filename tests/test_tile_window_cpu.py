"""The L2 budget that picks the row-tile list of a tile-kernel launch (``arrow_tile_rows_rule``), pinned without a GPU.

The CTAs of a launch share one atomic ticket, so the rows in flight are about ``resident CTAs x rows per tile``.  The rule
lets the X rows of that window (``resident CTAs x rows x k x element bytes``) take a quarter of the L2 and picks the
largest list that fits: 128 rows (float32, k <= 32), 64, 32, else 16.
"""
import numpy as np
import pytest

from arrow_matrix_b200 import _lib
from tests import tile_dispatch as td

H100 = dict(l2=50 << 20, ctas=4 * 132)        # H100 SXM: 50 MB L2, 132 SMs x 4 resident tile CTAs
B200 = dict(l2=126 << 20, ctas=4 * 148)


def rule(k, elem, dev, big_ok):
    return _lib.load_library().arrow_tile_rows_rule(k, elem, dev["l2"], dev["ctas"], int(big_ok))


def restated(k, elem, l2, ctas, big_ok):
    for rows in ((128,) if big_ok else ()) + (64, 32):
        if ctas * rows * k * elem <= l2 // 4:
            return rows
    return 16


@pytest.mark.parametrize("dev,elem,expected", [
    # k:            4    8   16   32   64  128  256
    (H100, 4, [128, 128, 128, 128, 64, 32, 16]),
    (H100, 8, [64, 64, 64, 64, 32, 16, 16]),
    (B200, 4, [128, 128, 128, 128, 64, 64, 32]),
    (B200, 8, [64, 64, 64, 64, 64, 32, 16]),
])
def test_rule_on_h100_and_b200(dev, elem, expected):
    ks = [4, 8, 16, 32, 64, 128, 256]
    got = [rule(k, elem, dev, elem == 4 and k <= 32) for k in ks]
    assert got == expected
    assert got == [restated(k, elem, dev["l2"], dev["ctas"], elem == 4 and k <= 32) for k in ks]


def test_rule_follows_the_window():
    # fewer resident CTAs (a capped grid) leave room for longer tiles; the floor is 16 rows
    assert rule(128, 4, dict(H100, ctas=2 * 132), False) == 64
    assert rule(128, 4, dict(H100, ctas=66 * 2), False) == 64
    assert rule(512, 8, H100, False) == 16
    # without a 128-row kernel for the shape the largest list is 64 rows
    assert rule(16, 4, H100, False) == 64
    for k in range(4, 260, 4):
        for elem in (4, 8):
            for dev in (H100, B200, dict(l2=40 << 20, ctas=4 * 114)):
                big_ok = elem == 4 and k <= 32
                assert rule(k, elem, dev, big_ok) == restated(k, elem, dev["l2"], dev["ctas"], big_ok)


def test_rule_refuses_bad_arguments():
    lib = _lib.load_library()
    for args in ((0, 4, 1 << 20, 4, 0), (16, 2, 1 << 20, 4, 0), (16, 4, 0, 4, 0), (16, 4, 1 << 20, 0, 0)):
        assert lib.arrow_tile_rows_rule(*args) < 0


def test_narrow_lists_fit_the_64_row_kernels():
    """the 16- and 32-row lists run on the TR = 64 / TN = 1024 instances: every tile within those bounds"""
    rng = np.random.default_rng(5)
    lens = rng.integers(0, 40, size=5000)
    lens[100:140] = rng.integers(250, 511, size=40)      # single rows above the narrow nnz caps
    lens[[7, 900]] = [512, 513]
    ip = np.concatenate([[0], np.cumsum(lens)])
    for rows_cap, nnz_cap in ((16, 256), (32, 512)):
        t = td.build_tiles(ip, rows_cap, nnz_cap)
        n = t[:, 1] - t[:, 0]
        assert (n <= rows_cap).all() and (t[:, 3] - t[:, 2] <= td.TILE_NNZ - 8).all()
        assert ((t[:, 3] - t[:, 2] <= nnz_cap - 4) | (n == 1)).all()
        assert 900 not in np.concatenate([np.arange(a, b) for a, b, _, _ in t])
