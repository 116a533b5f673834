"""The numpy restatements of the shared scan, block reduction and selection keys (oracle/prims.py) against independent
statements of what they compute: the fold against math.fsum, the keys' order against numpy's stable sorts, the scan
against cumsum.  And oracle.raster.nearest_resize, which the mask compaction is checked against, against torch."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import prims as P
from oracle import raster


def _spread(rng, n):
    """Values of both signs over 16 decades, so that the order of a sum's additions shows in its rounding."""
    return rng.standard_normal(n) * 10.0 ** rng.uniform(-8, 8, n)


@pytest.mark.parametrize("threads", [32, 64, 96, 128, 256, 1024])
def test_fold_agrees_with_fsum_within_its_rounding(threads):
    rng = np.random.default_rng(threads)
    x = _spread(rng, 40 * threads)
    got = P.block_reduce(x, threads, np.add, 0.0)
    depth = 5 + threads // 32                     # additions on the longest path: the xor tree, then the warp fold
    u = 2.0 ** -53
    for b in range(40):
        xb = x[b * threads:(b + 1) * threads]
        bound = depth * u / (1 - depth * u) * np.abs(xb).sum()
        assert abs(got[b] - math.fsum(xb)) <= bound
    # the fold is not the left-to-right sum: the restatement keeps the device's order, not another one
    left = np.array([sum(x[b * threads:(b + 1) * threads].tolist()) for b in range(40)])
    if threads >= 64:
        assert (got != left).any()


def test_fold_of_integers_and_extrema_is_exact():
    rng = np.random.default_rng(1)
    x = rng.integers(-2 ** 20, 2 ** 20, 8 * 256).astype(np.int32)
    assert np.array_equal(P.block_reduce(x, 256, np.add, np.int32(0)), x.reshape(8, -1).sum(1))
    q = rng.integers(0, 2 ** 64, 8 * 96, dtype=np.uint64)
    assert np.array_equal(P.block_reduce(q, 96, np.minimum, np.uint64(2 ** 64 - 1)), q.reshape(8, -1).min(1))
    assert np.array_equal(P.block_reduce(q, 96, np.maximum, np.uint64(0)), q.reshape(8, -1).max(1))


def test_fold_of_negative_zeros_takes_the_sign_of_init():
    r = P.block_reduce(np.full(128, -0.0), 128, np.add, 0.0)
    assert r.view(np.uint64)[0] == 0
    r = P.block_reduce(np.full(128, -0.0), 128, np.add, -0.0)
    assert np.signbit(r[0])


def test_exclusive_scan_is_cumsum_in_int64():
    a = np.array([5, 0, 2 ** 31 - 1, 7], np.int32)
    ex, total = P.exclusive_scan(a)
    assert ex.tolist() == [0, 5, 5, 2 ** 31 + 4] and total == 2 ** 31 + 11


def _finite_with_ties(rng, n):
    v = rng.integers(-20, 20, n).astype(np.float32) * np.float32(0.25)
    v[rng.random(n) < 0.1] = -0.0
    v[rng.random(n) < 0.1] = 0.0
    v[rng.random(n) < 0.05] = rng.choice(np.array([1e-45, -1e-45, 1e-39, -3e-40], np.float32), 1)
    return v


def test_sel_key_order_is_descending_value_then_ascending_index():
    rng = np.random.default_rng(2)
    for n in (1, 2, 33, 1000):
        v = _finite_with_ties(rng, n)
        k = P.sel_key(v)
        assert np.unique(k).size == n
        assert np.array_equal(np.argsort(k)[::-1], np.argsort(-v, kind="stable"))
        assert P.sel_index(k).tolist() == list(range(n))
        assert P.sel_index(k.max()) == P.first_argmax(v) == int(np.argmax(v))


def test_the_two_zeros_key_alike():
    assert P.ordered_bits(np.array([-0.0, 0.0], np.float32)).tolist() == [0x80000000, 0x80000000]
    k = P.sel_key(np.array([-0.0, 0.0], np.float32))
    assert k[0] > k[1]                                # equal values: the smaller index wins
    k = P.sel_key(np.array([0.0, -0.0], np.float32))
    assert k[0] > k[1]


def test_ordered_bits_keep_the_order_of_the_special_values():
    v = np.array([-np.inf, -3.4e38, -1.0, -1e-39, -1e-45, -0.0, 0.0, 1e-45, 1e-39, 1.0, 3.4e38, np.inf], np.float32)
    o = P.ordered_bits(v).astype(np.int64)
    assert (np.diff(o)[:5] > 0).all() and o[5] == o[6] and (np.diff(o)[6:] > 0).all()
    nan = np.array([0x7FC00000], np.uint32).view(np.float32)
    assert P.ordered_bits(nan)[0] > P.ordered_bits(np.array([np.inf], np.float32))[0]


def test_depth_key_order_is_ascending_z_then_ascending_id():
    rng = np.random.default_rng(3)
    for n in (1, 2, 33, 1000):
        z = np.abs(_finite_with_ties(rng, n))
        z[z == 0] = 0.0                              # z >= +0
        k = P.depth_key(z)
        assert np.array_equal(np.argsort(k), np.lexsort((np.arange(n), z)))
        assert int(np.argmin(k)) == P.smallest(z)


@pytest.mark.parametrize("n,W", [(33, 1023), (256, 1023), (100, 31), (7, 33), (1031, 1024), (341, 1024), (1, 1),
                                 (8, 1)])
def test_nearest_resize_is_torch_interpolate(n, W):
    a = np.arange(n * n, dtype=np.float32).reshape(n, n)
    want = F.interpolate(torch.from_numpy(a)[None, None], size=(W, W))[0, 0].numpy()
    assert np.array_equal(raster.nearest_resize(a, W), want)
