"""CPU oracle (test infrastructure, never on the product path): the shared pieces of the mesh, view and pose kernels
(avatarclip_b200/csrc/avc_common.cuh, avc_scan.cu) restated with numpy, bit for bit:

- ``exclusive_scan``: the exclusive prefix sum and the total in int64, so that a sum the device's int32 cannot hold
  shows up as a mismatch instead of wrapping the same way on both sides.
- ``block_reduce``: the fold of block_reduce -- per warp an xor tree (x[l] = x[l] op x[l ^ o] for o = 16, 8, 4, 2, 1),
  then the warp results folded onto ``init`` in warp order.  IEEE addition is commutative, so every lane of a warp
  holds the same sum and the restatement equals the device's bits.
- ``ordered_bits``, ``sel_key``, ``sel_index``, ``depth_key`` on uint32 / uint64 views, and the selections they make:
  the first argmax and the smallest (z, id).
"""
from __future__ import annotations

import numpy as np

_SIGN = np.uint32(0x80000000)
_LOW = np.uint64(0xFFFFFFFF)


def exclusive_scan(a):
    """(exclusive prefix sum [n] int64, total int64) of a in index order."""
    c = np.cumsum(np.asarray(a, dtype=np.int64))
    return np.concatenate([[0], c[:-1]]).astype(np.int64), int(c[-1])


def block_reduce(x, threads: int, op, init):
    """block_reduce over consecutive CTAs of ``threads`` (a multiple of 32) values of x: [blocks] results.  ``op`` is a
    numpy binary ufunc (np.add, np.minimum, np.maximum) applied elementwise, ``init`` a scalar of x's dtype."""
    x = np.asarray(x)
    assert threads % 32 == 0 and x.size % threads == 0
    w = x.reshape(-1, threads // 32, 32)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        w = op(w, w[..., lane ^ o])
    acc = np.full(w.shape[0], init, dtype=x.dtype)
    for k in range(w.shape[1]):
        acc = op(acc, w[:, k, 0])
    return acc


def ordered_bits(v):
    """float32 -> uint32 whose unsigned order is the float order; -0.0 maps to +0.0's bits."""
    u = np.ascontiguousarray(v, dtype=np.float32).view(np.uint32).copy()
    u[u == _SIGN] = 0
    return np.where(u & _SIGN, ~u, u | _SIGN).astype(np.uint32)


def sel_key(v, idx=None):
    """(ordered value bits, ~index) as uint64; idx defaults to 0..n-1."""
    v = np.asarray(v, dtype=np.float32)
    i = np.arange(v.size, dtype=np.uint64) if idx is None else np.asarray(idx).astype(np.uint64)
    return (ordered_bits(v).astype(np.uint64) << np.uint64(32)) | (_LOW - i)


def sel_index(key):
    return (_LOW - (np.asarray(key, dtype=np.uint64) & _LOW)).astype(np.int64)


def depth_key(z, idx=None):
    """(bits of z, id) as uint64 for z >= +0; idx defaults to 0..n-1."""
    z = np.ascontiguousarray(z, dtype=np.float32)
    i = np.arange(z.size, dtype=np.uint64) if idx is None else np.asarray(idx).astype(np.uint64)
    return (z.view(np.uint32).astype(np.uint64) << np.uint64(32)) | i


def first_argmax(v) -> int:
    """The first index of the largest value, the two zeros equal (np.argmax's rule; no NaN)."""
    v = np.asarray(v, dtype=np.float32)
    assert not np.isnan(v).any()
    return int(np.flatnonzero(v == v.max())[0])


def smallest(z) -> int:
    """The index of the smallest (z, index) for z >= +0: the first index of the smallest z."""
    z = np.asarray(z, dtype=np.float32)
    assert (z >= 0).all() and not np.signbit(z).any()
    return int(np.lexsort((np.arange(z.size), z))[0])
