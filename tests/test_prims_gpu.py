"""The shared scan, block reduction and selection keys (csrc/avc_common.cuh, avc_scan.cu) alone, through
avc_common_kernel_test, against their numpy restatements (oracle/prims.py, pinned by test_prims_cpu.py); then their
callers at the edges of those pieces, through the public entry points, against the callers' own oracles.

Every comparison is an equality: the pieces are integer or bit-level arithmetic, and block_reduce's fp64 fold is
restated in the device's order.  Outputs carry a guard past their end that must keep its bits.

Sizes: the device-wide scan runs in tiles of 2048 elements, and the scan of the tile sums in passes of 1024 tiles, so
n = 2047, 2048, 2049 land around one tile, 2048 * 1024 +- 1 around one pass, and 2048 * 2048 + 1 needs three passes."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import animate as OA
from oracle import decimate as OD
from oracle import prims as P
from oracle import raster
from oracle import shapegen as OS
from oracle import video as OV

pytestmark = pytest.mark.gpu

TILE, PASS = 2048, 2048 * 1024
U64_MAX = np.uint64(2 ** 64 - 1)
GUARD = 64
I32_GUARD = -0x21524111           # 0xdeadbeef as an int32

_F = None


def _fn():
    global _F
    if _F is None:
        from avatarclip_b200 import _lib
        f = _lib.lib().avc_common_kernel_test
        f.argtypes = [C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p]
        f.restype = C.c_int
        _F = (_lib, f)
    return _F


def _addr(t):
    return None if t is None else (t if isinstance(t, int) else t.data_ptr())


def _run(kind, dims, ins, outs):
    _lib, f = _fn()
    d = (C.c_int64 * len(dims))(*dims)
    pi = (C.c_void_p * max(len(ins), 1))(*[_addr(t) for t in ins])
    po = (C.c_void_p * len(outs))(*[_addr(t) for t in outs])
    _lib.check(f(kind, d, pi, po, _lib.stream_ptr()), f"avc_common_kernel_test({kind})")
    torch.cuda.synchronize()


def _dev(a):
    """numpy -> device tensor; uint64 and uint32 travel as int64 / int32 of the same bits."""
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a.copy()).cuda()


def _guarded(n, dtype, fill=I32_GUARD):
    return torch.full((n + GUARD,), fill, dtype=dtype, device="cuda")


def _bits(t, dtype):
    return t.cpu().numpy().view(dtype)


# ================================================================ exclusive_scan
def _scan_sums(n):
    out = C.c_int64(-1)
    _run(5, [n], [], [C.addressof(out)])
    return out.value


def _scan(a_np, garbage=None):
    n = a_np.size
    ns = _scan_sums(n)
    assert ns == -(-n // TILE)
    a = _guarded(n, torch.int32)
    a[:n] = torch.from_numpy(a_np).cuda()
    sums = _guarded(ns, torch.int32)
    if garbage is not None:
        sums[:ns] = torch.randint(-2 ** 31, 2 ** 31 - 1, (ns,), generator=torch.Generator().manual_seed(garbage),
                                  dtype=torch.int32).cuda()
    total = _guarded(1, torch.int32)
    _run(4, [n], [], [a, sums, total])
    assert (a[n:] == I32_GUARD).all() and (sums[ns:] == I32_GUARD).all() and (total[1:] == I32_GUARD).all()
    return a[:n].cpu().numpy(), int(total[0])


def _check_scan(a_np):
    ex, tot = P.exclusive_scan(a_np)
    for garbage in (None, 7):
        got, total = _scan(a_np, garbage)
        assert total == tot
        assert np.array_equal(got.astype(np.int64), ex)


@pytest.mark.parametrize("n", [1, 2, TILE - 1, TILE, TILE + 1, PASS - 1, PASS, PASS + 1, 2 * PASS + 1])
def test_exclusive_scan_at_tile_and_pass_boundaries(n):
    a = np.random.default_rng(n).integers(0, 100, n).astype(np.int32)
    _check_scan(a)


def test_exclusive_scan_of_zeros():
    _check_scan(np.zeros(2 * PASS + 1, np.int32))


@pytest.mark.parametrize("n", [3, TILE + 5, PASS + 1])
def test_exclusive_scan_total_of_int32_max(n):
    rng = np.random.default_rng(n)
    a = np.full(n, (2 ** 31 - 1) // n, np.int64)
    a[rng.integers(0, n)] += 2 ** 31 - 1 - a.sum()
    assert a.sum() == 2 ** 31 - 1
    _check_scan(a.astype(np.int32))


# ================================================================ block_reduce
OPS = {"f64_add": (0, np.float64, np.add, np.float64(0.0)), "i32_add": (1, np.int32, np.add, np.int32(0)),
       "u64_min": (2, np.uint64, np.minimum, U64_MAX), "u64_max": (3, np.uint64, np.maximum, np.uint64(0))}
BITS = {np.float64: np.uint64, np.int32: np.int32, np.uint64: np.uint64}


def _values(rng, dt, n):
    if dt == np.float64:
        return rng.standard_normal(n) * 10.0 ** rng.uniform(-8, 8, n)
    if dt == np.int32:
        return rng.integers(-2 ** 20, 2 ** 20, n).astype(np.int32)
    return rng.integers(0, 2 ** 64, n, dtype=np.uint64)


def _reduce(op, threads, blocks, x):
    """x [3][blocks threads] -> the [3][blocks threads] results every thread received."""
    code, dt = OPS[op][0], OPS[op][1]
    xd = _dev(x)
    r = torch.full((3 * blocks * threads + GUARD,), -1, dtype=xd.dtype, device="cuda")
    _run(0, [code, threads, blocks], [xd], [r])
    assert (r[3 * blocks * threads:] == -1).all()
    return r[:3 * blocks * threads].cpu().numpy().view(dt).reshape(3, -1)


@pytest.mark.parametrize("threads", [32, 64, 96, 128, 256, 1024])
@pytest.mark.parametrize("op", list(OPS))
def test_block_reduce_is_the_fold_in_every_thread(op, threads):
    """Three back-to-back calls on one red, each on its own inputs: every thread's three results equal the fold of
    its CTA's values for that call, bit for bit."""
    code, dt, fn, init = OPS[op]
    blocks = 67
    rng = np.random.default_rng(16 * threads + code)
    x = np.stack([_values(rng, dt, blocks * threads) for _ in range(3)])
    got = _reduce(op, threads, blocks, x)
    for c in range(3):
        want = np.repeat(P.block_reduce(x[c], threads, fn, init), threads)
        b = BITS[dt]
        assert np.array_equal(got[c].view(b), want.view(b)), (c, np.flatnonzero(got[c].view(b) != want.view(b))[:8])


@pytest.mark.parametrize("threads", [32, 96, 1024])
def test_block_reduce_of_negative_zeros_is_positive_zero(threads):
    """init (+0.0) decides the sign of a zero sum: every -0.0 input gives +0.0."""
    blocks = 5
    x = np.full((3, blocks * threads), -0.0)
    x[1] = np.random.default_rng(0).standard_normal(blocks * threads)
    got = _reduce("f64_add", threads, blocks, x)
    assert (got[0].view(np.uint64) == 0).all() and (got[2].view(np.uint64) == 0).all()


# ================================================================ block_exclusive_scan
@pytest.mark.parametrize("NT", [32, 128, 256, 1024])
def test_block_exclusive_scan_with_a_running_carry(NT):
    """Per CTA `rounds` calls on one warp_tot, each from the running carry (k_scan_top's loop): zeros, large values,
    a CTA of zeros only and one whose total is exactly INT32_MAX."""
    blocks, rounds = 9, 7
    m = rounds * NT
    rng = np.random.default_rng(NT)
    x = rng.integers(0, (2 ** 31 - 1) // m, (blocks, m)).astype(np.int64)
    x[rng.random((blocks, m)) < 0.5] = 0
    x[1] = 0
    x[2, rng.integers(0, m)] += 2 ** 31 - 1 - x[2].sum()
    x[3, :] = 0
    x[3, m - 1] = 2 ** 31 - 1
    ex = _guarded(blocks * m, torch.int32)
    tot = _guarded(blocks * NT, torch.int32)
    _run(1, [NT, blocks, rounds], [_dev(x.astype(np.int32))], [ex, tot])
    assert (ex[blocks * m:] == I32_GUARD).all() and (tot[blocks * NT:] == I32_GUARD).all()
    ex, tot = ex[:blocks * m].cpu().numpy().reshape(blocks, m), tot[:blocks * NT].cpu().numpy().reshape(blocks, NT)
    for b in range(blocks):
        want, total = P.exclusive_scan(x[b])
        assert np.array_equal(ex[b].astype(np.int64), want), b
        assert (tot[b] == total).all(), b


# ================================================================ keys and selection
def _special_floats():
    bits = np.array([0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000, 0x80800000,
                     0x3F800000, 0xBF800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000, 0xFF800000,    # +-0, subnormals,
                     0x7FC00000, 0x7F800001, 0x7FFFFFFF], np.uint32)                          # +-1, max, inf, +NaN
    rng = np.random.default_rng(11)
    finite = rng.integers(0, 0x7F800000, 4000, dtype=np.uint32) | (rng.integers(0, 2, 4000, dtype=np.uint32) << 31)
    ties = (rng.integers(-8, 8, 3000) * 0.5).astype(np.float32).view(np.uint32)
    zeros = np.where(rng.random(1000) < 0.5, 0x80000000, 0).astype(np.uint32)
    v = np.concatenate([bits, finite, ties, zeros, bits])
    return v[rng.permutation(v.size)].view(np.float32)


def test_keys_equal_their_restatement():
    """ordered_bits, sel_key, sel_index and depth_key over finite values, both zeros, subnormals, +-inf and positive
    NaNs; -0.0 keys as +0.0, so equal values tie by index."""
    v = _special_floats()
    n = v.size
    ob, sk, dk = _guarded(n, torch.int32), _guarded(n, torch.int64), _guarded(n, torch.int64)
    si = _guarded(n, torch.int32)
    _run(2, [n], [_dev(v)], [ob, sk, si, dk])
    for t in (ob, sk, si, dk):
        assert (t[n:] == I32_GUARD).all()
    assert np.array_equal(_bits(ob[:n], np.uint32), P.ordered_bits(v))
    assert np.array_equal(_bits(sk[:n], np.uint64), P.sel_key(v))
    assert np.array_equal(si[:n].cpu().numpy(), np.arange(n))
    assert np.array_equal(_bits(dk[:n], np.uint64), P.depth_key(v))


def _select(v, z, threads, blocks):
    mx, mn = _guarded(1, torch.int64), _guarded(1, torch.int64)
    best = _guarded(1, torch.int32)
    _run(3, [v.size, threads, blocks], [_dev(v), None if z is None else _dev(z)], [mx, mn, best])
    for t in (mx, mn, best):
        assert (t[1:] == I32_GUARD).all()
    return int(_bits(mx[:1], np.uint64)[0]), int(_bits(mn[:1], np.uint64)[0]), int(best[0])


@pytest.mark.parametrize("threads,blocks", [(256, 64), (32, 1000), (1024, 132), (1, 1)])
def test_selection_is_the_first_argmax_across_ctas(threads, blocks):
    """The 64-bit atomicMax of sel_key and atomicMin of depth_key from every thread of a grid-stride loop: the first
    index of the largest value and of the smallest z, with the tied entries handled by different CTAs."""
    n = 200_003 if threads > 1 else 5000
    rng = np.random.default_rng(threads)
    v = rng.integers(-50, 8, n).astype(np.float32)              # the maximum, 7, on ~n / 58 indices
    z = rng.integers(3, 60, n).astype(np.float32) * np.float32(0.125)
    z[rng.integers(n // 2, n, 40)] = np.float32(0.25)           # the smallest z, only in the second half
    mx, mn, best = _select(v, z, threads, blocks)
    assert best == P.first_argmax(v) and mx == int(P.sel_key(v).max())
    assert mn == int(P.depth_key(z).min()) and (mn & 0xFFFFFFFF) == P.smallest(z)
    # the largest value only twice, far apart; then a maximum of zeros whose first is -0.0
    v[:] = -1.0
    v[n - 3] = v[n // 3] = 2.5
    assert _select(v, None, threads, blocks)[2] == n // 3
    v[:] = -1.0
    zi = np.sort(rng.choice(n, 50, replace=False))
    v[zi] = 0.0
    v[zi[::2]] = -0.0
    mx, mn, best = _select(v, None, threads, blocks)
    assert best == zi[0] and mx == int(P.sel_key(v).max()) and mn == 2 ** 64 - 1


def test_the_two_zeros_tie_by_index():
    for v in ([-0.0, 0.0], [0.0, -0.0], [-1.0, -0.0, 0.0, -0.0]):
        v = np.array(v, np.float32)
        assert _select(v, None, 32, 1)[2] == P.first_argmax(v) == int(np.argmax(v))


# ================================================================ callers: mask compaction
def _compact(dil, W, cap):
    from avatarclip_b200 import _lib, views
    L = views._sigs()
    n = dil.shape[0]
    d = torch.from_numpy(dil.astype(np.uint8)).cuda()
    in_mask = torch.full((W * W + GUARD,), 0xAB, dtype=torch.uint8, device="cuda")
    pix, cnt = _guarded(cap, torch.int32), _guarded(1, torch.int32)
    _lib.check(L.avc_mask_compact(_lib.ptr(d), n, W, cap, _lib.ptr(in_mask), _lib.ptr(pix), _lib.ptr(cnt),
                                  _lib.stream_ptr()), "avc_mask_compact")
    torch.cuda.synchronize()
    assert (in_mask[W * W:] == 0xAB).all() and (cnt[1:] == I32_GUARD).all()
    return in_mask[:W * W].cpu().numpy(), pix.cpu().numpy(), int(cnt[0])


@pytest.mark.parametrize("W", [1, 31, 32, 33, 1023, 1024])
def test_mask_compact_at_canvas_edges(W):
    """Down- and up-sampling (n above and below W), empty, full and random masks, and a cap below the kept count:
    the first cap pixels in order, the count still the full total."""
    rng = np.random.default_rng(W)
    for n in sorted({max(1, W // 3), W + 7, 33}):
        for fill in ("random", "empty", "full"):
            dil = {"random": rng.random((n, n)) < 0.3, "empty": np.zeros((n, n), bool),
                   "full": np.ones((n, n), bool)}[fill]
            rm = raster.nearest_resize(dil, W).reshape(-1)
            want = np.flatnonzero(rm)
            got_m, pix, count = _compact(dil, W, W * W)
            assert np.array_equal(got_m, rm.astype(np.uint8)), (n, fill)
            assert count == want.size and np.array_equal(pix[:count], want), (n, fill)
            assert (pix[count:] == I32_GUARD).all()
            if want.size > 1:
                cap = want.size // 2
                _, pix, count = _compact(dil, W, cap)
                assert count == want.size and np.array_equal(pix[:cap], want[:cap]), (n, fill)
                assert (pix[cap:] == I32_GUARD).all()


# ================================================================ callers: vertex -> face adjacency
def _check_adjacency(faces, V):
    from avatarclip_b200 import video
    adj = video.adjacency(torch.from_numpy(np.ascontiguousarray(faces, np.int32)).cuda(), V)
    off, vf = OV.adjacency(faces, V)
    assert np.array_equal(adj.offsets.cpu().numpy(), off)
    assert np.array_equal(adj.vf[:int(off[-1])].cpu().numpy(), vf)


def _strip(V):
    """A triangle strip over vertices 0 .. V - 2 (the last vertex in no face)."""
    i = np.arange(max(V - 3, 1))
    return np.stack([i, i + 1 + i % 2, i + 2 - i % 2], 1) % V


def test_adjacency_of_degenerate_meshes():
    _check_adjacency(np.array([[0, 1, 2], [2, 0, 1]]), 1)             # V = 1: the indices >= V are skipped
    _check_adjacency(np.array([[0, 0, 0]]), 1)
    rng = np.random.default_rng(0)
    _check_adjacency(2 * rng.integers(0, 2500, (3000, 3)), 5000)      # the odd vertices in no face
    F = 1500                                                          # vertex 0 in every face
    i = np.arange(F)
    _check_adjacency(np.stack([np.zeros(F, np.int64), 1 + i, 1 + (i + 1) % F], 1), F + 1)
    _check_adjacency(rng.permutation(np.stack([1 + i, np.zeros(F, np.int64), 1 + (i + 1) % F], 1)), F + 1)


@pytest.mark.parametrize("V", [2, TILE - 1, TILE, TILE + 1, PASS - 1, PASS, PASS + 1, 2 * PASS + 1])
def test_adjacency_at_scan_boundaries(V):
    _check_adjacency(_strip(V), V)


# ================================================================ callers: selections
@pytest.mark.parametrize("N", [1, 31, 1023, 1024, 1025])
def test_cosine_topk_full_order(N):
    """k = N: the whole descending order of the device's own scores, ties to the smaller index; then all rows equal."""
    from avatarclip_b200 import animate as A
    g = torch.Generator(device="cuda").manual_seed(N)
    rows = torch.randn(N, 64, generator=g, device="cuda")
    vec = torch.randn(64, generator=g, device="cuda")
    if N > 4:
        rows[N // 2] = rows[N - 1] = rows[1]                       # three equal scores
    cos, idx = A.cosine_topk(rows, vec, N)
    c = cos.cpu().numpy()
    assert np.abs(c - OA.cosine(rows.cpu().numpy(), vec.cpu().numpy())).max() <= 1e-6
    assert np.array_equal(idx.cpu().numpy(), np.argsort(-c, kind="stable"))
    _, idx = A.cosine_topk(rows[:1].expand(N, 64).contiguous(), vec, N)
    assert np.array_equal(idx.cpu().numpy(), np.arange(N))


def test_pose_score_groups_of_one_and_ties_across_ctas():
    """One CTA per pose: a group of 1 selects 0; tied scores of poses in different CTAs select the first."""
    from avatarclip_b200 import animate as A
    g = torch.Generator().manual_seed(8)
    emb, text = torch.randn(3, 24, 64, generator=g), torch.randn(64, generator=g)
    score, best = A.pose_score(emb.cuda(), text.cuda(), 1)
    ref = OA.cosine(emb.double().mean(0), text)
    assert np.abs(score.cpu().numpy() - ref).max() <= 1e-6 and best.cpu().tolist() == [0] * 24
    emb[:, [9, 13, 14]] = text * 3                                   # group 1 (poses 8..15): 9 first
    emb[:, [23, 17]] = text * 2                                      # group 2 (poses 16..23): 17 first
    score, best = A.pose_score(emb.cuda(), text.cuda(), 8)
    s = score.cpu().numpy()
    assert s[9] == s[13] == s[14] and s[17] == s[23]
    assert best.cpu().tolist() == [P.first_argmax(s[k:k + 8]) for k in (0, 8, 16)]
    assert best.cpu().tolist()[1:] == [1, 1]


def test_codebook_argmax_of_one_row():
    from avatarclip_b200 import shapegen as S
    g = torch.Generator(device="cuda").manual_seed(1)
    Cb, e, d = (torch.randn(*s, generator=g, device="cuda") for s in ((1, 512), (512,), (512,)))
    cos, best = S.codebook_argmax(Cb, e, d)
    assert best == 0 and abs(cos.item() - OS.codebook_cos(Cb.cpu(), e.cpu(), d.cpu())[0]) <= 1e-6
    cos, best = S.codebook_argmax(e[None].clone(), e, d)             # C == e: cos 0
    assert best == 0 and cos.item() == 0.0


# ================================================================ callers: decimation budget
@pytest.mark.parametrize("name", ["sphere", "fan_boundary"])
def test_decimate_every_budget_of_the_first_rounds(name):
    """Every target from F - 1 down to F - 40: k_dc_cap's face budget lands on, and one face past, every prefix of
    the first round's selected collapses (two faces each inside, one on the boundary)."""
    from avatarclip_b200 import export as X
    from avatarclip_b200.drive import Mesh
    v, f = OD.sphere() if name == "sphere" else OD.fan(12)[:2]
    c = np.random.default_rng(5).random(v.shape).astype(np.float32)
    F = f.shape[0]
    for target in range(F - 1, F - 41, -1):
        m, rounds = X._decimate(Mesh(torch.from_numpy(v).cuda(), torch.from_numpy(f.astype(np.int32)).cuda(), c),
                                target)
        want = OD.decimate(v, f, target, colors=c)
        assert rounds == want["rounds"], target
        assert np.array_equal(m.triangles.cpu().numpy(), want["faces"]), target
        assert m.vertices.cpu().numpy().tobytes() == want["vertices"].tobytes(), target
        assert m.vertex_colors.tobytes() == want["colors"].tobytes(), target
