"""The store-only epilogue functors (value chain, feature bias, colour lin0, ReLU, plain store, ReLU-mask dgrad,
encoding-gradient accumulation, the GEMM self-test's plain store) through the wgmma NT tiles: values against fp64, the
bf16 split against the functor's own fp32 copy, sentinels around every output (rows >= M, columns past what the
functor writes) that must survive, and which store path each shape takes.  Outputs whose rows end on 16 bytes leave the
SM by TMA bulk stores through the epilogue ring; a launch with an output that does not (TMA bounds columns in whole 16
bytes) keeps register stores.  Shapes: ragged row counts, N = 217 in a 224-wide stash and a 256-wide skip input whose
columns 217..255 hold another kernel's data, N = 200 in a 224-wide stash (ring-stored zero padding), single 64-wide
column tiles, K = 39, 256 and 320 (streamed B), one and three bf16 products."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

BETA = 100.0
BAR = 3e-5
BAR_D1 = 2e-4
BAR_NP1 = 3e-5                 # NPROD = 1 against the fp64 product of the hi halves: only the fp32 sums differ
EXTRA = 5                      # sentinel rows below every output


def r8(n):
    return (n + 7) // 8 * 8


def r4(n):
    return (n + 3) // 4 * 4


def _lib():
    from avatarclip_b200 import _lib as L
    return L


def _epi_fn():
    L = _lib().lib()
    f = L.avc_tc_epi_test
    vp, i32 = C.c_void_p, C.c_int32
    f.argtypes = [i32, vp, vp, C.c_int64, i32, i32, i32, vp, vp, i32, vp, vp, C.c_float, C.c_float, vp, vp, i32, vp,
                  C.c_size_t, vp]
    f.restype = C.c_int
    return f


def _last_ring():
    f = _lib().lib().avc_tc_nt_last_ring
    f.restype = C.c_int
    return f()


def _ptr(t):
    return None if t is None else t.data_ptr()


def _sentinel_split(M, ld2):
    """[M + EXTRA][ld2] fp32 buffer holding bf16 pairs: known finite values everywhere (hi then lo halves of a row)."""
    pat = (torch.arange((M + EXTRA) * 2 * ld2, dtype=torch.float32) % 97 - 48.0).bfloat16()
    return pat.view(torch.float32).reshape(M + EXTRA, ld2).cuda()


def _split(x):
    hi = x.bfloat16()
    lo = (x - hi.float()).bfloat16()
    return hi.double(), lo.double()


def _run(kind, M, N, K, ldx, ld2, X=None, Y=None, v1=None, v2=None, s=1.0, seed=0, OUT2=None):
    """Returns the fp64 accumulator the tiles compute (up to their fp32 sums), the outputs, the split buffer before the
    call and whether the launch stored through the ring."""
    L, f = _lib(), _epi_fn()
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).cuda()
    B = (torch.randn(N, K, generator=g) * 0.1).cuda()
    if X is None:
        X = torch.zeros(M, 8, device="cuda")     # unused by this functor
    OUT = torch.full((M + EXTRA, ldx), float("nan"), device="cuda")
    if OUT2 is None:
        OUT2 = _sentinel_split(M, ld2)
    before = OUT2.clone()
    ws = torch.empty(4 * (M + N) * r8(K) + 4 * M * ldx + 8 * M * ld2 + 8192, dtype=torch.uint8, device="cuda")
    L.check(f(kind, A.data_ptr(), B.data_ptr(), M, N, K, 0, _ptr(X), _ptr(Y), ldx, _ptr(v1), _ptr(v2), s, 1.0,
              OUT.data_ptr(), OUT2.data_ptr(), ld2, ws.data_ptr(), ws.numel(), L.stream_ptr()), "avc_tc_epi_test")
    torch.cuda.synchronize()
    ring = _last_ring()
    (ah, al), (bh, bl) = _split(A), _split(B)
    if kind >= 100:      # one product of the hi halves
        return ah @ bh.t(), OUT, OUT2, before, ring
    # the three products of the two-term split in fp64 (sp' = sigmoid(100 z) would turn the split's own ~1e-5 error
    # into ~1e-4)
    return ah @ bh.t() + ah @ bl.t() + al @ bh.t(), OUT, OUT2, before, ring


def _err(got, ref):
    return (got.double() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _aligned(*cols_bytes):
    return all(c % 16 == 0 for c in cols_bytes)


def _check_store(OUT, OUT2, before, M, ncols, ext16, ld2):
    """OUT: columns < ncols written, the rest and rows >= M untouched.  Split: hi / lo = the split of OUT's fp32 values
    in columns < ext16, every other bf16 of the buffer unchanged."""
    assert not torch.isnan(OUT[:M, :ncols]).any()
    assert torch.isnan(OUT[:M, ncols:]).all() and torch.isnan(OUT[M:]).all()
    h16, b16 = OUT2.view(torch.bfloat16), before.view(torch.bfloat16)
    hi, lo = h16[:M, :ld2], h16[:M, ld2:]
    v = OUT[:M, :ext16]
    want_hi = v.bfloat16()
    want_lo = (v - want_hi.float()).bfloat16()
    assert torch.equal(hi[:, :ext16].view(torch.int16), want_hi.view(torch.int16))
    assert torch.equal(lo[:, :ext16].view(torch.int16), want_lo.view(torch.int16))
    mask = torch.ones_like(h16, dtype=torch.bool)
    mask[:M, :ext16] = False
    mask[:M, ld2:ld2 + ext16] = False
    assert torch.equal(h16[mask].view(torch.int16), b16[mask].view(torch.int16))


def _softplus(z):
    bz = BETA * z
    sp = torch.where(bz > 20.0, z, torch.log1p(torch.exp(torch.clamp(bz, max=20.0))) / BETA)
    d1 = torch.where(bz > 20.0, torch.ones_like(z), torch.sigmoid(bz))
    return sp, d1


# (M, N, K, ldx, ld2): ld2 = 256 at N = 217 is the skip-layer input, whose columns 217..255 hold the encoding
VALUE_SHAPES = [(1000, 217, 256, 224, 256), (300, 64, 39, 64, 64), (4133, 256, 256, 256, 256), (129, 39, 256, 40, 40),
                (513, 128, 39, 128, 136), (777, 200, 256, 224, 208), (700, 128, 320, 128, 128)]


@pytest.mark.parametrize("M,N,K,ldx,ld2", VALUE_SHAPES)
def test_value(M, N, K, ldx, ld2):
    g = torch.Generator().manual_seed(11)
    bias = (torch.randn(N, generator=g) * 0.02).cuda()
    ring_expected = _aligned(4 * N, 2 * N)       # OUT and its split end at column N; the sp' stash at ldx
    D1 = torch.full((M + EXTRA, ldx), float("nan"), device="cuda")
    if not ring_expected:
        D1[:, N:] = 0.0          # the register path writes the padding only up to N rounded to 4: the rest is the zeros
        #                          the stash is allocated with
    s = 0.7071067811865476
    acc, OUT, OUT2, before, ring = _run(6, M, N, K, ldx, ld2, Y=D1, v1=bias, s=s, seed=1)
    assert ring == int(ring_expected)
    sp, d1 = _softplus(acc + bias.double()[None, :])
    eo, ed = _err(OUT[:M, :N], sp * s), _err(D1[:M, :N], d1)
    print(M, N, K, "ring", ring, "out", eo, "sp'", ed)
    # sp' = sigmoid(100 z) has a slope of up to 25 in z: the fp32 sums of z (~3e-6 off at K = 256) move it by up to ~1e-4
    assert eo < BAR and ed < BAR_D1
    assert torch.all(D1[:M, N:] == 0)            # the stash padding is zero (written by the ring path) ...
    assert torch.isnan(D1[M:, :N]).all()         # ... and no row >= M is written
    _check_store(OUT, OUT2, before, M, N, N, ld2)


STORE_SHAPES = [(1000, 217, 256), (300, 64, 39), (4133, 256, 256), (129, 39, 256), (513, 128, 39), (700, 128, 320)]


@pytest.mark.parametrize("M,N,K", STORE_SHAPES)
def test_bias(M, N, K):
    ldx = r8(N)
    g = torch.Generator().manual_seed(12)
    bias = torch.randn(N, generator=g).cuda()
    acc, OUT, OUT2, before, ring = _run(7, M, N, K, ldx, ldx, v1=bias, seed=2)
    assert ring == int(_aligned(2 * r4(N)))
    e = _err(OUT[:M, :N], acc + bias.double()[None, :])
    print(M, N, K, "ring", ring, "bias", e)
    assert e < BAR
    assert torch.all(OUT[:M, N:r4(N)] == 0)
    _check_store(OUT, OUT2, before, M, r4(N), r4(N), ldx)


@pytest.mark.parametrize("nprod", [3, 1])
@pytest.mark.parametrize("M,N,K", STORE_SHAPES)
def test_store(M, N, K, nprod):
    ldx = r8(N)
    acc, OUT, OUT2, before, ring = _run(10 if nprod == 3 else 110, M, N, K, ldx, ldx, seed=3)
    assert ring == int(_aligned(2 * r4(N)))
    e = _err(OUT[:M, :N], acc)
    print(M, N, K, nprod, "ring", ring, "store", e)
    assert e < (BAR if nprod == 3 else BAR_NP1)
    assert torch.all(OUT[:M, N:r4(N)] == 0)
    _check_store(OUT, OUT2, before, M, r4(N), r4(N), ldx)


# EpiRelu / EpiColor0 read their bias in whole groups: the colour width is a multiple of 4
RELU_SHAPES = [(1000, 256, 256), (300, 64, 39), (4133, 128, 256), (129, 36, 256), (700, 128, 320)]


@pytest.mark.parametrize("nprod", [3, 1])
@pytest.mark.parametrize("M,N,K", RELU_SHAPES)
def test_relu(M, N, K, nprod):
    ldx = r8(N)
    g = torch.Generator().manual_seed(13)
    bias = torch.randn(N, generator=g).cuda()
    acc, OUT, OUT2, before, ring = _run(9 if nprod == 3 else 109, M, N, K, ldx, ldx, v1=bias, seed=4)
    assert ring == int(_aligned(2 * N))
    e = _err(OUT[:M, :N], torch.relu(acc + bias.double()[None, :]))
    print(M, N, K, nprod, "ring", ring, "relu", e)
    assert e < (BAR if nprod == 3 else BAR_NP1)
    _check_store(OUT, OUT2, before, M, N, N, ldx)


@pytest.mark.parametrize("nprod", [3, 1])
@pytest.mark.parametrize("M,N,K", RELU_SHAPES)
def test_color0(M, N, K, nprod):
    ldx = r8(N)
    g = torch.Generator().manual_seed(14)
    bias = torch.randn(N, generator=g).cuda()
    cin = torch.randn(M, 8, generator=g).cuda()
    WxT = torch.zeros(6, ldx)
    WxT[:, :N] = torch.randn(6, N, generator=g)
    WxT = WxT.cuda()
    acc, OUT, OUT2, before, ring = _run(8 if nprod == 3 else 108, M, N, K, ldx, ldx, X=cin, v1=bias, v2=WxT, seed=5)
    assert ring == 0             # colour lin0 keeps register stores
    ref = torch.relu(acc + bias.double()[None, :] + cin.double()[:, :6] @ WxT.double()[:, :N])
    e = _err(OUT[:M, :N], ref)
    print(M, N, K, nprod, "color0", e)
    assert e < (BAR if nprod == 3 else BAR_NP1)
    _check_store(OUT, OUT2, before, M, N, N, ldx)


@pytest.mark.parametrize("nprod", [3, 1])
@pytest.mark.parametrize("M,N,K", STORE_SHAPES)
def test_dgrad_relu_split(M, N, K, nprod):
    ldx = r8(N)
    g = torch.Generator().manual_seed(15)
    H = torch.zeros(M, ldx)
    H[:, :N] = torch.relu(torch.randn(M, N, generator=g))
    H = H.cuda()
    acc, OUT, OUT2, before, ring = _run(11 if nprod == 3 else 111, M, N, K, ldx, ldx, X=H, seed=6)
    assert ring == int(_aligned(2 * r4(N)))
    mask = (H[:, :N].bfloat16() != 0).double()
    e = _err(OUT[:M, :N], acc * mask)
    print(M, N, K, nprod, "ring", ring, "dgrad relu", e)
    assert e < (BAR if nprod == 3 else BAR_NP1)
    _check_store(OUT, OUT2, before, M, r4(N), r4(N), ldx)


@pytest.mark.parametrize("M,N,K", [(1000, 39, 256), (300, 64, 39), (129, 39, 39), (700, 39, 320)])
def test_ge(M, N, K):
    """ge += acc, ring-stored over the padded width: the padding columns and rows >= M come back bit for bit."""
    ld2 = r8(N)
    g = torch.Generator().manual_seed(16)
    GE = torch.randn(M + EXTRA, ld2, generator=g).cuda()
    ge0 = GE.clone()
    acc, _, GE, _, ring = _run(5, M, N, K, 8, ld2, OUT2=GE, seed=7)
    assert ring == 1
    e = _err(GE[:M, :N], ge0[:M, :N].double() + acc)
    print(M, N, K, "ge", e)
    assert e < BAR
    assert torch.equal(GE[:M, N:].view(torch.int32), ge0[:M, N:].view(torch.int32))
    assert torch.equal(GE[M:].view(torch.int32), ge0[M:].view(torch.int32))


@pytest.mark.parametrize("nprod", [3, 1])
@pytest.mark.parametrize("M,N,K", [(1000, 64, 256), (300, 37, 39), (129, 128, 320), (513, 200, 64)])
def test_plain_store(M, N, K, nprod):
    """The GEMM self-test's plain store: ring-stored when its rows (N floats) end on 16 bytes."""
    L = _lib()
    f = L.lib().avc_tc_gemm_nt_test
    vp = C.c_void_p
    f.argtypes = [vp, vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, vp, vp, C.c_size_t, vp]
    f.restype = C.c_int
    g = torch.Generator().manual_seed(17)
    A = torch.randn(M, K, generator=g).cuda()
    B = torch.randn(N, K, generator=g).cuda()
    Cm = torch.full((M + EXTRA, N), float("nan"), device="cuda")
    ws = torch.empty(4 * (M + N) * r8(K) + 8192, dtype=torch.uint8, device="cuda")
    L.check(f(A.data_ptr(), B.data_ptr(), M, N, K, nprod, Cm.data_ptr(), ws.data_ptr(), ws.numel(), L.stream_ptr()),
            "avc_tc_gemm_nt_test")
    torch.cuda.synchronize()
    assert _last_ring() == int(_aligned(4 * N))
    (ah, al), (bh, bl) = _split(A), _split(B)
    ref = ah @ bh.t() if nprod == 1 else ah @ bh.t() + ah @ bl.t() + al @ bh.t()
    e = _err(Cm[:M], ref)
    print(M, N, K, nprod, "plain", e)
    assert e < BAR
    assert torch.isnan(Cm[M:]).all()
