"""The staged epilogue functors (second-order sweep, value backward, gradient chain) through the wgmma NT tiles with the
output sets the renderer launches them with: their outputs are written over their staged operands in shared memory and
leave the SM by TMA bulk stores.  Values against fp64 restatements of the formulas, the store path the launch took,
sentinel rows below every output that must survive, zero padding columns, zbar_prev updated in place and the encoding
gradient accumulated.  Shapes: ragged row counts, N = 217 in a 224-wide stash (and a 256-wide ubar whose columns
224..255 belong to another kernel), single 64-wide column tiles, K = 39 and 256."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BETA = 100.0
BAR = 3e-5
EXTRA = 5                      # sentinel rows below every output


def r8(n):
    return (n + 7) // 8 * 8


def _lib():
    from avatarclip_b200 import _lib as L
    return L


def _run(kind, M, N, K, ldx, X, Y=None, v1=None, v2=None, s=1.0, s2=1.0, OUT=None, OUT2=None, ld2=8, Nv=0, seed=0):
    """Runs one avc_tc_epi_test launch; returns the fp64 accumulator and whether the launch stored through the ring."""
    L = _lib()
    f = L.lib().avc_tc_epi_test
    vp, i32 = C.c_void_p, C.c_int32
    f.argtypes = [i32, vp, vp, C.c_int64, i32, i32, i32, vp, vp, i32, vp, vp, C.c_float, C.c_float, vp, vp, i32, vp,
                  C.c_size_t, vp]
    f.restype = C.c_int
    ring = L.lib().avc_tc_nt_last_ring
    ring.restype = C.c_int
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).cuda()
    B = (torch.randn(N, K, generator=g) * 0.1).cuda()
    ws = torch.empty(4 * (M + N) * r8(K) + 4 * M * ldx + 8 * M * ld2 + 8192, dtype=torch.uint8, device="cuda")
    p = [None if t is None else t.data_ptr() for t in (X, Y, v1, v2, OUT, OUT2)]
    L.check(f(kind, A.data_ptr(), B.data_ptr(), M, N, K, Nv, p[0], p[1], ldx, p[2], p[3], s, s2, p[4], p[5], ld2,
              ws.data_ptr(), ws.numel(), L.stream_ptr()), "avc_tc_epi_test")
    torch.cuda.synchronize()
    return A.double() @ B.double().t(), ring()


def _err(got, ref):
    return (got.double() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _stash(M, N, ldx, g, lo=0.0, hi=1.0):
    """[M][ldx] fp32 stash with zero padding (columns >= N), like the sp' / qt / zbar stashes of the NeuS path."""
    x = torch.zeros(M, ldx)
    x[:, :N] = lo + (hi - lo) * torch.rand(M, N, generator=g)
    return x.cuda()


def _split_value(x):
    hi = x.bfloat16()
    lo = (x - hi.float()).bfloat16()
    return hi.double() + lo.double()


def _nan(M, cols):
    return torch.full((M + EXTRA, cols), float("nan"), device="cuda")


def _sentinel_split(M, ld2):
    """[M + EXTRA][ld2] fp32 buffer holding bf16 pairs (hi in columns [0, ld2), lo in [ld2, 2 ld2)): known values."""
    pat = (torch.arange((M + EXTRA) * 2 * ld2, dtype=torch.float32) % 97 - 48.0).bfloat16()
    return pat.view(torch.float32).reshape(M + EXTRA, ld2).cuda()


def _check_split(S, before, M, N, ext, ld2, ref):
    """The split in S: hi + lo = ref in columns < N, zeros in [N, ext), everything else as it was."""
    h16, b16 = S.view(torch.bfloat16), before.view(torch.bfloat16)
    hi, lo = h16[:M, :ld2], h16[:M, ld2:]
    e = _err(hi[:, :N].double() + lo[:, :N].double(), ref)
    assert e < BAR, e
    assert torch.all(hi[:, N:ext] == 0) and torch.all(lo[:, N:ext] == 0)
    mask = torch.ones_like(h16, dtype=torch.bool)
    mask[:M, :ext] = False
    mask[:M, ld2:ld2 + ext] = False
    assert torch.equal(h16[mask].view(torch.int16), b16[mask].view(torch.int16))
    return e


def _check_f32(OUT, M, N, ref):
    """fp32 output of the padded width: ref in columns < N, zero padding, rows >= M untouched (NaN)."""
    e = _err(OUT[:M, :N], ref)
    assert e < BAR, e
    assert torch.all(OUT[:M, N:] == 0)
    assert torch.isnan(OUT[M:]).all()
    return e


SHAPES = [(1000, 217, 256), (300, 64, 39), (4133, 256, 256), (129, 39, 256), (513, 128, 39)]


def _chain_bwd_inputs(M, N, ldx):
    g = torch.Generator().manual_seed(1)
    return _stash(M, N, ldx, g), _stash(M, N, ldx, g, -1.0, 1.0)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_chain_bwd_split(M, N, K):
    """zbar and the split of ubar_next (a hidden layer of the sweep); at N = 217 into a 256-wide skip input."""
    ldx = r8(N)
    ld2 = 256 if N == 217 else ldx
    D1, QT = _chain_bwd_inputs(M, N, ldx)
    Z, U16 = _nan(M, ldx), _sentinel_split(M, ld2)
    before = U16.clone()
    s = math.sqrt(0.5)
    acc, ring = _run(12, M, N, K, ldx, D1, QT, s=s, OUT=Z, OUT2=U16, ld2=ld2)
    assert ring == 1
    d = D1.double()[:, :N]
    ez = _check_f32(Z, M, N, BETA * (1.0 - d) * _split_value(QT)[:, :N] * acc)
    eu = _check_split(U16, before, M, N, ldx, ld2, d * acc * s)
    print(M, N, K, "zbar", ez, "ubar split", eu)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_chain_bwd_f32(M, N, K):
    """zbar and the fp32 copy of ubar_next (the last linear of the sweep): the copy is stored in two 8-column boxes."""
    ldx = r8(N)
    D1, QT = _chain_bwd_inputs(M, N, ldx)
    Z, U = _nan(M, ldx), _nan(M, ldx)
    s = math.sqrt(0.5)
    acc, ring = _run(0, M, N, K, ldx, D1, QT, s=s, OUT=Z, OUT2=U, ld2=ldx)
    assert ring == 1
    d = D1.double()[:, :N]
    ez = _check_f32(Z, M, N, BETA * (1.0 - d) * _split_value(QT)[:, :N] * acc)
    eu = _check_f32(U, M, N, d * acc * s)
    print(M, N, K, "zbar", ez, "ubar", eu)


def _dgrad_inputs(M, N, ldx, sdf):
    g = torch.Generator().manual_seed(2)
    D1 = _stash(M, N, ldx, g)
    ZB = torch.full((M + EXTRA, ldx), 7.0)          # rows >= M: sentinels
    ZB[:M] = 0.0
    ZB[:M, :N] = -1.0 + 2.0 * torch.rand(M, N, generator=g)
    sdfbar = torch.randn(M, generator=g).cuda() if sdf else None
    wsdf = torch.zeros(ldx)
    wsdf[:N] = torch.randn(N, generator=g)
    return D1, ZB.cuda(), sdfbar, wsdf.cuda() if sdf else None


def _dgrad_ref(D1, ZB, acc, sdfbar, wsdf, M, N, s, inv):
    ab = acc + (sdfbar.double()[:, None] * inv * wsdf.double()[None, :N] if sdfbar is not None else 0.0)
    return D1.double()[:, :N] * ab * s + ZB.double()[:M, :N]


@pytest.mark.parametrize("sdf", [False, True])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dgrad_split(M, N, K, sdf):
    """The split of the new zbar_prev only (the renderer's value backward); zbar_prev itself is only read."""
    ldx = r8(N)
    D1, ZB, sdfbar, wsdf = _dgrad_inputs(M, N, ldx, sdf)
    zb0 = ZB.clone()
    Z16 = _sentinel_split(M, ldx)
    before = Z16.clone()
    s, inv = 0.5, 1.0 / 3.0
    acc, ring = _run(14 if sdf else 13, M, N, K, ldx, D1, ZB, v1=sdfbar, v2=wsdf, s=s, s2=inv, OUT=_nan(M, 8),
                     OUT2=Z16, ld2=ldx)
    assert ring == 1
    e = _check_split(Z16, before, M, N, ldx, ldx, _dgrad_ref(D1, zb0, acc, sdfbar, wsdf, M, N, s, inv))
    assert torch.equal(ZB, zb0)
    print(M, N, K, sdf, "zbar_prev split", e)


@pytest.mark.parametrize("sdf", [False, True])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dgrad_in_place(M, N, K, sdf):
    """The fp32 zbar_prev, updated in place: its padding stays zero and its rows >= M keep their sentinels."""
    ldx = r8(N)
    D1, ZB, sdfbar, wsdf = _dgrad_inputs(M, N, ldx, sdf)
    zb0 = ZB.clone()
    s, inv = 0.5, 1.0 / 3.0
    acc, ring = _run(2 if sdf else 1, M, N, K, ldx, D1, ZB, v1=sdfbar, v2=wsdf, s=s, s2=inv)
    assert ring == 1
    e = _err(ZB[:M, :N], _dgrad_ref(D1, zb0, acc, sdfbar, wsdf, M, N, s, inv))
    print(M, N, K, sdf, "zbar_prev", e)
    assert e < BAR
    assert torch.all(ZB[:M, N:] == 0)
    assert torch.equal(ZB[M:], zb0[M:])


# (M, Nv, E, K): E > 0 is the chain into a skip layer, whose columns >= Nv accumulate into ge
CHAIN_SHAPES = [(1000, 217, 39, 256), (300, 64, 0, 39), (4133, 256, 0, 256), (129, 25, 39, 39)]


def _chain_inputs(M, Nv, E):
    ldx = max(r8(Nv), r8(E))
    g = torch.Generator().manual_seed(3)
    return ldx, _stash(M, Nv, ldx, g), torch.randn(M + EXTRA, ldx, generator=g).cuda()


@pytest.mark.parametrize("M,Nv,E,K", CHAIN_SHAPES)
def test_chain_split(M, Nv, E, K):
    """The split of qt_prev only (the renderer's gradient chain), with the ge columns accumulated by red.global."""
    ldx, D1, GE = _chain_inputs(M, Nv, E)
    ge0 = GE.clone()
    Q16 = _sentinel_split(M, ldx)
    before = Q16.clone()
    s = math.sqrt(0.5)
    acc, ring = _run(15, M, Nv + E, K, ldx, D1, s=s, OUT=GE, OUT2=Q16, ld2=ldx, Nv=Nv)
    assert ring == 1
    eq = _check_split(Q16, before, M, Nv, ldx, ldx, D1.double()[:, :Nv] * acc[:, :Nv] * s)
    print(M, Nv, E, K, "qt_prev split", eq)
    if E:
        ege = _err(GE[:M, :E], ge0[:M, :E].double() + acc[:, Nv:] * math.sqrt(0.5))
        print("ge", ege)
        assert ege < BAR
    assert torch.equal(GE[:M, E:], ge0[:M, E:]) and torch.equal(GE[M:], ge0[M:])


@pytest.mark.parametrize("M,Nv,E,K", CHAIN_SHAPES)
def test_chain_f32(M, Nv, E, K):
    """The fp32 qt_prev of the padded width (zero padding), rows >= M untouched."""
    ldx, D1, GE = _chain_inputs(M, Nv, E)
    ge0 = GE.clone()
    Q = _nan(M, ldx)
    s = math.sqrt(0.5)
    acc, ring = _run(3, M, Nv + E, K, ldx, D1, s=s, OUT=Q, OUT2=GE, ld2=ldx, Nv=Nv)
    assert ring == 1
    eq = _check_f32(Q, M, Nv, D1.double()[:, :Nv] * acc[:, :Nv] * s)
    print(M, Nv, E, K, "qt_prev", eq)
    if E:
        assert _err(GE[:M, :E], ge0[:M, :E].double() + acc[:, Nv:] * math.sqrt(0.5)) < BAR
    assert torch.equal(GE[M:], ge0[M:])
