"""The backward epilogue functors (second-order sweep, value backward, gradient chain, ReLU-mask dgrad, encoding-gradient
accumulation) through the wgmma NT tiles against an fp64 restatement of their formulas: ragged row counts, the padded
skip-layer width (N = 217 in a 224-wide stash), single 64-wide column tiles, K = 39 and K = 256."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BETA = 100.0
BAR = 3e-5


def r8(n):
    return (n + 7) // 8 * 8


def _lib_fn():
    from avatarclip_b200 import _lib
    L = _lib.lib()
    f = L.avc_tc_epi_test
    vp, i32 = C.c_void_p, C.c_int32
    f.argtypes = [i32, vp, vp, C.c_int64, i32, i32, i32, vp, vp, i32, vp, vp, C.c_float, C.c_float, vp, vp, i32, vp,
                  C.c_size_t, vp]
    f.restype = C.c_int
    return _lib, f


def _ptr(t):
    return None if t is None else t.data_ptr()


def _run(kind, M, N, K, ldx, X, Y=None, v1=None, v2=None, s=1.0, s2=1.0, OUT=None, OUT2=None, ld2=8, Nv=0, seed=0):
    _lib, f = _lib_fn()
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).cuda()
    B = (torch.randn(N, K, generator=g) * 0.1).cuda()
    ws = torch.empty(4 * (M + N) * r8(K) + 4 * M * ldx + 8192, dtype=torch.uint8, device="cuda")
    _lib.check(f(kind, A.data_ptr(), B.data_ptr(), M, N, K, Nv, _ptr(X), _ptr(Y), ldx, _ptr(v1), _ptr(v2), s, s2,
                 _ptr(OUT), _ptr(OUT2), ld2, ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "avc_tc_epi_test")
    torch.cuda.synchronize()
    return A.double() @ B.double().t()       # the fp64 accumulator


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


SHAPES = [(1000, 217, 256), (300, 64, 39), (4133, 256, 256), (129, 39, 256), (513, 128, 39)]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_chain_bwd(M, N, K):
    ldx = r8(N)
    g = torch.Generator().manual_seed(1)
    D1, QT = _stash(M, N, ldx, g), _stash(M, N, ldx, g, -1.0, 1.0)
    Z = torch.full((M, ldx), float("nan"), device="cuda")
    U = torch.full((M, ldx), float("nan"), device="cuda")
    s = math.sqrt(0.5)
    acc = _run(0, M, N, K, ldx, D1, QT, s=s, OUT=Z, OUT2=U, ld2=ldx)
    d = D1.double()[:, :N]
    u_ref = d * acc * s
    z_ref = BETA * (1.0 - d) * _split_value(QT)[:, :N] * acc
    eu, ez = _err(U[:, :N], u_ref), _err(Z[:, :N], z_ref)
    print(M, N, K, "ubar", eu, "zbar", ez)
    assert eu < BAR and ez < BAR
    # the padding columns of the last group come out zero (zero stash padding)
    n4 = (N + 3) // 4 * 4
    assert torch.all(Z[:, N:n4] == 0) and torch.all(U[:, N:n4] == 0)


@pytest.mark.parametrize("sdf", [False, True])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dgrad(M, N, K, sdf):
    ldx = r8(N)
    g = torch.Generator().manual_seed(2)
    D1, ZB = _stash(M, N, ldx, g), _stash(M, N, ldx, g, -1.0, 1.0)
    zb0 = ZB.double()[:, :N].clone()
    sdfbar = torch.randn(M, generator=g).cuda() if sdf else None
    wsdf = torch.zeros(ldx)
    wsdf[:N] = torch.randn(N, generator=g)
    wsdf = wsdf.cuda() if sdf else None
    s, inv = 0.5, 1.0 / 3.0
    acc = _run(2 if sdf else 1, M, N, K, ldx, D1, ZB, v1=sdfbar, v2=wsdf, s=s, s2=inv)
    ab = acc + (sdfbar.double()[:, None] * inv * wsdf.double()[None, :N] if sdf else 0.0)
    ref = D1.double()[:, :N] * ab * s + zb0
    e = _err(ZB[:, :N], ref)
    print(M, N, K, sdf, "zbar_prev", e)
    assert e < BAR


@pytest.mark.parametrize("M,Nv,E,K", [(1000, 217, 39, 256), (300, 64, 0, 39), (4133, 256, 0, 256), (129, 25, 39, 39)])
def test_chain(M, Nv, E, K):
    N = Nv + E
    ldx, ld2 = r8(Nv), r8(max(E, 1))
    g = torch.Generator().manual_seed(3)
    D1 = _stash(M, Nv, ldx, g)
    Q = torch.full((M, ldx), float("nan"), device="cuda")
    GE = torch.randn(M, ld2, generator=g).cuda()
    ge0 = GE.double().clone()
    s = math.sqrt(0.5)
    acc = _run(3, M, N, K, ldx, D1, s=s, OUT=Q, OUT2=GE, ld2=ld2, Nv=Nv)
    eq = _err(Q[:, :Nv], D1.double()[:, :Nv] * acc[:, :Nv] * s)
    print(M, Nv, E, K, "qt_prev", eq)
    assert eq < BAR
    assert torch.all(Q[:, Nv:ldx] == 0)          # the padding of qt_prev is zeroed
    if E:
        ege = _err(GE[:, :E], ge0[:, :E] + acc[:, Nv:] * math.sqrt(0.5))
        print("ge", ege)
        assert ege < BAR


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dgrad_relu(M, N, K):
    ldx = r8(N)
    g = torch.Generator().manual_seed(4)
    H = torch.zeros(M, ldx)
    H[:, :N] = torch.relu(torch.randn(M, N, generator=g))
    H = H.cuda()
    OUT = torch.full((M, ldx), float("nan"), device="cuda")
    acc = _run(4, M, N, K, ldx, H, OUT=OUT)
    mask = (H[:, :N].bfloat16() != 0).double()
    e = _err(OUT[:, :N], acc * mask)
    print(M, N, K, "dgrad relu", e)
    assert e < BAR


@pytest.mark.parametrize("M,N,K", [(1000, 39, 256), (300, 64, 39), (129, 39, 39)])
def test_ge(M, N, K):
    ld2 = r8(N)
    g = torch.Generator().manual_seed(5)
    GE = torch.randn(M, ld2, generator=g).cuda()
    ge0 = GE.double().clone()
    X = torch.zeros(M, 8, device="cuda")         # unused by this functor
    acc = _run(5, M, N, K, 8, X, OUT2=GE, ld2=ld2)
    e = _err(GE[:, :N], ge0[:, :N] + acc)
    print(M, N, K, "ge", e)
    assert e < BAR
