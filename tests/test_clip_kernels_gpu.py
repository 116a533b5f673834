"""Every kernel of the CLIP towers (avc_clip.cu) on its own inputs against its float64 reference (oracle/clip_kernels.py,
pinned against torch by test_clip_kernels_cpu.py), through avc_clip_kernel_test: the host code the towers use.

End-to-end parity cannot see a kernel error below ~1e-4 of the embedding (the fp32 / fp16 rounding floor), so each
kernel is checked here at the shapes where it can go wrong: both GEMM paths (M <= 128 wgmma, M > 128 mma.sync) with full
and ragged tiles and short last K splits, LayerNorm at its register-cache limit, the uncached row-scale branch, token
counts from 1 to the kernels' limits, non-square and extreme canvases, head widths that are not a multiple of 64.

fp32 outputs meet rel-to-max bars.  fp16 outputs must lie in [fp16(ref - delta), fp16(ref + delta)], delta a bound of
that stage's fp32 error: with delta under half an fp16 step, fp16(ref) or, within delta of the rounding midpoint, the
other neighbour.  Every output buffer has a NaN-patterned tail of at least one row (and rows the kernel must not write
keep their contents), checked bit for bit afterwards."""
import ctypes as C

import numpy as np
import pytest
import torch

import util_neus as U
from oracle import clip_kernels as ck

pytestmark = pytest.mark.gpu

GUARD = 256                  # at least; every guard also spans one full row of its buffer
NAN32, NAN16 = 0x7FC0DEAD, 0x7E55
# rel-to-max bars of the fp32 outputs: at most 4x the worst value of two full runs on an H100 80GB HBM3 (400 W limit)
BAR_GEMM = 5.5e-6           # measured 1.43e-6: fp32 accumulation over K <= 3072
BAR_LN = 6.5e-5             # 1.68e-5: the fp32 mean of rows at 1e3
BAR_LN_BWD = 3.9e-5         # 9.9e-6
BAR_ATT_BWD = 1e-3          # 2.56e-4: tf32 rounding of P and dS lands on the other side for a few entries
BAR_PRE_BWD = 5.5e-5        # 1.46e-5: the 1 x 1 canvas sums all 3 x 224^2 taps in fp32 atomics
BAR_HEAD = 2e-6             # 5.43e-7

_F = None


def _fn():
    global _F
    if _F is None:
        from avatarclip_b200 import _lib
        f = _lib.lib().avc_clip_kernel_test
        f.argtypes = [C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p]
        f.restype = C.c_int
        _F = (_lib, f)
    return _F


def _run(kind, dims, ins, outs):
    _lib, f = _fn()
    d = (C.c_int32 * len(dims))(*dims)
    pi = (C.c_void_p * len(ins))(*[None if t is None else t.data_ptr() for t in ins])
    po = (C.c_void_p * len(outs))(*[None if t is None else t.data_ptr() for t in outs])
    _lib.check(f(kind, d, pi, po, _lib.stream_ptr()), f"avc_clip_kernel_test({kind})")
    torch.cuda.synchronize()


class Out:
    """Device output buffer of `shape` followed by a NaN-patterned guard of at least one row (so a write to any column
    of row M lands in it); `init` fills the output part."""

    def __init__(self, shape, dtype=torch.float32, init=None):
        n = int(np.prod(shape))
        guard = max(GUARD, shape[-1])
        it = torch.int32 if dtype == torch.float32 else torch.int16
        self.full = torch.full((n + guard,), NAN32 if dtype == torch.float32 else NAN16, dtype=it,
                               device="cuda").view(dtype)
        self.t = self.full[:n].view(shape)
        if init is not None:
            self.t.copy_(init)
        self.n, self.it = n, it

    def intact(self):
        tail = self.full[self.n:].view(self.it).cpu()
        return bool(torch.all(tail == (NAN32 if self.it == torch.int32 else NAN16)))


def _rel(got, ref):
    return U.rel_to_max(got, ref)


def _faithful16(got, ref, delta):
    """(bad, off): outputs outside [fp16(ref - delta), fp16(ref + delta)], and outputs other than fp16(ref).  With delta
    under half an fp16 step this allows the other neighbour only where ref lies within delta of the midpoint."""
    g = got.detach().cpu().double()
    r, d = ref.detach().double().cpu(), delta.detach().double().cpu()
    lo, hi = ck.fp16(r - d), ck.fp16(r + d)
    bad = (g < lo) | (g > hi)
    if bad.any():
        i = int(torch.nonzero(bad.flatten())[0])
        print("fp16 mismatch: ref %.9g got %.9g delta %.3g" % (r.flatten()[i], g.flatten()[i],
                                                             d.expand_as(r).flatten()[i]))
    return int(bad.sum()), int((g != ck.fp16(r)).sum())


def _h(t):
    return t.half().cuda()


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------ GEMMs
M_ALL = [1, 50, 77, 100, 127, 128, 129, 150, 231]


def _operands(M, N, K, g):
    A = torch.randn(M, K, generator=g).half()
    Wt = (torch.randn(N, K, generator=g) * K ** -0.5).half()
    return A, Wt


# (N, K, ksplit) of the towers: image qkv / c_fc / input-gradient of out_proj and the patch embedding, text qkv / c_fc
@pytest.mark.parametrize("N,K,ks", [(2304, 768, 1), (1536, 512, 1), (768, 768, 1), (3072, 768, 1)])
@pytest.mark.parametrize("M", M_ALL)
def test_gemm_bias_store_and_store_unscale(M, N, K, ks):
    g = _gen(M * 7 + N)
    A, Wt = _operands(M, N, K, g)
    acc = ck.gemm(A, Wt)
    bias = torch.randn(N, generator=g)
    out = Out((M, N))
    _run(0, [M, N, K, ks], [_h(A), _h(Wt), bias.cuda()], [out.t])
    e0 = _rel(out.t, acc + bias.double())
    sc = torch.ldexp(torch.ones(M), torch.randint(-20, 20, (M,), generator=g))
    out2 = Out((M, N))
    _run(5, [M, N, K, ks], [_h(A), _h(Wt), sc.cuda()], [out2.t])
    e5 = _rel(out2.t, acc / sc.double()[:, None])
    U.log_parity("clip_kernel_gemm_store", {"M": M, "N": N, "K": K, "bias_store": e0, "store_unscale": e5})
    assert e0 < BAR_GEMM and e5 < BAR_GEMM and out.intact() and out2.intact()


# split-K accumulators: out_proj / c_proj (image and text), the input-gradients through c_fc and qkv, and K = 320 in
# 4 requested splits, which runs as 3 splits of 128, 128 and 64
@pytest.mark.parametrize("N,K,ks", [(768, 768, 2), (768, 3072, 4), (512, 512, 2), (512, 2048, 4), (768, 2304, 3),
                                    (64, 320, 4)])
@pytest.mark.parametrize("M", M_ALL)
def test_gemm_residual_and_accum_unscale(M, N, K, ks):
    g = _gen(M * 11 + K)
    A, Wt = _operands(M, N, K, g)
    acc = ck.gemm(A, Wt)
    bias = torch.randn(N, generator=g) * 4           # added once over the splits: a per-split bias would show
    x0 = torch.randn(M, N, generator=g)
    out = Out((M, N), init=x0)
    _run(1, [M, N, K, ks], [_h(A), _h(Wt), bias.cuda()], [out.t])
    e1 = _rel(out.t, x0.double() + acc + bias.double())
    sc = torch.ldexp(torch.ones(M), torch.randint(-20, 20, (M,), generator=g))
    out4 = Out((M, N), init=x0)
    _run(4, [M, N, K, ks], [_h(A), _h(Wt), sc.cuda()], [out4.t])
    e4 = _rel(out4.t, x0.double() + acc / sc.double()[:, None])
    U.log_parity("clip_kernel_gemm_accum", {"M": M, "N": N, "K": K, "ks": ks, "residual": e1, "accum_unscale": e4})
    assert e1 < BAR_GEMM and e4 < BAR_GEMM and out.intact() and out4.intact()


@pytest.mark.parametrize("N,K", [(3072, 768), (2048, 512)])
@pytest.mark.parametrize("M", M_ALL)
def test_gemm_fc_and_dfc(M, N, K):
    g = _gen(M * 13 + N)
    A, Wt = _operands(M, N, K, g)
    acc = ck.gemm(A, Wt)
    bias = torch.randn(N, generator=g) * 0.5
    pre, g16 = Out((M, N)), Out((M, N), torch.float16)
    _run(2, [M, N, K, 1], [_h(A), _h(Wt), bias.cuda()], [pre.t, g16.t])
    epre = _rel(pre.t, acc + bias.double())
    p32 = pre.t.double().cpu()          # the activation is checked on the kernel's own fp32 pre-activation
    gref = ck.quick_gelu(p32)
    bad_fc, m_fc = _faithful16(g16.t, gref, 2.0 ** -20 * (gref.abs() + p32.abs()))
    # EpiDfc: the incoming gradient times QuickGELU'(pre) of a given fp32 pre-activation
    pin = torch.randn(M, N, generator=g) * 2
    d16 = Out((M, N), torch.float16)
    _run(3, [M, N, K, 1], [_h(A), _h(Wt), pin.cuda()], [None, d16.t])
    dq = ck.quick_gelu_grad(pin.double())
    dref = acc * dq
    bad_dfc, m_dfc = _faithful16(d16.t, dref, dq.abs() * ck.gemm_delta(A, Wt) + acc.abs() * ck.quick_gelu_grad_err(pin))
    U.log_parity("clip_kernel_gemm_fc", {"M": M, "N": N, "K": K, "pre": epre, "g16_bad": bad_fc, "dfc16_bad": bad_dfc,
                                         "g16_off": m_fc, "dfc16_off": m_dfc})
    assert epre < BAR_GEMM and bad_fc == 0 and bad_dfc == 0
    assert pre.intact() and g16.intact() and d16.intact()


# patch embedding: np = 49 patches per image (ViT-B/32 at 224) and np = 16 (image 64, patch 16, width 128)
@pytest.mark.parametrize("B,np_,N,K", [(1, 49, 768, 3072), (2, 49, 768, 3072), (3, 49, 768, 3072), (7, 16, 128, 768),
                                       (8, 16, 128, 768), (9, 16, 128, 768)])
def test_gemm_patch_embedding_leaves_cls_rows_untouched(B, np_, N, K):
    g = _gen(B * np_)
    M, T = B * np_, np_ + 1
    A, Wt = _operands(M, N, K, g)
    acc = ck.gemm(A, Wt)
    x0 = torch.randn(B * T, N, generator=g)
    x = Out((B * T, N), init=x0)
    _run(6, [M, N, K, 4, np_], [_h(A), _h(Wt), None], [x.t])
    want = x0.double().clone()
    idx = torch.tensor([b * T + 1 + p for b in range(B) for p in range(np_)])
    want[idx] += acc
    e = _rel(x.t, want)
    cls = torch.arange(B) * T
    U.log_parity("clip_kernel_gemm_patch", {"B": B, "np": np_, "err": e})
    assert e < BAR_GEMM and x.intact()
    assert torch.equal(x.t.cpu()[cls].view(torch.int32), x0[cls].view(torch.int32))


# ------------------------------------------------------------------------------------------------------- LayerNorm
def _ln_inputs(M, Wd, g):
    x = torch.randn(M, Wd, generator=g) * (1 + torch.rand(M, 1, generator=g) * 3)
    x[::3] += 1e3                                      # a one-pass variance loses these rows
    gam = 1 + 0.1 * torch.randn(Wd, generator=g)
    bet = 0.1 * torch.randn(Wd, generator=g)
    return x, gam, bet


@pytest.mark.parametrize("Wd", [64, 512, 768, 832, 1024])
@pytest.mark.parametrize("M", [1, 101])
def test_layernorm(M, Wd):
    g = _gen(M + Wd)
    x, gam, bet = _ln_inputs(M, Wd, g)
    y32, y16, sx = Out((M, Wd)), Out((M, Wd), torch.float16), Out((M, Wd))
    _run(7, [M, Wd], [x.cuda(), gam.cuda(), bet.cuda()], [y32.t, y16.t, sx.t])
    e = _rel(y32.t, ck.layernorm(x, gam, bet))
    assert torch.equal(y16.t.cpu(), y32.t.cpu().half())
    assert torch.equal(sx.t.cpu().view(torch.int32), x.view(torch.int32))
    only16 = Out((M, Wd), torch.float16)
    _run(7, [M, Wd], [x.cuda(), gam.cuda(), bet.cuda()], [None, only16.t, None])
    assert torch.equal(only16.t.cpu().view(torch.int16), y16.t.cpu().view(torch.int16))
    U.log_parity("clip_kernel_layernorm", {"M": M, "Wd": Wd, "err": e})
    assert e < BAR_LN and y32.intact() and y16.intact() and sx.intact() and only16.intact()


@pytest.mark.parametrize("Wd", [64, 512, 768, 832, 1024])
@pytest.mark.parametrize("M", [1, 101])
def test_layernorm_backward(M, Wd):
    g = _gen(M * 3 + Wd)
    x, gam, _ = _ln_inputs(M, Wd, g)
    dy = torch.randn(M, Wd, generator=g)
    dx0 = torch.randn(M, Wd, generator=g)
    # accumulate into dx, clear dy, row-scaled fp16 copy: the form the towers' backward uses
    dyb, dx, d16, sc = Out((M, Wd), init=dy), Out((M, Wd), init=dx0), Out((M, Wd), torch.float16), Out((M,))
    _run(8, [M, Wd, 1, 1], [x.cuda(), gam.cuda()], [dyb.t, dx.t, d16.t, sc.t])
    e_acc = _rel(dx.t, ck.layernorm_bwd(x, dy, gam, dx0))
    assert torch.all(dyb.t == 0)
    dxk = dx.t.double().cpu()
    want16, want_sc = ck.to_half_rowscaled(dxk)
    assert torch.equal(sc.t.double().cpu(), want_sc)
    assert torch.equal(d16.t.double().cpu(), want16)
    # plain: dx overwritten, dy kept, no fp16 copy
    dyb2, dx2 = Out((M, Wd), init=dy), Out((M, Wd), init=dx0)
    _run(8, [M, Wd, 0, 0], [x.cuda(), gam.cuda()], [dyb2.t, dx2.t, None, None])
    e = _rel(dx2.t, ck.layernorm_bwd(x, dy, gam))
    assert torch.equal(dyb2.t.cpu().view(torch.int32), dy.view(torch.int32))
    U.log_parity("clip_kernel_layernorm_bwd", {"M": M, "Wd": Wd, "err": e, "err_accumulate": e_acc})
    assert e < BAR_LN_BWD and e_acc < BAR_LN_BWD
    assert all(o.intact() for o in (dyb, dx, d16, sc, dyb2, dx2))


# width 768 / 3 x 768 = 2304 (the register-cached limit) / 3 x 832 = 2496 and 3 x 1024 = 3072 (uncached)
@pytest.mark.parametrize("N", [64, 768, 2304, 2496, 3072])
def test_to_half_rowscaled(N):
    g = _gen(N)
    M = 101
    src = torch.randn(M, N, generator=g) * torch.ldexp(torch.ones(M, 1), torch.randint(-30, 30, (M, 1), generator=g))
    src[3] = 0
    src[4] = torch.randn(N, generator=g) * 1e-30
    src[5] = torch.randn(N, generator=g) * 1e30
    dst, sc = Out((M, N), torch.float16), Out((M,))
    _run(9, [M, N, N], [src.cuda(), None], [dst.t, sc.t])
    want16, want_sc = ck.to_half_rowscaled(src)
    assert torch.equal(sc.t.double().cpu(), want_sc)
    assert torch.equal(dst.t.double().cpu(), want16)
    assert dst.intact() and sc.intact()


def test_to_half_rowscaled_gathers_the_patch_rows():
    """The patch-gradient form: rows b*T + 1 + p of the token gradient, T = 50."""
    g = _gen(5)
    B, T, Wd = 3, 50, 768
    src = torch.randn(B * T, Wd, generator=g)
    rm = torch.tensor([b * T + 1 + p for b in range(B) for p in range(T - 1)], dtype=torch.int32)
    M = rm.numel()
    dst, sc = Out((M, Wd), torch.float16), Out((M,))
    _run(9, [M, Wd, Wd], [src.cuda(), rm.cuda()], [dst.t, sc.t])
    want16, want_sc = ck.to_half_rowscaled(src, rm)
    assert torch.equal(sc.t.double().cpu(), want_sc) and torch.equal(dst.t.double().cpu(), want16)
    assert dst.intact() and sc.intact()


# ------------------------------------------------------------------------------------------------------- attention
ATT = [(T, h) for T in (2, 17, 37, 50) for h in (1, 12, 16)]


@pytest.mark.parametrize("T,heads", ATT)
def test_attention(T, heads):
    g = _gen(T * heads)
    B, Wd = 2, 64 * heads
    qkv = torch.randn(B * T, 3 * Wd, generator=g)
    qkv[:, :Wd] *= 1.5                                   # sharper softmax rows
    o16 = Out((B * T, Wd), torch.float16)
    _run(10, [B, T, Wd, heads], [qkv.cuda()], [o16.t])
    ref, delta = ck.attention(qkv, B, T, heads)
    bad, off = _faithful16(o16.t, ref, delta)
    dO = torch.randn(B * T, Wd, generator=g)
    dq = Out((B * T, 3 * Wd))
    _run(11, [B, T, Wd, heads], [qkv.cuda(), dO.cuda()], [dq.t])
    e = _rel(dq.t, ck.attention_bwd(qkv, dO, B, T, heads))
    U.log_parity("clip_kernel_attention", {"T": T, "heads": heads, "o16_bad": bad, "o16_off": off, "bwd": e})
    assert bad == 0 and e < BAR_ATT_BWD and o16.intact() and dq.intact()


@pytest.mark.parametrize("T", [1, 31, 32, 33, 77, 128])
def test_causal_attention(T):
    g = _gen(T)
    B, heads = 2, 8
    Wd = 64 * heads
    qkv = torch.randn(B * T, 3 * Wd, generator=g)
    o16 = Out((B * T, Wd), torch.float16)
    _run(12, [B, T, Wd, heads], [qkv.cuda()], [o16.t])
    ref, delta = ck.causal_attention(qkv, B, T, heads)
    bad, off = _faithful16(o16.t, ref, delta)
    U.log_parity("clip_kernel_causal_attention", {"T": T, "o16_bad": bad, "o16_off": off})
    assert bad == 0 and o16.intact()
    # rows after position a change: rows 0..a of every sequence stay bit for bit
    a = T // 2
    q2 = qkv.clone().view(B, T, -1)
    q2[:, a + 1:] = torch.randn(q2[:, a + 1:].shape, generator=g)
    o2 = Out((B * T, Wd), torch.float16)
    _run(12, [B, T, Wd, heads], [q2.reshape(B * T, -1).cuda()], [o2.t])
    assert torch.equal(o2.t.view(B, T, Wd)[:, :a + 1].cpu().view(torch.int16),
                       o16.t.view(B, T, Wd)[:, :a + 1].cpu().view(torch.int16))


# --------------------------------------------------------------------------------------------------- preprocessing
CANVASES = [(224, 224, 2), (160, 160, 2), (256, 256, 2), (97, 300, 2), (1, 1, 2), (2000, 2000, 1)]


@pytest.mark.parametrize("H,W,B", CANVASES)
def test_preprocess_and_backward(H, W, B):
    g = _gen(H * W)
    IS, P = 224, 32
    canvas = torch.rand(B, H, W, 3, generator=g)
    ng = (IS // P) ** 2
    a0 = Out((B * ng, 3 * P * P), torch.float16)
    _run(13, [H, W, B, IS, P, 0], [canvas.cuda()], [a0.t])
    ref = ck.preprocess(canvas, IS, P, f32=True)
    # one fp32 step of each source position (fused or separate rounding), fp32 arithmetic on values of size ~4
    sy = torch.tensor([(y + 0.5) * H / IS for y in range(IS)], dtype=torch.float64)
    sx = torch.tensor([(x + 0.5) * W / IS for x in range(IS)], dtype=torch.float64)
    eps = 2.0 ** -23 * (sy[:, None] + sx[None, :] + 2) / 0.26
    delta = ck.im2col(eps.expand(B, 3, IS, IS), P) + 2.0 ** -20 * (ref.abs() + 4)
    bad, off = _faithful16(a0.t, ref, delta)
    dpatch = torch.randn(B * ng, 3 * P * P, generator=g)
    dc = Out((B, H, W, 3), init=torch.full((B, H, W, 3), 7.0))
    _run(14, [H, W, B, IS, P, 0], [dpatch.cuda()], [dc.t])
    want = ck.preprocess_bwd(dpatch, B, H, W, IS, P, f32=True)
    e = _rel(dc.t, want)
    Ry, Rx = ck.resize_matrix(H, IS, True), ck.resize_matrix(W, IS, True)
    unreached = ((Ry.sum(0) == 0)[:, None] | (Rx.sum(0) == 0)[None, :])
    assert torch.all(dc.t.cpu()[:, unreached] == 0)
    U.log_parity("clip_kernel_preprocess", {"H": H, "W": W, "a0_bad": bad, "a0_off": off, "bwd": e, "unreached": int(unreached.sum())})
    assert bad == 0 and e < BAR_PRE_BWD and a0.intact() and dc.intact()


def test_preprocess_mode1_is_a_plain_im2col():
    g = _gen(11)
    B, IS, P = 3, 224, 32
    img = torch.randn(B, 3, IS, IS, generator=g)
    ng = (IS // P) ** 2
    a0 = Out((B * ng, 3 * P * P), torch.float16)
    _run(13, [IS, IS, B, IS, P, 1], [img.cuda()], [a0.t])
    assert torch.equal(a0.t.cpu().view(torch.int16), ck.im2col(img, P).half().view(torch.int16))
    dpatch = torch.randn(B * ng, 3 * P * P, generator=g)
    dc = Out((B, 3, IS, IS))
    _run(14, [IS, IS, B, IS, P, 1], [dpatch.cuda()], [dc.t])
    assert torch.equal(dc.t.cpu().view(torch.int32), ck.col2im(dpatch, B, IS, P).contiguous().view(torch.int32))
    assert a0.intact() and dc.intact()


# ------------------------------------------------------------------------------------------------------------ head
@pytest.mark.parametrize("OD", [1, 64, 100, 512])
@pytest.mark.parametrize("B,T,Wd", [(2, 50, 768), (3, 1, 512)])
def test_head(B, T, Wd, OD):
    g = _gen(OD * 5 + T)
    x = torch.randn(B * T, Wd, generator=g) + 3
    gam, bet = 1 + 0.1 * torch.randn(Wd, generator=g), 0.1 * torch.randn(Wd, generator=g)
    proj = torch.randn(Wd, OD, generator=g) * Wd ** -0.5
    emb, yn = Out((B, OD)), Out((B, Wd))
    _run(15, [B, T, Wd, OD], [x.cuda(), gam.cuda(), bet.cuda(), proj.cuda()], [emb.t, yn.t])
    e_ref, y_ref = ck.head_proj(x, B, T, gam, bet, proj)
    errs = {"emb": _rel(emb.t, e_ref), "ynorm": _rel(yn.t, y_ref)}
    embk = emb.t.cpu()
    text = torch.randn(B, OD, generator=g)
    text[1] = 0                                          # zero text vector: no cosine gradient, cos 0
    cos = Out((B,))
    _run(16, [B, OD], [emb.t, text.cuda()], [cos.t])
    errs["cos"] = (cos.t.double().cpu() - ck.cosine(embk, text)).abs().max().item()
    g_cos, g_emb = torch.randn(B, generator=g), torch.randn(B, OD, generator=g)
    dx_x = None
    for name, gc, ge in (("g_cos", g_cos, None), ("g_emb", None, g_emb), ("both", g_cos, g_emb)):
        dy = Out((B, Wd))
        _run(17, [B, Wd, OD], [proj.cuda(), text.cuda(), emb.t, None if gc is None else gc.cuda(),
                               None if ge is None else ge.cuda()], [dy.t])
        want = ck.head_bwd_dy(proj, text, embk, gc, ge)
        # the size of the cosine term's parts, which cancel exactly when out_dim = 1
        parts = 0.0 if gc is None else (gc.abs() / embk.norm(dim=-1)).max().item() * proj.abs().sum(1).max().item()
        errs["dy_" + name] = (dy.t.double().cpu() - want).abs().max().item() / max(want.abs().max().item(), parts)
        dx = Out((B * T, Wd), init=torch.full((B * T, Wd), 5.0))
        _run(18, [B, T, Wd], [x.cuda(), gam.cuda(), dy.t], [dx.t])
        errs["dx_" + name] = _rel(dx.t, ck.head_bwd_ln(x, B, T, gam, dy.t.cpu()))
        rows = dx.t.view(B, T, Wd)[:, 1:]
        assert torch.all(rows == 0) and dy.intact() and dx.intact()
    U.log_parity("clip_kernel_head", {"B": B, "T": T, "Wd": Wd, "OD": OD, **errs})
    assert all(v < BAR_HEAD for v in errs.values()), errs
    assert emb.intact() and yn.intact() and cos.intact()


# ---------------------------------------------------------------------------------------------- end-of-text rows
@pytest.mark.parametrize("T", [1, 77, 128])
def test_text_eot_rows(T):
    g = _gen(T)
    B, Wd = 5, 512
    tok = torch.randint(0, 1000, (B, T), generator=g, dtype=torch.int32)
    tok[0, 0] = 5000                                     # maximum at position 0
    tok[1, T - 1] = 5000                                 # at T - 1
    tok[2, T // 3] = tok[2, (2 * T) // 3] = 5000         # a tie: the first one
    tok[3, :] = 7                                        # all equal: position 0
    x = torch.randn(B * T, Wd, generator=g)
    eot = Out((B, Wd))
    _run(19, [B, T, Wd], [tok.cuda(), x.cuda()], [eot.t])
    want = ck.text_eot_rows(tok, x, B, T).float()
    assert torch.equal(eot.t.cpu().view(torch.int32), want.view(torch.int32)) and eot.intact()
