"""The float64 references of the CLIP kernels (oracle/clip_kernels.py) against torch in float64 with their deliberate
rounding turned off, and their rounding helpers against hand-written bit patterns.  The GPU tests
(test_clip_kernels_gpu.py) trust these references, so they are pinned here first."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import clip_kernels as ck
from oracle.clip_vit import CLIP_MEAN, CLIP_STD

TOL = 1e-12


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-300)


def _f32(bits):
    return torch.from_numpy(np.array(bits, dtype=np.uint32).view(np.float32).astype(np.float64))


# ------------------------------------------------------------------------------------------------------------ rounding
def test_fp16_rounds_to_nearest_even_from_float64():
    one_ulp = 2.0 ** -10
    x = torch.tensor([1 + one_ulp / 2, 1 + 1.5 * one_ulp, -(1 + one_ulp / 2), 1 + one_ulp / 2 + 2.0 ** -40,
                      65504.0, 65520.0, 2.0 ** -25, 2.0 ** -25 + 2.0 ** -40, 3 * 2.0 ** -25], dtype=torch.float64)
    want = [1.0, 1 + 2 * one_ulp, -1.0, 1 + one_ulp, 65504.0, float("inf"), 0.0, 2.0 ** -24, 2.0 ** -23]
    assert ck.fp16(x).tolist() == want


def test_tf32_keeps_ten_bits_with_ties_away_from_zero():
    # 1 + 2^-11 is the midpoint between 1 and 1 + 2^-10: away from zero.  Just below it: down.
    x = _f32([0x3F801000, 0x3F800FFF, 0xBF801000, 0x3F803000, 0x3F802FFF, 0x7F7FFFFF, 0x00001000])
    got = ck.tf32(x).float().numpy().view(np.uint32).tolist()
    assert got == [0x3F802000, 0x3F800000, 0xBF802000, 0x3F804000, 0x3F802000, 0x7F800000, 0x00002000]


def test_row_scale_is_the_power_of_two_that_puts_the_max_in_1_2():
    mx = torch.tensor([1.0, 1.5, 1.9999999, 2.0, 0.75, 3e-39, 2.0 ** -149, 1e30, 3.4e38, 0.0, float("inf"),
                       float("nan")], dtype=torch.float64)
    sc = ck.row_scale(mx)
    assert sc.tolist() == [1.0, 1.0, 1.0, 0.5, 2.0, 2.0 ** 128, 2.0 ** 149, 2.0 ** -99, 2.0 ** -127, 1.0, 1.0, 1.0]
    fin = mx[:9]
    assert torch.all((fin * sc[:9] >= 1) & (fin * sc[:9] < 2))


def test_to_half_rowscaled_gathers_and_scales_rows():
    g = torch.Generator().manual_seed(0)
    src = torch.randn(5, 12, generator=g, dtype=torch.float64)
    src[1] = 0
    src[2] *= 1e-30
    rm = torch.tensor([4, 2, 1], dtype=torch.int32)
    h, sc = ck.to_half_rowscaled(src, rm)
    assert sc[2].item() == 1.0 and torch.all(h[2] == 0)
    assert torch.equal(h, ck.fp16(src[rm.long()] * sc[:, None]))
    assert torch.all(h.abs().amax(-1)[[0, 1]] < 2) and torch.all(h.abs().amax(-1)[[0, 1]] >= 1)


# ------------------------------------------------------------------------------------------------------ preprocessing
@pytest.mark.parametrize("H,W,IS", [(224, 224, 224), (160, 160, 224), (256, 256, 224), (97, 300, 224), (1, 1, 8),
                                    (500, 37, 64), (7, 5, 16)])
def test_resize_matches_interpolate(H, W, IS):
    g = torch.Generator().manual_seed(H + W)
    c = torch.rand(2, H, W, 3, generator=g, dtype=torch.float64)
    want = F.interpolate(c.permute(0, 3, 1, 2), size=(IS, IS), mode="bilinear", align_corners=False, antialias=False)
    assert _rel(ck.resize(c, IS), want) < TOL
    # adjoint: <R c, g> = <c, R^T g>
    gg = torch.randn(2, 3, IS, IS, generator=g, dtype=torch.float64)
    lhs = (ck.resize(c, IS) * gg).sum()
    rhs = (c * ck.resize_adjoint(gg, H, W)).sum()
    assert abs(lhs - rhs).item() < TOL * abs(lhs).item() + TOL


def test_preprocess_and_its_backward_match_autograd():
    g = torch.Generator().manual_seed(3)
    B, H, W, IS, P = 2, 97, 300, 64, 16
    c = torch.rand(B, H, W, 3, generator=g, dtype=torch.float64, requires_grad=True)
    mean = torch.tensor(CLIP_MEAN, dtype=torch.float32).double().view(1, 3, 1, 1)
    std = torch.tensor(CLIP_STD, dtype=torch.float32).double().view(1, 3, 1, 1)
    img = (F.interpolate(c.permute(0, 3, 1, 2), size=(IS, IS), mode="bilinear", align_corners=False) - mean) / std
    want = F.unfold(img, P, stride=P).transpose(1, 2).reshape(-1, 3 * P * P)
    assert _rel(ck.preprocess(c.detach(), IS, P), want) < TOL
    gp = torch.randn(want.shape, generator=g, dtype=torch.float64)
    (gc,) = torch.autograd.grad((want * gp).sum(), c)
    assert _rel(ck.preprocess_bwd(gp, B, H, W, IS, P), gc) < TOL
    assert torch.equal(ck.col2im(ck.im2col(img.detach(), P), B, IS, P), img.detach())


# --------------------------------------------------------------------------------------------- LayerNorm, attention
@pytest.mark.parametrize("Wd", [64, 768, 1024])
def test_layernorm_and_backward_match_autograd(Wd):
    g = torch.Generator().manual_seed(Wd)
    x = (torch.randn(9, Wd, generator=g, dtype=torch.float64) + 1e3).requires_grad_(True)
    gam, bet = 1 + 0.1 * torch.randn(Wd, generator=g, dtype=torch.float64), torch.randn(Wd, generator=g, dtype=torch.float64)
    y = F.layer_norm(x, (Wd,), gam, bet, 1e-5)
    assert _rel(ck.layernorm(x.detach(), gam, bet), y) < TOL
    dy, dx0 = torch.randn(9, Wd, generator=g, dtype=torch.float64), torch.randn(9, Wd, generator=g, dtype=torch.float64)
    (gx,) = torch.autograd.grad((y * dy).sum(), x)
    assert _rel(ck.layernorm_bwd(x.detach(), dy, gam), gx) < 1e-9       # x ~ 1e3: autograd's own cancellation
    assert _rel(ck.layernorm_bwd(x.detach(), dy, gam, dx0), gx + dx0) < 1e-9


def _qkv_autograd(B, T, heads, causal, g):
    W = 64 * heads
    qkv = torch.randn(B * T, 3 * W, generator=g, dtype=torch.float64, requires_grad=True)
    q, k, v = (t.reshape(B, T, heads, 64).transpose(1, 2) for t in qkv.split(W, 1))
    o = F.scaled_dot_product_attention(q, k, v, is_causal=causal, scale=0.125)
    return qkv, o.transpose(1, 2).reshape(B * T, W)


@pytest.mark.parametrize("B,T,heads", [(2, 2, 1), (1, 17, 12), (3, 50, 2)])
def test_attention_and_backward_match_autograd(B, T, heads):
    g = torch.Generator().manual_seed(T)
    qkv, o = _qkv_autograd(B, T, heads, False, g)
    got, delta = ck.attention(qkv.detach(), B, T, heads, rnd=False)
    assert _rel(got, o) < TOL and torch.all(delta > 0)
    dO = torch.randn(o.shape, generator=g, dtype=torch.float64)
    (gq,) = torch.autograd.grad((o * dO).sum(), qkv)
    assert _rel(ck.attention_bwd(qkv.detach(), dO, B, T, heads, rnd=False), gq) < TOL


@pytest.mark.parametrize("T", [1, 33, 128])
def test_causal_attention_matches_sdpa(T):
    g = torch.Generator().manual_seed(T)
    qkv, o = _qkv_autograd(2, T, 2, True, g)
    got, _ = ck.causal_attention(qkv.detach(), 2, T, 2)
    assert _rel(got, o) < TOL


def test_attention_rounding_moves_the_output_by_tf32_amounts():
    g = torch.Generator().manual_seed(1)
    qkv = torch.randn(50, 3 * 64, generator=g, dtype=torch.float64).float().double()
    o_exact, _ = ck.attention(qkv, 1, 50, 1, rnd=False)
    o_tf32, delta = ck.attention(qkv, 1, 50, 1)
    e = _rel(o_tf32, o_exact)
    assert 1e-5 < e < 3e-3
    assert delta.max().item() < 1e-3 * o_exact.abs().max().item()


# -------------------------------------------------------------------------------------------------------------- head
@pytest.mark.parametrize("zero_text", [False, True])
def test_head_backward_matches_autograd_of_cosine_similarity(zero_text):
    g = torch.Generator().manual_seed(7)
    B, T, Wd, OD = 3, 5, 128, 100
    x = torch.randn(B * T, Wd, generator=g, dtype=torch.float64, requires_grad=True)
    gam, bet = 1 + 0.1 * torch.randn(Wd, generator=g, dtype=torch.float64), torch.randn(Wd, generator=g, dtype=torch.float64)
    proj = torch.randn(Wd, OD, generator=g, dtype=torch.float64) / Wd ** 0.5
    text = torch.randn(B, OD, generator=g, dtype=torch.float64)
    if zero_text:
        text[1] = 0
    y = F.layer_norm(x.reshape(B, T, Wd)[:, 0], (Wd,), gam, bet, 1e-5)
    emb = y @ proj
    cos = torch.cosine_similarity(emb, text, dim=-1)
    e_ref, y_ref = ck.head_proj(x.detach(), B, T, gam, bet, proj)
    assert _rel(e_ref, emb) < TOL and _rel(y_ref, y) < TOL
    assert _rel(ck.cosine(emb.detach(), text), cos) < TOL
    g_cos, g_emb = torch.randn(B, generator=g, dtype=torch.float64), torch.randn(B, OD, generator=g, dtype=torch.float64)
    for gc, ge in ((g_cos, None), (None, g_emb), (g_cos, g_emb)):
        loss = (cos * gc).sum() if gc is not None else 0.0
        loss = loss + ((emb * ge).sum() if ge is not None else 0.0)
        gy, gx = torch.autograd.grad(loss, (y, x), retain_graph=True)
        dy = ck.head_bwd_dy(proj, text, emb.detach(), gc, ge)
        assert _rel(dy, gy) < TOL
        assert _rel(ck.head_bwd_ln(x.detach(), B, T, gam, dy), gx) < TOL


def test_eot_rows_take_the_first_maximum():
    tok = torch.tensor([[5, 9, 9, 1], [9, 1, 2, 3], [1, 2, 3, 9]])
    x = torch.arange(3 * 4 * 2, dtype=torch.float64).reshape(12, 2)
    assert ck.text_eot_rows(tok, x, 3, 4).tolist() == [x[1].tolist(), x[4].tolist(), x[11].tolist()]
