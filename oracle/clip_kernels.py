"""float64 references of the CLIP tower's kernels (avatarclip_b200/csrc/avc_clip.cu), one per kernel, on the inputs the
kernel reads (fp16 operands passed as their exact fp16 values), plus the rounding the kernels apply on purpose:

* ``fp16``: round-to-nearest-even to fp16 (every fp16 operand the kernels write);
* ``tf32``: ``cvt.rna.tf32.f32``, ten mantissa bits with ties away from zero (the attention kernels' q, k, v, P, dO, dS);
* ``row_scale``: the power-of-two scale of ``k_to_half_rowscaled`` / ``k_layernorm_bwd`` that puts max|row| in [1, 2).

Every function takes and returns torch float64 tensors (integer tensors for indices).  ``rnd=False`` turns the
deliberate tf32 rounding off, so that the formulas can be checked against torch autograd."""
from __future__ import annotations

import numpy as np
import torch

from .clip_vit import CLIP_MEAN, CLIP_STD

EPS_LN = 1e-5
ATT_SCALE = 0.125          # 1 / sqrt(64)


# ---------------------------------------------------------------------------------------------------------- rounding
def fp16(x: torch.Tensor) -> torch.Tensor:
    """Round to the nearest fp16, ties to even, straight from float64 (no intermediate fp32 rounding)."""
    with np.errstate(over="ignore"):
        return torch.from_numpy(x.detach().double().cpu().numpy().astype(np.float16).astype(np.float64))


def tf32(x: torch.Tensor) -> torch.Tensor:
    """``cvt.rna.tf32.f32`` of fp32 values: keep ten mantissa bits, round to nearest with ties away from zero."""
    u = x.detach().cpu().float().numpy().view(np.uint32).astype(np.uint64)
    finite = np.isfinite(x.detach().cpu().float().numpy())
    r = np.where(finite, (u + 0x1000) & 0xFFFFE000, u).astype(np.uint32)
    return torch.from_numpy(r.view(np.float32).astype(np.float64))


def tf32_ulp(x: torch.Tensor) -> torch.Tensor:
    """Spacing of the tf32 grid at |x| (2^(e - 10) for |x| in [2^e, 2^(e+1)))."""
    _, e = torch.frexp(x.abs().float().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), (e - 11).to(torch.int64))


def row_scale(mx: torch.Tensor) -> torch.Tensor:
    """2^(1 - e) for mx = m 2^e, m in [0.5, 1): mx * scale lands in [1, 2).  1 for a zero or non-finite max.
    The kernels compute the scale in fp32, where it is finite only for mx >= 2^-127 (e >= -126): a row whose largest
    nonzero magnitude is below that gets an infinite scale.  Tower gradient rows are either exactly zero (scale 1) or
    many orders of magnitude larger, so the kernels are not clamped; this reference keeps the exact power of two."""
    mx = mx.double()
    ok = (mx > 0) & torch.isfinite(mx)
    _, e = torch.frexp(torch.where(ok, mx, torch.ones_like(mx)))
    return torch.where(ok, torch.ldexp(torch.ones_like(mx), (1 - e).to(torch.int64)), torch.ones_like(mx))


# -------------------------------------------------------------------------------------------------------------- GEMM
def gemm(A: torch.Tensor, Wt: torch.Tensor) -> torch.Tensor:
    """acc[M][N] = A[M][K] . Wt[N][K]^T in float64."""
    return A.double() @ Wt.double().t()


def gemm_delta(A: torch.Tensor, Wt: torch.Tensor) -> torch.Tensor:
    """Bound of the fp32 accumulation error of ``gemm``: one rounding of the running sum per 8 of K, over sum |a w|."""
    K = A.shape[1]
    return 2.0 ** -24 * (K / 8 + 16) * (A.double().abs() @ Wt.double().abs().t())


def quick_gelu(p):
    return p * torch.sigmoid(1.702 * p)


def quick_gelu_grad(p):
    s = torch.sigmoid(1.702 * p)
    return s + 1.702 * p * s * (1 - s)


def quick_gelu_grad_err(p):
    """Bound of the fp32 evaluation error of quick_gelu_grad: a few roundings of its two terms, which cancel near
    p = -1.28 (no relative bound there)."""
    p = p.double()
    s = torch.sigmoid(1.702 * p)
    return 2.0 ** -20 * (s + 1.702 * p.abs() * s)


# --------------------------------------------------------------------------------------------------------- LayerNorm
def layernorm(x, g, b):
    x = x.double()
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    return (x - mean) / torch.sqrt(var + EPS_LN) * g.double() + b.double()


def layernorm_bwd(x, dy, g, dx0=None):
    """dx (+ dx0) = LN'(x)^T dy."""
    x, dy, g = x.double(), dy.double(), g.double()
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + EPS_LN)
    xh = (x - mean) * rstd
    dg = dy * g
    dx = rstd * (dg - dg.mean(-1, keepdim=True) - xh * (dg * xh).mean(-1, keepdim=True))
    return dx if dx0 is None else dx + dx0.double()


def to_half_rowscaled(src, row_map=None):
    """(fp16(row * scale), scale) of ``k_to_half_rowscaled``; rows gathered through row_map when given."""
    s = src.double() if row_map is None else src.double()[row_map.long()]
    sc = row_scale(s.abs().amax(-1))
    return fp16(s * sc[:, None]), sc


# --------------------------------------------------------------------------------------------------------- attention
def _heads(t, B, T, heads):
    return t.reshape(B, T, heads, -1).permute(0, 2, 1, 3)        # [B, heads, T, 64]


def _unheads(t):
    B, h, T, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(B * T, h * d)


def attention(qkv, B, T, heads, rnd=True):
    """``k_attention``: o[B*T][W] = softmax(q k^T / 8) v per head, with tf32 q, k, P, v when rnd.  Also returns
    delta, a bound of the kernel's fp32 error per element: accumulation and softmax error plus, for every P entry that
    lies within that error of a tf32 rounding midpoint, one tf32 step of P times |v|."""
    W = qkv.shape[1] // 3
    r = tf32 if rnd else (lambda t: t.double())
    q, k, v = (_heads(r(t), B, T, heads) for t in qkv.double().split(W, dim=1))
    S = q @ k.transpose(-1, -2) * ATT_SCALE
    P = torch.softmax(S, -1)
    Pr = r(P)
    o = _unheads(Pr @ v)
    eS = 2.0 ** -24 * 64 * ATT_SCALE * (q.abs() @ k.abs().transpose(-1, -2))
    eP = 2 * eS.amax(-1, keepdim=True) + (T + 32) * 2.0 ** -24
    amb = torch.zeros_like(P)
    if rnd:
        ulp = tf32_ulp(P)
        mid = (torch.floor(P / ulp) + 0.5) * ulp
        amb = torch.where((P - mid).abs() <= eP * P, ulp, amb)
    delta = _unheads((P * (eP + 64 * 2.0 ** -24)) @ v.abs() + amb @ v.abs())
    return o, delta


def attention_bwd(qkv, dO, B, T, heads, rnd=True):
    """``k_attention_bwd``: dqkv[B*T][3W] with P recomputed, tf32 q, k, v, dO, P, dS when rnd."""
    W = qkv.shape[1] // 3
    r = tf32 if rnd else (lambda t: t.double())
    q, k, v = (_heads(r(t), B, T, heads) for t in qkv.double().split(W, dim=1))
    do = _heads(r(dO.double()), B, T, heads)
    P = torch.softmax(q @ k.transpose(-1, -2) * ATT_SCALE, -1)
    dP = do @ v.transpose(-1, -2)
    dS = P * (dP - (P * dP).sum(-1, keepdim=True)) * ATT_SCALE
    dSr, Pr = r(dS), r(P)
    dq, dk, dv = dSr @ k, dSr.transpose(-1, -2) @ q, Pr.transpose(-1, -2) @ do
    return torch.cat([_unheads(dq), _unheads(dk), _unheads(dv)], 1)


def causal_attention(qkv, B, T, heads):
    """``k_causal_attention`` (fp32 FFMA, no tf32): o and a bound of its fp32 error per element."""
    W = qkv.shape[1] // 3
    q, k, v = (_heads(t, B, T, heads) for t in qkv.double().split(W, dim=1))
    mask = torch.full((T, T), float("-inf"), dtype=torch.float64).triu_(1)
    P = torch.softmax(q @ k.transpose(-1, -2) * ATT_SCALE + mask, -1)
    o = _unheads(P @ v)
    eS = 2.0 ** -24 * 72 * ATT_SCALE * (q.abs() @ k.abs().transpose(-1, -2))
    eP = 2 * eS.amax(-1, keepdim=True) + (T + 32) * 2.0 ** -24
    return o, _unheads((P * (eP + (T + 16) * 2.0 ** -24)) @ v.abs())


# ----------------------------------------------------------------------------------------------------- preprocessing
def resize_matrix(n_in: int, n_out: int, f32: bool = False) -> torch.Tensor:
    """[n_out][n_in] weights of the 1-D bilinear resize, align_corners=False, no antialias (torch's
    area_pixel_compute_source_index: negative source positions clamp to 0, the upper neighbour clamps to the edge).
    f32: the source positions as the kernels compute them, (d + 0.5) * fp32(n_in / n_out) - 0.5 rounded once to fp32
    (a fused multiply-add); their fractions are then exact."""
    R = torch.zeros(n_out, n_in, dtype=torch.float64)
    scale = float(np.float32(n_in) / np.float32(n_out)) if f32 else n_in / n_out
    for d in range(n_out):
        src = (d + 0.5) * scale - 0.5
        src = max(float(np.float32(src)) if f32 else src, 0.0)
        i0 = min(int(src), n_in - 1)
        i1 = i0 + (1 if i0 < n_in - 1 else 0)
        lam = src - i0
        R[d, i0] += 1 - lam
        R[d, i1] += lam
    return R


def resize(canvas, IS, f32=False):
    """[B][H][W][3] -> [B][3][IS][IS] bilinear."""
    c = canvas.double().permute(0, 3, 1, 2)
    Ry, Rx = resize_matrix(c.shape[2], IS, f32), resize_matrix(c.shape[3], IS, f32)
    return Ry @ c @ Rx.t()


def resize_adjoint(g, H, W, f32=False):
    """R^T: [B][3][IS][IS] -> [B][H][W][3]."""
    IS = g.shape[-1]
    Ry, Rx = resize_matrix(H, IS, f32), resize_matrix(W, IS, f32)
    return (Ry.t() @ g.double() @ Rx).permute(0, 2, 3, 1)


def _norm_consts():
    """Normalize's mean and std as the fp32 constants the kernels hold."""
    as64 = lambda v: torch.tensor(v, dtype=torch.float32).double().view(1, 3, 1, 1)
    return as64(CLIP_MEAN), as64(CLIP_STD)


def im2col(img, P):
    """[B][3][IS][IS] -> [B*g*g][3*P*P], row b*g*g + patch, column c*P*P + (y%P)*P + x%P."""
    B, C, IS, _ = img.shape
    g = IS // P
    return img.reshape(B, C, g, P, g, P).permute(0, 2, 4, 1, 3, 5).reshape(B * g * g, C * P * P)


def col2im(a, B, IS, P):
    g = IS // P
    return a.reshape(B, g, g, 3, P, P).permute(0, 3, 1, 4, 2, 5).reshape(B, 3, IS, IS)


def preprocess(canvas, IS, P, f32=False):
    """``k_preprocess`` mode 0 before the fp16 rounding: im2col((resize(canvas) - mean) / std)."""
    mean, std = _norm_consts()
    return im2col((resize(canvas, IS, f32) - mean) / std, P)


def preprocess_bwd(dpatch, B, H, W, IS, P, f32=False):
    """``k_preprocess_bwd`` mode 0: R^T (col2im(dpatch) / std)."""
    _, std = _norm_consts()
    return resize_adjoint(col2im(dpatch.double(), B, IS, P) / std, H, W, f32)


# -------------------------------------------------------------------------------------------------------------- head
def head_proj(x, B, T, g, b, proj):
    """``k_head_proj``: (emb[B][OD], ynorm[B][W]) = (LN(x[b, 0]) @ proj, LN(x[b, 0]))."""
    y = layernorm(x.double().reshape(B, T, -1)[:, 0], g, b)
    return y @ proj.double(), y


def cosine(emb, text):
    e, t = emb.double(), text.double()
    return (e * t).sum(-1) / torch.clamp(e.norm(dim=-1) * t.norm(dim=-1), min=1e-8)


def head_bwd_dy(proj, text, emb, g_cos=None, g_emb=None):
    """``k_head_bwd_dy``: dy[B][W] = proj . (g_cos d cos / d emb + g_emb); the cosine term is 0 for a zero vector."""
    e, t = emb.double(), text.double()
    de = torch.zeros_like(e)
    if g_cos is not None:
        na, nt = e.norm(dim=-1, keepdim=True), t.norm(dim=-1, keepdim=True)
        c = (e * t).sum(-1, keepdim=True)
        ok = (na > 0) & (nt > 0)
        d = t / (na * nt) - c * e / (na ** 3 * nt)
        de = de + torch.where(ok, g_cos.double()[:, None] * d, torch.zeros_like(d))
    if g_emb is not None:
        de = de + g_emb.double()
    return de @ proj.double().t()


def head_bwd_ln(x, B, T, g, dy):
    """``k_head_bwd_ln``: dx[B*T][W], LN backward on each image's row 0, zero elsewhere."""
    xr = x.double().reshape(B, T, -1)
    dx = torch.zeros_like(xr)
    dx[:, 0] = layernorm_bwd(xr[:, 0], dy, g)
    return dx.reshape(B * T, -1)


def text_eot_rows(tok, x, B, T):
    """``k_text_eot_rows``: x[b, argmax_t tok[b, t]] (first maximum)."""
    return x.double().reshape(B, T, -1)[torch.arange(B), tok.long().argmax(-1)]
