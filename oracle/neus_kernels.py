"""float64 references of the NeuS kernels outside the GEMM tiles (avc_neus_kernels.cuh): compositing, scalars,
placement, weight packing and its backward, the encoding, the thin contractions and the ends of the gradient chain; and
of the fused value-chain kernel (avc_chain.cu), which holds its own tiles.
One function per kernel, taking the fp32 inputs the kernel reads.  They run on whatever device the inputs live on.

The compositing forward is oracle.neus.composite itself; its backward is fp64 autograd through it, so the kernels'
hand-derived backward is checked against an independent derivation.  Where a kernel rounds on purpose like torch eager
fp32 (depth placement, mid-points, sample points, the ``radius < 1`` mask, y = scale x, the sqrt(1/2) skip copies), the
rounding is restated here as separately rounded fp32 operations, and the GPU tests compare those outputs exactly.
tests/test_neus_kernels_cpu.py pins each function against torch."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle import neus

F64 = torch.float64
COT_KEYS = ["color", "extra", "wsum", "wmax", "weights", "cdf", "gradients", "gerr"]


# --------------------------------------------------------------------------- scalars
def inv_s(variance: torch.Tensor, dtype=F64) -> torch.Tensor:
    """k_ctx_init: clip(exp(10 v), 1e-6, 1e6) (models/fields.py:276, renderer.py:234)."""
    return neus.inv_s_from_variance(variance.to(dtype))


def variance_grad(variance, invs_bar, g_sval, dtype=F64) -> torch.Tensor:
    """k_variance_grad: d/dv of invs_bar * inv_s(v) + sum(g_sval) / inv_s(v) (s_val = 1 / inv_s per ray), by autograd
    through the clip, whose backward passes the gradient at both bounds."""
    v = variance.detach().to(dtype).reshape(1).requires_grad_(True)
    s = neus.inv_s_from_variance(v)
    loss = invs_bar.to(dtype).sum() * s.sum()
    if g_sval is not None:
        loss = loss + (g_sval.to(dtype).reshape(-1, 1) * (1.0 / s)).sum()
    (g,) = torch.autograd.grad(loss, v)
    return g


# --------------------------------------------------------------------------- deliberate fp32 rounding
def fma_f32(a: float, b: float, c: float) -> float:
    """fp32 fused multiply-add: a * b + c rounded once (round to nearest even), from the exact rational value."""
    import numpy as np
    from fractions import Fraction
    a, b, c = (np.float32(v) for v in (a, b, c))
    exact = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    f = np.float32(float(exact))
    cands = [f, np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))]
    err = [abs(Fraction(float(v)) - exact) for v in cands]
    best = min(err)
    tied = [v for v, e in zip(cands, err) if e == best]
    return float(min(tied, key=lambda v: int(np.array(v).view(np.int32)) & 1))


def torch_linspace(start: float, end: float, n: int) -> torch.Tensor:
    """at::linspace in fp32 as its CUDA kernel computes it: step = (end - start) / (n - 1); the first n // 2 entries
    are fma(step, j, start), the rest fma(-step, n - 1 - j, end) (torch's build contracts both into FMAs)."""
    if n == 1:
        return torch.tensor([start], dtype=torch.float32)
    s, e = torch.tensor(start, dtype=torch.float32), torch.tensor(end, dtype=torch.float32)
    step = ((e - s) / torch.tensor(float(n - 1), dtype=torch.float32)).item()
    v = [fma_f32(step, j, s.item()) if j < n // 2 else fma_f32(-step, n - 1 - j, e.item()) for j in range(n)]
    return torch.tensor(v, dtype=torch.float32)


def coarse_z(near, far, jitter, n: int) -> torch.Tensor:
    """k_coarse_z as torch eager fp32 computes it on the GPU (renderer.py:305-306,319): near + (far - near) *
    linspace(0, 1, n), plus jitter * 2 / n, where torch divides by the scalar as a product with its fp32 reciprocal.
    near, far, jitter: [R] fp32."""
    z = near[:, None] + (far - near)[:, None] * torch_linspace(0.0, 1.0, n).to(near.device)
    if jitter is not None:
        z = z + jitter[:, None] * 2.0 * (torch.tensor(1.0) / torch.tensor(float(n))).to(near.device)
    return z


def mid_points(rays_o, rays_d, z, sample_dist: float):
    """Mid-points and sample points of the fine pass in torch eager fp32 (renderer.py:208-213): dist = z[j+1] - z[j]
    (sample_dist for the last), mid = z + dist * 0.5, x = o + d * mid.  Returns (mid [R,S], x [R,S,3])."""
    dist = torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], sample_dist)], -1)
    mid = z + dist * 0.5
    x = rays_o[:, None, :] + rays_d[:, None, :] * mid[..., None]
    return mid, x


def radius_f32(x) -> torch.Tensor:
    """sqrt((x0 x0 + x1 x1) + x2 x2) with every operation rounded to fp32 (ray_radius in the placement kernels)."""
    return torch.sqrt((x[..., 0] * x[..., 0] + x[..., 1] * x[..., 1]) + x[..., 2] * x[..., 2])


def split_bf16(v: torch.Tensor):
    """The two-term bf16 split of an fp32 tensor: hi = bf16 RNE of v, lo = bf16 RNE of fp32(v - hi)."""
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16)
    return hi, lo


# --------------------------------------------------------------------------- compositing
def _composite_inputs(rays_d, z, sdf, cin, rgb6, background, bg_kind, dtype):
    R, S = z.shape
    c = lambda t: t.detach().to(dtype)
    pts = c(cin[:, 0:3])
    normals = c(cin[:, 3:6])
    dirs = c(rays_d)[:, None, :].expand(R, S, 3).reshape(-1, 3)
    bg = None
    if bg_kind == 1:
        bg = c(background).reshape(1, 3)
    elif bg_kind == 2:
        bg = c(background).reshape(R, 1)
    y = c(rgb6[:, 0:6])
    return R, S, pts, normals, dirs, bg, c(sdf).reshape(-1, 1), y


def composite_fwd(rays_d, z, sdf, cin, rgb6, background, bg_kind: int, inv_s_val, cos_anneal: float,
                  sample_dist: float, eik_den_total=None, dtype=F64) -> Dict[str, torch.Tensor]:
    """k_composite_fwd on its own inputs: rays_d [R,3], z [R,S], sdf [P], cin [P,8] (points 0:3, normals 3:6), rgb6
    [P,8] (sigmoid outputs 0:6), background [3] / [R] / None, inv_s scalar tensor.  Returns the per-ray / per-sample
    outputs plus the per-ray eikonal partials eik_num / eik_den and gradient_error with normaliser eik_den_total."""
    R, S, pts, normals, dirs, bg, sd, y = _composite_inputs(rays_d, z, sdf, cin, rgb6, background, bg_kind, dtype)
    zz = z.detach().to(dtype)
    dists = torch.cat([zz[:, 1:] - zz[:, :-1], torch.full_like(zz[:, :1], sample_dist)], -1)
    s = torch.as_tensor(inv_s_val).to(dtype=dtype, device=zz.device).reshape(1, 1)
    den = None if eik_den_total is None else torch.as_tensor(eik_den_total).to(dtype)
    out = neus.composite(sd, normals, pts, y[:, 0:3].reshape(R, S, 3), y[:, 3:6].reshape(R, S, 3), dists, s, dirs, bg,
                         cos_anneal, relax_total=den)
    gnorm = torch.linalg.norm(normals.reshape(R, S, 3), ord=2, dim=-1)
    w = out["weights"]
    return {"color": out["color"], "extra": out["extra_color"], "weights": w, "cdf": out["cdf"],
            "wsum": w.sum(-1), "wmax": w.max(-1)[0], "s_val": (1.0 / s).reshape(1).expand(R),
            "eik_num": (out["relax"] * (gnorm - 1.0) ** 2).sum(-1), "eik_den": out["relax"].sum(-1),
            "gerr": out["gradient_error"]}


def first_argmax(w: torch.Tensor) -> torch.Tensor:
    """Index of the first largest entry of each row: where torch.max(dim) sends the gradient of a tie."""
    m = w.max(-1, keepdim=True)[0]
    idx = torch.arange(w.shape[-1], device=w.device).expand_as(w)
    return torch.where(w == m, idx, w.shape[-1]).min(-1)[0]


def composite_bwd(rays_d, z, sdf, cin, rgb6, background, bg_kind: int, inv_s_val, cos_anneal: float,
                  sample_dist: float, eik_den_total, cot: Dict[str, Optional[torch.Tensor]], weights_argmax=None,
                  dtype=F64) -> Dict[str, torch.Tensor]:
    """k_composite_bwd by autograd through composite_fwd: cotangents (any may be None) on color [R,3], extra [R,3],
    wsum [R], wmax [R], weights [R,S], cdf [R,S], gradients (the normals) [P,3], gerr [1].  The weight_max cotangent
    goes to the first maximum of ``weights_argmax`` (the forward's stored weights).  Returns y6bar [P,6] (the adjoint
    of the six head logits), sdfbar [P], nbar [P,3] and invs_bar [R] (per ray, the adjoint of inv_s through the
    compositing alone)."""
    R, S = z.shape
    sd = sdf.detach().to(dtype).reshape(-1).clone().requires_grad_(True)
    nrm = cin[:, 3:6].detach().to(dtype).clone().requires_grad_(True)
    y = rgb6[:, 0:6].detach().to(dtype)
    logit = (torch.log(y) - torch.log1p(-y)).requires_grad_(True)
    s = torch.as_tensor(inv_s_val).detach().to(dtype=dtype, device=nrm.device).reshape(1, 1).expand(R, 1).clone().requires_grad_(True)
    _, _, pts, _, dirs, bg, _, _ = _composite_inputs(rays_d, z, sdf, cin, rgb6, background, bg_kind, dtype)
    zz = z.detach().to(dtype)
    dists = torch.cat([zz[:, 1:] - zz[:, :-1], torch.full_like(zz[:, :1], sample_dist)], -1)
    den = None if eik_den_total is None else torch.as_tensor(eik_den_total).to(dtype)
    yy = torch.sigmoid(logit)
    c = neus.composite(sd.reshape(-1, 1), nrm, pts, yy[:, 0:3].reshape(R, S, 3), yy[:, 3:6].reshape(R, S, 3), dists,
                       s.expand(R, S).reshape(-1, 1), dirs, bg, cos_anneal, relax_total=den)
    w = c["weights"]
    outs = {"color": c["color"], "extra": c["extra_color"], "wsum": w.sum(-1), "weights": w, "cdf": c["cdf"],
            "gradients": nrm, "gerr": c["gradient_error"].reshape(1)}
    loss = torch.zeros((), dtype=dtype, device=nrm.device)
    for k, g in cot.items():
        if g is None:
            continue
        if k == "wmax":
            am = first_argmax((weights_argmax if weights_argmax is not None else w).detach())
            loss = loss + (g.to(dtype).reshape(-1) * w.gather(1, am[:, None]).reshape(-1)).sum()
        else:
            loss = loss + (outs[k] * g.to(dtype).reshape(outs[k].shape)).sum()
    if not loss.requires_grad:
        return {"y6bar": torch.zeros_like(logit), "sdfbar": torch.zeros_like(sd), "nbar": torch.zeros_like(nrm),
                "invs_bar": torch.zeros(R, dtype=dtype, device=nrm.device)}
    gl, gs, gn, gi = torch.autograd.grad(loss, [logit, sd, nrm, s], allow_unused=True)
    zl = lambda g, t: torch.zeros_like(t) if g is None else g
    return {"y6bar": zl(gl, logit), "sdfbar": zl(gs, sd), "nbar": zl(gn, nrm), "invs_bar": zl(gi, s).reshape(R)}


# --------------------------------------------------------------------------- placement
def upsample_cdf(rays_o, rays_d, z, sdf, inv_s_val: float, dtype=F64):
    """up_sample's cdf (renderer.py:133-177, sample_pdf :39-50) for rays [R,3], z / sdf [R,n]: [R,n] with cdf[:,0] = 0.
    The ``radius < 1`` mask comes from the fp32 points (separately rounded, as the kernel and torch eager compute it);
    everything after it in ``dtype``."""
    R, n = z.shape
    x = rays_o[:, None, :] + rays_d[:, None, :] * z[..., None]
    rad = radius_f32(x)
    inside = ((rad[:, :-1] < 1.0) | (rad[:, 1:] < 1.0)).to(dtype)
    zz, ss = z.to(dtype), sdf.to(dtype)
    prev_sdf, next_sdf = ss[:, :-1], ss[:, 1:]
    prev_z, next_z = zz[:, :-1], zz[:, 1:]
    mid_sdf = (prev_sdf + next_sdf) * 0.5
    cos_val = (next_sdf - prev_sdf) / (next_z - prev_z + 1e-5)
    prev_cos = torch.cat([torch.zeros(R, 1, dtype=dtype, device=z.device), cos_val[:, :-1]], dim=-1)
    cos_val = torch.minimum(prev_cos, cos_val).clip(-1e3, 0.0) * inside
    dist = next_z - prev_z
    pc = torch.sigmoid((mid_sdf - cos_val * dist * 0.5) * inv_s_val)
    nc = torch.sigmoid((mid_sdf + cos_val * dist * 0.5) * inv_s_val)
    alpha = (pc - nc + 1e-5) / (pc + 1e-5)
    trans = torch.cumprod(torch.cat([torch.ones(R, 1, dtype=dtype, device=z.device), 1.0 - alpha + 1e-7], -1), -1)[:, :-1]
    w = alpha * trans + 1e-5
    cdf = torch.cumsum(w / w.sum(-1, keepdim=True), -1)
    return torch.cat([torch.zeros(R, 1, dtype=dtype, device=z.device), cdf], -1)


def upsample_u(per: int) -> torch.Tensor:
    """The fp32 sample positions linspace(0.5 / per, 1 - 0.5 / per, per) of sample_pdf(det=True), with the ends
    rounded as k_upsample rounds them (0.5f / per, 1 - that)."""
    a = torch.tensor(0.5, dtype=torch.float32) / per
    return torch_linspace(a.item(), (1.0 - a).item(), per)


def invert_cdf(z, cdf, u, bins: Optional[torch.Tensor] = None, clamp=1e-5):
    """sample_pdf's inverse-CDF step (renderer.py:51-69) in the dtype of cdf: u [per] -> depths [R,per].  ``bins``
    ([R,per] int64, optional) forces the index of the cdf entry above u instead of searchsorted(right=True); ``clamp``
    (a number or [R,1]) is the threshold below which a bin's denominator is replaced by 1."""
    R, n = cdf.shape
    uu = u.to(cdf.dtype).to(cdf.device).expand(R, -1).contiguous()
    inds = torch.searchsorted(cdf, uu, right=True) if bins is None else bins
    below = (inds - 1).clamp(min=0)
    above = inds.clamp(max=n - 1)
    zz = z.to(cdf.dtype)
    cb, ca = cdf.gather(1, below), cdf.gather(1, above)
    zb, za = zz.gather(1, below), zz.gather(1, above)
    denom = ca - cb
    denom = torch.where(denom < clamp, torch.ones_like(denom), denom)
    return zb + (uu - cb) / denom * (za - zb)


def merge(z, sdf, newz, news):
    """cat_z_vals (renderer.py:179-193): stable sort of cat([z, newz]) (old entries first on ties); each sdf travels
    with its depth.  Returns (z_sorted, sdf_sorted or None)."""
    zs, idx = torch.sort(torch.cat([z, newz], -1), dim=-1, stable=True)
    so = None if news is None else torch.cat([sdf, news], -1).gather(1, idx)
    return zs, so


# --------------------------------------------------------------------------- weights
def effective_weight(v, g, dtype=F64) -> torch.Tensor:
    """k_pack_linear: W = g v / ||v|| per output row (torch.nn.utils.weight_norm, dim=0).  v [N,K], g [N] or [N,1]."""
    return neus.effective_weight({"w.weight_v": v.to(dtype), "w.weight_g": g.to(dtype).reshape(-1, 1)}, "w")


def wn_backward(v, g, wbar, dtype=F64):
    """k_wn_backward: with vhat = v / ||v||, gbar = sum_k Wbar vhat and vbar = g / ||v|| (Wbar - gbar vhat).  The bias
    gradient is a copy of the dense one (compared exactly).  Returns (gbar [N], vbar [N,K])."""
    v, g, wbar = v.to(dtype), g.to(dtype).reshape(-1, 1), wbar.to(dtype)
    nv = v.norm(dim=1, keepdim=True)
    vh = v / nv
    gbar = (wbar * vh).sum(1, keepdim=True)
    return gbar.reshape(-1), g / nv * (wbar - gbar * vh)


# --------------------------------------------------------------------------- encoding
def scaled(x, scale: float) -> torch.Tensor:
    """y = scale x rounded to fp32, the input of every sin / cos of the encoding kernels."""
    return x.float() * torch.tensor(scale, dtype=torch.float32)


def encode(x, scale: float, multires: int, dtype=F64) -> torch.Tensor:
    """encode_group: positional_encode(y) of the fp32 y = scale x, in ``dtype``.  x [P,3] -> [P, 3 (1 + 2 multires)]."""
    return neus.positional_encode(scaled(x, scale).to(dtype), multires)


def skip_copy(e32: torch.Tensor) -> torch.Tensor:
    """The skip layers' copy of an fp32 encoding: each value times the fp32 sqrt(1/2), rounded once."""
    return e32.float() * torch.tensor(0.70710678118654752440, dtype=torch.float32)


def sample_points(rays_o, rays_d, z) -> torch.Tensor:
    """k_encode_samples' points o + d z in torch eager fp32 (renderer.py:182, :337).  z [R,n] -> [R,n,3]."""
    return rays_o[:, None, :] + rays_d[:, None, :] * z[..., None]


def inside_sphere(x) -> torch.Tensor:
    """renderer.py:219: (||x|| < 1) with the norm rounded like the kernel (radius_f32)."""
    return (radius_f32(x) < 1.0).float()


# --------------------------------------------------------------------------- thin contractions
def sdf_head(in_l, K: int, wsdf, bsdf, scale: float, dtype=F64) -> torch.Tensor:
    """k_thin_nt<1, OutSdf>: (in_L[:, :K] . w_sdf + b_sdf) / scale: only the K inputs of the last linear."""
    return (in_l[:, :K].to(dtype) @ wsdf[:K].to(dtype) + bsdf.to(dtype).reshape(())) / scale


def color_heads(ch, W6, b6, dtype=F64) -> torch.Tensor:
    """k_thin_nt<6, OutHeads>: sigmoid(ch W6[0:6]^T + b6[0:6]) -> [P,6]."""
    return torch.sigmoid(ch.to(dtype) @ W6[0:6].to(dtype).T + b6[0:6].to(dtype))


def nbar_add(nbar, cbar, c0xT, dtype=F64) -> torch.Tensor:
    """k_thin_nt<6, OutNbarAdd>: nbar[:, 0:3] + cbar W0[:, 3:6]; c0xT is the packed [8][Hc] transpose of lin0's first
    columns."""
    return nbar[:, 0:3].to(dtype) + cbar.to(dtype) @ c0xT[3:6].to(dtype).T


def thin_tn(S, Hm, s_scale: float = 1.0, dtype=F64):
    """k_thin_tn: (s_scale S)^T Hm -> [NI, NC] and the bias sum sum_p s_scale S[p] -> [NI]."""
    Ss = S.to(dtype) * s_scale
    return Ss.T @ Hm.to(dtype), Ss.sum(0)


def colsum(X, scale: float = 1.0, dtype=F64) -> torch.Tensor:
    """k_colsum: scale sum_p X[p]."""
    return X.to(dtype).sum(0) * scale


def heads_dgrad(y6bar, W6, h, dtype=F64) -> torch.Tensor:
    """k_heads_dgrad: (y6bar[:, 0:6] W6[0:6]) [h > 0] (ReLU' (0) = 0)."""
    return (y6bar[:, 0:6].to(dtype) @ W6[0:6].to(dtype)) * (h > 0).to(dtype)


# --------------------------------------------------------------------------- value chain
SQRT_HALF = 0.70710678118654752440


def value_chain(x0, skip, weights, biases, w_sdf, b_sdf, skip_layer: Optional[int], scale: float, dtype=F64,
                split_acts: bool = False, pre: Optional[list] = None) -> torch.Tensor:
    """k_sdf_chain (avc_chain.cu) on its own inputs: the SDF value chain of models/fields.py:72-91 from the encoded
    points to the sdf.  x0 [P, K_0] is the layer-0 input, skip [P, E] the skip linear's encoding columns as the kernel
    reads them (already times sqrt(1/2)) or None, weights / biases the L hidden linears ([N_l, K_l], [N_l]), w_sdf [K_L]
    and b_sdf the sdf row of the last linear, skip_layer the index (1..L) of the linear that takes cat([h, enc]) / sqrt(2)
    or None.  Per hidden linear: z = h W^T + b, softplus with beta 100 and threshold 20, times sqrt(1/2) when the next
    linear takes the skip concat, then the concat.  sdf = (h . w_sdf + b_sdf) / scale.
    ``split_acts`` rounds every activation that feeds another hidden linear to fp32 and then to its two-term bf16 split
    (split_bf16), as the kernel's epilogue stores it; the last hidden activation meets the head unsplit, as in the kernel.
    ``pre`` (a list) receives each linear's pre-activation z."""
    h = x0.to(dtype)
    L = len(weights)
    for l in range(L):
        z = h @ weights[l].to(dtype).T + biases[l].to(dtype)
        if pre is not None:
            pre.append(z)
        a = neus.softplus100(z)
        if skip_layer == l + 1:
            a = a * SQRT_HALF
        if split_acts and l + 1 < L:
            hi, lo = split_bf16(a.float())
            a = hi.to(dtype) + lo.to(dtype)
        if skip_layer == l + 1:
            a = torch.cat([a, skip.to(dtype)], -1)
        h = a
    return (h @ w_sdf.to(dtype) + b_sdf.to(dtype).reshape(())) / scale


# --------------------------------------------------------------------------- gradient chain

def chain_start(wsdf, zprev, n_prev: int, K_last: int, skip_last: bool, E: int, dtype=F64):
    """k_chain_start: qt_{L-1} = sp'(z_{L-1}) * w_sdf[0:N_{L-1}] (times sqrt(1/2) when the last linear takes the skip
    concat) and ge = the encoding part of w_sdf, w_sdf[K-E:K] sqrt(1/2), or 0.  Returns (qt [P, n_prev], ge [P, E])."""
    s = SQRT_HALF if skip_last else 1.0
    w = wsdf.to(dtype)
    qt = zprev[:, :n_prev].to(dtype) * w[:n_prev] * s
    P = zprev.shape[0]
    ge = (w[K_last - E:K_last] * s).expand(P, E) if skip_last else torch.zeros(P, E, dtype=dtype, device=zprev.device)
    return qt, ge


def _bands(x, scale: float, multires: int, dtype):
    y = scaled(x, scale).to(dtype)
    return [(float(2 ** k), torch.sin(y * 2 ** k), torch.cos(y * 2 ** k)) for k in range(multires)]


def normal(ge, x, scale: float, multires: int, dtype=F64) -> torch.Tensor:
    """k_normal: n = D(y)^T ge with D the Jacobian of positional_encode at y = scale x (the scale of y and the 1 / scale
    of the sdf cancel).  ge [P, >= E], x [P,3] -> [P,3]."""
    g = ge.to(dtype)
    n = g[:, 0:3].clone()
    for k, (f, sn, cs) in enumerate(_bands(x, scale, multires, dtype)):
        n = n + f * (cs * g[:, 3 + 6 * k:6 + 6 * k] - sn * g[:, 6 + 6 * k:9 + 6 * k])
    return n


def dge(x, nbar, scale: float, multires: int, dtype=F64) -> torch.Tensor:
    """k_dge: gebar = D(y) nbar -> [P, E] (the same Jacobian as ``normal``, applied forward)."""
    nb = nbar[:, 0:3].to(dtype)
    cols = [nb]
    for f, sn, cs in _bands(x, scale, multires, dtype):
        cols += [f * cs * nb, -f * sn * nb]
    return torch.cat(cols, -1)


def fill_gebar(gebar, E: int) -> torch.Tensor:
    """k_fill_gebar: the skip half of ubar, fp32 gebar[:, 0:E] times the fp32 sqrt(1/2), rounded once."""
    return skip_copy(gebar[:, 0:E])
