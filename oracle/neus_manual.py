"""CPU oracle (test infrastructure, never on the product path): the fine pass of the
NeuS renderer with a HAND-DERIVED backward -- no autograd anywhere in this file.

Why it exists: the reference obtains its second-order terms from
``torch.autograd.grad(create_graph=True)`` (models/fields.py:96-107) and never writes
the formulas down.  The CUDA path must.  This file states them once, in the exact
step order the kernels of ``avatarclip_b200/csrc`` execute (the step names below are
the kernel names), and ``tests/test_oracle_manual.py`` proves them against
``oracle.neus`` autograd in fp64.  The GPU tests compare the whole render with this
oracle; tests/test_neus_kernels_gpu.py checks the compositing, scalar and placement
kernels alone against fp64 autograd of oracle.neus (oracle/neus_kernels.py).

Symbols (per sample point; P = rays x samples):
  y = scale * x, e = enc(y) [E];  in_l: input of linear l (after the optional skip
  concat /sqrt2), z_l = W_l in_l + b_l, a_{l+1} = softplus100(z_l);
  qt_l = d z_L[0] / d z_l,  u_l = W_l^T qt_l = d z_L[0] / d in_l,  ge = d z_L[0] / d e,
  n = grad_x sdf = D(y)^T ge  (D = d enc / d y).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch

from .neus import ColorConf, RenderConf, SDFConf, effective_weight, inv_s_from_variance

SQRT1_2 = 1.0 / math.sqrt(2.0)
BETA = 100.0
THRESH = 20.0


# ----------------------------------------------------------------------------- pointwise
def softplus_all(z):
    """softplus_beta(z), its first and second derivative with torch's threshold rule
    (beta*z > 20 -> identity, derivative 1, second derivative 0)."""
    bz = z * BETA
    lin = bz > THRESH
    sp = torch.where(lin, z, torch.log1p(torch.exp(torch.clamp(bz, max=THRESH))) / BETA)
    s1 = torch.where(lin, torch.ones_like(z), torch.sigmoid(bz))
    s2 = torch.where(lin, torch.zeros_like(z), BETA * s1 * (1.0 - s1))
    return sp, s1, s2


def encode(y, multires):
    outs = [y]
    for k in range(multires):
        f = float(2 ** k)
        outs += [torch.sin(y * f), torch.cos(y * f)]
    return torch.cat(outs, -1)


def enc_jacT_apply(y, multires, ge):
    """n = D(y)^T ge  -> [P,3]."""
    n = ge[:, 0:3].clone()
    for k in range(multires):
        f = float(2 ** k)
        n = n + f * torch.cos(y * f) * ge[:, 3 + 6 * k: 6 + 6 * k] - f * torch.sin(y * f) * ge[:, 6 + 6 * k: 9 + 6 * k]
    return n


def enc_jac_apply(y, multires, nbar):
    """gebar = D(y) nbar -> [P,E]."""
    outs = [nbar]
    for k in range(multires):
        f = float(2 ** k)
        outs += [f * torch.cos(y * f) * nbar, -f * torch.sin(y * f) * nbar]
    return torch.cat(outs, -1)


# ----------------------------------------------------------------------------- forward
def fine_forward(sdf_p, col_p, variance, sconf: SDFConf, cconf: ColorConf, rconf: RenderConf,
                 rays_o, rays_d, z_vals, background_rgb=None, cos_anneal_ratio=0.0):
    """Forward of render_core (models/renderer.py:195-300) in kernel order.  Returns
    (outputs dict with the reference's keys, stash for the backward)."""
    assert cconf.mode == "no_view_dir" and cconf.multires_view == 0 and rconf.extra_color
    R, S = z_vals.shape
    dt = z_vals.dtype
    Lr = sconf.n_lin - 1                      # index of the last SDF linear
    E = sconf.d_enc
    skip = set(sconf.skip_in)
    W = [effective_weight(sdf_p, f"lin{l}") for l in range(sconf.n_lin)]
    B = [sdf_p[f"lin{l}.bias"] for l in range(sconf.n_lin)]

    # --- k_points_encode
    sample_dist = 2.0 / rconf.n_samples
    dists = torch.cat([z_vals[:, 1:] - z_vals[:, :-1], torch.full((R, 1), sample_dist, dtype=dt)], -1)
    mid_z = z_vals + dists * 0.5
    x = (rays_o[:, None, :] + rays_d[:, None, :] * mid_z[..., None]).reshape(-1, 3)
    dirs = rays_d[:, None, :].expand(R, S, 3).reshape(-1, 3)
    y = x * sconf.scale
    e = encode(y, sconf.multires)

    # --- value chain: gemm + EpiValue per layer
    ins: List[torch.Tensor] = []
    zs: List[torch.Tensor] = []
    a = e
    for l in range(sconf.n_lin):
        inp = torch.cat([a, e], 1) * SQRT1_2 if l in skip else a
        ins.append(inp)
        z = inp @ W[l].t() + B[l]
        zs.append(z)
        if l < Lr:
            a = softplus_all(z)[0]
    sdf = zs[Lr][:, :1] / sconf.scale
    feat = zs[Lr][:, 1:]

    # --- gradient chain: k_chain_start, then gemm(q_l, W_l) + EpiChain for l = L-1 .. 0
    ge = torch.zeros(x.shape[0], E, dtype=dt)
    qts: List[Optional[torch.Tensor]] = [None] * sconf.n_lin     # qt_l for l < L (qt_L = e_0)
    u = W[Lr][0:1, :].expand(x.shape[0], -1)                      # u_L: constant row 0 of W_L
    for l in range(Lr, -1, -1):
        if l < Lr:
            u = qts[l] @ W[l]
        if l in skip:
            ge = ge + u[:, -E:] * SQRT1_2
            ua = u[:, :-E] * SQRT1_2
        else:
            ua = u
        if l == 0:
            ge = ge + ua
        else:
            qts[l - 1] = softplus_all(zs[l - 1])[1] * ua
    # --- k_normal
    n = enc_jacT_apply(y, sconf.multires, ge)

    # --- colour net
    Wc = [effective_weight(col_p, f"lin{l}") for l in range(cconf.n_lin)]
    Bc = [col_p[f"lin{l}.bias"] for l in range(cconf.n_lin)]
    Wx, Bx = effective_weight(col_p, "extra_lin"), col_p["extra_lin.bias"]
    cin6 = torch.cat([x, n], -1)
    hs: List[torch.Tensor] = []
    h = None
    for l in range(cconf.n_lin - 1):
        if l == 0:
            c = feat @ Wc[0][:, 6:].t() + cin6 @ Wc[0][:, :6].t() + Bc[0]   # EpiColor0: rank-6 update
        else:
            c = h @ Wc[l].t() + Bc[l]
        h = torch.relu(c)
        hs.append(h)
    W6 = torch.cat([Wc[-1], Wx], 0)
    b6 = torch.cat([Bc[-1], Bx], 0)
    rgb6 = torch.sigmoid(h @ W6.t() + b6)                                   # k_heads

    # --- k_composite (per ray)
    inv_s = inv_s_from_variance(variance)
    a_ = cos_anneal_ratio
    tc = (dirs * n).sum(-1, keepdim=True)
    ic = -(torch.relu(-tc * 0.5 + 0.5) * (1.0 - a_) + torch.relu(-tc) * a_)
    d = dists.reshape(-1, 1)
    en = sdf + ic * d * 0.5
    ep = sdf - ic * d * 0.5
    Pp = torch.sigmoid(ep * inv_s)
    Pn = torch.sigmoid(en * inv_s)
    araw = ((Pp - Pn + 1e-5) / (Pp + 1e-5)).reshape(R, S)
    alpha = araw.clip(0.0, 1.0)
    T = torch.cumprod(torch.cat([torch.ones(R, 1, dtype=dt), 1.0 - alpha + 1e-7], -1), -1)[:, :-1]
    w = alpha * T
    wsum = w.sum(-1, keepdim=True)
    rgb6r = rgb6.reshape(R, S, 6)
    color = (w[..., None] * rgb6r[..., :3]).sum(1)
    extra = (w[..., None] * rgb6r[..., 3:]).sum(1)
    if background_rgb is not None:
        extra = extra + background_rgb * (1.0 - wsum)
    xnorm = torch.linalg.norm(x, dim=-1).reshape(R, S)
    relax = (xnorm < 1.2).to(dt)
    gn = torch.linalg.norm(n, dim=-1).reshape(R, S)
    cnt = relax.sum()
    gerr = (relax * (gn - 1.0) ** 2).sum() / (cnt + 1e-5)

    out = {
        "color_fine": color, "extra_color_fine": extra,
        "s_val": (1.0 / inv_s).reshape(1, 1).expand(R, 1),
        "cdf_fine": Pp.reshape(R, S), "weight_sum": wsum, "weight_max": w.max(-1, keepdim=True)[0],
        "gradients": n.reshape(R, S, 3), "weights": w, "mid_z_vals": mid_z,
        "gradient_error": gerr, "inside_sphere": (xnorm < 1.0).to(dt),
    }
    stash = dict(R=R, S=S, x=x, y=y, e=e, dirs=dirs, dists=dists, ins=ins, zs=zs, qts=qts, ge=ge, n=n,
                 feat=feat, cin6=cin6, hs=hs, rgb6=rgb6, sdf=sdf, inv_s=inv_s, tc=tc, ic=ic, ep=ep, en=en,
                 Pp=Pp, Pn=Pn, araw=araw, alpha=alpha, T=T, w=w, relax=relax, gn=gn, cnt=cnt,
                 W=W, Wc=Wc, W6=W6, background=background_rgb, a=a_)
    return out, stash


# ----------------------------------------------------------------------------- backward
def weight_norm_backward(p, name, Wbar):
    """W = g v/||v||  ->  gbar = sum_in Wbar * vhat ;  vbar = g/||v|| (Wbar - gbar vhat)."""
    v, g = p[f"{name}.weight_v"], p[f"{name}.weight_g"]
    nv = v.norm(dim=1, keepdim=True)
    vhat = v / nv
    gbar = (Wbar * vhat).sum(1, keepdim=True)
    vbar = g / nv * (Wbar - gbar * vhat)
    return gbar, vbar


def fine_backward(sdf_p, col_p, variance, sconf: SDFConf, cconf: ColorConf, rconf: RenderConf,
                  st, cot: Dict[str, torch.Tensor]):
    """Backward of fine_forward.  ``cot`` maps output names (color_fine, extra_color_fine,
    s_val, cdf_fine, weight_sum, weight_max, gradients, weights, gradient_error) to
    cotangents; missing entries mean zero.  Returns parameter gradients keyed like the
    reference's named_parameters (``sdf.lin0.weight_g`` ...)."""
    R, S = st["R"], st["S"]
    dt = st["x"].dtype
    P = R * S
    E = sconf.d_enc
    Lr = sconf.n_lin - 1
    skip = set(sconf.skip_in)
    W, Wc, W6 = st["W"], st["Wc"], st["W6"]

    def get(k, shape):
        v = cot.get(k)
        return torch.zeros(shape, dtype=dt) if v is None else v.to(dt).reshape(shape)

    g_color, g_extra = get("color_fine", (R, 3)), get("extra_color_fine", (R, 3))
    g_wsum, g_wmax = get("weight_sum", (R, 1)), get("weight_max", (R, 1))
    g_w, g_cdf = get("weights", (R, S)), get("cdf_fine", (R, S))
    g_n, g_sval = get("gradients", (P, 3)), get("s_val", (R, 1))
    g_gerr = get("gradient_error", ())

    # --- k_composite_bwd (per ray)
    w, T, alpha, araw = st["w"], st["T"], st["alpha"], st["araw"]
    rgb6r = st["rgb6"].reshape(R, S, 6)
    wbar = g_w + g_wsum + (rgb6r[..., :3] * g_color[:, None, :]).sum(-1) + (rgb6r[..., 3:] * g_extra[:, None, :]).sum(-1)
    if st["background"] is not None:
        wbar = wbar - (g_extra * st["background"]).sum(-1, keepdim=True)
    amax = w.argmax(-1, keepdim=True)
    wbar = wbar + torch.zeros_like(w).scatter_(1, amax, g_wmax)
    rgb6bar = torch.cat([w[..., None] * g_color[:, None, :], w[..., None] * g_extra[:, None, :]], -1).reshape(P, 6)
    abar = torch.zeros_like(alpha)
    Tbar_next = torch.zeros(R, dtype=dt)
    for j in range(S - 1, -1, -1):                    # reverse scan, T_{j+1} = T_j (1 - a_j + 1e-7)
        abar[:, j] = wbar[:, j] * T[:, j] - Tbar_next * T[:, j]
        Tbar_next = wbar[:, j] * alpha[:, j] + Tbar_next * (1.0 - alpha[:, j] + 1e-7)
    abar = abar * ((araw >= 0.0) & (araw <= 1.0)).to(dt)
    abar = abar.reshape(P, 1)
    Pp, Pn, ep, en, inv_s = st["Pp"], st["Pn"], st["ep"], st["en"], st["inv_s"]
    den = Pp + 1e-5
    Ppbar = abar * Pn / (den * den) + g_cdf.reshape(P, 1)      # d alpha/d Pp = (den - num)/den^2 = Pn/den^2
    Pnbar = -abar / den
    dPp, dPn = Pp * (1.0 - Pp), Pn * (1.0 - Pn)
    epbar, enbar = Ppbar * dPp * inv_s, Pnbar * dPn * inv_s
    inv_s_bar = (Ppbar * dPp * ep + Pnbar * dPn * en).sum() - g_sval.sum() / (inv_s * inv_s)
    sdfbar = epbar + enbar
    d = st["dists"].reshape(P, 1)
    icbar = (enbar - epbar) * d * 0.5
    tc, a_ = st["tc"], st["a"]
    tcbar = icbar * (0.5 * (1.0 - a_) * (tc < 1.0).to(dt) + a_ * (tc < 0.0).to(dt))
    nbar = tcbar * st["dirs"] + g_n
    gn = st["gn"].reshape(P, 1)
    relax = st["relax"].reshape(P, 1)
    eik = g_gerr * relax * 2.0 * (gn - 1.0) / (st["cnt"] + 1e-5)
    nbar = nbar + torch.where(gn > 0, eik * st["n"] / gn.clamp(min=1e-30), torch.zeros_like(st["n"]))
    var_bar = inv_s_bar * 10.0 * inv_s if (1e-6 < float(torch.exp(variance * 10.0)) < 1e6) else torch.zeros((), dtype=dt)

    grads: Dict[str, torch.Tensor] = {"var.variance": var_bar.reshape(())}

    # --- colour heads: k_heads_bwd (thin gemm + thin wgrad)
    y6bar = rgb6bar * st["rgb6"] * (1.0 - st["rgb6"])
    hs = st["hs"]
    hbar = y6bar @ W6
    W6bar = y6bar.t() @ hs[-1]
    b6bar = y6bar.sum(0)
    nl = cconf.n_lin
    col_wbar = {f"lin{nl - 1}": (W6bar[:3], b6bar[:3]), "extra_lin": (W6bar[3:], b6bar[3:])}
    # --- colour hidden layers: dgrad gemm + EpiDgradRelu, wgrad
    featbar = None
    for l in range(nl - 2, -1, -1):
        cbar = hbar * (hs[l] > 0).to(dt)
        if l == 0:
            inp = torch.cat([st["cin6"], st["feat"]], 1)
            col_wbar["lin0"] = (cbar.t() @ inp, cbar.sum(0))
            featbar = cbar @ Wc[0][:, 6:]
            cin6bar = cbar @ Wc[0][:, :6]
            nbar = nbar + cin6bar[:, 3:6]                       # xbar (cols 0:3) is discarded: pts is a leaf
        else:
            col_wbar[f"lin{l}"] = (cbar.t() @ hs[l - 1], cbar.sum(0))
            hbar = cbar @ Wc[l]
    for name, (Wb, bb) in col_wbar.items():
        gbar, vbar = weight_norm_backward(col_p, name, Wb)
        grads[f"col.{name}.weight_g"], grads[f"col.{name}.weight_v"], grads[f"col.{name}.bias"] = gbar, vbar, bb

    # --- SDF: second-order sweep (forward order) -- k_dge, then gemm(ubar_l, W_l^T) + EpiChainBwd
    gebar = enc_jac_apply(st["y"], sconf.multires, nbar)
    Wbar = [torch.zeros_like(Wl) for Wl in W]
    z2bar: List[Optional[torch.Tensor]] = [None] * sconf.n_lin
    uabar = gebar
    zs, qts, ins = st["zs"], st["qts"], st["ins"]
    for l in range(0, Lr + 1):
        ubar = torch.cat([uabar * SQRT1_2, gebar * SQRT1_2], 1) if l in skip else uabar
        if l == Lr:
            Wbar[l][0, :] += ubar.sum(0)                        # qt_L = e_0: only row 0 of W_L is touched
            break
        Wbar[l] += qts[l].t() @ ubar                            # wgrad (qt_l, ubar_l)
        qbar = ubar @ W[l].t()                                  # gemm, forward shape
        _, s1, _ = softplus_all(zs[l])
        uabar = s1 * qbar                                       # -> ubar_{l+1}
        z2bar[l] = BETA * (1.0 - s1) * qts[l] * qbar            # = softplus'' * ua_{l+1} * qbar
    # --- SDF: value backward (reverse order) -- gemm(zbar_l, W_l) + EpiDgrad, wgrad
    zbar = torch.cat([sdfbar / sconf.scale, featbar], 1)
    bbar = [None] * sconf.n_lin
    for l in range(Lr, -1, -1):
        Wbar[l] += zbar.t() @ ins[l]
        bbar[l] = zbar.sum(0)
        if l == 0:
            break                                               # d/d e only feeds xbar: discarded
        inbar = zbar @ W[l]
        abar_l = inbar[:, :-E] * SQRT1_2 if l in skip else inbar
        zbar = softplus_all(zs[l - 1])[1] * abar_l + z2bar[l - 1]
    for l in range(sconf.n_lin):
        gbar, vbar = weight_norm_backward(sdf_p, f"lin{l}", Wbar[l])
        grads[f"sdf.lin{l}.weight_g"], grads[f"sdf.lin{l}.weight_v"], grads[f"sdf.lin{l}.bias"] = gbar, vbar, bbar[l]
    return grads
