"""CPU oracle (test infrastructure, never on the product path): NeuS renderer of
AvatarCLIP restated with plain torch ops; autograd provides every gradient.

All citations are relative to /root/reference/AvatarGen/AppearanceGen.
The functions work in whatever dtype the inputs carry (fp32 for parity with the
reference, fp64 for tight checks of the hand-derived backward).

Parameters are passed as flat dicts with the reference's own state-dict key
names (``lin0.weight_g``, ``lin0.weight_v``, ``lin0.bias``, ``extra_lin.*``,
``variance``) so shipped checkpoints and reference modules can be fed directly.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Optional, Sequence

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------- config
@dataclass
class SDFConf:
    """Constructor arguments of SDFNetwork (models/fields.py:10-21)."""
    d_in: int = 3
    d_out: int = 257
    d_hidden: int = 256
    n_layers: int = 8
    skip_in: Sequence[int] = (4,)
    multires: int = 6
    bias: float = 0.5
    scale: float = 1.0
    geometric_init: bool = True
    weight_norm: bool = True
    inside_outside: bool = False

    @property
    def d_enc(self) -> int:
        return self.d_in * (1 + 2 * self.multires) if self.multires > 0 else self.d_in

    @property
    def n_lin(self) -> int:
        return self.n_layers + 1

    def layer_dims(self):
        """(in, out) of every linear: models/fields.py:24-43."""
        dims = [self.d_enc] + [self.d_hidden] * self.n_layers + [self.d_out]
        out = []
        for l in range(len(dims) - 1):
            o = dims[l + 1] - dims[0] if (l + 1) in self.skip_in else dims[l + 1]
            out.append((dims[l], o))
        return out


@dataclass
class ColorConf:
    """Constructor arguments of RenderingNetwork (models/fields.py:112-122)."""
    d_feature: int = 256
    mode: str = "no_view_dir"
    d_in: int = 6
    d_out: int = 3
    d_hidden: int = 256
    n_layers: int = 4
    weight_norm: bool = True
    multires_view: int = 0
    squeeze_out: bool = True
    extra_color: bool = True

    @property
    def n_lin(self) -> int:
        return self.n_layers + 1

    def layer_dims(self):
        dims = [self.d_in + self.d_feature] + [self.d_hidden] * self.n_layers + [self.d_out]
        return [(dims[l], dims[l + 1]) for l in range(len(dims) - 1)]


@dataclass
class RenderConf:
    """Constructor arguments of NeuSRenderer (models/renderer.py:73-93)."""
    n_samples: int = 64
    n_importance: int = 64
    n_outside: int = 0
    up_sample_steps: int = 4
    perturb: float = 1.0
    extra_color: bool = True


# --------------------------------------------------------------------------- parameters
def init_sdf_params(conf: SDFConf, generator: Optional[torch.Generator] = None,
                    dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Geometric initialisation, models/fields.py:36-66 (restated; the pinning
    script checks the *forward*, not the RNG stream, against the reference).
    weight_norm stores g = ||v||_row, v = W (torch.nn.utils.weight_norm, dim=0)."""
    p: Dict[str, torch.Tensor] = {}
    dims = conf.layer_dims()
    n_lin = len(dims)
    d0 = conf.d_enc
    for l, (din, dout) in enumerate(dims):
        w = torch.empty(dout, din, dtype=dtype)
        b = torch.zeros(dout, dtype=dtype)
        if l == n_lin - 1:
            mean = math.sqrt(math.pi) / math.sqrt(din)
            if conf.inside_outside:
                mean, bias = -mean, conf.bias
            else:
                bias = -conf.bias
            w.normal_(mean, 1e-4, generator=generator)
            b.fill_(bias)
        elif conf.multires > 0 and l == 0:
            w.zero_()
            w[:, :3].normal_(0.0, math.sqrt(2) / math.sqrt(dout), generator=generator)
        elif conf.multires > 0 and l in conf.skip_in:
            w.normal_(0.0, math.sqrt(2) / math.sqrt(dout), generator=generator)
            w[:, -(d0 - 3):] = 0.0
        else:
            w.normal_(0.0, math.sqrt(2) / math.sqrt(dout), generator=generator)
        p[f"lin{l}.weight_g"] = w.norm(dim=1, keepdim=True)
        p[f"lin{l}.weight_v"] = w
        p[f"lin{l}.bias"] = b
    return p


def init_color_params(conf: ColorConf, generator: Optional[torch.Generator] = None,
                      dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """nn.Linear default init (kaiming-uniform a=sqrt(5)) + weight_norm,
    models/fields.py:136-149."""
    p: Dict[str, torch.Tensor] = {}

    def lin(name, din, dout):
        bound = 1.0 / math.sqrt(din)
        w = (torch.rand(dout, din, dtype=dtype, generator=generator) * 2 - 1) * bound
        b = (torch.rand(dout, dtype=dtype, generator=generator) * 2 - 1) * bound
        p[f"{name}.weight_g"] = w.norm(dim=1, keepdim=True)
        p[f"{name}.weight_v"] = w
        p[f"{name}.bias"] = b

    dims = conf.layer_dims()
    for l, (din, dout) in enumerate(dims):
        lin(f"lin{l}", din, dout)
    if conf.extra_color:
        lin("extra_lin", dims[-1][0], conf.d_out)
    return p


def effective_weight(p: Dict[str, torch.Tensor], name: str) -> torch.Tensor:
    """torch.nn.utils.weight_norm(dim=0): W = g * v / ||v||_2 per output row
    (applied at models/fields.py:65-66,142-143,148-149).  Plain ``weight`` keys
    (weight_norm=False) are passed through."""
    if f"{name}.weight" in p:
        return p[f"{name}.weight"]
    v = p[f"{name}.weight_v"]
    g = p[f"{name}.weight_g"]
    return g * v / v.norm(dim=1, keepdim=True)


# --------------------------------------------------------------------------- networks
def positional_encode(x: torch.Tensor, multires: int) -> torch.Tensor:
    """[x, sin(2^k x), cos(2^k x)]_{k<multires}; models/embedder.py:11-36 with the
    kwargs of get_embedder (:39-51): include_input, log-sampled bands 2^0..2^(L-1)."""
    if multires <= 0:
        return x
    outs = [x]
    for k in range(multires):
        f = float(2 ** k)
        outs.append(torch.sin(x * f))
        outs.append(torch.cos(x * f))
    return torch.cat(outs, dim=-1)


def softplus100(x: torch.Tensor) -> torch.Tensor:
    """nn.Softplus(beta=100) with torch's default threshold=20 (models/fields.py:70)."""
    return F.softplus(x, beta=100.0, threshold=20.0)


def sdf_forward(p: Dict[str, torch.Tensor], conf: SDFConf, x: torch.Tensor) -> torch.Tensor:
    """SDFNetwork.forward, models/fields.py:72-88.  Returns [P, d_out] = [sdf/scale, feat]."""
    inputs = positional_encode(x * conf.scale, conf.multires)
    h = inputs
    n_lin = conf.n_lin
    for l in range(n_lin):
        if l in conf.skip_in:
            h = torch.cat([h, inputs], dim=1) / math.sqrt(2)
        h = F.linear(h, effective_weight(p, f"lin{l}"), p[f"lin{l}.bias"])
        if l < n_lin - 1:
            h = softplus100(h)
    return torch.cat([h[:, :1] / conf.scale, h[:, 1:]], dim=-1)


def sdf_value(p, conf: SDFConf, x):
    """SDFNetwork.sdf, models/fields.py:90-91."""
    return sdf_forward(p, conf, x)[:, :1]


def sdf_gradient(p, conf: SDFConf, x: torch.Tensor, create_graph: bool = True) -> torch.Tensor:
    """SDFNetwork.gradient, models/fields.py:96-107: d sdf / d x via autograd with a
    retained graph so that second-order terms flow into the parameters."""
    if not x.requires_grad:
        x = x.detach().requires_grad_(True)
    y = sdf_value(p, conf, x)
    (g,) = torch.autograd.grad(y, x, torch.ones_like(y), create_graph=create_graph,
                               retain_graph=True)
    return g


def color_forward(p, conf: ColorConf, points, normals, view_dirs, feats) -> torch.Tensor:
    """RenderingNetwork.forward, models/fields.py:154-185 (multires_view = 0 in every
    shipped conf; the embedded-view variant is restated for completeness)."""
    if conf.multires_view > 0:
        view_dirs = positional_encode(view_dirs, conf.multires_view)
    if conf.mode == "idr":
        h = torch.cat([points, view_dirs, normals, feats], dim=-1)
    elif conf.mode == "no_view_dir":
        h = torch.cat([points, normals, feats], dim=-1)
    elif conf.mode == "no_normal":
        h = torch.cat([points, view_dirs, feats], dim=-1)
    else:
        raise ValueError(conf.mode)
    n_lin = conf.n_lin
    extra = None
    for l in range(n_lin):
        h_in = h
        h = F.linear(h_in, effective_weight(p, f"lin{l}"), p[f"lin{l}.bias"])
        if l < n_lin - 1:
            h = torch.relu(h)
        if conf.extra_color and l == n_lin - 2:
            # the extra head taps the activation *after* the last hidden ReLU (:177-178)
            extra = F.linear(h, effective_weight(p, "extra_lin"), p["extra_lin.bias"])
    if conf.extra_color:
        h = torch.cat([h, extra], dim=-1)
    if conf.squeeze_out:
        h = torch.sigmoid(h)
    return h


def inv_s_from_variance(variance: torch.Tensor) -> torch.Tensor:
    """SingleVarianceNetwork.forward + clip, models/fields.py:275-276, renderer.py:234."""
    return torch.exp(variance * 10.0).clip(1e-6, 1e6)


# --------------------------------------------------------------------------- sampling
def sample_pdf_det(bins: torch.Tensor, weights: torch.Tensor, n: int) -> torch.Tensor:
    """Deterministic inverse-CDF sampling; models/renderer.py:39-69 with det=True."""
    weights = weights + 1e-5
    pdf = weights / weights.sum(-1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], -1)
    u = torch.linspace(0.5 / n, 1.0 - 0.5 / n, n, dtype=bins.dtype)
    u = u.expand(list(cdf.shape[:-1]) + [n]).contiguous()
    inds = torch.searchsorted(cdf, u, right=True)
    below = (inds - 1).clamp(min=0)
    above = inds.clamp(max=cdf.shape[-1] - 1)
    cdf_b, cdf_a = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    bin_b, bin_a = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    denom = cdf_a - cdf_b
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    t = (u - cdf_b) / denom
    return bin_b + t * (bin_a - bin_b)


def up_sample(rays_o, rays_d, z_vals, sdf, n_importance: int, inv_s: float) -> torch.Tensor:
    """NeuSRenderer.up_sample, models/renderer.py:133-177."""
    R, n = z_vals.shape
    pts = rays_o[:, None, :] + rays_d[:, None, :] * z_vals[..., None]
    radius = torch.linalg.norm(pts, ord=2, dim=-1)
    inside = (radius[:, :-1] < 1.0) | (radius[:, 1:] < 1.0)
    sdf = sdf.reshape(R, n)
    prev_sdf, next_sdf = sdf[:, :-1], sdf[:, 1:]
    prev_z, next_z = z_vals[:, :-1], z_vals[:, 1:]
    mid_sdf = (prev_sdf + next_sdf) * 0.5
    cos_val = (next_sdf - prev_sdf) / (next_z - prev_z + 1e-5)
    prev_cos = torch.cat([torch.zeros(R, 1, dtype=z_vals.dtype), cos_val[:, :-1]], dim=-1)
    cos_val = torch.minimum(prev_cos, cos_val)
    cos_val = cos_val.clip(-1e3, 0.0) * inside
    dist = next_z - prev_z
    prev_esti = mid_sdf - cos_val * dist * 0.5
    next_esti = mid_sdf + cos_val * dist * 0.5
    prev_cdf = torch.sigmoid(prev_esti * inv_s)
    next_cdf = torch.sigmoid(next_esti * inv_s)
    alpha = (prev_cdf - next_cdf + 1e-5) / (prev_cdf + 1e-5)
    trans = torch.cumprod(torch.cat([torch.ones(R, 1, dtype=z_vals.dtype), 1.0 - alpha + 1e-7], -1), -1)[:, :-1]
    weights = alpha * trans
    return sample_pdf_det(z_vals, weights, n_importance).detach()


def hierarchical_z(sdf_fn, rconf: RenderConf, rays_o, rays_d, near, far,
                   jitter: Optional[torch.Tensor]) -> torch.Tensor:
    """Sample placement of NeuSRenderer.render, models/renderer.py:302-352 (n_outside=0).

    ``jitter`` is the per-ray offset ``(u - 0.5)`` of :317-319 (shape [R,1]) or None
    for perturb = 0; the caller owns the RNG so both sides see identical draws.
    ``sdf_fn`` maps [P,3] points to [P,1] sdf values (sdf_network.sdf)."""
    R = rays_o.shape[0]
    n = rconf.n_samples
    z = torch.linspace(0.0, 1.0, n, dtype=rays_o.dtype)
    z = near + (far - near) * z[None, :]
    if jitter is not None:
        z = z + jitter * 2.0 / n
    if rconf.n_importance > 0:
        with torch.no_grad():
            pts = rays_o[:, None, :] + rays_d[:, None, :] * z[..., None]
            sdf = sdf_fn(pts.reshape(-1, 3)).reshape(R, n)
            per = rconf.n_importance // rconf.up_sample_steps
            for i in range(rconf.up_sample_steps):
                new_z = up_sample(rays_o, rays_d, z, sdf, per, 64 * 2 ** i)
                last = (i + 1 == rconf.up_sample_steps)
                # cat_z_vals, models/renderer.py:179-193
                cat = torch.cat([z, new_z], dim=-1)
                z_sorted, index = torch.sort(cat, dim=-1)
                if not last:
                    npts = rays_o[:, None, :] + rays_d[:, None, :] * new_z[..., None]
                    new_sdf = sdf_fn(npts.reshape(-1, 3)).reshape(R, per)
                    sdf = torch.gather(torch.cat([sdf, new_sdf], dim=-1), 1, index)
                z = z_sorted
    return z


# --------------------------------------------------------------------------- render core
def render_core(sdf_p, col_p, variance, sconf: SDFConf, cconf: ColorConf, rconf: RenderConf,
                rays_o, rays_d, z_vals, sample_dist: float,
                background_rgb=None, cos_anneal_ratio: float = 0.0):
    """NeuSRenderer.render_core, models/renderer.py:195-300, n_outside = 0."""
    R, S = z_vals.shape
    dists = z_vals[..., 1:] - z_vals[..., :-1]
    dists = torch.cat([dists, torch.full_like(dists[..., :1], sample_dist)], -1)
    mid_z = z_vals + dists * 0.5
    pts = (rays_o[:, None, :] + rays_d[:, None, :] * mid_z[..., None]).reshape(-1, 3)
    dirs = rays_d[:, None, :].expand(R, S, 3).reshape(-1, 3)

    pts = pts.detach().requires_grad_(True)   # models/fields.py:97 (x.requires_grad_(True))
    out = sdf_forward(sdf_p, sconf, pts)
    sdf, feat = out[:, :1], out[:, 1:]
    grads = sdf_gradient(sdf_p, sconf, pts, create_graph=True)

    raw = color_forward(col_p, cconf, pts, grads, dirs, feat)
    if rconf.extra_color:
        raw = raw.reshape(R, S, 6)
        sampled, extra_sampled = raw[..., :3], raw[..., 3:]
    else:
        sampled, extra_sampled = raw.reshape(R, S, 3), None

    inv_s = inv_s_from_variance(variance).reshape(1, 1).expand(R * S, 1)
    c = composite(sdf, grads, pts, sampled, extra_sampled, dists, inv_s, dirs, background_rgb, cos_anneal_ratio)
    return {
        "color": c["color"], "extra_color": c["extra_color"], "sdf": sdf, "dists": dists,
        "gradients": grads.reshape(R, S, 3), "s_val": 1.0 / inv_s, "mid_z_vals": mid_z,
        "weights": c["weights"], "cdf": c["cdf"], "gradient_error": c["gradient_error"],
        "inside_sphere": c["inside"],
    }


def composite(sdf, grads, pts, sampled, extra_sampled, dists, inv_s, dirs, background_rgb=None,
              cos_anneal_ratio: float = 0.0, relax_total=None):
    """The compositing of render_core, models/renderer.py:234-286, on per-sample tensors: sdf [P,1], grads / pts /
    dirs [P,3] (P = R*S, ray-major), sampled / extra_sampled [R,S,3] (extra_sampled None without extra_color), dists
    [R,S], inv_s broadcastable to [P,1].  ``relax_total`` replaces the eikonal normaliser relax.sum() (the product sums
    it over every chunk of a call).  Also returns the per-ray ``relax`` mask and the per-sample ``alpha``."""
    R, S = dists.shape
    true_cos = (dirs * grads).sum(-1, keepdim=True)
    iter_cos = -(F.relu(-true_cos * 0.5 + 0.5) * (1.0 - cos_anneal_ratio)
                 + F.relu(-true_cos) * cos_anneal_ratio)
    d = dists.reshape(-1, 1)
    est_next = sdf + iter_cos * d * 0.5
    est_prev = sdf - iter_cos * d * 0.5
    prev_cdf = torch.sigmoid(est_prev * inv_s)
    next_cdf = torch.sigmoid(est_next * inv_s)
    pp = prev_cdf - next_cdf
    cc = prev_cdf
    alpha = ((pp + 1e-5) / (cc + 1e-5)).reshape(R, S).clip(0.0, 1.0)

    pts_norm = torch.linalg.norm(pts, ord=2, dim=-1, keepdim=True).reshape(R, S)
    inside = (pts_norm < 1.0).to(dists.dtype).detach()
    relax = (pts_norm < 1.2).to(dists.dtype).detach()

    ones = torch.ones(R, 1, dtype=dists.dtype, device=dists.device)
    trans = torch.cumprod(torch.cat([ones, 1.0 - alpha + 1e-7], -1), -1)[:, :-1]
    weights = alpha * trans
    wsum = weights.sum(-1, keepdim=True)
    color = (sampled * weights[..., None]).sum(1)
    extra_color = (extra_sampled * weights[..., None]).sum(1) if extra_sampled is not None else None
    if background_rgb is not None:
        if extra_sampled is not None:
            extra_color = extra_color + background_rgb * (1.0 - wsum)
        else:
            color = color + background_rgb * (1.0 - wsum)

    gnorm = torch.linalg.norm(grads.reshape(R, S, 3), ord=2, dim=-1)
    den = relax.sum() if relax_total is None else relax_total
    gerr = (relax * (gnorm - 1.0) ** 2).sum() / (den + 1e-5)
    return {"color": color, "extra_color": extra_color, "weights": weights, "cdf": cc.reshape(R, S),
            "gradient_error": gerr, "inside": inside, "relax": relax, "alpha": alpha}


def render(sdf_p, col_p, variance, sconf: SDFConf, cconf: ColorConf, rconf: RenderConf,
           rays_o, rays_d, near, far, jitter=None, background_rgb=None,
           cos_anneal_ratio: float = 0.0, z_vals: Optional[torch.Tensor] = None):
    """NeuSRenderer.render, models/renderer.py:302-397 (n_outside = 0).  Returns the same
    11 keys.  ``jitter``: see hierarchical_z.  ``z_vals`` (test hook): skip the sample
    placement and composite on the given sorted depths -- the placement is discontinuous
    (bin searches, ``radius < 1`` masks), so two fp32 implementations can legitimately
    place a few samples differently; feeding identical depths isolates the smooth part."""
    R = rays_o.shape[0]
    sample_dist = 2.0 / rconf.n_samples
    if z_vals is None:
        z = hierarchical_z(lambda x: sdf_value(sdf_p, sconf, x), rconf, rays_o, rays_d, near, far, jitter)
    else:
        z = z_vals
    S = z.shape[1]
    ret = render_core(sdf_p, col_p, variance, sconf, cconf, rconf, rays_o, rays_d, z, sample_dist,
                      background_rgb=background_rgb, cos_anneal_ratio=cos_anneal_ratio)
    w = ret["weights"]
    return {
        "color_fine": ret["color"],
        "extra_color_fine": ret["extra_color"],
        "s_val": ret["s_val"].reshape(R, S).mean(-1, keepdim=True),
        "cdf_fine": ret["cdf"],
        "weight_sum": w.sum(-1, keepdim=True),
        "weight_max": w.max(-1, keepdim=True)[0],
        "gradients": ret["gradients"],
        "weights": w,
        "mid_z_vals": ret["mid_z_vals"],
        "gradient_error": ret["gradient_error"],
        "inside_sphere": ret["inside_sphere"],
        "z_vals": z,           # extra (not in the reference dict): the sorted sample depths
    }


# --------------------------------------------------------------------------- rays
def near_far_from_sphere(rays_o, rays_d):
    """SMPL_Dataset.near_far_from_sphere, models/dataset.py:331-342 (is_sphere=False):
    mid = -(o.d)/(d.d); near = max(mid-1, 0); far = mid+1."""
    a = (rays_d ** 2).sum(-1, keepdim=True)
    b = 2.0 * (rays_o * rays_d).sum(-1, keepdim=True)
    mid = 0.5 * (-b) / a
    near = (mid - 1.0).clamp(min=0.0)
    far = mid + 1.0
    return near, far
