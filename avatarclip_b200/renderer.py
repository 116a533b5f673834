"""Host-side mirror of ``NeuSRenderer`` (AvatarGen/AppearanceGen/models/renderer.py:72-404).

Same constructor and ``render`` signature / returned dict as the reference; the computation is one
call into libavc_b200.so per direction (``avc_neus_render_fwd`` / ``avc_neus_render_bwd``) wrapped in a
``torch.autograd.Function`` so that ``loss.backward()`` and ``torch.optim.Adam`` in the reference's
``Runner`` keep working unmodified.  Parameters of the three networks are re-homed (once) into a
single flat fp32 vector whose layout is the C ABI's (include/avc_b200.h): that vector is what the
fused Adam and the multi-GPU gradient all-reduce operate on.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Tuple

import torch

from . import _lib
from ._lib import NeusCfg, NeusCotangents, NeusOutputs

_OUT_KEYS = ["color_fine", "extra_color_fine", "s_val", "cdf_fine", "weight_sum", "weight_max", "gradients",
             "weights", "mid_z_vals", "gradient_error", "inside_sphere"]
_NONDIFF = ("mid_z_vals", "inside_sphere", "z_vals")


def _skip_mask(skip_in) -> int:
    m = 0
    for s in skip_in:
        m |= 1 << int(s)
    return m


class FlatParams:
    """The flat parameter vector shared by the SDF, colour and variance modules."""

    def __init__(self, cfg: NeusCfg, sdf_network, deviation_network, color_network, device):
        L = _lib.lib()
        n = C.c_int64()
        _lib.check(L.avc_neus_param_count(C.byref(cfg), C.byref(n)), "avc_neus_param_count")
        self.n = int(n.value)
        self.cfg = cfg
        self.flat = torch.zeros(self.n, dtype=torch.float32, device=device)
        self.grad = torch.zeros(self.n, dtype=torch.float32, device=device)
        self.slots: List[Tuple[torch.nn.Parameter, int, int]] = []   # (param, offset, numel)

        def off(net, layer, which):
            o, m = C.c_int64(), C.c_int64()
            _lib.check(L.avc_neus_param_offset(C.byref(cfg), net, layer, which, C.byref(o), C.byref(m)),
                       "avc_neus_param_offset")
            return int(o.value), int(m.value)

        def bind(mod, net, layer):
            for which, name in ((0, "weight_g"), (1, "weight_v"), (2, "bias")):
                p = getattr(mod, name)
                o, m = off(net, layer, which)
                if p.numel() != m:
                    raise ValueError(f"parameter {name} of net {net} layer {layer}: {p.numel()} != {m}")
                self.slots.append((p, o, m))

        for l in range(cfg.sdf_n_layers + 1):
            bind(getattr(sdf_network, f"lin{l}"), 0, l)
        for l in range(cfg.col_n_layers + 1):
            bind(getattr(color_network, f"lin{l}"), 1, l)
        if getattr(color_network, "extra_color", True):
            bind(color_network.extra_lin, 2, 0)
        else:
            # RenderingNetwork(extra_color=False) has no second head (models/fields.py:147).  The kernels always evaluate
            # one: its slot holds the constant map W = g v / ||v|| = 0 (g = 0, v = 1, bias = 0); it is not a Parameter (not
            # trained, absent from state dicts), its output is dropped by NeuSRenderer.render and nothing back-propagates
            # into it (zero cotangent).
            o, m = off(2, 0, 1)
            self.flat[o:o + m] = 1.0
        o, m = off(3, 0, 0)
        self.slots.append((deviation_network.variance, o, m))
        self.rehome()

    def rehome(self):
        """Point every Parameter's storage at its slice of the flat vector (values preserved)."""
        with torch.no_grad():
            for p, o, m in self.slots:
                view = self.flat[o:o + m].view(p.shape)
                if p.data_ptr() != view.data_ptr():
                    view.copy_(p.data.to(self.flat.device, torch.float32))
                    p.data = view

    def is_homed(self) -> bool:
        base = self.flat.data_ptr()
        return all(p.data_ptr() == base + 4 * o for p, o, _ in self.slots)

    def params(self) -> List[torch.nn.Parameter]:
        return [p for p, _, _ in self.slots]

    def grad_views(self, grad: torch.Tensor):
        return [grad[o:o + m].view(p.shape) for p, o, m in self.slots]


def render_forward_raw(renderer, rays_o, rays_d, near, far, jitter, background, bg_kind, cos_anneal, z_in,
                       keep_ws: bool, out: Optional[Dict[str, torch.Tensor]] = None):
    """One avc_neus_render_fwd call.  Returns (outputs dict incl. z_vals, workspace, chunk)."""
    L = _lib.lib()
    fp: FlatParams = renderer._flat
    cfg = fp.cfg
    R = rays_o.shape[0]
    S = cfg.n_samples + cfg.n_importance
    dev = rays_o.device
    if out is None:
        f = dict(dtype=torch.float32, device=dev)
        out = {
            "color_fine": torch.empty(R, 3, **f), "extra_color_fine": torch.empty(R, 3, **f),
            "s_val": torch.empty(R, 1, **f), "cdf_fine": torch.empty(R, S, **f),
            "weight_sum": torch.empty(R, 1, **f), "weight_max": torch.empty(R, 1, **f),
            "gradients": torch.empty(R, S, 3, **f), "weights": torch.empty(R, S, **f),
            "mid_z_vals": torch.empty(R, S, **f), "gradient_error": torch.empty((), **f),
            "inside_sphere": torch.empty(R, S, **f), "z_vals": torch.empty(R, S, **f),
        }
    chunk = min(R, renderer.max_rays_per_chunk)
    ws = renderer._workspace(chunk, keep=keep_ws)
    o = NeusOutputs(**{k: out[k].data_ptr() for k in _lib._OUT_FIELDS})
    _lib.check(L.avc_neus_render_fwd(C.byref(cfg), _lib.ptr(fp.flat), _lib.ptr(rays_o), _lib.ptr(rays_d),
                                     _lib.ptr(near), _lib.ptr(far), _lib.ptr(jitter), _lib.ptr(background),
                                     bg_kind, _lib.ptr(z_in), float(cos_anneal), R, C.byref(o), _lib.ptr(ws),
                                     ws.numel(), chunk, _lib.stream_ptr()), "avc_neus_render_fwd")
    return out, ws, chunk


def render_backward_raw(renderer, rays_o, rays_d, background, bg_kind, cos_anneal, out, ws, chunk,
                        cot: Dict[str, Optional[torch.Tensor]], grad: Optional[torch.Tensor] = None, flags: int = 0):
    """One avc_neus_render_bwd call.  ``cot``: contiguous fp32 cotangents (missing / None = zero).
    Returns the flat parameter gradient."""
    L = _lib.lib()
    fp: FlatParams = renderer._flat
    c = NeusCotangents(**{k: (None if cot.get(k) is None else cot[k].data_ptr()) for k in _lib._COT_FIELDS})
    o = NeusOutputs(**{k: out[k].data_ptr() for k in _lib._OUT_FIELDS})
    if grad is None:
        grad = torch.empty_like(fp.flat)
    _lib.check(L.avc_neus_render_bwd(C.byref(fp.cfg), _lib.ptr(fp.flat), _lib.ptr(rays_o), _lib.ptr(rays_d),
                                     _lib.ptr(background), bg_kind, float(cos_anneal), rays_o.shape[0], C.byref(o),
                                     C.byref(c), _lib.ptr(grad), _lib.ptr(ws), ws.numel(), chunk, flags,
                                     _lib.stream_ptr()), "avc_neus_render_bwd")
    return grad


class _RenderFn(torch.autograd.Function):
    """Autograd seam.  ``hook`` is a dummy differentiable scalar that makes autograd call ``backward``; the
    parameter gradients are handed to the modules' Parameters directly as views of ONE flat gradient vector
    (accumulating into existing ``.grad`` like autograd would), so that neither 28 small copies nor 28
    AccumulateGrad nodes are needed per step."""

    @staticmethod
    def forward(ctx, renderer, hook, rays_o, rays_d, near, far, jitter, background, bg_kind, cos_anneal, z_in,
                need_grad):
        # ``need_grad`` is decided by the caller: inside Function.forward grad mode is always off.  With it the forward
        # stash lives in a workspace OWNED by this autograd node (a later render / sdf_query cannot overwrite it
        # before backward runs, e.g. when several views are accumulated before one backward()).
        out, ws, chunk = render_forward_raw(renderer, rays_o, rays_d, near, far, jitter, background, bg_kind,
                                            cos_anneal, z_in, keep_ws=need_grad)
        ctx.renderer, ctx.out, ctx.ws, ctx.chunk = renderer, out, ws, chunk
        ctx.rays = (rays_o, rays_d, background, bg_kind, float(cos_anneal))
        ctx.mark_non_differentiable(out["mid_z_vals"], out["inside_sphere"], out["z_vals"])
        return tuple(out[k] for k in _OUT_KEYS) + (out["z_vals"],)

    @staticmethod
    def backward(ctx, *gouts):
        renderer = ctx.renderer
        fp: FlatParams = renderer._flat
        rays_o, rays_d, background, bg_kind, cos_anneal = ctx.rays
        cot = {}
        for k, t in zip(_OUT_KEYS, gouts[:len(_OUT_KEYS)]):
            if k in _lib._COT_FIELDS and t is not None:
                cot[k] = t.contiguous().float()
        grad = render_backward_raw(renderer, rays_o, rays_d, background, bg_kind, cos_anneal, ctx.out, ctx.ws,
                                   ctx.chunk, cot)
        renderer.last_flat_grad = grad
        for p, view in zip(fp.params(), fp.grad_views(grad)):
            if p.requires_grad:
                p.grad = view if p.grad is None else p.grad + view
        ctx.ws = ctx.out = None                      # release the node-owned stash as soon as it was consumed
        return (None,) * 12


class NeuSRenderer:
    """Drop-in for models/renderer.py:72-404 (``n_outside`` must be 0 and ``nerf`` None, as in every
    shipped conf -- main.py:136; the reference's ``render_core_outside`` is dead code there).  ``extra_color`` True is the
    train_clip configuration (179 confs), False the NeuS pre-fit of confs/base_models/astrongman.conf."""

    def __init__(self, nerf, sdf_network, deviation_network, color_network, n_samples, n_importance, n_outside,
                 up_sample_steps, perturb, extra_color=False, engine: int = 0, max_rays_per_chunk: int = 4096,
                 color_products: Optional[int] = None, wgrad_products: Optional[int] = None):
        if n_outside != 0:
            raise NotImplementedError("n_outside > 0 (NeRF background) is not part of the AvatarCLIP hot path")
        if bool(extra_color) != bool(getattr(color_network, "extra_color", True)):
            raise ValueError("NeuSRenderer(extra_color=...) and RenderingNetwork(extra_color=...) must agree "
                             "(models/renderer.py:227-232 reshapes the colour net's output to 6 or 3 channels)")
        self.nerf = nerf
        self.sdf_network = sdf_network
        self.deviation_network = deviation_network
        self.color_network = color_network
        self.n_samples, self.n_importance, self.n_outside = int(n_samples), int(n_importance), int(n_outside)
        self.up_sample_steps, self.perturb, self.extra_color = int(up_sample_steps), perturb, bool(extra_color)
        self.max_rays_per_chunk = int(max_rays_per_chunk)
        self.cfg = NeusCfg(
            sdf_d_in=sdf_network.d_in, sdf_d_out=sdf_network.d_out, sdf_d_hidden=sdf_network.d_hidden,
            sdf_n_layers=sdf_network.n_layers, sdf_skip_mask=_skip_mask(sdf_network.skip_in),
            sdf_multires=sdf_network.multires, sdf_scale=sdf_network.scale,
            col_d_feature=color_network.d_feature, col_d_hidden=color_network.d_hidden,
            col_n_layers=color_network.n_layers,
            n_samples=self.n_samples, n_importance=self.n_importance, up_sample_steps=self.up_sample_steps,
            engine=int(engine),
            # tcgen05 engine: MMAs per product in the colour net; None -> AVC_COLOR_PRODUCTS (default 3 = split operands)
            color_products=int(os.environ.get("AVC_COLOR_PRODUCTS", "3") if color_products is None else color_products),
            # MMAs per product in the weight-gradient tiles; None -> AVC_WGRAD_PRODUCTS
            wgrad_products=int(os.environ.get("AVC_WGRAD_PRODUCTS", "3") if wgrad_products is None else wgrad_products))
        self._flat: Optional[FlatParams] = None
        self._hook = torch.zeros((), requires_grad=True)
        self._ws_cache: Dict[int, torch.Tensor] = {}
        self.last_flat_grad: Optional[torch.Tensor] = None
        sdf_network._avc_binding = self

    # ------------------------------------------------------------------ plumbing
    def _ensure_flat(self, device):
        if self._flat is None or self._flat.flat.device != device:
            self._flat = FlatParams(self.cfg, self.sdf_network, self.deviation_network, self.color_network, device)
        elif not self._flat.is_homed():
            self._flat.rehome()
        return self._flat

    def _make_hook(self, dev):
        self._hook = torch.zeros((), device=dev, requires_grad=True)
        return self._hook

    def flat_params(self, device=None) -> FlatParams:
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        return self._ensure_flat(device)

    def _workspace(self, chunk: int, keep: bool) -> torch.Tensor:
        size = C.c_size_t()
        _lib.check(_lib.lib().avc_neus_workspace_bytes(C.byref(self.cfg), chunk, C.byref(size)),
                   "avc_neus_workspace_bytes")
        dev = self._flat.flat.device
        if keep:     # owned by the autograd node until its backward ran
            return torch.empty(size.value, dtype=torch.uint8, device=dev)
        ws = self._ws_cache.get(chunk)
        if ws is None or ws.numel() < size.value or ws.device != dev:
            ws = torch.empty(size.value, dtype=torch.uint8, device=dev)
            self._ws_cache = {chunk: ws}
        return ws

    @staticmethod
    def _prep(t, shape=None):
        t = t.detach()
        if t.dtype != torch.float32:
            t = t.float()
        if shape is not None:
            t = t.reshape(shape)
        return t.contiguous()

    # ------------------------------------------------------------------ reference API
    def render(self, rays_o, rays_d, near, far, perturb_overwrite=-1, background_rgb=None, cos_anneal_ratio=0.0,
               jitter=None, z_vals=None):
        """models/renderer.py:302-397.  Extra keyword-only hooks (not in the reference): ``jitter`` injects
        the per-ray draw ``u - 0.5`` of :317-319; ``z_vals`` composites on given depths."""
        if not rays_o.is_cuda:
            raise _lib.AvcError("avatarclip_b200 has no CPU path: rays must live on a CUDA device")
        dev = rays_o.device
        fp = self._ensure_flat(dev)
        R = rays_o.shape[0]
        rays_o, rays_d = self._prep(rays_o, (R, 3)), self._prep(rays_d, (R, 3))
        near_t = self._prep(near, (R,)) if torch.is_tensor(near) else torch.full((R,), float(near), device=dev)
        far_t = self._prep(far, (R,)) if torch.is_tensor(far) else torch.full((R,), float(far), device=dev)
        perturb = self.perturb
        if perturb_overwrite >= 0:
            perturb = perturb_overwrite
        if jitter is not None:
            jit = self._prep(jitter, (R,))
        elif perturb > 0:
            jit = (torch.rand([R, 1], device=dev) - 0.5).reshape(R)           # renderer.py:317-319
        else:
            jit = None
        bg, bg_kind = None, 0
        if background_rgb is not None:
            bgt = self._prep(background_rgb)
            if bgt.numel() == 3:
                bg, bg_kind = bgt.reshape(3), 1
            elif bgt.numel() == R:
                bg, bg_kind = bgt.reshape(R), 2
            else:
                raise ValueError("background_rgb must be [1,3] or [R,1] (main.py:393-405)")
        color_bg = None
        if not self.extra_color and bg is not None:
            # renderer.py:277-281: without the extra head the fixed background goes onto `color` itself; the kernels put it
            # on the extra colour, so they run without one and the (differentiable) blend happens on their outputs
            color_bg, bg, bg_kind = (bg.reshape(1, 3) if bg_kind == 1 else bg.reshape(R, 1)), None, 0
        z_in = self._prep(z_vals, (R, self.n_samples + self.n_importance)) if z_vals is not None else None
        hook = self._hook if self._hook.device == dev else self._make_hook(dev)
        hook.requires_grad_(any(p.requires_grad for p in fp.params()))
        need_grad = bool(torch.is_grad_enabled() and hook.requires_grad)
        outs = _RenderFn.apply(self, hook, rays_o, rays_d, near_t, far_t, jit, bg, bg_kind, float(cos_anneal_ratio), z_in,
                               need_grad)
        ret = dict(zip(_OUT_KEYS, outs[:len(_OUT_KEYS)]))
        ret["z_vals"] = outs[-1]
        if not self.extra_color:                                           # renderer.py:272-281,379
            ret["extra_color_fine"] = None
            if color_bg is not None:
                ret["color_fine"] = ret["color_fine"] + color_bg * (1.0 - ret["weight_sum"])
        return ret

    def sdf_query(self, pts: torch.Tensor) -> torch.Tensor:
        """SDFNetwork.sdf (models/fields.py:90-91) on [P,3] points -> [P,1]."""
        if not pts.is_cuda:
            raise _lib.AvcError("avatarclip_b200 has no CPU path: points must live on a CUDA device")
        fp = self._ensure_flat(pts.device)
        pts = self._prep(pts, (-1, 3))
        P = pts.shape[0]
        out = torch.empty(P, 1, dtype=torch.float32, device=pts.device)
        chunk = max(1, min(self.max_rays_per_chunk, (P + self.cfg.n_samples + self.cfg.n_importance - 1)
                           // (self.cfg.n_samples + self.cfg.n_importance)))
        ws = self._workspace(chunk, keep=False)
        _lib.check(_lib.lib().avc_neus_sdf_query(C.byref(self.cfg), _lib.ptr(fp.flat), _lib.ptr(pts), P,
                                                 _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                   "avc_neus_sdf_query")
        return out

    def sdf_eval(self, pts: torch.Tensor, want_features: bool = True, want_gradient: bool = False):
        """SDFNetwork.forward (models/fields.py:72-88) and/or SDFNetwork.gradient (:96-107) on [P,3] points ->
        ([P, d_out] = (sdf, features) or None, [P,3] raw gradient or None).  Inference only (no autograd)."""
        if not pts.is_cuda:
            raise _lib.AvcError("avatarclip_b200 has no CPU path: points must live on a CUDA device")
        fp = self._ensure_flat(pts.device)
        pts = self._prep(pts, (-1, 3))
        P = pts.shape[0]
        S = self.cfg.n_samples + self.cfg.n_importance
        out = torch.empty(P, self.cfg.sdf_d_out, dtype=torch.float32, device=pts.device) if want_features else None
        grad = torch.empty(P, 3, dtype=torch.float32, device=pts.device) if want_gradient else None
        cfg0 = NeusCfg.from_buffer_copy(self.cfg)
        cfg0.engine = 0
        size = C.c_size_t()
        chunk = max(1, min(self.max_rays_per_chunk, (P + S - 1) // S))
        _lib.check(_lib.lib().avc_neus_workspace_bytes(C.byref(cfg0), chunk, C.byref(size)), "avc_neus_workspace_bytes")
        ws = torch.empty(size.value, dtype=torch.uint8, device=pts.device)
        _lib.check(_lib.lib().avc_neus_sdf_eval(C.byref(self.cfg), _lib.ptr(fp.flat), _lib.ptr(pts), P, _lib.ptr(out),
                                                _lib.ptr(grad), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                   "avc_neus_sdf_eval")
        return out, grad

    def extract_geometry(self, bound_min, bound_max, resolution, threshold=0.0):
        """models/renderer.py:399-404 (-> extract_geometry :27-36): the iso-surface {-sdf = threshold} of the
        resolution^3 grid over the bounding box.  Returns (vertices [V,3] float, triangles [T,3] int) as numpy arrays in
        world coordinates like the reference.  The reference triangulates with PyMCubes; here csrc/avc_mesh.cu runs
        marching tetrahedra on the device (same surface, different triangulation; normals point out of the body)."""
        import numpy as np
        L = _lib.lib()
        u = self.extract_fields(bound_min, bound_max, resolution).contiguous()
        dev = u.device
        N = int(resolution)
        counts = torch.empty((N - 1) ** 3, dtype=torch.int32, device=dev)
        _lib.check(L.avc_march_count(_lib.ptr(u), N, N, N, float(threshold), _lib.ptr(counts), _lib.stream_ptr()),
                   "avc_march_count")
        incl = torch.cumsum(counts, 0, dtype=torch.int64)
        T = int(incl[-1].item()) if incl.numel() else 0
        if T == 0:
            return np.zeros((0, 3), dtype=np.float64), np.zeros((0, 3), dtype=np.int64)
        if T > 2 ** 31 - 1:              # avc_march_emit's offsets are int32
            raise _lib.AvcError(f"extract_geometry: {T} triangles at resolution {N} exceed the int32 triangle offsets")
        offsets = (incl - counts).to(torch.int32)
        verts = torch.empty(T * 3, 3, dtype=torch.float32, device=dev)
        keys = torch.empty(T * 3, dtype=torch.int64, device=dev)
        _lib.check(L.avc_march_emit(_lib.ptr(u), N, N, N, float(threshold), _lib.ptr(offsets), _lib.ptr(verts),
                                    _lib.ptr(keys), _lib.stream_ptr()), "avc_march_emit")
        uniq, inv = torch.unique(keys, return_inverse=True)        # weld vertices on the same grid edge or grid point
        welded = torch.empty(uniq.numel(), 3, dtype=torch.float32, device=dev)
        welded[inv] = verts
        tri = inv.reshape(T, 3)
        good = (tri[:, 0] != tri[:, 1]) & (tri[:, 1] != tri[:, 2]) & (tri[:, 0] != tri[:, 2])   # collapsed on a grid point
        tri = tri[good]
        used = torch.zeros(uniq.numel(), dtype=torch.bool, device=dev)   # and the vertices only they referenced
        used[tri.reshape(-1)] = True
        welded = welded[used]
        tri = (torch.cumsum(used, 0) - 1)[tri]
        b_min = torch.as_tensor(np.asarray(bound_min, dtype=np.float32), device=dev)
        b_max = torch.as_tensor(np.asarray(bound_max, dtype=np.float32), device=dev)
        vertices = welded / (N - 1.0) * (b_max - b_min)[None, :] + b_min[None, :]          # renderer.py:33-35
        return vertices.double().cpu().numpy(), tri.cpu().numpy()

    def extract_fields(self, bound_min, bound_max, resolution):
        """models/renderer.py:10-25 with query_func = -sdf, evaluated in slabs on the device."""
        dev = self._flat.flat.device if self._flat is not None else torch.device("cuda")
        xs = torch.linspace(float(bound_min[0]), float(bound_max[0]), resolution, device=dev)
        ys = torch.linspace(float(bound_min[1]), float(bound_max[1]), resolution, device=dev)
        zs = torch.linspace(float(bound_min[2]), float(bound_max[2]), resolution, device=dev)
        u = torch.empty(resolution, resolution, resolution, dtype=torch.float32, device=dev)
        step = max(1, (1 << 22) // (resolution * resolution))
        for i in range(0, resolution, step):
            xx, yy, zz = torch.meshgrid(xs[i:i + step], ys, zs, indexing="ij")
            pts = torch.stack([xx, yy, zz], -1).reshape(-1, 3)
            u[i:i + step] = -self.sdf_query(pts).reshape(xx.shape)
        return u
