"""CPU oracle (test infrastructure / timed CPU baseline, never on the product path): one full
appearance-optimisation step of ``Runner.train_clip`` (AvatarGen/AppearanceGen/main.py:345-566) assembled from
the restated pieces -- render (oracle.neus), shading + losses (oracle.loss), CLIP tower (oracle.clip_vit),
``loss.backward()`` via autograd and ``torch.optim.Adam`` (main.py:145,536-538) -- exactly the work the
reference does per step on one device, in fp32 on the host cores.

The view is passed in as plain CPU tensors (fields of ``avatarclip_b200.workload.HostView``); this module does
not import the product package.
"""
from __future__ import annotations

from typing import Dict

import torch

from . import clip_vit, loss as oloss, neus


class OracleTrainer:
    def __init__(self, sconf: neus.SDFConf, cconf: neus.ColorConf, rconf: neus.RenderConf,
                 sdf_state: Dict[str, torch.Tensor], col_state: Dict[str, torch.Tensor], variance: float,
                 clip_state: Dict[str, torch.Tensor], text_emb: torch.Tensor, lr: float = 5e-4,
                 igr_weight: float = 0.1, mask_weight: float = 0.5, clip_weight: float = 1.0,
                 dtype=torch.float32, clip_conf: clip_vit.ViTConf = None, add_no_texture: bool = True,
                 texture_cast_light: bool = True):
        self.add_no_texture, self.texture_cast_light = add_no_texture, texture_cast_light     # main.py:509-534
        self.sconf, self.cconf, self.rconf = sconf, cconf, rconf
        self.clip_conf = clip_conf if clip_conf is not None else clip_vit.ViTConf()
        self.dtype = dtype
        self.sp = {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in sdf_state.items()}
        self.cp = {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in col_state.items()}
        self.var = torch.tensor(float(variance), dtype=dtype, requires_grad=True)
        self.clip_state = {k: v.to(dtype) for k, v in clip_state.items()}
        self.text = text_emb.to(dtype).reshape(-1, text_emb.shape[-1])
        if self.text.shape[0] == 1:
            self.text = self.text.expand(2, -1)
        self.w = (igr_weight, mask_weight, clip_weight)
        self.params = list(self.sp.values()) + list(self.cp.values()) + [self.var]
        self.opt = torch.optim.Adam(self.params, lr=lr)

    def named_params(self):
        return ([("sdf." + k, v) for k, v in self.sp.items()] + [("col." + k, v) for k, v in self.cp.items()]
                + [("var.variance", self.var)])

    def loss(self, view, cos_anneal: float = 1.0, use_jitter: bool = True, z_vals=None):
        """``z_vals`` (test hook, see ``neus.render``): composite on these sorted depths instead of placing samples."""
        dt = self.dtype
        igr, mw, cw = self.w
        o, d = view.rays_o.to(dt), view.rays_d.to(dt)
        near, far = view.near.to(dt).reshape(-1, 1), view.far.to(dt).reshape(-1, 1)
        jit = view.jitter.to(dt).reshape(-1, 1) if use_jitter else None
        if view.bg_choice == 0:
            bg = torch.ones(1, 3, dtype=dt)
        elif view.bg_choice in (1, 2):
            bg = view.ray_background.to(dt).reshape(-1, 1)
        else:
            bg = None
        out = neus.render(self.sp, self.cp, self.var, self.sconf, self.cconf, self.rconf, o, d, near, far,
                          jitter=jit, background_rgb=bg, cos_anneal_ratio=cos_anneal,
                          z_vals=None if z_vals is None else z_vals.to(dt))
        H, W = view.H, view.W
        dm = view.in_mask.reshape(H, W).bool()
        cbg = None if view.canvas_background is None else view.canvas_background.to(dt).reshape(-1, 1)
        stage = oloss.shading_and_losses(out, dm, H, W, view.true_rgb.to(dt), view.mask.to(dt).reshape(-1, 1),
                                         torch.as_tensor(view.light_dir, dtype=dt), view.ambience,
                                         background_choice=view.bg_choice, background_rgb=cbg,
                                         igr_weight=igr, mask_weight=mw, add_no_texture=self.add_no_texture,
                                         texture_cast_light=self.texture_cast_light)
        cos_t = clip_vit.clip_cosine(self.clip_state, stage["texture_canvas"], self.text[0], self.clip_conf)
        cos_s = clip_vit.clip_cosine(self.clip_state, stage["shading_canvas"], self.text[1], self.clip_conf) \
            if self.add_no_texture else None
        total = oloss.total_loss(stage, cos_t, cos_s, cw)
        return total, {"out": out, "stage": stage, "cos": torch.stack([cos_t, cos_s] if cos_s is not None else [cos_t])}

    def step(self, view, cos_anneal: float = 1.0):
        """zero_grad / backward / Adam.step (main.py:536-538).  Returns (loss, aux)."""
        total, aux = self.loss(view, cos_anneal)
        self.opt.zero_grad()
        total.backward()
        self.opt.step()
        return total.detach(), aux
