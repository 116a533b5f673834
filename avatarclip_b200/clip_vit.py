"""Host-side wrapper of the CLIP ViT-B/32 image tower kernels (libavc_b200.so, ``avc_clip_*``).

Drop-in for the two things the reference does with ``perceptor`` after ``clip.load('ViT-B/32')``
(AvatarGen/AppearanceGen/main.py:259-261,509-526):

* ``encode_image(img[B,3,224,224]) -> [B,512]``  (differentiable w.r.t. the image; weights frozen)
* the fused ``resize -> Normalize -> encode_image -> cosine(text)`` used by ``train_clip``:
  ``cosine(canvas[B,H,W,3], text_emb[B,512]) -> [B]``.

Weights come from an openai/CLIP state dict (``model.visual.state_dict()`` or ``ViT-B-32.pt``; keys with or
without the ``visual.`` prefix).  They are packed once: fp16 matrices (what ``clip.load`` keeps on CUDA) plus
transposed copies for the input-gradient GEMMs, fp32 LayerNorm / bias / embedding vectors.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import torch

from . import _lib

MAX_LAYERS = 24


class ClipCfg(C.Structure):
    _fields_ = [("image_size", C.c_int32), ("patch", C.c_int32), ("width", C.c_int32), ("layers", C.c_int32),
                ("heads", C.c_int32), ("mlp", C.c_int32), ("out_dim", C.c_int32)]


class ClipLayerW(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in
                ("ln1_g", "ln1_b", "ln2_g", "ln2_b", "w_qkv", "w_qkv_t", "b_qkv", "w_out", "w_out_t", "b_out",
                 "w_fc", "w_fc_t", "b_fc", "w_proj", "w_proj_t", "b_proj")]


class ClipW(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in
                ("w_patch", "w_patch_t", "cls", "pos", "ln_pre_g", "ln_pre_b", "ln_post_g", "ln_post_b", "proj")] + \
               [("layer", ClipLayerW * MAX_LAYERS)]


def _bind(L):
    if getattr(L, "_clip_bound", False):
        return
    vp, i32, sz = C.c_void_p, C.c_int32, C.c_size_t
    P = C.POINTER
    L.avc_clip_workspace_bytes.argtypes = [P(ClipCfg), i32, P(sz)]
    L.avc_clip_loss_fwd.argtypes = [P(ClipCfg), P(ClipW), vp, i32, i32, i32, i32, vp, vp, vp, vp, sz, vp]
    L.avc_clip_loss_bwd.argtypes = [P(ClipCfg), P(ClipW), i32, i32, i32, i32, vp, vp, vp, vp, vp, sz, vp]
    for n in ("avc_clip_workspace_bytes", "avc_clip_loss_fwd", "avc_clip_loss_bwd"):
        getattr(L, n).restype = C.c_int
    L._clip_bound = True


class _ClipFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tower, x, text, mode):
        L = _lib.lib()
        B = x.shape[0]
        H, W = (x.shape[1], x.shape[2]) if mode == 0 else (x.shape[2], x.shape[3])
        ws = tower._workspace(B)
        emb = torch.empty(B, tower.cfg.out_dim, dtype=torch.float32, device=x.device)
        cos = torch.empty(B, dtype=torch.float32, device=x.device)
        _lib.check(L.avc_clip_loss_fwd(C.byref(tower.cfg), C.byref(tower.w), _lib.ptr(x), H, W, B, mode,
                                       _lib.ptr(text), _lib.ptr(emb), _lib.ptr(cos), _lib.ptr(ws), ws.numel(),
                                       _lib.stream_ptr()), "avc_clip_loss_fwd")
        ctx.tower, ctx.ws, ctx.mode, ctx.shape = tower, ws, mode, tuple(x.shape)
        ctx.text = text
        return emb, cos

    @staticmethod
    def backward(ctx, g_emb, g_cos):
        L = _lib.lib()
        tower = ctx.tower
        B = ctx.shape[0]
        H, W = (ctx.shape[1], ctx.shape[2]) if ctx.mode == 0 else (ctx.shape[2], ctx.shape[3])
        ge = g_emb.contiguous().float() if g_emb is not None else None
        gc = g_cos.contiguous().float() if g_cos is not None else None
        dx = torch.empty(ctx.shape, dtype=torch.float32, device=ctx.text.device)
        _lib.check(L.avc_clip_loss_bwd(C.byref(tower.cfg), C.byref(tower.w), H, W, B, ctx.mode, _lib.ptr(ctx.text),
                                       _lib.ptr(gc), _lib.ptr(ge), _lib.ptr(dx), _lib.ptr(ctx.ws), ctx.ws.numel(),
                                       _lib.stream_ptr()), "avc_clip_loss_bwd")
        return None, dx, None, None


class WeightPacker:
    """Device copies of frozen weights for the library's weight structs: fp16 GEMM matrices (what ``clip.load`` keeps on
    CUDA) and fp32 vectors.  ``keep`` holds the tensors alive as long as the raw pointers are in use."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.keep = []

    def h16(self, t: torch.Tensor) -> int:
        t = t.detach().to(self.device, torch.float16).contiguous()
        self.keep.append(t)
        return t.data_ptr()

    def f32(self, t: torch.Tensor) -> int:
        t = t.detach().to(self.device, torch.float32).contiguous()
        self.keep.append(t)
        return t.data_ptr()

    def layer(self, lw: ClipLayerW, sd: Dict[str, torch.Tensor], p: str, transposed: bool):
        """One residual block ``p`` = "transformer.resblocks.{i}." into ``lw``; the transposed copies (input-gradient
        GEMMs) only when ``transposed``, else their pointers stay NULL."""
        h16, f32 = self.h16, self.f32
        lw.ln1_g, lw.ln1_b = f32(sd[p + "ln_1.weight"]), f32(sd[p + "ln_1.bias"])
        lw.ln2_g, lw.ln2_b = f32(sd[p + "ln_2.weight"]), f32(sd[p + "ln_2.bias"])
        for name, key in (("qkv", "attn.in_proj_weight"), ("out", "attn.out_proj.weight"),
                          ("fc", "mlp.c_fc.weight"), ("proj", "mlp.c_proj.weight")):
            setattr(lw, "w_" + name, h16(sd[p + key]))
            if transposed:
                setattr(lw, "w_" + name + "_t", h16(sd[p + key].t()))
        lw.b_qkv, lw.b_out = f32(sd[p + "attn.in_proj_bias"]), f32(sd[p + "attn.out_proj.bias"])
        lw.b_fc, lw.b_proj = f32(sd[p + "mlp.c_fc.bias"]), f32(sd[p + "mlp.c_proj.bias"])


class ClipImageTower:
    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", heads: int = None):
        L = _lib.lib()
        _bind(L)
        sd = {(k[len("visual."):] if k.startswith("visual.") else k): v for k, v in state_dict.items()}
        dev = torch.device(device)
        conv = sd["conv1.weight"]
        width, _, patch, _ = conv.shape
        tokens = sd["positional_embedding"].shape[0]
        grid = int(round((tokens - 1) ** 0.5))
        layers = len({k.split(".")[2] for k in sd if k.startswith("transformer.resblocks.")})
        mlp = sd["transformer.resblocks.0.mlp.c_fc.weight"].shape[0]
        out_dim = sd["proj"].shape[1]
        heads = heads or width // 64
        self.cfg = ClipCfg(image_size=grid * patch, patch=patch, width=width, layers=layers, heads=heads, mlp=mlp,
                           out_dim=out_dim)
        self.device = dev
        pk = WeightPacker(dev)
        self._keep = pk.keep
        self.w = ClipW()
        h16, f32 = pk.h16, pk.f32
        wp = conv.reshape(width, -1)
        self.w.w_patch, self.w.w_patch_t = h16(wp), h16(wp.t())
        self.w.cls, self.w.pos = f32(sd["class_embedding"]), f32(sd["positional_embedding"])
        self.w.ln_pre_g, self.w.ln_pre_b = f32(sd["ln_pre.weight"]), f32(sd["ln_pre.bias"])
        self.w.ln_post_g, self.w.ln_post_b = f32(sd["ln_post.weight"]), f32(sd["ln_post.bias"])
        self.w.proj = f32(sd["proj"].half())     # fp16-valued (as clip.load keeps it), stored fp32
        for i in range(layers):
            pk.layer(self.w.layer[i], sd, f"transformer.resblocks.{i}.", transposed=True)
        self._zero_text = None

    def _workspace(self, B: int) -> torch.Tensor:
        size = C.c_size_t()
        _lib.check(_lib.lib().avc_clip_workspace_bytes(C.byref(self.cfg), B, C.byref(size)), "avc_clip_workspace_bytes")
        return torch.empty(size.value, dtype=torch.uint8, device=self.device)

    # ------------------------------------------------------------------ reference-facing API
    def encode_image(self, image: torch.Tensor) -> torch.Tensor:
        """perceptor.encode_image (main.py:512): image [B,3,S,S] already normalised -> [B,out_dim]."""
        if not image.is_cuda:
            raise _lib.AvcError("avatarclip_b200 has no CPU path")
        B = image.shape[0]
        text = torch.ones(B, self.cfg.out_dim, dtype=torch.float32, device=image.device)
        emb, _ = _ClipFn.apply(self, image.contiguous().float(), text, 1)
        return emb

    def cosine(self, canvas: torch.Tensor, text_emb: torch.Tensor) -> torch.Tensor:
        """main.py:509-514 fused: canvas [B,H,W,3] in [0,1] -> resize 224 -> Normalize -> encode_image ->
        cosine with text_emb [B,out_dim] (or [out_dim], broadcast) -> [B]."""
        if not canvas.is_cuda:
            raise _lib.AvcError("avatarclip_b200 has no CPU path")
        B = canvas.shape[0]
        text = text_emb.detach().float().reshape(-1, self.cfg.out_dim)
        if text.shape[0] == 1 and B > 1:
            text = text.expand(B, -1)
        text = text.contiguous().to(canvas.device)
        _, cos = _ClipFn.apply(self, canvas.contiguous().float(), text, 0)
        return cos
