"""Host-side wrapper of the CLIP ViT-B/32 text tower kernel (libavc_b200.so, ``avc_clip_encode_text``) and the reader of
openai's ``ViT-B-32.pt``.

Replaces ``perceptor.encode_text(clip.tokenize([prompt]))`` of AvatarGen/AppearanceGen/main.py:273-288 (openai/CLIP
``CLIP.encode_text``): ``ClipTextTower(text_state_dict).encode_text(tokens[B,77]) -> [B,512]``, forward only (the
reference detaches the result).  Tokens come from ``clip_tokenizer.ClipTokenizer``.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Tuple

import torch

from . import _lib
from .clip_vit import MAX_LAYERS, ClipLayerW, WeightPacker

TEXT_PREFIXES = ("token_embedding.weight", "positional_embedding", "transformer.", "ln_final.", "text_projection")


class ClipTextCfg(C.Structure):
    _fields_ = [("context", C.c_int32), ("vocab", C.c_int32), ("width", C.c_int32), ("layers", C.c_int32),
                ("heads", C.c_int32), ("mlp", C.c_int32), ("out_dim", C.c_int32)]


class ClipTextW(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("token_emb", "pos", "ln_final_g", "ln_final_b", "proj")] + \
               [("layer", ClipLayerW * MAX_LAYERS)]


def _bind(L):
    if getattr(L, "_clip_text_bound", False):
        return
    vp, i32, sz = C.c_void_p, C.c_int32, C.c_size_t
    P = C.POINTER
    L.avc_clip_text_workspace_bytes.argtypes = [P(ClipTextCfg), i32, P(sz)]
    L.avc_clip_encode_text.argtypes = [P(ClipTextCfg), P(ClipTextW), vp, i32, vp, vp, sz, vp]
    L.avc_clip_text_workspace_bytes.restype = L.avc_clip_encode_text.restype = C.c_int
    L._clip_text_bound = True


def load_clip_model(path: str) -> Tuple[Dict[str, torch.Tensor], Dict[str, torch.Tensor]]:
    """Read an openai/CLIP checkpoint the way ``clip.load(..., jit=False)`` does: as a TorchScript archive (openai's
    ``ViT-B-32.pt``), else as a plain ``torch.save``d state dict.  Returns ``(visual, text)``: the ``visual.*`` tensors
    (prefix kept; ``ClipImageTower`` strips it) and the text tower's tensors (token / positional embedding,
    ``transformer.*``, ``ln_final.*``, ``text_projection``).  Other keys (``logit_scale``, ...) are dropped."""
    try:
        sd = torch.jit.load(path, map_location="cpu").state_dict()
    except RuntimeError:
        sd = torch.load(path, map_location="cpu")
    visual = {k: v for k, v in sd.items() if k.startswith("visual.")}
    text = {k: v for k, v in sd.items() if k.startswith(TEXT_PREFIXES)}
    return visual, text


class ClipTextTower:
    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda"):
        L = _lib.lib()
        _bind(L)
        sd = state_dict
        dev = torch.device(device)
        vocab, width = sd["token_embedding.weight"].shape
        layers = len({k.split(".")[2] for k in sd if k.startswith("transformer.resblocks.")})
        self.cfg = ClipTextCfg(context=sd["positional_embedding"].shape[0], vocab=vocab, width=width, layers=layers,
                               heads=width // 64, mlp=sd["transformer.resblocks.0.mlp.c_fc.weight"].shape[0],
                               out_dim=sd["text_projection"].shape[1])
        self.device = dev
        pk = WeightPacker(dev)
        self._keep = pk.keep
        self.w = ClipTextW()
        # fp16-valued (as clip.load keeps them), stored fp32
        self.w.token_emb = pk.f32(sd["token_embedding.weight"].half())
        self.w.pos = pk.f32(sd["positional_embedding"].half())
        self.w.proj = pk.f32(sd["text_projection"].half())
        self.w.ln_final_g, self.w.ln_final_b = pk.f32(sd["ln_final.weight"]), pk.f32(sd["ln_final.bias"])
        for i in range(layers):
            pk.layer(self.w.layer[i], sd, f"transformer.resblocks.{i}.", transposed=False)

    @property
    def context(self) -> int:
        return self.cfg.context

    def encode_text(self, tokens: torch.Tensor) -> torch.Tensor:
        """perceptor.encode_text (main.py:276): tokens [B, context] (``ClipTokenizer.tokenize``) -> [B, out_dim] fp32."""
        if self.device.type != "cuda":
            raise _lib.AvcError("avatarclip_b200 has no CPU path")
        if tokens.dim() != 2 or tokens.shape[1] != self.cfg.context:
            raise _lib.AvcError(f"encode_text: tokens must be [B, {self.cfg.context}], got {tuple(tokens.shape)}")
        tok = tokens.to(self.device, torch.int32).contiguous()
        lo, hi = int(tok.min()), int(tok.max())
        if lo < 0 or hi >= self.cfg.vocab:
            raise _lib.AvcError(f"encode_text: token ids must lie in [0, {self.cfg.vocab}), got [{lo}, {hi}]")
        L = _lib.lib()
        B = tok.shape[0]
        size = C.c_size_t()
        _lib.check(L.avc_clip_text_workspace_bytes(C.byref(self.cfg), B, C.byref(size)), "avc_clip_text_workspace_bytes")
        ws = torch.empty(size.value, dtype=torch.uint8, device=self.device)
        emb = torch.empty(B, self.cfg.out_dim, dtype=torch.float32, device=self.device)
        _lib.check(L.avc_clip_encode_text(C.byref(self.cfg), C.byref(self.w), _lib.ptr(tok), B, _lib.ptr(emb),
                                          _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "avc_clip_encode_text")
        return emb
