"""CPU oracle (test infrastructure, never on the product path): CLIP ViT-B/32 text tower.

PARITY UNPINNED, like ``oracle.clip_vit``: the arithmetic lives in openai/CLIP (unpinned third-party dependency,
AvatarCLIP ``requirements.txt:12``); the reference only calls it (AvatarGen/AppearanceGen/main.py:274-288
``clip.tokenize`` + ``perceptor.encode_text``, detached).  This file restates the published architecture (openai/CLIP
``clip/model.py``: ``CLIP.encode_text``, ``build_attention_mask``, ``ResidualAttentionBlock``, ``QuickGELU``, fp32
``LayerNorm``) and ``oracle/pin_clip_text.py`` cross-checks it against HuggingFace ``transformers``
``CLIPTextModelWithProjection`` on seeded random weights.

State-dict keys follow openai/CLIP: token_embedding.weight [49408,512], positional_embedding [77,512],
transformer.resblocks.{i}.{ln_1,ln_2}.{weight,bias}, .attn.in_proj_{weight,bias}, .attn.out_proj.{weight,bias},
.mlp.c_fc.{weight,bias}, .mlp.c_proj.{weight,bias}, ln_final.{weight,bias}, text_projection [512,512].
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict

import torch
import torch.nn.functional as F

from .clip_vit import quick_gelu


@dataclass
class TextConf:
    context: int = 77
    vocab: int = 49408
    width: int = 512
    layers: int = 12
    heads: int = 8
    mlp: int = 2048
    out_dim: int = 512


def random_text_state(conf: TextConf = TextConf(), seed: int = 0, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Seeded random weights with openai/CLIP's initialisation scales (``CLIP.initialize_parameters``: token std 0.02,
    positional std 0.01, attention / projection / fc stds from the width and depth, text_projection std W^-0.5), small
    random biases and LayerNorm jitter like ``clip_vit.random_vit_state``, rounded to fp16 values and returned as
    ``dtype``."""
    g = torch.Generator().manual_seed(seed)
    W = conf.width
    rn = lambda *s, std=1.0: torch.randn(*s, generator=g) * std
    sd: Dict[str, torch.Tensor] = {"token_embedding.weight": rn(conf.vocab, W, std=0.02),
                                   "positional_embedding": rn(conf.context, W, std=0.01)}
    proj_std = (W ** -0.5) * ((2 * conf.layers) ** -0.5)
    attn_std = W ** -0.5
    fc_std = (2 * W) ** -0.5
    for i in range(conf.layers):
        p = f"transformer.resblocks.{i}."
        for ln in ("ln_1", "ln_2"):
            sd[p + ln + ".weight"] = 1.0 + 0.05 * rn(W)
            sd[p + ln + ".bias"] = 0.05 * rn(W)
        sd[p + "attn.in_proj_weight"] = rn(3 * W, W, std=attn_std)
        sd[p + "attn.in_proj_bias"] = 0.02 * rn(3 * W)
        sd[p + "attn.out_proj.weight"] = rn(W, W, std=proj_std)
        sd[p + "attn.out_proj.bias"] = 0.02 * rn(W)
        sd[p + "mlp.c_fc.weight"] = rn(conf.mlp, W, std=fc_std)
        sd[p + "mlp.c_fc.bias"] = 0.02 * rn(conf.mlp)
        sd[p + "mlp.c_proj.weight"] = rn(W, conf.mlp, std=proj_std)
        sd[p + "mlp.c_proj.bias"] = 0.02 * rn(W)
    sd["ln_final.weight"] = 1.0 + 0.05 * rn(W)
    sd["ln_final.bias"] = 0.05 * rn(W)
    sd["text_projection"] = rn(W, conf.out_dim, std=W ** -0.5)
    return {k: v.half().to(dtype) for k, v in sd.items()}


def encode_text(sd: Dict[str, torch.Tensor], tokens: torch.Tensor, conf: TextConf = TextConf()) -> torch.Tensor:
    """``CLIP.encode_text`` (openai/CLIP clip/model.py): tokens [B, context] -> [B, out_dim], fp32 throughout."""
    B, T = tokens.shape
    W, Hh = conf.width, conf.heads
    hd = W // Hh
    x = sd["token_embedding.weight"][tokens.long()] + sd["positional_embedding"]
    mask = torch.full((T, T), float("-inf")).triu_(1)                    # build_attention_mask
    for i in range(conf.layers):
        p = f"transformer.resblocks.{i}."
        h = F.layer_norm(x, (W,), sd[p + "ln_1.weight"], sd[p + "ln_1.bias"], 1e-5)
        q, k, v = F.linear(h, sd[p + "attn.in_proj_weight"], sd[p + "attn.in_proj_bias"]).chunk(3, dim=-1)
        sh = lambda t: t.reshape(B, T, Hh, hd).permute(0, 2, 1, 3)       # [B, heads, T, hd]
        q, k, v = sh(q), sh(k), sh(v)
        att = torch.softmax((q @ k.transpose(-1, -2)) / math.sqrt(hd) + mask, dim=-1)
        o = (att @ v).permute(0, 2, 1, 3).reshape(B, T, W)
        x = x + F.linear(o, sd[p + "attn.out_proj.weight"], sd[p + "attn.out_proj.bias"])
        h = F.layer_norm(x, (W,), sd[p + "ln_2.weight"], sd[p + "ln_2.bias"], 1e-5)
        h = quick_gelu(F.linear(h, sd[p + "mlp.c_fc.weight"], sd[p + "mlp.c_fc.bias"]))
        x = x + F.linear(h, sd[p + "mlp.c_proj.weight"], sd[p + "mlp.c_proj.bias"])
    x = F.layer_norm(x, (W,), sd["ln_final.weight"], sd["ln_final.bias"], 1e-5)
    return x[torch.arange(B), tokens.long().argmax(dim=-1)] @ sd["text_projection"]
