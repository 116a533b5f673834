"""CPU oracle (test infrastructure, never on the product path): AvatarAnimate's motion stage (models/motion_generation.py)
restated in torch on the CPU, in fp64 by default -- the VPoser encoder, MotionInterpolation's latent interpolation, the
motion VAE's transformer decoder, the rotation chain (pytorch3d's rotation_6d_to_matrix, matrix_to_quaternion,
quaternion_to_axis_angle, axis_angle_to_matrix, matrix_to_rotation_6d, restated from their published algorithms),
MotionOptimizer's loss without the CLIP term and its Adam loop -- plus the seeded synthetic weights the tests and
oracle/pin_motion.py share.  Written with torch ops so that autograd gives the gradients the tests compare against.

PARITY UNPINNED for the VPoser encoder, as for the decoder (oracle/animate.py): ``human_body_prior`` is absent.
Restated from its published model: ``encoder_net`` = BatchFlatten, BatchNorm1d(63), Linear(63, 512), LeakyReLU(0.01),
BatchNorm1d(512), Dropout, Linear(512, 512), Linear(512, 512), NormalDistDecoder (``.mean`` = its ``mu`` Linear),
in eval mode (running statistics, eps 1e-5).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import animate as OA

ENCODER_SEED = 31
MOTION_VAE_SEED = 32
N_JOINTS = 21


def _t(x, dtype=torch.float64) -> torch.Tensor:
    return torch.as_tensor(x).detach().to(dtype)


# ---------------------------------------------------------------- VPoser encoder
def vposer_encoder_state(seed: int = ENCODER_SEED, n_in: int = 63, hidden: int = 512, latent: int = 32) -> dict:
    """encoder_net weights (nn.Linear / BatchNorm1d layouts) giving latents of about unit spread for poses of about
    0.3 rad."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, std: torch.randn(*s, generator=g) * std
    sd = {}
    for i, n in ((1, n_in), (4, hidden)):
        sd[f"encoder_net.{i}.weight"] = 1.0 + rn(n, std=0.1)
        sd[f"encoder_net.{i}.bias"] = rn(n, std=0.1)
        sd[f"encoder_net.{i}.running_mean"] = rn(n, std=0.1 if i == 1 else 0.2)
        sd[f"encoder_net.{i}.running_var"] = (0.3 if i == 1 else 0.5) + torch.rand(n, generator=g) * 0.2
    sd["encoder_net.2.weight"] = rn(hidden, n_in, std=1 / math.sqrt(n_in))
    sd["encoder_net.2.bias"] = rn(hidden, std=0.1)
    for i in (6, 7):
        sd[f"encoder_net.{i}.weight"] = rn(hidden, hidden, std=1 / math.sqrt(hidden))
        sd[f"encoder_net.{i}.bias"] = rn(hidden, std=0.05)
    sd["encoder_net.8.mu.weight"] = rn(latent, hidden, std=1 / math.sqrt(hidden))
    sd["encoder_net.8.mu.bias"] = rn(latent, std=0.05)
    sd["encoder_net.8.logvar.weight"] = rn(latent, hidden, std=1 / math.sqrt(hidden))
    sd["encoder_net.8.logvar.bias"] = rn(latent, std=0.05)
    return sd


def vposer_encode(x, sd, dtype=torch.float64) -> torch.Tensor:
    """VPoser.encode(x).mean, eval mode."""
    g = lambda k: _t(sd[f"encoder_net.{k}"], dtype)
    bn = lambda h, i: (h - g(f"{i}.running_mean")) / torch.sqrt(g(f"{i}.running_var") + 1e-5) * g(f"{i}.weight") + \
        g(f"{i}.bias")
    h = bn(_t(x, dtype).reshape(len(x), -1), 1)
    h = torch.nn.functional.leaky_relu(h @ g("2.weight").T + g("2.bias"), 0.01)
    h = bn(h, 4)
    h = h @ g("6.weight").T + g("6.bias")
    h = h @ g("7.weight").T + g("7.bias")
    return h @ g("8.mu.weight").T + g("8.mu.bias")


def interpolate(latents, anchor_position, num_frame: int, dtype=torch.float64) -> torch.Tensor:
    """MotionInterpolation's sequential accumulation latent[s + j + 1] = latent[s + j] + (end - start) / interval."""
    lat = _t(latents, dtype)
    out = torch.zeros(num_frame, lat.shape[1], dtype=dtype)
    out[0] = lat[0]
    for i in range(1, len(anchor_position)):
        s, e = anchor_position[i - 1], anchor_position[i]
        delta = (lat[i] - lat[i - 1]) / (e - s)
        for j in range(e - s):
            out[s + j + 1] = out[s + j] + delta
    return out


def interpolation_motion(poses, enc_sd, dec_sd, anchor_position=(0, 14, 29, 44, 59), num_frame: int = 60) -> np.ndarray:
    """MotionInterpolation.get_motion in fp64 -> [num_frame, 63]."""
    z = interpolate(vposer_encode(_t(poses)[:, :63], enc_sd), anchor_position, num_frame)
    return OA.vposer_decode(z.numpy(), dec_sd)[0].reshape(num_frame, 63)


# ---------------------------------------------------------------- rotation chain
def rotation_6d_to_matrix(d6: torch.Tensor) -> torch.Tensor:
    """Gram-Schmidt of the two 3-vectors (first three values, last three); the rows of the result are b1, b2, b3."""
    b1 = torch.nn.functional.normalize(d6[..., :3], dim=-1)
    a2 = d6[..., 3:]
    b2 = torch.nn.functional.normalize(a2 - (b1 * a2).sum(-1, keepdim=True) * b1, dim=-1)
    return torch.stack((b1, b2, torch.cross(b1, b2, dim=-1)), dim=-2)


def _sqrt_pos(x: torch.Tensor) -> torch.Tensor:
    """sqrt(max(0, x)) with a zero subgradient at x <= 0."""
    out = torch.zeros_like(x)
    pos = x > 0
    out[pos] = torch.sqrt(x[pos])
    return out


def matrix_to_quaternion(m: torch.Tensor) -> torch.Tensor:
    """The four candidate quaternions (r, i, j, k), each scaled by its own denominator 2 max(|q_c|, 0.1); the one
    whose |q_c| is largest (the first of equal ones) is returned."""
    e = [m[..., i, j] for i in range(3) for j in range(3)]
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = e
    qa = _sqrt_pos(torch.stack([1 + m00 + m11 + m22, 1 + m00 - m11 - m22, 1 - m00 + m11 - m22, 1 - m00 - m11 + m22], -1))
    cand = torch.stack([
        torch.stack([qa[..., 0] ** 2, m21 - m12, m02 - m20, m10 - m01], -1),
        torch.stack([m21 - m12, qa[..., 1] ** 2, m10 + m01, m02 + m20], -1),
        torch.stack([m02 - m20, m10 + m01, qa[..., 2] ** 2, m12 + m21], -1),
        torch.stack([m10 - m01, m20 + m02, m21 + m12, qa[..., 3] ** 2], -1)], -2)
    cand = cand / (2.0 * torch.maximum(qa[..., None], torch.tensor(0.1, dtype=qa.dtype)))
    idx = qa.argmax(-1)
    return torch.gather(cand, -2, idx[..., None, None].expand(*idx.shape, 1, 4)).squeeze(-2)


def _sin_half_over_angle(angles: torch.Tensor, half: torch.Tensor) -> torch.Tensor:
    small = angles.abs() < 1e-6
    safe = torch.where(small, torch.ones_like(angles), angles)
    return torch.where(small, 0.5 - angles * angles / 48, torch.sin(half) / safe)


def quaternion_to_axis_angle(q: torch.Tensor) -> torch.Tensor:
    norms = torch.norm(q[..., 1:], p=2, dim=-1, keepdim=True)
    half = torch.atan2(norms, q[..., :1])
    return q[..., 1:] / _sin_half_over_angle(2 * half, half)


def axis_angle_to_matrix(aa: torch.Tensor) -> torch.Tensor:
    angles = torch.norm(aa, p=2, dim=-1, keepdim=True)
    half = angles * 0.5
    q = torch.cat([torch.cos(half), aa * _sin_half_over_angle(angles, half)], -1)
    r, i, j, k = q.unbind(-1)
    two_s = 2.0 / (q * q).sum(-1)
    o = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return o.reshape(q.shape[:-1] + (3, 3))


def matrix_to_rotation_6d(m: torch.Tensor) -> torch.Tensor:
    return m[..., :2, :].reshape(m.shape[:-2] + (6,))


def rot6d_to_aa(d6: torch.Tensor) -> torch.Tensor:
    return quaternion_to_axis_angle(matrix_to_quaternion(rotation_6d_to_matrix(d6)))


# ---------------------------------------------------------------- motion VAE decoder
LAYER_KEYS = ("self_attn.in_proj_weight", "self_attn.in_proj_bias", "self_attn.out_proj.weight",
              "self_attn.out_proj.bias", "multihead_attn.in_proj_weight", "multihead_attn.in_proj_bias",
              "multihead_attn.out_proj.weight", "multihead_attn.out_proj.bias", "linear1.weight", "linear1.bias",
              "linear2.weight", "linear2.bias", "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias",
              "norm3.weight", "norm3.bias")


def motion_vae_state(seed: int = MOTION_VAE_SEED, latent: int = 256, num_layers: int = 4, n_out: int = 330) -> dict:
    """MotionOptimizer's decoder keys (``decoder.seqTransDecoder.layers.{l}.*``, ``decoder.final.*``) with nn.Linear /
    nn.LayerNorm layouts, scaled so that the 6D outputs spread over a wide range of joint rotations."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, std: torch.randn(*s, generator=g) * std
    D, F = latent, 4 * latent
    sd = {}
    for l in range(num_layers):
        p = f"decoder.seqTransDecoder.layers.{l}."
        for a in ("self_attn", "multihead_attn"):
            sd[p + f"{a}.in_proj_weight"] = rn(3 * D, D, std=1.5 / math.sqrt(D))
            sd[p + f"{a}.in_proj_bias"] = rn(3 * D, std=0.05)
            sd[p + f"{a}.out_proj.weight"] = rn(D, D, std=1 / math.sqrt(D))
            sd[p + f"{a}.out_proj.bias"] = rn(D, std=0.05)
        sd[p + "linear1.weight"] = rn(F, D, std=1 / math.sqrt(D))
        sd[p + "linear1.bias"] = rn(F, std=0.05)
        sd[p + "linear2.weight"] = rn(D, F, std=1 / math.sqrt(F))
        sd[p + "linear2.bias"] = rn(D, std=0.05)
        for n in (1, 2, 3):
            sd[p + f"norm{n}.weight"] = 1.0 + rn(D, std=0.1)
            sd[p + f"norm{n}.bias"] = rn(D, std=0.05)
    sd["decoder.final.weight"] = rn(n_out, D, std=0.3 / math.sqrt(D))
    sd["decoder.final.bias"] = torch.tensor([1.0, 0.0, 0.0, 0.0, 1.0, 0.0]).repeat(n_out // 6) + rn(n_out, std=0.2)
    return sd


def positional_table(num_frame: int, d_model: int) -> torch.Tensor:
    """SinusoidalPositionalEncoding's rows: sin / cos of position * exp(-2i log(10000) / d_model), in fp64."""
    pos = torch.arange(num_frame, dtype=torch.float64)[:, None]
    div = torch.exp(torch.arange(0, d_model, 2, dtype=torch.float64) * (-math.log(10000.0) / d_model))
    pe = torch.zeros(num_frame, d_model, dtype=torch.float64)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


def decoder(latent: torch.Tensor, sd: dict, num_layers: int = 4, num_heads: int = 4, num_frame: int = 60,
            pe: torch.Tensor = None) -> torch.Tensor:
    """MotionXTransformerDecoder(latent [D]) -> [num_frame, n_out] in latent's dtype: post-LN decoder layers (self
    attention, attention over the one memory token, exact-GELU feed-forward), LayerNorm eps 1e-5, then final."""
    dt = latent.dtype
    D = latent.numel()
    dh = D // num_heads
    g = lambda k: _t(sd[k], dt)
    x = (positional_table(num_frame, D) if pe is None else pe).to(dt)
    mem = latent.reshape(1, D)
    ln = lambda v, p: torch.nn.functional.layer_norm(v, (D,), g(p + ".weight"), g(p + ".bias"), 1e-5)
    for l in range(num_layers):
        p = f"decoder.seqTransDecoder.layers.{l}."
        qkv = x @ g(p + "self_attn.in_proj_weight").T + g(p + "self_attn.in_proj_bias")
        q, k, v = (qkv[:, i * D:(i + 1) * D].reshape(num_frame, num_heads, dh).transpose(0, 1) for i in range(3))
        a = torch.softmax(q @ k.transpose(1, 2) / math.sqrt(dh), -1) @ v
        a = a.transpose(0, 1).reshape(num_frame, D)
        x = ln(x + a @ g(p + "self_attn.out_proj.weight").T + g(p + "self_attn.out_proj.bias"), p + "norm1")
        Wv = g(p + "multihead_attn.in_proj_weight")[2 * D:]
        bv = g(p + "multihead_attn.in_proj_bias")[2 * D:]
        c = (mem @ Wv.T + bv) @ g(p + "multihead_attn.out_proj.weight").T + g(p + "multihead_attn.out_proj.bias")
        x = ln(x + c, p + "norm2")
        h = torch.nn.functional.gelu(x @ g(p + "linear1.weight").T + g(p + "linear1.bias"))
        x = ln(x + h @ g(p + "linear2.weight").T + g(p + "linear2.bias"), p + "norm3")
    return x @ g("decoder.final.weight").T + g("decoder.final.bias")


def decode(latent: torch.Tensor, sd: dict, **kw) -> torch.Tensor:
    """MotionOptimizer.decode -> [num_frame, 63]."""
    out = decoder(latent, sd, **kw)
    aa = rot6d_to_aa(out.reshape(-1, 6)).reshape(out.shape[0], -1)
    return aa[:, 3:66]


def loss(motion: torch.Tensor, poses: torch.Tensor, recon_coef, delta_coef: float) -> torch.Tensor:
    """get_motion's loss with clip_coef = 0 (torch.min's gradient goes to the index it returns)."""
    K, T = poses.shape[0], motion.shape[0]
    six = lambda a: matrix_to_rotation_6d(axis_angle_to_matrix(a.reshape(*a.shape[:-1], N_JOINTS, 3)))
    per = ((six(motion)[None] - six(poses.to(motion.dtype))[:, None]) ** 2).mean(-1).mean(-1)    # [K, T]
    value, _ = torch.min(per, dim=1)
    total = 0
    for j in range(K):
        total = total + value[j] * recon_coef[j]
    if delta_coef > 0:
        total = total - torch.nn.functional.mse_loss(motion[:-1], motion[1:]) * delta_coef
    return total


def optimize(sd: dict, poses, latent0, n_iter: int, recon_coef, delta_coef: float, lr: float = 0.01,
             dtype=torch.float64, **kw):
    """get_motion's loop (clip_coef = 0) with torch.optim.Adam on a CPU parameter of ``dtype``: (losses [n_iter],
    final latent, the motion of the last iteration [num_frame, 63])."""
    z = torch.nn.Parameter(_t(latent0, dtype).clone())
    opt = torch.optim.Adam([z], lr=lr)
    p = _t(poses, dtype)
    losses = []
    for _ in range(n_iter):
        motion = decode(z, sd, **kw)
        lo = loss(motion, p, recon_coef, delta_coef)
        opt.zero_grad()
        lo.backward()
        opt.step()
        losses.append(float(lo.detach()))
    return torch.tensor(losses, dtype=torch.float64), z.detach().clone(), motion.detach()
