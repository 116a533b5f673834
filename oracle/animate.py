"""CPU oracle (test infrastructure, never on the product path): AvatarAnimate's pose stage (models/pose_generation.py,
render.py) restated in numpy / torch CPU fp64 -- the VPoser decoder, the conditional RealNVP, SMPL with zero betas, the
batched textured render, the CLIP score, the codebook top-k and the duplicate suppression -- plus the seeded synthetic
weights the tests and oracle/pin_animate.py share.

PARITY UNPINNED for VPoser: ``human_body_prior`` (and the torchgeometry it calls) is neither vendored nor installed.
Restated from their published algorithms: ``decoder_net`` = Linear(32, 512), LeakyReLU(0.01), Dropout (identity in
eval), Linear(512, 512), LeakyReLU, Linear(512, 126), then ``ContinousRotReprDecoder`` (each joint's 6 values as a
[3, 2] matrix, b1 = normalize(col 0), b2 = normalize(col 1 - (b1 . col 1) b1), b3 = b1 x b2, R = [b1 b2 b3] as columns)
and ``matrot2aa`` = torchgeometry's ``rotation_matrix_to_angle_axis`` (``rotation_matrix_to_quaternion``'s four
branches on the transposed matrix with eps 1e-6, then ``quaternion_to_angle_axis``).  The textured rasteriser is
oracle/shapegen.py's (also unpinned).  Everything around them -- the RealNVP decode, the scorer, the search loops, the
sort, the codebook top-k and the suppression -- is the reference's own code, run by oracle/pin_animate.py.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import lbs as olbs
from oracle import shapegen as OS

ANGLES = (120, 150, 180, 210, 240)          # get_pose_feature's default cameras
CAMERA_DISTANCE = 2.0                       # render.py:13
ROT = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])   # render.py:25-28, applied as v @ ROT
GLOBAL_ORIENT = (math.pi / 2, 0.0, 0.0)     # get_pose_feature :71-72
VPOSER_SEED = 21
REALNVP_SEED = 22
CODEBOOK_SEED = 23
TEXT = "a rendered 3d man is crying"


def _d(t) -> np.ndarray:
    return np.asarray(torch.as_tensor(t).detach().cpu(), dtype=np.float64)


def leaky(x):
    return np.where(x > 0, x, 0.01 * x)


# ---------------------------------------------------------------- VPoser
def rot6d_to_matrix(x) -> np.ndarray:
    """ContinousRotReprDecoder: [..., 6] -> [..., 3, 3] (fp64)."""
    m = np.asarray(x, dtype=np.float64).reshape(-1, 3, 2)
    a, c = m[:, :, 0], m[:, :, 1]
    b1 = a / np.maximum(np.linalg.norm(a, axis=1, keepdims=True), 1e-12)
    u = c - (b1 * c).sum(1, keepdims=True) * b1
    b2 = u / np.maximum(np.linalg.norm(u, axis=1, keepdims=True), 1e-12)
    return np.stack([b1, b2, np.cross(b1, b2)], -1)


def matrot2aa(R) -> np.ndarray:
    """torchgeometry rotation_matrix_to_angle_axis of [N, 3, 3] in fp64 (the branch chosen on the same tests)."""
    R = np.asarray(R, dtype=np.float64).reshape(-1, 3, 3)
    m = np.transpose(R, (0, 2, 1))
    out = np.zeros((R.shape[0], 3))
    for i, t_ in enumerate(m):
        if t_[2, 2] < 1e-6:
            if t_[0, 0] > t_[1, 1]:
                t = 1 + t_[0, 0] - t_[1, 1] - t_[2, 2]
                q = [t_[1, 2] - t_[2, 1], t, t_[0, 1] + t_[1, 0], t_[2, 0] + t_[0, 2]]
            else:
                t = 1 - t_[0, 0] + t_[1, 1] - t_[2, 2]
                q = [t_[2, 0] - t_[0, 2], t_[0, 1] + t_[1, 0], t, t_[1, 2] + t_[2, 1]]
        elif t_[0, 0] < -t_[1, 1]:
            t = 1 - t_[0, 0] - t_[1, 1] + t_[2, 2]
            q = [t_[0, 1] - t_[1, 0], t_[2, 0] + t_[0, 2], t_[1, 2] + t_[2, 1], t]
        else:
            t = 1 + t_[0, 0] + t_[1, 1] + t_[2, 2]
            q = [t, t_[1, 2] - t_[2, 1], t_[2, 0] - t_[0, 2], t_[0, 1] - t_[1, 0]]
        q = np.asarray(q) / np.sqrt(t) * 0.5
        s2 = q[1] ** 2 + q[2] ** 2 + q[3] ** 2
        s = math.sqrt(s2)
        two_theta = 2 * (math.atan2(-s, -q[0]) if q[0] < 0 else math.atan2(s, q[0]))
        k = two_theta / s if s2 > 0 else 2.0
        out[i] = q[1:] * k
    return out


def vposer_decode(z, sd) -> tuple:
    """VPoser.decode(z)['pose_body'] [B, 21, 3] and the rotation matrices [B, 21, 3, 3], fp64."""
    g = lambda k: _d(sd[f"decoder_net.{k}"])
    h = leaky(_d(z) @ g("0.weight").T + g("0.bias"))
    h = leaky(h @ g("3.weight").T + g("3.bias"))
    o = h @ g("5.weight").T + g("5.bias")
    B = o.shape[0]
    R = rot6d_to_matrix(o.reshape(-1, 6))
    return matrot2aa(R).reshape(B, -1, 3), R.reshape(B, -1, 3, 3)


def vposer_state(seed: int = VPOSER_SEED, latent: int = 32, hidden: int = 512, n_joints: int = 21) -> dict:
    """decoder_net weights (nn.Linear layouts) scaled so that decoded poses spread over realistic joint angles."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, std: torch.randn(*s, generator=g) * std
    return {"decoder_net.0.weight": rn(hidden, latent, std=0.3), "decoder_net.0.bias": rn(hidden, std=0.1),
            "decoder_net.3.weight": rn(hidden, hidden, std=0.06), "decoder_net.3.bias": rn(hidden, std=0.1),
            "decoder_net.5.weight": rn(6 * n_joints, hidden, std=0.004),
            "decoder_net.5.bias": torch.tensor([1.0, 0.0, 0.0, 1.0, 0.0, 0.0]).repeat(n_joints)}


# ---------------------------------------------------------------- RealNVP
def realnvp_decode(z, feature, sd, n_block: int = 8) -> np.ndarray:
    """VPoserRealNVP.decode (:233-240) in fp64 with the feature repeated over the rows."""
    x = _d(z)
    f = np.broadcast_to(_d(feature).reshape(1, -1), (x.shape[0], _d(feature).size))
    mask = _d(sd["mask"]).reshape(n_block, -1)
    for i in range(n_block):
        m = mask[i]
        x_ = x * m
        trans = np.concatenate([x_, f], 1)
        net = lambda p: (lambda h: h @ _d(sd[f"{p}.{i}.4.weight"]).T + _d(sd[f"{p}.{i}.4.bias"]))(
            leaky(leaky(trans @ _d(sd[f"{p}.{i}.0.weight"]).T + _d(sd[f"{p}.{i}.0.bias"])) @
                  _d(sd[f"{p}.{i}.2.weight"]).T + _d(sd[f"{p}.{i}.2.bias"])))
        s = np.tanh(net("s")) * (1 - m)
        t = net("t") * (1 - m)
        x = x_ + (1 - m) * (x * np.exp(s) + t)
    return x


def realnvp_state(seed: int = REALNVP_SEED, dim: int = 32, hdim: int = 256, n_block: int = 8, feat: int = 512) -> dict:
    """``pose_realnvp.pth``'s ``state_dict``: s.{i} / t.{i} Sequential weights and the 0 / 1 ``mask`` [n_block, 1, dim]."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for p in ("s", "t"):
        for i in range(n_block):
            sd[f"{p}.{i}.0.weight"] = torch.randn(hdim, dim + feat, generator=g) * 0.05
            sd[f"{p}.{i}.0.bias"] = torch.randn(hdim, generator=g) * 0.05
            sd[f"{p}.{i}.2.weight"] = torch.randn(hdim, hdim, generator=g) * 0.06
            sd[f"{p}.{i}.2.bias"] = torch.randn(hdim, generator=g) * 0.05
            sd[f"{p}.{i}.4.weight"] = torch.randn(dim, hdim, generator=g) * 0.06
            sd[f"{p}.{i}.4.bias"] = torch.randn(dim, generator=g) * 0.05
    mask = torch.randn(n_block, 1, dim, generator=g)
    sd["mask"] = (mask > 0).float()
    return sd


# ---------------------------------------------------------------- SMPL, render, score
def smpl_vertices(smpl: dict, body_pose, global_orient=GLOBAL_ORIENT) -> np.ndarray:
    """smplx SMPL with zero betas: my_lbs on v_shaped = v_template of the 72-value pose (global_orient, body_pose padded
    with zeros) -> [B, V, 3] fp64."""
    bp = _d(body_pose).reshape(-1, _d(body_pose).shape[-1])
    B, nj = bp.shape[0], smpl["J_regressor"].shape[0]
    pose = np.zeros((B, nj * 3))
    pose[:, :3] = global_orient
    pose[:, 3:3 + bp.shape[1]] = bp
    vt = torch.as_tensor(_d(smpl["v_template"]))[None].expand(B, -1, -1)
    v, _ = olbs.my_lbs(vt, torch.from_numpy(pose), torch.as_tensor(_d(smpl["posedirs"])),
                       torch.as_tensor(_d(smpl["J_regressor"])), torch.as_tensor(smpl["parents"]).long(),
                       torch.as_tensor(_d(smpl["lbs_weights"])))
    return v.numpy()


def eye(elevation: float, azimuth: float):
    """neural_renderer's get_points_from_angles(2, elevation, azimuth) in degrees."""
    el, az = math.radians(elevation), math.radians(azimuth)
    return (CAMERA_DISTANCE * math.cos(el) * math.sin(az), CAMERA_DISTANCE * math.sin(el),
            -CAMERA_DISTANCE * math.cos(el) * math.cos(az))


def render_batch(verts, faces, textures, eyes) -> np.ndarray:
    """render.py:10-39 for explicit eyes: [A * B, 256, 256, 3] (angle-major) of the meshes [B, V, 3] times ROT."""
    v = np.asarray(verts, dtype=np.float64) @ ROT
    return np.stack([OS.raster_textured(v[b], faces, textures, e) for e in eyes for b in range(v.shape[0])])


def cosine(a, b, eps: float = 1e-8) -> np.ndarray:
    """F.cosine_similarity in fp64: each operand divided by max(|.|, eps)."""
    a, b = np.atleast_2d(_d(a)), np.atleast_2d(_d(b))
    a = a / np.maximum(np.linalg.norm(a, axis=1, keepdims=True), eps)
    b = b / np.maximum(np.linalg.norm(b, axis=1, keepdims=True), eps)
    return (a * b).sum(1)


def suppress(poses, threshold: float) -> list:
    """suppress_duplicated_poses (:304-317) on fp32 values: the kept indices in order."""
    p = np.asarray(poses, dtype=np.float32)
    kept = []
    for i in range(p.shape[0]):
        md = 10.0
        for j in kept:
            md = min(np.float32(np.abs(p[i] - p[j]).astype(np.float64).mean()), md)
        if not kept or md > np.float32(threshold):
            kept.append(i)
    return kept


def make_codebook(text_feature, seed: int = CODEBOOK_SEED, n: int = 256, latent: int = 32) -> dict:
    """``codebook.pth``: latents [n, 32] and embeddings [n, 512] whose cosines with the text feature are spread at least
    0.004 apart in their top 48 (no ties for the top-40), and whose top-40 latents come in near-duplicate pairs and
    triples so that the suppression has work to do.  The latents are scaled so that, through ``vposer_state``'s
    decoder, the planted duplicates lie within about 0.002 of their kept neighbour in mean absolute difference and
    every other pose at least 0.1 from every kept one: both sides clear of the 0.07 threshold."""
    g = torch.Generator().manual_seed(seed)
    t = torch.as_tensor(text_feature, dtype=torch.float64).reshape(-1)
    t = t / t.norm()
    r = torch.randn(n, t.numel(), generator=g, dtype=torch.float64)
    r = r - (r @ t)[:, None] * t
    r = r / r.norm(dim=1, keepdim=True)
    target = torch.linspace(0.9, -0.3, n, dtype=torch.float64)[torch.randperm(n, generator=g)]
    emb = target[:, None] * t + (1 - target[:, None] ** 2).sqrt() * r
    lat = torch.randn(n, latent, generator=g)
    order = torch.argsort(-target)
    for k in range(1, 40, 3):             # every third of the top-40 sits next to its predecessor
        lat[order[k]] = lat[order[k - 1]] + 0.01 * torch.randn(latent, generator=g)
    return {"codebook": 2.0 * lat, "codebook_embedding": emb.float()}
