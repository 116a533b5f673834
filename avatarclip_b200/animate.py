"""Host-side mirror of AvatarAnimate's pose stage (main.py with ``general.mode = pose``): candidate SMPL body poses
that a text prompt describes, written as ``candidate_%d.npy`` (63 float32 axis-angle values, joints 1-21) and
``candidate_%d.jpg``.

Two generators of models/pose_generation.py run here:
  * ``VPoserCodebook`` (:288-329): the CLIP cosine of every codebook embedding against the prompt, the top ``pre_topk``,
    their VPoser decodes, greedy duplicate suppression, the first ``topk``;
  * ``VPoserRealNVP`` (:176-285): per candidate ``num_batch`` x ``num_sample`` prior draws through the text-conditioned
    RealNVP and VPoser, each pose posed on SMPL, rendered with the UV texture from 5 cameras and scored by CLIP; the
    best of the batches is kept, then the candidates are sorted by a fresh score.
The gradient-based generators are refused before any file is read, each naming its own command: ``PoseOptimizer``
runs as ``python -m avatarclip_b200.pose_optimizer`` and ``VPoserOptimizer`` as ``python -m
avatarclip_b200.vposer_optimizer`` (the VPoser latent optimised through ``avc_vposer_decode_bwd``); the motion stage
(``general.mode = motion``) is ``python -m avatarclip_b200.motion``.

Everything on the hot path runs in libavc_b200.so: ``avc_vposer_decode``, ``avc_realnvp_decode``,
``avc_smpl_pose_batch``, ``avc_raster_textured_batch``, ``avc_clip_prep_nearest``, the CLIP towers,
``avc_pose_score``, ``avc_cosine_topk`` and ``avc_pose_suppress``; the jpg is drawn by ``avc_video_render``.

    python -m avatarclip_b200.animate --conf confs/pose_ablation/vposer_realnvp/cry.conf --smpl smpl.npz \\
        --clip_model ViT-B-32.pt --bpe bpe_simple_vocab_16e6.txt.gz
"""
from __future__ import annotations

import argparse
import ctypes as C
import glob
import math
import os
import sys
from typing import List, Mapping, NamedTuple, Optional, Sequence

import numpy as np
import torch

from . import _lib, drive, shapegen

ANGLES = (120, 150, 180, 210, 240)      # get_pose_feature's default cameras
CAMERA_DISTANCE = 2.0                   # render.py:13
ELEVATION_STD = 0.3                     # render.py:34: np.random.randn() * 0.3 degrees per camera per call
RENDER_ROT = np.array([[1, 0, 0], [0, 0, -1], [0, 1, 0]], dtype=np.float32)    # render.py:25-28 (v @ RENDER_ROT)
SCORE_ORIENT = (math.pi / 2, 0.0, 0.0)  # get_pose_feature :71-72
IMAGE_ORIENT = (math.pi, 0.0, 0.0)      # visualize.py:87-88
IMAGE_SIZE, IMAGE_FOCAL, IMAGE_DEPTH, IMAGE_GREY = 512, 5000.0, 25.0, 0.4    # visualize.py:20-38
IN_SCOPE = ("VPoserCodebook", "VPoserRealNVP")
OUT_OF_SCOPE = {"PoseOptimizer": "optimises SMPL theta through the rasteriser's gradient, so it runs as its own "
                                 "command: python -m avatarclip_b200.pose_optimizer",
                "VPoserOptimizer": "optimises the VPoser latent through the rasteriser's gradient and the VPoser "
                                   "decoder's, so it runs as its own command: python -m "
                                   "avatarclip_b200.vposer_optimizer"}
DEFAULT_PATHS = {"vposer": "data/vposer", "codebook": "data/codebook.pth",      # BasePoseGenerator / the
                 "realnvp": "data/pose_realnvp.pth"}                           # generators' constructor defaults
_RENDER_BYTES = 1 << 30                 # device bytes per chunk of renders (z-buffers, images, CLIP inputs)

_bound = None


def _L():
    global _bound
    L = _lib.lib()
    if _bound is None:
        vp, i32, f32, sz = C.c_void_p, C.c_int32, C.c_float, C.c_size_t
        P = C.POINTER
        L.avc_vposer_decode_workspace_bytes.argtypes = [i32, i32, i32, P(sz)]
        L.avc_vposer_decode.argtypes = [vp, i32, i32, vp, vp, i32, vp, vp, vp, vp, i32, vp, vp, vp, sz, vp]
        L.avc_realnvp_pack_floats.argtypes = [i32, i32, i32, P(sz)]
        L.avc_realnvp_pack.argtypes = [vp, i32, i32, i32, i32, vp, vp]
        L.avc_realnvp_decode_workspace_bytes.argtypes = [i32, i32, i32, P(sz)]
        L.avc_realnvp_decode.argtypes = [vp, i32, i32, vp, i32, vp, vp, vp, i32, i32, vp, vp, sz, vp]
        L.avc_smpl_pose_batch_workspace_bytes.argtypes = [i32, i32, P(sz)]
        L.avc_smpl_pose_batch.argtypes = [vp, vp, vp, vp, vp, i32, i32, vp, i32, i32, vp, vp, vp, vp, sz, vp]
        L.avc_raster_textured_batch_workspace_bytes.argtypes = [i32, i32, i32, i32, i32, P(sz)]
        L.avc_raster_textured_batch.argtypes = [vp, i32, i32, vp, vp, i32, i32, i32, vp, i32, vp, vp, i32, i32, vp,
                                                vp, sz, vp]
        L.avc_cosine_topk.argtypes = [vp, i32, i32, vp, f32, i32, vp, vp, vp]
        L.avc_pose_suppress.argtypes = [vp, i32, i32, f32, vp, vp, vp]
        L.avc_pose_score.argtypes = [vp, i32, i32, i32, vp, i32, vp, vp, vp, sz, vp]
        for n in ("avc_vposer_decode_workspace_bytes", "avc_vposer_decode", "avc_realnvp_pack_floats",
                  "avc_realnvp_pack", "avc_realnvp_decode_workspace_bytes",
                  "avc_realnvp_decode", "avc_smpl_pose_batch_workspace_bytes", "avc_smpl_pose_batch",
                  "avc_raster_textured_batch_workspace_bytes", "avc_raster_textured_batch", "avc_cosine_topk",
                  "avc_pose_suppress", "avc_pose_score"):
            getattr(L, n).restype = C.c_int
        _bound = L
    return L


def _dev(t: torch.Tensor, what: str) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.AvcError(f"{what}: avatarclip_b200 has no CPU path")
    return t.detach().float().contiguous()


def _host_f32(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def _hp(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def _ws(query, *args) -> C.c_size_t:
    need = C.c_size_t()
    _lib.check(query(*args, C.byref(need)), query.__name__)
    return need.value


# ---------------------------------------------------------------- device ops
def vposer_decode(z: torch.Tensor, dec: Mapping[str, torch.Tensor], return_matrot: bool = False):
    """VPoser.decode(z)['pose_body'] for z [B, latent] -> [B, n_joints, 3] (and [B, n_joints, 3, 3])."""
    z = _dev(z, "vposer_decode").reshape(z.shape[0], -1)
    w = [_dev(dec[f"decoder_net.{i}.{k}"], "vposer_decode") for i in (0, 3, 5) for k in ("weight", "bias")]
    H, Lz, O = w[0].shape[0], w[0].shape[1], w[4].shape[0]
    if z.shape[1] != Lz or O % 6 or tuple(w[2].shape) != (H, H) or w[4].shape[1] != H:
        raise _lib.AvcError(f"vposer_decode: z {tuple(z.shape)} against decoder_net {[tuple(t.shape) for t in w]}")
    B, nj = z.shape[0], O // 6
    L = _L()
    ws = torch.empty(_ws(L.avc_vposer_decode_workspace_bytes, Lz, H, nj), dtype=torch.uint8, device=z.device)
    pose = torch.empty(B, nj, 3, device=z.device)
    rot = torch.empty(B, nj, 3, 3, device=z.device) if return_matrot else None
    _lib.check(L.avc_vposer_decode(_lib.ptr(z), B, Lz, _lib.ptr(w[0]), _lib.ptr(w[1]), H, _lib.ptr(w[2]),
                                   _lib.ptr(w[3]), _lib.ptr(w[4]), _lib.ptr(w[5]), nj, _lib.ptr(pose), _lib.ptr(rot),
                                   _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "avc_vposer_decode")
    return (pose, rot) if return_matrot else pose


class RealNVPWeights(NamedTuple):
    """The coupling nets on the device: ``params`` in avc_realnvp_decode's layout, ``pack`` their transposed copies
    (avc_realnvp_pack, made once), ``mask`` [num_block, dim]."""
    params: torch.Tensor
    pack: torch.Tensor
    mask: torch.Tensor
    hidden: int
    feat_dim: int


def pack_realnvp(sd: Mapping[str, torch.Tensor], num_block: int, device) -> RealNVPWeights:
    """``pose_realnvp.pth``'s state dict on the device, packed for avc_realnvp_decode."""
    device = drive._cuda(device)
    parts = []
    for i in range(num_block):
        for p in ("s", "t"):
            for k in ("0.weight", "0.bias", "2.weight", "2.bias", "4.weight", "4.bias"):
                parts.append(torch.as_tensor(sd[f"{p}.{i}.{k}"]).float().reshape(-1))
    params = torch.cat(parts).to(device).contiguous()
    mask = torch.as_tensor(sd["mask"]).float().reshape(num_block, -1).to(device).contiguous()
    H, DE = torch.as_tensor(sd["s.0.0.weight"]).shape
    D = mask.shape[1]
    E = DE - D
    if params.numel() != 2 * num_block * (H * (D + E) + H + H * H + H + D * H + D):
        raise ValueError(f"RealNVP weights: {params.numel()} values do not form {num_block} blocks of dim {D}, "
                         f"hidden {H}, feature {E}")
    L = _L()
    pack = torch.empty(_ws(L.avc_realnvp_pack_floats, D, H, num_block), device=device)
    _lib.check(L.avc_realnvp_pack(_lib.ptr(params), D, E, H, num_block, _lib.ptr(pack), _lib.stream_ptr()),
               "avc_realnvp_pack")
    return RealNVPWeights(params, pack, mask, H, E)


def realnvp_decode(z: torch.Tensor, feature: torch.Tensor, w: RealNVPWeights) -> torch.Tensor:
    """VPoserRealNVP.decode(z, feature repeated over the rows) -> [B, dim]."""
    z = _dev(z, "realnvp_decode")
    f = _dev(feature, "realnvp_decode").reshape(-1)
    nb, D = w.mask.shape
    B = z.shape[0]
    if z.shape[1] != D or f.numel() != w.feat_dim:
        raise _lib.AvcError(f"realnvp_decode: z {tuple(z.shape)} and feature {f.numel()} against dim {D}, "
                            f"feature {w.feat_dim}")
    L = _L()
    ws = torch.empty(_ws(L.avc_realnvp_decode_workspace_bytes, D, w.hidden, nb), dtype=torch.uint8, device=z.device)
    x = torch.empty(B, D, device=z.device)
    _lib.check(L.avc_realnvp_decode(_lib.ptr(z), B, D, _lib.ptr(f), f.numel(), _lib.ptr(w.params), _lib.ptr(w.pack),
                                    _lib.ptr(w.mask), nb, w.hidden, _lib.ptr(x), _lib.ptr(ws), ws.numel(),
                                    _lib.stream_ptr()), "avc_realnvp_decode")
    return x


def smpl_pose_batch(s: dict, body_pose: torch.Tensor, global_orient=SCORE_ORIENT, post_rot=None) -> torch.Tensor:
    """smplx SMPL (zero betas) of body poses [B, 63 | 69] with one global orientation -> vertices [B, V, 3], optionally
    times ``post_rot`` (v @ post_rot)."""
    bp = _dev(body_pose, "smpl_pose_batch")
    bp = bp.reshape(bp.shape[0], -1)
    B, V, nj = bp.shape[0], s["v_template"].shape[0], s["J_regressor"].shape[0]
    L = _L()
    ws = torch.empty(_ws(L.avc_smpl_pose_batch_workspace_bytes, B, nj), dtype=torch.uint8, device=bp.device)
    out = torch.empty(B, V, 3, device=bp.device)
    go = _host_f32(global_orient).reshape(3)
    pr = None if post_rot is None else _host_f32(post_rot).reshape(9)
    _lib.check(L.avc_smpl_pose_batch(_lib.ptr(s["v_template"]), _lib.ptr(s["J_regressor"]), _lib.ptr(s["parents"]),
                                     _lib.ptr(s["posedirs"]), _lib.ptr(s["lbs_weights"]), V, nj, _lib.ptr(bp),
                                     bp.shape[1], B, _hp(go), None if pr is None else _hp(pr), _lib.ptr(out),
                                     _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "avc_smpl_pose_batch")
    return out


def raster_textured_batch(verts: torch.Tensor, faces: torch.Tensor, textures: torch.Tensor, eyes, group: int,
                          image_size: int = shapegen.IMAGE_SIZE, supersample: int = 2, at=(0.0, 0.0, 0.0),
                          up=(0.0, 1.0, 0.0)) -> torch.Tensor:
    """Renders of verts [B, V, 3] from eyes [ceil(B / group), A, 3] (mesh b uses eyes[b // group]) -> [A, B, n, n, 3]."""
    v = _dev(verts, "raster_textured_batch")
    f = faces.to(v.device, torch.int32).contiguous()
    t = _dev(textures, "raster_textured_batch")
    B, V = v.shape[0], v.shape[1]
    e = _host_f32(eyes).reshape(-1, 3)
    ng = (B + group - 1) // group
    A = e.shape[0] // ng
    if A * ng != e.shape[0] or tuple(t.shape) != (f.shape[0], t.shape[1], t.shape[1], t.shape[1], 3):
        raise _lib.AvcError(f"raster_textured_batch: {e.shape[0]} eyes for {ng} groups, textures {tuple(t.shape)}")
    L = _L()
    ws = torch.empty(_ws(L.avc_raster_textured_batch_workspace_bytes, V, A * B, ng * A, image_size, supersample),
                     dtype=torch.uint8, device=v.device)
    rgb = torch.empty(A, B, image_size, image_size, 3, device=v.device)
    a_, u_ = _host_f32(at).reshape(3), _host_f32(up).reshape(3)
    _lib.check(L.avc_raster_textured_batch(_lib.ptr(v), B, group, _lib.ptr(f), _lib.ptr(t), V, f.shape[0],
                                           t.shape[1], _hp(e), A, _hp(a_), _hp(u_), image_size, supersample,
                                           _lib.ptr(rgb), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
               "avc_raster_textured_batch")
    return rgb


def cosine_topk(rows: torch.Tensor, vec: torch.Tensor, k: int, eps: float = 1e-8):
    """(F.cosine_similarity(rows, vec) [N], torch.topk(., k) indices [k]) on the device."""
    r = _dev(rows, "cosine_topk")
    v = _dev(vec, "cosine_topk").reshape(-1)
    N, D = r.shape
    if v.numel() != D or not 1 <= k <= N:
        raise _lib.AvcError(f"cosine_topk: rows {tuple(r.shape)}, vector {v.numel()}, k {k}")
    cos = torch.empty(N, device=r.device)
    idx = torch.empty(k, dtype=torch.int32, device=r.device)
    _lib.check(_L().avc_cosine_topk(_lib.ptr(r), N, D, _lib.ptr(v), eps, k, _lib.ptr(cos), _lib.ptr(idx),
                                    _lib.stream_ptr()), "avc_cosine_topk")
    return cos, idx


def pose_suppress(poses: torch.Tensor, threshold: float) -> torch.Tensor:
    """suppress_duplicated_poses: the kept row indices (device int32) of poses [P <= 64, dim]."""
    p = _dev(poses, "pose_suppress").reshape(poses.shape[0], -1)
    keep = torch.empty(p.shape[0], dtype=torch.int32, device=p.device)
    count = torch.empty(1, dtype=torch.int32, device=p.device)
    _lib.check(_L().avc_pose_suppress(_lib.ptr(p), p.shape[0], p.shape[1], threshold, _lib.ptr(keep),
                                      _lib.ptr(count), _lib.stream_ptr()), "avc_pose_suppress")
    return keep[:int(count.item())]


def pose_score(emb: torch.Tensor, text: torch.Tensor, group: int):
    """(scores [B], per-group first argmax [ceil(B / group)]) of emb [A, B, dim] against text [dim]."""
    e = _dev(emb, "pose_score")
    t = _dev(text, "pose_score").reshape(-1)
    A, B, D = e.shape
    ng = (B + group - 1) // group
    ws = torch.empty(8 * ng, dtype=torch.uint8, device=e.device)
    score = torch.empty(B, device=e.device)
    best = torch.empty(ng, dtype=torch.int32, device=e.device)
    _lib.check(_L().avc_pose_score(_lib.ptr(e), A, B, D, _lib.ptr(t), group, _lib.ptr(score), _lib.ptr(best),
                                   _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "avc_pose_score")
    return score, best


# ---------------------------------------------------------------- loaders
VPOSER_ENCODER_KEYS = tuple([f"encoder_net.{i}.{k}" for i in (1, 4) for k in ("weight", "bias", "running_mean",
                                                                               "running_var")] +
                            [f"encoder_net.{i}.{k}" for i in (2, 6, 7, "8.mu") for k in ("weight", "bias")])


def load_vposer(path, encoder: bool = False) -> dict:
    """human_body_prior's ``load_model(path, remove_words_in_model_weights='vp_model.')``, decoder only: ``path`` is the
    VPoser directory (the last of ``snapshots/*.ckpt``, a Lightning checkpoint whose ``state_dict`` holds
    ``vp_model.decoder_net.{0,3,5}.{weight,bias}``), one such checkpoint file, or a state dict.  With ``encoder`` the
    result also holds ``VPOSER_ENCODER_KEYS`` (what ``VPoser.encode(x).mean`` reads)."""
    if isinstance(path, Mapping):
        sd = path
    else:
        fname = path
        if os.path.isdir(path):
            snaps = sorted(glob.glob(os.path.join(path, "snapshots", "*.ckpt")))
            if not snaps:
                raise FileNotFoundError(f"{path}: no snapshots/*.ckpt (a VPoser 2.x model directory)")
            fname = snaps[-1]
        ck = torch.load(fname, map_location="cpu", weights_only=False)
        sd = ck.get("state_dict", ck)
    sd = {k.replace("vp_model.", ""): v for k, v in sd.items()}
    keys = [f"decoder_net.{i}.{k}" for i in (0, 3, 5) for k in ("weight", "bias")]
    if encoder:
        keys += VPOSER_ENCODER_KEYS
    missing = [k for k in keys if k not in sd]
    if missing:
        raise ValueError(f"VPoser weights: missing {missing}")
    return {k: torch.as_tensor(sd[k]).float() for k in keys}


def load_realnvp(path) -> dict:
    """``pose_realnvp.pth``: ``torch.load(path)['state_dict']`` (or the state dict itself)."""
    data = path if isinstance(path, Mapping) else torch.load(path, map_location="cpu", weights_only=False)
    return data.get("state_dict", data)


def load_pose_codebook(path) -> tuple:
    """``codebook.pth``: (codebook latents [N, 32], codebook_embedding [N, 512])."""
    data = path if isinstance(path, Mapping) else torch.load(path, map_location="cpu", weights_only=False)
    return torch.as_tensor(data["codebook"]), torch.as_tensor(data["codebook_embedding"])


class Assets:
    """What BasePoseGenerator loads (:35-49): CLIP, SMPL, VPoser, and render.py's UV texture."""

    def __init__(self, smpl, clip: shapegen.ClipModels, vposer, uv_obj, device="cuda"):
        self.device = drive._cuda(device)
        self.smpl = drive.smpl_tensors(smpl, self.device)
        self.faces = torch.as_tensor(np.asarray(smpl["faces"], dtype=np.int32)).to(self.device)
        self.clip = clip
        # None: a generator that needs no VPoser (PoseOptimizer)
        self.vposer = None if vposer is None else {k: v.to(self.device) for k, v in load_vposer(vposer).items()}
        tex = uv_obj if isinstance(uv_obj, torch.Tensor) else shapegen.load_obj_textures(uv_obj, 8, self.device)
        if tex.shape[0] != self.faces.shape[0]:
            raise ValueError(f"the UV texture has {tex.shape[0]} faces, the SMPL mesh {self.faces.shape[0]}")
        self.textures = tex.to(self.device).float().contiguous()


class PoseScorer:
    """BasePoseGenerator's scoring (:56-99), batched.  The camera elevations come from numpy's global RNG in the
    reference's order: one ``np.random.randn()`` per angle per ``get_pose_feature`` call."""

    def __init__(self, assets: Assets, angles: Sequence[float] = ANGLES):
        self.a = assets
        self.angles = tuple(angles)

    def get_text_feature(self, text: str) -> torch.Tensor:
        c = self.a.clip
        return c.text.encode_text(c.tokenizer.tokenize(text, context_length=c.text.context)).float()[0]

    def draw_eyes(self, n_calls: int) -> np.ndarray:
        """[n_calls, A, 3]: the cameras of n_calls consecutive get_pose_feature calls."""
        out = np.empty((n_calls, len(self.angles), 3))
        for i in range(n_calls):
            for j, az in enumerate(self.angles):
                el = np.random.randn() * ELEVATION_STD
                out[i, j] = shapegen.handoff.get_points_from_angles(CAMERA_DISTANCE, el, az)
        return out

    def _chunk(self, group: int) -> int:
        n = shapegen.IMAGE_SIZE
        per_pose = len(self.angles) * (8 * (2 * n) ** 2 + 12 * n * n + 4 * 3 * 224 * 224 + 16 * self.a.smpl[
            "v_template"].shape[0]) + 12 * self.a.smpl["v_template"].shape[0]
        return max(group, (_RENDER_BYTES // per_pose) // group * group)

    def scores(self, poses: torch.Tensor, text_feature: torch.Tensor, group: int, eyes: np.ndarray):
        """get_pose_feature + the cosine for poses [B, 63 | 69] in groups of ``group`` rows, group g seen from eyes[g]:
        (scores [B], first argmax of each group [B / group])."""
        B = poses.shape[0]
        scores, best = [], []
        chunk = self._chunk(group)
        for b0 in range(0, B, chunk):
            p = poses[b0:b0 + chunk]
            v = smpl_pose_batch(self.a.smpl, p, SCORE_ORIENT, RENDER_ROT)
            imgs = raster_textured_batch(v, self.a.faces, self.a.textures, eyes[b0 // group:(b0 + p.shape[0] + group - 1)
                                                                               // group], group)
            A = imgs.shape[0]
            prep = shapegen.clip_prep_nearest(imgs.reshape(A * p.shape[0], *imgs.shape[2:]))
            emb = torch.cat([self.a.clip.image.encode_image(prep[i:i + 256]).float() for i in range(0, prep.shape[0], 256)])
            s, bst = pose_score(emb.reshape(A, p.shape[0], -1), text_feature, group)
            scores.append(s)
            best.append(bst)
        return torch.cat(scores), torch.cat(best)

    def sort_poses_by_score(self, text_feature: torch.Tensor, poses: List[torch.Tensor]) -> tuple:
        """sort_poses_by_score (:97-99): one fresh score per pose in list order, then a stable descending sort.
        Returns (the sorted poses, the scores in list order)."""
        sc, _ = self.scores(torch.stack(poses), text_feature, 1, self.draw_eyes(len(poses)))
        sc = sc.cpu().tolist()
        order = sorted(range(len(poses)), key=lambda i: sc[i], reverse=True)
        return [poses[i] for i in order], sc


class BasePoseGenerator:
    def __init__(self, name: str, assets: Assets, topk: int = 5, smpl_path=None, vposer_path=None):
        self.name = name
        self.topk = topk
        self.assets = assets
        self.scorer = PoseScorer(assets)

    def get_text_feature(self, text: str) -> torch.Tensor:
        return self.scorer.get_text_feature(text)


class VPoserCodebook(BasePoseGenerator):
    """:288-329 with the reference's constructor defaults."""

    def __init__(self, codebook_path="data/codebook.pth", pre_topk=40, filter_threshold=0.07, **kwargs):
        super().__init__(**kwargs)
        cb, emb = load_pose_codebook(codebook_path)
        self.codebook = cb.to(self.assets.device).float().contiguous()
        self.codebook_embedding = emb.to(self.assets.device).float().contiguous()
        self.pre_topk = pre_topk
        self.filter_threshold = filter_threshold
        self.last = {}

    def get_topk_poses(self, text: str) -> torch.Tensor:
        tf = self.get_text_feature(text)
        cos, idx = cosine_topk(self.codebook_embedding, tf, self.pre_topk)
        poses = vposer_decode(self.codebook[idx.long()], self.assets.vposer).reshape(self.pre_topk, -1)
        keep = pose_suppress(poses, self.filter_threshold)
        self.last = dict(cos=cos, topk=idx, keep=keep)
        return poses[keep.long()][:self.topk]


class VPoserRealNVP(BasePoseGenerator):
    """:176-285 with the reference's constructor defaults.  ``get_topk_poses(text, z=...)`` takes the prior draws
    [topk, num_batch * num_sample, dim] instead of drawing them with torch on the device."""

    def __init__(self, dim=32, hdim=256, num_block=8, num_sample=10, num_batch=50, ckpt_path="data/pose_realnvp.pth",
                 **kwargs):
        super().__init__(**kwargs)
        self.dim, self.hdim, self.num_block = dim, hdim, num_block
        self.num_sample, self.num_batch = num_sample, num_batch
        self.weights = pack_realnvp(load_realnvp(ckpt_path), num_block, self.assets.device)
        self.last = {}

    def get_pose(self, text_feature: torch.Tensor, z: Optional[torch.Tensor] = None) -> torch.Tensor:
        """All num_batch x num_sample draws of one candidate in one pass; the per-batch argmax, then the reference's
        running "beats the best so far, starting from 0" over the batches in order."""
        n = self.num_batch * self.num_sample
        if z is None:
            z = torch.randn(n, self.dim, device=self.assets.device)
        x = realnvp_decode(z.to(self.assets.device), text_feature, self.weights)
        poses = vposer_decode(x, self.assets.vposer).reshape(n, -1)
        scores, best = self.scorer.scores(poses, text_feature, self.num_sample, self.scorer.draw_eyes(self.num_batch))
        scores, best = scores.cpu().numpy(), best.cpu().numpy()
        self.last.setdefault("scores", []).append(scores)
        best_pose, best_score = None, 0.0
        for g in range(self.num_batch):
            i = g * self.num_sample + int(best[g])
            if scores[i] > best_score:
                best_pose, best_score = poses[i], float(scores[i])
        if best_pose is None:
            raise RuntimeError(f"VPoserRealNVP: none of the {n} sampled poses scored above 0 against the text")
        self.last.setdefault("best_scores", []).append(best_score)
        return best_pose

    def get_topk_poses(self, text: str, z: Optional[torch.Tensor] = None,
                       text_feature: Optional[torch.Tensor] = None) -> torch.Tensor:
        """:280-285.  ``text_feature`` [512], when given, stands in for the CLIP text encode of ``text``.  Afterwards
        ``self.last`` holds per candidate the scores of all its draws and the best score kept, and the sort's scores
        in candidate order."""
        tf = self.get_text_feature(text) if text_feature is None else text_feature.to(self.assets.device).float()
        self.last = {}
        poses = [self.get_pose(tf, None if z is None else z[i]) for i in range(self.topk)]
        poses, sc = self.scorer.sort_poses_by_score(tf, poses)
        self.last["sort_scores"] = sc
        return torch.stack(poses, 0)


def refusal(conf) -> Optional[str]:
    """Why ``conf`` cannot run here, or None."""
    mode = conf.get_string("general.mode", "pose")
    if mode != "pose":
        return (f"general.mode = {mode}: this command runs the pose stage only; the motion stage runs as python -m "
                "avatarclip_b200.motion")
    return pose_generator_refusal(conf)


def pose_generator_refusal(conf) -> Optional[str]:
    """Why the conf's pose_generator cannot run here, or None."""
    typ = conf.get("pose_generator", {}).get("type", None)
    if typ in OUT_OF_SCOPE:
        return f"pose_generator.type = {typ} is not available: it {OUT_OF_SCOPE[typ]}"
    if typ not in IN_SCOPE:
        return f"pose_generator.type = {typ!r} is unknown (available: {', '.join(IN_SCOPE)})"
    return None


def build_pose_generator(conf: dict, assets: Assets):
    """builder.py:13-22 for the two generators that need no gradient."""
    conf = dict(conf)
    name = conf.pop("type", None)
    if name in OUT_OF_SCOPE:
        raise NotImplementedError(f"{name} is not available: it {OUT_OF_SCOPE[name]}")
    cls = {"VPoserRealNVP": VPoserRealNVP, "VPoserCodebook": VPoserCodebook}.get(name)
    if cls is None:
        raise KeyError(f"unknown pose generator type {name!r}")
    return cls(name=name, assets=assets, **conf)


# ---------------------------------------------------------------- candidate images (visualize.py, unpinned)
def render_candidates(assets: Assets, poses: torch.Tensor) -> np.ndarray:
    """render_pose's picture of each pose: SMPL with global_orient (pi, 0, 0), rotated 180 degrees about x, seen from
    z = 25 with focal 5000 on 512 x 512, grey 0.4 on white.  Drawn by avc_video_render (its own shading; the
    reference's pyrender lights are not restated) -> [N, 512, 512, 3] uint8 RGB."""
    from . import video
    v = smpl_pose_batch(assets.smpl, poses, IMAGE_ORIENT)
    V = v.shape[1]
    # pyrender camera at (0, 0, 25) looking down -z, y up; rotating the mesh 180 degrees about x flips y and z, so the
    # camera frame (x right, y down, z forward) sees (x, y, z + 25) of the unrotated vertices
    cam = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, IMAGE_DEPTH, IMAGE_FOCAL], dtype=np.float32)
    adj = video.adjacency(assets.faces, V)
    grey = torch.full((V, 3), round(IMAGE_GREY * 255), dtype=torch.uint8, device=v.device)
    return video.render(v, assets.faces, adj, grey, np.stack([cam] * v.shape[0]), IMAGE_SIZE, 2).cpu().numpy()


# ---------------------------------------------------------------- CLI (main.py:15-35)
def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(
        prog="python -m avatarclip_b200.animate",
        description="Generate candidate SMPL body poses for the text of an AvatarAnimate conf (main.py, general.mode = "
                    "pose; VPoserCodebook or VPoserRealNVP): writes candidate_%%d.npy and candidate_%%d.jpg into "
                    "general.base_exp_dir.",
        epilog="Files: --codebook (codebook.pth), --realnvp (pose_realnvp.pth) and --uv_obj (smpl_uv.obj) are "
               "AvatarAnimate's data/ files; --vposer is the VPoser v2.0 model directory from human_body_prior "
               "(snapshots/*.ckpt); --clip_model / --bpe are openai's CLIP ViT-B/32 checkpoint and BPE merges file.  "
               "The SMPL .npz holds the arrays " + ", ".join(shapegen.SMPL_NPZ_KEYS) + " (see python -m "
               "avatarclip_b200.shapegen --help for the conversion from an smplx model folder).  A path given by a flag "
               "wins; without the flag a path in the conf's pose_generator block (codebook_path, ckpt_path, "
               "vposer_path) is used, and without either the reference's default shown with the flag.")
    p.add_argument("--conf", type=str, default="./confs/base.conf")
    p.add_argument("--smpl", required=True, help=".npz with the SMPL tensors and faces")
    for flag, what in (("--vposer", "VPoser 2.x model directory"), ("--codebook", "VPoserCodebook's codebook"),
                       ("--realnvp", "VPoserRealNVP's checkpoint")):
        p.add_argument(flag, type=str, default=None,
                       help=f"{what} (default: the conf's path, else {DEFAULT_PATHS[flag.lstrip('-')]})")
    p.add_argument("--uv_obj", type=str, default="data/smpl_uv.obj", help="SMPL mesh with UVs, its .mtl and image")
    p.add_argument("--clip_model", type=str, default="ViT-B-32.pt")
    p.add_argument("--bpe", type=str, default="bpe_simple_vocab_16e6.txt.gz")
    p.add_argument("--seed", type=int, default=None, help="seed numpy's and torch's generators first")
    p.add_argument("--device", default="cuda")
    return p


def parse_args(argv=None):
    """(args, conf, pose_generator kwargs); exits with a message for what cannot run, before any weights are read."""
    from . import conf as conf_mod
    parser = build_parser()
    a = parser.parse_args(argv)
    if not os.path.isfile(a.conf):
        parser.error(f"--conf: no such file: {a.conf}")
    conf = conf_mod.parse_file(a.conf)
    why = refusal(conf)
    if why:
        parser.error(why)
    return a, conf, resolve_pose_paths(parser, a, conf)


def resolve_pose_paths(parser, a, conf) -> dict:
    """The pose_generator kwargs with its weight path resolved (and ``a.vposer``), every file checked to exist."""
    pg = dict(conf["pose_generator"])
    # an explicit flag, else the conf's path, else the reference's default
    pick = lambda flag, key: getattr(a, flag) or pg.get(key) or DEFAULT_PATHS[flag]
    if pg["type"] == "VPoserCodebook":
        pg["codebook_path"] = pick("codebook", "codebook_path")
        need = [("codebook_path", pg["codebook_path"])]
    else:
        pg["ckpt_path"] = pick("realnvp", "ckpt_path")
        need = [("ckpt_path", pg["ckpt_path"])]
    pg.pop("smpl_path", None)
    a.vposer = pick("vposer", "vposer_path")
    pg.pop("vposer_path", None)
    need += [("--smpl", a.smpl), ("--uv_obj", a.uv_obj), ("--clip_model", a.clip_model), ("--bpe", a.bpe)]
    for flag, path in need:
        if not os.path.isfile(path):
            parser.error(f"{flag}: no such file: {path}")
    if not os.path.exists(a.vposer):
        parser.error(f"--vposer: no such directory or file: {a.vposer}")
    return pg


def write_candidates(out_dir: str, poses: torch.Tensor, images: np.ndarray) -> List[str]:
    import cv2
    os.makedirs(out_dir, exist_ok=True)
    written = []
    for i in range(poses.shape[0]):
        npy = os.path.join(out_dir, "candidate_%d.npy" % i)
        np.save(npy, poses[i].detach().cpu().numpy().astype(np.float32))
        jpg = os.path.join(out_dir, "candidate_%d.jpg" % i)
        cv2.imwrite(jpg, cv2.cvtColor(images[i], cv2.COLOR_RGB2BGR))
        written += [npy, jpg]
    return written


def main(argv=None) -> int:
    a, conf, pg = parse_args(argv)
    if a.seed is not None:
        np.random.seed(a.seed)
        torch.manual_seed(a.seed)
    smpl = shapegen.load_smpl_npz(a.smpl)
    clip = shapegen.load_clip(a.clip_model, a.bpe, a.device)
    assets = Assets(smpl, clip, a.vposer, a.uv_obj, a.device)
    text = conf.get_string("general.text")
    out_dir = conf.get_string("general.base_exp_dir")
    gen = build_pose_generator(pg, assets)
    poses = gen.get_topk_poses(text)
    write_candidates(out_dir, poses, render_candidates(assets, poses))
    print(f"{poses.shape[0]} candidate poses for {text!r} written to {out_dir}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
