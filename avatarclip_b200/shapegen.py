"""Host-side mirror of AvatarGen/ShapeGen: the coarse body shape from a text prompt, and its 108-view dataset.

``shape_gen`` (main.py:93-123) encodes a neutral and a target prompt with the CLIP ViT-B/32 text tower, decodes the
zero latent of the shape VAE (``LinearVAE.decode``), renders that mesh once with the SMPL UV texture
(``render_one_batch``, utils.py:9-35), encodes the render with the image tower, and picks the codebook entry whose CLIP
image embedding, seen from the neutral render, points most along the text direction:
``argmax_i normalize(C_i - e) . normalize(t - n)``.  That entry's latent is decoded and written as an OBJ
(``writeOBJ``).  ``render_coarse_shape`` is render.py's second step (render.py:109-139,140-170): the OBJ posed by
``stand_pose.npy`` or the T-pose through ``my_lbs`` and rendered into ``img/NNNN.png`` + ``transforms_train.json``
(``handoff.render_coarse_shape``), the directory ``--mode train`` reads.

Everything on the hot path runs in libavc_b200.so: ``avc_vae_decode``, ``avc_load_textures``, ``avc_raster_textured``,
``avc_clip_prep_nearest``, ``avc_codebook_argmax``, the CLIP towers and ``avc_lbs_fwd``.  No ``clip``, ``smplx`` or
``neural_renderer``: the prompts go through ``ClipTokenizer`` + ``ClipTextTower`` from ``ViT-B-32.pt`` and the BPE
merges file, SMPL comes from an ``.npz`` (see ``--help``).

    python -m avatarclip_b200.shapegen --target_txt "a 3d rendering of a strong man in unreal engine" \\
        --smpl smpl.npz --uv_obj data/smpl_uv.obj --clip_model ViT-B-32.pt --bpe bpe_simple_vocab_16e6.txt.gz \\
        --render_folder output/render
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import sys
from typing import Mapping, NamedTuple, Optional, Union

import numpy as np
import torch
from torch import nn

from . import _lib, drive, handoff

CLIP_SIZE = 224
TEXTURE_SIZE = 8           # utils.py:7,12
IMAGE_SIZE = 256           # Renderer() default
CAMERA_DISTANCE = 2.0      # utils.py:10
CAMERA_AZIMUTH = 150       # utils.py:21: range(150, 160, 10)
SMPL_NPZ_KEYS = drive.SMPL_KEYS + ("faces",)

_bound = None


def _L():
    global _bound
    L = _lib.lib()
    if _bound is None:
        vp, i32, sz = C.c_void_p, C.c_int32, C.c_size_t
        L.avc_vae_decode_workspace_bytes.argtypes = [i32, i32, C.POINTER(sz)]
        L.avc_vae_decode.argtypes = [vp, i32, i32, vp, vp, i32, vp, vp, vp, i32, vp, vp, sz, vp]
        L.avc_load_textures.argtypes = [vp, i32, i32, vp, vp, i32, i32, vp, vp]
        L.avc_raster_textured_workspace_bytes.argtypes = [i32, i32, i32, C.POINTER(sz)]
        L.avc_raster_textured.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp, i32, i32, vp, vp, sz, vp]
        L.avc_clip_prep_nearest.argtypes = [vp, i32, i32, i32, vp, vp]
        L.avc_codebook_argmax.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, sz, vp]
        for n in ("avc_vae_decode_workspace_bytes", "avc_vae_decode", "avc_load_textures",
                  "avc_raster_textured_workspace_bytes", "avc_raster_textured", "avc_clip_prep_nearest",
                  "avc_codebook_argmax"):
            getattr(L, n).restype = C.c_int
        _bound = L
    return L


def _cuda_tensor(t: torch.Tensor, what: str) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.AvcError(f"{what}: avatarclip_b200 has no CPU path")
    return t.detach().float().contiguous()


def _f3(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32).reshape(3))


# ---------------------------------------------------------------- device ops
def vae_decode(z: torch.Tensor, W1, b1, W2, b2, v_template) -> torch.Tensor:
    """``dec2(dec1(z)) + v_template`` (main.py:67-68) for z [B <= 8, L] on the device -> [B, D] fp32."""
    z = _cuda_tensor(z, "vae_decode")
    B, Lz = z.shape
    H, D = W1.shape[0], W2.shape[0]
    if tuple(W1.shape) != (H, Lz) or tuple(W2.shape) != (D, H) or b1.numel() != H or b2.numel() != D \
            or v_template.numel() != D:
        raise _lib.AvcError(f"vae_decode: inconsistent shapes z {tuple(z.shape)}, dec1 {tuple(W1.shape)}, "
                            f"dec2 {tuple(W2.shape)}, v_template {tuple(v_template.shape)}")
    L = _L()
    need = C.c_size_t()
    _lib.check(L.avc_vae_decode_workspace_bytes(B, H, C.byref(need)), "avc_vae_decode_workspace_bytes")
    ws = torch.empty(need.value, dtype=torch.uint8, device=z.device)
    out = torch.empty(B, D, dtype=torch.float32, device=z.device)
    ts = [_cuda_tensor(t, "vae_decode") for t in (W1, b1, W2, b2, v_template)]
    _lib.check(L.avc_vae_decode(_lib.ptr(z), B, Lz, _lib.ptr(ts[0]), _lib.ptr(ts[1]), H, _lib.ptr(ts[2]),
                                _lib.ptr(ts[3]), _lib.ptr(ts[4]), D, _lib.ptr(out), _lib.ptr(ws), ws.numel(),
                                _lib.stream_ptr()), "avc_vae_decode")
    return out


def load_textures(image: torch.Tensor, face_uv: torch.Tensor, is_update: torch.Tensor, textures: torch.Tensor):
    """One material of neural_renderer's load_textures: ``image`` [H,W,3] in [0,1] as stored (row 0 at the top),
    ``face_uv`` [F,3,2], ``is_update`` [F] -> ``textures`` [F,R,R,R,3] updated in place for the faces with
    is_update != 0."""
    img = _cuda_tensor(image, "load_textures")
    uv = _cuda_tensor(face_uv, "load_textures")
    upd = is_update.to(img.device, torch.int32).contiguous()
    if not (textures.is_cuda and textures.is_contiguous() and textures.dtype == torch.float32):
        raise _lib.AvcError("load_textures: textures must be a contiguous float32 CUDA tensor")
    F, R = textures.shape[0], textures.shape[1]
    if img.dim() != 3 or img.shape[2] != 3 or tuple(uv.shape) != (F, 3, 2) or upd.numel() != F \
            or tuple(textures.shape) != (F, R, R, R, 3):
        raise _lib.AvcError("load_textures: expected image [H,W,3], face_uv [F,3,2], is_update [F], "
                            "textures [F,R,R,R,3]")
    _lib.check(_L().avc_load_textures(_lib.ptr(img), img.shape[0], img.shape[1], _lib.ptr(uv), _lib.ptr(upd), F, R,
                                      _lib.ptr(textures), _lib.stream_ptr()), "avc_load_textures")
    return textures


def raster_textured(verts: torch.Tensor, faces: torch.Tensor, textures: torch.Tensor, eye, at=(0.0, 0.0, 0.0),
                    up=(0.0, 1.0, 0.0), image_size: int = IMAGE_SIZE, supersample: int = 2) -> torch.Tensor:
    """neural_renderer ``Renderer(camera_mode='look_at')`` of one textured mesh -> [n, n, 3] (row 0 at the top)."""
    v = _cuda_tensor(verts, "raster_textured").reshape(-1, 3)
    f = faces.to(v.device, torch.int32).contiguous().reshape(-1, 3)
    t = _cuda_tensor(textures, "raster_textured")
    R = t.shape[1]
    if tuple(t.shape) != (f.shape[0], R, R, R, 3):
        raise _lib.AvcError(f"raster_textured: textures must be [F={f.shape[0]}, R, R, R, 3], got {tuple(t.shape)}")
    L = _L()
    need = C.c_size_t()
    _lib.check(L.avc_raster_textured_workspace_bytes(v.shape[0], image_size, supersample, C.byref(need)),
               "avc_raster_textured_workspace_bytes")
    ws = torch.empty(need.value, dtype=torch.uint8, device=v.device)
    rgb = torch.empty(image_size, image_size, 3, dtype=torch.float32, device=v.device)
    e, a, u = _f3(eye), _f3(at), _f3(up)
    fp = lambda x: x.ctypes.data_as(C.c_void_p)
    _lib.check(L.avc_raster_textured(_lib.ptr(v), _lib.ptr(f), _lib.ptr(t), v.shape[0], f.shape[0], R, fp(e), fp(a),
                                     fp(u), image_size, supersample, _lib.ptr(rgb), _lib.ptr(ws), ws.numel(),
                                     _lib.stream_ptr()), "avc_raster_textured")
    return rgb


def clip_prep_nearest(images_hw3: torch.Tensor, size: int = CLIP_SIZE) -> torch.Tensor:
    """``F.interpolate(images, size)`` (nearest) + the CLIP Normalize (main.py:101-103): [B,n,n,3] -> [B,3,size,size]."""
    x = _cuda_tensor(images_hw3, "clip_prep_nearest")
    if x.dim() == 3:
        x = x[None]
    if x.dim() != 4 or x.shape[1] != x.shape[2] or x.shape[3] != 3:
        raise _lib.AvcError(f"clip_prep_nearest: expected [B, n, n, 3], got {tuple(images_hw3.shape)}")
    out = torch.empty(x.shape[0], 3, size, size, dtype=torch.float32, device=x.device)
    _lib.check(_L().avc_clip_prep_nearest(_lib.ptr(x), x.shape[0], x.shape[1], size, _lib.ptr(out), _lib.stream_ptr()),
               "avc_clip_prep_nearest")
    return out


def codebook_argmax(clip_codebook: torch.Tensor, image_emb: torch.Tensor, delta: torch.Tensor):
    """main.py:106-108: (cos [N] = normalize(C - e, dim=1) . normalize(delta), best = first argmax) on the device;
    ``best`` is a host int."""
    Cb = _cuda_tensor(clip_codebook, "codebook_argmax")
    e = _cuda_tensor(image_emb, "codebook_argmax").reshape(-1)
    d = _cuda_tensor(delta, "codebook_argmax").reshape(-1)
    if Cb.dim() != 2 or e.numel() != Cb.shape[1] or d.numel() != Cb.shape[1]:
        raise _lib.AvcError(f"codebook_argmax: codebook [N,D] with embeddings [D]; got {tuple(Cb.shape)}, "
                            f"{e.numel()}, {d.numel()}")
    N, D = Cb.shape
    cos = torch.empty(N, dtype=torch.float32, device=Cb.device)
    best = torch.empty(1, dtype=torch.int32, device=Cb.device)
    ws = torch.empty(8, dtype=torch.uint8, device=Cb.device)
    _lib.check(_L().avc_codebook_argmax(_lib.ptr(Cb), _lib.ptr(e), _lib.ptr(d), N, D, _lib.ptr(cos), _lib.ptr(best),
                                        _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "avc_codebook_argmax")
    return cos, int(best.item())


# ---------------------------------------------------------------- main.py:22-91
class LinearVAE(nn.Module):
    """main.py:22-68, state-dict compatible with ``model_VAE_16.pth`` (``enc1/enc2/dec1/dec2.{weight,bias}``).  Only
    ``decode`` runs (on the device, ``avc_vae_decode``); the encoder is loaded and kept, as the reference does.  The
    layers are created on the meta device: ``create_load_AE`` assigns the checkpoint's tensors."""

    def __init__(self, in_dim, latent_dim, v_template):
        super().__init__()
        self.v_template = v_template
        self.latent_dim = latent_dim
        self.enc1 = nn.Linear(in_dim, 8192, device="meta")
        self.enc2 = nn.Linear(8192, latent_dim * 2, device="meta")
        self.dec1 = nn.Linear(latent_dim, 8192, device="meta")
        self.dec2 = nn.Linear(8192, in_dim, device="meta")

    def decode(self, latent: torch.Tensor) -> torch.Tensor:
        """main.py:67-68: [B, latent_dim] -> [B, V, 3]; batches above 8 are decoded in chunks of 8."""
        z = latent.reshape(-1, self.latent_dim)
        vt = self.v_template.reshape(-1)
        outs = [vae_decode(z[i:i + 8], self.dec1.weight, self.dec1.bias, self.dec2.weight, self.dec2.bias, vt)
                for i in range(0, z.shape[0], 8)]
        return torch.cat(outs).reshape(z.shape[0], -1, 3)


def parse_prompt(prompt):
    """main.py:70-73: ``text[:weight[:stop]]`` split from the right, defaults weight 1 and stop -inf."""
    vals = prompt.rsplit(":", 2)
    vals = vals + ["", "1", "-inf"][len(vals):]
    return vals[0], float(vals[1]), float(vals[2])


def create_load_AE(in_dim, latent_dim, v_template, pth_fname, device="cuda"):
    """main.py:75-79: ``pth_fname`` is a ``model_VAE_16.pth`` path or its state dict."""
    model_AE = LinearVAE(in_dim, latent_dim, v_template)
    sd = pth_fname if isinstance(pth_fname, Mapping) else torch.load(pth_fname, map_location="cpu")
    model_AE.load_state_dict(sd, assign=True)
    model_AE = model_AE.eval().requires_grad_(False).to(device)
    model_AE.v_template = torch.as_tensor(v_template).to(device, torch.float32)
    return model_AE


def load_codebook(fname, device="cuda"):
    """main.py:87-91: the file holds a dict whose first key is the latent tensor [N,16] and whose value is the CLIP
    image embeddings [N,512] (a pickled tensor-keyed dict, hence ``weights_only=False``)."""
    codebook_dict = torch.load(fname, map_location="cpu", weights_only=False)
    for latents, clip_codebook in codebook_dict.items():
        return latents.to(device), clip_codebook.to(device)
    raise ValueError(f"{fname}: the codebook dict is empty")


# ---------------------------------------------------------------- OBJ files (utils.py:37-86)
def writeOBJ(file, V, F, Vt=None, Ft=None):
    """utils.py:37-60's format: ``v x y z`` with each value written by ``str``, then ``vt`` lines, then 1-based
    ``f a b c`` (``f a/ta b/tb c/tc`` with UV faces)."""
    if Vt is not None and len(F) != len(Ft):
        raise ValueError("Inconsistent data, mesh and UV map do not have the same number of faces")
    lines = ["v " + " ".join(str(x) for x in v) for v in V]
    if Vt is not None:
        lines += ["vt " + " ".join(str(x) for x in v) for v in Vt]
    if Ft:
        lines += ["f " + " ".join(f"{i + 1}/{j + 1}" for i, j in zip(f, ft)) for f, ft in zip(F, Ft)]
    else:
        lines += ["f " + " ".join(str(i + 1) for i in f) for f in F]
    with open(file, "w") as fp:
        fp.write("".join(line + "\n" for line in lines))


def readOBJ(file):
    """utils.py:62-86: (V float32 [N,3], F list of 0-based index lists, Vt float32 or None, Ft list or None)."""
    V, Vt, F, Ft = [], [], [], []
    with open(file) as fp:
        for line in fp:
            if line.startswith("v "):
                V.append([float(x) for x in line[2:].split()])
            elif line.startswith("vt "):
                Vt.append([float(x) for x in line[3:].split()])
            elif line.startswith("f "):
                corners = [c.split("/") for c in line[2:].split()]
                corners = [c for c in corners if c[0] != ""]
                F.append([int(c[0]) - 1 for c in corners])
                if "/" in line:
                    Ft.append([int(c[1]) - 1 for c in corners])
    if Ft and len(F) != len(Ft):
        raise ValueError("Inconsistent .obj file, mesh and UV map do not have the same number of faces")
    if not Ft:
        return np.array(V, np.float32), F, None, None
    return np.array(V, np.float32), F, np.array(Vt, np.float32), Ft


# ---------------------------------------------------------------- textures (utils.py:7, nr.load_obj)
def _read_image_rgb01(path: str) -> torch.Tensor:
    import cv2 as cv
    img = cv.imread(path, cv.IMREAD_UNCHANGED)
    if img is None:
        raise FileNotFoundError(f"cannot read the texture image {path}")
    if img.ndim == 2:
        img = np.stack([img] * 3, -1)
    elif img.shape[2] == 4:
        img = cv.cvtColor(img, cv.COLOR_BGRA2RGB)
    else:
        img = cv.cvtColor(img, cv.COLOR_BGR2RGB)
    scale = 65535.0 if img.dtype == np.uint16 else 255.0
    return torch.from_numpy(img.astype(np.float32) / np.float32(scale))


def read_uv_obj(obj_fname: str):
    """The texture half of ``nr.load_obj``: per triangle (fans for polygons) its UV triangle and material name, and the
    ``map_Kd`` image of every material of the ``mtllib`` files (paths relative to the OBJ).  Returns (face_uv [F,3,2]
    float32, materials [F] list, {material: image path})."""
    vt, face_uv, mats, mtls = [], [], [], []
    material = ""
    with open(obj_fname) as fp:
        lines = fp.readlines()
    for line in lines:
        tok = line.split()
        if not tok:
            continue
        if tok[0] == "vt":
            vt.append([float(t) for t in tok[1:3]])
        elif tok[0] == "usemtl":
            material = tok[1]
        elif tok[0] == "mtllib":
            mtls.append(os.path.join(os.path.dirname(obj_fname), tok[1]))
        elif tok[0] == "f":
            ti = [int(c.split("/")[1]) if "/" in c and "//" not in c else 0 for c in tok[1:]]
            for k in range(len(ti) - 2):
                face_uv.append((ti[0], ti[k + 1], ti[k + 2]))
                mats.append(material)
    vt = np.asarray(vt, dtype=np.float32).reshape(-1, 2)
    idx = np.asarray(face_uv, dtype=np.int64).reshape(-1, 3) - 1
    if idx.size and (idx.min() < 0 or idx.max() >= len(vt)):
        raise ValueError(f"{obj_fname}: a face has no UV index or one outside the {len(vt)} vt lines")
    images = {}
    for mtl in mtls:
        name = None
        with open(mtl) as fp:
            for line in fp:
                tok = line.split()
                if len(tok) >= 2 and tok[0] == "newmtl":
                    name = tok[1]
                elif len(tok) >= 2 and tok[0] == "map_Kd" and name is not None:
                    images[name] = os.path.join(os.path.dirname(obj_fname), tok[1])
    return vt[idx], mats, images


def load_obj_textures(obj_fname: str, texture_size: int = TEXTURE_SIZE, device="cuda") -> torch.Tensor:
    """``nr.load_obj(obj_fname, load_texture=True, texture_size)[2]`` (utils.py:7): [F,R,R,R,3] on the device, 1.0 for
    faces whose material has no ``map_Kd`` image."""
    face_uv, mats, images = read_uv_obj(obj_fname)
    if not images:
        raise ValueError(f"{obj_fname}: no material with a map_Kd image (load_obj raises 'Failed to load textures')")
    device = drive._cuda(device)
    F, R = face_uv.shape[0], texture_size
    tex = torch.ones(F, R, R, R, 3, dtype=torch.float32, device=device)
    uv = torch.from_numpy(face_uv).to(device)
    mats = np.asarray(mats)
    for name, path in images.items():
        upd = torch.from_numpy((mats == name).astype(np.int32)).to(device)
        load_textures(_read_image_rgb01(path).to(device), uv, upd, tex)
    return tex


def render_one_batch(v: torch.Tensor, f, texture: torch.Tensor) -> torch.Tensor:
    """utils.py:9-35 without the unused ``steady_image`` / ``detached_images``: each mesh of v [B,V,3] rendered from
    ``get_points_from_angles(2, 0, 150)`` with the UV texture [F,R,R,R,3] -> images [B,3,256,256]."""
    eye = handoff.get_points_from_angles(CAMERA_DISTANCE, 0, CAMERA_AZIMUTH)
    faces = torch.as_tensor(np.asarray(f, dtype=np.int32)).to(v.device)
    imgs = [raster_textured(v[b], faces, texture, eye) for b in range(v.shape[0])]
    return torch.stack(imgs).permute(0, 3, 1, 2).contiguous()


# ---------------------------------------------------------------- SMPL, CLIP
def load_smpl_npz(path: str) -> dict:
    """SMPL tensors from an ``.npz`` with the keys ``SMPL_NPZ_KEYS`` (drive's keys plus ``faces`` [F,3])."""
    with np.load(path) as z:
        d = {k: z[k] for k in SMPL_NPZ_KEYS if k in z.files}
    if "faces" not in d:
        raise ValueError(f"{path}: missing 'faces' (need {list(SMPL_NPZ_KEYS)})")
    drive._check_smpl(d)
    f = np.asarray(d["faces"])
    V = d["v_template"].shape[0]
    if f.ndim != 2 or f.shape[1] != 3 or f.size == 0 or f.min() < 0 or f.max() >= V:
        raise ValueError(f"{path}: faces must be [F, 3] indices into the {V} vertices, got {list(f.shape)}")
    d["faces"] = f.astype(np.int32)
    return d


class ClipModels(NamedTuple):
    image: object
    text: object
    tokenizer: object


def load_clip(clip_model, bpe, device="cuda") -> ClipModels:
    """main.py:81-85 without the ``clip`` package: ``clip_model`` is ``ViT-B-32.pt`` (or a (visual, text) pair of
    state dicts), ``bpe`` the merges file ``bpe_simple_vocab_16e6.txt.gz``."""
    from .clip_text import ClipTextTower, load_clip_model
    from .clip_tokenizer import ClipTokenizer
    from .clip_vit import ClipImageTower
    visual, text = load_clip_model(clip_model) if isinstance(clip_model, (str, os.PathLike)) else clip_model
    return ClipModels(ClipImageTower(visual, device), ClipTextTower(text, device), ClipTokenizer(str(bpe)))


class ShapeGenResult(NamedTuple):
    v: np.ndarray                # [V,3] the chosen shape
    f: np.ndarray                # [F,3]
    zero_beta_v: np.ndarray      # [V,3] the decoded zero latent
    best: int
    cos: torch.Tensor            # [N]
    neutral_image: torch.Tensor  # [1,3,256,256] the render of the zero latent
    image_embed: torch.Tensor    # [512]
    delta_embed: torch.Tensor    # [512]


def run_shape_gen(smpl, AE_path_fname, codebook_fname, neutral_txt, target_txt, clip: ClipModels, uv_obj,
                  device="cuda") -> ShapeGenResult:
    """main.py:93-123 with every intermediate of the search returned.  ``smpl``: ``load_smpl_npz``'s dict (only
    ``v_template`` and ``faces`` are used); ``uv_obj``: ``smpl_uv.obj`` or its [F,R,R,R,3] texture tensor."""
    device = drive._cuda(device)
    vt = torch.as_tensor(smpl["v_template"]).to(device, torch.float32)
    faces = np.asarray(smpl["faces"], dtype=np.int32)
    model_AE = create_load_AE(vt.numel(), 16, vt, AE_path_fname, device)
    codebook, clip_codebook = load_codebook(codebook_fname, device)
    texture = load_obj_textures(uv_obj, TEXTURE_SIZE, device) if isinstance(uv_obj, (str, os.PathLike)) else uv_obj
    if texture.shape[0] != faces.shape[0]:
        raise ValueError(f"the UV texture has {texture.shape[0]} faces, the SMPL mesh {faces.shape[0]}")

    ntxt, _, _ = parse_prompt(neutral_txt)
    ttxt, _, _ = parse_prompt(target_txt)
    ctx = clip.text.context
    nembed = clip.text.encode_text(clip.tokenizer.tokenize(ntxt, context_length=ctx)).float()
    tembed = clip.text.encode_text(clip.tokenizer.tokenize(ttxt, context_length=ctx)).float()
    delta_embed = (tembed - nembed).squeeze(0)

    v = model_AE.decode(torch.zeros(1, 16, device=device))
    zero_beta_v = v.clone()
    images = render_one_batch(v, faces, texture)
    prep = clip_prep_nearest(images.permute(0, 2, 3, 1))
    neutral_image_embed = clip.image.encode_image(prep).float().mean(0)

    cos, best = codebook_argmax(clip_codebook, neutral_image_embed, delta_embed)
    v = model_AE.decode(codebook[best].reshape(1, 16)).cpu().numpy()
    return ShapeGenResult(v.reshape(-1, 3), faces, zero_beta_v.cpu().numpy().reshape(-1, 3), best, cos, images,
                          neutral_image_embed, delta_embed)


def shape_gen(smpl, AE_path_fname, codebook_fname, neutral_txt, target_txt, clip: ClipModels, uv_obj,
              device="cuda"):
    """main.py:93-123: (v [V,3], f [F,3], zero_beta_v [V,3])."""
    r = run_shape_gen(smpl, AE_path_fname, codebook_fname, neutral_txt, target_txt, clip, uv_obj, device)
    return r.v, r.f, r.zero_beta_v


# ---------------------------------------------------------------- render.py
def coarse_shape_pose(pose_type: str, stand_pose: Optional[str] = None) -> np.ndarray:
    """render.py:150-157: ``stand_pose.npy`` as float32, or the T-pose (zeros with pose[0, 0] = pi / 2)."""
    if pose_type == "stand_pose":
        with open(stand_pose, "rb") as f:
            return np.load(f).astype(np.float32)
    if pose_type == "t_pose":
        pose = np.zeros([1, 24, 3], dtype=np.float32)
        pose[:, 0, 0] = np.pi / 2
        return pose
    raise NotImplementedError(pose_type)


def render_coarse_shape(pose, v_shaped, smpl, output_dir, device="cuda") -> str:
    """render.py:109-139: ``v_shaped`` [1,V,3] posed by ``pose`` (axis-angle, 24 joints) through ``my_lbs`` with
    pose2rot=False, then the 108 views + ``transforms_train.json`` of ``handoff.render_coarse_shape``."""
    from .lbs import my_lbs
    s = drive.smpl_tensors(smpl, device)
    nj = s["J_regressor"].shape[0]
    pose_rot = drive.batch_rodrigues(torch.as_tensor(np.asarray(pose, dtype=np.float32)).reshape(-1, 3))
    pose_rot = pose_rot.reshape(1, nj, 3, 3).to(s["v_template"].device)
    vs = torch.as_tensor(v_shaped).to(s["v_template"].device, torch.float32).reshape(1, -1, 3)
    vertices, _ = my_lbs(vs, pose_rot, s["v_template"], None, s["posedirs"], s["J_regressor"], s["parents"],
                         s["lbs_weights"], pose2rot=False)
    return handoff.render_coarse_shape(vertices[0], np.asarray(smpl["faces"], dtype=np.int32), output_dir, device)


# ---------------------------------------------------------------- CLI (main.py:125-152, render.py:140-170)
def output_fname(output_folder: str, target_txt: str) -> str:
    """main.py:147: the target prompt's words joined by ``_``."""
    return os.path.join(output_folder, "_".join(target_txt.split(" ")) + ".obj")


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(
        prog="python -m avatarclip_b200.shapegen",
        description="Generate the coarse SMPL body shape that a text prompt describes (AvatarGen/ShapeGen/main.py) and, "
                    "with --render_folder, its 108-view dataset for --mode train (ShapeGen/render.py).",
        epilog="The SMPL .npz holds the arrays " + ", ".join(SMPL_NPZ_KEYS) + ".  From an smplx model folder:  "
               "python -c \"import smplx, numpy as np; m = smplx.build_layer('models', model_type='smpl', "
               "gender='neutral'); d = {k: getattr(m, k).detach().cpu().numpy() for k in ('v_template', 'posedirs', "
               "'J_regressor', 'parents', 'lbs_weights')}; np.savez('smpl.npz', faces=m.faces.astype('int32'), **d)\"")
    p.add_argument("--AE_path_fname", type=str, default="./data/model_VAE_16.pth")
    p.add_argument("--codebook_fname", type=str, default="./data/codebook.pth")
    p.add_argument("--neutral_txt", type=str, default="a 3d rendering of a person in unreal engine")
    p.add_argument("--target_txt", type=str, default="a 3d rendering of a strong man in unreal engine")
    p.add_argument("--output_folder", type=str, default="./output/coarse_shape")
    p.add_argument("--smpl", required=True, help=".npz with the SMPL tensors and faces (see below)")
    p.add_argument("--uv_obj", type=str, default="./data/smpl_uv.obj",
                   help="SMPL mesh with UVs; its .mtl and texture image are found next to it")
    p.add_argument("--clip_model", type=str, default="ViT-B-32.pt", help="openai's CLIP ViT-B/32 checkpoint")
    p.add_argument("--bpe", type=str, default="bpe_simple_vocab_16e6.txt.gz", help="openai's CLIP BPE merges file")
    p.add_argument("--render_folder", type=str, default=None,
                   help="also write the 108-view dataset of the generated shape here (ShapeGen/render.py)")
    p.add_argument("--pose_type", type=str, choices=["stand_pose", "t_pose"], default="stand_pose")
    p.add_argument("--stand_pose", type=str, default="./output/stand_pose.npy", help="used with --pose_type stand_pose")
    p.add_argument("--device", default="cuda")
    return p


def parse_args(argv=None) -> argparse.Namespace:
    parser = build_parser()
    a = parser.parse_args(argv)
    files = [("--AE_path_fname", a.AE_path_fname), ("--codebook_fname", a.codebook_fname), ("--smpl", a.smpl),
             ("--uv_obj", a.uv_obj), ("--clip_model", a.clip_model), ("--bpe", a.bpe)]
    if a.render_folder is not None and a.pose_type == "stand_pose":
        files.append(("--stand_pose", a.stand_pose))
    for flag, path in files:
        if not os.path.isfile(path):
            parser.error(f"{flag}: no such file: {path}")
    return a


def main(argv=None) -> int:
    a = parse_args(argv)
    try:
        smpl = load_smpl_npz(a.smpl)
    except (ValueError, OSError) as e:
        build_parser().error(f"--smpl: {e}")
    print("Start generating coarse body shape given the target text: {}".format(a.target_txt))
    clip = load_clip(a.clip_model, a.bpe, a.device)
    v, f, _ = shape_gen(smpl, a.AE_path_fname, a.codebook_fname, a.neutral_txt, a.target_txt, clip, a.uv_obj, a.device)
    os.makedirs(a.output_folder, exist_ok=True)
    obj = output_fname(a.output_folder, a.target_txt)
    writeOBJ(obj, v, f)
    print("Results saved in {}".format(obj))
    if a.render_folder is not None:
        pose = coarse_shape_pose(a.pose_type, a.stand_pose)
        v_shaped, _, _, _ = readOBJ(obj)
        render_coarse_shape(pose, v_shaped.reshape(1, -1, 3), smpl, a.render_folder, a.device)
        print("Renderings written to: {}".format(a.render_folder))
    return 0


if __name__ == "__main__":
    sys.exit(main())
