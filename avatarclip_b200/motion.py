"""Host-side mirror of AvatarAnimate's motion stage (main.py with ``general.mode = motion``): the pose stage's candidate
poses, then a motion through them, written as ``motion.npy`` (float32 [num_frame, 69], ``pose_padding(motion)``) and
``motion.mp4``.

Two generators of models/motion_generation.py run here:
  * ``MotionInterpolation`` (:100-137): the candidates' VPoser latents (``avc_vposer_encode``), interpolated between the
    anchor frames by the reference's sequential fp32 accumulation, decoded by ``avc_vposer_decode``;
  * ``MotionOptimizer`` (:249-358) with ``clip_coef = 0``: the motion VAE decoder's latent optimised by Adam against
    the reconstruction (and delta) loss, ``avc_motion_optimize``.
A ``MotionOptimizer`` with ``clip_coef > 0`` is refused: its CLIP term (one camera at 150 degrees on every 30th frame)
runs as its own command, ``python -m avatarclip_b200.motion_clip``.  So are the pose generators ``animate`` refuses,
and any optimiser other than Adam.

    python -m avatarclip_b200.motion --conf confs/motion_ablation/baseline/walk.conf --smpl smpl.npz \\
        --clip_model ViT-B-32.pt --bpe bpe_simple_vocab_16e6.txt.gz
"""
from __future__ import annotations

import ctypes as C
import os
import sys
from typing import Mapping, NamedTuple, Optional, Sequence

import numpy as np
import torch

from . import _lib, animate

DEFAULT_MOTION_VAE = "data/motion_vae.pth"      # MotionOptimizer's ckpt_path default
# body_visualizer's imagearray2file writes the reference's motion.mp4; its frame rate is UNPINNED (the package is
# absent): 30 frames per second is assumed
MOTION_FPS = 30.0
IN_SCOPE = ("MotionInterpolation", "MotionOptimizer")
ADAM_KEYS = ("lr", "betas", "eps", "weight_decay", "amsgrad", "maximize", "foreach", "capturable", "differentiable",
             "fused")
OPTIMIZER_DEFAULTS = dict(latent_dim=256, num_layers=4, num_heads=4, ckpt_path=DEFAULT_MOTION_VAE, optim_name="Adam",
                          optim_cfg={"lr": 0.01}, num_iteration=5000, recon_coef=(1, 0.8, 0.6, 0.4, 0.2),
                          clip_coef=0.001, delta_coef=0.01, clip_num_part=30)
N_JOINTS = 21


class Dims(C.Structure):
    _fields_ = [("latent", C.c_int32), ("n_layers", C.c_int32), ("n_heads", C.c_int32), ("ff", C.c_int32),
                ("n_frames", C.c_int32), ("n_out", C.c_int32)]


_bound = None


def _L():
    global _bound
    L = _lib.lib()
    if _bound is None:
        vp, i32, f32, sz = C.c_void_p, C.c_int32, C.c_float, C.c_size_t
        P = C.POINTER
        L.avc_vposer_encode_workspace_bytes.argtypes = [i32, i32, i32, P(sz)]
        L.avc_vposer_encode.argtypes = [vp, i32, i32, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp, vp, sz, vp]
        L.avc_motion_param_count.argtypes = [P(Dims), P(C.c_int64)]
        L.avc_motion_workspace_bytes.argtypes = [P(Dims), P(sz)]
        L.avc_motion_decode.argtypes = [P(Dims), vp, vp, vp, vp, vp, sz, vp]
        L.avc_motion_optimize.argtypes = [P(Dims), vp, vp, vp, i32, vp, f32, f32, f32, f32, f32, i32, vp, vp, vp, vp,
                                          vp, vp, sz, vp]
        for n in ("avc_vposer_encode_workspace_bytes", "avc_vposer_encode", "avc_motion_param_count",
                  "avc_motion_workspace_bytes", "avc_motion_decode", "avc_motion_optimize"):
            getattr(L, n).restype = C.c_int
        _bound = L
    return L


# ---------------------------------------------------------------- VPoser encoder
def vposer_encode(x: torch.Tensor, enc: Mapping[str, torch.Tensor]) -> torch.Tensor:
    """VPoser.encode(x).mean for body poses x [B, 63] -> [B, latent]."""
    x = animate._dev(x, "vposer_encode")
    x = x.reshape(x.shape[0], -1)
    g = lambda k: animate._dev(enc[f"encoder_net.{k}"], "vposer_encode")
    bn = lambda i: torch.stack([g(f"{i}.{k}") for k in ("weight", "bias", "running_mean", "running_var")]).contiguous()
    W1, Wmu = g("2.weight"), g("8.mu.weight")
    H, NI, Lz = W1.shape[0], W1.shape[1], Wmu.shape[0]
    if x.shape[1] != NI:
        raise _lib.AvcError(f"vposer_encode: poses {tuple(x.shape)} against encoder_net.2 {tuple(W1.shape)}")
    bn1, bn2 = bn(1), bn(4)
    L = _L()
    ws = torch.empty(animate._ws(L.avc_vposer_encode_workspace_bytes, NI, H, Lz), dtype=torch.uint8, device=x.device)
    mu = torch.empty(x.shape[0], Lz, device=x.device)
    _lib.check(L.avc_vposer_encode(_lib.ptr(x), x.shape[0], NI, _lib.ptr(bn1), _lib.ptr(W1), _lib.ptr(g("2.bias")), H,
                                   _lib.ptr(bn2), _lib.ptr(g("6.weight")), _lib.ptr(g("6.bias")),
                                   _lib.ptr(g("7.weight")), _lib.ptr(g("7.bias")), _lib.ptr(Wmu),
                                   _lib.ptr(g("8.mu.bias")), Lz, _lib.ptr(mu), _lib.ptr(ws), ws.numel(),
                                   _lib.stream_ptr()), "avc_vposer_encode")
    return mu


def interpolate_latents(latents: np.ndarray, anchor_position: Sequence[int], num_frame: int) -> np.ndarray:
    """MotionInterpolation.get_motion's latents (:124-135): between consecutive anchors, delta = (end - start) /
    interval and latent[s + j + 1] = latent[s + j] + delta, accumulated in that order in fp32."""
    lat = np.asarray(latents, dtype=np.float32)
    out = np.zeros((num_frame, lat.shape[1]), dtype=np.float32)
    out[0] = lat[0]
    for i in range(1, len(anchor_position)):
        s, e = anchor_position[i - 1], anchor_position[i]
        delta = (lat[i] - lat[i - 1]) / np.float32(e - s)
        for j in range(e - s):
            out[s + j + 1] = out[s + j] + delta
    return out


# ---------------------------------------------------------------- motion VAE decoder
LAYER_KEYS = ("self_attn.in_proj_weight", "self_attn.in_proj_bias", "self_attn.out_proj.weight",
              "self_attn.out_proj.bias", "multihead_attn.in_proj_weight", "multihead_attn.in_proj_bias",
              "multihead_attn.out_proj.weight", "multihead_attn.out_proj.bias", "linear1.weight", "linear1.bias",
              "linear2.weight", "linear2.bias", "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias",
              "norm3.weight", "norm3.bias")


class MotionVAE(NamedTuple):
    """The decoder on the device: ``params`` in avc_motion_decode's layout, ``pe`` the positional rows [T, latent]."""
    dims: Dims
    params: torch.Tensor
    pe: torch.Tensor


def positional_table(num_frame: int, d_model: int) -> torch.Tensor:
    """SinusoidalPositionalEncoding's pe[:num_frame] (:145-152), computed in fp32 as the module computes it."""
    pe = torch.zeros(num_frame, d_model)
    position = torch.arange(0, num_frame, dtype=torch.float).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2).float() * (-np.log(10000.0) / d_model))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


def load_motion_vae(path, latent_dim: int = 256, num_layers: int = 4, num_heads: int = 4, num_frame: int = 60,
                    device="cuda") -> MotionVAE:
    """``motion_vae.pth``'s ``state_dict`` (or the state dict itself), the decoder's keys only (``get_motion`` never
    calls the encoder).  The reference loads with ``strict=False``, so a missing key would silently keep a random
    initialisation; here a missing key is an error.  ``decoder.pos_encoder.pe`` is taken from the checkpoint when it
    is there, else the module's own table."""
    data = path if isinstance(path, Mapping) else torch.load(path, map_location="cpu", weights_only=False)
    sd = data.get("state_dict", data)
    D, F = latent_dim, 4 * latent_dim
    pre = "decoder.seqTransDecoder.layers."
    keys = [f"{pre}{l}.{k}" for l in range(num_layers) for k in LAYER_KEYS] + ["decoder.final.weight",
                                                                               "decoder.final.bias"]
    missing = [k for k in keys if k not in sd]
    if missing:
        raise ValueError(f"motion VAE weights: missing {', '.join(missing[:4])}" +
                         (f" and {len(missing) - 4} more" if len(missing) > 4 else ""))
    t = lambda k: torch.as_tensor(sd[k]).float()
    n_out = t("decoder.final.weight").shape[0]
    want = {"self_attn.in_proj_weight": (3 * D, D), "self_attn.out_proj.weight": (D, D),
            "multihead_attn.in_proj_weight": (3 * D, D), "multihead_attn.out_proj.weight": (D, D),
            "linear1.weight": (F, D), "linear2.weight": (D, F)}
    for l in range(num_layers):
        for k, shape in want.items():
            if tuple(t(f"{pre}{l}.{k}").shape) != shape:
                raise ValueError(f"motion VAE weights: {pre}{l}.{k} is {tuple(t(f'{pre}{l}.{k}').shape)}, expected "
                                 f"{shape} for latent_dim {D}")
    if tuple(t("decoder.final.weight").shape) != (n_out, D):
        raise ValueError(f"motion VAE weights: decoder.final.weight is {tuple(t('decoder.final.weight').shape)}")
    parts = []
    for l in range(num_layers):
        g = lambda k: t(f"{pre}{l}.{k}").reshape(-1)
        parts += [g("self_attn.in_proj_weight"), g("self_attn.in_proj_bias"), g("self_attn.out_proj.weight"),
                  g("self_attn.out_proj.bias"), g("multihead_attn.in_proj_weight")[2 * D * D:],
                  g("multihead_attn.in_proj_bias")[2 * D:], g("multihead_attn.out_proj.weight"),
                  g("multihead_attn.out_proj.bias")] + [g(k) for k in LAYER_KEYS[8:]]
    parts += [t("decoder.final.weight").reshape(-1), t("decoder.final.bias").reshape(-1)]
    dims = Dims(D, num_layers, num_heads, F, num_frame, n_out)
    count = C.c_int64()
    rc = _L().avc_motion_param_count(C.byref(dims), C.byref(count))
    if rc == -1:
        raise ValueError(f"motion VAE: latent_dim {D}, {num_layers} layers, {num_heads} heads, {num_frame} frames, "
                         f"{n_out} outputs is a shape the device decoder does not support")
    _lib.check(rc, "avc_motion_param_count")
    params = torch.cat(parts)
    if params.numel() != count.value:
        raise ValueError(f"motion VAE weights: {params.numel()} values, the layout needs {count.value}")
    if "decoder.pos_encoder.pe" in sd:
        pe = t("decoder.pos_encoder.pe").reshape(-1, D)[:num_frame]
    else:
        pe = positional_table(num_frame, D)
    dev = animate.drive._cuda(device)
    return MotionVAE(dims, params.to(dev).contiguous(), pe.to(dev).contiguous())


def _motion_ws(w: MotionVAE) -> torch.Tensor:
    return torch.empty(animate._ws(_L().avc_motion_workspace_bytes, C.byref(w.dims)), dtype=torch.uint8,
                       device=w.params.device)


def motion_decode(latent: torch.Tensor, w: MotionVAE) -> torch.Tensor:
    """MotionOptimizer.decode(latent [latent_dim]) -> [num_frame, 63]."""
    z = animate._dev(latent, "motion_decode").reshape(-1)
    if z.numel() != w.dims.latent:
        raise _lib.AvcError(f"motion_decode: latent of {z.numel()} values, the decoder takes {w.dims.latent}")
    ws = _motion_ws(w)
    out = torch.empty(w.dims.n_frames, 3 * N_JOINTS, device=z.device)
    _lib.check(_L().avc_motion_decode(C.byref(w.dims), _lib.ptr(w.params), _lib.ptr(w.pe), _lib.ptr(z), _lib.ptr(out),
                                      _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "avc_motion_decode")
    return out


def motion_optimize(w: MotionVAE, poses: torch.Tensor, recon_coef: Sequence[float], delta_coef: float,
                    latent_init: torch.Tensor, n_iter: int, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                    record_loss: bool = False, return_grad: bool = False):
    """``n_iter`` iterations of get_motion's loop without the CLIP term from ``latent_init``, on the device without a
    host wait.  Returns (the latent after the last step, the motion decoded at the last iteration [num_frame, 63],
    each iteration's loss [n_iter] or None), and with ``return_grad`` the last iteration's latent gradient."""
    p = animate._dev(poses, "motion_optimize")
    p = p.reshape(p.shape[0], -1)[:, :3 * N_JOINTS].contiguous()
    z0 = animate._dev(latent_init, "motion_optimize").reshape(-1)
    K = p.shape[0]
    if z0.numel() != w.dims.latent or len(recon_coef) < K:
        raise _lib.AvcError(f"motion_optimize: latent of {z0.numel()} values for {w.dims.latent}, {len(recon_coef)} "
                            f"recon_coef for {K} poses")
    ws = _motion_ws(w)
    coef = animate._host_f32(list(recon_coef)[:K])
    z = torch.empty_like(z0)
    motion = torch.empty(w.dims.n_frames, 3 * N_JOINTS, device=z0.device)
    loss = torch.empty(n_iter, device=z0.device) if record_loss else None
    grad = torch.empty_like(z0) if return_grad else None
    _lib.check(_L().avc_motion_optimize(C.byref(w.dims), _lib.ptr(w.params), _lib.ptr(w.pe), _lib.ptr(p), K,
                                        animate._hp(coef), float(delta_coef), float(lr), float(betas[0]),
                                        float(betas[1]), float(eps), int(n_iter), _lib.ptr(z0), _lib.ptr(z),
                                        _lib.ptr(motion), _lib.ptr(loss), _lib.ptr(grad), _lib.ptr(ws), ws.numel(),
                                        _lib.stream_ptr()), "avc_motion_optimize")
    return (z, motion, loss, grad) if return_grad else (z, motion, loss)


def pose_padding(pose: torch.Tensor) -> torch.Tensor:
    """[..., 63] -> [..., 69] with six zeros (motion_generation.py:27-32)."""
    if pose.shape[-1] == 63:
        pose = torch.cat((pose, torch.zeros_like(pose)[..., :6]), dim=-1)
    return pose


# ---------------------------------------------------------------- generators
class MotionInterpolation:
    """:100-137 with the reference's defaults."""

    def __init__(self, vposer: Mapping[str, torch.Tensor], anchor_position=(0, 14, 29, 44, 59), num_frame: int = 60,
                 name: str = "MotionInterpolation", **_paths):
        anchor_position = tuple(int(a) for a in anchor_position)
        if anchor_position[0] != 0 or anchor_position[-1] != num_frame - 1:
            raise ValueError(f"MotionInterpolation: anchor_position {list(anchor_position)} must start at 0 and end at "
                             f"num_frame - 1 = {num_frame - 1}")
        self.name, self.vposer, self.anchor_position, self.num_frame = name, vposer, anchor_position, num_frame

    def get_motion(self, text: str, poses: torch.Tensor) -> torch.Tensor:
        poses = poses[:, :63]
        if len(self.anchor_position) > poses.shape[0]:
            raise ValueError(f"MotionInterpolation: {len(self.anchor_position)} anchors but only {poses.shape[0]} "
                             "candidate poses")
        lat = vposer_encode(poses, self.vposer).cpu().numpy()
        z = torch.from_numpy(interpolate_latents(lat, self.anchor_position, self.num_frame)).to(poses.device)
        motion = animate.vposer_decode(z, self.vposer).reshape(self.num_frame, 63)
        return pose_padding(motion)


class MotionOptimizer:
    """:249-358 without the CLIP term (``clip_coef`` must be 0), with the reference's defaults.

    ``get_motion(text, poses, latent=None)``: by default the initial latent is ``torch.randn(latent_dim)`` from torch's
    CPU generator, as the reference draws it.  The reference's seed -> latent mapping is not reproduced: there the draw
    follows the construction of modules from packages that are absent here (clip, smplx, VPoser), which consume the
    generator first.  Pass ``latent`` to start from a given one."""

    def __init__(self, device="cuda", name: str = "MotionOptimizer", num_frame: int = 60, **kw):
        cfg = dict(OPTIMIZER_DEFAULTS)
        cfg.update({k: v for k, v in kw.items() if k not in ("smpl_path", "vposer_path")})
        why = optimizer_refusal(cfg)
        if why:
            raise NotImplementedError(why)
        self.name, self.num_frame, self.cfg = name, num_frame, cfg
        self.vae = load_motion_vae(cfg["ckpt_path"], cfg["latent_dim"], cfg["num_layers"], cfg["num_heads"], num_frame,
                                   device)
        self.last = {}

    def get_motion(self, text: str, poses: torch.Tensor, latent: Optional[torch.Tensor] = None,
                   record_loss: bool = False) -> torch.Tensor:
        c = self.cfg
        K = poses.shape[0]
        if K > len(c["recon_coef"]):
            raise ValueError(f"MotionOptimizer: {K} candidate poses but {len(c['recon_coef'])} recon_coef entries")
        z0 = torch.randn(c["latent_dim"]) if latent is None else latent
        oc = dict(c["optim_cfg"])
        z, motion, loss = motion_optimize(self.vae, poses, c["recon_coef"], c["delta_coef"],
                                          z0.to(self.vae.params.device), c["num_iteration"], oc.get("lr", 1e-3),
                                          tuple(oc.get("betas", (0.9, 0.999))), oc.get("eps", 1e-8), record_loss)
        self.last = dict(latent_init=z0, latent=z, loss=loss)
        return pose_padding(motion)


def adam_refusal(mg: Mapping, who: str, default_cfg: Mapping) -> Optional[str]:
    """Why the optimiser settings (optim_name, optim_cfg) of ``who``'s conf block cannot run here, or None: only plain
    torch.optim.Adam runs (avc_adam_step_dev)."""
    name = mg.get("optim_name", "Adam")
    if name != "Adam":
        return f"{who} optim_name = {name} is not available: only Adam runs"
    cfg = dict(mg.get("optim_cfg", default_cfg))
    bad = sorted(set(cfg) - set(ADAM_KEYS))
    if bad:
        return f"{who} optim_cfg keys {bad} are not Adam's"
    if cfg.get("weight_decay", 0) or cfg.get("amsgrad", False) or cfg.get("maximize", False):
        return f"{who} optim_cfg: weight_decay, amsgrad and maximize are not available (plain Adam runs)"
    return None


def optimizer_refusal(mg: Mapping) -> Optional[str]:
    """Why a MotionOptimizer block cannot run here, or None."""
    clip_coef = float(mg.get("clip_coef", OPTIMIZER_DEFAULTS["clip_coef"]))
    if clip_coef > 0:
        return (f"MotionOptimizer with clip_coef = {clip_coef} does not run on this command: its CLIP term needs the "
                "rasteriser's gradient, so it runs as its own command, python -m avatarclip_b200.motion_clip "
                "(clip_coef = 0 runs here)")
    return adam_refusal(mg, "MotionOptimizer", OPTIMIZER_DEFAULTS["optim_cfg"])


def refusal(conf) -> Optional[str]:
    """Why ``conf`` cannot run as a motion, or None."""
    mode = conf.get_string("general.mode", "pose")
    if mode != "motion":
        return (f"general.mode = {mode}: this command runs the motion stage; run python -m avatarclip_b200.animate "
                "(PoseOptimizer confs: python -m avatarclip_b200.pose_optimizer)")
    why = animate.pose_generator_refusal(conf)
    if why:
        return why
    mg = conf.get("motion_generator", {})
    typ = mg.get("type", None)
    if typ not in IN_SCOPE:
        return f"motion_generator.type = {typ!r} is unknown (available: {', '.join(IN_SCOPE)})"
    if typ == "MotionOptimizer":
        return optimizer_refusal(mg)
    T = int(mg.get("num_frame", 60))
    anchors = list(mg.get("anchor_position", (0, 14, 29, 44, 59)))
    if anchors[0] != 0 or anchors[-1] != T - 1:
        return f"MotionInterpolation anchor_position {anchors} must start at 0 and end at num_frame - 1 = {T - 1}"
    return None


def build_motion_generator(conf: dict, vposer: Mapping[str, torch.Tensor], device="cuda"):
    """builder.py:25-33 for the two generators without a CLIP term."""
    conf = dict(conf)
    name = conf.pop("type", None)
    if name == "MotionInterpolation":
        return MotionInterpolation(vposer=vposer, name=name, **conf)
    if name == "MotionOptimizer":
        return MotionOptimizer(device=device, name=name, **conf)
    raise KeyError(f"unknown motion generator type {name!r}")


# ---------------------------------------------------------------- CLI (main.py:15-41)
def build_parser():
    p = animate.build_parser()
    p.prog = "python -m avatarclip_b200.motion"
    p.description = ("Generate a motion for the text of an AvatarAnimate conf (main.py, general.mode = motion; "
                     "MotionInterpolation, or MotionOptimizer with clip_coef = 0): writes candidate_%%d.npy / .jpg, "
                     "motion.npy [num_frame, 69] and motion.mp4 into general.base_exp_dir.")
    p.epilog += ("  --motion_vae is AvatarAnimate's data/motion_vae.pth (MotionOptimizer); without the flag the conf's "
                 "motion_generator.ckpt_path, else the default.  motion.mp4 plays at %g frames per second." % MOTION_FPS)
    p.add_argument("--motion_vae", type=str, default=None,
                   help=f"MotionOptimizer's checkpoint (default: the conf's ckpt_path, else {DEFAULT_MOTION_VAE})")
    return p


def parse_args(argv=None):
    """(args, conf, pose_generator kwargs, motion_generator kwargs); exits with a message for what cannot run, before
    any file but the conf is read."""
    from . import conf as conf_mod
    parser = build_parser()
    a = parser.parse_args(argv)
    if not os.path.isfile(a.conf):
        parser.error(f"--conf: no such file: {a.conf}")
    conf = conf_mod.parse_file(a.conf)
    why = refusal(conf)
    if why:
        parser.error(why)
    pg = animate.resolve_pose_paths(parser, a, conf)
    mg = dict(conf["motion_generator"])
    mg.pop("smpl_path", None)
    mg.pop("vposer_path", None)
    if mg["type"] == "MotionOptimizer":
        mg["ckpt_path"] = a.motion_vae or mg.get("ckpt_path") or DEFAULT_MOTION_VAE
        if not os.path.isfile(mg["ckpt_path"]):
            parser.error(f"ckpt_path: no such file: {mg['ckpt_path']}")
    return a, conf, pg, mg


def render_motion(assets: animate.Assets, motion: torch.Tensor) -> np.ndarray:
    """visualize.render_motion's frames: each frame drawn as animate's candidate images are -> [F, 512, 512, 3]."""
    return animate.render_candidates(assets, motion)


def write_motion(out_dir: str, motion: torch.Tensor, frames: np.ndarray) -> list:
    from . import video
    os.makedirs(out_dir, exist_ok=True)
    npy = os.path.join(out_dir, "motion.npy")
    np.save(npy, motion.detach().cpu().numpy().astype(np.float32))
    mp4 = os.path.join(out_dir, "motion.mp4")
    video.write_video(iter(frames), mp4, MOTION_FPS)
    return [npy, mp4]


def main(argv=None) -> int:
    from . import shapegen
    a, conf, pg, mg = parse_args(argv)
    if a.seed is not None:
        np.random.seed(a.seed)
        torch.manual_seed(a.seed)
    smpl = shapegen.load_smpl_npz(a.smpl)
    clip = shapegen.load_clip(a.clip_model, a.bpe, a.device)
    vp = animate.load_vposer(a.vposer, encoder=mg["type"] == "MotionInterpolation")
    assets = animate.Assets(smpl, clip, vp, a.uv_obj, a.device)
    text = conf.get_string("general.text")
    out_dir = conf.get_string("general.base_exp_dir")
    poses = animate.build_pose_generator(pg, assets).get_topk_poses(text)
    animate.write_candidates(out_dir, poses, animate.render_candidates(assets, poses))
    gen = build_motion_generator(mg, {k: v.to(assets.device) for k, v in vp.items()}, assets.device)
    motion = gen.get_motion(text, poses)
    write_motion(out_dir, motion, render_motion(assets, motion))
    print(f"a {motion.shape[0]}-frame motion for {text!r} written to {out_dir}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
