"""AvatarAnimate's ``MotionOptimizer`` with its CLIP term (models/motion_generation.py:249-358, ``clip_coef > 0``): the
paper's motion method, and what ``confs/base.conf`` and the ``confs/motion_ablation/motion_optimizer`` confs run.  The
pose stage's candidates, then the motion VAE decoder's latent optimised by Adam against

    sum_k recon_coef[k] min_t recon(motion[t], pose_k)
    + clip_coef sum_j (st + j P) / T (1 - cos(CLIP(render(SMPL(motion[st + j P]))), text))
    - delta_coef mse(motion[:-1], motion[1:])

with P = ``clip_num_part``, T = ``num_frame`` and, each iteration, ``st = np.random.randint(P)`` and one camera at
azimuth 150, distance 2 and elevation ``np.random.randn() * 0.3``, drawn in that order from numpy's global generator.
Written as ``motion``'s command writes it: ``candidate_%d.npy`` / ``.jpg``, ``motion.npy`` (float32 [T, 69]) and
``motion.mp4``.

One iteration is a fixed sequence of library calls with no host synchronisation:

    avc_motion_clip_forward (decoder -> motion [T, 63]) -> avc_motion_clip_select (the scored frames and weights)
    -> PoseStep.run (SMPL, textured render, CLIP tower, loss, and their backward, one row per scored frame)
    -> avc_motion_clip_backward (recon and delta loss, the CLIP rows' gradient through the rotation chain, the
       decoder's backward, Adam)

It is captured once as a CUDA graph and replayed ``num_iteration`` times.  Every iteration's draws are made on the host
up front; before each replay one device-to-device copy puts that iteration's camera bytes and ``st`` where the graph
reads them, as pose_optimizer does.

    python -m avatarclip_b200.motion_clip --conf confs/base.conf --smpl smpl.npz --uv_obj data/smpl_uv.obj \\
        --clip_model ViT-B-32.pt --bpe bpe_simple_vocab_16e6.txt.gz
"""
from __future__ import annotations

import ctypes as C
import os
import sys
from typing import Mapping, Optional, Tuple

import numpy as np
import torch

from . import _lib, animate, motion, pose_optimizer
from .handoff import get_points_from_angles

CLIP_AZIMUTH = 150.0                 # get_pose_feature(part_poses, (150,))
OPTIMIZER_DEFAULTS = motion.OPTIMIZER_DEFAULTS
ADAM_BETAS, ADAM_EPS = pose_optimizer.ADAM_BETAS, pose_optimizer.ADAM_EPS

_bound = None


def _L():
    global _bound
    L = pose_optimizer._L()
    motion._L()
    if _bound is None:
        vp, i32, f32, sz = C.c_void_p, C.c_int32, C.c_float, C.c_size_t
        P = C.POINTER
        L.avc_motion_clip_init.argtypes = [P(motion.Dims), vp, vp, vp, f32, vp, sz, vp]
        L.avc_motion_clip_forward.argtypes = [P(motion.Dims), vp, vp, vp, vp, sz, vp]
        L.avc_motion_clip_select.argtypes = [vp, i32, i32, f32, vp, i32, vp, vp, vp, vp]
        L.avc_motion_clip_backward.argtypes = [P(motion.Dims), vp, vp, vp, i32, vp, f32, i32, vp, vp, vp, vp, f32,
                                               f32, f32, vp, vp, vp, vp, sz, vp]
        L.avc_motion_clip_latent.argtypes = [P(motion.Dims), vp, vp, vp, vp, sz, vp]
        for n in ("avc_motion_clip_init", "avc_motion_clip_forward", "avc_motion_clip_select",
                  "avc_motion_clip_backward", "avc_motion_clip_latent"):
            getattr(L, n).restype = C.c_int
        _bound = L
    return L


def clip_rows(num_frame: int, clip_num_part: int) -> int:
    """The most frames one iteration scores: len(range(st, num_frame, clip_num_part)) at st = 0."""
    return -(-num_frame // clip_num_part)


def draw_iterations(n_iter: int, clip_num_part: int) -> Tuple[np.ndarray, np.ndarray]:
    """(st_idx int32 [n_iter], elevation [n_iter]) from numpy's global generator in the reference's order: per
    iteration np.random.randint(clip_num_part), then the camera's np.random.randn() * 0.3."""
    st, el = np.empty(n_iter, dtype=np.int32), np.empty(n_iter)
    for i in range(n_iter):
        st[i] = np.random.randint(clip_num_part)
        el[i] = np.random.randn() * animate.ELEVATION_STD
    return st, el


# ---------------------------------------------------------------- device ops
def select(motion_t: torch.Tensor, clip_num_part: int, clip_coef: float, st_idx: torch.Tensor, n_rows: int,
           pose=None, frame=None, weight=None):
    """avc_motion_clip_select: (pose [n_rows, 63], frame [n_rows] int32, weight [n_rows]) of motion [T, 63] and the
    device st_idx [1]."""
    dev = motion_t.device
    pose = torch.empty(n_rows, 63, device=dev) if pose is None else pose
    frame = torch.empty(n_rows, dtype=torch.int32, device=dev) if frame is None else frame
    weight = torch.empty(n_rows, device=dev) if weight is None else weight
    _lib.check(_L().avc_motion_clip_select(_lib.ptr(motion_t), motion_t.shape[0], int(clip_num_part), float(clip_coef),
                                           _lib.ptr(st_idx), int(n_rows), _lib.ptr(pose), _lib.ptr(frame),
                                           _lib.ptr(weight), _lib.stream_ptr()), "avc_motion_clip_select")
    return pose, frame, weight


class ClipMotionStep:
    """The motion side of one iteration on a persistent avc_motion workspace: ``init`` once, then per iteration
    ``forward`` -> (select, the pose rows' loss and gradient) -> ``backward``.  ``motion`` [T, 63] is written by both
    calls; ``loss`` [n_iter] and ``grad`` [latent] (when asked for) by ``backward``."""

    def __init__(self, vae: motion.MotionVAE, poses: torch.Tensor, recon_coef, delta_coef: float, n_iter: int,
                 record_grad: bool = False):
        self.vae, self.dims = vae, vae.dims
        dev = vae.params.device
        p = animate._dev(poses, "ClipMotionStep")
        self.poses = p.reshape(p.shape[0], -1)[:, :3 * motion.N_JOINTS].contiguous()
        K = self.poses.shape[0]
        if len(recon_coef) < K:
            raise _lib.AvcError(f"ClipMotionStep: {len(recon_coef)} recon_coef for {K} poses")
        self.coef = animate._host_f32(list(recon_coef)[:K])
        self.delta_coef = float(delta_coef)
        self.ws = motion._motion_ws(vae)
        self.motion = torch.empty(self.dims.n_frames, 3 * motion.N_JOINTS, device=dev)
        self.loss = torch.empty(n_iter, device=dev)
        self.grad = torch.empty(self.dims.latent, device=dev) if record_grad else None

    def _common(self):
        return C.byref(self.dims), _lib.ptr(self.vae.params), _lib.ptr(self.vae.pe)

    def init(self, latent: torch.Tensor, lr: float):
        z = animate._dev(latent, "ClipMotionStep").reshape(-1)
        if z.numel() != self.dims.latent:
            raise _lib.AvcError(f"ClipMotionStep: latent of {z.numel()} values, the decoder takes {self.dims.latent}")
        _lib.check(_L().avc_motion_clip_init(*self._common(), _lib.ptr(z), float(lr), _lib.ptr(self.ws),
                                             self.ws.numel(), _lib.stream_ptr()), "avc_motion_clip_init")

    def forward(self):
        _lib.check(_L().avc_motion_clip_forward(*self._common(), _lib.ptr(self.motion), _lib.ptr(self.ws),
                                                self.ws.numel(), _lib.stream_ptr()), "avc_motion_clip_forward")

    def backward(self, frame, weight, pose_grad, pose_loss, betas=ADAM_BETAS, eps: float = ADAM_EPS):
        _lib.check(_L().avc_motion_clip_backward(*self._common(), _lib.ptr(self.poses), self.poses.shape[0],
                                                 animate._hp(self.coef), self.delta_coef, frame.shape[0],
                                                 _lib.ptr(frame), _lib.ptr(weight), _lib.ptr(pose_grad),
                                                 _lib.ptr(pose_loss), float(betas[0]), float(betas[1]), float(eps),
                                                 _lib.ptr(self.motion), _lib.ptr(self.loss), _lib.ptr(self.grad),
                                                 _lib.ptr(self.ws), self.ws.numel(), _lib.stream_ptr()),
                   "avc_motion_clip_backward")

    def latent(self) -> torch.Tensor:
        out = torch.empty(self.dims.latent, device=self.motion.device)
        _lib.check(_L().avc_motion_clip_latent(*self._common(), _lib.ptr(out), _lib.ptr(self.ws), self.ws.numel(),
                                               _lib.stream_ptr()), "avc_motion_clip_latent")
        return out


# ---------------------------------------------------------------- the generator
def optimizer_refusal(mg: Mapping, num_frame: int = 60) -> Optional[str]:
    """Why a MotionOptimizer block cannot run on this command, or None."""
    clip_coef = float(mg.get("clip_coef", OPTIMIZER_DEFAULTS["clip_coef"]))
    if not clip_coef > 0:
        return (f"MotionOptimizer with clip_coef = {clip_coef} has no CLIP term: run python -m avatarclip_b200.motion "
                "(this command runs clip_coef > 0)")
    part = int(mg.get("clip_num_part", OPTIMIZER_DEFAULTS["clip_num_part"]))
    if part < 1 or part > num_frame:
        return (f"MotionOptimizer clip_num_part = {part} must be between 1 and num_frame = {num_frame} (above it the "
                "CLIP term scores an empty batch)")
    if int(mg.get("num_iteration", OPTIMIZER_DEFAULTS["num_iteration"])) < 1:
        return "MotionOptimizer num_iteration must be at least 1"
    return motion.adam_refusal(mg, "MotionOptimizer", OPTIMIZER_DEFAULTS["optim_cfg"])


class MotionOptimizer:
    """:249-358 with its CLIP term and the reference's constructor defaults.

    ``get_motion(text, poses, latent=None)``: the initial latent follows motion.MotionOptimizer's policy
    (``torch.randn(latent_dim)`` from torch's CPU generator, or ``latent``); every iteration's (st, elevation) is then
    drawn up front from numpy's global generator in the reference's order."""

    def __init__(self, assets: animate.Assets, name: str = "MotionOptimizer", num_frame: int = 60, **kw):
        cfg = dict(OPTIMIZER_DEFAULTS)
        cfg.update({k: v for k, v in kw.items() if k not in ("smpl_path", "vposer_path")})
        why = optimizer_refusal(cfg, num_frame)
        if why:
            raise NotImplementedError(why)
        self.assets, self.name, self.num_frame, self.cfg = assets, name, num_frame, cfg
        self.vae = motion.load_motion_vae(cfg["ckpt_path"], cfg["latent_dim"], cfg["num_layers"], cfg["num_heads"],
                                          num_frame, assets.device)
        self.last = {}

    def optimise(self, poses: torch.Tensor, latent: torch.Tensor, text_feature: torch.Tensor, st_idx: np.ndarray,
                 elevation: np.ndarray, record_grad: bool = False):
        """len(st_idx) Adam steps of the latent from ``latent``.  Returns (the latent after the last step, the motion
        decoded at the last iteration [T, 63]); self.last holds each iteration's loss (and latent gradient)."""
        c, dev = self.cfg, self.assets.device
        oc = dict(c["optim_cfg"])
        P, T, n = int(c["clip_num_part"]), self.num_frame, len(st_idx)
        R = clip_rows(T, P)
        ms = ClipMotionStep(self.vae, poses.to(dev), c["recon_coef"], c["delta_coef"], n, record_grad)
        step = pose_optimizer.PoseStep(self.assets, R, 1)
        step.set_text(text_feature.to(dev).float())
        # per iteration: the R rows' cameras (one eye), then st; one copy a replay puts a row where the graph reads it
        cb = step.cams.shape[1]
        eyes = np.stack([get_points_from_angles(animate.CAMERA_DISTANCE, e, CLIP_AZIMUTH) for e in elevation])
        cams = pose_optimizer.look_at_cams(np.repeat(eyes[:, None], R, 1), device=dev).view(n, R * cb)
        assert (R * cb) % 4 == 0
        table = torch.cat([cams, torch.from_numpy(np.asarray(st_idx, dtype=np.int32)).view(torch.uint8)
                           .reshape(n, 4).to(dev)], 1)
        cur = table[0].clone()
        step.cams = cur[:R * cb].view(R, cb)
        st_dev = cur[R * cb:].view(torch.int32)
        frame = torch.empty(R, dtype=torch.int32, device=dev)
        weight = torch.empty(R, device=dev)
        grads = torch.empty(n, self.vae.dims.latent, device=dev) if record_grad else None
        betas = tuple(float(b) for b in oc.get("betas", ADAM_BETAS))
        eps = float(oc.get("eps", ADAM_EPS))

        def front():
            ms.forward()
            select(ms.motion, P, float(c["clip_coef"]), st_dev, R, step.pose, frame, weight)
            step.run()

        ms.init(latent.to(dev).float(), float(oc.get("lr", 1e-3)))
        # capture on a side stream after one uncaptured pass without the backward (first-launch set-up)
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            front()
        torch.cuda.current_stream(dev).wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            front()
            ms.backward(frame, weight, step.grad, step.loss, betas, eps)
        for it in range(n):
            cur.copy_(table[it])
            g.replay()
            if grads is not None:
                grads[it].copy_(ms.grad)
        self.last = dict(loss=ms.loss, grad=grads)
        return ms.latent(), ms.motion.clone()

    def get_motion(self, text: str, poses: torch.Tensor, latent: Optional[torch.Tensor] = None,
                   text_feature: Optional[torch.Tensor] = None, record_grad: bool = False) -> torch.Tensor:
        """:306-358 -> [num_frame, 69].  ``text_feature`` [512] stands in for the CLIP text encode of ``text``.
        Afterwards ``self.last`` holds the initial latent, the draws, each iteration's loss (and latent gradient) and
        the final latent."""
        c = self.cfg
        K = poses.shape[0]
        if K > len(c["recon_coef"]):
            raise ValueError(f"MotionOptimizer: {K} candidate poses but {len(c['recon_coef'])} recon_coef entries")
        tf = (animate.PoseScorer(self.assets).get_text_feature(text) if text_feature is None else text_feature)
        z0 = torch.randn(c["latent_dim"]) if latent is None else latent
        st, el = draw_iterations(int(c["num_iteration"]), int(c["clip_num_part"]))
        z, m = self.optimise(poses[:, :63], z0, tf, st, el, record_grad)
        self.last = dict(self.last, latent_init=z0, st_idx=st, elevation=el, latent=z)
        return motion.pose_padding(m)


def refusal(conf) -> Optional[str]:
    """Why ``conf`` cannot run on this command, or None."""
    mode = conf.get_string("general.mode", "pose")
    if mode != "motion":
        return (f"general.mode = {mode}: this command runs the motion stage's MotionOptimizer with its CLIP term; the "
                "pose stage runs as python -m avatarclip_b200.animate (PoseOptimizer confs: python -m "
                "avatarclip_b200.pose_optimizer)")
    why = animate.pose_generator_refusal(conf)
    if why:
        return why
    mg = conf.get("motion_generator", {})
    typ = mg.get("type", None)
    if typ == "MotionInterpolation":
        return "motion_generator.type = MotionInterpolation has no CLIP term: run python -m avatarclip_b200.motion"
    if typ != "MotionOptimizer":
        return f"motion_generator.type = {typ!r} is unknown (this command runs MotionOptimizer with clip_coef > 0)"
    return optimizer_refusal(mg, int(mg.get("num_frame", 60)))


def build_motion_generator(conf: dict, assets: animate.Assets):
    """builder.py:25-33 for MotionOptimizer with its CLIP term."""
    conf = dict(conf)
    name = conf.pop("type", None)
    if name != "MotionOptimizer":
        raise KeyError(f"motion generator type {name!r} does not run on this command")
    return MotionOptimizer(assets, name=name, **conf)


# ---------------------------------------------------------------- CLI (main.py:15-41)
def build_parser():
    p = motion.build_parser()
    p.prog = "python -m avatarclip_b200.motion_clip"
    p.description = ("Generate a motion for the text of an AvatarAnimate conf with MotionOptimizer and its CLIP term "
                     "(main.py, general.mode = motion, clip_coef > 0; confs/base.conf and the motion_optimizer "
                     "confs): writes candidate_%%d.npy / .jpg, motion.npy [num_frame, 69] and motion.mp4 into "
                     "general.base_exp_dir.")
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
    mg["ckpt_path"] = a.motion_vae or mg.get("ckpt_path") or motion.DEFAULT_MOTION_VAE
    if not os.path.isfile(mg["ckpt_path"]):
        parser.error(f"ckpt_path: no such file: {mg['ckpt_path']}")
    return a, conf, pg, mg


def main(argv=None) -> int:
    from . import shapegen
    a, conf, pg, mg = parse_args(argv)
    if a.seed is not None:
        np.random.seed(a.seed)
        torch.manual_seed(a.seed)
    smpl = shapegen.load_smpl_npz(a.smpl)
    clip = shapegen.load_clip(a.clip_model, a.bpe, a.device)
    vp = animate.load_vposer(a.vposer, encoder=False)
    assets = animate.Assets(smpl, clip, vp, a.uv_obj, a.device)
    text = conf.get_string("general.text")
    out_dir = conf.get_string("general.base_exp_dir")
    poses = animate.build_pose_generator(pg, assets).get_topk_poses(text)
    animate.write_candidates(out_dir, poses, animate.render_candidates(assets, poses))
    m = build_motion_generator(mg, assets).get_motion(text, poses)
    motion.write_motion(out_dir, m, motion.render_motion(assets, m))
    print(f"a {m.shape[0]}-frame motion for {text!r} written to {out_dir}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
