"""AvatarAnimate's ``PoseOptimizer`` (models/pose_generation.py:102-135) on the GPU: SMPL body poses optimised by Adam
against a text prompt, written as ``candidate_%d.npy`` (69 float32 values, ``pose_padding``) and ``candidate_%d.jpg``.

Each of the ``topk`` candidates starts from ``torch.randn(63)`` and takes ``num_iteration`` Adam steps on
``1 - cosine(mean over 5 cameras of encode_image(render(SMPL(pose))), text_feature)``; the candidates are then sorted by
a fresh score (``PoseScorer.sort_poses_by_score``).  The ``topk`` candidates are independent, so they run as one batch
of rows: each row's gradient is that of its own loss, and Adam is elementwise.

One iteration is a fixed sequence of library calls with no host synchronisation:

    avc_smpl_pose_batch -> avc_raster_textured_batch_dev -> avc_clip_prep_nearest -> avc_clip_loss_fwd (tower)
    -> avc_pose_clip_loss -> avc_clip_loss_bwd -> avc_clip_prep_nearest_bwd -> avc_raster_textured_batch_bwd
    -> avc_smpl_pose_batch_bwd -> avc_adam_step_dev

It is captured once as a CUDA graph and replayed ``num_iteration`` times.  The cameras follow the trainer's pattern of
device-resident per-step inputs: every iteration's cameras (5 random elevations per candidate per iteration, drawn
from numpy's global generator in the reference's order) are made once into device memory, and before each replay one
device-to-device copy puts that iteration's cameras where the graph reads them.  That keeps the graph free of host
copies and leaves the draw order on the host, where the reference makes it.

    python -m avatarclip_b200.pose_optimizer --conf confs/pose_ablation/pose_optimizer/cry.conf --smpl smpl.npz \\
        --uv_obj data/smpl_uv.obj --clip_model ViT-B-32.pt --bpe bpe_simple_vocab_16e6.txt.gz
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import sys
from typing import Mapping, Optional

import numpy as np
import torch

from . import _lib, animate, motion, shapegen, video

OPTIMIZER_DEFAULTS = dict(optim_name="Adam", optim_cfg={"lr": 0.01}, num_iteration=500, topk=5)
ADAM_BETAS, ADAM_EPS = (0.9, 0.999), 1e-8      # torch.optim.Adam's defaults
POSE_DIM = 63

_bound = None


def _L():
    global _bound
    L = animate._L()
    shapegen._L()                              # binds avc_clip_prep_nearest
    if _bound is None:
        vp, i32, sz = C.c_void_p, C.c_int32, C.c_size_t
        P = C.POINTER
        L.avc_look_at_cam_bytes.argtypes = [P(sz)]
        L.avc_look_at_cams.argtypes = [vp, i32, vp, vp, i32, i32, vp, vp]
        L.avc_raster_textured_batch_dev.argtypes = [vp, i32, i32, vp, vp, i32, i32, i32, vp, i32, i32, i32, vp, vp, sz,
                                                    vp]
        L.avc_raster_textured_batch_bwd_workspace_bytes.argtypes = [i32, i32, i32, i32, P(sz)]
        L.avc_raster_textured_batch_bwd.argtypes = [vp, i32, i32, vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, vp, vp,
                                                    vp, sz, vp, sz, vp]
        L.avc_smpl_pose_batch_bwd_workspace_bytes.argtypes = [i32, i32, i32, P(sz)]
        L.avc_smpl_pose_batch_bwd.argtypes = [vp, vp, vp, vp, vp, i32, i32, vp, i32, i32, vp, vp, vp, vp, vp, sz, vp]
        L.avc_clip_prep_nearest_bwd.argtypes = [vp, i32, i32, i32, vp, vp]
        L.avc_pose_clip_loss.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp]
        for n in ("avc_look_at_cam_bytes", "avc_look_at_cams", "avc_raster_textured_batch_dev",
                  "avc_raster_textured_batch_bwd_workspace_bytes", "avc_raster_textured_batch_bwd",
                  "avc_smpl_pose_batch_bwd_workspace_bytes", "avc_smpl_pose_batch_bwd", "avc_clip_prep_nearest_bwd",
                  "avc_pose_clip_loss"):
            getattr(L, n).restype = C.c_int
        _bound = L
    return L


_hp, _host_f32, _ws, _dev = animate._hp, animate._host_f32, animate._ws, animate._dev


# ---------------------------------------------------------------- device ops
def look_at_cams(eyes, image_size: int = shapegen.IMAGE_SIZE, supersample: int = 2, at=(0.0, 0.0, 0.0),
                 up=(0.0, 1.0, 0.0), device="cuda") -> torch.Tensor:
    """The cameras of eyes [..., 3] as avc_raster_textured_batch makes them -> device bytes [N, cam_bytes]."""
    L = _L()
    e = _host_f32(eyes).reshape(-1, 3)
    nb = _ws(L.avc_look_at_cam_bytes)
    out = torch.empty(e.shape[0], nb, dtype=torch.uint8, device=device)
    _lib.check(L.avc_look_at_cams(_hp(e), e.shape[0], _hp(_host_f32(at).reshape(3)), _hp(_host_f32(up).reshape(3)),
                                  image_size, supersample, _lib.ptr(out), _lib.stream_ptr()), "avc_look_at_cams")
    return out


def raster_fwd_workspace(V: int, A: int, B: int, group: int, image_size: int, supersample: int, device) -> torch.Tensor:
    ng = (B + group - 1) // group
    return torch.empty(_ws(_L().avc_raster_textured_batch_workspace_bytes, V, A * B, ng * A, image_size, supersample),
                       dtype=torch.uint8, device=device)


def raster_bwd_workspace(F: int, A: int, B: int, image_size: int, supersample: int, device) -> torch.Tensor:
    return torch.empty(_ws(_L().avc_raster_textured_batch_bwd_workspace_bytes, F, A * B, image_size, supersample),
                       dtype=torch.uint8, device=device)


def raster_textured_batch_dev(verts, faces, textures, cams, A: int, group: int, rgb, ws,
                              image_size: int = shapegen.IMAGE_SIZE, supersample: int = 2):
    """avc_raster_textured_batch_dev into rgb [A, B, n, n, 3], the cameras (look_at_cams) in device memory."""
    B, V = verts.shape[0], verts.shape[1]
    _lib.check(_L().avc_raster_textured_batch_dev(_lib.ptr(verts), B, group, _lib.ptr(faces), _lib.ptr(textures), V,
                                                  faces.shape[0], textures.shape[1], _lib.ptr(cams), A, image_size,
                                                  supersample, _lib.ptr(rgb), _lib.ptr(ws), ws.numel(),
                                                  _lib.stream_ptr()), "avc_raster_textured_batch_dev")
    return rgb


def raster_textured_batch_bwd(verts, faces, textures, adj: video.Adjacency, A: int, group: int, g_rgb, fwd_ws, g_verts,
                              ws, image_size: int = shapegen.IMAGE_SIZE, supersample: int = 2):
    """avc_raster_textured_batch_bwd: g_verts [B, V, 3] from g_rgb [A, B, n, n, 3], after the forward that used fwd_ws."""
    B, V = verts.shape[0], verts.shape[1]
    _lib.check(_L().avc_raster_textured_batch_bwd(_lib.ptr(verts), B, group, _lib.ptr(faces), _lib.ptr(textures), V,
                                                  faces.shape[0], textures.shape[1], A, image_size, supersample,
                                                  _lib.ptr(adj.offsets), _lib.ptr(adj.vf), _lib.ptr(g_rgb),
                                                  _lib.ptr(g_verts), _lib.ptr(fwd_ws), fwd_ws.numel(), _lib.ptr(ws),
                                                  ws.numel(), _lib.stream_ptr()), "avc_raster_textured_batch_bwd")
    return g_verts


def smpl_pose_batch_bwd(s: dict, body_pose: torch.Tensor, g_verts: torch.Tensor, global_orient=animate.SCORE_ORIENT,
                        post_rot=animate.RENDER_ROT, out: Optional[torch.Tensor] = None,
                        ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    """d loss / d body_pose [B, P] of animate.smpl_pose_batch(s, body_pose, global_orient, post_rot) given g_verts."""
    B, P = body_pose.shape
    V, nj = s["v_template"].shape[0], s["J_regressor"].shape[0]
    L = _L()
    if ws is None:
        ws = torch.empty(_ws(L.avc_smpl_pose_batch_bwd_workspace_bytes, B, V, nj), dtype=torch.uint8,
                         device=body_pose.device)
    out = torch.empty(B, P, device=body_pose.device) if out is None else out
    go = _host_f32(global_orient).reshape(3)
    pr = None if post_rot is None else _host_f32(post_rot).reshape(9)
    _lib.check(L.avc_smpl_pose_batch_bwd(_lib.ptr(s["v_template"]), _lib.ptr(s["J_regressor"]), _lib.ptr(s["parents"]),
                                         _lib.ptr(s["posedirs"]), _lib.ptr(s["lbs_weights"]), V, nj,
                                         _lib.ptr(body_pose), P, B, _hp(go), None if pr is None else _hp(pr),
                                         _lib.ptr(g_verts), _lib.ptr(out), _lib.ptr(ws), ws.numel(),
                                         _lib.stream_ptr()), "avc_smpl_pose_batch_bwd")
    return out


def clip_prep_nearest_bwd(g_out: torch.Tensor, n: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """d loss / d images [B, n, n, 3] of shapegen.clip_prep_nearest given g_out [B, 3, S, S]."""
    B, S = g_out.shape[0], g_out.shape[-1]
    out = torch.empty(B, n, n, 3, device=g_out.device) if out is None else out
    _lib.check(_L().avc_clip_prep_nearest_bwd(_lib.ptr(g_out), B, n, S, _lib.ptr(out), _lib.stream_ptr()),
               "avc_clip_prep_nearest_bwd")
    return out


def pose_clip_loss(emb: torch.Tensor, text: torch.Tensor, loss: Optional[torch.Tensor] = None,
                   g_emb: Optional[torch.Tensor] = None):
    """(loss [B] = 1 - cos(mean_a emb[a, b], text), g_emb [A, B, D]) of emb [A, B, D]."""
    A, B, D = emb.shape
    loss = torch.empty(B, device=emb.device) if loss is None else loss
    g_emb = torch.empty_like(emb) if g_emb is None else g_emb
    _lib.check(_L().avc_pose_clip_loss(_lib.ptr(emb), A, B, D, _lib.ptr(text), _lib.ptr(loss), _lib.ptr(g_emb),
                                       _lib.stream_ptr()), "avc_pose_clip_loss")
    return loss, g_emb


# ---------------------------------------------------------------- one iteration on static buffers
class PoseStep:
    """The loss and pose gradient of B poses seen from A cameras each, on buffers allocated once, so that the
    sequence can be captured as a CUDA graph: ``pose`` [B, 63] and ``cams`` [B A cameras] are read, ``loss`` [B],
    ``grad`` [B, 63] and the intermediate ``rgb`` / ``prep`` / ``emb`` are written."""

    def __init__(self, assets: animate.Assets, B: int, A: int, image_size: int = shapegen.IMAGE_SIZE,
                 supersample: int = 2):
        a = assets
        dev = a.device
        self.a, self.B, self.A, self.n, self.ss = a, B, A, image_size, supersample
        L = _L()
        s = a.smpl
        V, nj = s["v_template"].shape[0], s["J_regressor"].shape[0]
        F = a.faces.shape[0]
        self.tower = a.clip.image
        D = self.tower.cfg.out_dim
        S = self.tower.cfg.image_size
        N = A * B
        self.pose = torch.zeros(B, POSE_DIM, device=dev)
        self.cams = torch.empty(B * A, _ws(L.avc_look_at_cam_bytes), dtype=torch.uint8, device=dev)
        self.verts = torch.empty(B, V, 3, device=dev)
        self.ws_smpl = torch.empty(_ws(L.avc_smpl_pose_batch_workspace_bytes, B, nj), dtype=torch.uint8, device=dev)
        self.rgb = torch.empty(A, B, image_size, image_size, 3, device=dev)
        self.ws_rf = raster_fwd_workspace(V, A, B, 1, image_size, supersample, dev)
        self.prep = torch.empty(N, 3, S, S, device=dev)
        self.text_rep = torch.empty(N, D, device=dev)
        self.emb = torch.empty(N, D, device=dev)
        self.cos = torch.empty(N, device=dev)
        self.ws_clip = self.tower._workspace(N)
        self.text = torch.empty(D, device=dev)
        self.loss = torch.empty(B, device=dev)
        self.g_emb = torch.empty(A, B, D, device=dev)
        self.g_prep = torch.empty(N, 3, S, S, device=dev)
        self.g_rgb = torch.empty(A, B, image_size, image_size, 3, device=dev)
        self.adj = video.adjacency(a.faces, V)
        self.ws_rb = raster_bwd_workspace(F, A, B, image_size, supersample, dev)
        self.g_verts = torch.empty(B, V, 3, device=dev)
        self.ws_sb = torch.empty(_ws(L.avc_smpl_pose_batch_bwd_workspace_bytes, B, V, nj), dtype=torch.uint8,
                                 device=dev)
        self.grad = torch.empty(B, POSE_DIM, device=dev)
        self._go = _host_f32(animate.SCORE_ORIENT).reshape(3)
        self._pr = _host_f32(animate.RENDER_ROT).reshape(9)

    def set_text(self, text_feature: torch.Tensor):
        self.text.copy_(text_feature.reshape(-1))
        self.text_rep.copy_(self.text[None].expand_as(self.text_rep))

    def run(self):
        """One forward and backward: the launches only, no host synchronisation."""
        L, a, s = _L(), self.a, self.a.smpl
        B, A, n = self.B, self.A, self.n
        V, nj = s["v_template"].shape[0], s["J_regressor"].shape[0]
        st = _lib.stream_ptr()
        cfg, w = C.byref(self.tower.cfg), C.byref(self.tower.w)
        S = self.tower.cfg.image_size
        N = A * B
        _lib.check(L.avc_smpl_pose_batch(_lib.ptr(s["v_template"]), _lib.ptr(s["J_regressor"]), _lib.ptr(s["parents"]),
                                         _lib.ptr(s["posedirs"]), _lib.ptr(s["lbs_weights"]), V, nj,
                                         _lib.ptr(self.pose), POSE_DIM, B, _hp(self._go), _hp(self._pr),
                                         _lib.ptr(self.verts), _lib.ptr(self.ws_smpl), self.ws_smpl.numel(), st),
                   "avc_smpl_pose_batch")
        raster_textured_batch_dev(self.verts, a.faces, a.textures, self.cams, A, 1, self.rgb, self.ws_rf, n, self.ss)
        _lib.check(L.avc_clip_prep_nearest(_lib.ptr(self.rgb), N, n, S, _lib.ptr(self.prep), st),
                   "avc_clip_prep_nearest")
        _lib.check(L.avc_clip_loss_fwd(cfg, w, _lib.ptr(self.prep), S, S, N, 1, _lib.ptr(self.text_rep),
                                       _lib.ptr(self.emb), _lib.ptr(self.cos), _lib.ptr(self.ws_clip),
                                       self.ws_clip.numel(), st), "avc_clip_loss_fwd")
        pose_clip_loss(self.emb.view(A, B, -1), self.text, self.loss, self.g_emb)
        _lib.check(L.avc_clip_loss_bwd(cfg, w, S, S, N, 1, _lib.ptr(self.text_rep), None, _lib.ptr(self.g_emb),
                                       _lib.ptr(self.g_prep), _lib.ptr(self.ws_clip), self.ws_clip.numel(), st),
                   "avc_clip_loss_bwd")
        clip_prep_nearest_bwd(self.g_prep, n, self.g_rgb.view(N, n, n, 3))
        raster_textured_batch_bwd(self.verts, a.faces, a.textures, self.adj, A, 1, self.g_rgb, self.ws_rf,
                                  self.g_verts, self.ws_rb, n, self.ss)
        smpl_pose_batch_bwd(s, self.pose, self.g_verts, animate.SCORE_ORIENT, animate.RENDER_ROT, self.grad,
                            self.ws_sb)


# ---------------------------------------------------------------- the generator
def optimizer_refusal(pg: Mapping, who: str = "PoseOptimizer") -> Optional[str]:
    """Why a PoseOptimizer (or ``who``'s) block's optimiser cannot run here, or None."""
    return motion.adam_refusal(pg, who, OPTIMIZER_DEFAULTS["optim_cfg"])


def adam_step(param: torch.Tensor, grad: torch.Tensor, m: torch.Tensor, v: torch.Tensor, state: torch.Tensor,
              betas, eps: float):
    """One torch.optim.Adam step of param by grad in place (avc_adam_step_dev; the step count and lr in state)."""
    _lib.check(_lib.lib().avc_adam_step_dev(_lib.ptr(param), _lib.ptr(grad), _lib.ptr(m), _lib.ptr(v), param.numel(),
                                            _lib.ptr(state), betas[0], betas[1], eps, 1.0, _lib.stream_ptr()),
               "avc_adam_step_dev")


def replay_iterations(step: PoseStep, cams: torch.Tensor, prime, body, grad: Optional[torch.Tensor] = None):
    """Capture body() (one iteration, ending in the parameter update) once as a CUDA graph and replay it once per
    iteration of cams [T, B A, cam_bytes], copying that iteration's cameras in first.  prime() -- the iteration
    without its update -- runs once before the capture, so that first-launch set-up stays outside the graph.  Returns
    step.loss after each replay [T, B] and, when grad is given, grad after each replay [T, *grad.shape] (else None)."""
    dev = step.pose.device
    T = cams.shape[0]
    losses = torch.empty(T, step.B, device=dev)
    grads = torch.empty(T, *grad.shape, device=dev) if grad is not None else None
    # capture on a side stream after one forward and backward without the update (first-launch set-up)
    step.cams.copy_(cams[0])
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        prime()
    torch.cuda.current_stream(dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        body()
    for it in range(T):
        step.cams.copy_(cams[it])
        g.replay()
        losses[it].copy_(step.loss)
        if grads is not None:
            grads[it].copy_(grad)
    return losses, grads


class PoseOptimizer(animate.BasePoseGenerator):
    """:102-135 with the reference's constructor defaults."""
    PARAM_DIM = POSE_DIM            # the optimised parameter of one candidate

    def __init__(self, optim_name="Adam", optim_cfg=None, num_iteration=500, topk=5, **kwargs):
        cfg = dict(OPTIMIZER_DEFAULTS["optim_cfg"] if optim_cfg is None else optim_cfg)
        why = optimizer_refusal(dict(optim_name=optim_name, optim_cfg=cfg), type(self).__name__)
        if why:
            raise NotImplementedError(why)
        super().__init__(topk=topk, **kwargs)
        self.num_iteration = int(num_iteration)
        self.lr = float(cfg.get("lr", 1e-3))
        self.betas = tuple(float(b) for b in cfg.get("betas", ADAM_BETAS))
        self.eps = float(cfg.get("eps", ADAM_EPS))
        self.last = {}

    def _cams(self, eyes: np.ndarray) -> torch.Tensor:
        """eyes [B, T, A, 3] -> each iteration's cameras [T, B A, cam_bytes] on the device."""
        B, T = eyes.shape[0], eyes.shape[1]
        return look_at_cams(np.ascontiguousarray(eyes.transpose(1, 0, 2, 3)), device=self.assets.device).view(
            T, B * eyes.shape[2], -1)

    def optimise(self, init: torch.Tensor, text_feature: torch.Tensor, eyes: np.ndarray,
                 record_grad: bool = False) -> torch.Tensor:
        """num_iteration Adam steps of the poses init [B, 63]; eyes [B, num_iteration, A, 3] are row b's cameras per
        iteration.  Returns the poses [B, 63]; self.last holds each iteration's loss (and pose gradient)."""
        dev = self.assets.device
        B, A = eyes.shape[0], eyes.shape[2]
        step = PoseStep(self.assets, B, A)
        step.set_text(text_feature.to(dev).float())
        step.pose.copy_(init.to(dev).float().reshape(B, POSE_DIM))
        m = torch.zeros_like(step.pose)
        v = torch.zeros_like(step.pose)
        state = torch.tensor([0.0, self.lr, 0.0, 0.0], device=dev)

        def body():
            step.run()
            adam_step(step.pose, step.grad, m, v, state, self.betas, self.eps)

        losses, grads = replay_iterations(step, self._cams(eyes), step.run, body, step.grad if record_grad else None)
        self.last = dict(loss=losses, grad=grads)
        return step.pose.clone()

    def get_topk_poses(self, text: str, init: Optional[torch.Tensor] = None,
                       text_feature: Optional[torch.Tensor] = None, record_grad: bool = False) -> torch.Tensor:
        """:133-135 -> [topk, 69].  ``init`` [topk, PARAM_DIM] stands in for the topk torch.randn(PARAM_DIM) draws and
        ``text_feature`` [512] for the CLIP text encode of ``text``.  Afterwards ``self.last`` holds the initial
        parameters, the eyes, each iteration's loss [num_iteration, topk] (and gradient) and the sort's scores."""
        tf = self.get_text_feature(text) if text_feature is None else text_feature.to(self.assets.device).float()
        if init is None:
            init = torch.stack([torch.randn(self.PARAM_DIM) for _ in range(self.topk)])
        init = torch.as_tensor(init, dtype=torch.float32).reshape(self.topk, self.PARAM_DIM)
        T = self.num_iteration
        eyes = self.scorer.draw_eyes(self.topk * T).reshape(self.topk, T, len(self.scorer.angles), 3)
        poses = self.optimise(init, tf, eyes, record_grad)
        last = dict(self.last, init=init, eyes=eyes)
        ranked, sc = self.scorer.sort_poses_by_score(tf, list(motion.pose_padding(poses)))
        self.last = dict(last, sort_scores=sc)
        return torch.stack(ranked, 0)


def refusal(conf) -> Optional[str]:
    """Why ``conf`` cannot run on this command, or None."""
    mode = conf.get_string("general.mode", "pose")
    if mode != "pose":
        return (f"general.mode = {mode}: this command runs the pose stage's PoseOptimizer; the motion stage runs as "
                "python -m avatarclip_b200.motion")
    pg = conf.get("pose_generator", {})
    typ = pg.get("type", None)
    if typ in animate.IN_SCOPE:
        return f"pose_generator.type = {typ}: this command runs PoseOptimizer; run python -m avatarclip_b200.animate"
    if typ == "VPoserOptimizer":
        return ("pose_generator.type = VPoserOptimizer: this command runs PoseOptimizer; VPoserOptimizer optimises the "
                "VPoser latent through the decoder's backward, so it runs as python -m avatarclip_b200.vposer_optimizer")
    if typ != "PoseOptimizer":
        return f"pose_generator.type = {typ!r} is unknown (this command runs PoseOptimizer)"
    return optimizer_refusal(pg)


# ---------------------------------------------------------------- CLI (main.py:15-35)
def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(
        prog="python -m avatarclip_b200.pose_optimizer",
        description="Optimise candidate SMPL body poses against the text of an AvatarAnimate conf (main.py, "
                    "general.mode = pose, pose_generator.type = PoseOptimizer): writes candidate_%%d.npy (69 values) "
                    "and candidate_%%d.jpg into general.base_exp_dir.",
        epilog="--uv_obj (smpl_uv.obj) is AvatarAnimate's data/ file; --clip_model / --bpe are openai's CLIP ViT-B/32 "
               "checkpoint and BPE merges file.  The SMPL .npz holds the arrays " + ", ".join(shapegen.SMPL_NPZ_KEYS) +
               " (see python -m avatarclip_b200.shapegen --help).")
    p.add_argument("--conf", type=str, default="./confs/base.conf")
    p.add_argument("--smpl", required=True, help=".npz with the SMPL tensors and faces")
    p.add_argument("--uv_obj", type=str, default="data/smpl_uv.obj", help="SMPL mesh with UVs, its .mtl and image")
    p.add_argument("--clip_model", type=str, default="ViT-B-32.pt")
    p.add_argument("--bpe", type=str, default="bpe_simple_vocab_16e6.txt.gz")
    p.add_argument("--seed", type=int, default=None, help="seed numpy's and torch's generators first")
    p.add_argument("--device", default="cuda")
    return p


def parse_args(argv=None):
    """(args, conf, PoseOptimizer kwargs); exits with a message for what cannot run, before any file but the conf is
    read."""
    from . import conf as conf_mod
    parser = build_parser()
    a = parser.parse_args(argv)
    if not os.path.isfile(a.conf):
        parser.error(f"--conf: no such file: {a.conf}")
    conf = conf_mod.parse_file(a.conf)
    why = refusal(conf)
    if why:
        parser.error(why)
    for flag, path in (("--smpl", a.smpl), ("--uv_obj", a.uv_obj), ("--clip_model", a.clip_model), ("--bpe", a.bpe)):
        if not os.path.isfile(path):
            parser.error(f"{flag}: no such file: {path}")
    pg = dict(conf["pose_generator"])
    pg.pop("type")
    for k in ("smpl_path", "vposer_path"):      # BasePoseGenerator's paths: --smpl stands in, VPoser is not used
        pg.pop(k, None)
    return a, conf, pg


def main(argv=None) -> int:
    a, conf, pg = parse_args(argv)
    if a.seed is not None:
        np.random.seed(a.seed)
        torch.manual_seed(a.seed)
    smpl = shapegen.load_smpl_npz(a.smpl)
    clip = shapegen.load_clip(a.clip_model, a.bpe, a.device)
    assets = animate.Assets(smpl, clip, None, a.uv_obj, a.device)
    text = conf.get_string("general.text")
    out_dir = conf.get_string("general.base_exp_dir")
    poses = PoseOptimizer(name="PoseOptimizer", assets=assets, **pg).get_topk_poses(text)
    animate.write_candidates(out_dir, poses, animate.render_candidates(assets, poses))
    print(f"{poses.shape[0]} candidate poses for {text!r} written to {out_dir}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
