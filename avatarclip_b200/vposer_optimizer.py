"""AvatarAnimate's ``VPoserOptimizer`` (models/pose_generation.py:138-173) on the GPU: SMPL body poses found by Adam in
VPoser's latent space against a text prompt, written as ``candidate_%d.npy`` (69 float32 values, ``pose_padding``) and
``candidate_%d.jpg``.

Each of the ``topk`` candidates starts from a latent ``torch.randn(32)`` and takes ``num_iteration`` Adam steps on
``1 - cosine(mean over 5 cameras of encode_image(render(SMPL(VPoser.decode(latent)))), text_feature)``, VPoser's
weights frozen.  The pose a candidate returns is the decode of its latent *before* the last Adam step: the reference
returns the last iteration's forward, so the final step moves the latent but not the output.  The candidates are then
sorted by a fresh score (``PoseScorer.sort_poses_by_score``).  As in ``pose_optimizer``, the candidates are independent
and Adam is elementwise, so all ``topk`` latents run as one batch of rows.

One iteration is a fixed sequence of library calls with no host synchronisation; its middle is
``pose_optimizer.PoseStep`` unchanged:

    avc_vposer_decode (latent -> PoseStep.pose) -> PoseStep.run() (SMPL, render, CLIP tower, loss and their backward
    to PoseStep.grad) -> avc_vposer_decode_bwd (PoseStep.grad -> d loss / d latent) -> avc_adam_step_dev

It is captured once as a CUDA graph and replayed ``num_iteration`` times by ``pose_optimizer.replay_iterations``, with
the cameras of each iteration copied in before its replay; the draws (the latents with torch, then candidate k's
``num_iteration`` x 5 elevations before candidate k + 1's, then the sort's, with numpy) stay on the host in the
reference's order.

    python -m avatarclip_b200.vposer_optimizer --conf confs/pose_ablation/vposer_optimizer/cry.conf --smpl smpl.npz \\
        --vposer data/vposer --uv_obj data/smpl_uv.obj --clip_model ViT-B-32.pt --bpe bpe_simple_vocab_16e6.txt.gz
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import sys
from typing import Mapping, Optional

import numpy as np
import torch

from . import _lib, animate, motion, motion_clip, shapegen
from . import pose_optimizer as PO

LATENT_DIM = 32                 # VPoserOptimizer.get_pose's torch.randn(32)

_bound = None


def _L():
    global _bound
    L = PO._L()
    if _bound is None:
        vp, i32, sz = C.c_void_p, C.c_int32, C.c_size_t
        L.avc_vposer_decode_bwd_workspace_bytes.argtypes = [i32, i32, i32, C.POINTER(sz)]
        L.avc_vposer_decode_bwd.argtypes = [vp, i32, i32, vp, vp, i32, vp, vp, vp, vp, i32, vp, vp, vp, vp, sz, vp]
        for n in ("avc_vposer_decode_bwd_workspace_bytes", "avc_vposer_decode_bwd"):
            getattr(L, n).restype = C.c_int
        _bound = L
    return L


# ---------------------------------------------------------------- device ops
def _decoder(dec: Mapping[str, torch.Tensor], latent: int):
    """(decoder_net's six tensors in avc_vposer_decode's order, hidden, n_joints), shapes checked against latent."""
    w = [animate._dev(dec[f"decoder_net.{i}.{k}"], "vposer decoder") for i in (0, 3, 5) for k in ("weight", "bias")]
    H, O = w[0].shape[0], w[4].shape[0]
    if w[0].shape[1] != latent or O % 6 or tuple(w[2].shape) != (H, H) or w[4].shape[1] != H:
        raise _lib.AvcError(f"vposer decoder: latent {latent} against decoder_net {[tuple(t.shape) for t in w]}")
    return w, H, O // 6


def vposer_workspace(dec: Mapping[str, torch.Tensor], latent: int = LATENT_DIM) -> torch.Tensor:
    """The workspace avc_vposer_decode and avc_vposer_decode_bwd take for this decoder."""
    w, H, nj = _decoder(dec, latent)
    return torch.empty(animate._ws(_L().avc_vposer_decode_bwd_workspace_bytes, latent, H, nj), dtype=torch.uint8,
                       device=w[0].device)


def vposer_decode_into(z: torch.Tensor, dec: Mapping[str, torch.Tensor], pose: torch.Tensor, ws: torch.Tensor):
    """avc_vposer_decode of the latents z [B, latent] into pose [B, n_joints * 3] on the caller's buffers."""
    w, H, nj = _decoder(dec, z.shape[1])
    _lib.check(_L().avc_vposer_decode(_lib.ptr(z), z.shape[0], z.shape[1], _lib.ptr(w[0]), _lib.ptr(w[1]), H,
                                      _lib.ptr(w[2]), _lib.ptr(w[3]), _lib.ptr(w[4]), _lib.ptr(w[5]), nj, _lib.ptr(pose),
                                      None, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "avc_vposer_decode")
    return pose


def vposer_decode_bwd(z: torch.Tensor, dec: Mapping[str, torch.Tensor], g_pose: torch.Tensor,
                      out: Optional[torch.Tensor] = None, pose_out: Optional[torch.Tensor] = None,
                      ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    """d loss / d z [B, latent] of VPoser.decode(z)['pose_body'] given g_pose = d loss / d pose_body [B, n_joints, 3]
    (or [B, n_joints * 3]).  pose_out [B, n_joints, 3], when given, receives the decode the backward recomputed."""
    z = animate._dev(z, "vposer_decode_bwd").reshape(z.shape[0], -1)
    B, Lz = z.shape
    w, H, nj = _decoder(dec, Lz)
    g = animate._dev(g_pose, "vposer_decode_bwd")
    if g.numel() != B * nj * 3:
        raise _lib.AvcError(f"vposer_decode_bwd: g_pose {tuple(g_pose.shape)} for {B} rows of {nj} joints")
    ws = vposer_workspace(dec, Lz) if ws is None else ws
    out = torch.empty(B, Lz, device=z.device) if out is None else out
    _lib.check(_L().avc_vposer_decode_bwd(_lib.ptr(z), B, Lz, _lib.ptr(w[0]), _lib.ptr(w[1]), H, _lib.ptr(w[2]),
                                          _lib.ptr(w[3]), _lib.ptr(w[4]), _lib.ptr(w[5]), nj, _lib.ptr(g),
                                          _lib.ptr(out), None if pose_out is None else _lib.ptr(pose_out),
                                          _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "avc_vposer_decode_bwd")
    return out


# ---------------------------------------------------------------- the generator
class VPoserOptimizer(PO.PoseOptimizer):
    """:138-173 with the reference's constructor defaults; the optimised parameter is each candidate's VPoser latent."""
    PARAM_DIM = LATENT_DIM

    def optimise(self, init: torch.Tensor, text_feature: torch.Tensor, eyes: np.ndarray,
                 record_grad: bool = False) -> torch.Tensor:
        """num_iteration Adam steps of the latents init [B, 32]; eyes [B, num_iteration, A, 3] are row b's cameras per
        iteration.  Returns the last iteration's decoded poses [B, 63] (of the latents before the last step); self.last
        holds each iteration's loss (and latent gradient) and the final latents."""
        dev = self.assets.device
        dec = self.assets.vposer
        B, A = eyes.shape[0], eyes.shape[2]
        _, _, nj = _decoder(dec, LATENT_DIM)
        if nj * 3 != PO.POSE_DIM:
            raise _lib.AvcError(f"VPoserOptimizer: the decoder gives {nj} joints, SMPL's body pose has 21")
        step = PO.PoseStep(self.assets, B, A)
        step.set_text(text_feature.to(dev).float())
        z = init.to(dev).float().reshape(B, LATENT_DIM).contiguous()
        g_z = torch.empty_like(z)
        ws = vposer_workspace(dec)
        m = torch.zeros_like(z)
        v = torch.zeros_like(z)
        state = torch.tensor([0.0, self.lr, 0.0, 0.0], device=dev)

        def forward_backward():
            vposer_decode_into(z, dec, step.pose, ws)
            step.run()
            vposer_decode_bwd(z, dec, step.grad, g_z, None, ws)

        def body():
            forward_backward()
            PO.adam_step(z, g_z, m, v, state, self.betas, self.eps)

        losses, grads = PO.replay_iterations(step, self._cams(eyes), forward_backward, body,
                                             g_z if record_grad else None)
        self.last = dict(loss=losses, grad=grads, latent=z.clone())
        return step.pose.clone()


def refusal(conf) -> Optional[str]:
    """Why ``conf`` cannot run on this command, or None."""
    mode = conf.get_string("general.mode", "pose")
    if mode != "pose":
        cmd = "motion_clip" if motion.refusal(conf) and motion_clip.refusal(conf) is None else "motion"
        return (f"general.mode = {mode}: this command runs the pose stage's VPoserOptimizer; this conf runs as "
                f"python -m avatarclip_b200.{cmd}")
    pg = conf.get("pose_generator", {})
    typ = pg.get("type", None)
    if typ in animate.IN_SCOPE:
        return f"pose_generator.type = {typ}: this command runs VPoserOptimizer; run python -m avatarclip_b200.animate"
    if typ == "PoseOptimizer":
        return ("pose_generator.type = PoseOptimizer: this command runs VPoserOptimizer; run python -m "
                "avatarclip_b200.pose_optimizer")
    if typ != "VPoserOptimizer":
        return f"pose_generator.type = {typ!r} is unknown (this command runs VPoserOptimizer)"
    return PO.optimizer_refusal(pg, "VPoserOptimizer")


# ---------------------------------------------------------------- CLI (main.py:15-35)
def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(
        prog="python -m avatarclip_b200.vposer_optimizer",
        description="Optimise candidate SMPL body poses in VPoser's latent space against the text of an AvatarAnimate "
                    "conf (main.py, general.mode = pose, pose_generator.type = VPoserOptimizer): writes "
                    "candidate_%%d.npy (69 values) and candidate_%%d.jpg into general.base_exp_dir.",
        epilog="--vposer is the VPoser v2.0 model directory from human_body_prior (snapshots/*.ckpt) or one checkpoint; "
               "without the flag the conf's pose_generator.vposer_path is used, and without either "
               f"{animate.DEFAULT_PATHS['vposer']}.  --uv_obj (smpl_uv.obj) is AvatarAnimate's data/ file; "
               "--clip_model / --bpe are openai's CLIP ViT-B/32 checkpoint and BPE merges file.  The SMPL .npz holds "
               "the arrays " + ", ".join(shapegen.SMPL_NPZ_KEYS) + " (see python -m avatarclip_b200.shapegen --help).")
    p.add_argument("--conf", type=str, default="./confs/base.conf")
    p.add_argument("--smpl", required=True, help=".npz with the SMPL tensors and faces")
    p.add_argument("--vposer", type=str, default=None,
                   help=f"VPoser 2.x model directory (default: the conf's path, else {animate.DEFAULT_PATHS['vposer']})")
    p.add_argument("--uv_obj", type=str, default="data/smpl_uv.obj", help="SMPL mesh with UVs, its .mtl and image")
    p.add_argument("--clip_model", type=str, default="ViT-B-32.pt")
    p.add_argument("--bpe", type=str, default="bpe_simple_vocab_16e6.txt.gz")
    p.add_argument("--seed", type=int, default=None, help="seed numpy's and torch's generators first")
    p.add_argument("--device", default="cuda")
    return p


def parse_args(argv=None):
    """(args, conf, VPoserOptimizer kwargs), args.vposer resolved; exits with a message for what cannot run, before
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
    pg = dict(conf["pose_generator"])
    pg.pop("type")
    # an explicit flag, else the conf's path, else the reference's default (as python -m avatarclip_b200.animate)
    a.vposer = a.vposer or pg.get("vposer_path") or animate.DEFAULT_PATHS["vposer"]
    for k in ("smpl_path", "vposer_path"):      # BasePoseGenerator's paths: --smpl and --vposer stand in
        pg.pop(k, None)
    for flag, path in (("--smpl", a.smpl), ("--uv_obj", a.uv_obj), ("--clip_model", a.clip_model), ("--bpe", a.bpe)):
        if not os.path.isfile(path):
            parser.error(f"{flag}: no such file: {path}")
    if not os.path.exists(a.vposer):
        parser.error(f"--vposer: no such directory or file: {a.vposer}")
    return a, conf, pg


def main(argv=None) -> int:
    a, conf, pg = parse_args(argv)
    if a.seed is not None:
        np.random.seed(a.seed)
        torch.manual_seed(a.seed)
    smpl = shapegen.load_smpl_npz(a.smpl)
    clip = shapegen.load_clip(a.clip_model, a.bpe, a.device)
    assets = animate.Assets(smpl, clip, a.vposer, a.uv_obj, a.device)
    text = conf.get_string("general.text")
    out_dir = conf.get_string("general.base_exp_dir")
    poses = VPoserOptimizer(name="VPoserOptimizer", assets=assets, **pg).get_topk_poses(text)
    animate.write_candidates(out_dir, poses, animate.render_candidates(assets, poses))
    print(f"{poses.shape[0]} candidate poses for {text!r} written to {out_dir}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
