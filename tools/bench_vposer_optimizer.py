"""Time AvatarAnimate's VPoserOptimizer on the device and print one JSON line.

The reference's defaults, topk 5 x num_iteration 500, on synthetic full-size weights (the real SMPL template with
seeded SMPL-shaped tensors, a seeded UV texture, random ViT-B/32 towers, oracle/animate.py's seeded VPoser decoder):
the whole ``get_topk_poses`` call in wall time ending in a device synchronise (draws, graph capture, 500 replays, the
sort), and, in a separate run of the same iteration launched stage by stage, the medians of CUDA-event times of its
parts: the VPoser decode, SMPL forward + render, CLIP prep + tower forward + loss + tower backward + prep backward, the
raster backward, the SMPL backward and the VPoser decoder's backward.  The card's name and power limit are read in the
same run.

    python tools/bench_vposer_optimizer.py [--reps 20] [--iters 500] [--topk 5]

The warm-up is one call at 2 iterations, so the timed call is the only one at the full size.
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_animate import _power_limit  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--topk", type=int, default=5)
    a = ap.parse_args()
    from avatarclip_b200 import _lib, animate as A, pose_optimizer as PO, shapegen as S, vposer_optimizer as VO
    from oracle import animate as O
    from oracle import drive as D
    from oracle import shapegen as OS
    tv, tf = D.template_obj()
    smpl = {k: np.asarray(v) for k, v in D.golden_smpl().items()}
    smpl["faces"] = tf
    with tempfile.TemporaryDirectory() as tmp:
        uv = OS.write_uv_obj(os.path.join(tmp, "uv"), smpl["v_template"], smpl["faces"])
        clip = S.load_clip(OS.clip_states(), OS.write_bpe(os.path.join(tmp, "bpe.txt.gz")))
        assets = A.Assets(smpl, clip, O.vposer_state(), uv)
    r = {"device": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "topk": a.topk, "iters": a.iters}
    tfeat = torch.randn(512, generator=torch.Generator().manual_seed(0)).cuda()
    np.random.seed(0)
    torch.manual_seed(0)
    VO.VPoserOptimizer(name="VPoserOptimizer", assets=assets, num_iteration=2, topk=a.topk).get_topk_poses(
        "", text_feature=tfeat)                          # warm-up: first launches of every kernel
    opt = VO.VPoserOptimizer(name="VPoserOptimizer", assets=assets, num_iteration=a.iters, topk=a.topk)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    opt.get_topk_poses("", text_feature=tfeat)
    torch.cuda.synchronize()
    r["call_s"] = time.perf_counter() - t0

    # one iteration, stage by stage
    step = PO.PoseStep(assets, a.topk, len(A.ANGLES))
    step.set_text(tfeat)
    z = torch.randn(a.topk, VO.LATENT_DIM, generator=torch.Generator().manual_seed(1)).cuda()
    g_z = torch.empty_like(z)
    ws_vp = VO.vposer_workspace(assets.vposer)
    step.cams.copy_(PO.look_at_cams(opt.scorer.draw_eyes(a.topk), device="cuda"))
    L, s = PO._L(), assets.smpl
    V, nj = s["v_template"].shape[0], s["J_regressor"].shape[0]
    B, Aa, n = step.B, step.A, step.n
    N, Sz = B * Aa, step.tower.cfg.image_size

    def render():
        _lib.check(L.avc_smpl_pose_batch(_lib.ptr(s["v_template"]), _lib.ptr(s["J_regressor"]), _lib.ptr(s["parents"]),
                                         _lib.ptr(s["posedirs"]), _lib.ptr(s["lbs_weights"]), V, nj,
                                         _lib.ptr(step.pose), 63, B, PO._hp(step._go), PO._hp(step._pr),
                                         _lib.ptr(step.verts), _lib.ptr(step.ws_smpl), step.ws_smpl.numel(),
                                         _lib.stream_ptr()), "avc_smpl_pose_batch")
        PO.raster_textured_batch_dev(step.verts, assets.faces, assets.textures, step.cams, Aa, 1, step.rgb, step.ws_rf)

    def clip_fb():
        st, cfg, w = _lib.stream_ptr(), C.byref(step.tower.cfg), C.byref(step.tower.w)
        _lib.check(L.avc_clip_prep_nearest(_lib.ptr(step.rgb), N, n, Sz, _lib.ptr(step.prep), st), "prep")
        _lib.check(L.avc_clip_loss_fwd(cfg, w, _lib.ptr(step.prep), Sz, Sz, N, 1, _lib.ptr(step.text_rep),
                                       _lib.ptr(step.emb), _lib.ptr(step.cos), _lib.ptr(step.ws_clip),
                                       step.ws_clip.numel(), st), "fwd")
        PO.pose_clip_loss(step.emb.view(Aa, B, -1), step.text, step.loss, step.g_emb)
        _lib.check(L.avc_clip_loss_bwd(cfg, w, Sz, Sz, N, 1, _lib.ptr(step.text_rep), None, _lib.ptr(step.g_emb),
                                       _lib.ptr(step.g_prep), _lib.ptr(step.ws_clip), step.ws_clip.numel(), st), "bwd")
        PO.clip_prep_nearest_bwd(step.g_prep, n, step.g_rgb.view(N, n, n, 3))

    def raster_bwd():
        PO.raster_textured_batch_bwd(step.verts, assets.faces, assets.textures, step.adj, Aa, 1, step.g_rgb, step.ws_rf,
                                     step.g_verts, step.ws_rb)

    def smpl_bwd():
        PO.smpl_pose_batch_bwd(s, step.pose, step.g_verts, out=step.grad, ws=step.ws_sb)

    def decode():
        VO.vposer_decode_into(z, assets.vposer, step.pose, ws_vp)

    def decode_bwd():
        VO.vposer_decode_bwd(z, assets.vposer, step.grad, g_z, None, ws_vp)

    parts = {"vposer_decode_ms": decode, "render_ms": render, "clip_fwd_bwd_ms": clip_fb, "raster_bwd_ms": raster_bwd,
             "smpl_bwd_ms": smpl_bwd, "vposer_decode_bwd_ms": decode_bwd}
    times = {k: [] for k in parts}
    for rep in range(a.reps + 2):
        for k, fn in parts.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            if rep >= 2:
                times[k].append(e0.elapsed_time(e1))
    for k, v in times.items():
        r[k] = float(np.median(v))
    print(json.dumps(r))


if __name__ == "__main__":
    main()
