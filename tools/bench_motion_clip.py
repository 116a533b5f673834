"""Time AvatarAnimate's MotionOptimizer with its CLIP term on the device and print JSON lines.

The shipped shape: latent 256, 4 layers, 60 frames, clip_num_part 30 (so 2 renders per iteration, at 256 x 256 with
2 x 2 supersampling), the full-size ViT-B/32 on seeded weights, the real SMPL template with seeded SMPL-shaped tensors
and a seeded UV texture.  One iteration launched stage by stage, the medians of CUDA-event times of its parts: the
decoder forward, the frame selection, SMPL forward + render, CLIP prep + tower forward + loss + tower backward + prep
backward, the raster backward, the SMPL backward and the motion backward (losses, the CLIP rows' gradient, the
decoder's backward and Adam).  The raster backward's serial edge sweeps depend on the pose, so the split is taken at
the initial latent and again at the latent the whole call ends with.  Between them, the wall time of one
``get_motion`` call at ``--iters`` iterations (base.conf's 5000 by default: draws, graph capture, the replays), ending
in a device synchronise.  The card's name and power limit are read in the same run.

    python tools/bench_motion_clip.py [--reps 20] [--iters 5000]
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


def _median_ms(fn, reps):
    t = []
    for rep in range(reps + 2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        if rep >= 2:
            t.append(e0.elapsed_time(e1))
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=5000)
    a = ap.parse_args()
    from avatarclip_b200 import _lib, animate as A, motion_clip as MC, pose_optimizer as PO, shapegen as S
    from oracle import drive as D
    from oracle import motion as OM
    from oracle import shapegen as OS
    tv, tf = D.template_obj()
    smpl = {k: np.asarray(v) for k, v in D.golden_smpl().items()}
    smpl["faces"] = tf
    with tempfile.TemporaryDirectory() as tmp:
        uv = OS.write_uv_obj(os.path.join(tmp, "uv"), smpl["v_template"], smpl["faces"])
        clip = S.load_clip(OS.clip_states(), OS.write_bpe(os.path.join(tmp, "bpe.txt.gz")))
        assets = A.Assets(smpl, clip, None, uv)
    r = {"device": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "latent": 256, "layers": 4,
         "frames": 60, "rows": MC.clip_rows(60, 30), "image": 256, "supersample": 2}
    gen = torch.Generator().manual_seed(0)
    tfeat = torch.randn(512, generator=gen).cuda()
    poses = (torch.randn(5, 63, generator=gen) * 0.3).cuda()
    opt = MC.MotionOptimizer(assets, ckpt_path=OM.motion_vae_state(), num_iteration=2)

    def split(latent):
        """One iteration stage by stage from ``latent``: the medians of its parts' CUDA-event times."""
        R = r["rows"]
        n_calls = 2 * (a.reps + 2) + 1
        ms = MC.ClipMotionStep(opt.vae, poses, [1, 0.8, 0.6, 0.4, 0.2], 0.01, n_calls)
        step = PO.PoseStep(assets, R, 1)
        step.set_text(tfeat)
        eye = PO.shapegen.handoff.get_points_from_angles(2.0, 0.1, MC.CLIP_AZIMUTH)
        step.cams.copy_(PO.look_at_cams(np.repeat(eye[None, None], R, 0), device="cuda").view(R, -1))
        st = torch.tensor([7], dtype=torch.int32, device="cuda")
        frame, weight = torch.empty(R, dtype=torch.int32, device="cuda"), torch.empty(R, device="cuda")
        ms.init(latent, 0.01)
        L, s = PO._L(), assets.smpl
        V, nj = s["v_template"].shape[0], s["J_regressor"].shape[0]
        N, n, Sz = R, step.n, step.tower.cfg.image_size

        def select():
            MC.select(ms.motion, 30, 0.001, st, R, step.pose, frame, weight)

        def render():
            _lib.check(L.avc_smpl_pose_batch(_lib.ptr(s["v_template"]), _lib.ptr(s["J_regressor"]),
                                             _lib.ptr(s["parents"]), _lib.ptr(s["posedirs"]), _lib.ptr(s["lbs_weights"]),
                                             V, nj,
                                             _lib.ptr(step.pose), 63, R, PO._hp(step._go), PO._hp(step._pr),
                                             _lib.ptr(step.verts), _lib.ptr(step.ws_smpl), step.ws_smpl.numel(),
                                             _lib.stream_ptr()), "avc_smpl_pose_batch")
            PO.raster_textured_batch_dev(step.verts, assets.faces, assets.textures, step.cams, 1, 1, step.rgb,
                                         step.ws_rf)

        def clip_fb():
            sp, cfg, w = _lib.stream_ptr(), C.byref(step.tower.cfg), C.byref(step.tower.w)
            _lib.check(L.avc_clip_prep_nearest(_lib.ptr(step.rgb), N, n, Sz, _lib.ptr(step.prep), sp), "prep")
            _lib.check(L.avc_clip_loss_fwd(cfg, w, _lib.ptr(step.prep), Sz, Sz, N, 1, _lib.ptr(step.text_rep),
                                           _lib.ptr(step.emb), _lib.ptr(step.cos), _lib.ptr(step.ws_clip),
                                           step.ws_clip.numel(), sp), "fwd")
            PO.pose_clip_loss(step.emb.view(1, R, -1), step.text, step.loss, step.g_emb)
            _lib.check(L.avc_clip_loss_bwd(cfg, w, Sz, Sz, N, 1, _lib.ptr(step.text_rep), None,
                                           _lib.ptr(step.g_emb), _lib.ptr(step.g_prep), _lib.ptr(step.ws_clip),
                                           step.ws_clip.numel(), sp), "bwd")
            PO.clip_prep_nearest_bwd(step.g_prep, n, step.g_rgb.view(N, n, n, 3))

        def raster_bwd():
            PO.raster_textured_batch_bwd(step.verts, assets.faces, assets.textures, step.adj, 1, 1, step.g_rgb,
                                         step.ws_rf, step.g_verts, step.ws_rb)

        def smpl_bwd():
            PO.smpl_pose_batch_bwd(s, step.pose, step.g_verts, out=step.grad, ws=step.ws_sb)

        def motion_bwd():
            ms.backward(frame, weight, step.grad, step.loss)

        parts = {"decoder_fwd_ms": ms.forward, "select_ms": select, "render_ms": render, "clip_fwd_bwd_ms": clip_fb,
                 "raster_bwd_ms": raster_bwd, "smpl_bwd_ms": smpl_bwd, "motion_bwd_adam_ms": motion_bwd}
        out = {k: _median_ms(fn, a.reps) for k, fn in parts.items()}
        out["parts_sum_ms"] = sum(out.values())
        return out

    z0 = torch.randn(256, generator=gen)
    r["split_at_start"] = split(z0.cuda())
    print(json.dumps(r), flush=True)

    # the whole call
    np.random.seed(0)
    torch.manual_seed(0)
    opt.get_motion("", poses, text_feature=tfeat)                   # warm-up: first launches at 2 iterations
    opt.cfg["num_iteration"] = a.iters
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    opt.get_motion("", poses, latent=z0, text_feature=tfeat)
    torch.cuda.synchronize()
    r["iters"] = a.iters
    r["call_s"] = time.perf_counter() - t0
    r["call_per_iter_ms"] = 1e3 * r["call_s"] / a.iters
    r["final_loss"] = float(opt.last["loss"][-1])
    print(json.dumps(r), flush=True)

    r["split_at_end"] = split(opt.last["latent"])
    print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
