"""Time AvatarAnimate's pose stage on the device and print one JSON line.

Per stage, the median of CUDA-event times over --reps calls after --warmup calls: the VPoser decode of 500 latents
(avc_vposer_decode), the RealNVP decode of 500 (avc_realnvp_decode), SMPL for 500 body poses (avc_smpl_pose_batch),
2 500 textured 256 x 256 renders (avc_raster_textured_batch), the CLIP image encode of 2 500 renders (nearest resize +
Normalize + ClipImageTower), and the codebook top-40 over 4 096 and 65 536 entries (avc_cosine_topk).  Then, in wall
time, one VPoserRealNVP.get_topk_poses at the reference's defaults (5 x 50 x 10 draws + 5 for the sort: 2 525 poses,
12 625 renders) and one VPoserCodebook.get_topk_poses.  The card's name and power limit are read in the same run.
All inputs are synthetic and seeded (oracle/animate.py, oracle/shapegen.py): SMPL-sized template, full-size VPoser and
RealNVP, random ViT-B/32 towers.

    python tools/bench_animate.py [--reps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _time(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import shapegen as S
    from oracle import animate as O
    from oracle import drive as D
    from oracle import shapegen as OS

    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit()}
    g = torch.Generator(device="cuda").manual_seed(0)
    tv, tf = D.template_obj()
    smpl = {k: np.asarray(v) for k, v in D.golden_smpl().items()}
    smpl["faces"] = tf
    with tempfile.TemporaryDirectory() as tmp:
        uv = OS.write_uv_obj(os.path.join(tmp, "uv"), tv, tf)
        clip = S.load_clip(OS.clip_states(), OS.write_bpe(os.path.join(tmp, "bpe.txt.gz")))
        assets = A.Assets(smpl, clip, O.vposer_state(), uv)
        z = torch.randn(500, 32, generator=g, device="cuda")
        res["vposer_decode_500_ms"] = _time(lambda: A.vposer_decode(z, assets.vposer), a.reps, a.warmup)
        nvp_w = A.pack_realnvp(O.realnvp_state(), 8, "cuda")
        f = torch.randn(512, generator=g, device="cuda") * 0.05
        res["realnvp_decode_500_ms"] = _time(lambda: A.realnvp_decode(z, f, nvp_w), a.reps, a.warmup)
        poses = A.vposer_decode(z, assets.vposer).reshape(500, -1)
        res["smpl_batch_500_ms"] = _time(lambda: A.smpl_pose_batch(assets.smpl, poses, A.SCORE_ORIENT, A.RENDER_ROT),
                                         a.reps, a.warmup)
        v = A.smpl_pose_batch(assets.smpl, poses, A.SCORE_ORIENT, A.RENDER_ROT)
        np.random.seed(0)
        eyes = A.PoseScorer(assets).draw_eyes(50)
        reps = max(3, a.reps // 4)
        res["raster_2500_ms"] = _time(lambda: [A.raster_textured_batch(v[i:i + 250], assets.faces, assets.textures,
                                                                       eyes[i // 10:(i + 250) // 10], 10)
                                               for i in range(0, 500, 250)], reps, 1)
        imgs = A.raster_textured_batch(v[:250], assets.faces, assets.textures, eyes[:25], 10).reshape(1250, 256, 256, 3)

        def encode():
            for _ in range(2):
                prep = S.clip_prep_nearest(imgs)
                for i in range(0, 1250, 256):
                    clip.image.encode_image(prep[i:i + 256])
        res["clip_encode_2500_ms"] = _time(encode, reps, 1)
        tfeat = torch.randn(512, generator=g, device="cuda")
        for N in (4096, 65536):
            cb = torch.randn(N, 512, generator=g, device="cuda")
            res[f"codebook_top40_{N}_ms"] = _time(lambda: A.cosine_topk(cb, tfeat, 40), a.reps, a.warmup)

        torch.save({"state_dict": O.realnvp_state()}, os.path.join(tmp, "nvp.pth"))
        torch.save(O.make_codebook(tfeat.cpu(), n=4096), os.path.join(tmp, "cb.pth"))
        nvp = A.build_pose_generator({"type": "VPoserRealNVP", "ckpt_path": os.path.join(tmp, "nvp.pth")}, assets)
        cbg = A.build_pose_generator({"type": "VPoserCodebook", "codebook_path": os.path.join(tmp, "cb.pth")}, assets)
        cbg.get_topk_poses(O.TEXT)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        cbg.get_topk_poses(O.TEXT)
        torch.cuda.synchronize()
        res["codebook_get_topk_poses_s"] = time.perf_counter() - t0
        try:
            t0 = time.perf_counter()
            nvp.get_topk_poses(O.TEXT)
            torch.cuda.synchronize()
            res["realnvp_get_topk_poses_s"] = time.perf_counter() - t0
        except RuntimeError as e:      # random weights: no draw of a candidate may score above 0
            res["realnvp_get_topk_poses_s"] = None
            res["realnvp_error"] = str(e)
    print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()
