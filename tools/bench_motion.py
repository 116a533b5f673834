"""Time AvatarAnimate's motion stage on the device and print one JSON line.

Medians of CUDA-event times over --reps calls after --warmup calls: the VPoser encode of 5 poses (avc_vposer_encode),
MotionInterpolation's interpolate + decode of 60 frames, one optimiser iteration (avc_motion_optimize with n = 1, which
includes its graph capture and instantiation), the shipped 5 000-iteration call, and the per-iteration time that
follows from it.  Then, in wall time, the whole command (``python -m avatarclip_b200.motion``, in-process) from files to
mp4 on a baseline conf at 5 000 iterations.  The card's name and power limit are read in the same run.  All inputs are
synthetic and seeded (oracle/motion.py, oracle/animate.py, oracle/shapegen.py): full-size VPoser, motion VAE decoder
(latent 256, 4 layers, 4 heads, FF 1024, 60 frames) and random ViT-B/32 towers.

    python tools/bench_motion.py [--reps 10] [--warmup 2]
"""
import argparse
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

from bench_animate import _power_limit, _time  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    from avatarclip_b200 import motion as M
    from oracle import animate as OA
    from oracle import drive as D
    from oracle import motion as OM
    from oracle import shapegen as OS
    dev = torch.device("cuda")
    vp = {k: v.to(dev) for k, v in {**OA.vposer_state(), **OM.vposer_encoder_state()}.items()}
    poses = (torch.randn(5, 63, generator=torch.Generator().manual_seed(0)) * 0.3).to(dev)
    vae = M.load_motion_vae(OM.motion_vae_state(), device=dev)
    z0 = torch.randn(256, generator=torch.Generator().manual_seed(1)).to(dev)
    interp = M.MotionInterpolation(vposer=vp)
    coef = [1.0] * 5
    r = {"device": torch.cuda.get_device_name(0), "power_limit": _power_limit()}
    r["vposer_encode_5_ms"] = _time(lambda: M.vposer_encode(poses, vp), a.reps, a.warmup)
    r["interpolate_decode_60_ms"] = _time(lambda: interp.get_motion("", poses), a.reps, a.warmup)
    r["motion_decode_ms"] = _time(lambda: M.motion_decode(z0, vae), a.reps, a.warmup)
    r["optimizer_1_iter_call_ms"] = _time(lambda: M.motion_optimize(vae, poses, coef, 0.0, z0, 1, lr=0.01), a.reps,
                                          a.warmup)
    r["optimizer_5000_iter_call_ms"] = _time(lambda: M.motion_optimize(vae, poses, coef, 0.0, z0, 5000, lr=0.01),
                                             max(3, a.reps // 3), 1)
    r["optimizer_per_iter_us"] = r["optimizer_5000_iter_call_ms"] * 1000 / 5000

    with tempfile.TemporaryDirectory() as tmp:
        tv, tf = D.template_obj()
        smpl = {k: np.asarray(v) for k, v in D.golden_smpl().items()}
        smpl["faces"] = tf
        np.savez(os.path.join(tmp, "smpl.npz"), **smpl)
        os.makedirs(os.path.join(tmp, "vposer", "snapshots"))
        torch.save({"state_dict": {"vp_model." + k: v.cpu() for k, v in vp.items()}},
                   os.path.join(tmp, "vposer", "snapshots", "V02_05.ckpt"))
        visual, text = OS.clip_states()
        torch.save({**{k: v.half() for k, v in visual.items()}, **{k: v.half() for k, v in text.items()}},
                   os.path.join(tmp, "clip.pt"))
        uv = OS.write_uv_obj(os.path.join(tmp, "data"), smpl["v_template"], smpl["faces"])
        torch.save(OA.make_codebook(torch.randn(512, generator=torch.Generator().manual_seed(0))),
                   os.path.join(tmp, "data", "codebook.pth"))
        torch.save({"state_dict": OM.motion_vae_state()}, os.path.join(tmp, "data", "motion_vae.pth"))
        conf = os.path.join(tmp, "walk.conf")
        with open(conf, "w") as f:
            f.write(f"general {{\n    base_exp_dir = {tmp}/exp\n    mode = motion\n    text = a rendered 3d man is "
                    "walking\n}\n\npose_generator {\n    type = VPoserCodebook\n}\n\nmotion_generator {\n    type = "
                    "MotionOptimizer\n    recon_coef = [1.0, 1.0, 1.0, 1.0, 1.0]\n    clip_coef = 0.0\n"
                    "    delta_coef = 0.0\n}\n")
        args = ["--conf", conf, "--smpl", os.path.join(tmp, "smpl.npz"), "--vposer", os.path.join(tmp, "vposer"),
                "--uv_obj", uv, "--codebook", os.path.join(tmp, "data", "codebook.pth"), "--motion_vae",
                os.path.join(tmp, "data", "motion_vae.pth"), "--clip_model", os.path.join(tmp, "clip.pt"), "--bpe",
                OS.write_bpe(os.path.join(tmp, "bpe.txt.gz")), "--seed", "0"]
        walls = []
        for _ in range(2):          # the first run loads the modules and picks the CLIP tower's algorithms
            torch.cuda.synchronize()
            t = time.perf_counter()
            M.main(args)
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t)
        r["command_files_to_mp4_s"] = walls[-1]
        r["command_first_run_s"] = walls[0]
    print(json.dumps(r))


if __name__ == "__main__":
    main()
