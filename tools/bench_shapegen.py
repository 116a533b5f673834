"""Time ShapeGen's stages on the device and print one JSON line.

Per stage, the median of CUDA-event times over --reps calls after --warmup calls: the shape-VAE decode of one latent
(avc_vae_decode, with the HBM bandwidth its 677 MB weight stream achieves), the texture loading of an SMPL-sized UV
mesh (avc_load_textures), the textured 256 x 256 render (avc_raster_textured), the CLIP image encode of that render
(nearest resize + Normalize + ClipImageTower), and the codebook score (avc_codebook_argmax).  Then one end-to-end
``run_shape_gen`` from files -- weight load, text encodes, decode, render, image encode, search, decode -- in wall time.
All inputs are synthetic and seeded (oracle/shapegen.py): SMPL-sized template, full-size VAE, random ViT-B/32 towers.

    python tools/bench_shapegen.py [--reps 50] [--warmup 5] [--codebook 4096]
"""
import argparse
import json
import os
import sys
import tempfile
import time

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--codebook", type=int, default=4096)
    a = ap.parse_args()
    from avatarclip_b200 import shapegen as S
    from oracle import drive as D
    from oracle import shapegen as O

    tv, tf = D.template_obj()
    vae = O.vae_state(tv)
    dev = {k: v.cuda() for k, v in vae.items()}
    vt = torch.from_numpy(tv).cuda().reshape(-1)
    z = torch.zeros(1, 16, device="cuda")
    res = {"gpu": torch.cuda.get_device_name(0)}
    res["decode_ms"] = _time(lambda: S.vae_decode(z, dev["dec1.weight"], dev["dec1.bias"], dev["dec2.weight"],
                                                  dev["dec2.bias"], vt), a.reps, a.warmup)
    res["decode_GBps"] = dev["dec2.weight"].numel() * 4 / (res["decode_ms"] * 1e-3) / 1e9
    z8 = torch.randn(8, 16, device="cuda")
    res["decode_b8_ms"] = _time(lambda: S.vae_decode(z8, dev["dec1.weight"], dev["dec1.bias"], dev["dec2.weight"],
                                                     dev["dec2.bias"], vt), a.reps, a.warmup)
    with tempfile.TemporaryDirectory() as tmp:
        obj = O.write_uv_obj(os.path.join(tmp, "uv"), tv, tf)
        face_uv, mats, images = S.read_uv_obj(obj)
        img = S._read_image_rgb01(images["skin"]).cuda()
        uv = torch.from_numpy(face_uv).cuda()
        upd = torch.ones(len(mats), dtype=torch.int32, device="cuda")
        tex = torch.ones(len(mats), 8, 8, 8, 3, device="cuda")
        res["texture_load_ms"] = _time(lambda: S.load_textures(img, uv, upd, tex), a.reps, a.warmup)
        tex = S.load_obj_textures(obj)
        v = S.vae_decode(z, dev["dec1.weight"], dev["dec1.bias"], dev["dec2.weight"], dev["dec2.bias"], vt)
        v = v.reshape(1, -1, 3)
        res["raster_ms"] = _time(lambda: S.render_one_batch(v, tf, tex), a.reps, a.warmup)
        images_ = S.render_one_batch(v, tf, tex)
        clip = S.load_clip(O.clip_states(), O.write_bpe(os.path.join(tmp, "bpe.txt.gz")))
        res["clip_encode_ms"] = _time(lambda: clip.image.encode_image(S.clip_prep_nearest(images_.permute(0, 2, 3, 1))),
                                      a.reps, a.warmup)
        g = torch.Generator(device="cuda").manual_seed(0)
        cb = torch.randn(a.codebook, 512, generator=g, device="cuda")
        e, d = torch.randn(512, device="cuda"), torch.randn(512, device="cuda")
        res["codebook"] = a.codebook
        res["score_ms"] = _time(lambda: S.codebook_argmax(cb, e, d), a.reps, a.warmup)

        torch.save(vae, os.path.join(tmp, "vae.pth"))
        torch.save({torch.randn(a.codebook, 16): cb.cpu()}, os.path.join(tmp, "codebook.pth"))
        smpl = {"v_template": tv, "faces": tf}
        del dev
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        S.run_shape_gen(smpl, os.path.join(tmp, "vae.pth"), os.path.join(tmp, "codebook.pth"), O.NEUTRAL_TXT,
                        O.TARGET_TXT, clip, obj)
        torch.cuda.synchronize()
        res["end_to_end_s"] = time.perf_counter() - t0
    print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()
