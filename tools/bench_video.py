"""Time video rendering (avatarclip_b200.video) stage by stage on an avatar-sized mesh.

The mesh is the one tools/bench_drive.py animates: the SMPL template in the stand pose subdivided three times (440 834
vertices, 881 664 faces), jittered, with seeded colours; the SMPL tensors are the tests' synthetic ones with the real
template and the motion is 120 seeded frames, rendered at 512 x 512 with 2 x 2 supersampling.  Every stage is timed with
CUDA events after one warm-up run, bracketed by device synchronisations:
  rig            read the PLY, rotate, cleanup_mesh, nearest template vertex, inverse LBS (drive.rig_mesh) + adjacency
  skin           avc_lbs_frames of all frames (kernel time)
  render         avc_video_render of all frames, one chunk at a time (kernel time; also per frame)
  d2h            the frames' copy to pinned host memory
  encode         write_video of the host frames (mp4v)
  total          iter_motion_frames + write_video, the whole call
Prints the card name and power limit with the medians of --repeats runs, and one JSON line.  Writes the videos under
--out_dir (a temporary directory when omitted).

    python tools/bench_video.py [--out_dir DIR] [--levels 3] [--frames 120] [--image_size 512] [--supersample 2]
"""
import argparse
import io
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from avatarclip_b200 import drive, handoff, video  # noqa: E402
from bench_drive import card  # noqa: E402
from oracle import drive as D  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out_dir", default=None)
    ap.add_argument("--levels", type=int, default=3)
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--image_size", type=int, default=512)
    ap.add_argument("--supersample", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_video needs a CUDA device")
    g = torch.load(os.path.join(ROOT, "tests", "golden", "ref_drive_small.pt"), weights_only=False)
    smpl = D.golden_smpl(g["smpl_seed"])
    stand_bytes = g["stand_pose_npy"].numpy().tobytes()
    v, f = D.bench_mesh(smpl, np.load(io.BytesIO(stand_bytes)), levels=a.levels)
    c = np.random.default_rng(2).integers(0, 256, v.shape, dtype=np.uint8)
    motion = np.random.default_rng(3).normal(0, 0.3, (a.frames, 72)).astype(np.float32)
    n, ss = a.image_size, a.supersample

    with tempfile.TemporaryDirectory() as tmp:
        out = a.out_dir or tmp
        os.makedirs(out, exist_ok=True)
        ply = handoff.write_ply(os.path.join(tmp, "avatar.ply"), v, f, c)
        mot = os.path.join(tmp, "motion.npy")
        np.save(mot, motion)
        stand = os.path.join(tmp, "stand_pose.npy")
        open(stand, "wb").write(stand_bytes)
        s = drive.smpl_tensors(smpl, "cuda")
        mp4 = os.path.join(out, "bench_motion.mp4")
        video.write_video(video.iter_motion_frames(ply, mot, s, stand, image_size=n, supersample=ss), mp4)  # warm-up

        def stages():
            st = {}
            ev = lambda: torch.cuda.Event(enable_timing=True)

            def run(name, fn):
                torch.cuda.synchronize()
                e0, e1 = ev(), ev()
                e0.record()
                r = fn()
                e1.record()
                torch.cuda.synchronize()
                st[name] = e0.elapsed_time(e1)
                return r

            m = run("rig", lambda: video.motion_rig(ply, mot, s, stand))
            mesh = m.rig.mesh
            V, F = mesh.vertices.shape[0], mesh.triangles.shape[0]
            adj = video.adjacency(mesh.triangles, V)
            colors = torch.from_numpy(mesh.vertex_colors).cuda()
            chunk = video._chunk_frames(V, F, n, ss, a.frames, None, True)
            verts = torch.empty(a.frames, V, 3, device="cuda")
            run("skin", lambda: video.skin(m, 0, a.frames, verts))
            flat = verts.reshape(-1, 3)
            cams = video.orbit_cameras(*video._bounding_sphere(flat.amin(0), flat.amax(0)), a.frames, n)
            rgb = torch.empty(a.frames, n, n, 3, dtype=torch.uint8, device="cuda")
            ws = torch.empty(video.render_workspace_bytes(V, F, chunk, n, ss), dtype=torch.uint8, device="cuda")

            def render_all():
                for f0 in range(0, a.frames, chunk):
                    k = min(chunk, a.frames - f0)
                    video.render(verts[f0:f0 + k], mesh.triangles, adj, colors, cams[f0:f0 + k], n, ss, out=rgb[f0:f0 + k],
                                 workspace=ws)
            run("render", render_all)
            host = torch.empty(rgb.shape, dtype=torch.uint8, pin_memory=True)
            run("d2h", lambda: host.copy_(rgb, non_blocking=True))
            frames = host.numpy()
            run("encode", lambda: video.write_video(iter(frames), os.path.join(out, "bench_encode.mp4")))
            run("total", lambda: video.write_video(
                video.iter_motion_frames(ply, mot, s, stand, image_size=n, supersample=ss), mp4))
            st["render per frame"] = st["render"] / a.frames
            return st, V, F, chunk

        runs = [stages() for _ in range(a.repeats)]
    name, limit = card()
    V, F, chunk = runs[0][1:]
    med = {k: float(np.median([r[0][k] for r in runs])) for k in runs[0][0]}
    print(f"card: {name}, power limit {limit}")
    print(f"mesh: {V} vertices / {F} faces; {a.frames} frames at {n} x {n}, {ss} x {ss} supersampling, "
          f"{chunk} frames per chunk; median of {a.repeats} runs after one warm-up")
    for k, ms in med.items():
        print(f"  {k:20s} {ms:9.3f} ms")
    print(json.dumps({"bench": "video", "card": name, "power_limit": limit, "vertices": int(V), "faces": int(F),
                      "frames": a.frames, "image_size": n, "supersample": ss, "frames_per_chunk": int(chunk),
                      "ms": med}))


if __name__ == "__main__":
    main()
