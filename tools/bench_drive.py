"""Time the mesh-animation step (avatarclip_b200.drive.generate_animation) stage by stage on an avatar-sized mesh.

The mesh is the SMPL template (tests/golden/ref_tree_template.tar.gz) in the stand pose, subdivided three times by
midpoint subdivision (440 834 vertices, 881 664 faces; the avatar the reference ships, Avatar2FBX/meshes/
abrahamlincoln.ply, has 185 428 vertices), jittered, plus a few singleton vertices for cleanup to remove.  The SMPL
tensors are the tests' synthetic ones with the real template; the motion is 120 seeded frames.  Every stage is timed
with CUDA events after one warm-up run, bracketed by device synchronisations, so the PLY and PC2 stages include their
file I/O.  Prints the card name and power limit with the numbers, and one JSON line.

    python tools/bench_drive.py [--levels 3] [--frames 120] [--repeats 3]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from avatarclip_b200 import drive, handoff  # noqa: E402
from oracle import drive as D  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
    except Exception:
        name, limit = torch.cuda.get_device_name(), "unknown"
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, default=3)
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_drive needs a CUDA device")
    g = torch.load(os.path.join(ROOT, "tests", "golden", "ref_drive_small.pt"), weights_only=False)
    smpl = D.golden_smpl(g["smpl_seed"])
    stand_bytes = g["stand_pose_npy"].numpy().tobytes()
    v, f = D.bench_mesh(smpl, np.load(io.BytesIO(stand_bytes)), levels=a.levels)
    v = np.concatenate([v, np.random.default_rng(1).normal(0, 1, (4, 3)).astype(np.float32)])
    c = np.random.default_rng(2).integers(0, 256, v.shape, dtype=np.uint8)
    motion = np.random.default_rng(3).normal(0, 0.3, (a.frames, 72)).astype(np.float32)

    with tempfile.TemporaryDirectory() as tmp:
        ply = handoff.write_ply(os.path.join(tmp, "avatar.ply"), v, f, c)
        mot = os.path.join(tmp, "motion.npy")
        np.save(mot, motion)
        stand = os.path.join(tmp, "stand_pose.npy")
        open(stand, "wb").write(stand_bytes)
        out = os.path.join(tmp, "out")
        s = drive.smpl_tensors(smpl, "cuda")
        drive.generate_animation(ply, mot, out, s, stand)          # warm-up: module load, allocator, page cache

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

            mesh = run("read_ply", lambda: drive.read_ply(ply))
            x = mesh.vertices
            mesh = run("rotate+cleanup_mesh", lambda: drive.cleanup_mesh(mesh._replace(
                vertices=torch.stack([x[:, 0], -x[:, 2], x[:, 1]], 1).contiguous())))
            run("write_ply", lambda: drive.write_ply(mesh, os.path.join(out, "avatar_cleaned_apose.ply")))
            tmpl, pose_rot, _ = run("load_template_smpl", lambda: drive.load_template_smpl(s, stand))
            near = run("find_nearest_ind", lambda: drive._nearest(mesh.vertices, tmpl["vertices"].reshape(-1, 3)))
            A0 = run("rel_transforms(stand)", lambda: drive._rel_transforms(s, pose_rot.reshape(1, 24, 9).contiguous(),
                                                                              False))
            tp = run("inv_lbs", lambda: drive._inv_lbs(mesh.vertices, near, s["lbs_weights"], A0[0]))
            mo = torch.from_numpy(drive._motion_axis_angle(mot)).cuda()
            A = run("rel_transforms(motion)", lambda: drive._rel_transforms(s, mo, True))
            buf = torch.empty(a.frames, tp.shape[0], 3, device="cuda")
            run("lbs_frames(kernel only)", lambda: drive._lbs_frames(tp, near, s["lbs_weights"], A, 0, a.frames, buf))
            torch.cuda.synchronize()
            e0, e1 = ev(), ev()
            e0.record()
            drive.generate_animation(ply, mot, out, s, stand)
            e1.record()
            torch.cuda.synchronize()
            st["generate_animation(total)"] = e0.elapsed_time(e1)
            st["pc2 frames+write (total - other stages)"] = st["generate_animation(total)"] - sum(
                st[k] for k in ("read_ply", "rotate+cleanup_mesh", "write_ply", "load_template_smpl",
                                "find_nearest_ind", "rel_transforms(stand)", "inv_lbs", "rel_transforms(motion)"))
            return st, mesh.vertices.shape[0], mesh.triangles.shape[0]

        runs = [stages() for _ in range(a.repeats)]
    name, limit = card()
    V, F = runs[0][1], runs[0][2]
    med = {k: float(np.median([r[0][k] for r in runs])) for k in runs[0][0]}
    print(f"card: {name}, power limit {limit}")
    print(f"mesh: {v.shape[0]} vertices / {f.shape[0]} faces in, {V} / {F} after cleanup; {a.frames} frames; "
          f"PC2 {32 + a.frames * V * 12} bytes; median of {a.repeats} runs after one warm-up")
    for k, ms in med.items():
        print(f"  {k:42s} {ms:9.3f} ms")
    print(json.dumps({"bench": "drive", "card": name, "power_limit": limit, "vertices_in": int(v.shape[0]),
                      "vertices": int(V), "faces": int(F), "frames": a.frames, "ms": med}))


if __name__ == "__main__":
    main()
