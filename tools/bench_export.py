"""Time the avatar export (avatarclip_b200.export) stage by stage on an avatar-sized mesh.

The mesh is tools/bench_drive.py's: the SMPL template in the stand pose, subdivided three times (440 834 vertices,
881 664 faces), jittered, with random colours; the SMPL tensors are the tests' synthetic ones with the real template;
the motion is 120 seeded frames.  Every stage is timed with CUDA events after one warm-up run, bracketed by device
synchronisations (so the PLY read and the .glb write include their file I/O); the median of ``--repeats`` runs is
reported.  Prints the card name and power limit with the numbers, the clustered vertex / triangle counts, the .glb size
next to the PC2 size drive writes for the same motion, and one JSON line.

    python tools/bench_export.py [--levels 3] [--frames 120] [--repeats 3]
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

from avatarclip_b200 import drive, handoff  # noqa: E402
from avatarclip_b200 import export as X  # noqa: E402
from bench_drive import card  # noqa: E402
from oracle import drive as D  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, default=3)
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_export needs a CUDA device")
    g = torch.load(os.path.join(ROOT, "tests", "golden", "ref_drive_small.pt"), weights_only=False)
    smpl = D.golden_smpl(g["smpl_seed"])
    stand_bytes = g["stand_pose_npy"].numpy().tobytes()
    v, f = D.bench_mesh(smpl, np.load(io.BytesIO(stand_bytes)), levels=a.levels)
    c = np.random.default_rng(2).integers(0, 256, v.shape, dtype=np.uint8)
    motion = np.random.default_rng(3).normal(0, 0.3, (a.frames, 72)).astype(np.float32)

    with tempfile.TemporaryDirectory() as tmp:
        ply = handoff.write_ply(os.path.join(tmp, "avatar.ply"), v, f, c)
        mot = os.path.join(tmp, "motion.npy")
        np.save(mot, motion)
        stand = os.path.join(tmp, "stand_pose.npy")
        open(stand, "wb").write(stand_bytes)
        s = drive.smpl_tensors(smpl, "cuda")
        X.export_avatar(ply, os.path.join(tmp, "warm.glb"), s, stand, mot)     # warm-up: module load, allocator, cache

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
            sm = run("simplify_mesh (cluster)", lambda: X.simplify_mesh(mesh))
            x = sm.vertices
            rot = torch.stack([x[:, 0], -x[:, 2], x[:, 1]], 1).contiguous()
            tmpl, pose_rot, _ = run("load_template_smpl", lambda: drive.load_template_smpl(s, stand))
            near = run("find_nearest_ind (f32)", lambda: X._nearest_f32(rot, tmpl["vertices"].reshape(-1, 3)))
            A0 = drive._rel_transforms(s, pose_rot.reshape(1, 24, 9).contiguous(), False)
            run("inv_lbs", lambda: drive._inv_lbs(rot, near, s["lbs_weights"], A0[0]))
            rig = X.rig_avatar(ply, s, stand)
            run("write_glb (no motion)", lambda: X.write_glb(rig, os.path.join(tmp, "a.glb")))
            run("write_glb (motion)", lambda: X.write_glb(rig, os.path.join(tmp, "b.glb"), mot))
            run("export_avatar (no motion)", lambda: X.export_avatar(ply, os.path.join(tmp, "c.glb"), s, stand))
            run("export_avatar (motion)", lambda: X.export_avatar(ply, os.path.join(tmp, "d.glb"), s, stand, mot))
            sizes = {k: os.path.getsize(os.path.join(tmp, k)) for k in ("c.glb", "d.glb")}
            return st, sm.vertices.shape[0], sm.triangles.shape[0], sizes

        runs = [stages() for _ in range(a.repeats)]
    name, limit = card()
    K, T, sizes = runs[0][1], runs[0][2], runs[0][3]
    med = {k: float(np.median([r[0][k] for r in runs])) for k in runs[0][0]}
    pc2 = 32 + a.frames * v.shape[0] * 12          # what drive writes for this mesh (cleanup keeps every vertex here)
    print(f"card: {name}, power limit {limit}")
    print(f"mesh: {v.shape[0]} vertices / {f.shape[0]} faces in, {K} / {T} after clustering; {a.frames} frames; "
          f"median of {a.repeats} runs after one warm-up")
    print(f"files: .glb {sizes['c.glb']} bytes without motion, {sizes['d.glb']} with it; PC2 of the same motion "
          f"{pc2} bytes")
    for k, ms in med.items():
        print(f"  {k:32s} {ms:9.3f} ms")
    print(json.dumps({"bench": "export", "card": name, "power_limit": limit, "vertices_in": int(v.shape[0]),
                      "faces_in": int(f.shape[0]), "vertices": int(K), "faces": int(T), "frames": a.frames,
                      "glb_bytes": sizes["c.glb"], "glb_motion_bytes": sizes["d.glb"], "pc2_bytes": pc2, "ms": med}))


if __name__ == "__main__":
    main()
