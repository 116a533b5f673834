"""Time quadric-error decimation (avc_mesh_decimate) on an avatar-sized mesh and the textured exports it enables.

The mesh is tools/bench_export.py's: the stand-pose template subdivided three times, 440 834 vertices and 881 664 faces
in the PLY frame.  Vertex clustering at resolution 256 keeps 803 006 of those faces.  For each of ``--targets``:
  decimate  ``export._decimate`` of the mesh as read: rounds, and CUDA events around one synchronised call
  reduce    ``export.reduce_mesh(mesh, 256, target)``, what ``export --target_faces`` runs (clustering, decimation,
            clustering), with the face count it keeps and its two-sided distance to the input (oracle/decimate.py,
            2 000 000 samples on the input), beside clustering alone at 256
Each time is the median of ``--repeats`` calls after one warm-up call.  Then ``export_avatar`` end to end (the PLY
file to the .glb) with and without ``--target_faces``, and the textured export of the reduced mesh at each of
``--texture_sizes``: the six-view render time and the .glb size.  The renders use a Runner of the shipped network size
at its geometric initialisation, as tools/bench_bake.py does.  Prints the card name and power limit and one JSON line.

    python tools/bench_decimate.py [--targets 50000,20000,13776] [--texture_sizes 1024,2048] [--bake_target 20000]
"""
import argparse
import io
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from avatarclip_b200 import bake, drive, handoff  # noqa: E402
from avatarclip_b200 import export as X  # noqa: E402
from bench_bake import make_conf, median, timed  # noqa: E402
from bench_drive import card  # noqa: E402
from oracle import decimate as O  # noqa: E402
from oracle import drive as D  # noqa: E402

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--targets", default="50000,20000,13776")
    ap.add_argument("--texture_sizes", default="1024,2048")
    ap.add_argument("--bake_target", type=int, default=20000)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decimate needs a CUDA device")
    g = torch.load(os.path.join(ROOT, "tests", "golden", "ref_drive_small.pt"), weights_only=False)
    smpl = D.golden_smpl(g["smpl_seed"])
    stand_bytes = g["stand_pose_npy"].numpy().tobytes()
    v, f = D.bench_mesh(smpl, np.load(io.BytesIO(stand_bytes)), levels=3)
    mesh = drive.Mesh(torch.from_numpy(v).cuda(), torch.from_numpy(f.astype(np.int32)).cuda(), None)
    cl = X.simplify_mesh(mesh, 256)
    SPACING = O.spacing_for(v, f)
    res = {"input_faces": int(f.shape[0]), "spacing": SPACING, "clustered_faces": int(cl.triangles.shape[0]),
           "clustered_distance": O.surface_distance(v, f, cl.vertices.cpu().numpy(), cl.triangles.cpu().numpy(),
                                                    SPACING), "targets": []}
    print(f"input {f.shape[0]} faces; clustered at 256: {res['clustered_faces']} faces, distance "
          f"{res['clustered_distance']}", flush=True)
    X._decimate(mesh, 50000)                                                   # warm-up
    X.reduce_mesh(mesh, 256, 50000)
    for t in map(int, a.targets.split(",")):
        ms_dec, (_, rounds) = median(lambda: X._decimate(mesh, t), a.repeats)
        ms_red, red = median(lambda: X.reduce_mesh(mesh, 256, t), a.repeats)
        d = O.surface_distance(v, f, red.vertices.cpu().numpy(), red.triangles.cpu().numpy(), SPACING)
        row = dict(target=t, rounds=rounds, decimate_ms=ms_dec, reduce_ms=ms_red, faces=int(red.triangles.shape[0]),
                   distance=d)
        res["targets"].append(row)
        print(f"target {t:6d}: {rounds} rounds, decimate {ms_dec:.1f} ms, reduce_mesh {ms_red:.1f} ms -> "
              f"{row['faces']} faces, distance mean {d['mean']:.3e} p99 {d['p99']:.3e} m", flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        ply = handoff.write_ply(os.path.join(tmp, "avatar.ply"), v, f, np.full(v.shape, 128, np.uint8))
        stand = os.path.join(tmp, "stand_pose.npy")
        open(stand, "wb").write(stand_bytes)
        s = drive.smpl_tensors(smpl, "cuda")
        out = os.path.join(tmp, "a.glb")
        X.export_avatar(ply, out, s, stand)                                      # warm-up
        e2e = {}
        for label, tf in (("clustered", None), (f"target_{a.bake_target}", a.bake_target)):
            e2e[label + "_ms"], _ = median(lambda: X.export_avatar(ply, out, s, stand, target_faces=tf), a.repeats)
            e2e[label + "_glb_bytes"] = os.path.getsize(out)
        res["export"] = e2e
        print(f"export_avatar end to end: {e2e}", flush=True)
        from avatarclip_b200.runner import Runner
        runner = Runner(make_conf(tmp, "shipped"), "validate_mesh", "smpl", device="cuda")
        rig = X.rig_avatar(ply, s, stand, ply_frame=True, target_faces=a.bake_target)
        vp, tri = torch.from_numpy(rig["vertices_ply"]).cuda(), torch.from_numpy(rig["triangles"]).cuda()
        bake.bake_texture(runner, vp, tri[:2000], 1024)                          # warm-up
        res["textured"] = []
        for T in map(int, a.texture_sizes.split(",")):
            cell = bake.atlas_grid(rig["triangles"].shape[0], T)[1]
            t_map, (owner, _, _) = timed(lambda: bake.texel_points(vp, tri, T))
            t_bake, (uv, tex) = timed(lambda: bake.bake_texture(runner, vp, tri, T))
            nrm = bake.vertex_normals(torch.from_numpy(rig["vertices"]).cuda(), tri).cpu().numpy()
            path = os.path.join(tmp, f"t{T}.glb")
            t0 = time.perf_counter()
            X.write_glb(dict(rig, normals=nrm), path, texture=(uv, tex))
            row = dict(texture=T, faces=int(rig["triangles"].shape[0]), cell=cell, used_texels=int((owner >= 0).sum()),
                       renders_ms=t_bake - t_map, glb_write_ms=1e3 * (time.perf_counter() - t0),
                       glb_bytes=os.path.getsize(path))
            res["textured"].append(row)
            print(f"textured T {T}: {row}", flush=True)
    name, limit = card()
    print(f"card: {name}, power limit {limit}; medians of {a.repeats} calls after one warm-up")
    print(json.dumps({"bench": "decimate", "card": name, "power_limit": limit, **res}))


if __name__ == "__main__":
    main()
