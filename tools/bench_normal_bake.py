"""Time the normal-map bake of the textured export (bake.bake_normal_map) phase by phase.

The mesh is tools/bench_bake.py's (the stand-pose template subdivided three times, in the PLY frame) reduced by
``export.rig_avatar(..., target_faces=20000)``, the engine-sized export.  The SDF is a Runner of the shipped network
size (confs/examples/hulk.conf: SDF 4 x 256) at its geometric initialisation, since the full-size pretrained checkpoint
is not part of the repository.  There most body texels find no sign change on their segment, but every texel runs
the same 16 + 12 sdf evaluations and one gradient whatever it finds, so the timing holds for a trained SDF.

Phases (wall clock around device synchronisations, ``bake_normal_map``'s ``timings``):
  frames            texel map, vertex normals, corner tangents, texel frames
  search_samples    16 samples per texel through avc_neus_sdf_query, and the bracket
  search_bisection  12 bisection steps, each one avc_neus_sdf_query pass over the texels
  gradient          avc_neus_sdf_eval's gradient at the snapped points
  encode            avc_bake_normal_encode and the copy to the host
then the bind pose's ``corner_tangents``, ``encode_png`` of the map and ``write_glb`` with texture and normal map.
One warm-up bake runs first; every number is the median of ``--repeats`` runs.  Prints the card name and power limit
read in the same process, and one JSON line.

    python tools/bench_normal_bake.py [--texture_sizes 1024,2048] [--target_faces 20000] [--repeats 3]
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
from avatarclip_b200.runner import Runner  # noqa: E402
from bench_bake import make_conf  # noqa: E402
from bench_drive import card  # noqa: E402
from oracle import drive as D  # noqa: E402


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--texture_sizes", default="1024,2048")
    ap.add_argument("--target_faces", type=int, default=20000)
    ap.add_argument("--resolution", type=int, default=X.DEFAULT_RESOLUTION)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_normal_bake needs a CUDA device")
    g = torch.load(os.path.join(ROOT, "tests", "golden", "ref_drive_small.pt"), weights_only=False)
    smpl = D.golden_smpl(g["smpl_seed"])
    stand_bytes = g["stand_pose_npy"].numpy().tobytes()
    v, f = D.bench_mesh(smpl, np.load(io.BytesIO(stand_bytes)), levels=3)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        runner = Runner(make_conf(tmp, "shipped"), "validate_mesh", "smpl", device="cuda")
        ply = handoff.write_ply(os.path.join(tmp, "avatar.ply"), v, f, np.full(v.shape, 128, np.uint8))
        stand = os.path.join(tmp, "stand_pose.npy")
        open(stand, "wb").write(stand_bytes)
        rig = X.rig_avatar(ply, drive.smpl_tensors(smpl, "cuda"), stand, a.resolution, ply_frame=True,
                           target_faces=a.target_faces)
        F = int(rig["triangles"].shape[0])
        vp = torch.from_numpy(rig["vertices_ply"]).cuda()
        tri = torch.from_numpy(rig["triangles"]).cuda()
        vb = torch.from_numpy(rig["vertices"]).cuda()
        rig["normals"] = bake.vertex_normals(vb, tri).cpu().numpy()
        bake.bake_normal_map(runner, vp, tri, 1024)                                    # warm-up
        for T in map(int, a.texture_sizes.split(",")):
            runs = []
            for _ in range(a.repeats):
                tm = {}
                ms, (image, stats) = wall(lambda: bake.bake_normal_map(runner, vp, tri, T, timings=tm))
                runs.append(dict({k: s * 1e3 for k, s in tm.items()}, bake=ms))
            st = {k: float(np.median([r[k] for r in runs])) for k in runs[0]}
            uv = bake.texel_points(vp, tri, T)[2]
            tr = [wall(lambda: bake.corner_tangents(vb, tri, torch.from_numpy(rig["normals"]), uv))
                  for _ in range(a.repeats)]
            st["tangents"], tg = float(np.median([t for t, _ in tr])), tr[-1][1]
            st["png"] = float(np.median([wall(lambda: bake.encode_png(image))[0] for _ in range(a.repeats)]))
            tex = np.zeros((T, T, 3), np.uint8)
            path = os.path.join(tmp, "n.glb")
            nm = (tg.cpu().numpy().reshape(-1, 4), image)
            st["glb"] = float(np.median([wall(lambda: X.write_glb(rig, path, texture=(uv.cpu().numpy(), tex),
                                                                  normal_map=nm))[0] for _ in range(a.repeats)]))
            n = stats["used"]
            evals = n * (bake.SNAP_SAMPLES + bake.SNAP_STEPS)
            row = dict(faces=F, texture=T, stats=stats, sdf_evaluations=evals,
                       sdf_evals_per_s=evals / ((st["search_samples"] + st["search_bisection"]) * 1e-3),
                       glb_bytes=os.path.getsize(path), ms=st)
            rows.append(row)
            print(f"{F:6d} faces  T {T:5d}  {n:9d} texels ({stats['converged']} converged, {stats['flat']} flat, "
                  f"{stats['back_facing']} back-facing)  " + "  ".join(f"{k} {ms:8.1f} ms" for k, ms in st.items())
                  + f"  {row['sdf_evals_per_s'] / 1e6:7.1f} M sdf/s", flush=True)
    name, limit = card()
    print(f"card: {name}, power limit {limit}; shipped network size at geometric init; medians of {a.repeats} runs "
          "after one warm-up bake")
    print(json.dumps({"bench": "normal_bake", "card": name, "power_limit": limit, "rows": rows}))


if __name__ == "__main__":
    main()
