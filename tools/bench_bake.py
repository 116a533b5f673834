"""Time the texture bake of the textured export (avatarclip_b200.bake) stage by stage.

The mesh is tools/bench_export.py's (the stand-pose template subdivided three times: 440 834 vertices in the PLY frame),
clustered at each ``--resolutions`` value; a texture too small for the faces is reported as refused.  The colour
field is a Runner of the shipped network size (confs/examples/hulk.conf: SDF 4 x 256, colour 2 x 256, 32 + 32 samples, 4
up-sampling steps) at its geometric initialisation, since the full-size pretrained checkpoint is not part of the repository; ``--conf small`` takes
confs/examples_small with its stand-pose checkpoint instead.  The rays a texel costs do not depend on the weights.

Stages, each timed with CUDA events bracketed by device synchronisations:
  texel map   ``bake.texel_points`` (avc_bake_texel_points)
  bake        ``bake.bake_texture``: the texel map, six-view renders of every used texel (``Runner.surface_colors``,
              65 536-ray chunks, mid-bin samples) and the scatter; renders = bake - texel map, reported as rays / s
  normals     ``bake.vertex_normals`` of the bind pose (adjacency included)
  png         ``bake.encode_png`` (cv2, on the host)
  glb         ``export.write_glb`` with the texture (PNG included)
One warm-up bake runs first; every stage is the median of ``--repeats`` runs (``--render_repeats`` for the bake,
which dominates).  Prints the card name and power limit with the numbers and one JSON line.

    python tools/bench_bake.py [--resolutions 64,96,128] [--texture_sizes 1024,2048,4096] [--conf shipped|small]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from avatarclip_b200 import bake, drive, handoff  # noqa: E402
from avatarclip_b200 import export as X  # noqa: E402
from avatarclip_b200.runner import Runner  # noqa: E402
from bench_drive import card  # noqa: E402
from oracle import drive as D  # noqa: E402
from util_neus import reference_tree  # noqa: E402


def make_conf(tmp: str, which: str) -> str:
    ag = reference_tree(os.path.join(tmp, "ref"))
    src = {"shipped": "confs/examples/hulk.conf", "small": "confs/examples_small/example.conf"}[which]
    text = open(os.path.join(ag, src)).read()
    for old, new in (("./exp/", os.path.join(tmp, "exp") + "/"), ("./data/", ag + "/data/"),
                     ("./pretrained_models/", ag + "/pretrained_models/")):
        text = text.replace(old, new)
    path = os.path.join(tmp, "bench.conf")
    open(path, "w").write(text)
    return path


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), r


def median(fn, n):
    runs = [timed(fn) for _ in range(n)]
    return float(np.median([t for t, _ in runs])), runs[-1][1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resolutions", default="64,96,128")
    ap.add_argument("--texture_sizes", default="1024,2048,4096")
    ap.add_argument("--conf", choices=("shipped", "small"), default="shipped")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--render_repeats", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bake needs a CUDA device")
    g = torch.load(os.path.join(ROOT, "tests", "golden", "ref_drive_small.pt"), weights_only=False)
    smpl = D.golden_smpl(g["smpl_seed"])
    stand_bytes = g["stand_pose_npy"].numpy().tobytes()
    v, f = D.bench_mesh(smpl, np.load(io.BytesIO(stand_bytes)), levels=3)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        runner = Runner(make_conf(tmp, a.conf), "validate_mesh", "smpl", device="cuda")
        ply = handoff.write_ply(os.path.join(tmp, "avatar.ply"), v, f, np.full(v.shape, 128, np.uint8))
        stand = os.path.join(tmp, "stand_pose.npy")
        open(stand, "wb").write(stand_bytes)
        s = drive.smpl_tensors(smpl, "cuda")
        rigs = {r: X.rig_avatar(ply, s, stand, r, ply_frame=True) for r in map(int, a.resolutions.split(","))}
        warm = rigs[min(rigs)]
        bake.bake_texture(runner, warm["vertices_ply"], warm["triangles"][:2000], 1024)     # warm-up
        for res, rig in rigs.items():
            vp = torch.from_numpy(rig["vertices_ply"]).cuda()
            tri = torch.from_numpy(rig["triangles"]).cuda()
            for T in map(int, a.texture_sizes.split(",")):
                try:
                    bake.atlas_grid(rig["triangles"].shape[0], T)
                except bake.AtlasTooSmall as e:
                    rows.append(dict(resolution=res, faces=int(rig["triangles"].shape[0]), texture=T, refused=str(e)))
                    print(f"res {res:4d}  T {T:5d}  refused: {e}", flush=True)
                    continue
                st = {}
                st["texel_map"], (owner, _, _) = median(lambda: bake.texel_points(vp, tri, T), a.repeats)
                used = int((owner >= 0).sum())
                st["bake"], (uv, tex) = median(lambda: bake.bake_texture(runner, vp, tri, T), a.render_repeats)
                st["renders"] = st["bake"] - st["texel_map"]
                st["normals"], nrm = median(lambda: bake.vertex_normals(torch.from_numpy(rig["vertices"]).cuda(), tri),
                                            a.repeats)
                st["png"], _ = median(lambda: bake.encode_png(tex), a.repeats)
                out = dict(rig, normals=nrm.cpu().numpy())
                path = os.path.join(tmp, "t.glb")
                st["glb"], _ = median(lambda: X.write_glb(out, path, texture=(uv, tex)), a.repeats)
                rays = 6 * used
                row = dict(resolution=res, faces=int(rig["triangles"].shape[0]), texture=T,
                           cell=bake.atlas_grid(rig["triangles"].shape[0], T)[1], used_texels=used, rays=rays,
                           mrays_per_s=rays / (st["renders"] * 1e3), glb_bytes=os.path.getsize(path), ms=st)
                rows.append(row)
                print(f"res {res:4d}  {row['faces']:7d} faces  T {T:5d}  cell {row['cell']:3d}  {used:9d} texels  "
                      + "  ".join(f"{k} {ms:9.1f} ms" for k, ms in st.items())
                      + f"  {row['mrays_per_s']:6.2f} Mrays/s  glb {row['glb_bytes'] / 2 ** 20:.1f} MiB", flush=True)
    name, limit = card()
    print(f"card: {name}, power limit {limit}; conf {a.conf}; medians of {a.repeats} runs ({a.render_repeats} for the "
          "bake) after one warm-up bake")
    print(json.dumps({"bench": "bake", "card": name, "power_limit": limit, "conf": a.conf, "rows": rows}))


if __name__ == "__main__":
    main()
