"""A-B check of a change to the wgmma NT tiles: one render forward + backward of the bench workload (bench view, synthetic
weights, seeded cotangents) through a given build of the library, outputs and flat gradient saved as .npy.

    AVC_B200_LIB=/path/to/libavc_b200.so python tools/nt_epilogue_ab.py --out DIR      # on the GPU, once per build
    python tools/nt_epilogue_ab.py --compare DIR_A DIR_B [DIR_A2]                      # anywhere

--compare reports, per output, whether A and B are bitwise equal, and the largest gradient difference between A and B;
with a second run of A (DIR_A2) also between A and A2: the split-K reductions of the TN tiles accumulate with
red.global.add, so two runs of the same build differ in the last bits of the gradient."""
import argparse
import glob
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(out_dir):
    sys.path.insert(0, ROOT)
    import torch
    from avatarclip_b200 import _lib, workload as WL
    from avatarclip_b200.renderer import render_backward_raw, render_forward_raw
    from avatarclip_b200.trainer import DeviceView
    dev = torch.device("cuda", 0)
    sp, cp = WL.synth_states(WL.B2_SDF_KW, WL.B2_COL_KW, seed=0)
    _, _, _, ren = WL.build_networks(WL.B2_SDF_KW, WL.B2_COL_KW, WL.B2_REN_KW, sp, cp, 0.3, dev, engine=1)
    ren._ensure_flat(dev)
    dv = DeviceView(WL.make_view(0, n_rays=512, H=224, W=224, seed=0, bg_choice=3), dev)
    jit = dv.jitter if ren.perturb > 0 else None
    out, ws, chunk = render_forward_raw(ren, dv.rays_o, dv.rays_d, dv.near, dv.far, jit, None, 0, 1.0, None,
                                        keep_ws=True)
    g = torch.Generator().manual_seed(7)
    cot = {k: torch.randn(out[k].shape, generator=g).to(dev) for k in _lib._COT_FIELDS}
    grad = render_backward_raw(ren, dv.rays_o, dv.rays_d, None, 0, 1.0, out, ws, chunk, cot)
    torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    for k, v in out.items():
        np.save(os.path.join(out_dir, f"out_{k}.npy"), v.detach().cpu().numpy())
    np.save(os.path.join(out_dir, "grad.npy"), grad.detach().cpu().numpy())
    print("wrote", out_dir, "lib", _lib.LIB_PATH)


def compare(a, b, a2=None):
    rep = {"outputs_bitwise_equal": {}}
    for f in sorted(glob.glob(os.path.join(a, "out_*.npy"))):
        k = os.path.basename(f)[4:-4]
        x, y = np.load(f), np.load(os.path.join(b, os.path.basename(f)))
        rep["outputs_bitwise_equal"][k] = bool(x.tobytes() == y.tobytes())
    ga, gb = np.load(os.path.join(a, "grad.npy")), np.load(os.path.join(b, "grad.npy"))
    scale = float(np.abs(ga).max())
    rep["grad_max_abs_diff_ab"] = float(np.abs(ga - gb).max())
    rep["grad_max_rel_to_max_ab"] = rep["grad_max_abs_diff_ab"] / scale
    if a2:
        ga2 = np.load(os.path.join(a2, "grad.npy"))
        rep["grad_max_abs_diff_aa"] = float(np.abs(ga - ga2).max())
        rep["grad_max_rel_to_max_aa"] = rep["grad_max_abs_diff_aa"] / scale
    print(json.dumps(rep, indent=1))
    return rep


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs="+", metavar="DIR")
    a = ap.parse_args()
    if a.out:
        run(a.out)
    if a.compare:
        compare(*a.compare[:3])
