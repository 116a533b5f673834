"""Stall probe of the wgmma NT tiles.

    python tools/nt_probe.py --build      # here (nvcc): avatarclip_b200/libavc_b200_probe.so = product objects, with
                                          # avc_neus.cu recompiled with -DAVC_NT_PROBE=1
    python tools/nt_probe.py --run OUT    # on the GPU: a few steps of the bench workload through the probe build,
                                          # per epilogue functor the share of its loop each warp role spent waiting

The probe adds a clock64 pair around every mbarrier wait of the three warp roles (TMA producer, MMA issuer, one epilogue
warp) and sums them per functor (avc_gemm_tc.cuh, AVC_NT_PROBE)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE_LIB = os.path.join(ROOT, "avatarclip_b200", "libavc_b200_probe.so")
NAMES = {1: "EpiValue", 2: "EpiChain", 3: "EpiChainBwd", 4: "EpiDgrad", 5: "EpiRelu", 6: "EpiDgradRelu", 7: "EpiColor0",
         8: "EpiStore", 9: "EpiBias", 10: "EpiGe", 0: "other"}


def build():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    g.build()
    obj_dir = os.path.join(ROOT, "build", "obj")
    probe_obj = os.path.join(ROOT, "build", "avc_neus_probe.o")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + g.NVCC_FLAGS + ["-DAVC_NT_PROBE=1", "-c", "-o", probe_obj,
                                                  os.path.join(ROOT, "avatarclip_b200", "csrc", "avc_neus.cu")], cwd=ROOT)
    objs = [os.path.join(obj_dir, f) for f in sorted(os.listdir(obj_dir)) if f.endswith(".o") and f != "avc_neus.o"]
    subprocess.check_call([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", PROBE_LIB, probe_obj] + objs,
                          cwd=ROOT)
    print("built", PROBE_LIB)


def run(out_path):
    os.environ["AVC_B200_LIB"] = PROBE_LIB
    sys.path.insert(0, ROOT)
    import torch
    from avatarclip_b200 import _lib, workload as WL
    from avatarclip_b200.clip_vit import ClipImageTower
    from avatarclip_b200.trainer import AppearanceTrainer, DeviceView
    dev = torch.device("cuda", 0)
    L = _lib.lib()
    L.avc_nt_probe_read.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    buf = (C.c_ulonglong * 128)()
    sp, cp = WL.synth_states(WL.B2_SDF_KW, WL.B2_COL_KW, seed=0)
    _, _, _, ren = WL.build_networks(WL.B2_SDF_KW, WL.B2_COL_KW, WL.B2_REN_KW, sp, cp, 0.3, dev, engine=1)
    tower = ClipImageTower(WL.random_vit_state(seed=0), device=dev)
    text = torch.randn(2, 512, generator=torch.Generator().manual_seed(5))
    tr = AppearanceTrainer(ren, tower, text, lr=5e-4, device=dev)
    view = DeviceView(WL.make_view(0, n_rays=512, H=224, W=224, seed=0, bg_choice=3), dev)
    for _ in range(3):
        tr.step(view)
    assert L.avc_nt_probe_read(buf, 1) == 0, "not a probe build"
    steps = 5
    for _ in range(steps):
        tr.step(view)
    assert L.avc_nt_probe_read(buf, 1) == 0
    rep = {}
    for i in range(16):
        v = [buf[i * 8 + j] for j in range(8)]
        if v[7] == 0:
            continue
        ctas = v[7]
        rep[NAMES.get(i, str(i))] = {
            "ctas_per_step": ctas / steps,
            # producer warp; consumer warpgroup 0 (its MMAs and epilogues)
            "loop_kcycles_per_cta": {"tma": v[1] / ctas / 1e3, "consumer": v[4] / ctas / 1e3},
            "tma_waits_free_stage": v[0] / max(v[1], 1),
            "consumer_waits_operands": v[3] / max(v[4], 1),
        }
    with open(out_path, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--build", action="store_true")
    ap.add_argument("--run", metavar="OUT")
    a = ap.parse_args()
    if a.build:
        build()
    if a.run:
        run(a.run)
