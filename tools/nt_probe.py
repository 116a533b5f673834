"""Stall probe of the wgmma NT tiles.

    python tools/nt_probe.py --build      # here (nvcc): avatarclip_b200/libavc_b200_probe.so = product objects, with
                                          # avc_neus.cu recompiled with -DAVC_NT_PROBE=1
    python tools/nt_probe.py --run OUT    # on the GPU: a few steps of the bench workload through the probe build,
                                          # per epilogue functor where each warp role's loop time went
    python tools/nt_probe.py --run OUT --lib OTHER.so --slots 9    # another probe build (9 slots: before the
                                          # store-drain slot existed, 8: before the epilogue-ring slot)

The probe takes clock64 stamps in the TMA producer and in the leading thread of each consumer warpgroup: the producer's
waits for a free stage, the consumers' waits for operands and for their turn at the tensor pipe, and the time from a
consumer's turn to its MMAs' completion and from there to the end of its epilogue, summed per functor
(avc_gemm_tc.cuh, AVC_NT_PROBE), and the consumers' waits for the epilogue operands staged in shared memory
(`waits_staged`, functors with a `Stage`), and their waits for the TMA stores of a ring slot to have read it before they
rewrite it (`waits_store_drain`, functors with an `Out`).  `busy_over_wall` is the MMA and epilogue time of both
consumer warpgroups over the loop time of one: above 1, the two worked at the same time (one's MMAs under the other's
epilogue)."""
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


def run(out_path, lib=PROBE_LIB, slots=10):
    os.environ["AVC_B200_LIB"] = lib
    sys.path.insert(0, ROOT)
    import torch
    from avatarclip_b200 import _lib, workload as WL
    from avatarclip_b200.clip_vit import ClipImageTower
    from avatarclip_b200.trainer import AppearanceTrainer, DeviceView
    dev = torch.device("cuda", 0)
    L = _lib.lib()
    L.avc_nt_probe_read.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    buf = (C.c_ulonglong * (16 * slots))()
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
        v = [buf[i * slots + j] for j in range(slots)] + [0] * (10 - slots)
        if v[7] == 0:
            continue
        ctas = v[7]
        cons = max(v[6], 1)      # loop cycles of both consumer warpgroups
        rep[NAMES.get(i, str(i))] = {
            "ctas_per_step": ctas / steps,
            "loop_kcycles_per_cta": {"producer": v[1] / ctas / 1e3, "consumer": v[6] / (2 * ctas) / 1e3},
            "producer_waits_free_stage": v[0] / max(v[1], 1),
            # shares of a consumer warpgroup's loop; the MMA share includes its operand and B-panel waits
            "consumer": {"waits_operands": v[2] / cons, "waits_turn": v[3] / cons, "mma": v[4] / cons,
                         "epilogue": v[5] / cons, "waits_staged": v[8] / cons, "waits_store_drain": v[9] / cons},
            "busy_over_wall": (v[4] + v[5]) / (cons / 2),
        }
    with open(out_path, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--build", action="store_true")
    ap.add_argument("--run", metavar="OUT")
    ap.add_argument("--lib", default=PROBE_LIB, help="probe build to load (default: the one --build makes)")
    ap.add_argument("--slots", type=int, default=10, help="counters per functor of that build")
    a = ap.parse_args()
    if a.build:
        build()
    if a.run:
        run(a.run, a.lib, a.slots)
