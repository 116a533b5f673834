"""Times SDFNetwork.sdf (value chain without a stash) on the wgmma engine, fused kernel vs layer-by-layer launches,
for the point counts of the placement passes and of a mesh grid, and reads the fused kernel's cycle counters
(AVC_CHAIN_DEBUG=1) at the placement passes' point counts.  Run on the GPU box: python tools/chain_probe.py"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from avatarclip_b200 import workload as WL  # noqa: E402


def main():
    sp, cp = WL.synth_states(WL.B2_SDF_KW, WL.B2_COL_KW, seed=0)
    sdf, col, var, ren = WL.build_networks(WL.B2_SDF_KW, WL.B2_COL_KW, WL.B2_REN_KW, sp, cp, 0.3, "cuda", engine=1, chunk=4096)
    out = {}
    for P in (8192, 32768, 1 << 20, 1 << 22):
        pts = (torch.rand(P, 3, device="cuda") - 0.5) * 2
        row = {}
        for mode in ("0", "1"):
            os.environ["AVC_FUSED_CHAIN"] = mode
            for _ in range(3):
                y = sdf.sdf(pts)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n = 10 if P <= 32768 else 3
            e0.record()
            for _ in range(n):
                y = sdf.sdf(pts)
            e1.record()
            torch.cuda.synchronize()
            row["fused_us" if mode == "1" else "layerwise_us"] = 1e3 * e0.elapsed_time(e1) / n
            row["checksum_" + mode] = float(y.double().sum())
        if P in (8192, 32768):       # stall picture of block 0 (cycle counters inside the kernel)
            import ctypes as C
            from avatarclip_b200 import _lib
            os.environ["AVC_FUSED_CHAIN"] = "1"
            os.environ["AVC_CHAIN_DEBUG"] = "1"
            sdf.sdf(pts)
            buf = (C.c_longlong * 8)()
            L = _lib.lib()
            L.avc_chain_debug_read.argtypes = [C.POINTER(C.c_longlong)]
            if L.avc_chain_debug_read(buf) == 0:
                n = max(1, buf[3])
                # consumer warpgroup 0 of block 0 per tile-layer: waits for its layer-0 input, for weight slabs, for
                # the MMA turn; MMAs (turn taken to accumulator ready, weight waits included); epilogue; loop total;
                # and the weight producer's waits for a free ring stage
                row["block0_cycles_per_tile_layer"] = {
                    "wait_A": buf[0] / n, "wait_W": buf[1] / n, "wait_turn": buf[4] / n, "mma": buf[6] / n,
                    "epi_work": buf[5] / n, "total": buf[2] / n, "producer_wait_free_stage": buf[7] / n,
                    "tile_layers": n, "epi_share": buf[5] / max(1, buf[2])}
            os.environ["AVC_CHAIN_DEBUG"] = "0"
        out[str(P)] = row
    print(json.dumps(out))


if __name__ == "__main__":
    main()
