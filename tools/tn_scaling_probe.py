"""Duration of the wgmma weight-gradient (TN) tile kernel against the reduction length P (N1 = N2 = 256, split operands):
the slope is the streaming cost, the intercept the fixed cost of a launch (set-up, first loads, atomics flush, tail).
    python tools/tn_scaling_probe.py OUT.json        # on an H100"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main(out_path):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from avatarclip_b200 import _lib
    L = _lib.lib()
    L.avc_tc_gemm_tn_test.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    dev = torch.device("cuda", 0)
    rep = {}
    for nprod in (3, 1):
        rows = []
        for P in (8192, 16384, 32768, 65536, 131072, 262144):
            A = torch.randn(P, 256, device=dev)
            B = torch.randn(P, 256, device=dev)
            Cm = torch.zeros(256, 256, device=dev)
            ws = torch.empty(4 * P * 512 + 4096, dtype=torch.uint8, device=dev)
            call = lambda: _lib.check(L.avc_tc_gemm_tn_test(A.data_ptr(), B.data_ptr(), P, 256, 256, nprod, Cm.data_ptr(), None,
                                                            ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "tn")
            for _ in range(3):
                call()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    call()
                torch.cuda.synchronize()
            us = [e.device_time for e in prof.events() if e.name and "gemm_tc_tn_kernel" in e.name]
            rows.append({"P": P, "us": sorted(us)[len(us) // 2], "operand_MB": P * 256 * 2 * 2 * (2 if nprod == 3 else 1) / 1e6})
        # least squares us = a + b * P over the four largest sizes
        xs = [r["P"] for r in rows[2:]]
        ys = [r["us"] for r in rows[2:]]
        n = len(xs)
        mx, my = sum(xs) / n, sum(ys) / n
        b = sum((x - mx) * (y - my) for x, y in zip(xs, ys)) / sum((x - mx) ** 2 for x in xs)
        a = my - b * mx
        rep["products_%d" % nprod] = {"runs": rows, "fixed_us": a, "us_per_65536_rows": b * 65536,
                                      "streaming_TBps": (65536 * 256 * 2 * 2 * (2 if nprod == 3 else 1) / 1e6) / (b * 65536)}
    with open(out_path, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main(sys.argv[1])
