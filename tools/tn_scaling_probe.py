"""Duration of the wgmma weight-gradient (TN) tile kernel against the reduction length P (N1 = N2 = 256, split operands):
the slope is the streaming cost, the intercept the fixed cost of a launch (set-up, first loads, atomics flush, tail).
The same fit for the other shapes a training step runs (256 x 39: the first SDF linear, BN = 64; 217 x 256: the skip
layer's input), and with --step the duration of every TN launch of one render forward + backward of the bench workload.
    python tools/tn_scaling_probe.py OUT.json [--step]        # on an H100 (AVC_B200_LIB selects another build)"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = ((256, 256), (256, 39), (217, 256))


def _fit(rows):
    """least squares us = a + b * P over the four largest sizes"""
    xs = [r["P"] for r in rows[-4:]]
    ys = [r["us"] for r in rows[-4:]]
    n = len(xs)
    mx, my = sum(xs) / n, sum(ys) / n
    b = sum((x - mx) * (y - my) for x, y in zip(xs, ys)) / sum((x - mx) ** 2 for x in xs)
    return my - b * mx, b


def step_launches():
    """Device durations (us) of the TN launches of one render forward + backward of the bench view, in launch order,
    with plain launches (under programmatic dependent launch a record includes the wait for the predecessor)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from avatarclip_b200 import _lib, workload as WL
    from avatarclip_b200.renderer import render_backward_raw, render_forward_raw
    from avatarclip_b200.trainer import DeviceView
    os.environ["AVC_TC_PDL"] = "0"
    dev = torch.device("cuda", 0)
    sp, cp = WL.synth_states(WL.B2_SDF_KW, WL.B2_COL_KW, seed=0)
    _, _, _, ren = WL.build_networks(WL.B2_SDF_KW, WL.B2_COL_KW, WL.B2_REN_KW, sp, cp, 0.3, dev, engine=1)
    ren._ensure_flat(dev)
    dv = DeviceView(WL.make_view(0, n_rays=512, H=224, W=224, seed=0, bg_choice=3), dev)
    jit = dv.jitter if ren.perturb > 0 else None

    def once():
        out, ws, chunk = render_forward_raw(ren, dv.rays_o, dv.rays_d, dv.near, dv.far, jit, None, 0, 1.0, None,
                                            keep_ws=True)
        cot = {k: torch.ones_like(out[k]) for k in _lib._COT_FIELDS}
        render_backward_raw(ren, dv.rays_o, dv.rays_d, None, 0, 1.0, out, ws, chunk, cot)

    for _ in range(3):
        once()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        once()
        torch.cuda.synchronize()
    os.environ.pop("AVC_TC_PDL")
    evs = sorted((e for e in prof.events() if e.name and "gemm_tc_tn_kernel" in e.name), key=lambda e: e.time_range.start)
    us = [round(e.device_time, 1) for e in evs]
    return {"kernels": sorted({e.name for e in evs}), "us": us, "launches": len(us), "total_us": round(sum(us), 1)}


def main(out_path, step=False):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from avatarclip_b200 import _lib
    L = _lib.lib()
    L.avc_tc_gemm_tn_test.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    dev = torch.device("cuda", 0)
    rep = {"device": torch.cuda.get_device_name(0), "lib": _lib.LIB_PATH}
    r8 = lambda n: (n + 7) // 8 * 8

    def time_tn(P, N1, N2, nprod):
        A = torch.randn(P, N1, device=dev)
        B = torch.randn(P, N2, device=dev)
        Cm = torch.zeros(N1, N2, device=dev)
        cs = torch.zeros(N1, device=dev)
        ws = torch.empty(4 * P * (r8(N1) + r8(N2)) + 4096, dtype=torch.uint8, device=dev)
        call = lambda: _lib.check(L.avc_tc_gemm_tn_test(A.data_ptr(), B.data_ptr(), P, N1, N2, nprod, Cm.data_ptr(),
                                                        cs.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "tn")
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(7):
                call()
            torch.cuda.synchronize()
        us = [e.device_time for e in prof.events() if e.name and "gemm_tc_tn_kernel" in e.name]
        return sorted(us)[len(us) // 2]

    for nprod in (3, 1):
        for N1, N2 in SHAPES:
            rows = []
            for P in (8192, 16384, 32768, 65536, 131072, 262144):
                us = time_tn(P, N1, N2, nprod)
                rows.append({"P": P, "us": us, "operand_MB": P * (N1 + N2) * 2 * (2 if nprod == 3 else 1) / 1e6})
            a, b = _fit(rows)
            mb65 = 65536 * (r8(N1) + r8(N2)) * 2 * (2 if nprod == 3 else 1) / 1e6
            rep["products_%d_%dx%d" % (nprod, N1, N2)] = {
                "runs": rows, "us_at_65536": next(r["us"] for r in rows if r["P"] == 65536), "fixed_us": a,
                "us_per_65536_rows": b * 65536, "streaming_TBps": mb65 / (b * 65536)}
    if step:
        rep["step_tn_launches"] = step_launches()
    with open(out_path, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main(sys.argv[1], step="--step" in sys.argv[2:])
