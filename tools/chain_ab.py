"""A-B check of a change to the fused SDF value-chain kernel (csrc/avc_chain.cu): the sample placement of the bench
workload's render (512 rays, 64 coarse samples, 4 up-sampling rounds of 16 on bench.py's 8 x 256 network) restated
kernel by kernel through avc_neus_kernel_test -- coarse depths (kind 6), encoding (13), the fused chain (27),
k_upsample (7), k_merge (8) -- through a given build of the library.  Saves the sdf of each of the four placement passes
and the depths and sdf after every k_merge as .npy.

    AVC_B200_LIB=/path/to/libavc_b200.so python tools/chain_ab.py --out DIR      # on the GPU, once per build
    python tools/chain_ab.py --compare DIR_A DIR_B                                 # anywhere

    python tools/chain_ab.py --compare-dumps DIR_A DIR_B [DIR_A2]                  # two bench.py --dump-outputs DIRs

--compare reports per array whether A and B are bitwise equal.  --compare-dumps does the same for the outputs of
bench.py --dump-outputs (take them with --steps 1 --warmup 0: later steps start from weights that Adam moved by a
gradient with run-to-run noise) and reports the largest difference of the flat gradient, with a second run of A (DIR_A2) also
between A and A2: the TN tiles' split-K reductions accumulate with red.global.add, so two runs of one build differ in
the last bits of the gradient."""
import argparse
import glob
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R, N0, PER, STEPS = 512, 64, 16, 4


def run(out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import test_neus_chain_kernels_gpu as K
    import test_neus_value_chain_gpu as V
    from avatarclip_b200 import _lib
    net = V.ChainNet(V.CONFIGS["b2"], seed=0)          # bench.py's network: 8 x 256, the skip concat into linear 4
    S = N0 + PER * STEPS
    g = torch.Generator().manual_seed(3)
    d = torch.tensor([0.0, 0.0, -1.0]) + 0.3 * torch.randn(R, 3, generator=g)
    d = (d / d.norm(dim=-1, keepdim=True)).cuda()
    o = (torch.tensor([0.0, 0.0, 1.8]) + 0.05 * torch.randn(R, 3, generator=g)).cuda()
    near = torch.full((R,), 0.8, device="cuda")
    far = torch.full((R,), 2.8, device="cuda")
    jit = (torch.rand(R, generator=g) - 0.5).cuda()

    def encode(z, nz, pitch):
        E, EP = net.E, net.EP
        p0 = K._pair(R * nz, EP)
        ps, dims_s = None, ([0] * 4, [0] * 4)
        if net.ls is not None:
            lk = net.lin[net.ls]
            ps = K._pair(R * nz, lk["Kp"])
            dims_s = ([lk["Kp"], 0, 0, 0], [lk["K"] - E, 0, 0, 0])
        dims = [net.mr, EP, 0 if ps is None else 1] + dims_s[0] + dims_s[1] + [nz, pitch, R]
        K._run(13, dims, [net.scale], [o, d, z], [None] * 5 + [p0, ps, None, None, None])
        return p0, ps

    def chain(z, nz, pitch, out_nz, out_pitch):
        p0, ps = encode(z, nz, pitch)
        sdf = torch.zeros(R, out_pitch, device="cuda")
        K._run(27, [R * nz, out_nz, out_pitch], [], [net.cfg, net.pack, net.pk_pair, p0, ps], [sdf])
        return sdf

    arrays = {}
    zc = torch.zeros(R, S, device="cuda")
    K._run(6, [N0, S, R], [], [near, far, jit], [zc])
    sc = chain(zc, N0, S, N0, S)                          # coarse pass: sdf written at (p / 64) * S + p % 64
    arrays["sdf_pass0"] = sc[:, :N0]
    n = N0
    for i in range(STEPS):
        last = i + 1 == STEPS
        newz = torch.zeros(R, PER, device="cuda")
        K._run(7, [n, S, R, PER], [64.0 * (1 << i)], [o, d, zc, sc], [newz])
        news = None
        if not last:
            news = chain(newz, PER, PER, 0, PER)          # up-sampling pass: dense [R][PER]
            arrays[f"sdf_pass{i + 1}"] = news
        zo, so = torch.zeros(R, S, device="cuda"), torch.zeros(R, S, device="cuda")
        K._run(8, [n, S, R, PER, S], [], [zc, sc, newz, news], [zo, so])
        n += PER
        arrays[f"z_merge{i}"] = zo[:, :n]
        if not last:
            arrays[f"sdf_merge{i}"] = so[:, :n]
        zc, sc = zo, so
    torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    for k, v in arrays.items():
        np.save(os.path.join(out_dir, k + ".npy"), v.detach().cpu().numpy())
    print("wrote", out_dir, "lib", _lib.LIB_PATH, "arrays", sorted(arrays))


def compare(a, b):
    rep = {}
    for f in sorted(glob.glob(os.path.join(a, "*.npy"))):
        k = os.path.basename(f)[:-4]
        x, y = np.load(f), np.load(os.path.join(b, os.path.basename(f)))
        rep[k] = bool(x.shape == y.shape and x.tobytes() == y.tobytes())
    rep["all_bitwise_equal"] = all(rep.values())
    print(json.dumps(rep, indent=1))
    return rep


def compare_dumps(a, b, a2=None):
    rep = {"bitwise_equal_ab": {}, "bitwise_equal_aa": {}}
    for k in ("color_fine", "extra_color_fine", "weight_sum", "loss", "clip_cos"):
        x, y = np.load(os.path.join(a, k + ".npy")), np.load(os.path.join(b, k + ".npy"))
        rep["bitwise_equal_ab"][k] = bool(x.tobytes() == y.tobytes())
        if a2:
            rep["bitwise_equal_aa"][k] = bool(x.tobytes() == np.load(os.path.join(a2, k + ".npy")).tobytes())
    ga, gb = np.load(os.path.join(a, "grad.npy")), np.load(os.path.join(b, "grad.npy"))
    scale = float(np.abs(ga).max())
    rep["grad_max_rel_to_max_ab"] = float(np.abs(ga - gb).max()) / scale
    if a2:
        rep["grad_max_rel_to_max_aa"] = float(np.abs(ga - np.load(os.path.join(a2, "grad.npy"))).max()) / scale
    print(json.dumps(rep, indent=1))
    return rep


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2, metavar="DIR")
    ap.add_argument("--compare-dumps", nargs="+", metavar="DIR")
    args = ap.parse_args()
    if args.out:
        run(args.out)
    if args.compare:
        compare(*args.compare)
    if args.compare_dumps:
        compare_dumps(*args.compare_dumps[:3])
