"""The fused SDF value-chain kernel (k_sdf_chain, csrc/avc_chain.cu) on its own inputs against its float64 restatement
(oracle/neus_kernels.py::value_chain, pinned against oracle.neus.sdf_value by test_neus_kernels_cpu.py), through kind 27
of avc_neus_kernel_test: value_chain_fused as the render calls it, on the packed weights kind 10 writes and the encoded
pairs kind 12 writes, so the chain sees exactly what a render gives it.

Conventions as in test_neus_chain_kernels_gpu.py:
- Every output buffer has a NaN-patterned guard that must keep its bits; the gap columns [nz, pitch) of a strided
  output keep their NaN bits.
- Inputs the kernel must not read are NaN: the padding columns [K, Kp) of the in0 pair, every column of the skip pair
  outside [skip_col0, skip_col0 + E), and everything in the packed buffer and its pair but the hidden linears' weights
  and biases and the sdf row.
- The reference is the fp64 chain on the kernel's own inputs: W = hi + lo of the packed pair, the fp32 biases, the
  layer-0 input and the skip columns as hi + lo of their pairs.  The bar is max(4 x the error of the fp32 twin that
  splits every stored activation as the kernel's epilogue does, a floor), relative to the largest reference entry.
- The small point counts are prefixes of a configuration's 128 x SMs + 1-point sample, judged on the sample's scale and
  bar (the twin's error on one point is a single draw), and must give the sample run's bits."""
import ctypes as C

import pytest
import torch

import test_neus_chain_kernels_gpu as K
import util_neus as U
from oracle import neus
from oracle import neus_kernels as nk

pytestmark = pytest.mark.gpu

F64 = torch.float64
AVC_E_BADCFG = -1
# the bar's floor binds where the twin splits nothing (one hidden linear: the twin's error 2.4e-7, the kernel's 1.5e-6 on
# an H100 80GB HBM3 at 700 W; everywhere else the kernel measured 1.5-2.6 x the twin's error)
FLOOR = 5e-6
SDF_BAR = 5e-5          # the public sdf query against the fp32 network (test_neus_gpu.py)
BENCH_RAYS = 12544      # rays of bench.py's training step
KIND = 27


# --------------------------------------------------------------------------- configurations
def _kw(H, L, skip, mr, scale):
    d_out = 257 if H == 256 else 9
    sdf_kw = dict(d_in=3, d_out=d_out, d_hidden=H, n_layers=L, skip_in=list(skip), multires=mr, bias=0.5, scale=scale,
                  geometric_init=True, weight_norm=True)
    col_kw = dict(d_feature=d_out - 1, mode="no_view_dir", d_in=6, d_out=3, d_hidden=64, n_layers=1, weight_norm=True,
                  multires_view=0, squeeze_out=True, extra_color=True)
    ren_kw = dict(n_samples=16, n_importance=16, n_outside=0, up_sample_steps=4, perturb=1.0, extra_color=True)
    return sdf_kw, col_kw, ren_kw


# name: (sdf_kw, col_kw, ren_kw, gain of the hidden weights)
CONFIGS = {
    "shipped": U.CASES["shipped"][:3] + (1.0,),     # 256 x 4, the skip concat at the head
    "b2": U.CASES["b2"][:3] + (1.0,),               # 256 x 8, skip inside (linear 3 is 217 wide): bench.py's network
    "l1": _kw(128, 1, (), 6, 1.0) + (1.0,),         # one hidden linear: its epilogue is the head's
    "l10": _kw(64, 10, (1,), 6, 1.0) + (1.0,),      # kMaxHidden linears; skip right after linear 0 (25 wide)
    "w80": _kw(80, 4, (3,), 4, 1.0) + (1.0,),       # partial last k-block (80 = 64 + 16), E = 27, linear 2 53 wide
    "w136": _kw(136, 3, (), 6, 1.0) + (1.0,),       # partial last k-block, no skip
    "w200": _kw(200, 3, (2,), 10, 1.0) + (1.0,),    # E = 63, linear 1 137 wide, partial k-blocks
    "col1": _kw(64, 3, (2,), 10, 1.0) + (1.0,),     # linear 1 is one column wide (64 - 63)
    "w16": _kw(16, 3, (2,), 0, 1.0) + (1.0,),       # multires 0 (E = 3), linear 1 13 wide
    "hot": _kw(128, 4, (2,), 6, 2.5) + (4.0,),      # scale 2.5, weights x 4: both softplus branches (|beta z| > 20)
}
# refused by chain::supported (or by value_chain_fused): the layer-by-layer launches run them
REFUSED = {
    "L11": _kw(64, 11, (4,), 6, 1.0) + (1.0,),
    "w264": _kw(264, 3, (2,), 6, 1.0) + (1.0,),
    "skip2x": _kw(64, 5, (2, 4), 6, 1.0) + (1.0,),
}
ACCEPTED_EDGES = {
    "L10": CONFIGS["l10"],
    "w256": _kw(256, 3, (), 6, 1.0) + (1.0,),
}

HEAD = K.HEAD
LIN = K.LIN


def _rc(kind, dims, ins, outs):
    """avc_neus_kernel_test's return code (no check)."""
    _lib, f = K._fn()
    d = (C.c_int64 * len(dims))(*dims)
    fsc = (C.c_float * 1)(0.0)
    pi = (C.c_void_p * len(ins))(*[K._addr(t) for t in ins])
    po = (C.c_void_p * len(outs))(*[K._addr(t) for t in outs])
    rc = f(kind, d, fsc, pi, po, _lib.stream_ptr())
    torch.cuda.synchronize()
    return rc


class ChainNet:
    """A configuration on the wgmma engine: the product modules, its plan's layout (kind 9), the packed weights and their
    pair (kind 10) with every float the chain must not read set to NaN, and the kernel's weights as the reference
    takes them."""

    def __init__(self, spec, seed=5):
        sdf_kw, col_kw, ren_kw, gain = spec
        self.sconf, _, _ = U.confs_from_kw(sdf_kw, col_kw, ren_kw)
        sp, cp = U.synth_state(sdf_kw, col_kw, seed)
        g = torch.Generator().manual_seed(seed + 100)
        for l in range(sdf_kw["n_layers"]):      # non-zero biases (the geometric init leaves them 0), the gain
            b = sp[f"lin{l}.bias"]
            sp[f"lin{l}.bias"] = b + 0.05 * torch.randn(b.shape, generator=g)
            sp[f"lin{l}.weight_g"] = sp[f"lin{l}.weight_g"] * gain
        self.sp = sp
        self.sdf, _, _, self.ren = U.build_product(sdf_kw, col_kw, ren_kw, sp, cp, 0.3, "cuda", engine=1)
        self.cfg = self.ren.cfg
        self.flat = self.ren.flat_params(torch.device("cuda", torch.cuda.current_device())).flat
        self.scale, self.mr = float(sdf_kw["scale"]), int(sdf_kw["multires"])
        buf = (C.c_int64 * (16 + 11 * 40))(*([-7] * (16 + 11 * 40)))
        K._run(9, [], [], [self.cfg], [buf])
        lay = dict(zip(HEAD, buf[:16]))
        self.__dict__.update(lay)
        self.lin = [dict(zip(LIN, buf[16 + 11 * i:27 + 11 * i])) for i in range(self.L + 1)]
        skips = [l for l in range(1, self.L + 1) if self.lin[l]["skip"]]
        self.ls = skips[0] if skips else None
        pf = self.pack_floats
        pk = K.Out((pf,))
        pair = torch.full((2 * pf,), float("nan"), dtype=torch.bfloat16, device="cuda")
        K._run(10, [], [], [self.cfg, self.flat], [pk.t, pair])
        assert pk.intact()
        pack = pk.t
        keep = torch.zeros(pf, dtype=torch.bool, device="cuda")         # what the chain reads of the fp32 pack
        keepw = torch.zeros(pf, dtype=torch.bool, device="cuda")        # ... and of the pair
        self.W, self.b = [], []
        hi, lo = pair[:pf], pair[pf:]
        for l in range(self.L):
            d = self.lin[l]
            N, Kk, Kp = d["N"], d["K"], d["Kp"]
            blk = slice(d["pk_W"], d["pk_W"] + N * Kp)
            keepw[blk].view(N, Kp)[:, :Kk] = True
            self.W.append(hi[blk].view(N, Kp)[:, :Kk].double() + lo[blk].view(N, Kp)[:, :Kk].double())
            keep[d["pk_b"]:d["pk_b"] + N] = True
            self.b.append(pack[d["pk_b"]:d["pk_b"] + N].clone())
        KL = self.lin[self.L]["K"]
        keep[self.pk_wsdf:self.pk_wsdf + KL] = True
        keep[self.pk_bsdf] = True
        self.w_sdf = pack[self.pk_wsdf:self.pk_wsdf + KL].clone()
        self.b_sdf = pack[self.pk_bsdf:self.pk_bsdf + 1].clone()
        pack[~keep] = float("nan")
        pair[:pf][~keepw] = float("nan")
        pair[pf:][~keepw] = float("nan")
        self.pack, self.pk_pair = pack, pair

    def encode(self, pts):
        """kind 12 as the render's wgmma targets: the in0 pair and the skip linear's pair; then NaN in every column the
        chain must not read.  Returns (in0 pair, skip pair or None)."""
        P = pts.shape[0]
        E, EP = self.E, self.EP
        p0 = K._pair(P, EP)
        ps, dims_s = None, ([0] * 4, [0] * 4)
        if self.ls is not None:
            d = self.lin[self.ls]
            ps = K._pair(P, d["Kp"])
            dims_s = ([d["Kp"], 0, 0, 0], [d["K"] - E, 0, 0, 0])
        dims = [self.mr, EP, 0 if ps is None else 1] + dims_s[0] + dims_s[1] + [P]
        K._run(12, dims, [self.scale], [pts], [None] * 5 + [p0, ps, None, None, None])
        p0[:, E:EP] = float("nan")
        p0[:, EP + E:] = float("nan")
        if ps is not None:
            Kp, c0 = self.lin[self.ls]["Kp"], self.lin[self.ls]["K"] - E
            for h in (0, Kp):
                ps[:, h:h + c0] = float("nan")
                ps[:, h + c0 + E:h + Kp] = float("nan")
        return p0, ps

    def run(self, p0, ps, P, nz=0, pitch=0, out=None):
        """kind 27 on the first P rows of the pairs -> the Out it wrote (NaN-patterned, guarded)."""
        if out is None:
            out = K.Out((P // nz, pitch) if nz else (P,))
        K._run(KIND, [P, nz, pitch], [], [self.cfg, self.pack, self.pk_pair, p0, ps], [out.t])
        return out

    def reference(self, p0, ps, P, dtype=F64, split_acts=False, pre=None):
        """value_chain on the kernel's own inputs, on the device of the pairs."""
        E, EP = self.E, self.EP
        x0 = p0[:P, :E].double() + p0[:P, EP:EP + E].double()
        skip = None
        if ps is not None:
            Kp, c0 = self.lin[self.ls]["Kp"], self.lin[self.ls]["K"] - E
            skip = ps[:P, c0:c0 + E].double() + ps[:P, Kp + c0:Kp + c0 + E].double()
            skip = skip.to(dtype)
        return nk.value_chain(x0.to(dtype), skip, self.W, self.b, self.w_sdf, self.b_sdf, self.ls, self.scale,
                              dtype=dtype, split_acts=split_acts, pre=pre)

    def check(self, label, got, p0, ps, P):
        ref = self.reference(p0, ps, P)
        twin = self.reference(p0, ps, P, dtype=torch.float32, split_acts=True)
        e, b = K._rel(got, ref), K._bar(ref, twin, FLOOR)
        print(f"[worst] value_chain {label} P {P} err {e:.2e} bar {b:.1e} (twin {K._rel(twin, ref):.2e})")
        assert e <= b, (label, P, e, b)


_NETS = {}


def _net(name):
    if name not in _NETS:
        spec = CONFIGS.get(name) or REFUSED.get(name) or ACCEPTED_EDGES[name]
        _NETS[name] = ChainNet(spec)
    return _NETS[name]


def _points(P, seed):
    return ((torch.rand(P, 3, generator=torch.Generator().manual_seed(seed)) - 0.5) * 2).cuda()


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _bits(t):
    return t.contiguous().view(torch.int32)


# --------------------------------------------------------------------------- every configuration, every tile edge
_SAMPLES = {}


def _sample(name):
    """The configuration's sample: 128 x SMs + 1 encoded points (one tile per CTA, and a second trip of the persistent
    loop on CTA 0), the kernel's output on all of them, the fp64 reference, its pre-activations and the bar."""
    if name not in _SAMPLES:
        net = _net(name)
        P = 128 * _sms() + 1
        p0, ps = net.encode(_points(P, 1))
        out = net.run(p0, ps, P)
        assert out.intact()
        pre = []
        ref = net.reference(p0, ps, P, pre=pre)
        twin = net.reference(p0, ps, P, dtype=torch.float32, split_acts=True)
        print(f"[sample] value_chain {name} P {P} twin {K._rel(twin, ref):.2e}")
        _SAMPLES[name] = (net, p0, ps, out.t, ref, K._bar(ref, twin, FLOOR), pre)
    return _SAMPLES[name]


PS = [1, 64, 65, 127, 128, 129, "sms", "sms+1"]


@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("name", list(CONFIGS))
def test_value_chain(name, P):
    """The first P points of the configuration's sample, on the same buffers: one partial tile (1, 64, 65, 127 points:
    one or both warpgroups, the rows >= P zero-filled by TMA and their skip columns zero), exactly one tile, one tile and
    one row, one tile per SM with and without one more.  Each meets the sample's bar, relative to the sample's largest
    reference entry (one point's sdf alone can be near 0), and gives the bits of the whole sample's run: a row's result
    does not depend on how many rows the launch has."""
    net, p0, ps, full, ref, bar, pre = _sample(name)
    Pf = full.shape[0]
    P = {"sms": Pf - 1, "sms+1": Pf}.get(P, P)
    got = full
    if P < Pf:
        out = net.run(p0, ps, P)
        assert out.intact()
        got = out.t
    e = (got.double() - ref[:P]).abs().max().item() / ref.abs().max().item()
    print(f"[worst] value_chain {name} P {P} err {e:.2e} bar {bar:.1e}")
    assert e <= bar, (name, P, e, bar)
    assert torch.equal(_bits(got), _bits(full[:P]))
    if name == "hot":
        bz = torch.cat([100.0 * z.reshape(-1) for z in pre])
        assert bool((bz > 20).any()) and bool((bz < -20).any()), "both softplus branches"


# --------------------------------------------------------------------------- the benchmark step's placement passes
_BIG = {}


def _big(name, P):
    """Encoded pairs of P points (cached: the 400 k-point inputs are shared by the tests below)."""
    key = (name, P)
    if key not in _BIG:
        net = _net(name)
        pts = _points(P, 7)
        if P >= 1037:       # rows 37..1036 are the 1 000 points test_position_independent evaluates alone
            pts[37:1037] = _points(1000, 11)
        _BIG[key] = net.encode(pts)
    return _BIG[key]


def test_coarse_pass_strided_and_stable():
    """bench.py's coarse pass: 12 544 rays x 32 samples on its network, the sdf written at (p / 32) * 64 + p % 32 --
    3 136 tiles, about 24 per CTA, so the W ring, the afree / a0full parities and the tile counter wrap many times.  The
    strided output is the dense output scattered, bit for bit; the gap columns keep their NaN bits; a second call gives
    the same bits; the dense output meets the bar against the fp64 chain (computed on the device).  Measured on an H100
    80GB HBM3 at 700 W: 8.7e-6 against a bar of 1.5e-5."""
    name, nz, pitch = "b2", 32, 64
    P = BENCH_RAYS * nz
    net = _net(name)
    p0, ps = _big(name, P)
    st = net.run(p0, ps, P, nz, pitch)
    assert st.intact()
    assert K._untouched(st.t[:, nz:])
    dense = net.run(p0, ps, P)
    assert dense.intact()
    assert torch.equal(_bits(st.t[:, :nz]).reshape(-1), _bits(dense.t))
    again = net.run(p0, ps, P)
    assert torch.equal(_bits(again.t), _bits(dense.t))
    net.check(f"{name} coarse", dense.t, p0, ps, P)


@pytest.mark.parametrize("name", ["b2", "shipped"])
def test_upsample_pass(name):
    """An up-sampling pass of the benchmark step: 12 544 rays x 8 new samples, dense.  Measured (H100 80GB HBM3, 700 W):
    b2 8.0e-6 against 1.4e-5, shipped 6.7e-6 against 1.6e-5."""
    P = BENCH_RAYS * 8
    net = _net(name)
    p0, ps = _big(name, P)
    out = net.run(p0, ps, P)
    assert out.intact()
    net.check(f"{name} upsample", out.t, p0, ps, P)


def test_position_independent():
    """The first 1 000 points give the same bits evaluated alone (8 tiles, one per CTA) and as rows 37.. of the coarse
    pass's 401 408 points (every row in another tile, warpgroup and CTA, about 24 tiles per CTA): each row's MMAs, its
    epilogue and the head's butterfly do not depend on where the row sits (DESIGN.md §3.1: placement is discontinuous
    in the sdf)."""
    name = "b2"
    net = _net(name)
    P = BENCH_RAYS * 32
    p0, ps = _big(name, P)
    big = net.run(p0, ps, P)
    q0, qs = net.encode(_points(1000, 11))
    assert torch.equal(q0.view(torch.int16), p0[37:1037].view(torch.int16))
    alone = net.run(q0, qs, 1000)
    assert alone.intact()
    assert torch.equal(_bits(alone.t), _bits(big.t[37:1037]))


def test_map_cache():
    """The TMA maps are cached by pointer and shape: on the same buffers P = 77, then 5 000, then 77 again each match
    their own reference, and the 77-point runs leave rows >= 77 of the output untouched."""
    net = _net("shipped")
    p0, ps = net.encode(_points(5000, 3))
    out = K.Out((5000,))
    for P in (77, 5000, 77):
        out.t.view(torch.int32).fill_(K.NANBITS)
        net.run(p0, ps, P, out=out)
        assert out.intact()
        if P < 5000:
            assert K._untouched(out.t[P:])
        net.check("shipped map cache", out.t[:P], p0, ps, P)


# --------------------------------------------------------------------------- where the fused kernel stops
@pytest.mark.parametrize("name,fused", [("L11", False), ("w264", False), ("skip2x", False), ("L10", True),
                                        ("w256", True)])
def test_supported_edges(name, fused):
    """kind 27 refuses 11 hidden linears, a 264-wide layer and two skip linears with AVC_E_BADCFG (and writes
    nothing), and runs 10 hidden linears and 256-wide layers.  The public sdf query still matches the fp32 network on
    the refused shapes: the layer-by-layer launches run them."""
    net = _net(name)
    P = 1001
    pts = _points(P, 13)
    p0, ps = net.encode(pts)
    out = K.Out((P,))
    rc = _rc(KIND, [P, 0, 0], [net.cfg, net.pack, net.pk_pair, p0, ps], [out.t])
    if fused:
        assert rc == 0 and out.intact()
        net.check(name, out.t, p0, ps, P)
    else:
        assert rc == AVC_E_BADCFG, rc
        assert K._untouched(out.full)
        got = net.sdf.sdf(pts).cpu()
        want = neus.sdf_value(net.sp, net.sconf, pts.cpu())
        e = U.rel_to_max(got, want)
        print(f"[worst] sdf query {name} (layer by layer) err {e:.2e} bar {SDF_BAR:.0e}")
        assert e < SDF_BAR, e


@pytest.mark.parametrize("name", list(CONFIGS))
def test_sdf_query_both_paths(name, monkeypatch):
    """The public sdf query on engine 1 with AVC_FUSED_CHAIN=0 (the layer-by-layer launches every refused configuration
    runs) and with it unset (the fused kernel) meets the 5e-5 bar against the fp32 network at every accepted shape."""
    net = _net(name)
    P = 4099
    pts = _points(P, 17)
    want = neus.sdf_value(net.sp, net.sconf, pts.cpu())
    for env in ("0", None):
        if env is None:
            monkeypatch.delenv("AVC_FUSED_CHAIN", raising=False)
        else:
            monkeypatch.setenv("AVC_FUSED_CHAIN", env)
        e = U.rel_to_max(net.sdf.sdf(pts).cpu(), want)
        print(f"[worst] sdf query {name} AVC_FUSED_CHAIN={env} err {e:.2e} bar {SDF_BAR:.0e}")
        assert e < SDF_BAR, (env, e)
