"""The NeuS kernels between the GEMM tiles -- weight packing, weight-norm backward, positional encoding, the thin (<= 8
wide) contractions, the start and end of the gradient chain and its second-order adjoint -- on their own inputs against
their float64 references (oracle/neus_kernels.py, pinned against torch autograd by test_neus_kernels_cpu.py), through
avc_neus_kernel_test: the host helpers the render launches them with, on the plan of a whole configuration.

Conventions as in test_neus_kernels_gpu.py:
- Every output buffer has a NaN-patterned guard that must keep its bits; padding the kernels write must be exactly 0,
  columns they must not write keep their NaN bits.
- Inputs a kernel must not read (the padding columns [K, Kp) nothing writes, y6bar[:, 6:8], ...) are NaN.
- Outputs that are copies or deliberate fp32 roundings (biases, identity columns, the sqrt(1/2) skip copies, sample
  points, mid_z, the |x| < 1 mask, bf16 splits) are compared exactly; everything else meets a rel-to-max bar of
  max(4 x the error of an fp32 twin of the reference on the same inputs, a floor).  Packed weights and the weight-norm
  gradient are compared per row (their rows span four decades)."""
import ctypes as C
import math

import pytest
import torch

from oracle import neus_kernels as nk

pytestmark = pytest.mark.gpu

F64 = torch.float64
NANBITS = 0x7FC0DEAD
GUARD = 64
FLOOR_FWD = 2e-6
FLOOR_BWD = 2e-5

_F = None


def _fn():
    global _F
    if _F is None:
        from avatarclip_b200 import _lib
        f = _lib.lib().avc_neus_kernel_test
        f.argtypes = [C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_float), C.POINTER(C.c_void_p),
                      C.POINTER(C.c_void_p), C.c_void_p]
        f.restype = C.c_int
        _F = (_lib, f)
    return _F


def _addr(t):
    if t is None:
        return None
    if isinstance(t, torch.Tensor):
        return t.data_ptr()
    return C.addressof(t)       # host structures: the configuration, the layout array


def _run(kind, dims, fs, ins, outs):
    _lib, f = _fn()
    d = (C.c_int64 * max(len(dims), 1))(*dims)
    fsc = (C.c_float * max(len(fs), 1))(*fs)
    pi = (C.c_void_p * max(len(ins), 1))(*[_addr(t) for t in ins])
    po = (C.c_void_p * max(len(outs), 1))(*[_addr(t) for t in outs])
    _lib.check(f(kind, d, fsc, pi, po, _lib.stream_ptr()), f"avc_neus_kernel_test({kind})")
    torch.cuda.synchronize()


class Out:
    """fp32 device buffer of `shape`, NaN-patterned, followed by a NaN-patterned guard of at least one row."""

    def __init__(self, shape, init=None):
        n = math.prod(shape)
        self.full = torch.full((n + max(GUARD, shape[-1]),), NANBITS, dtype=torch.int32, device="cuda").view(torch.float32)
        self.t = self.full[:n].view(shape)
        if init is not None:
            self.t.copy_(init)
        self.n = n

    def intact(self):
        return bool(torch.all(self.full[self.n:].view(torch.int32) == NANBITS))


def _untouched(t):
    return bool(torch.all(t.contiguous().view(torch.int32) == NANBITS))


def _pair(rows, ld):
    """A bf16 pair buffer [rows][2 ld] (hi, then lo, per row), NaN-filled."""
    return torch.full((rows, 2 * ld), float("nan"), dtype=torch.bfloat16, device="cuda")


def _split_equal(pair, ld, v, cols):
    """pair[:, cols] (hi) and pair[:, ld + cols] (lo) are exactly the two-term split of the fp32 values v[:, cols]."""
    hi, lo = nk.split_bf16(v[:, cols].contiguous())
    return (torch.equal(pair[:, cols].view(torch.int16), hi.view(torch.int16))
            and torch.equal(pair[:, ld + cols.start:ld + cols.stop].view(torch.int16), lo.view(torch.int16)))


def _rel(got, ref):
    got, ref = got.double(), ref.double().to(got.device)
    m = ref.abs().max().item()
    if m == 0.0:
        return 0.0 if torch.all(got == 0).item() else math.inf
    return (got - ref).abs().max().item() / m


def _bar(ref64, ref32, floor):
    return max(4.0 * _rel(ref32, ref64), floor)


def _check(name, got, ref, twin, floor):
    e, b = _rel(got, ref), _bar(ref, twin, floor)
    print(f"[worst] {name} err {e:.2e} bar {b:.1e}")
    assert e <= b, (name, e, b)


# --------------------------------------------------------------------------- configurations
class NeusCfg(C.Structure):
    _fields_ = [
        ("sdf_d_in", C.c_int32), ("sdf_d_out", C.c_int32), ("sdf_d_hidden", C.c_int32),
        ("sdf_n_layers", C.c_int32), ("sdf_skip_mask", C.c_uint32), ("sdf_multires", C.c_int32),
        ("sdf_scale", C.c_float),
        ("col_d_feature", C.c_int32), ("col_d_hidden", C.c_int32), ("col_n_layers", C.c_int32),
        ("n_samples", C.c_int32), ("n_importance", C.c_int32), ("up_sample_steps", C.c_int32),
        ("engine", C.c_int32), ("color_products", C.c_int32), ("wgrad_products", C.c_int32),
    ]


# name: (H, n_layers, skip_in, d_out, multires, scale, Hc, col_n_layers, engine)
CFGS = {
    "bench": (256, 8, (4,), 257, 6, 1.0, 256, 4, 1),
    "shipped": (256, 4, (4,), 257, 6, 1.0, 256, 2, 1),
    "examples_small": (128, 3, (3,), 129, 6, 1.0, 128, 1, 1),
    "tiny": (48, 3, (2,), 33, 6, 1.0, 40, 2, 0),
    "skiplast": (64, 4, (4,), 65, 6, 1.0, 64, 1, 1),
    "h52": (52, 3, (2,), 33, 6, 1.0, 44, 2, 0),
    "h44_skiplast": (44, 2, (2,), 33, 6, 1.0, 44, 1, 0),
    "scale0.5": (48, 3, (2,), 33, 6, 0.5, 40, 2, 0),
    "scale2": (64, 4, (4,), 65, 6, 2.0, 64, 1, 1),
    "mr0": (72, 3, (2,), 33, 0, 1.0, 40, 2, 1),
    "mr1": (72, 3, (2,), 33, 1, 2.0, 40, 2, 1),
    "mr7": (72, 3, (3,), 33, 7, 0.5, 40, 2, 0),
    "mr10": (72, 3, (2,), 33, 10, 2.0, 40, 2, 1),
}

HEAD = ["L", "Lc", "E", "EP", "F", "Fp", "Hc", "pack_floats", "n_params", "off_var", "pk_wsdf", "pk_bsdf", "pk_c0x",
        "pk_c0xT", "pk_W6", "pk_b6"]
LIN = ["K", "N", "Kp", "Np", "skip", "off_g", "off_v", "off_b", "pk_W", "pk_WT", "pk_b"]


class Net:
    """A configuration, its plan's layout (kind 9) and synthetic flat parameters."""

    def __init__(self, name, seed=0, engine=None):
        H, L, skip, d_out, mr, scale, Hc, Lc, eng = CFGS[name]
        self.name, self.multires, self.scale = name, mr, scale
        self.cfg = NeusCfg(sdf_d_in=3, sdf_d_out=d_out, sdf_d_hidden=H, sdf_n_layers=L,
                           sdf_skip_mask=sum(1 << l for l in skip), sdf_multires=mr, sdf_scale=scale,
                           col_d_feature=d_out - 1, col_d_hidden=Hc, col_n_layers=Lc, n_samples=64, n_importance=64,
                           up_sample_steps=4, engine=eng if engine is None else engine, color_products=0,
                           wgrad_products=0)
        buf = (C.c_int64 * (16 + 11 * 40))(*([-7] * (16 + 11 * 40)))
        _run(9, [], [], [self.cfg], [buf])
        lay = dict(zip(HEAD, buf[:16]))
        n_lin = lay["L"] + 1 + lay["Lc"] + 1 + 1
        self.lin = [dict(zip(LIN, buf[16 + 11 * i:27 + 11 * i])) for i in range(n_lin)]
        assert buf[16 + 11 * n_lin] == -7
        self.__dict__.update(lay)
        self.sdf = self.lin[:self.L + 1]
        self.col = self.lin[self.L + 1:self.L + 2 + self.Lc]
        self.extra = self.lin[-1]
        assert self.E == 3 * (1 + 2 * mr) and self.Hc == Hc and self.F == d_out - 1
        g = torch.Generator().manual_seed(seed)
        p = torch.full((self.n_params,), float("nan"))
        for i, d in enumerate(self.lin):
            N, K = d["N"], d["K"]
            decades = torch.logspace(-2, 2, N)[torch.randperm(N, generator=g)]
            p[d["off_v"]:d["off_v"] + N * K] = (torch.randn(N, K, generator=g) * decades[:, None]).reshape(-1)
            gg = torch.randn(N, generator=g)
            gg[0] = -abs(gg[0]) - 0.1                              # a negative g in every linear
            p[d["off_g"]:d["off_g"] + N] = gg
            p[d["off_b"]:d["off_b"] + N] = torch.randn(N, generator=g)
        p[self.off_var] = 0.3
        assert not torch.isnan(p).any()
        self.params = p

    def vgb(self, d, flat=None):
        p = self.params if flat is None else flat
        N, K = d["N"], d["K"]
        return (p[d["off_v"]:d["off_v"] + N * K].view(N, K), p[d["off_g"]:d["off_g"] + N],
                p[d["off_b"]:d["off_b"] + N])

    def pack(self):
        """kind 10 on this configuration: the packed buffer (device) and, for the wgmma engine, its bf16 pair."""
        pk = Out((self.pack_floats,))
        pair = torch.full((2 * self.pack_floats,), float("nan"), dtype=torch.bfloat16, device="cuda") \
            if self.cfg.engine == 1 else None
        _run(10, [], [], [self.cfg, self.params.cuda()], [pk.t, pair])
        assert pk.intact()
        return pk.t, pair


_NETS = {}


def _net(name):
    if name not in _NETS:
        _NETS[name] = Net(name)
    return _NETS[name]


# --------------------------------------------------------------------------- packing
def _expected_pack(net):
    """The fp64 packed buffer placed by hand from the layout: (ref, class 0 zero / 1 weight / 2 bias, per-entry row
    scale, fp32 twin)."""
    pf = net.pack_floats
    ref, twin = torch.zeros(pf, dtype=F64), torch.zeros(pf, dtype=F64)
    cls = torch.zeros(pf, dtype=torch.int8)
    rs = torch.ones(pf, dtype=F64)

    def put(idx, W, W32, c):
        idx = torch.as_tensor(idx).reshape(-1)
        assert torch.all(cls[idx] == 0), "layout overlap"
        ref[idx] = W.reshape(-1).double()
        twin[idx] = W32.reshape(-1).double()
        cls[idx] = c
        if c == 1:
            rs[idx] = W.abs().amax(-1, keepdim=True).expand_as(W).reshape(-1)

    def lin(d):
        v, g, b = net.vgb(d)
        return nk.effective_weight(v, g), nk.effective_weight(v, g, dtype=torch.float32), b

    ar = torch.arange
    for l, d in enumerate(net.sdf):
        W, W32, b = lin(d)
        N, K, Kp, Np = d["N"], d["K"], d["Kp"], d["Np"]
        n, k = ar(N)[:, None], ar(K)[None, :]
        if l < net.L:
            put(d["pk_W"] + n * Kp + k, W, W32, 1)
            put(d["pk_WT"] + k * Np + n, W, W32, 1)
            put(d["pk_b"] + ar(N), b, b, 2)
        else:
            put(net.pk_wsdf + ar(K)[None, :], W[0:1], W32[0:1], 1)
            put(torch.tensor([net.pk_bsdf]), b[0:1], b[0:1], 2)
            n1 = ar(N - 1)[:, None]
            put(d["pk_W"] + n1 * Kp + k, W[1:], W32[1:], 1)
            put(d["pk_WT"] + k * net.Fp + n1, W[1:], W32[1:], 1)
            put(d["pk_b"] + ar(N - 1), b[1:], b[1:], 2)
    Hc = net.Hc
    for l, d in enumerate(net.col):
        W, W32, b = lin(d)
        N, K = d["N"], d["K"]
        n = ar(N)[:, None]
        if l == 0:
            kf, kx = ar(K - 6)[None, :], ar(6)[None, :]
            put(d["pk_W"] + n * net.Fp + kf, W[:, 6:], W32[:, 6:], 1)
            put(d["pk_WT"] + kf * Hc + n, W[:, 6:], W32[:, 6:], 1)
            put(net.pk_c0x + n * 8 + kx, W[:, :6], W32[:, :6], 1)
            put(net.pk_c0xT + kx * Hc + n, W[:, :6], W32[:, :6], 1)
            put(d["pk_b"] + ar(N), b, b, 2)
        elif l < net.Lc:
            k = ar(K)[None, :]
            put(d["pk_W"] + n * Hc + k, W, W32, 1)
            put(d["pk_WT"] + k * Hc + n, W, W32, 1)
            put(d["pk_b"] + ar(N), b, b, 2)
    for h, d in enumerate((net.col[net.Lc], net.extra)):      # the two colour heads -> rows 0..2 / 3..5 of W6
        W, W32, b = lin(d)
        n, k = ar(3)[:, None], ar(Hc)[None, :]
        put(net.pk_W6 + (n + 3 * h) * Hc + k, W, W32, 1)
        put(net.pk_b6 + 3 * h + ar(3), b, b, 2)
    return ref, cls, rs, twin


@pytest.mark.parametrize("name", ["bench", "shipped", "examples_small", "tiny", "skiplast", "h52", "h44_skiplast",
                                  "mr0", "mr10"])
def test_pack(name):
    """k_pack_linear (+ k_split_bf16): every weight at its place (per row within the bar), every bias copied exactly,
    every other float of the pack exactly 0; the wgmma engine's pair is exactly the split of the fp32 pack."""
    net = _net(name)
    got, pair = net.pack()
    got = got.cpu()
    ref, cls, rs, twin = _expected_pack(net)
    w = cls == 1
    e = ((got.double() - ref).abs() / rs)[w].max().item()
    b = max(4.0 * ((twin - ref).abs() / rs)[w].max().item(), 1e-6)
    print(f"[worst] pack {name} err {e:.2e} bar {b:.1e}")
    assert e <= b, (e, b)
    assert torch.equal(got[cls == 2], ref[cls == 2].float())
    assert torch.all(got[cls == 0] == 0) and not torch.signbit(got[cls == 0]).any()
    if pair is not None:
        hi, lo = nk.split_bf16(got)
        assert torch.equal(pair[:net.pack_floats].cpu().view(torch.int16), hi.view(torch.int16))
        assert torch.equal(pair[net.pack_floats:].cpu().view(torch.int16), lo.view(torch.int16))


@pytest.mark.parametrize("name", ["bench", "shipped", "examples_small", "tiny", "h52"])
def test_weight_norm_backward(name):
    """k_wn_backward for every linear in one launch: gbar and vbar per row within the bar (one Wbar row orthogonal to its
    v row), the bias gradient an exact copy, the variance slot untouched."""
    net = _net(name)
    g = torch.Generator().manual_seed(3)
    wbar = torch.randn(net.n_params, generator=g)
    for d in net.lin:
        v, _, _ = net.vgb(d)
        wb = wbar[d["off_v"]:d["off_v"] + d["N"] * d["K"]].view(d["N"], d["K"])
        r = min(1, d["N"] - 1)
        wb[r] -= (wb[r].double() @ v[r].double() / (v[r].double() @ v[r].double()) * v[r].double()).float()
    grads = Out((net.n_params,))
    _run(11, [], [], [net.cfg, net.params.cuda(), wbar.cuda()], [grads.t])
    assert grads.intact()
    gt = grads.t.cpu()
    assert _untouched(gt[net.off_var:net.off_var + 1])
    worst = {"gbar": (0.0, 0.0), "vbar": (0.0, 0.0)}
    for d in net.lin:
        v, gg, _ = net.vgb(d)
        N, K = d["N"], d["K"]
        wb = wbar[d["off_v"]:d["off_v"] + N * K].view(N, K)
        gref, vref = nk.wn_backward(v, gg, wb)
        g32, v32 = nk.wn_backward(v, gg, wb, dtype=torch.float32)
        gv, _, gb = net.vgb(d, gt)
        gg_got = gt[d["off_g"]:d["off_g"] + N]
        assert torch.equal(gb, wbar[d["off_b"]:d["off_b"] + N])
        e = _rel(gg_got, gref)
        bar = _bar(gref, g32, FLOOR_FWD)
        assert e <= bar, ("gbar", d, e, bar)
        rs = vref.abs().amax(1, keepdim=True)
        ev = ((gv.double() - vref).abs() / rs).max().item()
        bv = max(4.0 * ((v32.double() - vref).abs() / rs).max().item(), FLOOR_FWD)
        assert ev <= bv, ("vbar", d, ev, bv)
        worst["gbar"] = max(worst["gbar"], (e, bar))
        worst["vbar"] = max(worst["vbar"], (ev, bv))
    for k, (e, b) in worst.items():
        print(f"[worst] wn_backward {k} {name} err {e:.2e} bar {b:.1e}")


# --------------------------------------------------------------------------- encoding
def _edge_points(P, g):
    x = torch.randn(P, 3, generator=g) * 0.6
    x[0] = 0.0
    if P > 2:
        x[1] = torch.tensor([1.0, 0.0, 0.0])
        x[2] = torch.tensor([0.0, 0.6, -0.8]) / torch.tensor([0.0, 0.6, -0.8]).norm()
    return x


def _targets(E, EP, n_skip, extra=9):
    """Skip targets laid out as the render lays them out: column K - E of a [P][Kp] input, K = H, Kp = round_up(H, 8)
    (H = 4 mod 8 leaves the columns [K, Kp) unwritten)."""
    ks = []
    for s in range(n_skip):
        K = ((E + extra + 4 * s + 3) // 4) * 4
        ks.append((K, ((K + 7) // 8) * 8))
    return ks


def _encode(kind, P, mr, scale, ins, fs_extra, dims_extra, n_skip, fp32_in0, fp32_skip, pairs, extra_outs=()):
    E = 3 * (1 + 2 * mr)
    EP = ((E + 7) // 8) * 8
    ks = _targets(E, EP, n_skip)
    in0 = Out((P, EP)) if fp32_in0 else None
    sk = [Out((P, Kp)) if fp32_skip[s] else None for s, (K, Kp) in enumerate(ks)]
    p0 = _pair(P, EP) if pairs else None
    ps = [_pair(P, Kp) if pairs else None for K, Kp in ks]
    dims = [mr, EP, n_skip] + [Kp for K, Kp in ks] + [0] * (4 - n_skip) + [K - E for K, Kp in ks] + [0] * (4 - n_skip)
    outs = [None if in0 is None else in0.t] + [None if o is None else o.t for o in sk] + [None] * (4 - n_skip)
    outs += [p0] + ps + [None] * (4 - n_skip) + list(extra_outs)
    _run(kind, dims + dims_extra, [scale] + fs_extra, ins, outs)
    for o in [in0] + sk:
        assert o is None or o.intact()
    return E, EP, ks, in0, sk, p0, ps


def _check_encoding(name, x, mr, scale, E, EP, ks, in0, sk, p0, ps):
    """Identity columns exact, sin / cos within the bar, padding exactly 0, skip copies exactly sqrt(1/2) times the
    in0 values, the columns around each skip copy untouched, pairs exactly the split."""
    e = in0.t
    y = nk.scaled(x, scale).to(e.device)
    assert torch.equal(e[:, 0:3], y)
    assert torch.all(e[:, E:EP] == 0)
    if mr > 0:
        dev = "cuda" if x.shape[0] > 4096 else "cpu"
        ref = nk.encode(x.to(dev), scale, mr)
        tw = nk.encode(x.to(dev), scale, mr, dtype=torch.float32)
        _check("encode " + name, e[:, 3:E], ref[:, 3:E], tw[:, 3:E], FLOOR_FWD)
    for s, (K, Kp) in enumerate(ks):
        if sk[s] is None:
            continue
        o = sk[s].t
        assert torch.equal(o[:, K - E:K], nk.skip_copy(e[:, 0:E]))
        assert _untouched(o[:, :K - E]) and _untouched(o[:, K:])
        if ps[s] is not None:
            assert _split_equal(ps[s], Kp, o, slice(K - E, K))
    if p0 is not None:
        assert _split_equal(p0, EP, e, slice(0, EP))


ENC = [  # P, multires, scale
    (1, 6, 1.0), (3, 0, 2.0), (5, 1, 0.5), (33, 7, 1.0), (127, 10, 2.0), (129, 6, 0.5), (1001, 10, 1.0),
    (65536, 6, 1.0)]


@pytest.mark.parametrize("P,mr,scale", ENC)
def test_encode_points(P, mr, scale):
    """k_encode_points with fp32 targets and pairs (engine 0 plus splits), then the wgmma form: in0 and the first skip
    target fp32-free, the pairs bit-identical to the first run's."""
    g = torch.Generator().manual_seed(P + mr)
    x = _edge_points(P, g)
    n_skip = 2
    r = _encode(12, P, mr, scale, [x.cuda()], [], [P], n_skip, True, [True, True], True)
    E, EP, ks, in0, sk, p0, ps = r
    _check_encoding("points", x, mr, scale, *r)
    r2 = _encode(12, P, mr, scale, [x.cuda()], [], [P], n_skip, False, [False, True], True)
    assert torch.equal(r2[5].view(torch.int16), p0.view(torch.int16))
    for s, (K, Kp) in enumerate(ks):
        cols = slice(K - E, K)
        assert torch.equal(r2[6][s][:, cols].view(torch.int16), ps[s][:, cols].view(torch.int16))
        assert torch.equal(r2[6][s][:, Kp + K - E:Kp + K].view(torch.int16), ps[s][:, Kp + K - E:Kp + K].view(torch.int16))
    assert torch.equal(r2[4][1].t.view(torch.int32), sk[1].t.view(torch.int32))


def _rays(R, g):
    d = torch.randn(R, 3, generator=g) * 0.25 + torch.tensor([0.0, 0.0, -1.0])
    d = d / d.norm(dim=-1, keepdim=True)
    o = torch.tensor([0.0, 0.0, 1.8]) + 0.05 * torch.randn(R, 3, generator=g)
    return o, d


@pytest.mark.parametrize("nz,pitch,Rc,mr,scale", [(64, 128, 512, 6, 1.0), (16, 16, 512, 6, 1.0), (3, 5, 7, 10, 2.0),
                                                  (1, 1, 1, 0, 0.5), (33, 40, 31, 7, 1.0)])
def test_encode_samples(nz, pitch, Rc, mr, scale):
    """k_encode_samples: point p = r nz + j from z[r][j] (row pitch), o + d z rounded like torch eager."""
    g = torch.Generator().manual_seed(nz * 7 + Rc)
    o, d = _rays(Rc, g)
    z = torch.full((Rc, pitch), float("nan"))
    z[:, :nz] = torch.sort(torch.rand(Rc, nz, generator=g) * 2 + 0.8, -1)[0]
    P = nz * Rc
    r = _encode(13, P, mr, scale, [o.cuda(), d.cuda(), z.cuda()], [], [nz, pitch, Rc], 1, True, [True], True)
    x = nk.sample_points(o, d, z[:, :nz]).reshape(P, 3)
    _check_encoding("samples", x, mr, scale, *r)


@pytest.mark.parametrize("S,Rc,mr,scale,outs", [(128, 512, 6, 1.0, True), (64, 4096, 6, 1.0, False),
                                                (3, 5, 10, 2.0, True), (1, 33, 0, 0.5, True), (40, 129, 7, 1.0, True)])
def test_encode_fine(S, Rc, mr, scale, outs):
    """k_encode_fine: mid-points (the last sample of a ray at sample_dist), cin = (x, 0, 0, 0, 0, 0), mid_z and the
    |x| < 1 mask exactly as torch eager rounds them; points at the origin and exactly on |x| = 1."""
    g = torch.Generator().manual_seed(S + Rc)
    o, d = _rays(Rc, g)
    z = torch.sort(torch.rand(Rc, S, generator=g) * 2 + 0.8, -1)[0]
    sdist = 2.0 / 64
    if S >= 3 and Rc >= 2:
        o[0], d[0] = torch.zeros(3), torch.tensor([1.0, 0.0, 0.0])
        z[0, 0], z[0, 1], z[0, 2] = -0.25, 0.25, 0.75          # mid-points 0 (the origin) and 0.5
        o[1], d[1] = torch.zeros(3), torch.tensor([0.0, 0.0, 1.0])
        z[1, 0], z[1, 1] = 0.75, 1.25                          # mid-point exactly 1: |x| = 1
        z[1, 2:] = torch.sort(torch.rand(S - 2, generator=g), -1)[0] + 1.25
    P = Rc * S
    cin = Out((P, 8))
    mid, ins = (Out((P,)), Out((P,))) if outs else (None, None)
    extra = [cin.t, None if mid is None else mid.t, None if ins is None else ins.t]
    r = _encode(14, P, mr, scale, [o.cuda(), d.cuda(), z.cuda()], [sdist], [S, Rc], 2, True, [True, True], True, extra)
    m, x = nk.mid_points(o, d, z, sdist)
    x = x.reshape(P, 3)
    want = torch.zeros(P, 8)
    want[:, 0:3] = x
    assert cin.intact() and torch.equal(cin.t.cpu(), want)
    if outs:
        assert mid.intact() and ins.intact()
        assert torch.equal(mid.t.cpu(), m.reshape(-1))
        assert torch.equal(ins.t.cpu(), nk.inside_sphere(x))
        if S >= 3 and Rc >= 2:
            assert ins.t[S].item() == 0.0 and torch.equal(cin.t[S, 0:3].cpu(), torch.tensor([0.0, 0.0, 1.0]))
    _check_encoding("fine", x, mr, scale, *r)


# --------------------------------------------------------------------------- thin contractions
ROWS = [1, 3, 5, 33, 127, 129, 1001]


def _nan_pad(t, K):
    t[:, K:] = float("nan")
    return t


@pytest.mark.parametrize("name,P,nz,pitch", [("h52", 1, 0, 0), ("h52", 129, 0, 0), ("h44_skiplast", 1001, 0, 0),
                                             ("tiny", 127, 0, 0), ("examples_small", 33, 0, 0),
                                             ("scale0.5", 1001, 0, 0), ("scale2", 5, 0, 0),
                                             ("bench", 65536, 0, 0), ("bench", 32768, 64, 128),
                                             ("shipped", 262144, 0, 0)])
def test_sdf_head(name, P, nz, pitch):
    """k_thin_nt<1, OutSdf> as the value chain launches it: reduces over the K inputs of the last linear only (the
    columns [K, Kp) of in[L] are NaN, as the render leaves them), 1 / scale, the [r][j] pitch mapping."""
    net = _net(name)
    pack, _ = net.pack()
    d = net.sdf[net.L]
    K, Kp = d["K"], d["Kp"]
    g = torch.Generator().manual_seed(P)
    inl = _nan_pad(torch.rand(P, Kp, generator=g) * 0.5, K)
    if nz:
        Rc = P // nz
        out = Out((Rc, pitch))
    else:
        out = Out((P,))
    _run(15, [P, nz, pitch], [], [net.cfg, inl.cuda(), pack], [out.t])
    assert out.intact()
    got = out.t[:, :nz].reshape(-1) if nz else out.t
    if nz:
        assert _untouched(out.t[:, nz:])
    dev = "cuda" if P > 4096 else "cpu"
    ws, bs = pack[net.pk_wsdf:net.pk_wsdf + Kp].to(dev), pack[net.pk_bsdf:net.pk_bsdf + 1].to(dev)
    ref = nk.sdf_head(inl.to(dev), K, ws, bs, net.scale)
    tw = nk.sdf_head(inl.to(dev), K, ws, bs, net.scale, dtype=torch.float32)
    _check("sdf_head", got, ref, tw, FLOOR_FWD)


def _relu_acts(P, Hc, g):
    h = torch.relu(torch.randn(P, Hc, generator=g))      # exact zeros at the ReLU mask
    return h


@pytest.mark.parametrize("name,P", [("tiny", 1), ("tiny", 5), ("skiplast", 127), ("examples_small", 1001),
                                    ("bench", 65536)])
def test_color_heads_and_nbar(name, P):
    """k_thin_nt<6, OutHeads> (rgb6[:, 6:8] exactly 0) and k_thin_nt<6, OutNbarAdd> (nbar[:, 3] untouched, rows of
    nbar = 0 included)."""
    net = _net(name)
    pack, _ = net.pack()
    Hc = net.Hc
    g = torch.Generator().manual_seed(P)
    ch = _relu_acts(P, Hc, g)
    rgb6 = Out((P, 8))
    _run(16, [P], [], [net.cfg, ch.cuda(), pack], [rgb6.t])
    assert rgb6.intact() and torch.all(rgb6.t[:, 6:8] == 0)
    dev = "cuda" if P > 4096 else "cpu"
    W6, b6 = pack[net.pk_W6:net.pk_W6 + 8 * Hc].view(8, Hc).to(dev), pack[net.pk_b6:net.pk_b6 + 8].to(dev)
    _check("color_heads", rgb6.t[:, 0:6], nk.color_heads(ch.to(dev), W6, b6),
           nk.color_heads(ch.to(dev), W6, b6, dtype=torch.float32), FLOOR_FWD)
    cbar = torch.randn(P, Hc, generator=g)
    nb0 = torch.randn(P, 4, generator=g)
    nb0[::2] = 0.0
    nbar = Out((P, 4), init=nb0.cuda())
    _run(17, [P], [], [net.cfg, cbar.cuda(), pack], [nbar.t])
    assert nbar.intact() and torch.equal(nbar.t[:, 3].cpu(), nb0[:, 3])
    c0xT = pack[net.pk_c0xT:net.pk_c0xT + 8 * Hc].view(8, Hc).to(dev)
    _check("nbar_add", nbar.t[:, 0:3], nk.nbar_add(nb0.to(dev), cbar.to(dev), c0xT),
           nk.nbar_add(nb0.to(dev), cbar.to(dev), c0xT, dtype=torch.float32), FLOOR_BWD)


@pytest.mark.parametrize("name,P", [("tiny", 3), ("h52", 129), ("examples_small", 1001), ("bench", 65536)])
def test_heads_dgrad(name, P):
    """k_heads_dgrad: cbar = (y6bar W6) [h > 0] with h exactly 0 on part of the mask, y6bar[:, 6:8] NaN (unread); the
    fp32 copy and the pair, then the pair alone (the wgmma form) bit-identical."""
    net = _net(name)
    pack, _ = net.pack()
    Hc = net.Hc
    g = torch.Generator().manual_seed(P + 1)
    h = _relu_acts(P, Hc, g)
    y6 = torch.randn(P, 8, generator=g)
    y6[:, 6:8] = float("nan")
    cb, pr = Out((P, Hc)), _pair(P, Hc)
    _run(20, [P], [], [net.cfg, y6.cuda(), pack, h.cuda()], [cb.t, pr])
    assert cb.intact()
    dev = "cuda" if P > 4096 else "cpu"
    W6 = pack[net.pk_W6:net.pk_W6 + 8 * Hc].view(8, Hc).to(dev)
    ref = nk.heads_dgrad(y6.to(dev), W6, h.to(dev))
    _check("heads_dgrad", cb.t, ref, nk.heads_dgrad(y6.to(dev), W6, h.to(dev), dtype=torch.float32), FLOOR_BWD)
    assert torch.all(cb.t.cpu()[h == 0] == 0)
    assert _split_equal(pr, Hc, cb.t, slice(0, Hc))
    pr2 = _pair(P, Hc)
    _run(20, [P], [], [net.cfg, y6.cuda(), pack, h.cuda()], [None, pr2])
    assert torch.equal(pr2.view(torch.int16), pr.view(torch.int16))


TN = [  # NI, P, NC, form
    (6, 1, 40, "heads"), (6, 3, 256, "heads"), (6, 129, 300, "heads"), (6, 1001, 128, "lin0"), (6, 65536, 256, "heads"),
    (6, 65536, 256, "lin0"), (1, 5, 52, "sdf"), (1, 33, 520, "sdf"), (1, 127, 257, "sdf"), (1, 65536, 256, "sdf"),
    (6, 262144, 256, "heads")]


@pytest.mark.parametrize("NI,P,NC,form", TN)
def test_thin_tn(NI, P, NC, form):
    """k_thin_tn in the three forms the backward launches: the colour heads (rows 0..2 / 3..5 split into two linears,
    both bias sums), colour lin0's first six columns (si = 1, sc = K, no bias) and the sdf row (s_scale = 1 / scale).
    NC below and above one 256-thread block: the bias sum is counted once.  Outputs accumulate into random values."""
    g = torch.Generator().manual_seed(P * 3 + NC)
    lds = 8 if NI == 6 else 1
    ldh = NC + (4 if NC % 8 else 8)
    S = torch.randn(P, lds, generator=g)
    if NI == 6:
        S[:, 6:] = float("nan")
    Hm = _nan_pad(torch.randn(P, ldh, generator=g), NC)
    s_scale = 0.5 if form == "sdf" else 1.0
    K = NC + 6
    if form == "heads":
        si, sc, split = NC, 1, 3
        out, out2 = Out((3, NC), torch.randn(3, NC, generator=g).cuda()), Out((3, NC), torch.randn(3, NC, generator=g).cuda())
        bo, bo2 = Out((3,), torch.randn(3, generator=g).cuda()), Out((3,), torch.randn(3, generator=g).cuda())
    elif form == "lin0":
        si, sc, split = 1, K, 6
        out, out2, bo, bo2 = Out((NC, K), torch.randn(NC, K, generator=g).cuda()), None, None, None
    else:
        si, sc, split = 0, 1, 1
        out, out2 = Out((NC,), torch.randn(NC, generator=g).cuda()), None
        bo, bo2 = Out((1,), torch.randn(1, generator=g).cuda()), None
    init = [None if o is None else o.t.clone() for o in (out, bo, out2, bo2)]
    _run(18, [NI, lds, ldh, NC, P, si, sc, split], [s_scale], [S.cuda(), Hm.cuda()],
         [None if o is None else o.t for o in (out, bo, out2, bo2)])
    for o in (out, bo, out2, bo2):
        assert o is None or o.intact()
    dev = "cuda" if P > 4096 else "cpu"
    Sv, Hv = S[:, :NI].to(dev), Hm[:, :NC].to(dev)
    rw, rb = nk.thin_tn(Sv, Hv, s_scale)
    tw, tb = nk.thin_tn(Sv, Hv, s_scale, dtype=torch.float32)
    if form == "heads":
        got_w = torch.cat([out.t - init[0], out2.t - init[2]], 0)
        got_b = torch.cat([bo.t - init[1], bo2.t - init[3]], 0)
    elif form == "lin0":
        got_w = (out.t - init[0])[:, 0:6].T
        assert torch.equal(out.t[:, 6:], init[0][:, 6:])
        got_b = None
    else:
        got_w, got_b = (out.t - init[0])[None, :], bo.t - init[1]
    # the accumulation into the initial values adds one rounding of the initial magnitude
    fl = FLOOR_BWD * max(1.0, init[0].abs().max().item() / max(rw.abs().max().item(), 1e-30))
    _check(f"thin_tn<{NI}> {form}", got_w, rw, tw, fl)
    if got_b is not None:
        flb = FLOOR_BWD * max(1.0, init[1].abs().max().item() / max(rb.abs().max().item(), 1e-30))
        _check(f"thin_tn<{NI}> bias", got_b, rb, tb, flb)


@pytest.mark.parametrize("P,NC,ld,scale", [(1, 52, 56, 1.0), (3, 257, 264, 1.0), (5, 8, 8, 0.5), (7, 44, 48, 1.0),
                                           (9, 256, 256, 1.0), (33, 520, 520, 1.0), (1001, 129, 136, 0.5),
                                           (65536, 256, 256, 1.0), (262144, 256, 264, 1.0)])
def test_colsum(P, NC, ld, scale):
    """k_colsum: the 8-way unrolled column sums, rows past a multiple of 8, columns [NC, ld) NaN (unread)."""
    g = torch.Generator().manual_seed(P + NC)
    X = _nan_pad(torch.randn(P, ld, generator=g), NC)
    init = torch.randn(NC, generator=g)
    out = Out((NC,), init.cuda())
    _run(19, [ld, NC, P], [scale], [X.cuda()], [out.t])
    assert out.intact()
    dev = "cuda" if P > 4096 else "cpu"
    ref = nk.colsum(X[:, :NC].to(dev), scale)
    fl = FLOOR_BWD * max(1.0, init.abs().max().item() / max(ref.abs().max().item(), 1e-30))
    _check("colsum", out.t - init.cuda(), ref, nk.colsum(X[:, :NC].to(dev), scale, dtype=torch.float32), fl)


# --------------------------------------------------------------------------- gradient chain
@pytest.mark.parametrize("name,P", [("bench", 65536), ("shipped", 1001), ("examples_small", 129), ("skiplast", 5),
                                    ("h52", 33), ("h44_skiplast", 127), ("mr10", 3), ("mr0", 1)])
def test_chain_start(name, P):
    """k_chain_start: qt[L-1] = sp'(z) w_sdf (sqrt(1/2) when the last linear takes the skip concat), its padding exactly
    0 (the stash's padding is NaN here), ge = the encoding part of w_sdf or 0, ge[:, E:EP] exactly 0."""
    net = _net(name)
    pack, _ = net.pack()
    dp, dL = net.sdf[net.L - 1], net.sdf[net.L]
    Np, N = dp["Np"], dp["N"]
    g = torch.Generator().manual_seed(P + 5)
    zp = _nan_pad(torch.rand(P, Np, generator=g), N)
    zp[::4, : N // 2] = 0.0
    qt, ge, pr = Out((P, Np)), Out((P, net.EP)), _pair(P, Np)
    _run(21, [P], [], [net.cfg, pack, zp.cuda()], [qt.t, ge.t, pr])
    assert qt.intact() and ge.intact()
    dev = "cuda" if P > 4096 else "cpu"
    ws = pack[net.pk_wsdf:net.pk_wsdf + dL["Kp"]].to(dev)
    rq, rg = nk.chain_start(ws, zp.to(dev), N, dL["K"], bool(dL["skip"]), net.E)
    tq, tg = nk.chain_start(ws, zp.to(dev), N, dL["K"], bool(dL["skip"]), net.E, dtype=torch.float32)
    _check("chain_start qt", qt.t[:, :N], rq, tq, FLOOR_FWD)
    assert torch.all(qt.t[:, N:] == 0) and torch.all(ge.t[:, net.E:] == 0)
    if dL["skip"]:
        _check("chain_start ge", ge.t[:, :net.E], rg, tg, FLOOR_FWD)
    else:
        assert torch.all(ge.t == 0)
    assert _split_equal(pr, Np, qt.t, slice(0, Np))
    pr2 = _pair(P, Np)
    _run(21, [P], [], [net.cfg, pack, zp.cuda()], [None, ge.t, pr2])
    assert torch.equal(pr2.view(torch.int16), pr.view(torch.int16))


@pytest.mark.parametrize("name,P", [("bench", 65536), ("tiny", 1), ("scale0.5", 33), ("scale2", 129), ("mr0", 5),
                                    ("mr1", 127), ("mr7", 1001), ("mr10", 1001)])
def test_normal(name, P):
    """k_normal: n = D(y)^T ge (the scale of y = scale x and the 1 / scale of the sdf cancel), frequencies past 7 lanes
    for multires = 10, none for multires = 0; ge[:, E:EP] NaN (unread); cin[:, 6:8] untouched; points at the origin and
    on |x| = 1."""
    net = _net(name)
    g = torch.Generator().manual_seed(P + 9)
    x = _edge_points(P, g)
    ge = _nan_pad(torch.randn(P, net.EP, generator=g), net.E)
    cin = Out((P, 8))
    cin.t[:, 0:3] = x.cuda()
    gr = Out((P, 3))
    _run(22, [P], [], [net.cfg, ge.cuda()], [cin.t, gr.t])
    assert cin.intact() and gr.intact()
    assert torch.equal(cin.t[:, 0:3].cpu(), x) and _untouched(cin.t[:, 6:8])
    assert torch.equal(cin.t[:, 3:6], gr.t)
    dev = "cuda" if P > 4096 else "cpu"
    ref = nk.normal(ge.to(dev), x.to(dev), net.scale, net.multires)
    tw = nk.normal(ge.to(dev), x.to(dev), net.scale, net.multires, dtype=torch.float32)
    _check(f"normal mr{net.multires}", gr.t, ref, tw, FLOOR_FWD)


@pytest.mark.parametrize("name,P", [("bench", 65536), ("tiny", 3), ("scale0.5", 33), ("scale2", 129), ("mr0", 5),
                                    ("mr1", 127), ("mr7", 1001), ("mr10", 1001), ("h52", 1)])
def test_dge(name, P):
    """k_dge: gebar = D(y) nbar into gebar and ubar_0 (padding exactly 0, rows with nbar = 0 exactly 0), the pair
    exactly the split of ubar_0; then the wgmma form (no fp32 ubar_0) bit-identical."""
    net = _net(name)
    g = torch.Generator().manual_seed(P + 11)
    x = _edge_points(P, g)
    cin = torch.full((P, 8), float("nan"))
    cin[:, 0:3] = x
    cin[:, 3:6] = torch.randn(P, 3, generator=g)
    nb = torch.randn(P, 4, generator=g)
    nb[:, 3] = float("nan")
    nb[1::3, 0:3] = 0.0
    Kp0 = net.sdf[0]["Kp"]
    ub, gb, pr = Out((P, Kp0)), Out((P, net.EP)), _pair(P, Kp0)
    _run(23, [P], [], [net.cfg, cin.cuda(), nb.cuda()], [ub.t, gb.t, pr])
    assert ub.intact() and gb.intact()
    E = net.E
    assert torch.equal(ub.t[:, :net.EP], gb.t) and torch.all(ub.t[:, E:] == 0) and torch.all(gb.t[:, E:] == 0)
    assert torch.all(gb.t[1::3] == 0)
    dev = "cuda" if P > 4096 else "cpu"
    ref = nk.dge(x.to(dev), nb.to(dev), net.scale, net.multires)
    tw = nk.dge(x.to(dev), nb.to(dev), net.scale, net.multires, dtype=torch.float32)
    _check(f"dge mr{net.multires}", gb.t[:, :E], ref, tw, FLOOR_BWD)
    assert _split_equal(pr, Kp0, ub.t, slice(0, Kp0))
    gb2, pr2 = Out((P, net.EP)), _pair(P, Kp0)
    _run(23, [P], [], [net.cfg, cin.cuda(), nb.cuda()], [None, gb2.t, pr2])
    assert torch.equal(gb2.t, gb.t) and torch.equal(pr2.view(torch.int16), pr.view(torch.int16))


@pytest.mark.parametrize("name,P", [("bench", 65536), ("tiny", 5), ("mr10", 129), ("mr0", 33), ("h52", 1001),
                                    ("mr7", 1)])
def test_fill_gebar(name, P):
    """k_fill_gebar: ubar_l[:, K-E:K] = gebar[:, :E] sqrt(1/2) exactly, every other column untouched, the pair exactly
    the split of those columns."""
    net = _net(name)
    l = next(i for i, d in enumerate(net.sdf) if d["skip"])
    d = net.sdf[l]
    K, Kp, E = d["K"], d["Kp"], net.E
    g = torch.Generator().manual_seed(P + 13)
    ge = _nan_pad(torch.randn(P, net.EP, generator=g), E)
    ub, pr = Out((P, Kp)), _pair(P, Kp)
    _run(24, [P, l], [], [net.cfg, ge.cuda()], [ub.t, pr])
    assert ub.intact()
    assert torch.equal(ub.t[:, K - E:K].cpu(), nk.fill_gebar(ge, E))
    assert _untouched(ub.t[:, :K - E]) and _untouched(ub.t[:, K:])
    assert _split_equal(pr, Kp, ub.t, slice(K - E, K))


# --------------------------------------------------------------------------- evaluator plumbing
@pytest.mark.parametrize("name,P", [("tiny", 1), ("tiny", 1001), ("examples_small", 65536)])
def test_evaluator_plumbing(name, P):
    """k_points_to_cin and k_assemble_sdf_feat (avc_neus_sdf_eval): exact copies."""
    net = _net(name)
    g = torch.Generator().manual_seed(P)
    x = torch.randn(P, 3, generator=g)
    cin = Out((P, 8))
    _run(25, [P], [], [x.cuda()], [cin.t])
    want = torch.zeros(P, 8)
    want[:, 0:3] = x
    assert cin.intact() and torch.equal(cin.t.cpu(), want)
    sdf = torch.randn(P, generator=g)
    feat = torch.randn(P, net.Fp, generator=g)
    out = Out((P, net.F + 1))
    _run(26, [P], [], [net.cfg, sdf.cuda(), feat.cuda()], [out.t])
    assert out.intact() and torch.equal(out.t.cpu(), torch.cat([sdf[:, None], feat[:, :net.F]], 1))

