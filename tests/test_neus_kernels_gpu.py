"""The compositing, scalar and placement kernels of the NeuS path on their own inputs against their float64 references
(oracle/neus_kernels.py, pinned against torch by test_neus_kernels_cpu.py), through avc_neus_kernel_test: the host
helpers the render launches them with.

The end-to-end parity bars (5e-2 per gradient tensor, 97 % of depths within 3e-3) cannot see a slightly wrong kernel
that only moves a small tensor or a few samples.  Here:
- Every output buffer has a NaN-patterned guard of at least one row that must keep its bits; y6bar[:, 6:8], nbar[:, 3]
  and placement columns past n are exactly 0 / untouched.
- Outputs the kernel rounds like torch eager fp32 (coarse depths, the merge permutation, per-ray relax counts) are
  compared exactly.
- Everything else meets a rel-to-max bar of max(4 x the error of an fp32 twin of the reference on the same inputs,
  a floor): the twin is the same reference run in fp32 on the CPU, so the bar follows the conditioning of each case
  (saturated sigmoids divide by 1 - alpha + 1e-7).
- k_coarse_z is compared bit for bit with torch eager on the GPU: torch.linspace's CUDA kernel (FMAs from both ends)
  and torch's division by a scalar (a product with the fp32 reciprocal).
- k_upsample's depths must lie within the bar of the fp64 depth in the fp64 bin, except where u lies within the knot
  window of an fp64 cdf knot or a bin's denominator near the 1e-5 clamp (see test_upsample)."""
import ctypes as C
import math

import pytest
import torch

from oracle import neus_kernels as nk

pytestmark = pytest.mark.gpu

GUARD = 64
NANBITS = 0x7FC0DEAD
FLOOR_FWD = 2e-6
FLOOR_BWD = 2e-5
CTX_INV_S, CTX_EIK_NUM, CTX_EIK_DEN, CTX_INVS_BAR = 0, 1, 2, 3

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


def _run(kind, dims, fs, ins, outs):
    _lib, f = _fn()
    d = (C.c_int64 * max(len(dims), 1))(*dims)
    fsc = (C.c_float * max(len(fs), 1))(*fs)
    pi = (C.c_void_p * max(len(ins), 1))(*[None if t is None else t.data_ptr() for t in ins])
    po = (C.c_void_p * max(len(outs), 1))(*[None if t is None else t.data_ptr() for t in outs])
    _lib.check(f(kind, d, fsc, pi, po, _lib.stream_ptr()), f"avc_neus_kernel_test({kind})")
    torch.cuda.synchronize()


class Out:
    """fp32 device buffer of `shape` followed by a NaN-patterned guard of at least one row."""

    def __init__(self, shape, init=None):
        n = math.prod(shape)
        self.full = torch.full((n + max(GUARD, shape[-1]),), NANBITS, dtype=torch.int32, device="cuda").view(torch.float32)
        self.t = self.full[:n].view(shape)
        if init is not None:
            self.t.copy_(init)
        self.n = n

    def intact(self):
        return bool(torch.all(self.full[self.n:].view(torch.int32) == NANBITS))


def _rel(got, ref):
    got, ref = got.double(), ref.double().to(got.device)
    m = ref.abs().max().item()
    if m == 0.0:
        return 0.0 if torch.all(got == 0).item() else math.inf
    return (got - ref).abs().max().item() / m


def _ctx(inv_s, eik_den=0.0):
    c = Out((8,))
    c.t.zero_()
    c.t[CTX_INV_S] = inv_s
    c.t[CTX_EIK_DEN] = eik_den
    return c


# --------------------------------------------------------------------------- compositing inputs
def _composite_case(R, S, seed, inv_s, special=True):
    """Rays and per-sample inputs with the edges compositing can get wrong: saturated sigmoids (|sdf| * inv_s >> 90),
    equal neighbouring depths (dist = 0), normals along the ray (true_cos exactly 1), across it (exactly 0), and zero."""
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(R, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    z = torch.sort(torch.rand(R, S, generator=g) * 2 + 0.5, -1)[0]
    P = R * S
    cin = torch.zeros(P, 8)
    cin[:, 0:3] = torch.randn(P, 3, generator=g) * 0.4
    r = cin[:, 0:3].double().norm(dim=-1)
    cin[(r - 1.2).abs() < 1e-4, 0:3] *= 0.99       # keep every point clear of the relax boundary (tested on its own)
    nrm = torch.randn(P, 3, generator=g) * 0.6
    sdf = (torch.rand(P, generator=g) - 0.5) * (4.0 / max(inv_s, 1.0) + 0.02)
    if special and R >= 3:
        d[0] = torch.tensor([0.0, 0.0, -1.0])
        nrm[0:S:3] = torch.tensor([0.0, 0.0, -1.0])          # true_cos = 1 exactly
        nrm[1:S:3] = torch.tensor([1.0, 0.0, 0.0])           # true_cos = 0 exactly
        nrm[2:S:3] = 0.0                                      # gn = 0
        sdf[S:2 * S] = torch.where(torch.arange(S) % 2 == 0, 1.0, -1.0) * 2.0   # saturated: araw exactly 0 / 1
        if S >= 4:
            z[2, 1] = z[2, 2] = z[2, 3]                      # dist = 0
    cin[:, 3:6] = nrm
    rgb6 = torch.zeros(P, 8)
    rgb6[:, 0:6] = torch.rand(P, 6, generator=g) * 0.9 + 0.05
    bgs = {0: None, 1: torch.rand(3, generator=g), 2: torch.rand(R, generator=g)}
    return d, z, sdf, cin, rgb6, bgs, g


def _check_points_clear_of_relax(cin):
    r = cin[:, 0:3].double().norm(dim=-1)
    assert (r - 1.2).abs().min().item() > 1e-5       # this generator keeps every point clear of the relax boundary


def _fwd(d, z, sdf, cin, rgb6, bg, bg_kind, inv_s, anneal, sdist, ctx):
    R, S = z.shape
    P = R * S
    outs = [Out((R, 3)), Out((R, 3)), Out((R,)), Out((R, S)), Out((R,)), Out((R,)), Out((R, S)), Out((R, 4))]
    cu = lambda t: None if t is None else t.cuda()
    _run(1, [S, R, bg_kind], [anneal, sdist], [cu(d), cu(z), cu(sdf), cu(cin), cu(rgb6), cu(bg)],
         [o.t for o in outs] + [ctx.t])
    assert all(o.intact() for o in outs) and ctx.intact()
    names = ["color", "extra", "s_val", "cdf", "wsum", "wmax", "weights", "ray_part"]
    return {k: o.t for k, o in zip(names, outs)}


FWD_CASES = [  # S, R, bg_kind, cos_anneal, inv_s
    (2, 1, 0, 0.0, 1.0), (31, 7, 1, 0.3, 64.0), (32, 8, 2, 1.0, 532.0), (33, 9, 0, 0.3, 20.0), (40, 1025, 1, 1.0, 64.0),
    (2, 50176, 2, 0.3, 532.0), (128, 9, 2, 0.0, 2e4), (200, 9, 1, 0.3, 64.0), (256, 7, 2, 0.3, 532.0),
    (256, 1025, 0, 1.0, 20.0)]


def _twin_bar(ref64, ref32, floor):
    return max(4.0 * _rel(ref32, ref64), floor)


@pytest.mark.parametrize("S,R,bg_kind,anneal,inv_s", FWD_CASES)
def test_composite(S, R, bg_kind, anneal, inv_s):
    d, z, sdf, cin, rgb6, bgs, g = _composite_case(R, S, seed=S * 7 + R, inv_s=inv_s)
    _check_points_clear_of_relax(cin)
    bg = bgs[bg_kind]
    sdist = 2.0 / max(S // 2, 1)
    eden = float(R * S) * 0.9
    ctx = _ctx(inv_s, eden)
    out = _fwd(d, z, sdf, cin, rgb6, bg, bg_kind, inv_s, anneal, sdist, ctx)
    inv = torch.tensor(inv_s, dtype=torch.float32).item()
    dev = "cuda" if R * S > 4096 else "cpu"
    cv = lambda t: None if t is None else t.to(dev)
    args = (cv(d), cv(z), cv(sdf), cv(cin), cv(rgb6), cv(bg), bg_kind, torch.tensor(inv), anneal, sdist)
    ref = nk.composite_fwd(*args, eden)
    tw = nk.composite_fwd(d, z, sdf, cin, rgb6, bg, bg_kind, torch.tensor(inv), anneal, sdist, eden,
                          dtype=torch.float32)
    worst = {}
    for k in ("color", "extra", "wsum", "wmax", "weights", "cdf"):
        e, bar = _rel(out[k], ref[k]), _twin_bar(ref[k], tw[k], FLOOR_FWD)
        worst[k] = (e, bar)
        assert e <= bar, (k, e, bar)
    assert torch.all(out["s_val"] == torch.tensor(1.0, device="cuda") / torch.tensor(inv, device="cuda"))
    rp = out["ray_part"]
    assert torch.equal(rp[:, 1].cpu().double(), ref["eik_den"].cpu())                 # exact per-ray relax counts
    e = _rel(rp[:, 0], ref["eik_num"])
    assert e <= _twin_bar(ref["eik_num"], tw["eik_num"], FLOOR_FWD), e
    c = ctx.t.cpu().double()
    want_den = torch.tensor(eden, dtype=torch.float32) + torch.tensor(ref["eik_den"].sum().item(), dtype=torch.float32)
    assert c[CTX_EIK_DEN].item() == want_den.item()
    assert abs(c[CTX_EIK_NUM].item() - ref["eik_num"].sum().item()) <= 1e-5 * max(ref["eik_num"].sum().item(), 1e-30)
    # k_finalize_fwd on that ctx
    gerr = Out((1,))
    _run(4, [], [], [ctx.t], [gerr.t])
    want = ctx.t[CTX_EIK_NUM].double() / (ctx.t[CTX_EIK_DEN].double() + 1e-5)
    assert gerr.intact() and abs(gerr.t.double().item() - want.item()) <= 2e-7 * abs(want.item())
    print(S, R, bg_kind, anneal, inv_s, {k: f"{v[0]:.2e}/{v[1]:.1e}" for k, v in worst.items()})


def _bwd(d, z, sdf, cin, rgb6, bg, bg_kind, anneal, sdist, ctx, cot, weights):
    R, S = z.shape
    P = R * S
    outs = [Out((P, 8)), Out((P,)), Out((P, 4)), Out((R, 4))]
    cu = lambda t: None if t is None else t.float().cuda()
    keys = ["color", "extra", "wsum", "wmax", "weights", "cdf", "gradients", "gerr"]
    _run(2, [S, R, bg_kind], [anneal, sdist],
         [cu(d), cu(z), cu(sdf), cu(cin), cu(rgb6), cu(bg)] + [cu(cot.get(k)) for k in keys] + [cu(weights)],
         [o.t for o in outs] + [ctx.t])
    assert all(o.intact() for o in outs) and ctx.intact()
    y6, sb, nb, rp = (o.t for o in outs)
    assert torch.all(y6[:, 6:8] == 0) and torch.all(nb[:, 3] == 0)
    return y6, sb, nb, rp


def _cots(R, S, g):
    return {"color": torch.randn(R, 3, generator=g), "extra": torch.randn(R, 3, generator=g),
            "wsum": torch.randn(R, generator=g), "wmax": torch.randn(R, generator=g),
            "weights": torch.randn(R, S, generator=g), "cdf": torch.randn(R, S, generator=g),
            "gradients": torch.randn(R * S, 3, generator=g) * 0.05, "gerr": torch.randn(1, generator=g)}


def _check_bwd(d, z, sdf, cin, rgb6, bg, bg_kind, inv_s, anneal, sdist, eden, cot, weights_in, tag):
    R, S = z.shape
    ctx = _ctx(inv_s, eden)
    y6, sb, nb, rp = _bwd(d, z, sdf, cin, rgb6, bg, bg_kind, anneal, sdist, ctx, cot, weights_in)
    inv = torch.tensor(inv_s, dtype=torch.float32).item()
    dev = "cuda" if R * S > 4096 else "cpu"
    cv = lambda t: None if t is None else t.to(dev)
    wa = None if weights_in is None else cv(weights_in)
    ref = nk.composite_bwd(cv(d), cv(z), cv(sdf), cv(cin), cv(rgb6), cv(bg), bg_kind, torch.tensor(inv), anneal, sdist,
                           eden, {k: cv(v) for k, v in cot.items()}, wa)
    tw = nk.composite_bwd(d, z, sdf, cin, rgb6, bg, bg_kind, torch.tensor(inv), anneal, sdist, eden, cot,
                          weights_in, dtype=torch.float32)
    worst = {}
    for k, got in (("y6bar", y6[:, 0:6]), ("sdfbar", sb), ("nbar", nb[:, 0:3]), ("invs_bar", rp[:, 2])):
        e, bar = _rel(got, ref[k]), _twin_bar(ref[k], tw[k], FLOOR_BWD)
        worst[k] = (e, bar)
        assert e <= bar, (tag, k, e, bar)
    tot = ref["invs_bar"].sum().item()
    scale = ref["invs_bar"].abs().sum().item()
    assert abs(ctx.t[CTX_INVS_BAR].item() - tot) <= max(FLOOR_BWD * scale, 4 * worst["invs_bar"][0] * scale + 1e-30)
    print(tag, {k: f"{v[0]:.2e}/{v[1]:.1e}" for k, v in worst.items()})


@pytest.mark.parametrize("S,R,bg_kind,anneal,inv_s", FWD_CASES)
def test_composite_bwd_all_cotangents(S, R, bg_kind, anneal, inv_s):
    d, z, sdf, cin, rgb6, bgs, g = _composite_case(R, S, seed=S * 7 + R, inv_s=inv_s)
    sdist = 2.0 / max(S // 2, 1)
    eden = float(R * S) * 0.9
    ctx = _ctx(inv_s, eden)
    w = _fwd(d, z, sdf, cin, rgb6, bgs[bg_kind], bg_kind, inv_s, anneal, sdist, ctx)["weights"].cpu()
    _check_bwd(d, z, sdf, cin, rgb6, bgs[bg_kind], bg_kind, inv_s, anneal, sdist, eden, _cots(R, S, g), w,
               f"all S={S} R={R}")


@pytest.mark.parametrize("key", ["color", "extra", "wsum", "wmax", "weights", "cdf", "gradients", "gerr"])
@pytest.mark.parametrize("bg_kind", [0, 1, 2])
def test_composite_bwd_single_cotangent(key, bg_kind):
    S, R, inv_s, anneal = 40, 9, 64.0, 0.3
    d, z, sdf, cin, rgb6, bgs, g = _composite_case(R, S, seed=3, inv_s=inv_s)
    sdist, eden = 0.05, 300.0
    ctx = _ctx(inv_s, eden)
    w = _fwd(d, z, sdf, cin, rgb6, bgs[bg_kind], bg_kind, inv_s, anneal, sdist, ctx)["weights"].cpu()
    cot = {key: _cots(R, S, g)[key]}
    _check_bwd(d, z, sdf, cin, rgb6, bgs[bg_kind], bg_kind, inv_s, anneal, sdist, eden, cot,
               w if key == "wmax" else None, f"{key} bg={bg_kind}")


def test_weight_max_ties_across_lane_blocks():
    """weight_max's cotangent goes to the FIRST largest stored weight: ties at j = 5 / 37 (same lane, two blocks), at
    j = 6 / 37 (two lanes), and a row of zeros (index 0)."""
    S, R, inv_s = 64, 3, 64.0
    d, z, sdf, cin, rgb6, bgs, g = _composite_case(R, S, seed=9, inv_s=inv_s)
    w = torch.rand(R, S, generator=g) * 0.1
    w[0, 5] = w[0, 37] = w[0, 40] = 0.5
    w[1, 6] = w[1, 37] = 0.5
    w[2] = 0.0
    cot = {"wmax": torch.randn(R, generator=g)}
    _check_bwd(d, z, sdf, cin, rgb6, None, 0, inv_s, 0.0, 0.03, 100.0, cot, w, "ties")


def test_relax_count_matches_composite_at_the_boundary():
    """Points within a few ulp of |x| = 1.2: k_relax_count (own fp32 points) and k_composite_fwd (points from cin) count
    exactly the same samples per ray, and agree with the fp64 count wherever |x| is not within 2 ulp of 1.2."""
    R, S = 512, 32
    g = torch.Generator().manual_seed(21)
    d = torch.randn(R, 3, generator=g)
    d = (d / d.norm(dim=-1, keepdim=True)).double()
    o = (torch.randn(R, 3, generator=g) * 0.2).double()
    # evenly spaced depths; sample jc's mid-point lands on |o + d m| = 1.2, the whole ray shifted by up to +-6 ulp
    b = (o * d).sum(-1)
    m = -b + torch.sqrt(b * b - (o * o).sum(-1) + 1.44)
    h = 0.01
    jc = torch.randint(0, S - 1, (R, 1), generator=g)
    z = (m[:, None] - h / 2 + (torch.arange(S)[None, :] - jc) * h).float()
    z = z + torch.randint(-6, 7, (R, 1), generator=g).float() * 2.4e-7
    sdist = h
    o32, d32 = o.float(), d.float()
    mid, x = nk.mid_points(o32, d32, z, sdist)
    cin = torch.zeros(R * S, 8)
    cin[:, 0:3] = x.reshape(-1, 3)
    cin[:, 3:6] = 1.0
    rgb6 = torch.full((R * S, 8), 0.5)
    ctx = _ctx(64.0, 0.0)
    out = _fwd(d32, z, torch.zeros(R * S), cin, rgb6, None, 0, 64.0, 0.0, sdist, ctx)
    rp = Out((R, 4))
    ctx2 = _ctx(64.0, 0.0)
    _run(3, [S, R], [sdist], [o32.cuda(), d32.cuda(), z.cuda()], [rp.t, ctx2.t])
    assert rp.intact() and ctx2.intact()
    assert torch.equal(rp.t[:, 1], out["ray_part"][:, 1])
    assert ctx2.t[CTX_EIK_DEN].item() == ctx.t[CTX_EIK_DEN].item()
    r = x.double().norm(dim=-1)
    amb = (r - 1.2).abs() <= 2 * 1.2e-7
    lo = ((r < 1.2) & ~amb).sum(-1).double()
    hi = ((r < 1.2) | amb).sum(-1).double()
    cnt = rp.t[:, 1].cpu().double()
    assert torch.all((cnt >= lo) & (cnt <= hi))
    print("relax: ambiguous points", int(amb.sum()), "of", R * S, "boundary-adjacent", int(((r - 1.2).abs() < 1e-5).sum()))


# --------------------------------------------------------------------------- scalars
def _variance_points():
    vs = [0.0, math.log(64.0) / 10, math.log(532.0) / 10, math.log(2e4) / 10, -2.0, 2.0, 0.3]
    for t in (1e6, 1e-6):       # the fp32 neighbours of ln(bound) / 10
        v = torch.tensor(math.log(t) / 10, dtype=torch.float32)
        for k in range(-3, 4):
            vv = v
            for _ in range(abs(k)):
                vv = torch.nextafter(vv, torch.tensor(math.copysign(math.inf, k)))
            vs.append(vv.item())
    return vs


@pytest.mark.parametrize("with_sval", [True, False])
def test_ctx_init_and_variance_grad(with_sval):
    vs = _variance_points()
    g = torch.Generator().manual_seed(5)
    R = 1025
    for v in vs:
        params = torch.tensor([7.0, v, 3.0], dtype=torch.float32).cuda()
        ctx = Out((8,), init=torch.full((8,), 5.0))
        _run(0, [1, 1], [], [params], [ctx.t])
        c = ctx.t.cpu()
        assert ctx.intact() and c[CTX_EIK_NUM] == 0 and c[CTX_EIK_DEN] == 0 and c[CTX_INVS_BAR] == 0
        ref = nk.inv_s(torch.tensor(v, dtype=torch.float32)).item()
        assert abs(c[CTX_INV_S].item() - ref) <= 1.5e-6 * ref, (v, c[CTX_INV_S].item(), ref)
        # zero_sums = 0 keeps the sums
        ctx2 = Out((8,), init=torch.full((8,), 5.0))
        _run(0, [1, 0], [], [params], [ctx2.t])
        assert ctx2.t[CTX_EIK_NUM].item() == 5.0 and ctx2.t[CTX_EIK_DEN].item() == 5.0 and ctx2.t[CTX_INVS_BAR] == 0
        # k_variance_grad with an inv_s adjoint in ctx
        ctx.t[CTX_INVS_BAR] = 0.37
        gs = torch.randn(R, generator=g) if with_sval else None
        gv = Out((1,))
        _run(5, [1, R], [], [params, ctx.t, None if gs is None else gs.cuda()], [gv.t])
        want = nk.variance_grad(torch.tensor(v, dtype=torch.float32), torch.tensor(0.37, dtype=torch.float32), gs).item()
        assert gv.intact()
        if want == 0.0:
            assert gv.t.item() == 0.0, v
        else:
            assert abs(gv.t.item() - want) <= 2e-5 * abs(want) + 1e-6 * abs(10 * ref * 0.37), (v, gv.t.item(), want)


# --------------------------------------------------------------------------- placement
@pytest.mark.parametrize("n", [2, 3, 10, 32, 63, 64, 96, 128])
@pytest.mark.parametrize("jit", ["none", "rand", "ends"])
def test_coarse_z_exact(n, jit):
    """Coarse depths bit for bit as torch eager computes renderer.py:305-306,319 on the GPU."""
    R, pitch = 300, n + 5
    g = torch.Generator().manual_seed(n)
    near = (torch.rand(R, generator=g) * 0.5).cuda()
    far = near + 1.0 + torch.rand(R, generator=g).cuda()
    j = {"none": None, "rand": torch.rand(R, generator=g) - 0.5,
         "ends": torch.where(torch.arange(R) % 2 == 0, 0.5, -0.5)}[jit]
    j = None if j is None else j.cuda()
    z = Out((R, pitch))
    _run(6, [n, pitch, R], [], [near, far, j], [z.t])
    ref = near[:, None] + (far - near)[:, None] * torch.linspace(0.0, 1.0, n, device="cuda")[None, :]
    if j is not None:
        ref = ref + j[:, None] * 2.0 / n
    assert torch.equal(z.t[:, :n], ref)
    assert torch.equal(z.t[:, :n].cpu(), nk.coarse_z(near.cpu(), far.cpu(), None if j is None else j.cpu(), n))
    assert torch.all(z.t[:, n:].view(torch.int32) == NANBITS) and z.intact()


@pytest.mark.parametrize("per", [1, 8, 16, 32, 33, 63, 64])
def test_linspace_reference_matches_torch_cuda(per):
    """The restated at::linspace (oracle/neus_kernels.py) that k_upsample's sample positions follow equals
    torch.linspace on the device, for the coarse grid and for sample_pdf's u."""
    u = torch.linspace(0.5 / per, 1.0 - 0.5 / per, per, device="cuda").cpu()
    assert torch.equal(nk.upsample_u(per), u)
    for n in (per, 2 * per + 1):
        assert torch.equal(nk.torch_linspace(0.0, 1.0, n), torch.linspace(0.0, 1.0, n, device="cuda").cpu())


@pytest.mark.parametrize("n,per,news", [(32, 8, True), (64, 64, True), (192, 64, False), (192, 64, True), (1, 1, True),
                                        (255, 1, True), (100, 33, False)])
def test_merge_exact(n, per, news):
    R = 77
    g = torch.Generator().manual_seed(n + per)
    pitch, pitch_o = n + 3, n + per + 2
    z = torch.sort(torch.rand(R, n, generator=g), -1)[0]
    newz = torch.sort(torch.rand(R, per, generator=g), -1)[0]
    k = min(n, per)
    newz[:, :k:2] = z[:, :k:2]                       # ties between old and new depths
    newz = torch.sort(newz, -1)[0]
    sdf = torch.randn(R, n, generator=g)
    ns = torch.randn(R, per, generator=g) if news else None
    zp = torch.full((R, pitch), float("nan"))
    zp[:, :n] = z
    sp = torch.full((R, pitch), float("nan"))
    sp[:, :n] = sdf
    zo, so = Out((R, pitch_o)), Out((R, pitch_o))
    _run(8, [n, pitch, R, per, pitch_o], [], [zp.cuda(), sp.cuda(), newz.cuda(), None if ns is None else ns.cuda()],
         [zo.t, so.t])
    rz, rs = nk.merge(z, sdf, newz, ns)
    assert torch.equal(zo.t[:, :n + per].cpu(), rz)
    assert torch.all(zo.t[:, n + per:].view(torch.int32) == NANBITS) and zo.intact() and so.intact()
    if news:
        assert torch.equal(so.t[:, :n + per].cpu(), rs)
    else:
        assert torch.all(so.t.view(torch.int32) == NANBITS)


def _upsample_case(kind, R, n, g):
    o = torch.tensor([0.0, 0.0, 1.8]) + 0.05 * torch.randn(R, 3, generator=g)
    d = torch.tensor([0.0, 0.0, -1.0]) + 0.3 * torch.randn(R, 3, generator=g)
    if kind == "miss":                  # rays that miss the unit sphere: no section is inside, cos_val = 0
        d = torch.tensor([1.0, 0.0, -0.3]) + 0.05 * torch.randn(R, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    z = torch.sort(torch.rand(R, n, generator=g) * 2.0 + 0.8, -1)[0]
    if kind == "uniform":               # constant sdf on even depths: knots at j / (n - 1), u on every other knot
        z = (torch.linspace(0.8, 2.8, n)[None, :] + torch.zeros(R, 1)).contiguous()
    x = o[:, None, :] + d[:, None, :] * z[..., None]
    if kind in ("constant", "uniform"):
        sdf = torch.full((R, n), 0.3)
    elif kind == "sharp":               # a thin shell: cdf plateaus (increments below 1e-5) away from it
        sdf = x.norm(dim=-1) - 0.6
    else:
        sdf = x.norm(dim=-1) - 0.6 + 0.01 * torch.randn(R, n, generator=g)
    return o, d, z, sdf


@pytest.mark.parametrize("kind,n,per,inv_s", [("smooth", 64, 16, 64.0), ("smooth", 192, 64, 512.0),
                                              ("sharp", 33, 8, 128.0), ("sharp", 255, 1, 512.0), ("miss", 64, 33, 64.0),
                                              ("constant", 40, 64, 64.0), ("uniform", 65, 32, 64.0),
                                              ("smooth", 2, 8, 64.0)])
def test_upsample(kind, n, per, inv_s):
    """Each new depth lies within the bar of the fp64 depth in the fp64 bin.  The bar and the knot window follow the
    fp32 twin: DELTA_r = 4 x the twin's worst cdf error on ray r (at least 1e-6).  Where u lies within DELTA_r of an fp64
    knot (or the bin's fp64 denominator within DELTA_r of the 1e-5 clamp), either neighbouring bin (or clamp outcome)
    is accepted, with the depth matching the fp64 value for the choice the kernel made."""
    R = 500
    g = torch.Generator().manual_seed(n * 3 + per)
    o, d, z, sdf = _upsample_case(kind, R, n, g)
    pitch = n + 4
    zp = torch.zeros(R, pitch)
    zp[:, :n] = z
    sp = torch.zeros(R, pitch)
    sp[:, :n] = sdf
    nz = Out((R, per))
    _run(7, [n, pitch, R, per], [inv_s], [o.cuda(), d.cuda(), zp.cuda(), sp.cuda()], [nz.t])
    assert nz.intact()
    got = nz.t.cpu().double()
    cdf = nk.upsample_cdf(o, d, z, sdf, inv_s)
    twin = nk.upsample_cdf(o, d, z, sdf, inv_s, dtype=torch.float32).double()
    delta = torch.clamp(4.0 * (twin - cdf).abs().max(-1, keepdim=True)[0], min=1e-6)      # [R, 1]
    u = nk.upsample_u(per).double()
    inds = torch.searchsorted(cdf, u.expand(R, -1).contiguous(), right=True)
    near_knot = (u[None, :, None] - cdf[:, None, :]).abs().min(-1)[0] < delta
    zd = z.double()
    zmax = zd.abs().max()
    best = torch.full_like(got, math.inf)
    for off in (-1, 0, 1):
        b = (inds + off).clamp(0, n)
        hi_i, lo_i = b.clamp(max=n - 1), (b - 1).clamp(min=0)
        width = (zd.gather(1, hi_i) - zd.gather(1, lo_i)).abs()
        den = cdf.gather(1, hi_i) - cdf.gather(1, lo_i)
        near_clamp = (den - 1e-5).abs() < delta
        for th in (1e-5, 1e-5 - delta, 1e-5 + delta):
            cand = nk.invert_cdf(zd, cdf, u, bins=b, clamp=th)
            dn = torch.where(den < th, torch.ones_like(den), den)
            # fp32 cdf error delta / 4, scaled by width / denom, plus a few ulp of the depth
            bar = width * delta / dn + 4e-7 * zmax
            ok = ((off == 0) | near_knot) & ((th == 1e-5) | near_clamp)
            best = torch.where(ok, torch.minimum(best, (got - cand).abs() / bar), best)
    bad = best > 1.0
    print(kind, n, per, "ambiguous samples", int(near_knot.sum()), "of", R * per, "worst dz / bar",
          best.max().item(), "median delta", delta.median().item())
    assert not bad.any(), (int(bad.sum()), best[bad][:5].tolist())
