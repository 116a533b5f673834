"""The float64 references of the NeuS kernels outside the GEMM tiles (oracle/neus_kernels.py) against torch: autograd
through oracle.neus in fp64 (and, for packing, encoding, thin contractions and the gradient chain, torch._weight_norm,
the JVP / VJP of positional_encode, F.linear and oracle.neus.sdf_gradient), torch's conventions the kernels adopt (clip / clamp backward inclusive at
the bounds, ReLU' (0) = 0, first-index max, searchsorted(right=True), at::linspace), and the deliberate rounding
(bf16 split, separately rounded fp32 placement arithmetic) against hand-written bit patterns."""
import math

import numpy as np
import pytest
import torch

from oracle import neus
from oracle import neus_kernels as nk

F64 = torch.float64


def _case(R=5, S=40, seed=0, inv_s=20.0):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(R, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    z = torch.sort(torch.rand(R, S, generator=g) * 2 + 0.5, -1)[0]
    P = R * S
    cin = torch.zeros(P, 8)
    cin[:, 0:3] = torch.randn(P, 3, generator=g) * 0.5
    cin[:, 3:6] = torch.randn(P, 3, generator=g)
    rgb6 = torch.zeros(P, 8)
    rgb6[:, 0:6] = torch.rand(P, 6, generator=g) * 0.9 + 0.05
    sdf = torch.randn(P, generator=g) * 0.1
    return d, z, sdf, cin, rgb6, torch.tensor(inv_s)


def _cots(R, S, g):
    return {"color": torch.randn(R, 3, generator=g), "extra": torch.randn(R, 3, generator=g),
            "wsum": torch.randn(R, generator=g), "wmax": torch.randn(R, generator=g),
            "weights": torch.randn(R, S, generator=g), "cdf": torch.randn(R, S, generator=g),
            "gradients": torch.randn(R * S, 3, generator=g) * 0.05, "gerr": torch.randn(1, generator=g)}


@pytest.mark.parametrize("bg_kind", [0, 1, 2])
def test_composite_bwd_matches_finite_differences(bg_kind):
    R, S = 3, 37
    d, z, sdf, cin, rgb6, s = _case(R, S, seed=bg_kind)
    g = torch.Generator().manual_seed(11)
    bg = {0: None, 1: torch.rand(3, generator=g), 2: torch.rand(R, generator=g)}[bg_kind]
    cot = _cots(R, S, g)
    args = (d, z, sdf, cin, rgb6, bg, bg_kind)
    b = nk.composite_bwd(*args, s, 0.3, 0.02, 50.0, cot)

    def loss(sdf_, cin_, rgb_, s_):
        o = nk.composite_fwd(d, z, sdf_, cin_, rgb_, bg, bg_kind, s_, 0.3, 0.02, 50.0)
        am = nk.first_argmax(o["weights"])
        tot = sum((o[k] * cot[k].double().reshape(o[k].shape)).sum() for k in ("color", "extra", "wsum", "weights",
                                                                                  "cdf"))
        tot = tot + (o["weights"].gather(1, am[:, None]).reshape(-1) * cot["wmax"].double()).sum()
        tot = tot + (cin_[:, 3:6].double() * cot["gradients"].double()).sum() + o["gerr"] * cot["gerr"].double()[0]
        return tot.item()

    h = 1e-6
    sdf64, cin64, rgb64, s64 = sdf.double(), cin.double(), rgb6.double(), s.double()
    for p in (0, 41, 77):
        e = torch.zeros_like(sdf64); e[p] = h
        fd = (loss(sdf64 + e, cin64, rgb64, s64) - loss(sdf64 - e, cin64, rgb64, s64)) / (2 * h)
        assert abs(fd - b["sdfbar"][p].item()) < 1e-6 * max(1.0, abs(fd))
        for a in range(3):
            e = torch.zeros_like(cin64); e[p, 3 + a] = h
            fd = (loss(sdf64, cin64 + e, rgb64, s64) - loss(sdf64, cin64 - e, rgb64, s64)) / (2 * h)
            assert abs(fd - b["nbar"][p, a].item()) < 1e-6 * max(1.0, abs(fd))
        for i in range(6):      # y6bar is the adjoint of the logit: d/dy * y (1 - y)
            e = torch.zeros_like(rgb64); e[p, i] = h
            fd = (loss(sdf64, cin64, rgb64 + e, s64) - loss(sdf64, cin64, rgb64 - e, s64)) / (2 * h)
            y = rgb64[p, i].item()
            assert abs(fd * y * (1 - y) - b["y6bar"][p, i].item()) < 1e-6 * max(1.0, abs(fd))
    fd = (loss(sdf64, cin64, rgb64, s64 + h * 100) - loss(sdf64, cin64, rgb64, s64 - h * 100)) / (2 * h * 100)
    assert abs(fd - b["invs_bar"].sum().item()) < 1e-6 * max(1.0, abs(fd))


def test_composite_matches_render_core_autograd():
    """composite_fwd / composite_bwd equal oracle.neus.render_core's compositing and its autograd in fp64."""
    R, S = 4, 33
    d, z, sdf, cin, rgb6, s = _case(R, S, seed=5)
    var = torch.tensor(math.log(20.0) / 10, dtype=F64)
    inv = neus.inv_s_from_variance(var)
    o = nk.composite_fwd(d, z, sdf, cin, rgb6, None, 0, inv, 0.5, 0.03)
    # the same numbers straight through neus.composite with leaves that need grad
    z64 = z.double()
    dists = torch.cat([z64[:, 1:] - z64[:, :-1], torch.full((R, 1), 0.03, dtype=F64)], -1)
    sd = sdf.double().reshape(-1, 1).requires_grad_(True)
    c = neus.composite(sd, cin[:, 3:6].double(), cin[:, 0:3].double(), rgb6[:, 0:3].double().reshape(R, S, 3),
                       rgb6[:, 3:6].double().reshape(R, S, 3), dists, inv.reshape(1, 1),
                       d.double()[:, None, :].expand(R, S, 3).reshape(-1, 3), None, 0.5)
    assert torch.equal(o["weights"], c["weights"].detach()) and torch.equal(o["color"], c["color"].detach())
    (gs,) = torch.autograd.grad(c["color"].sum(), sd)
    b = nk.composite_bwd(d, z, sdf, cin, rgb6, None, 0, inv, 0.5, 0.03, None,
                         {"color": torch.ones(R, 3)})
    assert (b["sdfbar"] - gs.reshape(-1)).abs().max().item() < 1e-10 * max(1.0, gs.abs().max().item())


def test_torch_conventions():
    # clip / clamp backward pass the gradient at both bounds
    x = torch.tensor([0.0, 0.5, 1.0, -1e-9, 1 + 1e-9], dtype=F64, requires_grad=True)
    (g,) = torch.autograd.grad(x.clip(0.0, 1.0).sum(), x)
    assert g.tolist() == [1.0, 1.0, 1.0, 0.0, 0.0]
    # ReLU' (0) = 0
    x = torch.tensor([0.0, 1.0, -1.0], dtype=F64, requires_grad=True)
    (g,) = torch.autograd.grad(torch.relu(x).sum(), x)
    assert g.tolist() == [0.0, 1.0, 0.0]
    # max(dim) sends a tied gradient to the first index; first_argmax agrees
    w = torch.zeros(2, 64, dtype=F64)
    w[0, 5] = w[0, 37] = w[0, 40] = 0.75
    w[1, 6] = w[1, 37] = 0.5
    w.requires_grad_(True)
    (g,) = torch.autograd.grad(w.max(-1)[0].sum(), w)
    assert g[0].nonzero().flatten().tolist() == [5] and g[1].nonzero().flatten().tolist() == [6]
    assert nk.first_argmax(w.detach()).tolist() == [5, 6]
    # searchsorted(right=True) = number of entries <= u
    cdf = torch.tensor([[0.0, 0.25, 0.25, 0.5, 1.0]], dtype=F64)
    u = torch.tensor([[0.0, 0.25, 0.3, 1.0]], dtype=F64)
    assert torch.searchsorted(cdf, u, right=True).tolist() == [[(cdf[0] <= v).sum().item() for v in u[0]]]


def test_fma_f32():
    # (1 + 2^-23)^2 = 1 + 2^-22 + 2^-46: fused, the 2^-46 survives; a separately rounded product would give 0
    a = 1.0 + 2 ** -23
    assert nk.fma_f32(a, a, -(1.0 + 2 ** -22)) == 2 ** -46
    assert nk.fma_f32(a, a, 0.0) == 1.0 + 2 ** -22
    # a tie rounds to even: 1 + 2^-24 lies halfway between 1 and 1 + 2^-23
    assert nk.fma_f32(2 ** -24, 1.0, 1.0) == 1.0
    assert nk.fma_f32(3 * 2 ** -24, 1.0, 1.0) == 1.0 + 2 ** -22


@pytest.mark.parametrize("start,end", [(0.0, 1.0), (0.5 / 33, 1 - 0.5 / 33), (0.5 / 64, 1 - 0.5 / 64), (0.1, 0.7)])
def test_linspace_halves(start, end):
    """at::linspace as its CUDA kernel computes it (the reference renders on the GPU; the GPU tests compare with
    torch.linspace on the device): fused multiply-adds from both ends."""
    s, e = np.float32(start), np.float32(end)
    for n in [2, 3, 9, 10, 33, 63, 64, 65, 128, 256]:
        step = np.float32((e - s) / np.float32(n - 1))
        got = nk.torch_linspace(start, end, n).numpy()
        for j in range(n):
            k = j if j < n // 2 else n - 1 - j
            base, sg = (s, 1.0) if j < n // 2 else (e, -1.0)
            # the exact value base + sg * step * k lies within half an ulp of the result
            exact = float(base) + sg * float(step) * k
            assert abs(float(got[j]) - exact) <= 0.5 * float(np.spacing(np.float32(got[j]))), (n, j)
        assert got[0] == s and (n < 2 or got[-1] == e)


def test_split_bf16_bits():
    v = torch.tensor([1.0, 1.00390625, 1.0 + 2 ** -9 + 2 ** -20, -3.1415927, 0.0, 1e-30], dtype=torch.float32)
    hi, lo = nk.split_bf16(v)
    hb = hi.view(torch.int16).numpy().astype(np.uint16).tolist()
    lb = lo.view(torch.int16).numpy().astype(np.uint16).tolist()
    # 1 + 2^-8 is a tie between 1 and 1 + 2^-7: RNE keeps the even 0x3f80, remainder 2^-8 = 0x3b80.
    # 1 + 2^-9 + 2^-20 rounds down to 1; its remainder 2^-9 (1 + 2^-11) rounds to 2^-9 = 0x3b00.
    # -pi = 0xc0490fdb -> 0xc049 (-3.140625), remainder -0.00096774 = -2^-11 * 1.9819 -> 0xba7e.
    assert hb[:4] == [0x3F80, 0x3F80, 0x3F80, 0xC049] and lb[:4] == [0, 0x3B80, 0x3B00, 0xBA7E]
    assert hb[4] == 0 and lb[4] == 0
    assert (hi.float() + lo.float() - v).abs().max().item() <= 2 ** -16 * v.abs().max().item()


def test_placement_rounding():
    g = torch.Generator().manual_seed(3)
    near, far = torch.rand(50, generator=g), torch.rand(50, generator=g) + 1.5
    jit = torch.rand(50, generator=g) - 0.5
    for n in (2, 3, 32, 63, 64):
        z = nk.coarse_z(near, far, jit, n)
        # each operation rounded on its own: the same as doing it in fp64 and rounding after every step
        lin = nk.torch_linspace(0.0, 1.0, n).double()
        r64 = (near.double()[:, None] + ((far.double() - near.double()).float().double()[:, None] * lin).float().double())
        rcp = np.float32(1.0) / np.float32(n)
        r64 = r64.float().double() + ((jit.double() * 2.0).float().double() * float(rcp)).float().double()[:, None]
        assert torch.equal(z, r64.float())
    o, d = torch.randn(6, 3, generator=g), torch.randn(6, 3, generator=g)
    z = torch.sort(torch.rand(6, 20, generator=g) * 3, -1)[0]
    mid, x = nk.mid_points(o, d, z, 2.0 / 64)
    dists = torch.cat([z[:, 1:] - z[:, :-1], torch.full((6, 1), 2.0 / 64)], -1)
    assert torch.equal(mid, z + dists * 0.5)
    assert torch.equal(x, o[:, None, :] + d[:, None, :] * mid[..., None])


def test_variance_grad():
    g_sval = torch.randn(9, dtype=F64)
    for v in (0.0, 0.3, 1.0):
        e = math.exp(10 * v)
        ib = 0.7
        got = nk.variance_grad(torch.tensor(v, dtype=F64), torch.tensor(ib, dtype=F64), g_sval).item()
        assert got == pytest.approx((ib - g_sval.sum().item() / e ** 2) * 10 * e, rel=1e-12)
    assert nk.variance_grad(torch.tensor(2.0), torch.tensor(0.7), g_sval).item() == 0.0


def test_no_fp32_variance_hits_a_clip_bound():
    """k_variance_grad zeroes the gradient unless 1e-6 < exp(10 v) < 1e6 strictly, torch's clip backward passes it at
    the bounds.  The two can only differ when the fp32 exp(fl(10 v)) equals a bound exactly: the nearest fp32 v come
    within 6.7 ulp of 1e-6f and 12.2 ulp of 1e6f (correctly rounded), beyond the 2 ulp of device expf."""
    for target in (1e6, 1e-6):
        t32 = np.float32(target)
        cur = np.float32(math.log(target) / 10)
        for _ in range(64):
            cur = np.nextafter(cur, np.float32(-np.inf))
        near = []
        for _ in range(128):
            x = np.float32(cur * np.float32(10.0))
            near.append(abs(math.exp(float(x)) - float(t32)) / float(np.spacing(t32)))
            cur = np.nextafter(cur, np.float32(np.inf))
        assert min(near) > 4.0, (target, min(near))


def test_merge_is_stable():
    z = torch.tensor([[0.1, 0.2, 0.2, 0.5]])
    newz = torch.tensor([[0.2, 0.3, 0.5]])
    s, ns = torch.tensor([[1.0, 2.0, 3.0, 4.0]]), torch.tensor([[-1.0, -2.0, -3.0]])
    zo, so = nk.merge(z, s, newz, ns)
    assert torch.equal(zo, torch.tensor([[0.1, 0.2, 0.2, 0.2, 0.3, 0.5, 0.5]]))
    assert so.tolist() == [[1.0, 2.0, 3.0, -1.0, -2.0, 4.0, -3.0]]


def test_upsample_reference_matches_oracle():
    g = torch.Generator().manual_seed(4)
    R, n, per = 6, 40, 16
    o = torch.tensor([0.0, 0.0, 1.8]) + 0.05 * torch.randn(R, 3, generator=g)
    d = torch.tensor([0.0, 0.0, -1.0]) + 0.2 * torch.randn(R, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    z = torch.sort(torch.rand(R, n, generator=g) * 2 + 0.8, -1)[0]
    sdf = (o[:, None, :] + d[:, None, :] * z[..., None]).norm(dim=-1) - 0.6
    cdf = nk.upsample_cdf(o, d, z, sdf, 64.0)
    got = nk.invert_cdf(z, cdf, nk.upsample_u(per).double())
    ref = neus.up_sample(o.double(), d.double(), z.double(), sdf.double(), per, 64.0)
    # the oracle takes the radius mask in fp64 and its u from an fp64 linspace: equal wherever neither matters
    assert (got - ref).abs().max().item() < 1e-6


# --------------------------------------------------------------------------- weights, encoding, thin ops, gradient chain
def _wide_rows(N, K, seed):
    """Weight rows over six decades, negative g, and (for the backward) a Wbar row orthogonal to its v row."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(N, K, generator=g, dtype=F64) * torch.logspace(-3, 3, N, dtype=F64)[:, None]
    gg = torch.randn(N, generator=g, dtype=F64) * 3
    gg[0] = -abs(gg[0])
    wbar = torch.randn(N, K, generator=g, dtype=F64)
    wbar[1] -= (wbar[1] @ v[1]) / (v[1] @ v[1]) * v[1]
    return v, gg, wbar


def test_pack_and_wn_backward_match_torch_weight_norm():
    v, gg, wbar = _wide_rows(7, 45, 0)
    vv, g2 = v.clone().requires_grad_(True), gg.reshape(-1, 1).clone().requires_grad_(True)
    W = torch._weight_norm(vv, g2, 0)
    assert (nk.effective_weight(v, gg) - W.detach()).abs().max().item() <= 1e-14 * W.abs().max().item()
    gv, gg_ = torch.autograd.grad((W * wbar).sum(), [vv, g2])
    gbar, vbar = nk.wn_backward(v, gg, wbar)
    assert (gbar - gg_.reshape(-1)).abs().max().item() <= 1e-12 * gg_.abs().max().item()
    for n in range(7):      # per row: the rows span six decades
        assert (vbar[n] - gv[n]).abs().max().item() <= 1e-12 * gv[n].abs().max().item()
    assert abs(gbar[1].item()) <= 1e-12 * wbar[1].norm().item()        # Wbar orthogonal to v: no g gradient


def _edge_points(P, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(P, 3, generator=g) * 0.6
    x[0] = 0.0                                          # the origin
    x[1] = torch.tensor([1.0, 0.0, 0.0])                # exactly on |x| = 1
    x[2] = torch.tensor([0.0, -1.0, 0.0])
    return x


@pytest.mark.parametrize("multires", [0, 1, 6, 7, 10])
@pytest.mark.parametrize("scale", [0.5, 1.0, 2.0])
def test_normal_and_dge_match_autograd_of_positional_encode(multires, scale):
    """k_normal is the VJP and k_dge the JVP of x -> positional_encode(scale x), both divided by scale (the sdf carries
    1 / scale)."""
    P = 9
    x = _edge_points(P, multires)
    E = 3 * (1 + 2 * multires)
    g = torch.Generator().manual_seed(100 + multires)
    ge = torch.randn(P, E + 5, generator=g, dtype=F64)
    nbar = torch.randn(P, 4, generator=g, dtype=F64)
    nbar[3] = 0.0
    enc = lambda xx: neus.positional_encode(xx * scale, multires)
    assert torch.equal(nk.encode(x, scale, multires), enc(x.double()))       # scale is a power of 2: y exact
    _, vjp = torch.func.vjp(enc, x.double())
    (want_n,) = vjp(ge[:, :E])
    got_n = nk.normal(ge, x, scale, multires)
    assert (got_n - want_n / scale).abs().max().item() <= 1e-12 * max(1.0, want_n.abs().max().item())
    _, want_g = torch.func.jvp(enc, (x.double(),), (nbar[:, 0:3],))
    got_g = nk.dge(x, nbar, scale, multires)
    assert got_g.shape == (P, E)
    assert (got_g - want_g / scale).abs().max().item() <= 1e-12 * max(1.0, want_g.abs().max().item())
    assert torch.all(got_g[3] == 0)


def test_thin_contractions_match_linear_autograd():
    g = torch.Generator().manual_seed(8)
    P, Hc, K = 37, 20, 44
    F_ = torch.nn.functional
    # sdf head: F.linear over the first K inputs, divided by scale
    inl = torch.randn(P, K + 4, generator=g, dtype=F64)
    w, b = torch.randn(K + 4, generator=g, dtype=F64), torch.randn(1, generator=g, dtype=F64)
    want = F_.linear(inl[:, :K], w[:K].reshape(1, K), b).reshape(-1) / 2.0
    assert (nk.sdf_head(inl, K, w, b, 2.0) - want).abs().max().item() <= 1e-13
    # heads: sigmoid of two linears on one activation; heads_dgrad = d/d pre-activation through the ReLU
    pre = torch.randn(P, Hc, generator=g, dtype=F64)
    pre[::3, 2] = 0.0                                   # h exactly 0 at the ReLU mask
    W6 = torch.randn(8, Hc, generator=g, dtype=F64)
    b6 = torch.randn(8, generator=g, dtype=F64)
    pr = pre.clone().requires_grad_(True)
    y = F_.linear(torch.relu(pr), W6[0:6], b6[0:6])
    assert (nk.color_heads(torch.relu(pre), W6, b6) - torch.sigmoid(y.detach())).abs().max().item() <= 1e-14
    y6bar = torch.randn(P, 8, generator=g, dtype=F64)
    (gp,) = torch.autograd.grad((y * y6bar[:, 0:6]).sum(), pr)
    assert (nk.heads_dgrad(y6bar, W6, torch.relu(pre)) - gp).abs().max().item() <= 1e-13
    # weight / bias gradients of F.linear: thin_tn (with s_scale) and colsum
    hm = torch.randn(P, Hc, generator=g, dtype=F64)
    Wl = torch.randn(6, Hc, generator=g, dtype=F64, requires_grad=True)
    bl = torch.randn(6, generator=g, dtype=F64, requires_grad=True)
    S = torch.randn(P, 6, generator=g, dtype=F64)
    gw, gb = torch.autograd.grad((F_.linear(hm, Wl, bl) * S * 0.5).sum(), [Wl, bl])
    tw, tb = nk.thin_tn(S, hm, 0.5)
    assert (tw - gw).abs().max().item() <= 1e-13 and (tb - gb).abs().max().item() <= 1e-13
    assert (nk.colsum(S, 0.5) - gb).abs().max().item() <= 1e-13
    # nbar += cbar W0[:, 3:6]: the adjoint of colour lin0's normal inputs
    cin6 = torch.randn(P, 6, generator=g, dtype=F64, requires_grad=True)
    W0x = torch.randn(Hc, 6, generator=g, dtype=F64)
    cbar = torch.randn(P, Hc, generator=g, dtype=F64)
    (gc,) = torch.autograd.grad((F_.linear(cin6, W0x) * cbar).sum(), cin6)
    c0xT = torch.zeros(8, Hc, dtype=F64)
    c0xT[0:6] = W0x.T
    nb = torch.randn(P, 4, generator=g, dtype=F64)
    assert (nk.nbar_add(nb, cbar, c0xT) - (nb[:, 0:3] + gc[:, 3:6])).abs().max().item() <= 1e-13


def _softplus_d1(z):
    return torch.where(z * 100.0 > 20.0, torch.ones_like(z), torch.sigmoid(z * 100.0))


@pytest.mark.parametrize("skip_in,multires,scale", [((2,), 6, 1.0), ((3,), 10, 2.0), ((1, 3), 7, 0.5), ((), 0, 2.0)])
def test_gradient_chain_references_match_sdf_gradient(skip_in, multires, scale):
    """k_chain_start -> the reverse sweep of the EpiChain GEMMs -> k_normal, composed from the references, is
    oracle.neus.sdf_gradient (autograd of SDFNetwork.forward) on a small network."""
    conf = neus.SDFConf(d_out=9, d_hidden=76, n_layers=3, skip_in=skip_in, multires=multires, scale=scale)
    g = torch.Generator().manual_seed(multires)
    p = {k: v.double() + 0.05 * torch.randn(v.shape, generator=g, dtype=F64)
         for k, v in neus.init_sdf_params(conf, g).items()}
    x = _edge_points(11, 1).double()
    want = neus.sdf_gradient(p, conf, x.clone(), create_graph=False)
    L, E = conf.n_layers, conf.d_enc
    W = [neus.effective_weight(p, f"lin{l}") for l in range(L + 1)]
    enc = neus.positional_encode(x * scale, multires)
    h, d1 = enc, []
    for l in range(L + 1):
        if l in skip_in:
            h = torch.cat([h, enc], -1) / math.sqrt(2)
        z = torch.nn.functional.linear(h, W[l], p[f"lin{l}.bias"])
        if l < L:
            d1.append(_softplus_d1(z))
            h = neus.softplus100(z)
    n_prev = W[L - 1].shape[0]
    qt, ge = nk.chain_start(W[L][0], d1[L - 1], n_prev, W[L].shape[1], L in skip_in, E)
    ge = ge.clone()
    for l in range(L - 1, 0, -1):
        u = qt @ W[l]
        if l in skip_in:
            np_ = W[l - 1].shape[0]
            ge = ge + u[:, np_:] * nk.SQRT_HALF
            u = u[:, :np_] * nk.SQRT_HALF
        qt = d1[l - 1] * u
    ge = ge + qt @ W[0]
    got = nk.normal(ge, x, scale, multires)
    assert (got - want).abs().max().item() <= 1e-12 * max(1.0, want.abs().max().item())

