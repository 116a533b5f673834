"""Fused train step (render -> shading/losses -> CLIP x2 -> backward -> Adam) against the CPU oracle step."""
import numpy as np
import pytest
import torch

import util_neus as U
from oracle import clip_vit as cv
from oracle.train_step import OracleTrainer

pytestmark = pytest.mark.gpu


def _setup(case, n_rays, H, bg_choice, seed=0, engine=0, add_no_texture=True, texture_cast_light=True):
    from avatarclip_b200.clip_vit import ClipImageTower
    from avatarclip_b200.trainer import AppearanceTrainer, DeviceView
    from avatarclip_b200.workload import make_view
    sdf_kw, col_kw, ren_kw, _ = U.CASES[case]
    sconf, cconf, rconf = U.confs_from_kw(sdf_kw, col_kw, ren_kw)
    sp, cp = U.synth_state(sdf_kw, col_kw, seed)
    clip_sd = cv.random_vit_state(seed=seed)
    text = torch.randn(2, 512, generator=torch.Generator().manual_seed(seed + 5))
    sdf, col, var, ren = U.build_product(sdf_kw, col_kw, ren_kw, sp, cp, 0.3, "cuda", engine=engine)
    tower = ClipImageTower(clip_sd, device="cuda")
    flags = dict(add_no_texture=add_no_texture, texture_cast_light=texture_cast_light)
    tr = AppearanceTrainer(ren, tower, text, lr=5e-4, **flags)
    orc = OracleTrainer(sconf, cconf, rconf, sp, cp, 0.3, clip_sd, text, lr=5e-4, **flags)
    hv = make_view(3, n_rays=n_rays, H=H, W=H, seed=seed, bg_choice=bg_choice)
    return tr, orc, hv, DeviceView(hv, "cuda"), (sdf, col, var)


@pytest.mark.parametrize("case,n_rays,H,bg", [("tiny", 120, 64, 3), ("shipped", 96, 80, 1), ("tiny", 150, 72, 0)])
def test_fused_step_matches_oracle(case, n_rays, H, bg):
    tr, orc, hv, dv, mods = _setup(case, n_rays, H, bg)
    # ---- loss and gradient
    grad = tr.forward_backward(dv).clone()
    loss_p = tr.loss_value().item()
    total, aux = orc.loss(hv)
    gs = torch.autograd.grad(total, [v for _, v in orc.named_params()], allow_unused=True, retain_graph=True)
    loss_o = total.item()
    print(f"loss product {loss_p:.6f} oracle {loss_o:.6f}; cos product {tr.cos.tolist()} oracle {aux['cos'].tolist()}")
    assert abs(loss_p - loss_o) / abs(loss_o) < 1e-3
    views = dict(zip([n for n, _ in [("sdf." + k, v) for k, v in mods[0].named_parameters()]
                      + [("col." + k, v) for k, v in mods[1].named_parameters()]
                      + [("var." + k, v) for k, v in mods[2].named_parameters()]], [None] * 999))
    fp = tr.fp
    named = {}
    for (p, o, m) in fp.slots:
        for pre, mod in (("sdf.", mods[0]), ("col.", mods[1]), ("var.", mods[2])):
            for k, q in mod.named_parameters():
                if q is p:
                    named[pre + k] = grad[o:o + m].view(p.shape).cpu()
    worst = 0.0
    gnorm_o = torch.cat([g.reshape(-1) for g in gs if g is not None]).norm().item()
    diff2 = 0.0
    for (k, v), g in zip(orc.named_params(), gs):
        g = torch.zeros_like(v) if g is None else g
        diff2 += (named[k] - g).double().pow(2).sum().item()
        worst = max(worst, U.rel_to_max(named[k], g))
    rel_l2 = diff2 ** 0.5 / gnorm_o
    print(f"flat-gradient rel-L2 err {rel_l2:.3e}; worst per-tensor rel-to-max {worst:.3e}")
    U.log_parity("fused_step", {"case": case, "engine": 0, "bg": bg, "loss_rel": abs(loss_p - loss_o) / abs(loss_o),
                                "grad_rel_l2": rel_l2, "worst_grad": worst})
    assert abs(loss_p - loss_o) / abs(loss_o) < 1e-4      # fp32 engine: measured ~1e-6
    assert rel_l2 < 1e-3
    # ---- one optimiser step: parameters move identically (Adam normalises, so compare the update direction)
    before = {k: v.detach().clone() for k, v in orc.named_params()}
    flat_before = tr.fp.flat.clone()
    tr.optimizer_step()
    orc.opt.zero_grad()
    total.backward()
    orc.opt.step()
    upd_p = (tr.fp.flat - flat_before)
    assert torch.isfinite(upd_p).all()
    assert abs(upd_p.abs().max().item() - 5e-4) < 1e-5     # first Adam step moves every coordinate by ~lr


def test_graph_replay_matches_eager_steps():
    """The captured-graph step (device-resident Adam state and per-view draws) reproduces the eager sequence of
    C-ABI calls: same parameters after 4 steps over changing views and a changing learning rate."""
    from avatarclip_b200.trainer import DeviceView
    from avatarclip_b200.workload import make_view
    views = [make_view(i, n_rays=120, H=64, W=64, seed=1, bg_choice=3) for i in range(3)]
    lrs = [5e-4, 5e-4, 3e-4, 1e-4]
    finals, losses_ = [], []
    for mode in ("eager", "graph"):
        tr, _, _, _, _ = _setup("tiny", 120, 64, 3)
        dv = DeviceView(views[0], "cuda")
        ls = []
        for i, lr in enumerate(lrs):
            dv.upload(views[i % 3])
            if mode == "eager":
                ls.append(tr.step(dv, lr=lr).item())
            else:
                ls.append(tr.replay(dv, lr=lr).item())
        assert tr.iter_step == len(lrs)
        finals.append(tr.fp.flat.clone())
        losses_.append(ls)
    print("losses eager", losses_[0], "graph", losses_[1])
    # the only non-determinism is the order of fp32 atomics in the weight-gradient reductions
    assert np.allclose(losses_[0], losses_[1], rtol=2e-4, atol=1e-5)
    d = (finals[0] - finals[1]).abs().max().item()
    print(f"max parameter difference after {len(lrs)} steps: {d:.3e}")
    assert d < 2e-4      # Adam's sign-like first steps amplify tiny gradient differences near zero; lr-scale bound
    # the light direction / ambience really are taken from the uploaded view, not frozen at capture time
    a = tr.replay(dv, lr=0.0).item()
    hv2 = make_view(1, n_rays=120, H=64, W=64, seed=1, bg_choice=3)
    hv2.scalars.copy_(torch.tensor([0.0, -1.0, 0.0, 0.9]))
    hv2.flat = None
    hv2.pack()
    dv.upload(hv2)
    b = tr.replay(dv, lr=0.0).item()
    assert a != b


def test_fused_step_tcgen05_engine_matches_oracle():
    """The fused step with the tcgen05 engine (what bench.py runs): loss and flat gradient against the CPU oracle step on
    the shipped-size networks (widths are multiples of 8, as engine 1 requires)."""
    tr, orc, hv, dv, mods = _setup("shipped", 96, 80, 3, engine=1)
    grad = tr.forward_backward(dv).clone()
    loss_p = tr.loss_value().item()
    total, aux = orc.loss(hv)
    params = [v for _, v in orc.named_params()]
    gs = torch.autograd.grad(total, params, allow_unused=True)
    loss_o = total.item()
    print(f"engine 1: loss product {loss_p:.6f} oracle {loss_o:.6f}")
    assert abs(loss_p - loss_o) / abs(loss_o) < 1e-3
    named = {}
    for (p, o, m) in tr.fp.slots:
        for pre, mod in (("sdf.", mods[0]), ("col.", mods[1]), ("var.", mods[2])):
            for k, q in mod.named_parameters():
                if q is p:
                    named[pre + k] = grad[o:o + m].view(p.shape).cpu()
    diff2, ref2 = 0.0, 0.0
    for (k, v), g in zip(orc.named_params(), gs):
        g = torch.zeros_like(v) if g is None else g
        diff2 += (named[k] - g).double().pow(2).sum().item()
        ref2 += g.double().pow(2).sum().item()
    rel_l2 = (diff2 / ref2) ** 0.5
    print(f"engine 1: flat-gradient rel-L2 err {rel_l2:.3e}")
    U.log_parity("fused_step", {"case": "shipped", "engine": 1, "bg": 3, "loss_rel": abs(loss_p - loss_o) / abs(loss_o),
                                "grad_rel_l2": rel_l2})
    assert rel_l2 < 1e-3


@pytest.mark.parametrize("no_tex,cast,bg,engine", [(False, False, 3, 0), (True, False, 1, 1), (False, True, 0, 0)])
def test_fused_step_with_the_ablation_switches_matches_oracle(no_tex, cast, bg, engine):
    """train.add_no_texture / train.texture_cast_light switched off as in confs/ablation/*_0..2.conf (main.py:425,509-534):
    the first CLIP term then sees the un-shaded extra colour and / or the second term is absent.  Loss and flat gradient of
    the fused step against the CPU oracle step with the same switches."""
    tr, orc, hv, dv, mods = _setup("shipped", 96, 80, bg, engine=engine, add_no_texture=no_tex, texture_cast_light=cast)
    grad = tr.forward_backward(dv).clone()
    loss_p = tr.loss_value().item()
    total, aux = orc.loss(hv)
    gs = torch.autograd.grad(total, [v for _, v in orc.named_params()], allow_unused=True)
    loss_o = total.item()
    named = {}
    for (p, o, m) in tr.fp.slots:
        for pre, mod in (("sdf.", mods[0]), ("col.", mods[1]), ("var.", mods[2])):
            for k, q in mod.named_parameters():
                if q is p:
                    named[pre + k] = grad[o:o + m].view(p.shape).cpu()
    diff2, ref2 = 0.0, 0.0
    for (k, v), g in zip(orc.named_params(), gs):
        g = torch.zeros_like(v) if g is None else g
        diff2 += (named[k] - g).double().pow(2).sum().item()
        ref2 += g.double().pow(2).sum().item()
    rel_l2 = (diff2 / ref2) ** 0.5
    loss_rel = abs(loss_p - loss_o) / abs(loss_o)
    print(f"add_no_texture {no_tex} texture_cast_light {cast} engine {engine}: loss product {loss_p:.6f} oracle {loss_o:.6f} "
          f"({loss_rel:.2e}); flat-gradient rel-L2 {rel_l2:.3e}")
    U.log_parity("fused_step_ablation", {"add_no_texture": no_tex, "texture_cast_light": cast, "engine": engine, "bg": bg,
                                         "loss_rel": loss_rel, "grad_rel_l2": rel_l2})
    assert loss_rel < 1e-4 and rel_l2 < 1e-3


def test_fused_adam_matches_torch_adam_over_5_steps():
    """avc_adam_step (eager) and avc_adam_step_dev (device-resident step counter / lr, the CUDA-graph variant) against
    torch.optim.Adam (main.py:145: lr only, default betas / eps, no weight decay) on identical gradient sequences."""
    import ctypes as C
    from avatarclip_b200 import _lib
    L = _lib.lib()
    n = 100_003
    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(n, generator=g)
    grads = [torch.randn(n, generator=g) * (10.0 ** (i - 2)) for i in range(5)]      # magnitudes 1e-2 .. 1e2
    lrs = [5e-4, 5e-4, 4e-4, 1e-4, 3e-5]
    ref = torch.nn.Parameter(p0.clone().cuda())
    opt = torch.optim.Adam([ref], lr=lrs[0])
    pa, ma, va = p0.clone().cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    pb, mb, vb = p0.clone().cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    state = torch.zeros(4, dtype=torch.float32, device="cuda")
    for i, (gr, lr) in enumerate(zip(grads, lrs)):
        gd = gr.cuda()
        for grp in opt.param_groups:
            grp["lr"] = lr
        ref.grad = gd.clone()
        opt.step()
        _lib.check(L.avc_adam_step(_lib.ptr(pa), _lib.ptr(gd), _lib.ptr(ma), _lib.ptr(va), n, lr, 0.9, 0.999, 1e-8,
                                   i + 1, 1.0, _lib.stream_ptr()), "avc_adam_step")
        state[1].fill_(lr)
        _lib.check(L.avc_adam_step_dev(_lib.ptr(pb), _lib.ptr(gd), _lib.ptr(mb), _lib.ptr(vb), n, _lib.ptr(state), 0.9,
                                       0.999, 1e-8, 1.0, _lib.stream_ptr()), "avc_adam_step_dev")
        da = (pa - ref.detach()).abs().max().item()
        db = (pb - ref.detach()).abs().max().item()
        print(f"step {i + 1}: max |param - torch.optim.Adam| eager {da:.2e} device-state {db:.2e}")
        assert da <= 1e-6 and db <= 1e-6, (i, da, db)
    st = opt.state[ref]
    assert (ma - st["exp_avg"]).abs().max().item() <= 1e-6 * st["exp_avg"].abs().max().item() + 1e-12
    assert ((va - st["exp_avg_sq"]).abs() / (st["exp_avg_sq"].abs() + 1e-30)).max().item() <= 1e-5
    assert int(state[0].item()) == 5


def test_two_renders_then_one_backward_accumulates():
    """ADVICE r1: a forward's stash must survive other renders / sdf queries issued before its backward (accumulating
    two views before one backward() -- the N-view accumulation the multi-GPU path is defined to equal)."""
    sdf_kw, col_kw, ren_kw, _ = U.CASES["tiny"]
    sp, cp = U.synth_state(sdf_kw, col_kw, 0)
    sdf, col, var, ren = U.build_product(sdf_kw, col_kw, ren_kw, sp, cp, 0.3, "cuda")
    rays = [U.make_rays(40, s) for s in (1, 2)]

    def loss_of(out):
        return out["extra_color_fine"].sum() + 0.1 * out["gradient_error"] + (out["weights"] ** 2).sum()

    def run(idx):
        o, d, near, far, jit = (t.cuda() for t in rays[idx])
        return ren.render(o, d, near, far, perturb_overwrite=1, jitter=jit, cos_anneal_ratio=1.0)

    def flat_grad():
        return torch.cat([p.grad.reshape(-1) for m in (sdf, col, var) for p in m.parameters()]).clone()

    def zero():
        for m in (sdf, col, var):
            for p in m.parameters():
                p.grad = None

    sep = []
    for i in range(2):
        zero()
        loss_of(run(i)).backward()
        sep.append(flat_grad())
    zero()
    a = run(0)
    b = run(1)                                   # a second forward before a's backward
    _ = sdf.sdf(torch.rand(1000, 3, device="cuda"))   # and an unrelated query through the shared workspace
    (loss_of(a) + loss_of(b)).backward()
    both = flat_grad()
    want = sep[0] + sep[1]
    err = (both - want).abs().max().item() / want.abs().max().item()
    print("accumulated-two-views gradient error vs sum of separate backwards:", err)
    assert err < 1e-5
