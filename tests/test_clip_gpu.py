"""GPU parity of the CLIP ViT-B/32 image tower + cosine loss against the CPU oracle (oracle/clip_vit.py:
the published architecture restated and cross-checked against HF transformers; PARITY UNPINNED w.r.t.
openai/CLIP itself -- see oracle/__init__.py).

The tower's GEMMs run on the wgmma kernel when the token rows fit one 128-row tile (M = 50 B <= 128: one or two
images) and on the mma.sync kernel otherwise; the three-image cases run every GEMM of the forward and the backward on
the mma.sync kernel (M = 150, patch embedding M = 147)."""
import pytest
import torch

from oracle import clip_vit as cv
import util_neus as U

pytestmark = pytest.mark.gpu


def _tower(seed=0):
    from avatarclip_b200.clip_vit import ClipImageTower
    sd = cv.random_vit_state(seed=seed)
    return sd, ClipImageTower(sd, device="cuda")


@pytest.mark.parametrize("H,images", [(160, 2), (224, 2), (256, 2), (224, 3)])
def test_clip_cosine_and_canvas_gradient(H, images):
    sd, tower = _tower()
    g = torch.Generator().manual_seed(H)
    # smooth-ish image content (renders are smooth) + noise background
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, H), indexing="ij")
    base = torch.stack([0.5 + 0.4 * torch.sin(6 * xx + 2 * yy), 0.5 + 0.4 * torch.cos(5 * yy), xx * yy], -1)
    imgs = [(base + 0.1 * torch.randn(H, H, 3, generator=g)).clamp(0, 1), torch.rand(H, H, 3, generator=g)]
    if images > 2:
        imgs.append((base.flip(0) + 0.1 * torch.randn(H, H, 3, generator=g)).clamp(0, 1))
    canv = torch.stack(imgs)
    text = torch.randn(images, 512, generator=g)
    # oracle (fp32, fp16-valued weights)
    co = canv.clone().requires_grad_(True)
    cos_o = torch.stack([cv.clip_cosine(sd, co[b], text[b]) for b in range(images)])
    w = torch.tensor([1.0, -0.7, 0.4][:images])
    (go,) = torch.autograd.grad((cos_o * w).sum(), co)
    # product
    cp = canv.cuda().requires_grad_(True)
    cos_p = tower.cosine(cp, text.cuda())
    (cos_p * w.cuda()).sum().backward()
    # north_star: CLIP loss (1 - cos) within 1e-3 relative
    loss_o, loss_p = 1.0 - cos_o.detach(), 1.0 - cos_p.detach().cpu()
    rel = ((loss_o - loss_p).abs() / loss_o.abs()).max().item()
    gerr = U.rel_to_max(cp.grad, go)
    U.log_parity("clip_tower", {"images": images, "H": H, "clip_loss_rel": rel, "canvas_grad_rel_to_max": gerr})
    print(f"H={H} images={images}: cos oracle {cos_o.tolist()} product {cos_p.tolist()} loss rel err {rel:.2e} "
          f"canvas-grad err {gerr:.2e}")
    assert rel < 1e-3
    assert gerr < 2e-2      # fp16 GEMM operands (as in the reference's CUDA path); fp32 accumulate


@pytest.mark.parametrize("batch", [1, 3])
def test_encode_image_matches_oracle(batch):
    sd, tower = _tower(seed=3)
    g = torch.Generator().manual_seed(9)
    img = torch.randn(batch, 3, 224, 224, generator=g)
    want = cv.encode_image(sd, img)
    got = tower.encode_image(img.cuda()).cpu()
    assert U.rel_to_max(got, want) < 5e-3


def _autograd_case(conf, B, H, W, seed, use_cos, use_emb, mode=0):
    """Oracle autograd and the product on one batch: loss = sum_b w_b cos_b (use_cos) + <g, emb> (use_emb)."""
    from avatarclip_b200.clip_vit import ClipImageTower
    sd = cv.random_vit_state(conf, seed=seed)
    tower = ClipImageTower(sd, device="cuda")
    g = torch.Generator().manual_seed(seed + 1)
    if mode == 0:
        x = torch.rand(B, H, W, 3, generator=g)
        img_o = lambda t: torch.cat([cv.preprocess(t[b], conf.image_size) for b in range(B)])
    else:
        x = torch.randn(B, 3, conf.image_size, conf.image_size, generator=g)
        img_o = lambda t: t
    text = torch.randn(B, conf.out_dim, generator=g)
    wc, ge = torch.randn(B, generator=g), torch.randn(B, conf.out_dim, generator=g)
    xo = x.clone().requires_grad_(True)
    emb_o = cv.encode_image(sd, img_o(xo), conf)
    cos_o = torch.cosine_similarity(emb_o, text, dim=-1)
    loss_o = (cos_o * wc).sum() * use_cos + (emb_o * ge).sum() * use_emb
    (gx_o,) = torch.autograd.grad(loss_o, xo)
    from avatarclip_b200.clip_vit import _ClipFn
    xp = x.cuda().requires_grad_(True)
    emb_p, cos_p = _ClipFn.apply(tower, xp, text.cuda(), mode)
    loss_p = (cos_p * wc.cuda()).sum() * use_cos + (emb_p * ge.cuda()).sum() * use_emb
    loss_p.backward()
    return {"emb": U.rel_to_max(emb_p, emb_o), "cos": (cos_p.detach().cpu() - cos_o.detach()).abs().max().item(),
            "grad": U.rel_to_max(xp.grad, gx_o)}


SMALL = cv.ViTConf(image_size=64, patch=16, width=128, layers=2, heads=2, mlp=256, out_dim=100)


@pytest.mark.parametrize("name,conf,B,H,W", [
    # token rows 119 / 136 / 153, patch rows 112 / 128 / 144: both GEMM paths on either side of M = 128
    ("small", SMALL, 7, 64, 80), ("small", SMALL, 8, 97, 61), ("small", SMALL, 9, 48, 200),
    ("width1024", cv.ViTConf(image_size=64, patch=32, width=1024, layers=1, heads=16, mlp=1024, out_dim=512), 2, 70, 50),
    ("tokens2", cv.ViTConf(image_size=32, patch=32, width=128, layers=2, heads=2, mlp=256, out_dim=64), 3, 40, 33)])
def test_tower_shapes_against_autograd(name, conf, B, H, W):
    """Non-square canvases and a loss through both the embedding and the cosine."""
    r = _autograd_case(conf, B, H, W, seed=B, use_cos=1.0, use_emb=1.0)
    U.log_parity("clip_tower_shapes", {"case": name, "B": B, "H": H, "W": W, **r})
    print(name, B, r)
    # measured on an H100 (400 W): emb <= 2.45e-4, |cos| <= 4.12e-5, grad <= 8.87e-4 -- the fp16 / tf32 operand floor
    assert r["emb"] < 9.5e-4 and r["cos"] < 1.6e-4 and r["grad"] < 3.5e-3


@pytest.mark.parametrize("use_cos", [0.0, 1.0])
def test_encode_image_backward(use_cos):
    """input_mode 1 (encode_image with autograd): the gradient through g_emb, alone and with g_cos."""
    r = _autograd_case(cv.ViTConf(), 2, 224, 224, seed=4, use_cos=use_cos, use_emb=1.0, mode=1)
    U.log_parity("clip_encode_image_backward", {"use_cos": use_cos, **r})
    print(use_cos, r)
    assert r["emb"] < 1e-3 and r["grad"] < 3e-3            # measured 2.97e-4 / 7.93e-4 on an H100 (400 W)
