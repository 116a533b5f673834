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
