"""Shading / canvas / loss stage (csrc/avc_loss.cu, AvatarGen/AppearanceGen/main.py:417-497,528-534) called DIRECTLY through
the C ABI against tests/golden/loss_stage.pt -- the vectors oracle/pin_loss_stage.py recorded by executing the reference's own
source lines (background modes 3 / 1 / 0, mask_weight 0 included; cases 3-6: the add_no_texture / texture_cast_light switch
combinations of confs/ablation/*_0..2.conf).  Modes 1 and 2 reach the kernels as the same per-pixel background field
(main.py:411-414,461-465); the chessboard field itself is checked in tests/test_view_gpu.py.

The backward needs d loss / d canvases, which in the step comes from the CLIP tower: here it is taken from the CPU oracle tower
at the REFERENCE canvases, so the test isolates the stage's own kernels."""
import os

import pytest
import torch

import util_neus as U
from oracle import clip_vit as cv

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss_stage.pt")
NAMES = ("color_fine", "extra_color_fine", "gradients", "weights", "weight_sum", "gradient_error")


def _inputs(c, dev):
    from avatarclip_b200.losses import StepInputs
    H = c["H"]
    igr_w, mask_w, clip_w = c["weights"]
    dm = c["dilated_mask"].reshape(-1)
    ro = {k: c["render_out"][k].float().contiguous().to(dev) for k in NAMES}
    ro["gradient_error"] = ro["gradient_error"].reshape(1)
    ro["weight_sum"] = ro["weight_sum"].reshape(-1)
    mask = (c["mask"] > 0.5).float() if mask_w > 0.0 else torch.ones_like(c["mask"])          # main.py:407-410
    choice = c["choice_i"]
    bg = c["background_rgb"].reshape(-1).to(dev) if choice in (1, 2) else None
    si = StepInputs(torch.nonzero(dm).reshape(-1).to(torch.int32).to(dev), dm.to(torch.uint8).to(dev), c["true_rgb"].to(dev),
                    mask.to(dev), H, H, c["light_dir"].float().tolist(), c["ambience"], bg_choice=choice, background=bg,
                    igr_weight=igr_w, mask_weight=mask_w, clip_weight=clip_w, add_no_texture=c["flags"][0],
                    texture_cast_light=c["flags"][1])
    return ro, si


@pytest.mark.parametrize("case", [0, 1, 2, 3, 4, 5, 6])
def test_loss_stage_kernels_match_reference_lines(case):
    from avatarclip_b200 import losses as PL
    c = torch.load(GOLDEN, map_location="cpu", weights_only=False)["cases"][case]
    H = c["H"]
    igr_w, mask_w, clip_w = c["weights"]
    no_tex, cast = c["flags"]
    ref = c["ref"]
    ro, si = _inputs(c, "cuda")
    canv, scal = PL.stage_forward(ro, si)
    torch.cuda.synchronize()
    assert torch.isfinite(canv).all()                      # canvas 1 is written in every configuration (B = 2 CLIP batch)
    e_tex = (canv[0].reshape(-1, 3).cpu() - ref["texture_shading"]).abs().max().item()
    # the reference computes rand_shading_rgb whenever either switch is on (main.py:425); it feeds a loss term only with
    # add_no_texture
    e_sh = 0.0 if ref["rand_shading_rgb"] is None else \
        (canv[1].reshape(-1, 3).cpu() - ref["rand_shading_rgb"]).abs().max().item()
    s = scal.cpu()
    base_ref = ref["color_fine_loss"] + ref["eikonal_loss"] * igr_w + ref["mask_loss"] * mask_w             # main.py:528-531
    rel = {k: abs(s[i].item() - float(v)) / max(abs(float(v)), 1e-30)
           for k, i, v in (("color", PL.S_COLOR, ref["color_fine_loss"]), ("eikonal", PL.S_EIK, ref["eikonal_loss"]),
                           ("bce", PL.S_BCE, ref["mask_loss"]), ("psnr", PL.S_PSNR, ref["psnr"]),
                           ("base", PL.S_BASE, base_ref))}
    # d (clip terms) / d canvases from the oracle tower at the reference canvases
    clip_state = cv.random_vit_state(seed=c["clip_seed"])
    t = ref["texture_shading"].reshape(H, H, 3).clone().requires_grad_(True)
    sh = (ref["rand_shading_rgb"] if ref["rand_shading_rgb"] is not None else canv[1].reshape(-1, 3).cpu()) \
        .reshape(H, H, 3).clone().requires_grad_(True)
    clip_terms = (1.0 - cv.clip_cosine(clip_state, t, c["text"])) * clip_w + (1.0 - cv.clip_cosine(clip_state, sh, c["text"])) * clip_w
    gt, gs = torch.autograd.grad(clip_terms.sum(), [t, sh])
    # without add_no_texture the trainer still runs the B = 2 CLIP batch: the stage must IGNORE the second canvas' cotangent
    d_canv = torch.stack([gt, gs]).float().contiguous().cuda()
    cot = PL.stage_backward(ro, si, d_canv, scal)
    torch.cuda.synchronize()
    g_err = {k: U.rel_to_max(cot[k].reshape(-1), c["ref_grads"][k].reshape(-1)) for k in NAMES}
    print(f"case {case} (bg {c['choice_i']}, add_no_texture {no_tex}, texture_cast_light {cast}): canvases {e_tex:.2e} / {e_sh:.2e}; scalars {rel}; cotangents {g_err}")
    U.log_parity("loss_stage_direct", {"case": case, "bg": c["choice_i"], "flags": list(c["flags"]), "canvas_abs": max(e_tex, e_sh),
                                       "scalars_rel": max(rel.values()), "cotangents_rel_to_max": max(g_err.values())})
    assert e_tex < 2e-6 and e_sh < 2e-6
    assert max(rel.values()) < 5e-6, rel
    assert max(g_err.values()) < 5e-5, g_err


def test_loss_stage_rejects_bad_arguments():
    """Error behaviour of the C entry point (include/avc_b200.h): a missing background field for modes 1 / 2 and an
    out-of-range mode are refused with an error code, nothing is launched."""
    from avatarclip_b200 import losses as PL
    from avatarclip_b200._lib import AvcError
    c = torch.load(GOLDEN, map_location="cpu", weights_only=False)["cases"][0]
    ro, si = _inputs(c, "cuda")
    si.bg_choice = 2
    with pytest.raises(AvcError):
        PL.stage_forward(ro, si)
    si.bg_choice = 7
    with pytest.raises(AvcError):
        PL.stage_forward(ro, si)
