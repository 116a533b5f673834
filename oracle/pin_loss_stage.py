"""Pin oracle/loss.py (shading / canvases / losses, cameras, ray generators, schedules) against the UNMODIFIED
reference source, executed in place.

`AvatarGen/AppearanceGen/main.py` and `models/{utils,dataset}.py` cannot be imported here (clip, smplx,
neural_renderer, pyhocon, trimesh are not installed), but the code of this path is plain torch / numpy.  This script
therefore reads the reference FILES, cuts out exactly the line ranges the oracle cites, dedents them and `exec`s them
with stand-ins for the objects around them (`self`, the renderer's result dict, a CLIP tower) -- the arithmetic that
runs is the reference's own text, byte for byte:

    main.py:417-534            the whole loss stage of Runner.train_clip (mask_sum ... loss += ...)
    main.py:571-586            get_cos_anneal_ratio, update_learning_rate
    models/utils.py:6-27,59-64 norm_np_arr + lookat, sphere_coord
    models/dataset.py:252-293,331-342   gen_rays_silhouettes, gen_rays_pose, near_far_from_sphere

It asserts equality with the oracle's restatement (values and gradients w.r.t. every differentiable renderer output)
and writes `tests/golden/loss_stage.pt` (inputs + the reference's outputs), which `tests/test_oracle_golden.py`
replays without /root/reference.  Run in the build container only:  python -m oracle.pin_loss_stage

CLIP: the perceptor is the oracle's own ViT (random weights) on both sides -- this pins the code AROUND the tower
(resize, Normalize, mean over the batch, cosine), not the tower.  torchvision here is 0.26 (antialias defaults to
True); the canvases are 112 x 112 and 224 x 224, i.e. up-sampling / identity, where antialiasing has no effect, so the
reference lines give the same numbers as under the torchvision 0.8 they were written for.
"""
from __future__ import annotations

import math
import os
import sys
import textwrap
import types

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.path.join(os.environ.get("AVC_REFERENCE", "/root/reference"), "AvatarGen/AppearanceGen")

from oracle import clip_vit as cv          # noqa: E402
from oracle import loss as ol              # noqa: E402


def cut(path, first, last, expect_first, expect_last):
    """Lines first..last (1-based, inclusive) of a reference file, dedented; the anchors guard against drift."""
    lines = open(os.path.join(REF, path)).read().split("\n")
    body = lines[first - 1:last]
    assert expect_first in body[0], (path, first, body[0])
    assert expect_last in body[-1], (path, last, body[-1])
    return textwrap.dedent("\n".join(body)) + "\n"


def rel(a, b):
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-30))


# ------------------------------------------------------------------------------------------------ inputs
def synthetic_inputs(H, seed, choice_i):
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(H), indexing="ij")
    r2 = (yy - (H - 1) / 2.0) ** 2 + (xx - (H - 1) / 2.0) ** 2
    dilated = r2 < (0.33 * H) ** 2
    inner = r2 < (0.25 * H) ** 2
    R, S = int(dilated.sum()), 12
    ro = {
        "color_fine": torch.rand(R, 3, generator=g),
        "extra_color_fine": torch.rand(R, 3, generator=g),
        "gradients": torch.randn(R, S, 3, generator=g),
        "weights": torch.rand(R, S, generator=g) / S,
        "weight_sum": torch.rand(R, 1, generator=g),
        "gradient_error": torch.rand((), generator=g),
        "s_val": torch.rand(R, 1, generator=g), "cdf_fine": torch.rand(R, S, generator=g),
        "weight_max": torch.rand(R, 1, generator=g),
    }
    ro["gradients"][3] = 0.0                      # a ray whose normal is exactly zero (the 1e-7 guards)
    true_rgb = inner.reshape(-1, 1).float().repeat(1, 3) * (0.3 + 0.7 * torch.rand(H * H, 3, generator=g))
    mask = torch.zeros_like(true_rgb)
    mask[true_rgb != 0] = 1
    mask = mask[..., :1]
    background_rgb = None
    if choice_i == 0:
        background_rgb = torch.ones([1, 3])
    elif choice_i in (1, 2):
        background_rgb = torch.clamp(0.5 + 0.2 * torch.randn(H, H, 1, generator=g), 0, 1).reshape(-1, 1)
    return ro, dilated, true_rgb, mask, background_rgb, S


# ------------------------------------------------------------------------------------------------ reference run
def run_reference_stage(snippet, ro, dilated, true_rgb, mask, background_rgb, choice_i, H, S, clip_state, text,
                        theta, phi, np_seed, weights, flags=(True, True)):
    igr_w, mask_w, clip_w = weights
    add_no_texture, texture_cast_light = flags
    from torchvision import transforms
    leaves = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in ro.items()}

    class Renderer:
        n_samples, n_importance = S // 2, S - S // 2
        def render(self, *a, **k):
            return leaves

    perceptor = types.SimpleNamespace(encode_image=lambda x: cv.encode_image(clip_state, x))
    self = types.SimpleNamespace(
        renderer=Renderer(), get_cos_anneal_ratio=lambda: 1.0, add_no_texture=add_no_texture,
        texture_cast_light=texture_cast_light,
        use_silhouettes=True, use_face_prompt=False, use_back_prompt=False, igr_weight=igr_w, mask_weight=mask_w,
        clip_weight=clip_w, perceptor=perceptor, encoded_text=text,
        clip_normalizer=transforms.Normalize((0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)),
        resize=transforms.RandomResizedCrop(224, scale=(1, 1)),                      # main.py:266
        random_perspective=transforms.RandomPerspective(p=0, distortion_scale=0.5))  # main.py:267
    ns = dict(torch=torch, np=np, F=F, transforms=transforms, self=self, sphere_coord=REF_FUNCS["sphere_coord"],
              rays_o=None, rays_d=None, near=None, far=None, H=H, W=H, dilated_mask=dilated, choice_i=choice_i,
              background_rgb=background_rgb, true_rgb=true_rgb, theta=theta, phi=phi, iter_i=1, is_front=1)
    # main.py:407-415 (the two statements just before the cut, restated here because they sit in the same block)
    ns["mask"] = (mask > 0.5).float() if mask_w > 0.0 else torch.ones_like(mask)
    ns["masked_background_rgb"] = background_rgb.reshape(H, H, 1)[dilated].reshape(-1, 1) if choice_i in (1, 2) \
        else background_rgb
    np.random.seed(np_seed)
    # the only shim: `.cuda()` (main.py:462,481,485 -- a device move, no arithmetic) is the identity on this GPU-less box
    saved_cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self_, *a, **k: self_
    try:
        exec(compile(snippet, "main.py:417-534", "exec"), ns)
    finally:
        torch.Tensor.cuda = saved_cuda
    loss = ns["loss"]
    diff = [k for k in ("color_fine", "extra_color_fine", "gradients", "weights", "weight_sum", "gradient_error")]
    grads = torch.autograd.grad(loss, [leaves[k] for k in diff], allow_unused=True)
    out = {k: ns[k].detach() for k in ("loss", "color_fine_loss", "mask_loss", "eikonal_loss", "psnr", "cosine")}
    # the image the first CLIP term saw (main.py:509-520): texture_shading, or the extra-colour canvas without cast light
    out["texture_shading"] = (ns["texture_shading"] if texture_cast_light else ns["extra_color_fine"]).detach()
    out["cosine_shading"] = ns["cosine_shading"].detach() if add_no_texture else None
    out["rand_shading_rgb"] = ns["rand_shading_rgb"].detach() if (add_no_texture or texture_cast_light) else None
    out["grads"] = {k: (torch.zeros_like(leaves[k]) if g is None else g.detach()) for k, g in zip(diff, grads)}
    return out


def run_oracle_stage(ro, dilated, true_rgb, mask, background_rgb, choice_i, H, clip_state, text, light_dir, ambience,
                     weights, flags=(True, True)):
    igr_w, mask_w, clip_w = weights
    add_no_texture, texture_cast_light = flags
    leaves = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in ro.items()}
    m = (mask > 0.5).float() if mask_w > 0.0 else torch.ones_like(mask)
    st = ol.shading_and_losses(leaves, dilated, H, H, true_rgb, m, torch.as_tensor(light_dir, dtype=torch.float32),
                               float(ambience), choice_i, background_rgb if choice_i in (1, 2) else None, igr_w, mask_w,
                               add_no_texture=add_no_texture, texture_cast_light=texture_cast_light)
    c_tex = cv.clip_cosine(clip_state, st["texture_canvas"], text)
    c_sh = cv.clip_cosine(clip_state, st["shading_canvas"], text) if add_no_texture else None
    loss = ol.total_loss(st, c_tex, c_sh, clip_w)
    diff = ["color_fine", "extra_color_fine", "gradients", "weights", "weight_sum", "gradient_error"]
    grads = torch.autograd.grad(loss, [leaves[k] for k in diff], allow_unused=True)
    out = {"loss": loss.detach(), "color_fine_loss": st["color_loss"].detach(), "mask_loss": st["mask_loss"].detach(),
           "eikonal_loss": st["eikonal_loss"].detach(), "psnr": st["psnr"].detach(), "cosine": c_tex.detach(),
           "cosine_shading": None if c_sh is None else c_sh.detach(),
           "texture_shading": st["texture_canvas"].reshape(-1, 3).detach(),
           "rand_shading_rgb": None if st["shading_canvas"] is None else st["shading_canvas"].reshape(-1, 3).detach()}
    out["grads"] = {k: (torch.zeros_like(leaves[k]) if g is None else g.detach()) for k, g in zip(diff, grads)}
    return out


REF_FUNCS = {}


def load_reference_functions():
    ns = dict(np=np, torch=torch)
    exec(cut("models/utils.py", 6, 27, "def norm_np_arr", "return"), ns)
    exec(cut("models/utils.py", 59, 64, "def sphere_coord", "])"), ns)
    REF_FUNCS["lookat"], REF_FUNCS["sphere_coord"] = ns["lookat"], ns["sphere_coord"]
    from scipy import ndimage
    dns = dict(np=np, torch=torch, ndimage=ndimage)
    exec(cut("models/dataset.py", 252, 275, "def gen_rays_silhouettes", "return masked_rays_o"), dns)
    exec(cut("models/dataset.py", 277, 293, "def gen_rays_pose", "return rays_o, rays_v"), dns)
    exec(cut("models/dataset.py", 331, 342, "def near_far_from_sphere", "return near, far"), dns)
    for k in ("gen_rays_silhouettes", "gen_rays_pose", "near_far_from_sphere"):
        REF_FUNCS[k] = dns[k]
    mns = dict(np=np, torch=torch)
    exec(cut("main.py", 571, 586, "def get_cos_anneal_ratio", "g['lr']"), mns)
    REF_FUNCS["get_cos_anneal_ratio"], REF_FUNCS["update_learning_rate"] = mns["get_cos_anneal_ratio"], mns["update_learning_rate"]


def fake_dataset(Hfull=256, fov=math.pi / 3):
    focal = .5 * Hfull / np.tan(.5 * fov)                                   # dataset.py:235-236
    K = torch.from_numpy(np.array([[focal, 0, 0.5 * Hfull], [0, focal, 0.5 * Hfull], [0, 0, 1]])).cpu()
    ds = types.SimpleNamespace(H=Hfull, W=Hfull, K=K)
    ds.gen_rays_pose = lambda pose, resolution_level=1: REF_FUNCS["gen_rays_pose"](ds, pose, resolution_level)
    return ds


def main():
    torch.manual_seed(0)
    load_reference_functions()
    worst = {}

    def note(name, err, tol):
        worst[name] = max(worst.get(name, 0.0), err)
        assert err <= tol, f"{name}: {err:.3e} > {tol:.1e}"

    # ---- cameras, schedules
    for eye, at in (((0.3, 0.2, 1.4), (0.0, 0.1, 0.0)), ((-1.2, 0.0, 0.7), (0.05, -0.1, 0.02))):
        note("lookat", rel(ol.lookat(eye, at), REF_FUNCS["lookat"](np.array(eye), np.array(at), np.array([0, 1, 0]))), 1e-12)
    for th, ph in ((0.3, 1.1), (2.0, -0.4)):
        note("sphere_coord", rel(ol.sphere_coord(th, ph), REF_FUNCS["sphere_coord"](th, ph)), 1e-15)
    for it in (0, 100, 499, 500, 7000, 29999):
        r = types.SimpleNamespace(iter_step=it, warm_up_end=500, end_iter=30000, learning_rate_alpha=0.05, learning_rate=5e-4,
                                  anneal_end=0.0, optimizer=types.SimpleNamespace(param_groups=[{"lr": None}]))
        REF_FUNCS["update_learning_rate"](r)
        note("learning_rate_factor", abs(r.optimizer.param_groups[0]["lr"] - 5e-4 * ol.learning_rate_factor(it, 500, 30000, 0.05)), 1e-18)
        for ae in (0.0, 5000.0):
            r.anneal_end = ae
            note("cos_anneal_ratio", abs(float(REF_FUNCS["get_cos_anneal_ratio"](r)) - ol.cos_anneal_ratio(it, ae)), 0.0)

    # ---- ray generators (dataset.py:252-293, 331-342)
    ds = fake_dataset()
    pose = torch.from_numpy(ol.lookat((0.4, 0.1, 1.5), (0.0, 0.0, 0.0))).float()
    ro_ref, rv_ref = REF_FUNCS["gen_rays_pose"](ds, pose, 4)
    ro_o, rv_o = ol.pinhole_rays(pose, 64, 64)
    note("gen_rays_pose.rays_d", rel(rv_o, rv_ref), 1e-6)
    note("gen_rays_pose.rays_o", rel(ro_o, ro_ref), 0.0)
    yy, xx = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    sil = (((yy - 128) ** 2 + (xx - 120) ** 2) < 40 ** 2).astype(np.float32)
    mo, mv, Wc, dm = REF_FUNCS["gen_rays_silhouettes"](ds, pose, 12544, sil)
    o_all, v_all = ol.pinhole_rays(pose, Wc, Wc)
    note("gen_rays_silhouettes.rays_d", rel(v_all[dm], mv), 1e-6)
    note("gen_rays_silhouettes.rays_o", rel(o_all[dm], mo), 0.0)
    near_ref, far_ref = REF_FUNCS["near_far_from_sphere"](ds, mo.float(), mv.float())
    import oracle.neus as on
    near_o, far_o = on.near_far_from_sphere(mo.float(), mv.float())
    note("near_far.near", rel(near_o, near_ref), 1e-6)
    note("near_far.far", rel(far_o, far_ref), 1e-6)

    # ---- the loss stage, main.py:417-534
    snippet = cut("main.py", 417, 534, "mask_sum = mask.sum() + 1e-5", "loss += (1.0 - cosine_shading) * self.clip_weight")
    clip_state = cv.random_vit_state(seed=3)
    text = torch.randn(1, 512, generator=torch.Generator().manual_seed(11))
    golden = {"cases": []}
    # the 64 x 64 cases are also written to the golden fixture (small); all canvases are <= 224 (up-sampling / identity)
    # flags = (add_no_texture, texture_cast_light): (True, True) is confs/examples*; the 48 x 48 cases are the switches of
    # confs/ablation/*_0.conf (no shading block at all, black background), *_1.conf (the same with background
    # augmentation), *_2.conf (shading term, un-shaded texture) and the remaining combination
    T2 = (True, True)
    for (H, choice_i, seed, weights, flags) in (
            (112, 3, 1, (0.1, 0.5, 1.0), T2), (112, 1, 2, (0.1, 0.5, 1.0), T2), (224, 0, 3, (0.2, 0.0, 0.7), T2),
            (112, 2, 4, (0.1, 0.1, 1.0), T2), (64, 3, 5, (0.1, 0.5, 1.0), T2), (64, 1, 6, (0.1, 0.5, 1.0), T2),
            (64, 0, 7, (0.3, 0.0, 0.5), T2),
            (48, 3, 8, (0.1, 0.5, 1.0), (False, False)), (48, 1, 9, (0.1, 1.0, 1.0), (False, False)),
            (48, 0, 10, (0.1, 0.5, 1.0), (True, False)), (48, 3, 11, (0.1, 0.5, 0.8), (False, True))):
        ro, dilated, true_rgb, mask, bg, S = synthetic_inputs(H, seed, choice_i)
        theta, phi, np_seed = 1.2 + 0.1 * seed, 0.4 * seed, 100 + seed
        np.random.seed(np_seed)                     # replay the snippet's three draws (main.py:433, 440)
        u1, u2 = np.random.uniform(-np.pi / 4, np.pi / 4), np.random.uniform(-np.pi / 4, np.pi / 4)
        light_dir = REF_FUNCS["sphere_coord"](theta + u1, phi + u2)
        ambience = np.random.uniform(0, 0.2)
        ref = run_reference_stage(snippet, ro, dilated, true_rgb, mask, bg, choice_i, H, S, clip_state, text, theta, phi,
                                  np_seed, weights, flags)
        orc = run_oracle_stage(ro, dilated, true_rgb, mask, bg, choice_i, H, clip_state, text, light_dir, ambience, weights,
                               flags)
        for k in ("loss", "color_fine_loss", "mask_loss", "eikonal_loss", "psnr", "cosine", "cosine_shading",
                  "texture_shading", "rand_shading_rgb"):
            if k == "rand_shading_rgb" and not flags[0]:
                continue                            # computed by the reference (with cast light) but feeds no loss term
            assert (orc[k] is None) == (ref[k] is None), k
            if ref[k] is not None:
                note("stage." + k, rel(orc[k], ref[k]), 2e-6)
        for k in ref["grads"]:
            note("stage.grad." + k, rel(orc["grads"][k], ref["grads"][k]), 2e-5)
        if H <= 64:
            golden["cases"].append({"H": H, "choice_i": choice_i, "weights": weights, "flags": flags,
                                    "render_out": ro, "dilated_mask": dilated,
                                    "true_rgb": true_rgb, "mask": mask, "background_rgb": bg,
                                    "light_dir": torch.as_tensor(light_dir), "ambience": float(ambience), "clip_seed": 3,
                                    "text": text, "ref": {k: v for k, v in ref.items() if k != "grads"},
                                    "ref_grads": ref["grads"]})
        print(f"case H={H} bg={choice_i} flags={flags}: loss ref {float(ref['loss']):.6f} oracle {float(orc['loss']):.6f}")
    # ray fixture: a smaller ray budget keeps the file small (the 12 544-ray case above is asserted, not stored)
    mo2, mv2, Wc2, dm2 = REF_FUNCS["gen_rays_silhouettes"](ds, pose, 2048, sil)
    n2, f2 = REF_FUNCS["near_far_from_sphere"](ds, mo2.float(), mv2.float())
    golden["rays"] = {"pose": pose, "sil_center": (128, 120), "sil_radius": 40, "max_ray_num": 2048, "canvas": int(Wc2),
                      "dilated_mask": dm2, "rays_o": mo2.float(), "rays_d": mv2.float(), "near": n2, "far": f2}
    out = os.path.join(ROOT, "tests", "golden", "loss_stage.pt")
    torch.save(golden, out)
    print("pinned against the reference source; worst relative errors:")
    for k, v in sorted(worst.items()):
        print(f"  {k:34s} {v:.3e}")
    print("wrote", out, os.path.getsize(out) // 1024, "KB")


if __name__ == "__main__":
    main()
