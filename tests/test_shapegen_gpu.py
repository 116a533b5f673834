"""ShapeGen on the device: every kernel of avc_shape.cu against the fp64 oracle (oracle/shapegen.py) or torch on its own
inputs, the end-to-end shape_gen on the seeded inputs of tests/golden/ref_shapegen_small.pt, and the command line
from a prompt to the 108-view dataset.  Reads only tests/golden and synthetic data."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import drive as D
from oracle import shapegen as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_shapegen_small.pt")
EYE150 = (2 * math.sin(math.radians(150)), 0.0, -2 * math.cos(math.radians(150)))


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def template():
    return D.template_obj()


@pytest.fixture(scope="module")
def uv_dir(tmp_path_factory, template):
    d = tmp_path_factory.mktemp("uv")
    O.write_uv_obj(str(d), *template)
    return d


@pytest.mark.parametrize("B", [1, 2, 8])
def test_vae_decode_vs_fp64(B):
    from avatarclip_b200 import shapegen as S
    g = torch.Generator(device="cuda").manual_seed(B)
    for D_out, H in ((20670, 8192), (1001, 1028)):
        rn = lambda *s, std: torch.randn(*s, generator=g, device="cuda") * std
        z, W1, b1 = rn(B, 16, std=1.0), rn(H, 16, std=0.25), rn(H, std=0.25)
        W2, b2, vt = rn(D_out, H, std=2e-3), rn(D_out, std=1e-2), rn(D_out, std=0.5)
        out = S.vae_decode(z, W1, b1, W2, b2, vt)
        ref = (z.double() @ W1.double().T + b1.double()) @ W2.double().T + b2.double() + vt.double()
        err = ((out.double() - ref).abs().max() / ref.abs().max()).item()
        assert err <= 1e-5, (B, D_out, H, err)


def test_load_textures_vs_oracle(uv_dir):
    from avatarclip_b200 import shapegen as S
    obj = str(uv_dir / "smpl_uv.obj")
    tex = S.load_obj_textures(obj).cpu().numpy()
    ref = O.load_obj_textures(obj)
    assert tex.shape == ref.shape == (13776, 8, 8, 8, 3)
    assert np.abs(tex - ref).max() <= 1e-6
    face_uv, mats, _ = O.read_uv_obj(obj)
    bare = np.asarray(mats) == "bare"
    assert bare.any() and (tex[bare] == 1.0).all()


def _compare_raster(img, ref):
    sil, rsil = img.sum(-1) > 0, ref.sum(-1) > 0
    n = sil.size
    mismatch = (sil != rsil).mean()
    off = (np.abs(img - ref).max(-1) > 1e-4).mean()
    return mismatch, off, n


@pytest.mark.parametrize("case", ["smpl_150", "crossing_z0", "empty"])
def test_raster_textured_vs_oracle(case, template, uv_dir):
    from avatarclip_b200 import shapegen as S
    tv, tf = template
    tex_d = S.load_obj_textures(str(uv_dir / "smpl_uv.obj"))
    tex = tex_d.double().cpu().numpy()
    v = tv + np.random.default_rng(1).normal(0, 2e-3, tv.shape).astype(np.float32)
    at, eye, n = (0.0, 0.0, 0.0), EYE150, 256
    if case == "crossing_z0":       # the eye inside the body's bounding box: faces on both sides of the camera plane
        eye, at, n = (0.05, 0.2, 0.02), (0.05, 0.2, -1.0), 128
    elif case == "empty":
        eye, at, n = EYE150, (EYE150[0] * 2, 0.0, EYE150[2] * 2), 64
    img = S.raster_textured(torch.from_numpy(v).cuda(), torch.from_numpy(tf).cuda(), tex_d, eye, at, image_size=n)
    img = img.cpu().numpy()
    ref = O.raster_textured(v, tf, tex, eye, at, n=n)
    if case == "empty":
        assert not img.any() and not ref.any()
        return
    mismatch, off, _ = _compare_raster(img, ref)
    cover = (ref.sum(-1) > 0).mean()
    assert cover > 0.02, cover
    assert mismatch < 2e-3 and off < 5e-3, (case, mismatch, off)
    if case == "crossing_z0":
        cam = (np.asarray(v, np.float64) - eye) @ O.look_at_camera(eye, at)[1]
        assert (cam[:, 2] <= 0).any() and (cam[:, 2] > 0).any()


def test_raster_textured_analytic_constant_colour():
    """A +y facing triangle with a constant texture is fully lit: the kernel's inner pixels equal the colour."""
    from avatarclip_b200 import shapegen as S
    v = torch.tensor([[-0.6, 0.0, -0.6], [0.6, 0.0, -0.6], [0.0, 0.0, 0.6]], device="cuda")
    colour = torch.tensor([0.8, 0.4, 0.2], device="cuda")
    tex = colour.expand(1, 8, 8, 8, 3).contiguous()
    img = S.raster_textured(v, torch.tensor([[0, 1, 2]], device="cuda"), tex, (1.0, 1.2, 1.6), image_size=64)
    hit = img[img.sum(-1) > 0]
    assert hit.shape[0] > 40
    inner = (hit - colour).abs().max(-1).values <= 1e-6
    assert inner.float().mean() > 0.6 and (hit <= colour + 1e-6).all()


def test_clip_prep_nearest_vs_torch():
    from avatarclip_b200 import shapegen as S
    img = torch.rand(2, 3, 256, 256, device="cuda")
    out = S.clip_prep_nearest(img.permute(0, 2, 3, 1))
    ref = F.interpolate(img, size=224)
    ref -= torch.from_numpy(np.array([0.48145466, 0.4578275, 0.40821073])).reshape(1, 3, 1, 1).cuda()
    ref /= torch.from_numpy(np.array([0.26862954, 0.26130258, 0.27577711])).reshape(1, 3, 1, 1).cuda()
    assert (out - ref).abs().max().item() <= 1e-6
    odd = torch.rand(1, 3, 97, 97, device="cuda")
    ref = (F.interpolate(odd, size=224).double() - torch.tensor(O.CLIP_MEAN, device="cuda").view(1, 3, 1, 1).double())
    ref = ref.float().double() / torch.tensor(O.CLIP_STD, device="cuda").view(1, 3, 1, 1).double()
    assert (S.clip_prep_nearest(odd.permute(0, 2, 3, 1)).double() - ref).abs().max().item() <= 1e-6


def test_codebook_argmax_vs_fp64_and_first_index_on_ties():
    from avatarclip_b200 import shapegen as S
    g = torch.Generator(device="cuda").manual_seed(0)
    N, Dm = 1000, 512
    Cb = torch.randn(N, Dm, generator=g, device="cuda")
    e = torch.randn(Dm, generator=g, device="cuda")
    d = torch.randn(Dm, generator=g, device="cuda")
    cos, best = S.codebook_argmax(Cb, e, d)
    ref = O.codebook_cos(Cb.cpu(), e.cpu(), d.cpu())
    assert np.abs(cos.cpu().numpy() - ref).max() <= 1e-6 and best == int(np.argmax(ref))
    # a constructed tie: rows 300 and 700 hold the same best entry -> the first one wins
    Cb[300] = Cb[700] = e + 3.0 * d
    cos, best = S.codebook_argmax(Cb, e, d)
    assert best == 300 and cos[300].item() == cos[700].item()
    # the upstream expression agrees
    up = (F.normalize(Cb - e, dim=1) * F.normalize(d.reshape(-1), dim=0)).sum(-1)
    assert int(up.argmax()) == 300 and (up - cos).abs().max().item() <= 1e-6
    # a zero row (C_i == e): F.normalize's clamp gives cos 0
    Cb[5] = e
    cos, _ = S.codebook_argmax(Cb, e, d)
    assert cos[5].item() == 0.0


def _clip_models(tmp_path):
    from avatarclip_b200 import shapegen as S
    return S.load_clip(O.clip_states(), O.write_bpe(tmp_path / "bpe.txt.gz"))


def test_shape_gen_end_to_end_on_the_golden_inputs(golden, template, uv_dir, tmp_path):
    from avatarclip_b200 import shapegen as S
    tv, tf = template
    torch.save({golden["codebook_latents"]: golden["codebook_emb"]}, tmp_path / "codebook.pth")
    smpl = {"v_template": tv, "faces": tf}
    r = S.run_shape_gen(smpl, O.vae_state(tv), str(tmp_path / "codebook.pth"), golden["neutral_txt"],
                        golden["target_txt"], _clip_models(tmp_path), str(uv_dir / "smpl_uv.obj"))
    assert r.best == golden["best"]
    cos = r.cos.cpu().numpy()
    top = np.sort(cos)[::-1]
    assert top[0] - top[1] >= 0.05
    assert np.abs(cos - golden["cos"].numpy()).max() < 0.02          # fp16 towers against the fp32 oracle towers
    assert np.abs(r.v - golden["v"].numpy()).max() <= 1e-5
    assert np.abs(r.zero_beta_v - golden["zero_beta_v"].numpy()).max() <= 1e-5
    img = r.neutral_image[0].permute(1, 2, 0).cpu().numpy()
    mismatch, off, _ = _compare_raster(img, golden["neutral_image"].float().permute(1, 2, 0).numpy())
    assert mismatch < 2e-3 and (np.abs(img - golden["neutral_image"].float().permute(1, 2, 0).numpy()).max(-1) > 1e-3).mean() < 5e-3


def test_cli_prompt_to_obj_and_dataset(tmp_path):
    """The CLI on a small synthetic body: the OBJ reads back, --render_folder writes the 108 views that
    SMPL_Dataset loads."""
    from avatarclip_b200 import shapegen as S
    from avatarclip_b200.dataset import SMPL_Dataset
    from avatarclip_b200.workload import synthetic_body_mesh
    from oracle import lbs as olbs
    bv, bf = synthetic_body_mesh(12, 16)
    V = bv.shape[0]
    sm = {k: v.numpy() for k, v in olbs.synthetic_smpl(V=V, seed=4).items() if k in D.SMPL_KEYS}
    sm["v_template"] = bv
    np.savez(tmp_path / "smpl.npz", faces=bf, **sm)
    vae = O.vae_state(bv)
    torch.save(vae, tmp_path / "vae.pth")
    lat = torch.randn(6, 16, generator=torch.Generator().manual_seed(0))
    torch.save({lat: torch.randn(6, 512, generator=torch.Generator().manual_seed(1))}, tmp_path / "codebook.pth")
    visual, text = O.clip_states()
    torch.save({**{k: v.half() for k, v in visual.items()}, **{k: v.half() for k, v in text.items()}},
               tmp_path / "clip.pt")
    uv = O.write_uv_obj(str(tmp_path / "uv"), bv, bf)
    np.save(tmp_path / "stand.npy", np.zeros((1, 72), np.float32))
    out, render = tmp_path / "out", tmp_path / "render"
    rc = S.main(["--AE_path_fname", str(tmp_path / "vae.pth"), "--codebook_fname", str(tmp_path / "codebook.pth"),
                 "--smpl", str(tmp_path / "smpl.npz"), "--uv_obj", uv, "--clip_model", str(tmp_path / "clip.pt"),
                 "--bpe", O.write_bpe(tmp_path / "bpe.txt.gz"), "--target_txt", "a big man", "--output_folder",
                 str(out), "--render_folder", str(render), "--stand_pose", str(tmp_path / "stand.npy")])
    assert rc == 0
    V_, F_, _, _ = S.readOBJ(str(out / "a_big_man.obj"))
    assert V_.shape == (V, 3) and np.array_equal(np.asarray(F_), bf)
    decoded = O.vae_decode(lat, vae["dec1.weight"], vae["dec1.bias"], vae["dec2.weight"], vae["dec2.bias"], bv)
    assert min(np.abs(decoded[i].reshape(-1, 3) - V_).max() for i in range(6)) <= 1e-5
    meta = json.load(open(render / "transforms_train.json"))
    assert len(meta["frames"]) == 108 and len(os.listdir(render / "img")) == 108
    ds = SMPL_Dataset({"data_dir": str(render)})
    assert ds.n_images == 108 and float(ds.masks.mean()) > 0.01


def test_error_codes_and_cpu_tensors():
    from avatarclip_b200 import _lib, shapegen as S
    L = S._L()
    sz = C.c_size_t()
    st = _lib.stream_ptr()
    buf = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    p = _lib.ptr(buf)
    assert L.avc_vae_decode_workspace_bytes(9, 8192, C.byref(sz)) == -3
    assert L.avc_vae_decode_workspace_bytes(1, 8190, C.byref(sz)) == -3
    assert L.avc_vae_decode_workspace_bytes(1, 8192, None) == -2
    assert L.avc_vae_decode(None, 1, 16, p, p, 8192, p, p, p, 100, p, p, buf.numel(), st) == -2
    assert L.avc_vae_decode(p, 1, 16, p, p, 8192, p, p, p, 100, p, p, 16, st) == -3
    assert L.avc_load_textures(p, 4, 4, p, p, 1, 1, p, st) == -3
    assert L.avc_load_textures(None, 4, 4, p, p, 1, 8, p, st) == -2
    assert L.avc_raster_textured_workspace_bytes(10, 64, 5, C.byref(sz)) == -3
    e = C.cast((C.c_float * 3)(0.0, 0.0, 2.0), C.c_void_p)
    up = C.cast((C.c_float * 3)(0.0, 1.0, 0.0), C.c_void_p)
    assert L.avc_raster_textured(p, p, p, 3, 1, 8, e, e, up, 16, 2, p, p, buf.numel(), st) == -1     # eye == at
    assert L.avc_raster_textured(p, p, p, 3, 1, 8, e, None, up, 16, 2, p, p, buf.numel(), st) == -2
    assert L.avc_clip_prep_nearest(p, 0, 8, 224, p, st) == -3
    assert L.avc_codebook_argmax(p, p, p, 4, 8, p, p, p, 4, st) == -3
    assert L.avc_codebook_argmax(p, p, None, 4, 8, p, p, p, 8, st) == -2
    with pytest.raises(_lib.AvcError):
        S.vae_decode(torch.zeros(1, 16), torch.zeros(8, 16), torch.zeros(8), torch.zeros(4, 8), torch.zeros(4),
                     torch.zeros(4))
    with pytest.raises(_lib.AvcError):
        S.raster_textured(torch.zeros(3, 3), torch.zeros(1, 3, dtype=torch.int32), torch.ones(1, 8, 8, 8, 3),
                          (0, 0, 2))
    with pytest.raises(_lib.AvcError):
        S.codebook_argmax(torch.zeros(4, 8, device="cuda"), torch.zeros(8), torch.ones(8, device="cuda"))
    with pytest.raises(_lib.AvcError):
        S.load_textures(torch.zeros(4, 4, 3), torch.zeros(1, 3, 2), torch.ones(1), torch.ones(1, 8, 8, 8, 3))
    torch.cuda.synchronize()
