"""AvatarAnimate's motion stage on the device: avc_vposer_encode, avc_motion_decode and avc_motion_optimize against fp64
(oracle/motion.py), the optimiser's trajectory against what the reference computed (tests/golden/ref_motion_small.pt),
and the command line on synthetic files.  Reads only tests/golden and synthetic data."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import animate as OA
from oracle import drive as D
from oracle import motion as OM
from oracle import shapegen as OS

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_motion_small.pt")


def _err(out, ref):
    ref = torch.as_tensor(ref, dtype=torch.float64)
    return float((torch.as_tensor(out).detach().cpu().double() - ref).abs().max() / ref.abs().max())


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def vae():
    from avatarclip_b200 import motion as M
    return M.load_motion_vae(OM.motion_vae_state())


@pytest.mark.parametrize("B", [1, 5, 37])
def test_vposer_encode_vs_fp64(B):
    from avatarclip_b200 import motion as M
    sd = OM.vposer_encoder_state()
    x = torch.randn(B, 63, generator=torch.Generator().manual_seed(B)) * 0.4
    got = M.vposer_encode(x.cuda(), {k: v.cuda() for k, v in sd.items()})
    ref = OM.vposer_encode(x, sd)
    twin = _err(OM.vposer_encode(x, sd, dtype=torch.float32), ref)
    assert got.shape == (B, 32) and _err(got, ref) <= max(4 * twin, 2e-6)


def test_motion_decode_vs_fp64(vae, golden):
    from avatarclip_b200 import motion as M
    sd = OM.motion_vae_state()
    z = golden["optimizer"]["delta0"]["latent_init"]
    got = M.motion_decode(z.cuda(), vae)
    ref = OM.decode(z.double(), sd)
    twin = _err(OM.decode(z.float(), sd, pe=OM.positional_table(60, 256).float()), ref)
    print(f"decode: device {_err(got, ref):.2e}, fp32 twin {twin:.2e}")
    assert got.shape == (60, 63) and _err(got, ref) <= max(4 * twin, 2e-6)


# rotations whose 6D forms take matrix_to_quaternion's four argmax branches, one near pi, one below the small-angle
# threshold (its decoder rows are zero so that it stays there)
BRANCH_ROTVECS = [[0.3, -0.2, 0.1], [math.pi * 0.9, 0.1, 0.0], [0.1, math.pi * 0.9, 0.0], [0.0, 0.2, math.pi * 0.9],
                  [math.pi - 0.01, 0.0, 0.0], [0.0, 0.0, 0.0], [1.2, -0.6, 0.4], [-0.5, 1.1, -0.9]]


def _branch_state():
    from scipy.spatial.transform import Rotation
    D, L = 64, 2
    sd = OM.motion_vae_state(seed=5, latent=D, num_layers=L, n_out=132)
    six = np.stack([Rotation.from_rotvec(v).as_matrix()[:2].reshape(6) for v in BRANCH_ROTVECS])
    bias = np.tile(six, (3, 1))[:22]
    W = sd["decoder.final.weight"] * 0.05
    W[5 * 6:6 * 6] = 0                    # decoder joint 5 (motion joint 4): the identity rotation, exactly
    sd["decoder.final.weight"], sd["decoder.final.bias"] = W, torch.from_numpy(bias.reshape(-1)).float()
    return sd, D, L


def test_rotation_chain_every_branch_vs_fp64():
    """Forward and latent gradient of a small decoder whose outputs sit on every branch of the chain, against fp64
    autograd."""
    from avatarclip_b200 import motion as M
    sd, D, L = _branch_state()
    w = M.load_motion_vae(sd, latent_dim=D, num_layers=L, num_heads=2)
    z = torch.randn(D, generator=torch.Generator().manual_seed(1))
    out = OM.decoder(z.double(), sd, num_layers=L, num_heads=2).reshape(60, 22, 6)[:, 1:]
    m = OM.rotation_6d_to_matrix(out)
    e = [m[..., i, j] for i in range(3) for j in range(3)]
    qa = torch.stack([1 + e[0] + e[4] + e[8], 1 + e[0] - e[4] - e[8], 1 - e[0] + e[4] - e[8], 1 - e[0] - e[4] + e[8]], -1)
    assert set(qa.argmax(-1).flatten().tolist()) == {0, 1, 2, 3}
    aa = OM.rot6d_to_aa(out)
    assert float(aa.norm(dim=-1).max()) > math.pi - 0.05 and float(aa.norm(dim=-1).min()) < 1e-6
    got = M.motion_decode(z.cuda(), w)
    assert _err(got, aa.reshape(60, 63)) <= 2e-5
    poses = aa.reshape(60, 63)[[3, 17, 31, 44, 58]].float() + 0.05 * torch.randn(5, 63, generator=torch.Generator()
                                                                                     .manual_seed(2))
    zz = z.double().requires_grad_()
    OM.loss(OM.decode(zz, sd, num_layers=L, num_heads=2), poses.double(), [1, 0.8, 0.6, 0.4, 0.2], 0.01).backward()
    _, _, _, g = M.motion_optimize(w, poses.cuda(), [1, 0.8, 0.6, 0.4, 0.2], 0.01, z.cuda(), 1, return_grad=True)
    print(f"branch gradient err {_err(g, zz.grad):.2e}")
    assert _err(g, zz.grad) <= 1e-4


@pytest.mark.parametrize("delta_coef", [0.0, 0.01])
def test_one_iteration_gradient_vs_fp64(vae, golden, delta_coef):
    from avatarclip_b200 import motion as M
    z0, poses = golden["optimizer"]["delta"]["latent_init"], golden["poses"]
    coef = [1, 0.8, 0.6, 0.4, 0.2]
    z = z0.double().requires_grad_()
    lo = OM.loss(OM.decode(z, OM.motion_vae_state()), poses.double(), coef, delta_coef)
    lo.backward()
    _, _, loss, g = M.motion_optimize(vae, poses.cuda(), coef, delta_coef, z0.cuda(), 1, record_loss=True,
                                      return_grad=True)
    print(f"one-iteration gradient err {_err(g, z.grad):.2e}, loss {float(loss[0]):.6f} vs {float(lo.detach()):.6f}")
    assert _err(g, z.grad) <= 1e-4 and abs(float(loss[0]) - float(lo.detach())) <= 1e-5 * abs(float(lo.detach()))


@pytest.mark.parametrize("run", ["delta0", "delta"])
def test_trajectory_vs_reference(vae, golden, run):
    """Over the pinned iterations the device's losses follow the reference's.  The bar is 20 times the oracle's own
    fp32-vs-fp64 divergence over the same iterations (relative to the largest loss), at least 1e-5."""
    from avatarclip_b200 import motion as M
    r, c = golden["optimizer"][run], golden["optimizer_conf"][run]
    n = golden["num_iter"]
    l64, _, _ = OM.optimize(OM.motion_vae_state(), golden["poses"], r["latent_init"], n, c["recon_coef"],
                            c["delta_coef"])
    l32, _, _ = OM.optimize(OM.motion_vae_state(), golden["poses"], r["latent_init"], n, c["recon_coef"],
                            c["delta_coef"], dtype=torch.float32)
    bar = max(20 * _err(l32, l64), 1e-5)
    z, motion, loss = M.motion_optimize(vae, golden["poses"].cuda(), c["recon_coef"], c["delta_coef"],
                                        r["latent_init"].cuda(), n, lr=c["lr"], record_loss=True)
    e = _err(loss, r["loss"])
    print(f"{run}: loss err {e:.2e} (bar {bar:.2e}), latent {_err(z, r['latent']):.2e}, "
          f"motion {_err(motion, r['motion'][:, :63]):.2e}")
    assert e <= bar
    assert _err(z, r["latent"]) <= 1e-3 and _err(motion, r["motion"][:, :63]) <= 1e-3


def test_long_run_stays_finite_and_near_the_oracle(vae, golden):
    """The shipped 5000 iterations (baseline conf) stay finite; the final loss is within 5% of the oracle's fp32 CPU
    run from the same latent."""
    from avatarclip_b200 import motion as M
    r = golden["optimizer"]["delta0"]
    n = golden["long_iter"]
    z, motion, loss = M.motion_optimize(vae, golden["poses"].cuda(), [1.0] * 5, 0.0, r["latent_init"].cuda(), n,
                                        lr=0.01, record_loss=True)
    ref = golden["oracle_fp32_long_loss"]
    print(f"{n} iterations: final loss {float(loss[-1]):.6f}, oracle fp32 {float(ref[-1]):.6f}")
    assert torch.isfinite(loss).all() and torch.isfinite(motion).all() and torch.isfinite(z).all()
    assert abs(float(loss[-1]) - float(ref[-1])) <= 0.05 * float(ref[-1])


def test_determinism(vae, golden):
    from avatarclip_b200 import motion as M
    r = golden["optimizer"]["delta"]
    a = M.motion_optimize(vae, golden["poses"].cuda(), [1, 0.8, 0.6, 0.4, 0.2], 0.01, r["latent_init"].cuda(), 30)
    b = M.motion_optimize(vae, golden["poses"].cuda(), [1, 0.8, 0.6, 0.4, 0.2], 0.01, r["latent_init"].cuda(), 30)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(M.motion_decode(a[0], vae), M.motion_decode(a[0], vae))


def test_interpolation_vs_golden(golden):
    from avatarclip_b200 import motion as M
    vp = {k: v.cuda() for k, v in {**OA.vposer_state(), **OM.vposer_encoder_state()}.items()}
    got = M.MotionInterpolation(vposer=vp).get_motion("", golden["poses"].cuda())
    assert got.shape == (60, 69) and _err(got, golden["interpolation"]) <= 1e-5
    with pytest.raises(ValueError, match="anchors"):
        M.MotionInterpolation(vposer=vp).get_motion("", golden["poses"][:3].cuda())


@pytest.mark.parametrize("kind", ["MotionInterpolation", "MotionOptimizer"])
def test_cli_writes_motion(tmp_path, monkeypatch, kind):
    from avatarclip_b200 import motion as M
    tv, tf = D.template_obj()
    smpl = {k: np.asarray(v) for k, v in D.golden_smpl().items()}
    smpl["faces"] = tf
    np.savez(tmp_path / "smpl.npz", **smpl)
    os.makedirs(tmp_path / "vposer" / "snapshots")
    torch.save({"state_dict": {"vp_model." + k: v for k, v in {**OA.vposer_state(), **OM.vposer_encoder_state()}.items()}},
               tmp_path / "vposer" / "snapshots" / "V02_05_epoch=13_val_loss=0.03.ckpt")
    visual, text = OS.clip_states()
    torch.save({**{k: v.half() for k, v in visual.items()}, **{k: v.half() for k, v in text.items()}},
               tmp_path / "clip.pt")
    uv = OS.write_uv_obj(str(tmp_path / "data"), smpl["v_template"], smpl["faces"])
    torch.save(OA.make_codebook(torch.randn(512, generator=torch.Generator().manual_seed(0))),
               tmp_path / "data" / "codebook.pth")
    torch.save({"state_dict": OM.motion_vae_state()}, tmp_path / "data" / "motion_vae.pth")
    block = "type = MotionInterpolation" if kind == "MotionInterpolation" else \
        "type = MotionOptimizer\n    num_iteration = 20\n    clip_coef = 0.0\n    delta_coef = 0.0"
    (tmp_path / "m.conf").write_text("general {\n    base_exp_dir = ./exp/m\n    mode = motion\n    text = a rendered 3d "
                                     "man is walking\n}\n\npose_generator {\n    type = VPoserCodebook\n}\n\n"
                                     f"motion_generator {{\n    {block}\n}}\n")
    monkeypatch.chdir(tmp_path)
    rc = M.main(["--conf", "m.conf", "--smpl", "smpl.npz", "--vposer", "vposer", "--uv_obj", uv, "--clip_model",
                 "clip.pt", "--bpe", OS.write_bpe(tmp_path / "bpe.txt.gz"), "--seed", "0"])
    assert rc == 0
    out = tmp_path / "exp" / "m"
    import cv2
    for i in range(5):
        assert np.load(out / f"candidate_{i}.npy").shape == (63,) and (out / f"candidate_{i}.jpg").exists()
    m = np.load(out / "motion.npy")
    assert m.shape == (60, 69) and m.dtype == np.float32 and np.isfinite(m).all() and not m[:, 63:].any()
    cap = cv2.VideoCapture(str(out / "motion.mp4"))
    frames = []
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        frames.append(fr)
    cap.release()
    assert len(frames) == 60 and frames[0].shape == (512, 512, 3)
    assert any((f < 200).any(axis=-1).mean() > 0.005 for f in frames)
