"""VPoserOptimizer without a device: which confs the command runs and how it refuses the rest, the fp64 autograd
restatement of VPoser's decode (oracle/vposer_optimizer.py) against the numpy decode and central differences on every
branch of matrot2aa, and the reference's own loop as tests/golden/ref_vposer_optimizer_small.pt recorded it."""
import glob
import os
import tarfile

import numpy as np
import pytest
import torch

from oracle import animate as O
from oracle import vposer_optimizer as OV

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def confs(tmp_path_factory):
    d = tmp_path_factory.mktemp("vposer_optimizer_confs")
    with tarfile.open(os.path.join(GOLDEN, "ref_animate_confs.tar.gz")) as tf:
        tf.extractall(d, filter="data")
    return sorted(glob.glob(str(d / "confs" / "**" / "*.conf"), recursive=True))


def test_conf_classification(confs):
    """Of the 85 shipped confs the command runs exactly the 12 vposer_optimizer ones, and names the command that runs
    each of the others."""
    from avatarclip_b200 import conf
    from avatarclip_b200 import vposer_optimizer as VO
    assert len(confs) == 85
    runs, refused = [], []
    for p in confs:
        c = conf.parse_file(p)
        why = VO.refusal(c)
        (runs if why is None else refused).append((p, c, why))
    assert len(runs) == 12 and all("/pose_ablation/vposer_optimizer/" in p for p, _, _ in runs)
    po = [w for p, _, w in refused if "/pose_ablation/pose_optimizer/" in p]
    assert len(po) == 12 and all("avatarclip_b200.pose_optimizer" in w for w in po)
    gen = [w for p, c, w in refused if c["pose_generator"]["type"] in ("VPoserCodebook", "VPoserRealNVP")
           and c.get_string("general.mode") == "pose"]
    assert len(gen) == 24 and all("avatarclip_b200.animate" in w for w in gen)
    mot = [(c, w) for p, c, w in refused if c.get_string("general.mode") == "motion"]
    assert len(mot) == 37
    from avatarclip_b200 import motion, motion_clip
    for c, w in mot:            # the motion command that runs the conf (motion when neither does)
        clip_only = motion.refusal(c) is not None and motion_clip.refusal(c) is None
        assert w.endswith("avatarclip_b200.motion_clip" if clip_only else "avatarclip_b200.motion")
    assert any(w.endswith("motion_clip") for _, w in mot) and any(w.endswith(".motion") for _, w in mot)


def test_cli_refuses_before_reading_files(confs, capsys):
    """Every refusal exits non-zero with its reason, although --smpl names no file; a runnable conf reaches the file
    checks."""
    from avatarclip_b200 import conf
    from avatarclip_b200 import vposer_optimizer as VO
    for p in confs:
        why = VO.refusal(conf.parse_file(p))
        with pytest.raises(SystemExit) as e:
            VO.parse_args(["--conf", p, "--smpl", "/nonexistent.npz"])
        err = capsys.readouterr().err
        assert e.value.code != 0
        assert (why in " ".join(err.split())) if why else ("--smpl: no such file" in err)


def test_vposer_path_from_the_conf(tmp_path, capsys):
    """Without --vposer the conf's pose_generator.vposer_path is used, and a missing one is reported by that path."""
    from avatarclip_b200 import vposer_optimizer as VO
    files = {}
    for k in ("smpl", "uv_obj", "clip_model", "bpe"):
        files[k] = tmp_path / k
        files[k].write_bytes(b"")
    c = tmp_path / "c.conf"
    c.write_text("general {\n    base_exp_dir = ./x\n    mode = pose\n    text = a man\n}\n"
                 f"pose_generator {{\n    type = VPoserOptimizer\n    vposer_path = {tmp_path}/nowhere\n}}\n")
    args = ["--conf", str(c)] + [x for k, p in files.items() for x in (f"--{k}", str(p))]
    with pytest.raises(SystemExit):
        VO.parse_args(args)
    assert f"--vposer: no such directory or file: {tmp_path}/nowhere" in capsys.readouterr().err
    (tmp_path / "vp").mkdir()
    a, _, pg = VO.parse_args(args + ["--vposer", str(tmp_path / "vp")])
    assert a.vposer == str(tmp_path / "vp") and "vposer_path" not in pg and "type" not in pg


def test_adam_refusals(tmp_path, capsys):
    from avatarclip_b200 import vposer_optimizer as VO
    c = tmp_path / "c.conf"
    c.write_text("general {\n    base_exp_dir = ./x\n    mode = pose\n    text = a man\n}\n"
                 "pose_generator {\n    type = VPoserOptimizer\n    optim_name = SGD\n}\n")
    with pytest.raises(SystemExit) as e:
        VO.parse_args(["--conf", str(c), "--smpl", "/nonexistent.npz"])
    assert e.value.code != 0 and "VPoserOptimizer optim_name = SGD" in capsys.readouterr().err
    with pytest.raises(NotImplementedError, match="VPoserOptimizer optim_name = SGD"):
        VO.VPoserOptimizer(optim_name="SGD", name="VPoserOptimizer", assets=None)


def test_other_commands_name_this_one(confs):
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import conf
    from avatarclip_b200 import pose_optimizer as PO
    c = conf.parse_file([p for p in confs if "/pose_ablation/vposer_optimizer/" in p][0])
    assert "avatarclip_b200.vposer_optimizer" in A.refusal(c)
    assert "avatarclip_b200.vposer_optimizer" in PO.refusal(c)


# ---------------------------------------------------------------- the fp64 restatement
def test_restatement_forward_equals_the_numpy_decode():
    for sd in (O.vposer_state(), OV.steered_state()):
        z = torch.randn(9, 32, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
        pose, _ = O.vposer_decode(z.numpy(), sd)
        assert np.abs(OV.decode(z, sd).numpy() - pose).max() <= 1e-12


def test_restatement_gradient_vs_central_differences():
    """Autograd of the masked restatement against central differences in fp64, on latents whose joints take all four
    quaternion branches and both atan2 branches (oracle.vposer_optimizer.steered_state)."""
    sd = {k: v.double() for k, v in OV.steered_state().items()}
    z = torch.randn(3, 32, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    R = OV.decoder_rotations(z, sd)
    assert set(OV.branches(R).tolist()) == {0, 1, 2, 3}
    assert set(OV.atan2_negative(R).tolist()) == {False, True}
    g = torch.randn(3, 21, 3, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    zz = z.clone().requires_grad_(True)
    (OV.decode(zz, sd) * g).sum().backward()
    f = lambda x: float((OV.decode(x, sd) * g).sum())
    h = 1e-6
    num = torch.zeros_like(z)
    for b in range(3):
        for k in range(32):
            e = torch.zeros_like(z)
            e[b, k] = h
            num[b, k] = (f(z + e) - f(z - e)) / (2 * h)
    assert float((zz.grad - num).abs().max()) <= 1e-7 * float(num.abs().max())


# ---------------------------------------------------------------- the reference's loop (oracle/pin_vposer_optimizer.py)
@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "ref_vposer_optimizer_small.pt"), map_location="cpu", weights_only=False)


def test_loop_against_the_reference(golden):
    """What the reference's own VPoserOptimizer did: the torch.randn(32) draws in order, the numpy elevations
    (candidate k's num_iteration x 5 before candidate k + 1's, then the sort's), torch Adam at lr 0.01 on the recorded
    gradients reproducing the recorded latents, and a returned pose that is the decode of the latent *before* the last
    step, padded and sorted by the recorded scores."""
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import motion as M
    K, T = golden["conf"]["topk"], golden["conf"]["num_iteration"]
    torch.manual_seed(golden["torch_seed"])
    assert torch.equal(torch.stack([torch.randn(32) for _ in range(K)]), golden["init"])
    np.random.seed(golden["np_seed"])
    eyes = A.PoseScorer(None).draw_eyes(K * T + K)
    np.testing.assert_allclose(eyes, golden["eyes"].double().numpy(), rtol=0, atol=1e-6)
    for k in range(K):
        p = torch.nn.Parameter(golden["init"][k].clone())
        opt = torch.optim.Adam([p], lr=0.01)
        for t in range(T):
            assert torch.equal(p.data, golden["latents"][k, t])
            p.grad = golden["grads"][k, t].clone()
            opt.step()
        assert not torch.equal(p.data, golden["latents"][k, T - 1])      # the last step moved the latent ...
    before = OV.decode(golden["latents"][:, T - 1].double(), O.vposer_state()).reshape(K, 63).float()
    assert torch.equal(before, golden["poses"])                          # ... but the output is the decode before it
    sc = golden["sort_scores"].tolist()
    order = sorted(range(K), key=lambda i: sc[i], reverse=True)
    np.testing.assert_array_equal(golden["files"].numpy(), M.pose_padding(before[order]).numpy())
    assert golden["files"].shape == (K, 69) and (golden["files"][:, 63:] == 0).all()
    assert (golden["loss"] > 0).all() and float(golden["grads"].abs().max()) > 0
