"""The three SMPL posing paths share one kinematic core (avatarclip_b200/csrc/avc_smpl.cuh): ``avc_lbs_fwd`` (my_lbs),
``avc_smpl_pose_batch`` (AvatarAnimate's poses) and ``avc_lbs_rel_transforms`` followed by ``avc_lbs_frames`` (drive,
export, video).  With the pose blend shapes zeroed, all three skin the bare template, so they must agree bit for bit."""
import pytest
import torch

from oracle import drive as D

pytestmark = pytest.mark.gpu

B = 37   # rows: several 8-row skinning tiles and a ragged last one, several 4-row chain CTAs


@pytest.fixture(scope="module")
def smpl():
    from avatarclip_b200 import drive
    s = drive.smpl_tensors(D.golden_smpl())
    s["posedirs"] = torch.zeros_like(s["posedirs"])
    return s


def _axis_angle(seed: int) -> torch.Tensor:
    """[B, 24, 3] axis-angle poses, components in [-1.5, 1.5]; row 0 is the zero pose (angle = |eps|)."""
    g = torch.Generator().manual_seed(seed)
    p = (torch.rand(B, 24, 3, generator=g) * 2 - 1) * 1.5
    p[0] = 0
    return p


def _lbs_rows(s, pose, pose2rot):
    from avatarclip_b200.lbs import my_lbs
    return torch.cat([my_lbs(s["v_template"][None], row.reshape(1, -1).cuda(), None, None, s["posedirs"],
                             s["J_regressor"], s["parents"], s["lbs_weights"], pose2rot=pose2rot)[0] for row in pose])


def _drive_frames(s, pose, pose2rot):
    from avatarclip_b200 import drive
    A = drive._rel_transforms(s, pose.cuda().contiguous(), pose2rot)
    out = torch.empty(pose.shape[0], s["v_template"].shape[0], 3, device="cuda")
    return drive._lbs_frames(s["v_template"], None, s["lbs_weights"], A, 0, pose.shape[0], out)


@pytest.mark.parametrize("P", [69, 63])
@pytest.mark.parametrize("orient", ["score", "drawn"])
def test_axis_angle_paths_equal(smpl, P, orient):
    from avatarclip_b200 import animate
    pose = _axis_angle(3 if orient == "score" else 4)
    go = torch.tensor(animate.SCORE_ORIENT) if orient == "score" else pose[1, 0].clone()
    pose[:, 0] = go
    pose.view(B, -1)[:, 3 + P:] = 0      # smpl_pose_batch zero-pads body_pose past P
    ref = _lbs_rows(smpl, pose, True)
    batch = animate.smpl_pose_batch(smpl, pose.view(B, -1)[:, 3:3 + P].contiguous().cuda(), global_orient=go)
    frames = _drive_frames(smpl, pose, True)
    torch.cuda.synchronize()
    assert torch.isfinite(ref).all() and ref.abs().max() > 0
    assert torch.equal(batch, ref)
    assert torch.equal(frames, ref)


def test_rotation_matrix_paths_equal(smpl):
    from avatarclip_b200 import drive
    pose = _axis_angle(5)
    rot = drive.batch_rodrigues(pose.reshape(-1, 3)).reshape(B, 24, 9).contiguous()
    ref = _lbs_rows(smpl, rot, False)
    frames = _drive_frames(smpl, rot, False)
    torch.cuda.synchronize()
    assert torch.isfinite(ref).all() and ref.abs().max() > 0
    assert torch.equal(frames, ref)
    assert not torch.equal(ref[1], ref[2])
