"""SMPL_Dataset (avatarclip_b200/dataset.py) loading the directories the reference SHIPS (data/zero_beta_{tpose,standpose}_render:
108 PNGs + transforms_train.json each) against the reference's own constructor lines (models/dataset.py:204-250) executed in
place; the render directories and what the reference made of them are stored under tests/golden/.  Stand-ins: `imageio.imread` (not installed) -> cv2 with
BGR(A) -> RGB(A) reordering; `torch.device('cuda')` -> cpu (a device move, no arithmetic); `pose_spherical` (render_poses, unused by
the Runner) -> a stub.  Everything else -- image scaling, the W-axis flip of :222, masks, poses, focal, K, bounding box -- is the
reference's text."""
import os
import textwrap
import types

import numpy as np
import pytest
import torch

REF = os.path.join(os.environ.get("AVC_REFERENCE", ""), "AvatarGen/AppearanceGen")


class _Conf(dict):
    def get_string(self, k):
        return self[k]


def _reference_dataset(data_dir):
    import cv2 as cv
    import json
    lines = open(os.path.join(REF, "models", "dataset.py")).read().split("\n")[203:250]
    assert lines[0].strip().startswith("def __init__(self, conf)") and "Load data: End" in lines[-1]
    body = textwrap.dedent("\n".join(lines)).replace("torch.device('cuda')", "torch.device('cpu')")
    body = body.replace("super(SMPL_Dataset, self).__init__()", "pass")

    def imread(fname):
        img = cv.imread(fname, cv.IMREAD_UNCHANGED)
        return img[:, :, [2, 1, 0] + ([3] if img.shape[2] == 4 else [])]

    ns = dict(np=np, torch=torch, os=os, json=json, imageio=type("I", (), {"imread": staticmethod(imread)}),
              pose_spherical=lambda *a: torch.eye(4))
    exec(body, ns)
    obj = type("RefDataset", (), {})()
    ns["__init__"](obj, _Conf(data_dir=data_dir))
    return obj


def _digest(t):
    import hashlib
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("name", ["zero_beta_tpose_render", "zero_beta_standpose_render"])
def test_shipped_render_directory_loads_like_the_reference(name, tmp_path):
    """The render directories are stored under tests/golden/ (util_neus.reference_tree), and so is what the reference's
    constructor made of them (images and masks as sha256 digests of their bytes)."""
    from avatarclip_b200.dataset import SMPL_Dataset
    from util_neus import reference_golden, reference_tree
    data_dir = os.path.join(reference_tree(tmp_path), "data", name)

    def reference():
        d = _reference_dataset(os.path.join(REF, "data", name))
        return dict(n_images=d.n_images, H=d.H, W=d.W, focal=d.focal, image_pixels=d.image_pixels, images=_digest(d.images),
                    masks=_digest(d.masks), poses=d.poses, K=d.K, object_bbox_min=d.object_bbox_min,
                    object_bbox_max=d.object_bbox_max, images_lis=[os.path.relpath(f, REF) for f in d.images_lis])
    ref = types.SimpleNamespace(**reference_golden(f"dataset_{name}", reference))
    ours = SMPL_Dataset(_Conf(data_dir=data_dir), device="cpu")
    assert ours.n_images == ref.n_images == 108 and (ours.H, ours.W) == (ref.H, ref.W) == (256, 256)
    assert ours.focal == ref.focal and ours.image_pixels == ref.image_pixels
    assert _digest(ours.images) == ref.images and _digest(ours.masks) == ref.masks
    assert torch.equal(ours.poses, ref.poses) and torch.equal(ours.K, ref.K)
    assert np.array_equal(ours.object_bbox_min, ref.object_bbox_min) and np.array_equal(ours.object_bbox_max, ref.object_bbox_max)
    assert [os.path.relpath(f, os.path.dirname(os.path.dirname(data_dir))) for f in ours.images_lis] == ref.images_lis
    img = ours.image_at(58, 4)                                   # the validation camera of train_clip (main.py:557)
    assert img.shape == (64, 64, 3)
