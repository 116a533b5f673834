"""CPU oracle (test infrastructure, never on the product path): AvatarGen/AppearanceGen/drive.py's generate_animation
(:308-361) restated step by step on numpy / torch CPU, with the LBS pieces of oracle/lbs.py.

The island search of ``cleanup_mesh`` (:172-210) is restated as connected components of the triangle-edge graph
(scipy) with the reference's choice rule: the largest island by vertex count, and among equal sizes the one the
reference's scan in vertex order finds first, i.e. the one with the smallest vertex index.  ``find_nearest_ind``
(:235-240) is the reference's float64 expression, evaluated in chunks of query points so that it fits in memory.

o3d SEMANTICS UNPINNED: open3d is not installable here, so what ``TriangleMesh.remove_vertices_by_index`` keeps (the
surviving vertices in order with their colours, the triangles whose three corners survive, re-indexed) is restated
from its documentation, both here and in the stand-in oracle/pin_drive.py runs drive.py with.
"""
from __future__ import annotations

import io
import os
import struct
import tarfile

import numpy as np
import torch

from oracle import lbs as olbs

ROT = np.array([[1, 0, 0], [0, 0, 1], [0, -1, 0]], dtype=np.float32)     # drive.py:318-323
SMPL_KEYS = ("v_template", "posedirs", "J_regressor", "parents", "lbs_weights")
_GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def template_obj():
    """The SMPL template shipped with the reference (data/zero_beta_smpl.obj, stored in
    tests/golden/ref_tree_template.tar.gz): vertices [6890,3] float32, faces [13776,3] int32."""
    with tarfile.open(os.path.join(_GOLDEN, "ref_tree_template.tar.gz")) as tf:
        text = tf.extractfile("data/zero_beta_smpl.obj").read().decode()
    vs, fs = [], []
    for line in io.StringIO(text):
        if line.startswith("v "):
            vs.append([float(t) for t in line.split()[1:4]])
        elif line.startswith("f "):
            idx = [int(t.split("/")[0]) - 1 for t in line.split()[1:]]
            fs += [[idx[0], idx[k], idx[k + 1]] for k in range(1, len(idx) - 1)]
    return np.asarray(vs, dtype=np.float32), np.asarray(fs, dtype=np.int32)


def golden_smpl(seed: int = 11) -> dict:
    """synthetic_smpl tensors (SMPL-shaped, random) with the real template as v_template."""
    tv, _ = template_obj()
    d = olbs.synthetic_smpl(V=tv.shape[0], seed=seed)
    return dict(v_template=torch.from_numpy(tv), posedirs=d["posedirs"], J_regressor=d["J_regressor"],
                parents=d["parents"], lbs_weights=d["lbs_weights"])


def subdivide(v: np.ndarray, f: np.ndarray):
    """One round of midpoint subdivision: every triangle becomes four, one new vertex per edge (appended)."""
    f = np.asarray(f, dtype=np.int64)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    uniq, inv = np.unique(e, axis=0, return_inverse=True)
    inv = inv.reshape(-1) + v.shape[0]
    n = f.shape[0]
    ab, bc, ca = inv[:n], inv[n:2 * n], inv[2 * n:]
    a, b, c = f[:, 0], f[:, 1], f[:, 2]
    nf = np.concatenate([np.stack(t, 1) for t in ((a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca))])
    nv = np.concatenate([v, 0.5 * (v[uniq[:, 0]] + v[uniq[:, 1]])]).astype(np.float32)
    return nv, nf.astype(np.int32)


def bench_mesh(smpl: dict, stand_pose: np.ndarray, levels: int = 3, seed: int = 0, jitter: float = 1e-3):
    """An avatar-sized mesh in the PLY frame of validate_mesh: the template in the stand pose, subdivided ``levels``
    times (6890 -> 27554 -> 110210 -> 440834 vertices), jittered, rotated so that ``rotate`` brings it back."""
    _, f = template_obj()
    v = load_template(smpl, stand_pose)[0].numpy()
    for _ in range(levels):
        v, f = subdivide(v, f)
    v = v + np.random.default_rng(seed).normal(0, jitter, v.shape).astype(np.float32)
    return np.stack([v[:, 0], v[:, 2], -v[:, 1]], 1).astype(np.float32), f


def rotate(v) -> np.ndarray:
    """drive.py:317-323 in float64: (x, y, z) -> (x, -z, y)."""
    return np.matmul(np.asarray(v, dtype=np.float64), ROT)


def components(V: int, faces) -> np.ndarray:
    """Per vertex, the smallest vertex index of its connected component (triangle edges; isolated vertices alone)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    r = np.concatenate([f[:, 0], f[:, 1], f[:, 2]])
    c = np.concatenate([f[:, 1], f[:, 2], f[:, 0]])
    n, lab = connected_components(coo_matrix((np.ones(r.size), (r, c)), shape=(V, V)), directed=False)
    first = np.full(n, V, dtype=np.int64)
    np.minimum.at(first, lab, np.arange(V))
    return first[lab]


def cleanup_mesh(v, faces, colors=None):
    """drive.py:172-210 -> (kept vertex indices, vertices, re-indexed faces, colours)."""
    v = np.asarray(v)
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    lab = components(v.shape[0], f)
    roots, sizes = np.unique(lab, return_counts=True)          # roots ascending = the reference's discovery order
    keep_label = roots[np.argmax(sizes)]                       # argmax: the first of equal maxima
    keep = lab == keep_label
    idx = np.nonzero(keep)[0]
    new = np.cumsum(keep) - 1
    fk = f[keep[f].all(1)]
    return idx, v[keep], new[fk].astype(np.int32), None if colors is None else np.asarray(colors)[keep]


def find_nearest_ind(new_vertices, template_vertices, chunk: int = 2048) -> np.ndarray:
    """drive.py:235-240: argmin over the template of ((tv - v) ** 2).sum(-1) in float64, ties to the first index."""
    tv = np.asarray(template_vertices, dtype=np.float32).reshape(1, -1, 3)
    nv = np.asarray(new_vertices, dtype=np.float64).reshape(-1, 1, 3)
    out = np.empty(nv.shape[0], dtype=np.int64)
    for i in range(0, nv.shape[0], chunk):
        out[i:i + chunk] = np.argmin(((tv - nv[i:i + chunk]) ** 2).sum(-1), 1)
    return out


def rel_transforms(smpl: dict, pose_rot: torch.Tensor) -> torch.Tensor:
    """A [1, nj, 4, 4] of drive.py:243-245 (beta = 0, so v_shaped = v_template)."""
    J = torch.einsum("bik,ji->bjk", smpl["v_template"][None], smpl["J_regressor"])
    return olbs.batch_rigid_transform(pose_rot, J, smpl["parents"])[1]


def load_template(smpl: dict, stand_pose: np.ndarray):
    """drive.py:223-233 -> (template vertices [V,3], pose_rot [1,nj,3,3])."""
    pose_rot = olbs.batch_rodrigues(torch.from_numpy(np.asarray(stand_pose)).reshape(-1, 3)).reshape(1, -1, 3, 3)
    verts, _ = olbs.my_lbs(smpl["v_template"][None], pose_rot, smpl["posedirs"], smpl["J_regressor"], smpl["parents"],
                           smpl["lbs_weights"], pose2rot=False)
    return verts[0], pose_rot


def inv_lbs(smpl: dict, vertices, blend_weights, pose_rot) -> torch.Tensor:
    """drive.py:242-253: torch.inverse(sum_j w_j A_j) . [p; 1], rows 0-2, in float32."""
    nj = smpl["J_regressor"].shape[0]
    T = torch.matmul(blend_weights[None], rel_transforms(smpl, pose_rot).view(1, nj, 16)).view(1, -1, 4, 4)
    p = torch.as_tensor(np.asarray(vertices), dtype=torch.float32).reshape(1, -1, 3)
    ph = torch.cat([p, torch.ones(1, p.shape[1], 1)], dim=2)
    return torch.matmul(torch.inverse(T), ph.unsqueeze(-1))[0, :, :3, 0]


def lbs(smpl: dict, tpose, blend_weights, pose_rot) -> torch.Tensor:
    """drive.py:255-265 (no pose blend shapes)."""
    nj = smpl["J_regressor"].shape[0]
    T = torch.matmul(blend_weights[None], rel_transforms(smpl, pose_rot).view(1, nj, 16)).view(1, -1, 4, 4)
    vh = torch.cat([tpose.reshape(1, -1, 3), torch.ones(1, tpose.shape[0], 1)], dim=2)
    return torch.matmul(T, vh.unsqueeze(-1))[0, :, :3, 0]


def read_pose_my(poses: np.ndarray):
    """drive.py:282-293 on the loaded array."""
    out = []
    for i in range(poses.shape[0]):
        p = np.array(poses[i, :72])
        p[:3] = 0
        p[0] = np.pi / 2
        out.append(olbs.batch_rodrigues(torch.from_numpy(p).reshape(-1, 3)).view(1, 24, 3, 3))
    return out


def pc2_bytes(frames) -> bytes:
    """drive.py:295-305."""
    fr = np.asarray([np.asarray(f) for f in frames], dtype="<f4")
    return struct.pack("<12siiffi", b"POINTCACHE2\0", 1, fr.shape[1], 0, 60, fr.shape[0]) + fr.tobytes()


def generate(mesh_v, mesh_f, mesh_c, smpl: dict, stand_pose: np.ndarray, motion: np.ndarray) -> dict:
    """generate_animation (drive.py:317-361) on a mesh as read from its PLY."""
    keep_idx, v, f, c = cleanup_mesh(rotate(mesh_v), mesh_f, mesh_c)
    template, pose_rot = load_template(smpl, stand_pose)
    nearest = find_nearest_ind(v, template.numpy())
    w = smpl["lbs_weights"][torch.from_numpy(nearest)]
    tpose = inv_lbs(smpl, v, w, pose_rot)
    poses = read_pose_my(motion)
    frames = torch.stack([lbs(smpl, tpose, w, p) for p in poses])
    return dict(keep_idx=keep_idx, cleaned_v=v.astype(np.float32), cleaned_f=f, cleaned_c=c, template=template,
                pose_rot=pose_rot, nearest=nearest, tpose=tpose, pose_list=torch.cat(poses), frames=frames,
                pc2=pc2_bytes(frames.numpy()))
