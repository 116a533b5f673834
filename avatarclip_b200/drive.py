"""Host-side mirror of AvatarGen/AppearanceGen/drive.py: animate a generated avatar mesh with SMPL's skeleton.

``generate_animation`` (drive.py:308-361) reads the PLY ``Runner.validate_mesh`` exports, rotates it from the NeuS
frame into SMPL's ((x, y, z) -> (x, -z, y)), keeps its largest connected piece (``cleanup_mesh``), gives every vertex
the skin weights of its nearest vertex of the SMPL template in the stand pose (``load_template_smpl`` /
``find_nearest_ind``), un-poses it to the zero pose (``inv_lbs``) and skins it through a motion (``read_pose_my`` /
``lbs``), writing ``<name>_cleaned_apose.ply`` and a PC2 point cache ``<motion>.pc2`` that a mesh-cache modifier
(Blender and other DCC tools) plays on that PLY.  The reference's paths are hard-coded; here they are arguments.

Everything runs in libavc_b200.so (``avc_nearest_vertex``, ``avc_mesh_components``, ``avc_lbs_rel_transforms``,
``avc_inv_lbs``, ``avc_lbs_frames``, and ``avc_lbs_fwd`` for the template).  The frames are computed and written
chunk by chunk through a pinned host buffer, so a long motion never has to fit in host memory.

``smplx`` and ``SMPL_NEUTRAL.pkl`` are not needed: pass the SMPL tensors as a mapping, or any object with the
attributes ``v_template``, ``posedirs``, ``J_regressor``, ``parents`` and ``lbs_weights`` (a ``smplx`` SMPL layer has
exactly these).  ``shapedirs`` is not used: drive.py fixes beta = 0.  ``read_pose_seq`` (a dataset-specific pickle
folder, unused by drive.py itself) is not mirrored.

    python -m avatarclip_b200.drive --mesh exp/.../meshes/00029500.ply --motion action.npy --smpl smpl.npz \\
        --stand_pose ShapeGen/output/stand_pose.npy --out_dir out/
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import struct
import sys
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import _lib, handoff

SMPL_KEYS = ("v_template", "posedirs", "J_regressor", "parents", "lbs_weights")
PC2_SAMPLE_RATE = 60
# (x, y, z) -> (x, -z, y): drive.py:318-323 multiplies the row vectors by this matrix
NEUS_TO_SMPL = np.array([[1, 0, 0], [0, 0, 1], [0, -1, 0]], dtype=np.float32)
_CHUNK_BYTES = 256 << 20       # device + pinned buffer budget per chunk of frames (two of each are live)


class Mesh(NamedTuple):
    """A triangle mesh on the device: vertices [V,3] float32, triangles [F,3] int32, colours [V,3] uint8 (host) or None."""
    vertices: torch.Tensor
    triangles: torch.Tensor
    vertex_colors: Optional[np.ndarray] = None


_bound = None


def _L():
    global _bound
    L = _lib.lib()
    if _bound is None:
        vp, i32, sz = C.c_void_p, C.c_int32, C.c_size_t
        L.avc_nearest_vertex.argtypes = [vp, i32, vp, i32, vp, vp]
        L.avc_mesh_components_workspace_bytes.argtypes = [i32, C.POINTER(sz)]
        L.avc_mesh_components.argtypes = [vp, i32, i32, vp, vp, vp, sz, vp]
        L.avc_lbs_rel_transforms.argtypes = [vp, vp, vp, i32, i32, vp, i32, i32, vp, vp, vp]
        L.avc_inv_lbs.argtypes = [vp, vp, i32, vp, i32, i32, vp, vp, vp]
        L.avc_lbs_frames.argtypes = [vp, vp, i32, vp, i32, i32, vp, i32, i32, i32, vp, vp]
        for n in ("avc_nearest_vertex", "avc_mesh_components_workspace_bytes", "avc_mesh_components",
                  "avc_lbs_rel_transforms", "avc_inv_lbs", "avc_lbs_frames"):
            getattr(L, n).restype = C.c_int
        _bound = L
    return L


def _cuda(device) -> torch.device:
    device = torch.device(device)
    if device.type != "cuda":
        raise _lib.AvcError("avatarclip_b200 has no CPU path")
    return device


def _f32(t, device) -> torch.Tensor:
    return torch.as_tensor(t).detach().to(device, torch.float32).contiguous()


# ---------------------------------------------------------------- SMPL tensors
def _check_smpl(d: dict) -> dict:
    missing = [k for k in SMPL_KEYS if k not in d or d[k] is None]
    if missing:
        raise ValueError(f"SMPL tensors: missing {missing} (need {list(SMPL_KEYS)})")
    shp = {k: tuple(np.shape(d[k])) for k in SMPL_KEYS}
    vt = shp["v_template"]
    if len(vt) != 2 or vt[1] != 3 or vt[0] < 1:
        raise ValueError(f"SMPL v_template: expected [V, 3], got {list(vt)}")
    V = vt[0]
    jr = shp["J_regressor"]
    if len(jr) != 2 or jr[1] != V or not 1 <= jr[0] <= 32:
        raise ValueError(f"SMPL J_regressor: expected [n_joints <= 32, {V}], got {list(jr)}")
    nj = jr[0]
    want = {"parents": (nj,), "lbs_weights": (V, nj), "posedirs": ((nj - 1) * 9, V * 3)}
    for k, s in want.items():
        if shp[k] != s:
            raise ValueError(f"SMPL {k}: expected {list(s)}, got {list(shp[k])}")
    par = np.asarray(torch.as_tensor(d["parents"]).cpu()).astype(np.int64)
    if par[0] != -1 or any(not 0 <= par[j] < j for j in range(1, nj)):
        raise ValueError("SMPL parents: expected parents[0] = -1 and 0 <= parents[j] < j")
    return d


def smpl_tensors(smpl, device="cuda") -> dict:
    """The SMPL tensors drive.py reads from its smplx layer, on ``device``: a mapping, or an object with the attributes
    ``v_template`` [V,3], ``posedirs`` [(nj-1)*9, V*3], ``J_regressor`` [nj,V], ``parents`` [nj], ``lbs_weights``
    [V,nj] (an ``smplx`` SMPL layer)."""
    device = _cuda(device)
    get = (lambda k: smpl.get(k)) if hasattr(smpl, "keys") else (lambda k: getattr(smpl, k, None))
    d = _check_smpl({k: get(k) for k in SMPL_KEYS})
    out = {k: _f32(d[k], device) for k in ("v_template", "posedirs", "J_regressor", "lbs_weights")}
    out["parents"] = torch.as_tensor(d["parents"]).to(device, torch.int32).contiguous()
    return out


def load_smpl_npz(path: str) -> dict:
    """SMPL tensors from an ``.npz`` with the keys ``SMPL_KEYS`` (see ``--help`` for the conversion from smplx)."""
    with np.load(path) as z:
        return _check_smpl({k: z[k] for k in SMPL_KEYS if k in z.files})


# ---------------------------------------------------------------- mesh I/O and cleanup (drive.py:162-210)
def read_ply(fname: str, device="cuda") -> Mesh:
    """drive.py:162-167 for the PLY ``Runner.validate_mesh`` writes (``handoff.read_ply``)."""
    device = _cuda(device)
    v, f, c = handoff.read_ply(fname)
    if f.size and (f.min() < 0 or f.max() >= v.shape[0]):
        raise ValueError(f"{fname}: a face index lies outside [0, {v.shape[0]})")
    return Mesh(_f32(v, device), torch.as_tensor(f, dtype=torch.int32).to(device).contiguous(), c)


def write_ply(mesh: Mesh, fname: str) -> str:
    """drive.py:169-170 (``handoff.write_ply``: float32 positions, the colours, int32 faces)."""
    return handoff.write_ply(fname, mesh.vertices.cpu().numpy(), mesh.triangles.cpu().numpy(), mesh.vertex_colors)


def cleanup_mesh(mesh: Mesh) -> Mesh:
    """drive.py:172-210: keep the largest connected piece (by vertex count; among equal sizes the one with the smallest
    vertex index), its vertices in their original order with their colours, and the triangles among them."""
    v, f = mesh.vertices, mesh.triangles
    device = _cuda(v.device)
    V, F = v.shape[0], f.shape[0]
    L = _L()
    need = C.c_size_t()
    _lib.check(L.avc_mesh_components_workspace_bytes(V, C.byref(need)), "avc_mesh_components_workspace_bytes")
    ws = torch.empty(need.value, dtype=torch.uint8, device=device)
    labels = torch.empty(V, dtype=torch.int32, device=device)
    kept = torch.empty(2, dtype=torch.int32, device=device)
    f = f.to(device, torch.int32).contiguous()
    _lib.check(L.avc_mesh_components(_lib.ptr(f) if F else None, F, V, _lib.ptr(labels), _lib.ptr(kept), _lib.ptr(ws),
                                     ws.numel(), _lib.stream_ptr()), "avc_mesh_components")
    keep = labels == kept[0]
    new_index = torch.cumsum(keep, 0, dtype=torch.int32) - 1
    # the three corners of a triangle share a component, so its first corner decides (remove_vertices_by_index)
    tri = f[keep[f[:, 0].long()]] if F else f
    colors = None if mesh.vertex_colors is None else mesh.vertex_colors[keep.cpu().numpy()]
    return Mesh(v[keep].contiguous(), new_index[tri.long()].contiguous(), colors)


# ---------------------------------------------------------------- poses (drive.py:13-49, 223-233, 282-293)
def batch_rodrigues(rot_vecs: torch.Tensor, epsilon: float = 1e-8) -> torch.Tensor:
    """drive.py:13-49, on the host: [N,3] axis-angle -> [N,3,3] rotation matrices (pose decoding only)."""
    n = rot_vecs.shape[0]
    angle = torch.norm(rot_vecs + epsilon, dim=1, keepdim=True, p=2)
    rot_dir = rot_vecs / angle
    cos, sin = torch.cos(angle)[:, None], torch.sin(angle)[:, None]
    rx, ry, rz = torch.split(rot_dir, 1, dim=1)
    zeros = torch.zeros((n, 1), dtype=rot_vecs.dtype)
    K = torch.cat([zeros, -rz, ry, rz, zeros, -rx, -ry, rx, zeros], dim=1).view(n, 3, 3)
    return torch.eye(3, dtype=rot_vecs.dtype)[None] + sin * K + (1 - cos) * torch.bmm(K, K)


def _motion_axis_angle(fname: str) -> np.ndarray:
    """drive.py:283-290: rows [F, >=72] -> pose[:72] with the global orientation replaced by (pi/2, 0, 0)."""
    poses = np.load(fname)
    if poses.ndim != 2 or poses.shape[1] < 72 or poses.shape[0] < 1:
        raise ValueError(f"{fname}: expected a motion of shape [frames, >= 72], got {list(poses.shape)}")
    p = np.array(poses[:, :72])
    p[:, :3] = 0
    p[:, 0] = np.pi / 2
    return p


def read_pose_my(fname: str):
    """drive.py:282-293: one [1,24,3,3] rotation tensor per frame (host tensors, as the reference returns)."""
    p = torch.from_numpy(_motion_axis_angle(fname))
    return list(batch_rodrigues(p.reshape(-1, 3)).view(-1, 1, 24, 3, 3).unbind(0))


def load_template_smpl(smpl_model, pose_fname: str, device="cuda"):
    """drive.py:223-233: the SMPL template posed by ``stand_pose.npy`` with pose blend shapes (``my_lbs``, beta = 0).
    Returns ({'vertices': [1,V,3]}, pose_rot [1,24,3,3], beta [1,10]) on ``device``."""
    from .lbs import my_lbs
    s = smpl_tensors(smpl_model, device)
    nj = s["J_regressor"].shape[0]
    with open(pose_fname, "rb") as f:
        pose = torch.from_numpy(np.load(f))
    pose_rot = batch_rodrigues(pose.reshape(-1, 3)).reshape(1, nj, 3, 3).to(s["v_template"].device, torch.float32)
    verts, _ = my_lbs(s["v_template"][None], pose_rot.reshape(1, -1), None, None, s["posedirs"], s["J_regressor"],
                      s["parents"], s["lbs_weights"], pose2rot=False)
    return {"vertices": verts}, pose_rot, torch.zeros(1, 10, device=s["v_template"].device)


# ---------------------------------------------------------------- nearest vertex, inverse LBS, LBS (drive.py:235-265)
def _nearest(query: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    out = torch.empty(query.shape[0], dtype=torch.int32, device=query.device)
    _lib.check(_L().avc_nearest_vertex(_lib.ptr(query), query.shape[0], _lib.ptr(ref), ref.shape[0], _lib.ptr(out),
                                       _lib.stream_ptr()), "avc_nearest_vertex")
    return out


def find_nearest_ind(new_vertices, template_object) -> torch.Tensor:
    """drive.py:235-240: per mesh vertex, the index of the nearest template vertex (float64 squared distance, ties to
    the first).  The vertices are taken as float32, the precision of the PLY.  Returns int64 [N] on the device."""
    tv = template_object["vertices"]
    device = _cuda(tv.device)
    return _nearest(_f32(new_vertices, device).reshape(-1, 3), _f32(tv, device).reshape(-1, 3)).long()


def _rel_transforms(s: dict, pose: torch.Tensor, pose2rot: bool, return_joints: bool = False):
    """A [frames, nj, 12] for beta = 0 (drive.py:243-245); with ``return_joints``, (A, J [nj, 3] = J_regressor .
    v_template)."""
    nj, V = s["J_regressor"].shape
    frames = pose.shape[0]
    A = torch.empty(frames, nj, 12, dtype=torch.float32, device=pose.device)
    joints = torch.empty(nj, 3, dtype=torch.float32, device=pose.device)
    _lib.check(_L().avc_lbs_rel_transforms(_lib.ptr(s["v_template"]), _lib.ptr(s["J_regressor"]), _lib.ptr(s["parents"]),
                                           V, nj, _lib.ptr(pose), 1 if pose2rot else 0, frames, _lib.ptr(joints),
                                           _lib.ptr(A), _lib.stream_ptr()), "avc_lbs_rel_transforms")
    return (A, joints) if return_joints else A


def _zero_beta(beta):
    if beta is not None and bool(torch.as_tensor(beta).ne(0).any()):
        raise NotImplementedError("drive.py fixes beta = 0; shapes with non-zero beta are not supported")


def _inv_lbs(verts, nearest, weights, A) -> torch.Tensor:
    N = verts.shape[0]
    out = torch.empty(N, 3, dtype=torch.float32, device=verts.device)
    _lib.check(_L().avc_inv_lbs(_lib.ptr(verts), _lib.ptr(nearest), N, _lib.ptr(weights), weights.shape[0],
                                weights.shape[1], _lib.ptr(A), _lib.ptr(out), _lib.stream_ptr()), "avc_inv_lbs")
    return out


def _lbs_frames(tpose, nearest, weights, A, begin, count, out) -> torch.Tensor:
    _lib.check(_L().avc_lbs_frames(_lib.ptr(tpose), _lib.ptr(nearest), tpose.shape[0], _lib.ptr(weights),
                                   weights.shape[0], weights.shape[1], _lib.ptr(A), A.shape[0], begin, count,
                                   _lib.ptr(out), _lib.stream_ptr()), "avc_lbs_frames")
    return out


def inv_lbs(smpl_model, vertices, blend_weights, pose, beta=None) -> torch.Tensor:
    """drive.py:242-253: un-pose ``vertices`` [N,3] posed by ``pose`` [1,nj,3,3] with per-vertex ``blend_weights``
    [N,nj] -> [N,3] (T^-1 . [p; 1] in fp64, rounded to float32)."""
    device = _cuda(blend_weights.device)
    _zero_beta(beta)
    s = smpl_tensors(smpl_model, device)
    nj = s["J_regressor"].shape[0]
    A = _rel_transforms(s, _f32(pose, device).reshape(1, nj, 9), False)
    return _inv_lbs(_f32(vertices, device).reshape(-1, 3), None, _f32(blend_weights, device), A[0])


def lbs(smpl_model, tpose_vertices, blend_weights, pose, beta=None) -> torch.Tensor:
    """drive.py:255-265: skin ``tpose_vertices`` [N,3] with ``blend_weights`` [N,nj] by ``pose`` [1,nj,3,3] (no pose
    blend shapes) -> [N,3]."""
    device = _cuda(blend_weights.device)
    _zero_beta(beta)
    s = smpl_tensors(smpl_model, device)
    nj = s["J_regressor"].shape[0]
    A = _rel_transforms(s, _f32(pose, device).reshape(1, nj, 9), False)
    tp = _f32(tpose_vertices, device).reshape(-1, 3)
    return _lbs_frames(tp, None, _f32(blend_weights, device), A, 0, 1,
                       torch.empty(tp.shape[0], 3, dtype=torch.float32, device=device))


# ---------------------------------------------------------------- PC2 (drive.py:295-305)
def pc2_header(vcount: int, num_samples: int) -> bytes:
    """drive.py:296-301: start frame 0 and sample rate 60, both stored as float32."""
    return struct.pack("<12siiffi", b"POINTCACHE2\0", 1, vcount, 0, PC2_SAMPLE_RATE, num_samples)


def write_pc2(fname: str, vertices_list) -> str:
    """drive.py:295-305: the header, then the frames as little-endian float32 [F][V][3]."""
    frames = [np.asarray(torch.as_tensor(v).detach().cpu(), dtype="<f4").reshape(-1, 3) for v in vertices_list]
    with open(fname, "wb") as fp:
        fp.write(pc2_header(frames[0].shape[0], len(frames)))
        for fr in frames:
            fp.write(fr.tobytes())
    return fname


# ---------------------------------------------------------------- generate_animation (drive.py:308-361)
def generate_animation(mesh_ply: str, motion_npy: str, out_dir: str, smpl, stand_pose_npy: str,
                       frames_per_chunk: Optional[int] = None, device="cuda"):
    """drive.py:308-361 with its hard-coded paths as arguments.  Writes ``out_dir/<mesh name>_cleaned_apose.ply`` and
    ``out_dir/<motion name>.pc2``; returns both paths."""
    device = _cuda(device)
    s = smpl_tensors(smpl, device)
    nj = s["J_regressor"].shape[0]
    if nj != 24:
        raise ValueError(f"read_pose_my decodes 24 SMPL joints per frame; the SMPL tensors have {nj}")
    motion = torch.from_numpy(_motion_axis_angle(motion_npy)).to(device, torch.float32).contiguous()
    mesh = read_ply(mesh_ply, device)
    v = mesh.vertices
    mesh = cleanup_mesh(mesh._replace(vertices=torch.stack([v[:, 0], -v[:, 2], v[:, 1]], 1).contiguous()))
    os.makedirs(out_dir, exist_ok=True)
    name = os.path.splitext(os.path.basename(mesh_ply))[0]
    ply_path = write_ply(mesh, os.path.join(out_dir, f"{name}_cleaned_apose.ply"))

    template, pose_rot, _ = load_template_smpl(s, stand_pose_npy, device)
    nearest = _nearest(mesh.vertices, template["vertices"].reshape(-1, 3))
    A_stand = _rel_transforms(s, pose_rot.reshape(1, nj, 9).contiguous(), False)
    tpose = _inv_lbs(mesh.vertices, nearest, s["lbs_weights"], A_stand[0])

    A = _rel_transforms(s, motion, True)
    frames, N = A.shape[0], tpose.shape[0]
    chunk = max(1, min(frames, frames_per_chunk or _CHUNK_BYTES // (N * 12)))
    dev_buf = [torch.empty(chunk, N, 3, dtype=torch.float32, device=device) for _ in range(2)]
    host_buf = [torch.empty(chunk, N, 3, dtype=torch.float32, pin_memory=True) for _ in range(2)]
    done = [torch.cuda.Event() for _ in range(2)]
    pc2_path = os.path.join(out_dir, os.path.splitext(os.path.basename(motion_npy))[0] + ".pc2")
    with open(pc2_path, "wb") as fp:
        fp.write(pc2_header(N, frames))
        pending = None
        # chunk k is computed and copied while the host writes chunk k-1; buffer k % 2 is free again because the
        # write of chunk k-2 finished in the previous iteration
        for k, f0 in enumerate(range(0, frames, chunk)):
            b, n = k % 2, min(chunk, frames - f0)
            _lbs_frames(tpose, nearest, s["lbs_weights"], A, f0, n, dev_buf[b])
            host_buf[b][:n].copy_(dev_buf[b][:n], non_blocking=True)
            done[b].record()
            if pending is not None:
                pb, pn = pending
                done[pb].synchronize()
                fp.write(host_buf[pb][:pn].numpy().data)
            pending = (b, n)
        pb, pn = pending
        done[pb].synchronize()
        fp.write(host_buf[pb][:pn].numpy().data)
    return ply_path, pc2_path


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(
        prog="python -m avatarclip_b200.drive",
        description="Animate a generated avatar mesh (AvatarGen/AppearanceGen/drive.py): keep its largest piece, rig it "
                    "with the skin weights of the nearest SMPL template vertex, un-pose it and skin it through a "
                    "motion into a PC2 point cache.",
        epilog="The SMPL .npz holds the arrays " + ", ".join(SMPL_KEYS) + ".  From an smplx model folder:  python -c "
               "\"import smplx, numpy as np; m = smplx.build_layer('models', model_type='smpl', gender='neutral'); "
               "np.savez('smpl.npz', **{k: getattr(m, k).detach().cpu().numpy() for k in "
               "('v_template', 'posedirs', 'J_regressor', 'parents', 'lbs_weights')})\"")
    p.add_argument("--mesh", required=True, help="PLY written by --mode validate_mesh")
    p.add_argument("--motion", required=True, help=".npy of shape [frames, >= 72] (SMPL axis-angle per frame)")
    p.add_argument("--smpl", required=True, help=".npz with the SMPL tensors (see below)")
    p.add_argument("--stand_pose", required=True, help="ShapeGen/output/stand_pose.npy: the pose the mesh stands in")
    p.add_argument("--out_dir", required=True)
    p.add_argument("--frames_per_chunk", type=int, default=None, help="frames computed per device chunk")
    p.add_argument("--device", default="cuda")
    return p


def main(argv=None) -> int:
    parser = build_parser()
    a = parser.parse_args(argv)
    for flag, path in (("--mesh", a.mesh), ("--motion", a.motion), ("--smpl", a.smpl), ("--stand_pose", a.stand_pose)):
        if not os.path.isfile(path):
            parser.error(f"{flag}: no such file: {path}")
    if a.frames_per_chunk is not None and a.frames_per_chunk < 1:
        parser.error("--frames_per_chunk must be >= 1")
    try:
        smpl = load_smpl_npz(a.smpl)
    except (ValueError, OSError) as e:
        parser.error(f"--smpl: {e}")
    ply, pc2 = generate_animation(a.mesh, a.motion, a.out_dir, smpl, a.stand_pose, a.frames_per_chunk, a.device)
    print(ply)
    print(pc2)
    return 0


if __name__ == "__main__":
    sys.exit(main())
