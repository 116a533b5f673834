"""Export a generated avatar as a rigged, skinned glTF 2.0 binary (.glb): the open counterpart of Avatar2FBX.

Avatar2FBX/export_fbx.py (:44-118) takes the PLY ``Runner.validate_mesh`` exports, simplifies it by vertex clustering
(``simplify_mesh``, open3d's ``simplify_vertex_clustering`` at voxel = max extent / 256), rotates it from the NeuS frame
into SMPL's ((x, y, z) -> (x, -z, y)), gives every vertex the skin weights of its nearest SMPL template vertex in the
stand pose (``find_nearest_ind``, float32 distances), un-poses it to SMPL's zero pose (``inv_lbs``) and hands the result
to Autodesk's FBX SDK rigged to SMPL's 24 joints under Mixamo's bone names.  Here the same rig is written as a .glb,
which Blender, three.js, Unity and Unreal import directly, with no SDK; optionally with the joint rotations of a motion
``.npy`` (the file ``avatarclip_b200.drive`` reads) as keyframes.

Everything on the mesh runs in libavc_b200.so: ``avc_mesh_cluster``, ``avc_mesh_decimate``, ``avc_nearest_vertex_f32``,
``avc_lbs_fwd`` (the template), ``avc_lbs_rel_transforms`` and ``avc_inv_lbs``.

With ``--target_faces N``, when the clustering keeps more than N faces, the mesh as read is first decimated by
quadric-error edge collapse (``decimate_mesh``) to N faces (or N - 1), keeping its topology, and then clustered
(``reduce_mesh``): vertex clustering alone removes few faces from a finely tessellated mesh, and the texture atlas
needs a few faces per texel cell.  The rig, the bake and the glTF then see the reduced mesh.

The file:
  * Frame and units: the bind pose is SMPL's zero pose in SMPL's canonical frame, which is glTF's (+Y up, facing +Z);
    lengths in metres (the reference's x100 is an FBX unit convention).
  * Mesh: one primitive.  POSITION float32 with min / max; indices uint32; COLOR_0 float32 RGB, the PLY's display
    (sRGB-encoded) colours decoded to linear as glTF defines COLOR_0 (the reference's FBX passes them through raw);
    JOINTS_n / WEIGHTS_n hold every non-zero weight of ``lbs_weights[nearest]``, largest first, in as many sets of
    four as the vertex with the most influences needs, not renormalised (SMPL's rows sum to 1).  Viewers that read only
    set 0 (three.js, for one) drop the influences beyond the four largest.
  * Skeleton: 24 joint nodes with Mixamo's names for the SMPL joints, the parent table of the SMPL tensors, translation
    J_j - J_parent(j) (the root's J_0), no rest rotation; inverseBindMatrices translate(-J_j).  The joint matrix G_j .
    IBM_j is then SMPL's relative transform A_j, so glTF skinning equals ``drive.lbs``.
  * Animation (with a motion): joints 1-23 get a rotation channel, the motion's axis-angle as unit quaternions
    (x, y, z, w), each key sign-aligned with the previous one so that slerp takes the short arc; key k at k / fps,
    LINEAR.  The root has no channel: drive replaces the global orientation by (pi/2, 0, 0) in its z-up frame, which
    is the identity in glTF's y-up frame, and reads no translation.  So at every frame p_drive = R_x(pi/2) (p_glb - J_0)
    + J_0.

  * Texture (with ``--conf``): ``bake.bake_texture`` fills a per-face atlas from the NeuS run's colour field.  The
    primitive then has one vertex per face corner (the atlas splits every face off its neighbours; positions and skin
    weights are the shared vertex's), NORMAL (``bake.vertex_normals`` of the bind pose, smooth across the split),
    TEXCOORD_0 (origin at the top left) and no COLOR_0.  The material's baseColorTexture is a PNG in a buffer view,
    its bytes the sRGB ``to8b`` bytes the PLY holds; the sampler is LINEAR without mipmaps (a face's footprint never
    leaves its own texels) and CLAMP_TO_EDGE.
  * Normal map (with ``--normal_map``, which needs ``--conf``): ``bake.bake_normal_map`` bakes the SDF's normals in
    each texel's tangent frame on the same atlas.  The primitive also has TANGENT (float VEC4, per corner,
    ``bake.corner_tangents`` of the bind pose's positions and NORMALs; w = +-1 so that w cross(N, T) points towards
    the image's top, glTF's "+Y up"), a second PNG (linear data, no sRGB) and the material's normalTexture
    {index 1, texCoord 0}.  The map is baked in the PLY frame.  The rotation into SMPL's frame is proper, so its
    tangent-space values carry over exactly; the un-posing is linear-blend skinning, under which they carry over to
    first order, the standard assumption of a skinned normal map.

Left out: FBX itself (it needs Autodesk's proprietary SDK; Blender converts the .glb to FBX), the reference's all-zero
blend shape, non-zero beta (Avatar2FBX fixes beta = 0) and ``cleanup_mesh`` (Avatar2FBX does not run it).

    python -m avatarclip_b200.export --mesh exp/.../meshes/00029500.ply --smpl smpl.npz \\
        --stand_pose stand_pose.npy [--motion action.npy --fps 30] [--target_faces 20000] --out avatar.glb \\
        [--conf confs/examples/hulk.conf [--case smpl] [--checkpoint ckpt_030000.pth] [--texture_size 2048]
         [--normal_map]]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import struct
import sys

import numpy as np
import torch

from . import _lib, bake, drive
from .drive import Mesh, _cuda, _f32

# The SMPL joints under Mixamo's bone names, in SMPL's joint order
MIXAMO_NAMES = (
    "Hips", "LeftUpLeg", "RightUpLeg", "Spine", "LeftLeg", "RightLeg", "Spine1", "LeftFoot", "RightFoot", "Spine2",
    "LeftToeBase", "RightToeBase", "Neck", "LeftShoulder", "RightShoulder", "Head", "LeftArm", "RightArm",
    "LeftForeArm", "RightForeArm", "LeftHand", "RightHand", "LeftHandMiddle1", "RightHandMiddle1")
JOINT_NAMES = tuple("mixamorig:" + n for n in MIXAMO_NAMES)
DEFAULT_RESOLUTION = 256

_bound = None


def _L():
    global _bound
    L = drive._L()
    if _bound is None:
        vp, i32, sz = C.c_void_p, C.c_int32, C.c_size_t
        L.avc_nearest_vertex_f32.argtypes = [vp, i32, vp, i32, vp, vp]
        L.avc_mesh_cluster_workspace_bytes.argtypes = [i32, i32, C.POINTER(sz)]
        L.avc_mesh_cluster.argtypes = [vp, vp, i32, vp, i32, i32, vp, vp, vp, vp, vp, sz, vp]
        L.avc_mesh_decimate_workspace_bytes.argtypes = [i32, i32, C.POINTER(sz)]
        L.avc_mesh_decimate.argtypes = [vp, vp, i32, vp, i32, i32, vp, vp, vp, vp, vp, sz, vp]
        for n in ("avc_nearest_vertex_f32", "avc_mesh_cluster_workspace_bytes", "avc_mesh_cluster",
                  "avc_mesh_decimate_workspace_bytes", "avc_mesh_decimate"):
            getattr(L, n).restype = C.c_int
        _bound = L
    return L


# ---------------------------------------------------------------- ply_utils.py:16-19, 84-89
def simplify_mesh(mesh: Mesh, resolution: int = DEFAULT_RESOLUTION) -> Mesh:
    """ply_utils.py:16-19: open3d's vertex clustering with voxel = max(max_bound - min_bound) / ``resolution``,
    averaging positions and colours (semantics in include/avc_b200.h, ``avc_mesh_cluster``).  The colours of the
    result are float32 [K,3] in [0, 1] on the host (open3d's c / 255), or None."""
    v, f = mesh.vertices, mesh.triangles
    device = _cuda(v.device)
    v = _f32(v, device).reshape(-1, 3)
    f = f.to(device, torch.int32).contiguous().reshape(-1, 3)
    V, F = v.shape[0], f.shape[0]
    L = _L()
    need = C.c_size_t()
    _lib.check(L.avc_mesh_cluster_workspace_bytes(V, F, C.byref(need)), "avc_mesh_cluster_workspace_bytes")
    ws = torch.empty(need.value, dtype=torch.uint8, device=device)
    col = None
    if mesh.vertex_colors is not None:
        col = torch.as_tensor(np.ascontiguousarray(mesh.vertex_colors, dtype=np.uint8)).to(device).reshape(-1, 3)
    v_out = torch.empty(V, 3, dtype=torch.float32, device=device)
    c_out = None if col is None else torch.empty(V, 3, dtype=torch.float32, device=device)
    f_out = torch.empty(max(F, 1), 3, dtype=torch.int32, device=device)
    counts = torch.empty(2, dtype=torch.int32, device=device)
    _lib.check(L.avc_mesh_cluster(_lib.ptr(v), _lib.ptr(col), V, _lib.ptr(f) if F else None, F, int(resolution),
                                  _lib.ptr(v_out), _lib.ptr(c_out), _lib.ptr(f_out) if F else None, _lib.ptr(counts),
                                  _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "avc_mesh_cluster")
    K, T = counts.tolist()
    return Mesh(v_out[:K], f_out[:T], None if c_out is None else c_out[:K].cpu().numpy())


def decimate_mesh(mesh: Mesh, target_faces: int) -> Mesh:
    """Quadric-error edge collapse to ``target_faces`` (semantics in include/avc_b200.h, ``avc_mesh_decimate``): the
    result has target_faces - 1 or target_faces faces, or more when no edge can collapse without breaking the
    topology or flipping a face.  Colours, when given, are float [N,3] in any scale and are interpolated along each
    collapsed edge.  Vertices and faces keep their input order.  The ends of non-manifold edges never move, so a
    mesh with many of them (a vertex-clustered one) stops early: ``reduce_mesh`` decimates before clustering."""
    return _decimate(mesh, target_faces)[0]


def _decimate(mesh: Mesh, target_faces: int):
    """``decimate_mesh`` and the number of collapse rounds it ran."""
    v, f = mesh.vertices, mesh.triangles
    device = _cuda(v.device)
    v = _f32(v, device).reshape(-1, 3)
    f = f.to(device, torch.int32).contiguous().reshape(-1, 3)
    V, F = v.shape[0], f.shape[0]
    L = _L()
    need = C.c_size_t()
    _lib.check(L.avc_mesh_decimate_workspace_bytes(V, F, C.byref(need)), "avc_mesh_decimate_workspace_bytes")
    ws = torch.empty(need.value, dtype=torch.uint8, device=device)
    col = None if mesh.vertex_colors is None else _f32(torch.as_tensor(mesh.vertex_colors), device).reshape(-1, 3)
    v_out = torch.empty(V, 3, dtype=torch.float32, device=device)
    c_out = None if col is None else torch.empty(V, 3, dtype=torch.float32, device=device)
    f_out = torch.empty(F, 3, dtype=torch.int32, device=device)
    counts = torch.empty(3, dtype=torch.int32, device=device)
    _lib.check(L.avc_mesh_decimate(_lib.ptr(v), _lib.ptr(col), V, _lib.ptr(f), F, int(target_faces), _lib.ptr(v_out),
                                   _lib.ptr(c_out), _lib.ptr(f_out), _lib.ptr(counts), _lib.ptr(ws), ws.numel(),
                                   _lib.stream_ptr()), "avc_mesh_decimate")
    K, T, rounds = counts.tolist()
    return Mesh(v_out[:K], f_out[:T], None if c_out is None else c_out[:K].cpu().numpy()), rounds


def reduce_mesh(mesh: Mesh, resolution: int = DEFAULT_RESOLUTION, target_faces: int | None = None) -> Mesh:
    """``simplify_mesh`` at ``resolution``; with ``target_faces``, when the clustering keeps more faces than that, the
    input is first decimated to ``target_faces`` (``decimate_mesh``) and the result clustered.  Clustering a finely
    tessellated mesh keeps most of its faces and leaves non-manifold edges (triangles beside their reverses) whose
    ends the collapse must not move, so the decimation runs on the mesh as read; the clustering after it only merges
    what falls in one voxel and keeps at most target_faces faces.  Colours are decimated on the 0-255 scale and rounded
    to the nearest byte before the clustering.  When the clustering alone keeps at most ``target_faces`` faces, the
    result is the clustering's, byte for byte."""
    clustered = simplify_mesh(mesh, resolution)
    if target_faces is None or clustered.triangles.shape[0] <= target_faces:
        return clustered
    col = None if mesh.vertex_colors is None else np.asarray(mesh.vertex_colors, dtype=np.float32)
    dec = decimate_mesh(Mesh(mesh.vertices, mesh.triangles, col), target_faces)
    c8 = None if dec.vertex_colors is None else np.clip(np.rint(dec.vertex_colors), 0, 255).astype(np.uint8)
    return simplify_mesh(Mesh(dec.vertices, dec.triangles, c8), resolution)


def _nearest_f32(query: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    out = torch.empty(query.shape[0], dtype=torch.int32, device=query.device)
    _lib.check(_L().avc_nearest_vertex_f32(_lib.ptr(query), query.shape[0], _lib.ptr(ref), ref.shape[0],
                                           _lib.ptr(out), _lib.stream_ptr()), "avc_nearest_vertex_f32")
    return out


def find_nearest_ind(new_vertices, template_object) -> torch.Tensor:
    """ply_utils.py:84-89: per mesh vertex, the index of the nearest template vertex by the float32 squared distance
    ((dx*dx + dy*dy) + dz*dz, each operation rounded), ties to the first.  Returns int64 [N] on the device."""
    tv = template_object["vertices"]
    device = _cuda(tv.device)
    return _nearest_f32(_f32(new_vertices, device).reshape(-1, 3), _f32(tv, device).reshape(-1, 3)).long()


# ---------------------------------------------------------------- export_fbx.py:44-109
def rig_avatar(mesh_ply: str, smpl, stand_pose_npy: str, resolution: int = DEFAULT_RESOLUTION, device="cuda",
               ply_frame: bool = False, target_faces: int | None = None) -> dict:
    """export_fbx.py:50-109 for one PLY: the content of the reference's ``smpl_object``, in metres, as host arrays:
    ``vertices`` [N,3] T-pose (SMPL's zero pose), ``triangles`` [T,3], ``joints`` [24,3] (J_regressor . v_template),
    ``nearest`` [N] (template vertex whose weights each vertex takes), ``colors`` [N,3] float32 in [0, 1] or None,
    plus what the skin needs: ``lbs_weights`` [M,24] and ``parents`` [24] of the SMPL tensors, and ``name``.
    ``ply_frame`` adds ``vertices_ply`` [N,3] float32: the clustered vertices in the PLY (NeuS) frame, before the
    rotation and the un-posing, where ``bake.bake_texture`` reads the colour field.  ``target_faces`` bounds the
    faces (``reduce_mesh``)."""
    device = _cuda(device)
    s = drive.smpl_tensors(smpl, device)
    nj = s["J_regressor"].shape[0]
    if nj != len(JOINT_NAMES):
        raise ValueError(f"the skeleton has the {len(JOINT_NAMES)} SMPL joints; the SMPL tensors have {nj}")
    mesh = reduce_mesh(drive.read_ply(mesh_ply, device), resolution, target_faces)
    v = mesh.vertices
    rot = torch.stack([v[:, 0], -v[:, 2], v[:, 1]], 1).contiguous()          # export_fbx.py:57-62
    template, pose_rot, _ = drive.load_template_smpl(s, stand_pose_npy, device)
    nearest = _nearest_f32(rot, template["vertices"].reshape(-1, 3))
    A_stand, joints = drive._rel_transforms(s, pose_rot.reshape(1, nj, 9).contiguous(), False, return_joints=True)
    tpose = drive._inv_lbs(rot, nearest, s["lbs_weights"], A_stand[0])
    rig = dict(name=os.path.splitext(os.path.basename(mesh_ply))[0], vertices=tpose.cpu().numpy(),
               triangles=mesh.triangles.cpu().numpy(), joints=joints.cpu().numpy(),
               nearest=nearest.cpu().numpy().astype(np.int64), colors=mesh.vertex_colors,
               lbs_weights=s["lbs_weights"].cpu().numpy(), parents=s["parents"].cpu().numpy().astype(np.int64))
    if ply_frame:
        rig["vertices_ply"] = v.cpu().numpy()
    return rig


# ---------------------------------------------------------------- glTF 2.0 binary
def srgb_to_linear(c) -> np.ndarray:
    """The sRGB decoding function (IEC 61966-2-1), elementwise on values in [0, 1]."""
    c = np.asarray(c, dtype=np.float64)
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


def axis_angle_to_quat(r) -> np.ndarray:
    """[..., 3] axis-angle -> [..., 4] unit quaternions (x, y, z, w), in float64."""
    r = np.asarray(r, dtype=np.float64)
    ang = np.linalg.norm(r, axis=-1, keepdims=True)
    half = 0.5 * ang
    k = np.where(ang > 0, np.sin(half) / np.where(ang > 0, ang, 1.0), 0.5)     # sin(a/2)/a -> 1/2 as a -> 0
    q = np.concatenate([r * k, np.cos(half)], -1)
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def _np(x):
    return None if x is None else np.asarray(torch.as_tensor(x).detach().cpu())


def _skin_sets(weights: np.ndarray):
    """Every non-zero weight per vertex, largest first, in sets of four: (joints [S][N,4] uint8, weights [S][N,4])."""
    nz = (weights != 0).sum(1)
    n_sets = max(1, int(-(-int(nz.max(initial=0)) // 4)))
    order = np.argsort(-weights, axis=1, kind="stable")[:, :4 * n_sets]
    w = np.take_along_axis(weights, order, 1).astype(np.float32)
    j = np.where(w != 0, order, 0).astype(np.uint8)              # unused slots: joint 0 with weight 0
    return [j[:, 4 * s:4 * s + 4] for s in range(n_sets)], [w[:, 4 * s:4 * s + 4] for s in range(n_sets)]


class _Glb:
    """Accumulates tightly packed buffer views (4-byte aligned) and accessors."""

    def __init__(self):
        self.blob, self.views, self.accessors = bytearray(), [], []

    def add(self, arr: np.ndarray, comp: int, typ: str, target=None, minmax: bool = False) -> int:
        data = np.ascontiguousarray(arr).tobytes()
        view = {"buffer": 0, "byteOffset": len(self.blob), "byteLength": len(data)}
        if target:
            view["target"] = target
        self.blob += data + b"\0" * (-len(data) % 4)
        self.views.append(view)
        n = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4, "MAT4": 16}[typ]
        acc = {"bufferView": len(self.views) - 1, "componentType": comp, "count": int(arr.size // n), "type": typ}
        if minmax:
            a = np.asarray(arr, dtype=np.float64).reshape(-1, n)
            acc["min"], acc["max"] = a.min(0).tolist(), a.max(0).tolist()
        self.accessors.append(acc)
        return len(self.accessors) - 1

    def add_bytes(self, data: bytes) -> int:
        """A buffer view of raw bytes (an embedded image): returns its index."""
        self.views.append({"buffer": 0, "byteOffset": len(self.blob), "byteLength": len(data)})
        self.blob += data + b"\0" * (-len(data) % 4)
        return len(self.views) - 1


def write_glb(rig: dict, path: str, motion_npy: str | None = None, fps: float = 30, texture=None,
              normal_map=None) -> str:
    """Write ``rig`` (``rig_avatar``'s dictionary; host arrays or tensors) as a glTF 2.0 binary at ``path``; with
    ``motion_npy`` (rows [F, >= 72] of SMPL axis-angle, as ``drive`` reads them) also one animation of F keys at
    ``fps``; with ``texture`` = (uv [3T,2], image uint8 [H,W,3] RGB), ``bake.bake_texture``'s result, a textured
    primitive, which also needs ``rig["normals"]`` [N,3]; with ``normal_map`` = (tangents [3T,4], image uint8
    [H,W,3]), ``bake.corner_tangents`` and ``bake.bake_normal_map``'s image, also TANGENT and a normalTexture (it
    needs ``texture``).  Layout in the module docstring.  Returns ``path``."""
    FLOAT, UINT, UBYTE = 5126, 5125, 5121
    pos = _np(rig["vertices"]).astype(np.float32).reshape(-1, 3)
    tri = _np(rig["triangles"]).astype(np.uint32).reshape(-1, 3)
    J = _np(rig["joints"]).astype(np.float32).reshape(-1, 3)
    parents = _np(rig["parents"]).astype(np.int64).reshape(-1)
    weights = _np(rig["lbs_weights"]).astype(np.float32)[_np(rig["nearest"]).astype(np.int64).reshape(-1)]
    nj = J.shape[0]
    if nj != len(JOINT_NAMES) or parents.shape[0] != nj or weights.shape[1] != nj:
        raise ValueError(f"write_glb: expected {len(JOINT_NAMES)} joints, got joints {list(J.shape)}, parents "
                         f"{list(parents.shape)}, weights {list(weights.shape)}")
    if fps <= 0:
        raise ValueError(f"write_glb: fps must be > 0, got {fps}")
    motion = None if motion_npy is None else drive._motion_axis_angle(motion_npy)
    if normal_map is not None:
        if texture is None:
            raise ValueError("write_glb: a normal map needs the colour texture (texture=)")
        tangents = _np(normal_map[0]).astype(np.float32).reshape(-1, 4)
        nmap = np.asarray(_np(normal_map[1]), dtype=np.uint8)
        if tangents.shape[0] != tri.size or nmap.ndim != 3 or nmap.shape[2] != 3:
            raise ValueError(f"write_glb: normal_map needs tangents [{tri.size}, 4] and an RGB image [H, W, 3], got "
                             f"tangents {list(tangents.shape)}, image {list(nmap.shape)}")

    if texture is not None:
        uv, image = _np(texture[0]).astype(np.float32).reshape(-1, 2), np.asarray(_np(texture[1]), dtype=np.uint8)
        if rig.get("normals") is None:
            raise ValueError("write_glb: a textured primitive needs rig['normals'] (bake.vertex_normals)")
        if uv.shape[0] != tri.size or image.ndim != 3 or image.shape[2] != 3:
            raise ValueError(f"write_glb: texture needs uv [{tri.size}, 2] and an RGB image [H, W, 3], got uv "
                             f"{list(uv.shape)}, image {list(image.shape)}")
        corner = tri.reshape(-1).astype(np.int64)           # one vertex per face corner: the UV seams split every face
        normals = _np(rig["normals"]).astype(np.float32).reshape(-1, 3)[corner]
        pos, weights, tri = pos[corner], weights[corner], np.arange(tri.size, dtype=np.uint32).reshape(-1, 3)

    g = _Glb()
    attrs = {"POSITION": g.add(pos, FLOAT, "VEC3", 34962, minmax=True)}
    if texture is not None:
        attrs["NORMAL"] = g.add(normals, FLOAT, "VEC3", 34962)
        attrs["TEXCOORD_0"] = g.add(uv, FLOAT, "VEC2", 34962)
        if normal_map is not None:
            attrs["TANGENT"] = g.add(tangents, FLOAT, "VEC4", 34962)
    elif rig.get("colors") is not None:
        col = srgb_to_linear(np.clip(_np(rig["colors"]).reshape(-1, 3), 0.0, 1.0)).astype(np.float32)
        attrs["COLOR_0"] = g.add(col, FLOAT, "VEC3", 34962)
    js, ws = _skin_sets(weights)
    for s, (j, w) in enumerate(zip(js, ws)):
        attrs[f"JOINTS_{s}"] = g.add(j, UBYTE, "VEC4", 34962)
        attrs[f"WEIGHTS_{s}"] = g.add(w, FLOAT, "VEC4", 34962)
    indices = g.add(tri.reshape(-1), UINT, "SCALAR", 34963)
    ibm = np.tile(np.eye(4, dtype=np.float32), (nj, 1, 1))
    ibm[:, :3, 3] = -J                                               # translate(-J_j)
    ibm_acc = g.add(ibm.transpose(0, 2, 1), FLOAT, "MAT4")           # column-major

    rel = J - np.where(parents[:, None] >= 0, J[np.maximum(parents, 0)], 0)
    nodes = [{"name": rig.get("name") or "avatar", "mesh": 0, "skin": 0}]
    for j in range(nj):
        node = {"name": JOINT_NAMES[j], "translation": rel[j].astype(np.float64).tolist()}
        kids = [1 + c for c in range(nj) if parents[c] == j]
        if kids:
            node["children"] = kids
        nodes.append(node)
    roots = [1 + j for j in range(nj) if parents[j] < 0]
    gltf = {
        "asset": {"version": "2.0", "generator": "avatarclip_b200.export"},
        "scene": 0,
        "scenes": [{"nodes": [0] + roots}],
        "nodes": nodes,
        "meshes": [{"name": nodes[0]["name"], "primitives": [{"attributes": attrs, "indices": indices, "material": 0,
                                                              "mode": 4}]}],
        "materials": [{"name": "vertex_colour", "pbrMetallicRoughness": {"baseColorFactor": [1, 1, 1, 1],
                                                                         "metallicFactor": 0.0,
                                                                         "roughnessFactor": 1.0}}],
        "skins": [{"name": "smpl", "joints": [1 + j for j in range(nj)], "skeleton": roots[0],
                   "inverseBindMatrices": ibm_acc}],
    }
    if texture is not None:
        png = g.add_bytes(bake.encode_png(image))
        gltf["materials"] = [{"name": "baked_texture", "pbrMetallicRoughness": {"baseColorTexture": {"index": 0},
                                                                              "metallicFactor": 0.0,
                                                                              "roughnessFactor": 1.0}}]
        gltf["textures"] = [{"sampler": 0, "source": 0}]
        gltf["samplers"] = [{"magFilter": 9729, "minFilter": 9729, "wrapS": 33071, "wrapT": 33071}]   # LINEAR, CLAMP
        gltf["images"] = [{"bufferView": png, "mimeType": "image/png"}]
        if normal_map is not None:
            gltf["materials"][0]["normalTexture"] = {"index": 1, "texCoord": 0}
            gltf["textures"].append({"sampler": 0, "source": 1})
            gltf["images"].append({"bufferView": g.add_bytes(bake.encode_png(nmap)), "mimeType": "image/png"})
    if motion is not None:
        q = axis_angle_to_quat(motion[:, 3:3 * nj].reshape(motion.shape[0], nj - 1, 3))     # [F, nj-1, 4]
        for k in range(1, q.shape[0]):                                 # short arc between successive keys
            flip = (q[k] * q[k - 1]).sum(-1) < 0
            q[k, flip] = -q[k, flip]
        times = g.add((np.arange(q.shape[0], dtype=np.float64) / fps).astype(np.float32), FLOAT, "SCALAR",
                      minmax=True)
        samplers, channels = [], []
        for j in range(1, nj):
            out = g.add(q[:, j - 1].astype(np.float32), FLOAT, "VEC4")
            samplers.append({"input": times, "output": out, "interpolation": "LINEAR"})
            channels.append({"sampler": len(samplers) - 1, "target": {"node": 1 + j, "path": "rotation"}})
        name = os.path.splitext(os.path.basename(motion_npy))[0]
        gltf["animations"] = [{"name": name, "samplers": samplers, "channels": channels}]
    gltf.update(accessors=g.accessors, bufferViews=g.views, buffers=[{"byteLength": len(g.blob)}])

    js_bytes = json.dumps(gltf, separators=(",", ":")).encode("utf-8")
    js_bytes += b" " * (-len(js_bytes) % 4)
    total = 12 + 8 + len(js_bytes) + 8 + len(g.blob)
    with open(path, "wb") as fp:
        fp.write(struct.pack("<4sII", b"glTF", 2, total))
        fp.write(struct.pack("<II", len(js_bytes), 0x4E4F534A) + js_bytes)
        fp.write(struct.pack("<II", len(g.blob), 0x004E4942) + bytes(g.blob))
    return path


def export_avatar(mesh_ply: str, out_glb: str, smpl, stand_pose_npy: str, motion_npy: str | None = None,
                  fps: float = 30, resolution: int = DEFAULT_RESOLUTION, device="cuda", conf: str | None = None,
                  case: str = "smpl", checkpoint: str | None = None, texture_size: int | None = None,
                  target_faces: int | None = None, normal_map: bool = False) -> str:
    """``rig_avatar`` + ``write_glb``: the .glb of one PLY, optionally animated by ``motion_npy``.  With ``conf`` (the
    NeuS run's conf) the mesh also gets a texture of ``texture_size`` (default ``bake.DEFAULT_TEXTURE_SIZE``) baked
    from the run's colour field: the Runner is built as ``--mode validate_mesh`` builds it (its last checkpoint), or
    from ``checkpoint`` (a path, or a name under the run's checkpoints directory).  ``target_faces`` bounds the
    faces (``reduce_mesh``); the texture atlas is then sized for the reduced mesh.  When decimation stops above the target, one line on stderr says how many faces it reached.  ``normal_map`` (needs
    ``conf``) also bakes a tangent-space normal map from the run's SDF (``bake.bake_normal_map``); one line on stderr
    counts its flat and back-facing texels when there are any.  Returns the path."""
    if target_faces is not None and target_faces < 1:
        raise ValueError(f"export_avatar: target_faces must be >= 1, got {target_faces}")
    if conf is None and (checkpoint is not None or texture_size is not None or normal_map):
        raise ValueError("export_avatar: checkpoint, texture_size and normal_map need conf (the NeuS run to bake from)")
    if motion_npy is not None:
        drive._motion_axis_angle(motion_npy)           # reject a bad motion before the GPU work
    rig = rig_avatar(mesh_ply, smpl, stand_pose_npy, resolution, device, ply_frame=conf is not None,
                     target_faces=target_faces)
    if target_faces is not None and len(rig["triangles"]) > target_faces:
        print(f"export: decimation stopped at {len(rig['triangles'])} faces, above --target_faces {target_faces}: "
              "no further edge collapse keeps the topology and the face orientations", file=sys.stderr)
    texture = None
    if conf is not None:
        from .runner import Runner
        T = bake.DEFAULT_TEXTURE_SIZE if texture_size is None else int(texture_size)
        bake.atlas_grid(len(rig["triangles"]), T)      # refuse a texture too small for the faces before any render
        runner = Runner(conf, "validate_mesh", case, is_continue=checkpoint is None, device=device)
        if checkpoint is not None:
            runner.load_checkpoint(checkpoint)
        texture = bake.bake_texture(runner, rig["vertices_ply"], rig["triangles"], T)
        rig["normals"] = bake.vertex_normals(torch.from_numpy(rig["vertices"]).to(_cuda(device)),
                                             torch.from_numpy(rig["triangles"])).cpu().numpy()
    nmap = None
    if normal_map:
        image, stats = bake.bake_normal_map(runner, rig["vertices_ply"], rig["triangles"], T)
        tangents = bake.corner_tangents(torch.from_numpy(rig["vertices"]).to(_cuda(device)), rig["triangles"],
                                        torch.from_numpy(rig["normals"]), texture[0])
        nmap = (tangents.cpu().numpy().reshape(-1, 4), image)
        if stats["flat"] or stats["back_facing"]:
            print(f"export: normal map: {stats['flat']} of {stats['used']} texels flat (no zero crossing within the "
                  f"search, or a vanishing gradient), {stats['back_facing']} back-facing", file=sys.stderr)
    out_dir = os.path.dirname(os.path.abspath(out_glb))
    os.makedirs(out_dir, exist_ok=True)
    return write_glb(rig, out_glb, motion_npy, fps, texture=texture, normal_map=nmap)


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(
        prog="python -m avatarclip_b200.export",
        description="Export a generated avatar mesh as a rigged, skinned glTF 2.0 binary (Avatar2FBX's rig: vertex "
                    "clustering, the skin weights of the nearest SMPL template vertex, un-posed to SMPL's zero pose, "
                    "24 joints under Mixamo's names), optionally animated by an SMPL motion.",
        epilog="The SMPL .npz holds the arrays " + ", ".join(drive.SMPL_KEYS) + " (see python -m avatarclip_b200.drive "
               "--help for writing it from smplx).")
    p.add_argument("--mesh", required=True, help="PLY written by --mode validate_mesh")
    p.add_argument("--smpl", required=True, help=".npz with the SMPL tensors")
    p.add_argument("--stand_pose", required=True, help="stand_pose.npy: the pose the mesh stands in")
    p.add_argument("--motion", default=None, help=".npy of shape [frames, >= 72] (SMPL axis-angle per frame)")
    p.add_argument("--fps", type=float, default=30.0, help="keyframes per second of the motion")
    p.add_argument("--resolution", type=int, default=DEFAULT_RESOLUTION,
                   help="voxel = largest extent / resolution for the vertex clustering")
    p.add_argument("--target_faces", type=int, default=None,
                   help="at most this many faces: when the clustering keeps more, decimate the mesh by quadric-error "
                        "edge collapse to this many, then cluster")
    p.add_argument("--out", required=True, help="the .glb to write")
    p.add_argument("--device", default="cuda")
    t = p.add_argument_group("texture", "bake a base-colour texture from the NeuS run that made the mesh")
    t.add_argument("--conf", default=None, help="the run's conf (as --mode validate_mesh reads it)")
    t.add_argument("--case", default=None, help="CASE_NAME of the conf (default smpl)")
    t.add_argument("--checkpoint", default=None,
                   help="ckpt_XXXXXX.pth under the run's checkpoints directory, or a path (default: the last one)")
    t.add_argument("--texture_size", type=int, default=None,
                   help=f"texels per side of the square texture (default {bake.DEFAULT_TEXTURE_SIZE})")
    t.add_argument("--normal_map", action="store_true",
                   help="also bake a tangent-space normal map from the run's SDF (glTF normalTexture and TANGENT)")
    return p


def main(argv=None) -> int:
    parser = build_parser()
    a = parser.parse_args(argv)
    if a.conf is None:
        for flag, val in (("--case", a.case), ("--checkpoint", a.checkpoint), ("--texture_size", a.texture_size),
                          ("--normal_map", a.normal_map or None)):
            if val is not None:
                parser.error(f"{flag} needs --conf (the NeuS run to bake the texture from)")
    if a.target_faces is not None and a.target_faces < 1:
        parser.error("--target_faces must be >= 1")
    if a.texture_size is not None and not 1 <= a.texture_size <= bake.MAX_TEXTURE_SIZE:
        parser.error(f"--texture_size must be in [1, {bake.MAX_TEXTURE_SIZE}]")
    for flag, path in (("--mesh", a.mesh), ("--smpl", a.smpl), ("--stand_pose", a.stand_pose), ("--motion", a.motion),
                       ("--conf", a.conf)):
        if path is not None and not os.path.isfile(path):
            parser.error(f"{flag}: no such file: {path}")
    if not a.fps > 0:
        parser.error("--fps must be > 0")
    if not 1 <= a.resolution <= (1 << 21) - 2:
        parser.error("--resolution must be in [1, 2097150]")
    try:
        smpl = drive.load_smpl_npz(a.smpl)
    except (ValueError, OSError) as e:
        parser.error(f"--smpl: {e}")
    if np.shape(smpl["J_regressor"])[0] != len(JOINT_NAMES):
        parser.error(f"--smpl: the skeleton has the {len(JOINT_NAMES)} SMPL joints, the file "
                     f"{np.shape(smpl['J_regressor'])[0]}")
    if a.motion is not None:
        try:
            drive._motion_axis_angle(a.motion)
        except (ValueError, OSError) as e:
            parser.error(f"--motion: {e}")
    if a.conf is None:
        print(export_avatar(a.mesh, a.out, smpl, a.stand_pose, a.motion, a.fps, a.resolution, a.device,
                            target_faces=a.target_faces))
        return 0
    try:
        out = export_avatar(a.mesh, a.out, smpl, a.stand_pose, a.motion, a.fps, a.resolution, a.device, conf=a.conf,
                            case=a.case or "smpl", checkpoint=a.checkpoint, texture_size=a.texture_size,
                            target_faces=a.target_faces, normal_map=a.normal_map)
    except bake.AtlasTooSmall as e:
        parser.error(f"--texture_size: {e}")
    print(out)
    return 0


if __name__ == "__main__":
    sys.exit(main())
