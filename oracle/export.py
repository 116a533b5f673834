"""CPU oracle (test infrastructure, never on the product path): Avatar2FBX/export_fbx.py (:44-118) restated on numpy /
torch CPU, plus a small glTF 2.0 binary reader and skinner for checking the files avatarclip_b200.export writes.

o3d SEMANTICS UNPINNED: open3d is absent, so ``TriangleMesh.simplify_vertex_clustering`` (ply_utils.py:16-19) is restated
from open3d's published ``TriangleMesh::SimplifyVertexClustering``, both here and in the stand-in oracle/pin_avatar2fbx.py
runs export_fbx.py with:
  * voxel of a vertex: idx = floor((v - (min_bound - voxel / 2)) / voxel) per axis, in float64;
  * output vertex k is the k-th distinct voxel in order of its first vertex (input index order); vertices in no triangle
    are clustered too;
  * positions and colours: the float64 mean over the voxel (colours as open3d reads them, c / 255);
  * triangles remapped in input order; dropped when two corners share a voxel, or when an earlier kept triangle is one of
    its rotations (a reversed triangle is not); a kept triangle keeps the rotation it first appeared in.
Everything after the clustering (rotation, float32 nearest search, weight gather, ``inv_lbs``, ``tpose_joints``, x100,
colour cast) is pinned against the unmodified export_fbx.py by oracle/pin_avatar2fbx.py.
"""
from __future__ import annotations

import json
import struct

import numpy as np
import torch

from oracle import drive as D

KEY_BITS = 21


# ---------------------------------------------------------------- open3d's simplify_vertex_clustering (restated)
def voxel_size(v, resolution: int = 256) -> float:
    """ply_utils.py:17: max(max_bound - min_bound) / resolution, in float64."""
    v = np.asarray(v, dtype=np.float64)
    return max(v.max(0) - v.min(0)) / resolution


def cluster(v, faces, colors=None, voxel: float | None = None, resolution: int = 256):
    """simplify_vertex_clustering(voxel, Average) -> (vertices [K,3] float64, triangles [T,3] int64, colours [K,3]
    float64 or None, cluster of every input vertex [V]).  ``colors`` are float (open3d's c / 255); ``voxel`` defaults to
    Avatar2FBX's ``voxel_size(v, resolution)``."""
    v = np.asarray(v, dtype=np.float64).reshape(-1, 3)
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    if voxel is None:
        voxel = voxel_size(v, resolution)
    if voxel > 0:
        lo = v.min(0) - voxel * 0.5
        idx = np.floor((v - lo) / voxel).astype(np.int64)
    else:                                   # every vertex is the same point
        idx = np.zeros(v.shape, dtype=np.int64)
    key = (idx[:, 0] << (2 * KEY_BITS)) | (idx[:, 1] << KEY_BITS) | idx[:, 2]
    _, first, inv = np.unique(key, return_index=True, return_inverse=True)
    rank = np.empty(first.size, dtype=np.int64)
    rank[np.argsort(first, kind="stable")] = np.arange(first.size)     # numbered in order of their first vertex
    cl = rank[inv.reshape(-1)]
    K = first.size
    cnt = np.bincount(cl, minlength=K).astype(np.float64)
    mean = lambda x: np.stack([np.bincount(cl, weights=x[:, a], minlength=K) for a in range(3)], 1) / cnt[:, None]
    out_c = None if colors is None else mean(np.asarray(colors, dtype=np.float64).reshape(-1, 3))
    t = cl[f]
    t = t[(t[:, 0] != t[:, 1]) & (t[:, 0] != t[:, 2]) & (t[:, 1] != t[:, 2])]
    # the rotation that puts the smallest index first identifies a triangle up to rotation
    r = np.argmin(t, 1)
    canon = np.stack([t[np.arange(len(t)), (r + k) % 3] for k in range(3)], 1)
    if len(t):
        _, keep = np.unique(canon, axis=0, return_index=True)
        t = t[np.sort(keep)]
    return mean(v), t, out_c, cl


def simplify(v, faces, colors_u8=None, resolution: int = 256):
    """What the product's ``simplify_mesh`` returns for a PLY's float32 positions and uint8 colours: (vertices [K,3]
    float32, triangles [T,3] int32, colours [K,3] float32 or None)."""
    c = None if colors_u8 is None else np.asarray(colors_u8, dtype=np.float64) / 255.0
    ov, t, oc, _ = cluster(np.asarray(v, dtype=np.float32), faces, c, resolution=resolution)
    return ov.astype(np.float32), t.astype(np.int32), None if oc is None else oc.astype(np.float32)


# ---------------------------------------------------------------- export_fbx.py:55-109
def find_nearest_ind(new_vertices, template_vertices, chunk: int = 1024) -> np.ndarray:
    """ply_utils.py:84-89 with both operands float32: the float32 ((tv - v) ** 2).sum(-1), ties to the first index."""
    tv = np.asarray(template_vertices, dtype=np.float32).reshape(1, -1, 3)
    nv = np.asarray(new_vertices, dtype=np.float32).reshape(-1, 1, 3)
    out = np.empty(nv.shape[0], dtype=np.int64)
    for i in range(0, nv.shape[0], chunk):
        out[i:i + chunk] = np.argmin(((tv - nv[i:i + chunk]) ** 2).sum(-1), 1)
    return out


def smpl_object(v, faces, colors_u8, smpl: dict, stand_pose: np.ndarray, resolution: int = 256) -> dict:
    """export_fbx.py:50-109 on a mesh as read from its PLY (float32 positions, uint8 colours): the content of
    ``smpl_object`` (centimetres, as the reference hands it to the FBX SDK) plus the nearest indices."""
    sv, t, c = simplify(v, faces, colors_u8, resolution)
    rot = np.matmul(sv, D.ROT)                                       # float32, export_fbx.py:57-62
    template, pose_rot = D.load_template(smpl, stand_pose)
    nearest = find_nearest_ind(rot, template.numpy())
    w = smpl["lbs_weights"][torch.from_numpy(nearest)]
    tpose = D.inv_lbs(smpl, rot, w, pose_rot)                        # ply_utils.py:91-102 (float32 torch.inverse)
    joints = torch.einsum("bik,ji->bjk", smpl["v_template"][None], smpl["J_regressor"])[0]
    return dict(vertices=tpose * 100, triangles=t, joints=joints * 100, nearest=nearest, colors=c, simplified=sv,
                pose_rot=pose_rot)


def wide_smpl(smpl: dict, every: int = 7, joints: int = 6, seed: int = 3) -> dict:
    """``smpl`` with every ``every``-th template vertex skinned to ``joints`` joints (rows still sum to 1): more
    influences than one glTF weight set holds."""
    g = torch.Generator().manual_seed(seed)
    w = smpl["lbs_weights"].clone()
    rows = torch.arange(0, w.shape[0], every)
    w[rows] = 0
    for r in rows.tolist():
        idx = torch.randperm(w.shape[1], generator=g)[:joints]
        w[r, idx] = torch.rand(joints, generator=g) + 0.1
    w = w / w.sum(1, keepdim=True)
    return dict(smpl, lbs_weights=w)


# ---------------------------------------------------------------- glTF 2.0 binary reader and skinner
_COMP = {5120: np.int8, 5121: np.uint8, 5122: np.int16, 5123: np.uint16, 5125: np.uint32, 5126: np.float32}
_NCOMP = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4, "MAT4": 16}


def read_glb(path: str) -> dict:
    """Parse a .glb: {'json': the glTF JSON, 'bin': the binary chunk, 'header': (magic, version, length),
    'chunks': [(type, offset, length)]}."""
    data = open(path, "rb").read()
    magic, version, length = struct.unpack_from("<4sII", data, 0)
    chunks, off = [], 12
    while off < len(data):
        n, typ = struct.unpack_from("<II", data, off)
        chunks.append((typ, off + 8, n))
        off += 8 + n
    js = [c for c in chunks if c[0] == 0x4E4F534A][0]
    bn = [c for c in chunks if c[0] == 0x004E4942]
    g = json.loads(data[js[1]:js[1] + js[2]].decode("utf-8"))
    b = data[bn[0][1]:bn[0][1] + bn[0][2]] if bn else b""
    return {"json": g, "bin": b, "header": (magic, version, length), "chunks": chunks, "size": len(data)}


def accessor(glb: dict, i: int) -> np.ndarray:
    """Decode accessor ``i`` (tightly packed views) -> [count, ncomp] (MAT4 as [count, 4, 4] row-major matrices)."""
    g = glb["json"]
    a = g["accessors"][i]
    bv = g["bufferViews"][a["bufferView"]]
    dt = np.dtype(_COMP[a["componentType"]]).newbyteorder("<")
    n = _NCOMP[a["type"]]
    off = bv.get("byteOffset", 0) + a.get("byteOffset", 0)
    x = np.frombuffer(glb["bin"], dtype=dt, count=a["count"] * n, offset=off).reshape(a["count"], n)
    if a["type"] == "MAT4":
        return x.reshape(-1, 4, 4).transpose(0, 2, 1).astype(np.float64)    # glTF matrices are column-major
    return x


def quat_to_mat(q) -> np.ndarray:
    x, y, z, w = [float(t) for t in q]
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def node_worlds(glb: dict, frame: int | None = None) -> list:
    """World matrices of every node from its TRS; with ``frame``, the rotations / translations of animation 0 at
    keyframe ``frame`` replace the nodes' own."""
    g = glb["json"]
    nodes = g["nodes"]
    trs = [dict(t=np.array(n.get("translation", [0, 0, 0]), dtype=np.float64),
                r=np.array(n.get("rotation", [0, 0, 0, 1]), dtype=np.float64),
                s=np.array(n.get("scale", [1, 1, 1]), dtype=np.float64)) for n in nodes]
    if frame is not None:
        an = g["animations"][0]
        for ch in an["channels"]:
            smp = an["samplers"][ch["sampler"]]
            val = accessor(glb, smp["output"])[frame].astype(np.float64)
            trs[ch["target"]["node"]][{"rotation": "r", "translation": "t", "scale": "s"}[ch["target"]["path"]]] = val
    local = []
    for d in trs:
        m = np.eye(4)
        m[:3, :3] = quat_to_mat(d["r"]) * d["s"][None]
        m[:3, 3] = d["t"]
        local.append(m)
    parent = {c: i for i, n in enumerate(nodes) for c in n.get("children", [])}
    world = [None] * len(nodes)

    def w(i):
        if world[i] is None:
            world[i] = local[i] if i not in parent else w(parent[i]) @ local[i]
        return world[i]
    return [w(i) for i in range(len(nodes))]


def skin(glb: dict, frame: int | None = None) -> np.ndarray:
    """Skinned POSITION of the first skinned mesh node: sum over all JOINTS_n / WEIGHTS_n sets of w * (G_j . IBM_j)."""
    g = glb["json"]
    node = [n for n in g["nodes"] if "skin" in n and "mesh" in n][0]
    sk = g["skins"][node["skin"]]
    prim = g["meshes"][node["mesh"]]["primitives"][0]
    worlds = node_worlds(glb, frame)
    ibm = accessor(glb, sk["inverseBindMatrices"])
    jm = np.stack([worlds[j] @ ibm[k] for k, j in enumerate(sk["joints"])])
    p = accessor(glb, prim["attributes"]["POSITION"]).astype(np.float64)
    ph = np.concatenate([p, np.ones((p.shape[0], 1))], 1)
    out = np.zeros_like(p)
    s = 0
    while f"JOINTS_{s}" in prim["attributes"]:
        J = accessor(glb, prim["attributes"][f"JOINTS_{s}"]).astype(np.int64)
        W = accessor(glb, prim["attributes"][f"WEIGHTS_{s}"]).astype(np.float64)
        for k in range(4):
            out += W[:, k:k + 1] * np.einsum("vij,vj->vi", jm[J[:, k]], ph)[:, :3]
        s += 1
    return out
