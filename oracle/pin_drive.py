"""Pin oracle/drive.py against the reference's own drive.py (AvatarGen/AppearanceGen/drive.py) run in THIS container,
and record what the reference computed as tests/golden/ref_drive_small.pt.

drive.py imports ``open3d``, ``smplx`` and ``tqdm``, none of which is installed.  This script puts stand-ins for them
in ``sys.modules`` and executes the UNMODIFIED drive.py text:
  * ``smplx``: ``build_layer`` returns a layer holding the SMPL tensors whose forward is the reference's own ``my_lbs``
    (models/utils.py, imported unmodified with drive.py's in-tree smplx.lbs copies standing in for ``smplx.lbs``, as
    oracle/pin_lbs.py does), with pose2rot = False as smplx's layers run it;
  * ``open3d``: a small ``TriangleMesh`` restatement (``vertices``, ``compute_adjacency_list``, ``adjacency_list``,
    ``remove_vertices_by_index``).  Its removal semantics are UNPINNED: o3d is absent, so they are restated from its
    documentation (surviving vertices in order with their colours; triangles whose corners all survive, re-indexed);
  * ``tqdm``: the identity.
``generate_animation`` itself hard-codes its input and output paths, so its body (:317-361) is followed call by call
here, with the reference's functions.  Nothing of the reference is copied into this repository.

Inputs: the half above y = 0 of the shipped template (ref_tree_template.tar.gz, 6890 vertices) posed by the shipped
stand_pose.npy (stored in the golden): 3406 vertices, which the cut leaves as one island of 1992 and ~530 small islands
and singletons; jittered, rotated into the PLY frame, with extra islands (singletons and a small piece), the vertex
order shuffled.  The whole 6890-vertex posed template is the nearest-vertex reference set.  A second small mesh whose
two largest pieces tie; synthetic_smpl tensors (seed SMPL_SEED, re-created by the tests) with the real template as
v_template; a seeded [5, 75] motion.  Half a body keeps the golden small: the PC2 frames dominate its size.

    python -m oracle.pin_drive
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

REF_AG = "/root/reference/AvatarGen/AppearanceGen"
STAND_POSE = "/root/reference/AvatarGen/ShapeGen/output/stand_pose.npy"
GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
SMPL_SEED = 11


class _TriangleMesh:
    """Stand-in for open3d.geometry.TriangleMesh (the members drive.py uses)."""

    def __init__(self, vertices, triangles, vertex_colors):
        self.vertices = np.asarray(vertices, dtype=np.float64)
        self.triangles = np.asarray(triangles, dtype=np.int64).reshape(-1, 3)
        self.vertex_colors = np.asarray(vertex_colors)
        self.adjacency_list = []

    def compute_adjacency_list(self):
        adj = [set() for _ in range(len(self.vertices))]
        for a, b, c in self.triangles.tolist():
            adj[a].update((b, c))
            adj[b].update((a, c))
            adj[c].update((a, b))
        self.adjacency_list = adj

    def remove_vertices_by_index(self, indices):
        keep = np.ones(len(self.vertices), dtype=bool)
        keep[np.asarray(indices, dtype=np.int64)] = False
        new = np.cumsum(keep) - 1
        self.vertices = np.asarray(self.vertices)[keep]
        self.vertex_colors = self.vertex_colors[keep]
        self.triangles = new[self.triangles[keep[self.triangles].all(1)]]
        self.adjacency_list = []


def _install_stand_ins(src: str):
    ns = {}
    fake_lbs = types.ModuleType("smplx.lbs")
    smplx = types.ModuleType("smplx")
    smplx.lbs = fake_lbs

    class _Layer:
        def __init__(self, smpl):
            for k, v in smpl.items():
                setattr(self, k, v)
            self.shapedirs = torch.zeros(smpl["v_template"].shape[0], 3, 10)

        def __call__(self, betas, body_pose, global_orient):
            from models import utils as ref_utils
            full = torch.cat([global_orient, body_pose], dim=1)
            v_shaped = self.v_template[None] + ns["blend_shapes"](betas, self.shapedirs)
            verts, joints = ref_utils.my_lbs(v_shaped, full, self.v_template, self.shapedirs, self.posedirs,
                                             self.J_regressor, self.parents, self.lbs_weights, pose2rot=False)
            return {"vertices": verts, "joints": joints}

    smplx.build_layer = lambda folder, **kw: _Layer(_SMPL)
    o3d = types.ModuleType("open3d")
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a, dtype=np.float64))
    o3d.geometry = types.SimpleNamespace(TriangleMesh=_TriangleMesh)
    tqdm = types.ModuleType("tqdm")
    tqdm.tqdm = lambda it, *a, **k: it
    sys.modules.update({"smplx": smplx, "smplx.lbs": fake_lbs, "open3d": o3d, "tqdm": tqdm,
                        "neural_renderer": types.ModuleType("neural_renderer")})
    exec(compile(src, os.path.join(REF_AG, "drive.py"), "exec"), ns)
    for k in ("vertices2joints", "blend_shapes", "batch_rigid_transform", "transform_mat", "batch_rodrigues"):
        setattr(fake_lbs, k, ns[k])
    fake_lbs.__all__ = ["vertices2joints", "blend_shapes", "batch_rigid_transform", "transform_mat", "batch_rodrigues"]
    sys.path.insert(0, REF_AG)
    return ns


_SMPL = None


def _shuffled(v, faces, colors, rng):
    perm = rng.permutation(v.shape[0])          # new position i holds old vertex perm[i]
    inv = np.empty_like(perm)
    inv[perm] = np.arange(perm.size)
    return v[perm], inv[faces].astype(np.int32), colors[perm]


def golden_inputs(stand_pose: np.ndarray):
    from oracle import drive as D
    rng = np.random.default_rng(5)
    _, tf = D.template_obj()
    posed, _ = D.load_template(_SMPL, stand_pose)
    p = posed.numpy() + rng.normal(0, 2e-3, posed.shape).astype(np.float32)
    # the half of the template above y = 0: the cut splits it into one large island and ~530 small ones and singletons
    sel = posed.numpy()[:, 1] > 0
    p = p[sel]
    body_f = (np.cumsum(sel) - 1)[tf[sel[tf].all(1)]]
    body = np.stack([p[:, 0], p[:, 2], -p[:, 1]], 1).astype(np.float32)     # D.rotate maps it back onto p
    V = body.shape[0]
    piece = (rng.normal(0, 0.05, (5, 3)) + [0.8, 0.0, 0.3]).astype(np.float32)
    piece_f = np.array([[0, 1, 2], [0, 2, 3], [0, 3, 4], [0, 4, 1]]) + V + 3
    singles = rng.normal(0, 0.5, (3, 3)).astype(np.float32)
    v = np.concatenate([body, singles, piece])
    f = np.concatenate([body_f, piece_f]).astype(np.int32)
    c = rng.integers(0, 256, (v.shape[0], 3), dtype=np.uint8)
    mesh = _shuffled(v, f, c, rng)
    # two pieces of 6 vertices tie for largest; a piece of 3 and 4 singletons
    strip = np.array([[0, 1, 2], [1, 3, 2], [2, 3, 4], [3, 5, 4]])
    tv = rng.normal(0, 1, (19, 3)).astype(np.float32)
    tfaces = np.concatenate([strip, strip + 6, [[12, 13, 14]]]).astype(np.int32)
    tie = _shuffled(tv, tfaces, rng.integers(0, 256, (19, 3), dtype=np.uint8), rng)
    motion = rng.normal(0, 0.3, (5, 75)).astype(np.float32)
    return mesh, tie, motion


def main():
    global _SMPL
    from oracle import drive as D
    _SMPL = D.golden_smpl(SMPL_SEED)
    src = open(os.path.join(REF_AG, "drive.py")).read()
    ns = _install_stand_ins(src)
    stand_bytes = open(STAND_POSE, "rb").read()
    stand = np.load(STAND_POSE)
    (mv, mf, mc), (tv, tf, tc), motion = golden_inputs(stand)

    with tempfile.TemporaryDirectory() as tmp:
        pose_fname = os.path.join(tmp, "stand_pose.npy")
        motion_fname = os.path.join(tmp, "action.npy")
        open(pose_fname, "wb").write(stand_bytes)
        np.save(motion_fname, motion)
        # generate_animation (drive.py:317-361), call by call
        mesh = _TriangleMesh(mv, mf, mc)
        ori_vertices = np.asarray(mesh.vertices)
        rot_ori_vertices = np.matmul(ori_vertices, np.array([[1, 0, 0], [0, 0, 1], [0, -1, 0]], dtype=np.float32))
        mesh.vertices = ns["o3d"].utility.Vector3dVector(rot_ori_vertices)
        mesh = ns["cleanup_mesh"](mesh)
        smpl_model = ns["init_smpl_model"]("unused")
        template_object, pose_rot, beta = ns["load_template_smpl"](smpl_model, pose_fname)
        nearest_ind = ns["find_nearest_ind"](np.asarray(mesh.vertices), template_object)
        smpl_blend_weights = smpl_model.lbs_weights
        mesh_blend_weights = torch.gather(smpl_blend_weights, 0, torch.from_numpy(nearest_ind).unsqueeze(-1).repeat(
            1, smpl_blend_weights.shape[-1]))
        tpose_vertices = ns["inv_lbs"](smpl_model, np.asarray(mesh.vertices), mesh_blend_weights, pose_rot, beta)
        pose_list = ns["read_pose_my"](motion_fname)
        vertices_list = [ns["lbs"](smpl_model, tpose_vertices, mesh_blend_weights, p, beta) for p in pose_list]
        pc2_fname = os.path.join(tmp, "action.pc2")
        ns["write_pc2"](pc2_fname, vertices_list)
        pc2 = open(pc2_fname, "rb").read()
        tie_mesh = ns["cleanup_mesh"](_TriangleMesh(tv, tf, tc))

    ref = dict(cleaned_v=np.asarray(mesh.vertices).astype(np.float32), cleaned_f=mesh.triangles.astype(np.int32),
               cleaned_c=mesh.vertex_colors, template=template_object["vertices"][0], pose_rot=pose_rot,
               nearest=nearest_ind.astype(np.int32), tpose=tpose_vertices, pose_list=torch.cat(pose_list),
               pc2=np.frombuffer(pc2, dtype=np.uint8).copy())
    assert np.array_equal(ref["cleaned_v"].astype(np.float64), np.asarray(mesh.vertices))   # float32-exact positions

    # the restatement against the reference
    o = D.generate(mv, mf, mc, _SMPL, stand, motion)
    ot = D.cleanup_mesh(tv, tf, tc)
    checks = {
        "cleaned_v": np.array_equal(o["cleaned_v"], ref["cleaned_v"]),
        "cleaned_f": np.array_equal(o["cleaned_f"], ref["cleaned_f"]),
        "cleaned_c": np.array_equal(o["cleaned_c"], ref["cleaned_c"]),
        "nearest": np.array_equal(o["nearest"], ref["nearest"]),
        "tie": np.array_equal(ot[1], tie_mesh.vertices.astype(np.float32)) and np.array_equal(ot[2], tie_mesh.triangles),
        "pc2_header": o["pc2"][:32] == pc2[:32],
    }
    e_t = (o["template"] - ref["template"]).abs().max().item()
    e_tp = (o["tpose"] - ref["tpose"]).abs().max().item()
    fr_ref = np.frombuffer(pc2[32:], dtype="<f4")
    e_fr = np.abs(np.frombuffer(o["pc2"][32:], dtype="<f4") - fr_ref).max()
    e_rot = (o["pose_list"] - ref["pose_list"]).abs().max().item()
    print(f"[pin_drive] exact: {checks}")
    print(f"[pin_drive] max abs err template {e_t:.2e}, T-pose {e_tp:.2e}, frames {e_fr:.2e}, read_pose_my {e_rot:.2e}")
    print(f"[pin_drive] mesh {len(mv)} -> {len(ref['cleaned_v'])} vertices, {len(mf)} -> {len(ref['cleaned_f'])} faces;"
          f" tie mesh keeps {len(tie_mesh.vertices)} of {len(tv)}")
    assert all(checks.values()) and max(e_t, e_tp, e_fr, e_rot) <= 1e-6

    rec = dict(smpl_seed=SMPL_SEED, smpl_sums={k: float(v.double().sum()) for k, v in _SMPL.items()},
               stand_pose_npy=np.frombuffer(stand_bytes, dtype=np.uint8).copy(), motion=motion, mesh=dict(v=mv, f=mf, c=mc),
               tie=dict(v=tv, f=tf, c=tc, cleaned_v=tie_mesh.vertices.astype(np.float32),
                        cleaned_f=tie_mesh.triangles.astype(np.int32), cleaned_c=tie_mesh.vertex_colors),
               ref=ref)
    # numpy arrays as tensors: torch.save stores tensor storages raw, numpy arrays through pickle's text encoding
    as_t = lambda x: ({k: as_t(v) for k, v in x.items()} if isinstance(x, dict) else
                      torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x)
    os.makedirs(GOLDEN, exist_ok=True)
    torch.save(as_t(rec), os.path.join(GOLDEN, "ref_drive_small.pt"))


if __name__ == "__main__":
    main()
