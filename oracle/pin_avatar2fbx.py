"""Pin oracle/export.py against the reference's own Avatar2FBX/export_fbx.py run in THIS container, and record what the
reference computed as tests/golden/ref_avatar2fbx_small.pt.

export_fbx.py imports ``open3d``, ``smplx``, ``tqdm`` and Autodesk's FBX SDK (``FbxCommon`` / ``fbx``), none of which is
installed.  This script puts stand-ins for them in ``sys.modules`` and runs the UNMODIFIED export_fbx.py as ``__main__``
with ``runpy``, in a temporary directory holding ``meshes/<name>.ply`` and ``poses/stand_pose.npy``:
  * ``open3d``: a ``TriangleMesh`` whose ``io.read_triangle_mesh`` reads the PLY as open3d does (float64 positions,
    colours c / 255) and whose ``simplify_vertex_clustering`` is oracle/export.py's restatement.  That part is
    UNPINNED (open3d is absent);
  * ``smplx``: ``build_layer`` returns a layer holding the SMPL tensors (with a zero ``shapedirs``, beta = 0) whose
    forward is the reference's own ``my_lbs`` (AvatarGen/AppearanceGen/models/utils.py, unmodified, with ply_utils.py's
    smplx helpers standing in for ``smplx.lbs``), as oracle/pin_drive.py does;
  * ``FbxCommon`` / ``fbx``: permissive no-ops;
  * ``utils.fbx_utils``: its ``CreateScene`` records the ``smpl_object`` it is handed and returns True.
So every step after the clustering is the reference's: the rotation, the float32 nearest search, the weight gather,
``inv_lbs``, ``tpose_joints``, the x100 and the colour cast.  Nothing of the reference is copied into this repository.

Inputs: the head of the real template (ref_tree_template.tar.gz) posed by the shipped stand_pose.npy, subdivided three
times (the vertex density of an avatar mesh, so that clustering merges about a third of the vertices), jittered, rotated into the PLY frame, plus two
isolated vertices at (-1, -1, -1) and (1, 1, 1) m around the body (so the voxel is an avatar's, exactly 2^-7 m).  Appended: a
vertex exactly on a voxel boundary, each rotation of one triangle plus its reversed copy, and a degenerate triangle.  SMPL: the tests' synthetic
tensors (seed SMPL_SEED) and a variant with six non-zero weights on every seventh template vertex.

    python -m oracle.pin_avatar2fbx
"""
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

REF = "/root/reference"
REF_A2F = os.path.join(REF, "Avatar2FBX")
REF_AG = os.path.join(REF, "AvatarGen", "AppearanceGen")
GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
SMPL_SEED = 11
MESH_NAME = "avatar"


class _Permissive:
    """Any attribute is a call that returns another permissive object (the FBX SDK's managers and settings)."""

    def __getattr__(self, name):
        return lambda *a, **k: _Permissive()


def _install_stand_ins(recorded: list, smpl_holder: dict):
    from avatarclip_b200 import handoff
    from oracle import export as E

    class _TriangleMesh:
        def __init__(self, vertices, triangles, colors):
            self.vertices = np.asarray(vertices, dtype=np.float64)
            self.triangles = np.asarray(triangles, dtype=np.int64).reshape(-1, 3)
            self.vertex_colors = np.asarray(colors, dtype=np.float64)

        def get_min_bound(self):
            return self.vertices.min(0)

        def get_max_bound(self):
            return self.vertices.max(0)

        def simplify_vertex_clustering(self, voxel_size, contraction):
            assert contraction == "Average"
            v, t, c, _ = E.cluster(self.vertices, self.triangles, self.vertex_colors, voxel=voxel_size)
            return _TriangleMesh(v, t, c)

    def read_triangle_mesh(fname):
        v, f, c = handoff.read_ply(fname)
        return _TriangleMesh(v, f, np.asarray(c, dtype=np.float64) / 255.0)

    o3d = types.ModuleType("open3d")
    o3d.io = types.SimpleNamespace(read_triangle_mesh=read_triangle_mesh)
    o3d.geometry = types.SimpleNamespace(SimplificationContraction=types.SimpleNamespace(Average="Average"),
                                         TriangleMesh=_TriangleMesh)

    fake_lbs = types.ModuleType("smplx.lbs")
    smplx = types.ModuleType("smplx")
    smplx.lbs = fake_lbs

    class _Layer:
        def __init__(self, smpl):
            for k, v in smpl.items():
                setattr(self, k, v)
            self.shapedirs = torch.zeros(smpl["v_template"].shape[0], 3, 10)

        def __call__(self, betas, body_pose, global_orient):
            pu = sys.modules["utils.ply_utils"]
            for k in ("vertices2joints", "blend_shapes", "batch_rigid_transform", "transform_mat", "batch_rodrigues"):
                setattr(fake_lbs, k, getattr(pu, k))
            fake_lbs.__all__ = ["vertices2joints", "blend_shapes", "batch_rigid_transform", "transform_mat",
                                "batch_rodrigues"]
            from models import utils as ref_utils
            full = torch.cat([global_orient, body_pose], dim=1)
            v_shaped = self.v_template[None] + pu.blend_shapes(betas, self.shapedirs)
            verts, joints = ref_utils.my_lbs(v_shaped, full, self.v_template, self.shapedirs, self.posedirs,
                                             self.J_regressor, self.parents, self.lbs_weights, pose2rot=False)
            return {"vertices": verts, "joints": joints}

    smplx.build_layer = lambda folder, **kw: _Layer(smpl_holder["smpl"])
    tqdm = types.ModuleType("tqdm")
    tqdm.tqdm = lambda it, *a, **k: it
    fbx = types.ModuleType("fbx")
    fbx.EXP_FBX_EMBEDDED = "EXP_FBX_EMBEDDED"
    fbx.__all__ = ["EXP_FBX_EMBEDDED"]
    fbx_common = types.ModuleType("FbxCommon")
    fbx_common.InitializeSdkObjects = lambda: (_Permissive(), _Permissive())
    fbx_common.SaveScene = lambda *a, **k: True
    fbx_common.__all__ = []
    fbx_utils = types.ModuleType("utils.fbx_utils")

    def CreateScene(manager, scene, smpl_object):
        recorded.append(smpl_object)
        return True
    fbx_utils.CreateScene = CreateScene
    fbx_utils.__all__ = ["CreateScene"]
    sys.modules.update({"open3d": o3d, "smplx": smplx, "smplx.lbs": fake_lbs, "tqdm": tqdm, "fbx": fbx,
                        "FbxCommon": fbx_common, "utils.fbx_utils": fbx_utils,
                        "neural_renderer": types.ModuleType("neural_renderer")})
    sys.path[:0] = [REF_A2F, REF_AG]


def golden_inputs(smpl: dict, stand_pose: np.ndarray):
    """(v [V,3] float32 PLY frame, f [F,3] int32, c [V,3] uint8, boundary vertex index, isolated vertex index)."""
    from oracle import drive as D
    from oracle import export as E
    rng = np.random.default_rng(7)
    _, tf = D.template_obj()
    posed = D.load_template(smpl, stand_pose)[0].numpy()
    sel = posed[:, 2] > 0.35                   # the head: a small cut, subdivided to an avatar's vertex density
    f = (np.cumsum(sel) - 1)[tf[sel[tf].all(1)]]
    v = posed[sel]
    for _ in range(3):
        v, f = D.subdivide(v, f)
    v = v + rng.normal(0, 5e-4, v.shape).astype(np.float32)
    v = np.stack([v[:, 0], v[:, 2], -v[:, 1]], 1).astype(np.float32)     # D.rotate maps it back
    # two isolated vertices around the whole body's bounds: the voxel is an avatar's, 2 / 256 = 2^-7 exactly
    v = np.concatenate([v, np.full((1, 3), -1.0, np.float32), np.full((1, 3), 1.0, np.float32)])
    vox = E.voxel_size(v)
    lo = -1.0 - vox * 0.5
    assert vox == 2.0 ** -7
    # a vertex of the head moved so that its x lies exactly on a voxel boundary (lo + k * vox is a float32)
    p = v[v.shape[0] // 3].copy()
    bnd = np.array([lo + np.round((p[0] - lo) / vox) * vox, p[1], p[2]], dtype=np.float32)
    q = (np.float64(bnd[0]) - lo) / vox
    assert q == np.floor(q)
    V = v.shape[0]
    v = np.concatenate([v, bnd[None]])
    a, b, c = f[len(f) // 2]
    extra = np.array([[V, a, b], [b, c, a], [c, a, b], [a, b, c], [a, c, b], [a, a, b]])
    f = np.concatenate([f, extra]).astype(np.int32)
    col = rng.integers(0, 256, (v.shape[0], 3), dtype=np.uint8)
    return v, f, col, V, V - 1


def main():
    from avatarclip_b200 import handoff
    from oracle import drive as D
    from oracle import export as E
    smpl = D.golden_smpl(SMPL_SEED)
    wide = E.wide_smpl(smpl)
    stand_path = os.path.join(REF_A2F, "poses", "stand_pose.npy")
    stand_bytes = open(stand_path, "rb").read()
    stand = np.load(stand_path)
    v, f, c, i_bnd, i_iso = golden_inputs(smpl, stand)

    recorded, found = [], []
    holder = {"smpl": smpl}
    _install_stand_ins(recorded, holder)
    import utils.ply_utils as pu                  # export_fbx.py star-imports it: wrap its search to see the indices
    search = pu.find_nearest_ind
    pu.find_nearest_ind = lambda new_vertices, template_object: found.append(
        search(new_vertices, template_object)) or found[-1]
    refs = {}
    for name, s in (("ref", smpl), ("ref_wide", wide)):
        holder["smpl"] = s
        del recorded[:], found[:]
        cwd = os.getcwd()
        with tempfile.TemporaryDirectory() as tmp:
            for d in ("meshes", "poses", "outputs"):
                os.makedirs(os.path.join(tmp, d))
            handoff.write_ply(os.path.join(tmp, "meshes", MESH_NAME + ".ply"), v, f, c)
            open(os.path.join(tmp, "poses", "stand_pose.npy"), "wb").write(stand_bytes)
            try:
                os.chdir(tmp)
                runpy.run_path(os.path.join(REF_A2F, "export_fbx.py"), run_name="__main__")
            finally:
                os.chdir(cwd)
        assert len(recorded) == 1 and len(found) == 1
        obj, nearest = recorded[0], np.asarray(found[0])
        w_ref = np.asarray(obj["blend_weights"]).T                      # [N, 24]
        o = E.smpl_object(v, f, c, s, stand)
        checks = {
            "name": obj["name"] == MESH_NAME,
            "triangles": np.array_equal(o["triangles"], np.asarray(obj["triangles"])),
            "colors": np.array_equal(o["colors"], obj["colors"]),
            "nearest": np.array_equal(o["nearest"], nearest),
            "blend_weights": np.array_equal(s["lbs_weights"][torch.from_numpy(nearest)].numpy(), w_ref),
        }
        e_v = (o["vertices"] - obj["vertices"]).abs().max().item()
        e_j = (o["joints"] - torch.as_tensor(obj["joints"])).abs().max().item()
        print(f"[pin_avatar2fbx] {name}: exact {checks}; max abs err T-pose {e_v:.2e} cm, joints {e_j:.2e} cm")
        assert all(checks.values()) and e_v <= 1e-4 and e_j <= 1e-4
        refs[name] = dict(vertices=obj["vertices"].detach().float(), joints=torch.as_tensor(obj["joints"]).float(),
                          nearest=nearest.astype(np.int32), max_influences=int((w_ref > 0).sum(1).max()))
        if name == "ref":
            refs[name].update(triangles=np.asarray(obj["triangles"]).astype(np.int32), colors=obj["colors"])
    sv = E.simplify(v, f, c)[0]
    lab = E.cluster(v.astype(np.float32), f)[3]
    print(f"[pin_avatar2fbx] mesh {len(v)} -> {len(sv)} vertices, {len(f)} -> {len(refs['ref']['triangles'])} "
          f"triangles; most influences per vertex: {refs['ref']['max_influences']} / {refs['ref_wide']['max_influences']}")
    assert refs["ref_wide"]["max_influences"] > 4
    assert lab[i_iso] not in set(lab[f.reshape(-1)].tolist())        # the isolated vertex is a voxel of its own

    rec = dict(smpl_seed=SMPL_SEED, smpl_sums={k: float(t.double().sum()) for k, t in smpl.items()},
               wide_sum=float(wide["lbs_weights"].double().sum()),
               stand_pose_npy=np.frombuffer(stand_bytes, dtype=np.uint8).copy(),
               mesh=dict(v=v, f=f, c=c, boundary_vertex=i_bnd, isolated_vertex=i_iso), **refs)
    as_t = lambda x: ({k: as_t(t) for k, t in x.items()} if isinstance(x, dict) else
                      torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x)
    os.makedirs(GOLDEN, exist_ok=True)
    torch.save(as_t(rec), os.path.join(GOLDEN, "ref_avatar2fbx_small.pt"))


if __name__ == "__main__":
    main()
