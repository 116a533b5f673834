"""Mesh animation kernels (avc_drive.cu) against what the reference's drive.py computed (tests/golden/ref_drive_small.pt)
and against host restatements at the size of a shipped avatar mesh."""
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch

import util_neus as U
from oracle import drive as D

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_drive_small.pt")


@pytest.fixture(scope="module")
def g():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def smpl(g):
    s = D.golden_smpl(g["smpl_seed"])
    assert {k: float(v.double().sum()) for k, v in s.items()} == g["smpl_sums"]
    return s


@pytest.fixture(scope="module")
def big(g, smpl):
    """The mesh tools/bench_drive.py times: the template subdivided three times (440 834 vertices), in the SMPL frame."""
    v, f = D.bench_mesh(smpl, np.load(io.BytesIO(g["stand_pose_npy"].numpy().tobytes())), levels=3)
    return D.rotate(v).astype(np.float32), f


def _frames(pc2: bytes, V: int):
    return np.frombuffer(pc2[32:], dtype="<f4").reshape(-1, V, 3)


def _components(v_count, faces):
    from avatarclip_b200 import _lib, drive
    L = drive._L()
    f = torch.as_tensor(faces, dtype=torch.int32).cuda().contiguous()
    need = C.c_size_t()
    _lib.check(L.avc_mesh_components_workspace_bytes(v_count, C.byref(need)), "ws")
    ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    labels = torch.empty(v_count, dtype=torch.int32, device="cuda")
    kept = torch.empty(2, dtype=torch.int32, device="cuda")
    _lib.check(L.avc_mesh_components(_lib.ptr(f) if f.numel() else None, f.shape[0], v_count, _lib.ptr(labels),
                                     _lib.ptr(kept), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "components")
    return labels.cpu().numpy(), kept.cpu().numpy()


# ---------------------------------------------------------------- nearest vertex
def test_nearest_equals_reference(g):
    from avatarclip_b200.drive import find_nearest_ind
    r = g["ref"]
    got = find_nearest_ind(r["cleaned_v"].cuda(), {"vertices": r["template"][None].cuda()})
    assert torch.equal(got.cpu(), r["nearest"].long())


def test_nearest_ties_go_to_first_index():
    from avatarclip_b200.drive import find_nearest_ind
    rng = np.random.default_rng(0)
    ref = rng.normal(0, 1, (1000, 3)).astype(np.float32)       # M not a multiple of the shared-memory tile
    ref[700] = ref[300]
    ref[900] = ref[300]
    ref[999] = ref[5]
    q = np.concatenate([ref[[700, 900, 300, 999, 5]], np.array([[10.0, 0, 0], [-10.0, 0, 0]], np.float32)])
    ref[0], ref[1] = [11.0, 0, 0], [9.0, 0, 0]                  # [10, 0, 0] lies exactly halfway between 0 and 1
    ref[2], ref[3] = [-9.0, 0, 0], [-11.0, 0, 0]                # and [-10, 0, 0] between 2 and 3
    got = find_nearest_ind(torch.from_numpy(q).cuda(), {"vertices": torch.from_numpy(ref).cuda()[None]}).cpu().numpy()
    assert got.tolist() == [300, 300, 300, 5, 5, 0, 2]
    assert got.tolist() == D.find_nearest_ind(q, ref).tolist()


def test_nearest_on_avatar_sized_mesh(g, smpl, big):
    from avatarclip_b200.drive import find_nearest_ind
    v, _ = big
    assert v.shape[0] >= 185428
    tmpl = D.load_template(smpl, np.load(io.BytesIO(g["stand_pose_npy"].numpy().tobytes())))[0]
    got = find_nearest_ind(torch.from_numpy(v).cuda(), {"vertices": tmpl[None].cuda()}).cpu().numpy()
    sub = np.sort(np.random.default_rng(1).choice(v.shape[0], 16384, replace=False))
    assert np.array_equal(got[sub], D.find_nearest_ind(v[sub], tmpl.numpy()))


# ---------------------------------------------------------------- connected components
def test_components_partition_on_avatar_sized_mesh(big):
    v, f = big
    V = v.shape[0]
    # cut the mesh: drop the triangles touching a band of vertices, and add singletons at the end
    drop = np.zeros(V + 5, dtype=bool)
    drop[np.random.default_rng(2).choice(V, 2000, replace=False)] = True
    f = f[~drop[f].any(1)]
    labels, kept = _components(V + 5, f)
    want = D.components(V + 5, f)
    assert np.array_equal(labels, want)                      # labels are the smallest index: same partition
    roots, sizes = np.unique(want, return_counts=True)
    assert kept.tolist() == [roots[np.argmax(sizes)], sizes.max()]
    assert labels[V:].tolist() == list(range(V, V + 5))


def test_components_singletons_only():
    labels, kept = _components(7, np.zeros((0, 3), np.int32))
    assert labels.tolist() == list(range(7)) and kept.tolist() == [0, 1]


def test_cleanup_equals_reference(g):
    from avatarclip_b200.drive import Mesh, cleanup_mesh
    m, r = g["mesh"], g["ref"]
    v = torch.from_numpy(D.rotate(m["v"].numpy()).astype(np.float32)).cuda()
    out = cleanup_mesh(Mesh(v, m["f"].cuda(), m["c"].numpy()))
    assert torch.equal(out.vertices.cpu(), r["cleaned_v"])
    assert torch.equal(out.triangles.cpu(), r["cleaned_f"])
    assert np.array_equal(out.vertex_colors, r["cleaned_c"].numpy())
    t = g["tie"]
    out = cleanup_mesh(Mesh(t["v"].cuda(), t["f"].cuda(), t["c"].numpy()))
    assert torch.equal(out.vertices.cpu(), t["cleaned_v"]) and torch.equal(out.triangles.cpu(), t["cleaned_f"])
    assert np.array_equal(out.vertex_colors, t["cleaned_c"].numpy())


# ---------------------------------------------------------------- inverse LBS, LBS, chunked frames
def test_inv_lbs_and_lbs_match_reference(g, smpl):
    from avatarclip_b200.drive import inv_lbs, lbs
    r = g["ref"]
    s = {k: v.cuda() for k, v in smpl.items()}
    w = s["lbs_weights"][r["nearest"].long().cuda()]
    beta = torch.zeros(1, 10)
    tpose = inv_lbs(s, r["cleaned_v"].cuda(), w, r["pose_rot"].cuda(), beta)
    e_t = (tpose.cpu() - r["tpose"]).abs().max().item()
    frames = _frames(r["pc2"].numpy().tobytes(), len(r["cleaned_v"]))
    e_f = max(np.abs(lbs(s, r["tpose"].cuda(), w, r["pose_list"][i:i + 1].cuda(), beta).cpu().numpy() - frames[i]).max()
              for i in range(len(frames)))
    back = lbs(s, tpose, w, r["pose_rot"].cuda(), beta)          # skinning the un-posed mesh by the stand pose
    e_b = (back.cpu() - r["cleaned_v"]).abs().max().item()
    U.log_parity("drive_inv_lbs_lbs", {"tpose": e_t, "frames": float(e_f), "round_trip": e_b})
    assert e_t <= 1e-5 and e_f <= 1e-5 and e_b <= 1e-5
    with pytest.raises(NotImplementedError):
        inv_lbs(s, r["cleaned_v"].cuda(), w, r["pose_rot"].cuda(), torch.ones(1, 10))


def _write_inputs(g, tmp_path):
    from avatarclip_b200 import handoff
    m = g["mesh"]
    ply = handoff.write_ply(str(tmp_path / "General.ply"), m["v"].numpy(), m["f"].numpy(), m["c"].numpy())
    motion = str(tmp_path / "raising_both_arms.npy")
    np.save(motion, g["motion"].numpy())
    stand = tmp_path / "stand_pose.npy"
    stand.write_bytes(g["stand_pose_npy"].numpy().tobytes())
    return ply, motion, str(stand)


def test_generate_animation_end_to_end(g, smpl, tmp_path):
    from avatarclip_b200 import handoff
    from avatarclip_b200.drive import find_nearest_ind, generate_animation, load_template_smpl
    r = g["ref"]
    ply, motion, stand = _write_inputs(g, tmp_path)
    out_ply, out_pc2 = generate_animation(ply, motion, str(tmp_path / "out"), smpl, stand)
    assert os.path.basename(out_ply) == "General_cleaned_apose.ply"
    assert os.path.basename(out_pc2) == "raising_both_arms.pc2"
    v, f, c = handoff.read_ply(out_ply)
    assert np.array_equal(v, r["cleaned_v"].numpy()) and np.array_equal(f, r["cleaned_f"].numpy())
    assert np.array_equal(c, r["cleaned_c"].numpy())
    pc2, ref_pc2 = open(out_pc2, "rb").read(), r["pc2"].numpy().tobytes()
    assert pc2[:32] == ref_pc2[:32] and len(pc2) == len(ref_pc2)
    # the template comes from avc_lbs_fwd, whose last bits may differ from the reference's: a near-tie may pick another
    # template vertex.  Vertices whose index agrees must agree to 1e-5.
    tmpl, _, _ = load_template_smpl(smpl, stand)
    near = find_nearest_ind(r["cleaned_v"].cuda(), tmpl).cpu()
    same = (near == r["nearest"].long()).numpy()
    n_diff = int((~same).sum())
    V = len(r["cleaned_v"])
    err = np.abs(_frames(pc2, V) - _frames(ref_pc2, V))[:, same].max()
    U.log_parity("drive_generate_animation", {"nearest_differ": n_diff, "of": V, "frames_err": float(err)})
    print(f"[drive] nearest indices differing from the reference: {n_diff} of {V}; frames max abs err {err:.2e}")
    assert same.mean() >= 0.999 and err <= 1e-5


def test_chunked_frames_write_the_same_file(g, smpl, tmp_path):
    from avatarclip_b200.drive import generate_animation
    ply, _, stand = _write_inputs(g, tmp_path)
    motion = str(tmp_path / "long.npy")
    np.save(motion, np.random.default_rng(3).normal(0, 0.3, (37, 72)).astype(np.float32))
    _, one = generate_animation(ply, motion, str(tmp_path / "a"), smpl, stand, frames_per_chunk=37)
    _, many = generate_animation(ply, motion, str(tmp_path / "b"), smpl, stand, frames_per_chunk=5)
    assert open(one, "rb").read() == open(many, "rb").read()


# ---------------------------------------------------------------- argument checks
def test_abi_rejects_bad_arguments():
    from avatarclip_b200 import drive
    L = drive._L()
    t = torch.zeros(64, 32, device="cuda")
    p = C.c_void_p(t.data_ptr())
    sz = C.c_size_t()
    E_BADCFG, E_NULL, E_SIZE = -1, -2, -3
    assert L.avc_nearest_vertex(None, 4, p, 4, p, None) == E_NULL
    assert L.avc_nearest_vertex(p, 4, p, 0, p, None) == E_SIZE
    assert L.avc_nearest_vertex(p, 0, p, 4, p, None) == E_SIZE
    assert L.avc_mesh_components_workspace_bytes(0, C.byref(sz)) == E_SIZE
    assert L.avc_mesh_components_workspace_bytes(4, None) == E_NULL
    assert L.avc_mesh_components(None, 3, 4, p, p, p, 1024, None) == E_NULL
    assert L.avc_mesh_components(p, 3, 4, p, p, p, 1, None) == E_SIZE
    assert L.avc_mesh_components(p, -1, 4, p, p, p, 1024, None) == E_SIZE
    assert L.avc_lbs_rel_transforms(p, p, p, 8, 33, p, 1, 1, p, p, None) == E_BADCFG
    assert L.avc_lbs_rel_transforms(p, p, p, 8, 0, p, 1, 1, p, p, None) == E_BADCFG
    assert L.avc_lbs_rel_transforms(p, p, p, 8, 24, p, 1, 0, p, p, None) == E_SIZE
    assert L.avc_lbs_rel_transforms(p, None, p, 8, 24, p, 1, 1, p, p, None) == E_NULL
    assert L.avc_inv_lbs(p, None, 8, p, 4, 24, p, p, None) == E_SIZE           # no gather: needs a row per vertex
    assert L.avc_inv_lbs(p, p, 8, p, 4, 40, p, p, None) == E_BADCFG
    assert L.avc_inv_lbs(p, p, 8, None, 4, 24, p, p, None) == E_NULL
    assert L.avc_lbs_frames(p, p, 8, p, 4, 24, p, 5, 3, 3, p, None) == E_SIZE   # frames 3..5 of 5
    assert L.avc_lbs_frames(p, p, 8, p, 4, 24, p, 5, -1, 2, p, None) == E_SIZE
    assert L.avc_lbs_frames(p, p, 8, p, 4, 24, p, 5, 0, 0, p, None) == E_SIZE
    assert L.avc_lbs_frames(p, p, 8, p, 4, 0, p, 5, 0, 1, p, None) == E_BADCFG
    assert L.avc_lbs_frames(p, p, 8, p, 4, 24, p, 5, 0, 1, None, None) == E_NULL
    torch.cuda.synchronize()


def test_cpu_tensors_raise(g, smpl):
    from avatarclip_b200 import AvcError
    from avatarclip_b200 import drive
    with pytest.raises(AvcError):
        drive.find_nearest_ind(g["ref"]["cleaned_v"].cuda(), {"vertices": g["ref"]["template"][None]})
    with pytest.raises(AvcError):
        drive.cleanup_mesh(drive.Mesh(g["mesh"]["v"], g["mesh"]["f"], None))
