"""The tangent-space normal map on the GPU (avc_bake.cu, bake.bake_normal_map, export's --normal_map): corner tangents
and texel frames against the fp64 oracle (oracle/normal_map.py), the zero-set snap against the oracle's search on the
SDF in fp64, the map's agreement with the SDF's normals, and the export end to end on the small stand-pose checkpoint
of tests/golden/ref_tree_checkpoint.tar."""
import io
import os

import numpy as np
import pytest
import torch

import util_neus as U
from oracle import bake as B
from oracle import drive as D
from oracle import export as E
from oracle import neus
from oracle import normal_map as NM

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_avatar2fbx_small.pt")


@pytest.fixture(scope="module")
def g():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def smpl(g):
    return D.golden_smpl(g["smpl_seed"])


def _deg(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    c = (a * b).sum(-1) / (np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1))
    return np.degrees(np.arccos(np.clip(c, -1, 1)))


# ---------------------------------------------------------------- tangents and frames
def _check_tangents_and_frames(v, f, T, name):
    from avatarclip_b200 import bake
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    nrm = bake.vertex_normals(vt, ft)
    owner, _, uv = bake.texel_points(vt, ft, T)
    tg = bake.corner_tangents(vt, ft, nrm, uv)
    assert torch.equal(tg, bake.corner_tangents(vt, ft, nrm, uv))
    n64, uv64, tg32 = nrm.cpu().double().numpy(), uv.cpu().double().numpy().reshape(-1, 3, 2), tg.cpu().numpy()
    want = NM.corner_tangents(v, f, n64, uv64)
    # conditioning: float32 positions and UV differences, then the Gram-Schmidt's cancellation
    p = v.astype(np.float64)[f]
    e1, e2 = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    du1, dv1 = uv64[:, 1, 0] - uv64[:, 0, 0], uv64[:, 1, 1] - uv64[:, 0, 1]
    du2, dv2 = uv64[:, 2, 0] - uv64[:, 0, 0], uv64[:, 2, 1] - uv64[:, 0, 1]
    tf = e1 * dv2[:, None] - e2 * dv1[:, None]
    nc = n64[f]
    o = np.linalg.norm(tf[:, None] - (tf[:, None] * nc).sum(-1, keepdims=True) * nc, axis=-1)
    scale = np.abs(p).sum((1, 2))[:, None] * (np.abs(du1) + np.abs(dv1) + np.abs(du2) + np.abs(dv2))[:, None]
    cond = np.maximum(1.0, scale / np.maximum(o, 1e-300))
    err = np.abs(tg32[..., :3] - want[..., :3]).max(-1)
    assert (err <= 1e-6 * cond).all(), float((err / cond).max())
    bf = e2 * du1[:, None] - e1 * du2[:, None]
    side = np.abs((np.cross(nc, want[..., :3]) * bf[:, None]).sum(-1)) / np.linalg.norm(bf, axis=-1)[:, None]
    firm = side > 1e-4
    assert np.array_equal(tg32[..., 3][firm], want[..., 3][firm])
    # texel frames from the kernel's tangents and normals
    texels = torch.nonzero(owner >= 0).reshape(-1).int()
    fr = bake.texel_frames(ft, nrm, tg, T, texels).cpu().double().numpy()
    tx = texels.cpu().numpy()
    wfr = NM.texel_frames(f, n64, tg32.astype(np.float64), T, tx)
    own, b = NM.texel_bary(tx, f.shape[0], T)
    Ns = (b[..., None] * n64[f[own]]).sum(1)
    Ti = (b[..., None] * tg32[own][..., :3].astype(np.float64)).sum(1)
    Nu = Ns / np.linalg.norm(Ns, axis=1, keepdims=True)
    oT = np.linalg.norm(Ti - (Ti * Nu).sum(1, keepdims=True) * Nu, axis=1)
    fcond = np.maximum.reduce([np.ones(len(tx)), 1 / np.linalg.norm(Ns, axis=1), np.linalg.norm(Ti, axis=1) / oT])
    wsum = np.abs((b * tg32[own][..., 3]).sum(1))
    ok = wsum > 1e-6
    ferr = np.abs(fr - wfr).max(-1)
    assert (ferr[:, [0, 2]].max(1) <= 2e-6 * fcond).all() and (ferr[ok, 1] <= 4e-6 * fcond[ok]).all()
    U.log_parity(f"normal_bake_frames_{name}", {"F": int(f.shape[0]), "T": T, "texels": int(len(tx)),
                                                "tangent_err_over_cond": float((err / cond).max()),
                                                "frame_err_over_cond": float((ferr.max(1) / fcond).max())})


def test_tangents_and_frames_on_hand_built_meshes():
    quad = (np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float32), np.array([[0, 1, 2], [0, 2, 3]], np.int32))
    _check_tangents_and_frames(*quad, 32, "quad")
    v, f = D.template_obj()
    _check_tangents_and_frames(v.astype(np.float32), f[:999].astype(np.int32), 512, "template_999")
    # a degenerate face (a repeated vertex) takes the fallback frame
    ff = np.concatenate([f[:10], [[0, 0, 1]]]).astype(np.int32)
    _check_tangents_and_frames(v.astype(np.float32), ff, 64, "degenerate")


def test_tangents_and_frames_on_clustered_avatar(g, smpl):
    from avatarclip_b200 import export as X
    from avatarclip_b200.drive import Mesh
    stand = np.load(io.BytesIO(g["stand_pose_npy"].numpy().tobytes()))
    v, f = D.bench_mesh(smpl, stand, levels=1)
    m = X.simplify_mesh(Mesh(torch.from_numpy(v).cuda(), torch.from_numpy(f.astype(np.int32)).cuda(), None), 128)
    _check_tangents_and_frames(m.vertices.cpu().numpy(), m.triangles.cpu().numpy(), 2048, "avatar")


def test_abi_rejects_bad_arguments():
    from avatarclip_b200 import bake
    L = bake._L()
    t = torch.zeros(64, device="cuda")
    p = t.data_ptr()
    E_BADCFG, E_NULL, E_SIZE = -1, -2, -3
    assert L.avc_bake_corner_tangents(p, p, p, None, 3, 1, p, None) == E_NULL
    assert L.avc_bake_corner_tangents(p, p, p, p, 3, 0, p, None) == E_SIZE
    assert L.avc_bake_texel_frames(p, p, p, 3, 1, 7, p, 1, p, None) == E_BADCFG
    assert L.avc_bake_texel_frames(p, p, p, 3, 1, 64, p, 0, p, None) == E_SIZE
    assert L.avc_bake_snap_samples(p, p, 1, 0.0, p, None) == E_BADCFG
    assert L.avc_bake_snap_samples(p, p, 1, float("nan"), p, None) == E_BADCFG
    assert L.avc_bake_snap_bracket(p, 0, 1.0, p, p, None) == E_SIZE
    assert L.avc_bake_snap_midpoints(p, None, p, 1, p, None) == E_NULL
    assert L.avc_bake_snap_bisect(p, 1, p, None, None) == E_NULL
    assert L.avc_bake_normal_encode(p, p, p, p, 1, 0, p, p, None) == E_SIZE
    torch.cuda.synchronize()


# ---------------------------------------------------------------- the NeuS run
def _conf(tmp_path):
    ag = U.reference_tree(tmp_path / "ref")
    text = open(os.path.join(ag, "confs/examples_small/example.conf")).read()
    for old, new in (("./exp/", str(tmp_path / "exp") + "/"), ("./data/", ag + "/data/"),
                     ("./pretrained_models/", ag + "/pretrained_models/")):
        text = text.replace(old, new)
    text = text.replace("        extra_color = True\n", "")
    p = tmp_path / "example.conf"
    p.write_text(text)
    return str(p)


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    """The small stand-pose run, its validate_mesh(resolution=64) mesh decimated to 400 faces, and the SDF in fp64."""
    from avatarclip_b200 import export as X
    from avatarclip_b200.drive import read_ply
    from avatarclip_b200.runner import Runner
    tmp = tmp_path_factory.mktemp("normal_bake_run")
    conf = _conf(tmp)
    r = Runner(conf, "validate_mesh", "smpl", device="cuda")
    r.iter_step = 100
    ply = r.validate_mesh(resolution=64)
    ckpt = r.save_checkpoint()
    m = X.decimate_mesh(read_ply(ply, "cuda"), 400)
    c = dict(r.conf["model.sdf_network"])
    sconf = neus.SDFConf(**{k: (tuple(v) if k == "skip_in" else v) for k, v in c.items()})
    p64 = {k: v.detach().double().cpu() for k, v in r.sdf_network.state_dict().items()}
    return dict(conf=conf, r=r, ply=ply, ckpt=os.path.basename(ckpt), v=m.vertices.contiguous(),
                f=m.triangles.contiguous(), sconf=sconf, p64=p64)


def _sdf64(run, x):
    with torch.no_grad():
        x = torch.as_tensor(np.asarray(x, np.float64))
        return torch.cat([neus.sdf_value(run["p64"], run["sconf"], x[i:i + 32768]).reshape(-1)
                          for i in range(0, x.shape[0], 32768)]).numpy()


def _grad64(run, x):
    x = torch.as_tensor(np.asarray(x, np.float64))
    return torch.cat([neus.sdf_gradient(run["p64"], run["sconf"], x[i:i + 16384], create_graph=False).detach()
                      for i in range(0, x.shape[0], 16384)]).numpy()


def _pipeline(run, T):
    """The kernel's texels, frames, points, snap and map: a dict of host arrays."""
    from avatarclip_b200 import bake
    v, f = run["v"], run["f"]
    owner, pts, uv = bake.texel_points(v, f, T)
    nrm = bake.vertex_normals(v, f)
    used = torch.nonzero(owner >= 0).reshape(-1).int()
    fr = bake.texel_frames(f, nrm, bake.corner_tangents(v, f, nrm, uv), T, used)
    p0 = pts[used.long()].contiguous()
    D = bake.search_length(v, f)
    x, br, st = bake.snap_to_zero_set(run["r"], p0, fr, D)
    image, stats = bake.bake_normal_map(run["r"], v, f, T)
    return dict(texels=used.cpu().numpy(), frames=fr.cpu().double().numpy(), p0=p0.cpu().double().numpy(), D=D,
                x=x.cpu().double().numpy(), bracket=br.cpu().double().numpy(), state=st.cpu().numpy(),
                image=image, stats=stats)


@pytest.fixture(scope="module")
def baked(run):
    return _pipeline(run, 256)


def test_snap_equals_the_fp64_search(run, baked):
    k = baked
    D = k["D"]
    n = k["texels"].size
    assert k["stats"]["used"] == n and 0 < k["stats"]["converged"] <= n
    sample = np.sort(np.random.default_rng(0).choice(n, min(n, 2000), replace=False))
    p0, N = k["p0"][sample], k["frames"][sample, 2]
    # the fp32 chain against fp64 at the sample points bounds where a sign may differ
    pts = (p0[:, None] + NM.offsets(D)[None, :, None] * N[:, None]).reshape(-1, 3).astype(np.float32)
    s32 = run["r"].renderer.sdf_query(torch.from_numpy(pts).cuda()).reshape(-1).cpu().double().numpy()
    s64 = _sdf64(run, pts.astype(np.float64))
    e = float(np.abs(s32 - s64).max())
    bound = 4 * e + 1e-7
    lo, hi, st, x64, s_or = NM.snap(p0, N, D, lambda q: _sdf64(run, q))
    tie = NM.ties(s_or, bound)
    keep = ~tie
    assert keep.mean() > 0.9, keep.mean()
    assert np.array_equal(k["state"][sample][keep], st[keep])
    w = (2 * D / 15) / 2 ** NM.STEPS
    tk = k["bracket"][sample].mean(1)
    t64 = (lo + hi) * 0.5
    gN = np.abs((_grad64(run, x64) * N).sum(1))
    conv = keep & (st != 0)
    tol = 2 * w + 4 * bound / np.maximum(gN, 0.05)
    assert (np.abs(tk - t64)[conv] <= tol[conv]).all(), float((np.abs(tk - t64)[conv] / tol[conv]).max())
    # converged points sit on the zero set within the bisection bound
    kc = k["state"][sample] != 0
    gk = _grad64(run, k["x"][sample][kc])
    assert (np.abs(_sdf64(run, k["x"][sample][kc])) <= np.linalg.norm(gk, axis=1) * w * 0.51 + bound).all()
    U.log_parity("normal_bake_snap", {"texels": int(n), "sampled": int(sample.size), "ties": int(tie.sum()),
                                      "converged": k["stats"]["converged"], "sdf_fp32_err": e, "D": D})


def test_map_bytes_do_not_depend_on_the_chunk(run, baked):
    from avatarclip_b200 import bake
    for chunk in (1000, 4097, 1 << 20):
        img, stats = bake.bake_normal_map(run["r"], run["v"], run["f"], 256, chunk=chunk)
        assert np.array_equal(img, baked["image"]) and stats == baked["stats"], chunk
    img, _ = bake.bake_normal_map(run["r"], run["v"], run["f"], 256)
    assert np.array_equal(img, baked["image"])
    own = B.texel_owner(run["f"].shape[0], 256).reshape(-1)
    assert (baked["image"].reshape(-1, 3)[own < 0] == 0).all()


def test_map_decodes_to_the_sdf_normal_and_beats_the_mesh_normal(run, baked):
    k = baked
    c = np.flatnonzero(k["state"] != 0)
    rgb = k["image"].reshape(-1, 3)[k["texels"][c]]
    fr = k["frames"][c]
    g64 = _grad64(run, k["x"][c])
    live = np.linalg.norm(g64, axis=1) >= 1e-5
    c, rgb, fr, g64 = c[live], rgb[live], fr[live], g64[live]
    ok = (fr[:, 2] * g64).sum(1) > 0                        # back-facing texels are counted, not checked here
    dec = NM.decode(rgb, fr[:, 0], fr[:, 1], fr[:, 2])
    err = _deg(dec, g64)[ok]
    assert err.max() <= 0.5, float(err.max())
    plain = _deg(fr[:, 2], g64)[ok]
    med_map, med_plain = float(np.median(err)), float(np.median(plain))
    print(f"[normal_bake] median angle to the SDF normal: {med_plain:.3f} deg interpolated, {med_map:.3f} deg mapped "
          f"({ok.sum()} texels)")
    U.log_parity("normal_bake_purpose", {"texels": int(ok.sum()), "median_deg_interpolated": med_plain,
                                         "median_deg_mapped": med_map, "max_deg_mapped": float(err.max())})
    assert med_map < 0.25 * med_plain and med_map < 0.5


def _glb_frames(glb, F, T, texels):
    """glTF's decode inputs at texel centres: the primitive's NORMAL and TANGENT interpolated as a viewer does."""
    prim = glb["json"]["meshes"][0]["primitives"][0]
    at = prim["attributes"]
    n = E.accessor(glb, at["NORMAL"]).astype(np.float64).reshape(F, 3, 3)
    t = E.accessor(glb, at["TANGENT"]).astype(np.float64).reshape(F, 3, 4)
    own, b = NM.texel_bary(texels, F, T)
    N = (b[..., None] * n[own]).sum(1)
    N /= np.linalg.norm(N, axis=1, keepdims=True)
    Tt = NM.tangent_against((b[..., None] * t[own][..., :3]).sum(1), N)
    w = np.where((b * t[own][..., 3]).sum(1) >= 0, 1.0, -1.0)
    return Tt, w[:, None] * np.cross(N, Tt), N


def _png(glb, i):
    import cv2 as cv
    j = glb["json"]
    bv = j["bufferViews"][j["images"][i]["bufferView"]]
    return cv.imdecode(np.frombuffer(glb["bin"][bv["byteOffset"]:bv["byteOffset"] + bv["byteLength"]], np.uint8),
                       cv.IMREAD_UNCHANGED)[..., ::-1]


def test_export_with_zero_stand_pose_decodes_to_the_rotated_sdf_normal(run, g, smpl, tmp_path):
    """A zero stand pose makes the un-posing the identity: the bind pose is the PLY frame rotated by (x, -z, y)."""
    from avatarclip_b200 import bake
    from avatarclip_b200 import export as X
    stand = np.load(io.BytesIO(g["stand_pose_npy"].numpy().tobytes()))
    zero = tmp_path / "zero_pose.npy"
    np.save(zero, np.zeros_like(stand))
    T = 256
    out = X.export_avatar(run["ply"], str(tmp_path / "z.glb"), smpl, str(zero), resolution=64, conf=run["conf"],
                          checkpoint=run["ckpt"], texture_size=T, target_faces=400, normal_map=True)
    rig = X.rig_avatar(run["ply"], smpl, str(zero), 64, ply_frame=True, target_faces=400)
    F = rig["triangles"].shape[0]
    glb = E.read_glb(out)
    at = glb["json"]["meshes"][0]["primitives"][0]["attributes"]
    assert all(glb["json"]["accessors"][at[a]]["count"] == 3 * F for a in at)
    uv = E.accessor(glb, at["TEXCOORD_0"]).astype(np.float64)
    assert np.abs(uv - B.uv(F, T).reshape(-1, 2)).max() <= 1e-7
    nmap = _png(glb, 1).reshape(-1, 3)
    kr = dict(run, v=torch.from_numpy(rig["vertices_ply"]).cuda(), f=torch.from_numpy(rig["triangles"]).cuda())
    k = _pipeline(kr, T)
    assert np.array_equal(nmap, k["image"].reshape(-1, 3))
    c = np.flatnonzero(k["state"] != 0)
    c = np.sort(np.random.default_rng(1).choice(c, min(c.size, 3000), replace=False))
    g64 = _grad64(run, k["x"][c])
    rot = np.stack([g64[:, 0], -g64[:, 2], g64[:, 1]], 1)
    Tt, Bt, N = _glb_frames(glb, F, T, k["texels"][c])
    # the frames carry over where the bind pose's normals and tangents are the PLY frame's rotated; a vertex whose
    # face normals nearly cancel, or a degenerate face's fallback axis, may round differently in the two frames
    fr = k["frames"][c]
    fr_rot = np.stack([fr[..., 0], -fr[..., 2], fr[..., 1]], -1)
    same = np.abs(np.stack([Tt, Bt, N], 1) - fr_rot).max((1, 2)) <= 1e-3
    ok = same & ((N * rot).sum(1) > 0) & (np.linalg.norm(g64, axis=1) >= 1e-5)
    dec = NM.decode(nmap[k["texels"][c]], Tt, Bt, N)
    err = _deg(dec, rot)[ok]
    U.log_parity("normal_bake_export_zero_pose", {"faces": F, "texels": int(ok.sum()), "frames_differ":
                                                  int((~same).sum()), "max_deg": float(err.max()),
                                                  "median_deg": float(np.median(err))})
    print(f"[normal_bake] zero stand pose: {ok.sum()} texels within {err.max():.3f} deg; {(~same).sum()} of {c.size} "
          "with frames that differ between the PLY frame and the bind pose")
    assert same.mean() > 0.97 and ok.mean() > 0.9 and err.max() <= 0.5, float(err.max())
    assert bake.search_length(rig["vertices_ply"], rig["triangles"]) > 0


def test_export_with_golden_stand_pose(run, g, smpl, tmp_path):
    from avatarclip_b200 import export as X
    stand = tmp_path / "stand_pose.npy"
    stand.write_bytes(g["stand_pose_npy"].numpy().tobytes())
    out = X.export_avatar(run["ply"], str(tmp_path / "s.glb"), smpl, str(stand), resolution=64, conf=run["conf"],
                          checkpoint=run["ckpt"], texture_size=256, target_faces=400, normal_map=True)
    glb = E.read_glb(out)
    j = glb["json"]
    prim = j["meshes"][0]["primitives"][0]
    at = prim["attributes"]
    n = j["accessors"][at["POSITION"]]["count"]
    assert {"POSITION", "NORMAL", "TANGENT", "TEXCOORD_0"} <= set(at)
    assert all(j["accessors"][at[a]]["count"] == n for a in at) and n % 3 == 0
    assert j["materials"][prim["material"]]["normalTexture"] == {"index": 1, "texCoord": 0}
    t = E.accessor(glb, at["TANGENT"])
    assert np.abs(np.linalg.norm(t[:, :3], axis=1) - 1).max() < 1e-5 and set(np.unique(t[:, 3])) <= {-1.0, 1.0}
    assert _png(glb, 1).shape == (256, 256, 3)
