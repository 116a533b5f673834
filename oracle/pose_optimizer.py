"""CPU oracle (test infrastructure, never on the product path): the backward of AvatarAnimate's PoseOptimizer chain
(models/pose_generation.py:102-135) in fp64 -- the textured rasteriser's gradient (neural_renderer's, Kato et al.
2018: the light, ``backward_pixel_map``'s edge sweep and the projection), SMPL's gradient by torch autograd through
``oracle.lbs.my_lbs``, the nearest-resize backward and the pose CLIP loss.

PARITY UNPINNED for the rasteriser's gradient: neural_renderer is neither vendored by the reference nor installed, so
``backward_pixel_map`` is restated from its published algorithm.  The sweep takes the face-index map and the
supersampled colour map as inputs, so a device kernel can be checked on its own maps; the pixel choices (pixel
coordinates, edge crossings and their floor / ceil) are made in fp32 one rounded operation at a time, as the device
makes them, and every sum is fp64.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import lbs as olbs
from oracle import shapegen as OS

EPS = 1e-4                      # neural_renderer's DEFAULT_EPS
ROT = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])   # render.py:25-28, applied as v @ ROT
GLOBAL_ORIENT = (math.pi / 2, 0.0, 0.0)
f32 = np.float32


def edge_sweep(pxy, f: int, fidx: np.ndarray, rgb: np.ndarray, g: np.ndarray, eps: float = EPS, skip=()) -> np.ndarray:
    """backward_pixel_map of face f (rgb only) -> d loss / d (x, y) [3, 2] (fp64) of its corners pxy [3, 2] (NDC, in
    the winding of the drawn copy).  fidx [is, is] the face-index map (-1 background), rgb [is, is, 3] the supersampled
    colour map, g [is, is, 3] the gradient at each supersample; row 0 at the top.  An edge whose end points share the
    swept coordinate contributes nothing; an opposite edge parallel to the sweep bounds the in-sweep at the edge pixel.
    ``skip`` lists (edge, axis) parts to leave out (edge e runs from corner e to corner e + 1; axis 0 sweeps columns)."""
    is_ = fidx.shape[0]
    fis = f32(is_)
    pxy = np.asarray(pxy, dtype=f32)
    pp = f32(0.5) * ((pxy * fis + fis) - f32(1.0))        # each operation rounded to fp32
    out = np.zeros((3, 2))
    rgb = np.asarray(rgb, dtype=np.float64)
    g = np.asarray(g, dtype=np.float64)
    for e in range(3):
        pi = (e, (e + 1) % 3, (e + 2) % 3)
        for axis in range(2):
            if (e, axis) in skip:
                continue
            p = np.array([[pp[k][axis], pp[k][1 - axis]] for k in pi], dtype=f32)
            if p[0, 0] == p[1, 0]:
                continue
            direction = -1 if p[0, 0] < p[1, 0] else 1
            if axis == 1:
                direction = -direction
            span = f32(p[1, 0] - p[0, 0])
            slope = f32(f32(p[1, 1] - p[0, 1]) / span)
            d0_from = max(int(math.ceil(min(p[0, 0], p[1, 0]))), 0)
            d0_to = min(int(math.floor(max(p[0, 0], p[1, 0]))), is_ - 1)
            for d0 in range(d0_from, d0_to + 1):
                fd0 = f32(d0)
                d1_cross = f32(f32(slope * f32(fd0 - p[0, 0])) + p[0, 1])
                d1_in = int(math.floor(d1_cross)) if direction > 0 else int(math.ceil(d1_cross))
                d1_out = d1_in + direction
                if not (0 <= d1_in < is_ and 0 <= d1_out < is_):
                    continue
                if axis == 0:
                    pix = lambda d1: (is_ - 1 - d1, np.full_like(d1, d0))
                else:
                    pix = lambda d1: (np.full_like(d1, is_ - 1 - d0), d1)
                rin, rout = rgb[pix(np.array(d1_in))], rgb[pix(np.array(d1_out))]
                P0, P1, D0, DC = float(p[0, 0]), float(p[1, 0]), float(d0), float(d1_cross)

                def add(d1, diff):          # the pixels d1 [k] with their diff [k] > 0
                    base = (d1 - DC) * 2.0 / is_
                    if P1 != D0:
                        dist = (P1 - P0) / (P1 - D0) * base
                        dist = np.where(dist > 0, dist + eps, dist - eps)
                        out[pi[0], 1 - axis] -= (diff / dist).sum()
                    if P0 != D0:
                        dist = (P1 - P0) / (D0 - P0) * base
                        dist = np.where(dist > 0, dist + eps, dist - eps)
                        out[pi[1], 1 - axis] -= (diff / dist).sum()

                if fidx[pix(np.array(d1_in))] == f:                # out: to the border
                    lim = is_ - 1 if direction > 0 else 0
                    d1 = np.arange(min(d1_out, lim), max(d1_out, lim) + 1)
                    r, c = pix(d1)
                    diff = ((rgb[r, c] - rin) * g[r, c]).sum(1)
                    add(d1[diff > 0], diff[diff > 0])
                with np.errstate(divide="ignore", invalid="ignore"):  # in: to the opposite edge, f's pixels
                    if (fd0 - p[0, 0]) * (fd0 - p[2, 0]) < 0:
                        c2 = f32(f32(f32(f32(p[2, 1] - p[0, 1]) / f32(p[2, 0] - p[0, 0])) * f32(fd0 - p[0, 0])) + p[0, 1])
                    else:
                        c2 = f32(f32(f32(f32(p[1, 1] - p[2, 1]) / f32(p[1, 0] - p[2, 0])) * f32(fd0 - p[2, 0])) + p[2, 1])
                lim = d1_in
                if np.isfinite(c2):
                    lim = int(min(max(math.ceil(c2) if direction > 0 else math.floor(c2), -1), is_))
                d1 = np.arange(max(min(d1_in, lim), 0), min(max(d1_in, lim), is_ - 1) + 1)
                r, c = pix(d1)
                diff = ((rgb[r, c] - rout) * g[r, c]).sum(1)
                sel = (fidx[r, c] == f) & (diff > 0)
                add(d1[sel], diff[sel])
    return out


def face_light(v0, v1, v2, eye):
    """(light, s, n) of render.py's lighting for one face in fp64."""
    a, b = v0 - v1, v2 - v1
    n = np.cross(a, b)
    nl = max(np.linalg.norm(n), 1e-5)
    s = 1.0 if np.dot(n, eye - v1) >= 0 else -1.0
    return 0.5 + 0.5 * max(s * n[1] / nl, 0.0), s, n


def light_backward(v0, v1, v2, eye, dlight):
    """d loss / d (v0, v1, v2) [3, 3] of light = 0.5 + 0.5 relu(s n_y / max(|n|, 1e-5)) given d loss / d light."""
    _, s, _ = face_light(v0, v1, v2, eye)
    with torch.enable_grad():                  # also when called from inside an autograd backward
        t = torch.tensor(np.stack([v0, v1, v2]), dtype=torch.float64, requires_grad=True)
        a, b = t[0] - t[1], t[2] - t[1]
        n = torch.linalg.cross(a, b)
        light = 0.5 + 0.5 * torch.relu(s * n[1] / torch.clamp(torch.linalg.norm(n), min=1e-5))
        (light * dlight).backward()
    return t.grad.numpy()


def raster_backward_image(verts, faces, proj, eye, rot, fidx, rgb_ss, g_rgb, ss: int) -> np.ndarray:
    """d loss / d verts [V, 3] (fp64) of one image from its device maps: proj [V, 3] the projected (x_ndc, y_ndc, z_cam),
    eye / rot the look_at camera (rot's columns are the camera axes, as OS.look_at_camera returns), fidx [is, is],
    rgb_ss [is, is, 3] the supersampled lit colours, g_rgb [n, n, 3] the image gradient."""
    v = np.asarray(verts, dtype=np.float64)
    faces = np.asarray(faces, dtype=np.int64)
    is_ = fidx.shape[0]
    g_ss = np.repeat(np.repeat(np.asarray(g_rgb, dtype=np.float64), ss, 0), ss, 1) / (ss * ss)
    inv_w = 1.0 / np.tan(np.deg2rad(30.0))
    out = np.zeros_like(v)
    for f in np.unique(fidx[fidx >= 0]):
        idx = faces[f]
        # (a) light: d light = sum over f's supersamples of g_ss . (lit / light)
        light, _, _ = face_light(v[idx[0]], v[idx[1]], v[idx[2]], eye)
        m = fidx == f
        dlight = float((g_ss[m] * np.asarray(rgb_ss, dtype=np.float64)[m]).sum()) / light
        out[idx] += light_backward(v[idx[0]], v[idx[1]], v[idx[2]], eye, dlight)
    for f in np.unique(fidx[fidx >= 0]):       # a face that wins no supersample gets no gradient
        idx = faces[f]
        q = np.asarray(proj, dtype=f32)[idx]
        if (q[:, 2] <= 0).any():
            continue
        front = (q[2, 1] - q[0, 1]) * (q[1, 0] - q[0, 0]) >= (q[1, 1] - q[0, 1]) * (q[2, 0] - q[0, 0])
        order = [0, 1, 2] if front else [2, 1, 0]
        gxy = edge_sweep(q[order, :2], f, fidx, rgb_ss, g_ss)
        # (c) projection: x' = x_c / z_c / tan 30, c = (v - eye) @ rot
        for k, o in enumerate(order):
            x, y, z = (float(c) for c in q[o])
            gc = np.array([gxy[k, 0] * inv_w / z, gxy[k, 1] * inv_w / z, -(gxy[k, 0] * x + gxy[k, 1] * y) / z])
            out[idx[o]] += rot @ gc
    return out


def smpl_pose_grad(s: dict, body_pose, g_verts, global_orient=GLOBAL_ORIENT, post_rot=ROT) -> np.ndarray:
    """d loss / d body_pose [B, P] of SMPL (zero betas) times post_rot, given g_verts [B, V, 3]: torch fp64 autograd
    through oracle.lbs.my_lbs."""
    dt = torch.float64
    bp = torch.tensor(np.asarray(body_pose, dtype=np.float64), dtype=dt, requires_grad=True)
    B, P = bp.shape
    nj = np.asarray(s["J_regressor"]).shape[0]
    full = torch.cat([torch.tensor(global_orient, dtype=dt).expand(B, 3), bp,
                      torch.zeros(B, 3 * (nj - 1) - P, dtype=dt)], 1)
    v_t = torch.as_tensor(np.asarray(s["v_template"]), dtype=dt)
    verts, _ = olbs.my_lbs(v_t[None].expand(B, -1, -1), full, torch.as_tensor(np.asarray(s["posedirs"]), dtype=dt),
                           torch.as_tensor(np.asarray(s["J_regressor"]), dtype=dt),
                           torch.as_tensor(np.asarray(s["parents"]), dtype=torch.long),
                           torch.as_tensor(np.asarray(s["lbs_weights"]), dtype=dt))
    if post_rot is not None:
        verts = verts @ torch.as_tensor(np.asarray(post_rot), dtype=dt)
    (verts * torch.as_tensor(np.asarray(g_verts), dtype=dt)).sum().backward()
    return bp.grad.numpy()


def clip_prep_nearest_bwd(g_out, n: int) -> np.ndarray:
    """d loss / d images [B, n, n, 3] of OS.clip_prep_nearest given g_out [B, 3, S, S]."""
    g = np.asarray(g_out, dtype=np.float64)
    B, _, S, _ = g.shape
    idx = np.minimum(np.floor(np.arange(S, dtype=f32) * (f32(n) / f32(S))).astype(np.int64), n - 1)
    out = np.zeros((B, n, n, 3))
    gs = g / np.asarray(OS.CLIP_STD, dtype=np.float64)[None, :, None, None]
    for y in range(S):
        for x in range(S):
            out[:, idx[y], idx[x], :] += gs[:, :, y, x]
    return out


def pose_clip_loss(emb, text):
    """(loss [B], g_emb [A, B, D]) of loss[b] = 1 - F.cosine_similarity(mean_a emb[a][b], text, eps=1e-8) in fp64."""
    e = torch.tensor(np.asarray(emb, dtype=np.float64), requires_grad=True)
    t = torch.as_tensor(np.asarray(text, dtype=np.float64)).reshape(1, -1)
    loss = 1 - F.cosine_similarity(e.mean(0), t.expand(e.shape[1], -1), dim=1, eps=1e-8)
    loss.sum().backward()
    return loss.detach().numpy(), e.grad.numpy()


def raster_maps(verts, faces, textures, eye, n: int = 256, ss: int = 2):
    """oracle/shapegen.py's textured render with the maps its backward reads: (rgb [n, n, 3], fidx [is, is], rgb_ss
    [is, is, 3], proj [V, 3]) in fp64.  The supersamples are the pixels of the same render at n ss with one sample
    each; the face of each supersample is read from a render whose texture holds the face's index + 1, divided by a
    render whose texture is 1 (both are that face's light times the constant)."""
    v = np.asarray(verts, dtype=np.float64)
    tex = np.asarray(textures, dtype=np.float64)
    is_ = n * ss
    rgb_ss = OS.raster_textured(v, faces, tex, eye, n=is_, ss=1)
    ids = np.broadcast_to((np.arange(tex.shape[0], dtype=np.float64) + 1)[:, None, None, None, None], tex.shape)
    lid = OS.raster_textured(v, faces, ids, eye, n=is_, ss=1)[..., 0]
    light = OS.raster_textured(v, faces, np.ones_like(tex), eye, n=is_, ss=1)[..., 0]
    fidx = np.where(light > 0, np.rint(lid / np.where(light > 0, light, 1.0)) - 1, -1).astype(np.int64)
    e, rot = OS.look_at_camera(eye)
    cam = (v - e) @ rot
    w = np.tan(np.deg2rad(30.0))
    proj = np.stack([cam[:, 0] / cam[:, 2] / w, cam[:, 1] / cam[:, 2] / w, cam[:, 2]], 1)
    return rgb_ss.reshape(n, ss, n, ss, 3).mean(axis=(1, 3)), fidx, rgb_ss, proj
