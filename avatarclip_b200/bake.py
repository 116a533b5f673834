"""Bake the NeuS colour field of a trained avatar into a texture for its exported mesh.

``bake_texture`` lays the clustered mesh's faces out on a closed-form atlas (``avc_bake_texel_points``: faces 2k and
2k + 1 share square cell k of a T x T texture, each on its side of the cell's diagonal), puts every used texel's centre
on its face's surface in the PLY (NeuS) frame, and colours it the way ``Runner.validate_mesh`` colours a vertex
(``Runner.surface_colors``: the best of six axis views, ``to8b``).  The renders use mid-bin samples (no jitter), so a
texel's bytes depend on its point alone.  ``export.write_glb`` stores the result as an sRGB PNG with ``TEXCOORD_0`` and
smooth ``NORMAL``s (``vertex_normals``).

``bake_normal_map`` bakes the SDF's own normals into a tangent-space normal map on the same atlas, so a reduced mesh
shades with the trained surface's detail.  Each used texel gets a (T, B, N) frame (``corner_tangents``: dP/du per face
corner, MikkTSpace's result for an atlas where every face is its own island; ``texel_frames``: interpolated at the
texel centre), searches the segment p + t N, t in [-D, D], D = 2 x the mesh's mean edge length, for the SDF's zero set
(16 samples, the sign change nearest t = 0, 12 bisection steps, all through ``avc_neus_sdf_query``), and stores the
SDF gradient at the snapped point in its frame as glTF's normalTexture bytes.  Texels with no sign change keep the
flat (128, 128, 255).  The colour texture's points are not snapped: that would change its bytes.

Not done: chart-based unwrapping or area-proportional packing (every face gets the same cell area), mipmap-safe gutters
(the sampler has no mipmaps), and occlusion or curvature maps.
"""
from __future__ import annotations

import ctypes as C
import time

import numpy as np
import torch

from . import _lib, video
from .drive import _cuda, _f32

DEFAULT_TEXTURE_SIZE = 2048
MIN_CELL = 8                 # texels per cell side (avc_bake_atlas_grid)
MAX_TEXTURE_SIZE = 16384
RAY_CHUNK = 1 << 16          # rays per render call of the bake
POINT_CHUNK = 1 << 21        # texel points per surface_colors call: bounds the six views' colour and depth buffers
SNAP_SAMPLES = 16            # search samples per texel (avc_bake_snap_samples)
SNAP_STEPS = 12              # bisection steps of the zero-set search
SNAP_CHUNK = 1 << 18         # texels per sample-evaluation pass: bounds the [chunk, 16, 3] sample points

_bound = None


class AtlasTooSmall(ValueError):
    """The texture is too small for the faces: its cells would be narrower than MIN_CELL texels."""


def _L():
    global _bound
    L = _lib.lib()
    if _bound is None:
        vp, i32 = C.c_void_p, C.c_int32
        L.avc_bake_atlas_grid.argtypes = [i32, i32, C.POINTER(i32), C.POINTER(i32)]
        L.avc_bake_texel_points.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, vp]
        L.avc_bake_vertex_normals.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
        L.avc_bake_corner_tangents.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
        L.avc_bake_texel_frames.argtypes = [vp, vp, vp, i32, i32, i32, vp, i32, vp, vp]
        L.avc_bake_snap_samples.argtypes = [vp, vp, i32, C.c_float, vp, vp]
        L.avc_bake_snap_bracket.argtypes = [vp, i32, C.c_float, vp, vp, vp]
        L.avc_bake_snap_midpoints.argtypes = [vp, vp, vp, i32, vp, vp]
        L.avc_bake_snap_bisect.argtypes = [vp, i32, vp, vp, vp]
        L.avc_bake_normal_encode.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp]
        for n in ("avc_bake_atlas_grid", "avc_bake_texel_points", "avc_bake_vertex_normals", "avc_bake_corner_tangents",
                  "avc_bake_texel_frames", "avc_bake_snap_samples", "avc_bake_snap_bracket", "avc_bake_snap_midpoints",
                  "avc_bake_snap_bisect", "avc_bake_normal_encode"):
            getattr(L, n).restype = C.c_int
        _bound = L
    return L


def atlas_grid(F: int, texture_size: int):
    """(m, c) of the atlas: an m x m grid of cells c texels wide.  Raises AtlasTooSmall when the cells would be
    narrower than MIN_CELL texels, naming the smallest texture size that fits."""
    m, c = C.c_int32(), C.c_int32()
    rc = _L().avc_bake_atlas_grid(int(F), int(texture_size), C.byref(m), C.byref(c))
    if rc == -1:
        raise AtlasTooSmall(f"a {texture_size} x {texture_size} texture gives the {F} faces cells of {c.value} texels; "
                         f"they need at least {MIN_CELL}.  The smallest texture size that fits is {MIN_CELL * m.value}; "
                         "or lower --resolution for fewer faces")
    _lib.check(rc, "avc_bake_atlas_grid")
    return m.value, c.value


def texel_points(vertices: torch.Tensor, triangles: torch.Tensor, texture_size: int, with_uv: bool = True):
    """``avc_bake_texel_points``: (owner [T*T] int32, points [T*T,3] float32, uv [3F,2] float32 or None) on the device."""
    device = _cuda(vertices.device)
    v = _f32(vertices, device).reshape(-1, 3)
    f = triangles.to(device, torch.int32).contiguous().reshape(-1, 3)
    T = int(texture_size)
    atlas_grid(f.shape[0], T)
    owner = torch.empty(T * T, dtype=torch.int32, device=device)
    points = torch.empty(T * T, 3, dtype=torch.float32, device=device)
    uv = torch.empty(f.shape[0] * 3, 2, dtype=torch.float32, device=device) if with_uv else None
    _lib.check(_L().avc_bake_texel_points(_lib.ptr(v), _lib.ptr(f), v.shape[0], f.shape[0], T, _lib.ptr(owner),
                                          _lib.ptr(points), _lib.ptr(uv), _lib.stream_ptr()), "avc_bake_texel_points")
    return owner, points, uv


def vertex_normals(vertices, triangles) -> torch.Tensor:
    """``avc_bake_vertex_normals`` on device tensors: unit smooth normals [V,3] (face cross products summed in face
    order)."""
    device = _cuda(torch.as_tensor(vertices).device)
    v = _f32(torch.as_tensor(vertices), device).reshape(-1, 3)
    f = torch.as_tensor(triangles).to(device, torch.int32).contiguous().reshape(-1, 3)
    adj = video.adjacency(f, v.shape[0])
    out = torch.empty(v.shape[0], 3, dtype=torch.float32, device=device)
    _lib.check(_L().avc_bake_vertex_normals(_lib.ptr(v), _lib.ptr(f), _lib.ptr(adj.offsets), _lib.ptr(adj.vf),
                                            v.shape[0], f.shape[0], _lib.ptr(out), _lib.stream_ptr()),
               "avc_bake_vertex_normals")
    return out


def bake_texture(runner, vertices_ply_frame, triangles, texture_size: int = DEFAULT_TEXTURE_SIZE,
                 ray_chunk: int = RAY_CHUNK, point_chunk: int = POINT_CHUNK):
    """The atlas of ``triangles`` over ``vertices_ply_frame`` (the clustered mesh before ``rig_avatar``'s rotation and
    un-posing) and its colours from ``runner``'s NeuS field -> (uv [3F,2] float32, texture uint8 [T,T,3] RGB, row 0
    at the top), host arrays.  Unused texels are 0."""
    device = _cuda(runner.device)
    v = _f32(torch.as_tensor(vertices_ply_frame), device).reshape(-1, 3)
    f = torch.as_tensor(triangles).to(device, torch.int32).reshape(-1, 3)
    T = int(texture_size)
    owner, points, uv = texel_points(v, f, T)
    used = torch.nonzero(owner >= 0).reshape(-1)
    texture = np.zeros((T * T, 3), dtype=np.uint8)
    idx = used.cpu().numpy()
    for s in range(0, used.numel(), point_chunk):
        texture[idx[s:s + point_chunk]] = runner.surface_colors(points[used[s:s + point_chunk]], chunk=ray_chunk,
                                                                perturb=0)
    return uv.cpu().numpy(), texture.reshape(T, T, 3)


def corner_tangents(vertices, triangles, normals, uv) -> torch.Tensor:
    """``avc_bake_corner_tangents`` on device tensors: [F,3,4] per face corner the unit tangent (dP/du Gram-Schmidt'd
    against the corner's normal) and the handedness w = +-1 (B = w cross(N, T) points towards the image's top)."""
    device = _cuda(torch.as_tensor(vertices).device)
    v = _f32(torch.as_tensor(vertices), device).reshape(-1, 3)
    f = torch.as_tensor(triangles).to(device, torch.int32).contiguous().reshape(-1, 3)
    n = _f32(torch.as_tensor(normals), device).reshape(-1, 3)
    w = _f32(torch.as_tensor(uv), device).reshape(-1, 3, 2)
    if n.shape[0] != v.shape[0] or w.shape[0] != f.shape[0]:
        raise ValueError(f"corner_tangents: normals [{v.shape[0]}, 3] and uv [{3 * f.shape[0]}, 2] expected, got "
                         f"{list(n.shape)} and {list(w.reshape(-1, 2).shape)}")
    out = torch.empty(f.shape[0], 3, 4, dtype=torch.float32, device=device)
    _lib.check(_L().avc_bake_corner_tangents(_lib.ptr(v), _lib.ptr(f), _lib.ptr(n), _lib.ptr(w), v.shape[0],
                                             f.shape[0], _lib.ptr(out), _lib.stream_ptr()), "avc_bake_corner_tangents")
    return out


def texel_frames(triangles, normals, tangents, texture_size: int, texels) -> torch.Tensor:
    """``avc_bake_texel_frames``: [n,3,3] rows T, B, N of the texels (indices y T + x) on the device."""
    device = _cuda(torch.as_tensor(normals).device)
    f = torch.as_tensor(triangles).to(device, torch.int32).contiguous().reshape(-1, 3)
    n = _f32(torch.as_tensor(normals), device).reshape(-1, 3)
    tg = _f32(torch.as_tensor(tangents), device).reshape(-1, 3, 4)
    idx = torch.as_tensor(texels).to(device, torch.int32).contiguous().reshape(-1)
    out = torch.empty(idx.numel(), 3, 3, dtype=torch.float32, device=device)
    _lib.check(_L().avc_bake_texel_frames(_lib.ptr(f), _lib.ptr(n), _lib.ptr(tg), n.shape[0], f.shape[0],
                                          int(texture_size), _lib.ptr(idx), idx.numel(), _lib.ptr(out),
                                          _lib.stream_ptr()), "avc_bake_texel_frames")
    return out


def search_length(vertices, triangles) -> float:
    """D of the zero-set search: 2 x the mean length of the faces' edges (fp64 on the host)."""
    v = torch.as_tensor(vertices).detach().cpu().double().reshape(-1, 3)
    f = torch.as_tensor(triangles).detach().cpu().long().reshape(-1, 3)
    p = v[f]
    e = torch.cat([p[:, 1] - p[:, 0], p[:, 2] - p[:, 1], p[:, 0] - p[:, 2]])
    return 2.0 * float(e.norm(dim=1).mean())


def _sdf(runner, pts: torch.Tensor, chunk: int) -> torch.Tensor:
    """``avc_neus_sdf_query`` on [P,3] points, ``chunk`` points per call -> [P]."""
    out = torch.empty(pts.shape[0], dtype=torch.float32, device=pts.device)
    for s in range(0, pts.shape[0], chunk):
        out[s:s + chunk] = runner.renderer.sdf_query(pts[s:s + chunk]).reshape(-1)
    return out


def snap_to_zero_set(runner, points, frames, D: float, chunk: int = SNAP_CHUNK, timings: dict | None = None):
    """The zero-set search of ``bake_normal_map`` for texel points [n,3] along their frames' N (include/avc_b200.h,
    avc_bake_snap_*) -> (snapped points [n,3], bracket [n,2] = (lo, hi), state [n] int32: 0 no sign change), on the
    device.  ``chunk`` texels are sampled per sdf pass; the result does not depend on it."""
    L, st = _L(), _lib.stream_ptr()
    n = points.shape[0]
    bracket = torch.empty(n, 2, dtype=torch.float32, device=points.device)
    state = torch.empty(n, dtype=torch.int32, device=points.device)
    for s in range(0, n, chunk):
        m = min(chunk, n - s)
        samples = torch.empty(m, SNAP_SAMPLES, 3, dtype=torch.float32, device=points.device)
        _lib.check(L.avc_bake_snap_samples(_lib.ptr(points[s:]), _lib.ptr(frames[s:]), m, float(D), _lib.ptr(samples),
                                           st), "avc_bake_snap_samples")
        sdf = _sdf(runner, samples.reshape(-1, 3), m * SNAP_SAMPLES)
        _lib.check(L.avc_bake_snap_bracket(_lib.ptr(sdf), m, float(D), _lib.ptr(bracket[s:]), _lib.ptr(state[s:]), st),
                   "avc_bake_snap_bracket")
    _mark(timings, "search_samples")
    mid = torch.empty(n, 3, dtype=torch.float32, device=points.device)
    for _ in range(SNAP_STEPS):
        _lib.check(L.avc_bake_snap_midpoints(_lib.ptr(points), _lib.ptr(frames), _lib.ptr(bracket), n, _lib.ptr(mid),
                                             st), "avc_bake_snap_midpoints")
        sdf = _sdf(runner, mid, chunk * SNAP_SAMPLES)
        _lib.check(L.avc_bake_snap_bisect(_lib.ptr(sdf), n, _lib.ptr(bracket), _lib.ptr(state), st),
                   "avc_bake_snap_bisect")
    _lib.check(L.avc_bake_snap_midpoints(_lib.ptr(points), _lib.ptr(frames), _lib.ptr(bracket), n, _lib.ptr(mid), st),
               "avc_bake_snap_midpoints")
    _mark(timings, "search_bisection")
    return mid, bracket, state


def _mark(timings, name):
    """With a ``timings`` dict: the seconds since the last mark, after a device synchronise, under ``name``."""
    if timings is None:
        return
    torch.cuda.synchronize()
    now = time.perf_counter()
    timings[name] = now - timings.get("_t", now)
    timings["_t"] = now


def bake_normal_map(runner, vertices_ply_frame, triangles, texture_size: int = DEFAULT_TEXTURE_SIZE,
                    chunk: int = SNAP_CHUNK, timings: dict | None = None):
    """The tangent-space normal map of ``triangles`` over ``vertices_ply_frame`` (the atlas of ``bake_texture``) from
    ``runner``'s SDF -> (image uint8 [T,T,3] RGB, row 0 at the top, host; stats dict: used, converged, flat,
    back_facing texels).  Frames come from the PLY-frame positions and their ``vertex_normals``, where the SDF lives.
    Unused texels are 0; texels with no sign change on their segment, or |grad sdf| < 1e-6, get (128, 128, 255)
    (flat); back-facing texels (the SDF's normal at or past 90 degrees from the mesh's) are encoded and counted.
    ``timings``, when given, receives the seconds of each phase (frames, search_samples, search_bisection, gradient,
    encode)."""
    device = _cuda(runner.device)
    _mark(timings, "_start")
    v = _f32(torch.as_tensor(vertices_ply_frame), device).reshape(-1, 3)
    f = torch.as_tensor(triangles).to(device, torch.int32).contiguous().reshape(-1, 3)
    T = int(texture_size)
    owner, points, uv = texel_points(v, f, T)
    normals = vertex_normals(v, f)
    used = torch.nonzero(owner >= 0).reshape(-1).to(torch.int32)
    n = used.numel()
    frames = texel_frames(f, normals, corner_tangents(v, f, normals, uv), T, used)
    p0 = points[used.long()].contiguous()
    _mark(timings, "frames")
    snapped, _, state = snap_to_zero_set(runner, p0, frames, search_length(v, f), chunk, timings)
    grad = torch.empty(n, 3, dtype=torch.float32, device=device)
    for s in range(0, n, chunk * SNAP_SAMPLES):
        grad[s:s + chunk * SNAP_SAMPLES] = runner.renderer.sdf_eval(snapped[s:s + chunk * SNAP_SAMPLES],
                                                                    want_features=False, want_gradient=True)[1]
    _mark(timings, "gradient")
    image = torch.zeros(T * T, 3, dtype=torch.uint8, device=device)
    counts = torch.empty(2, dtype=torch.int32, device=device)
    _lib.check(_L().avc_bake_normal_encode(_lib.ptr(frames), _lib.ptr(grad), _lib.ptr(state), _lib.ptr(used), n, T,
                                           _lib.ptr(image), _lib.ptr(counts), _lib.stream_ptr()),
               "avc_bake_normal_encode")
    flat, back = counts.tolist()
    stats = dict(used=n, converged=int((state != 0).sum()), flat=flat, back_facing=back)
    out = image.cpu().numpy().reshape(T, T, 3)
    _mark(timings, "encode")
    if timings is not None:
        timings.pop("_start", None), timings.pop("_t", None)
    return out, stats


def encode_png(texture: np.ndarray) -> bytes:
    """The RGB uint8 [H,W,3] texture as PNG bytes (``cv2.imencode``, which takes BGR)."""
    import cv2 as cv
    ok, buf = cv.imencode(".png", np.ascontiguousarray(np.asarray(texture, dtype=np.uint8)[..., ::-1]))
    if not ok:
        raise RuntimeError("cv2.imencode('.png') failed")
    return buf.tobytes()
