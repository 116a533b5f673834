"""Bake the NeuS colour field of a trained avatar into a texture for its exported mesh.

``bake_texture`` lays the clustered mesh's faces out on a closed-form atlas (``avc_bake_texel_points``: faces 2k and
2k + 1 share square cell k of a T x T texture, each on its side of the cell's diagonal), puts every used texel's centre
on its face's surface in the PLY (NeuS) frame, and colours it the way ``Runner.validate_mesh`` colours a vertex
(``Runner.surface_colors``: the best of six axis views, ``to8b``).  The renders use mid-bin samples (no jitter), so a
texel's bytes depend on its point alone.  ``export.write_glb`` stores the result as an sRGB PNG with ``TEXCOORD_0`` and
smooth ``NORMAL``s (``vertex_normals``).

Not done: chart-based unwrapping or area-proportional packing (every face gets the same cell area), mipmap-safe gutters
(the sampler has no mipmaps), normal maps, and snapping texel points onto the SDF's zero set.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib, video
from .drive import _cuda, _f32

DEFAULT_TEXTURE_SIZE = 2048
MIN_CELL = 8                 # texels per cell side (avc_bake_atlas_grid)
MAX_TEXTURE_SIZE = 16384
RAY_CHUNK = 1 << 16          # rays per render call of the bake
POINT_CHUNK = 1 << 21        # texel points per surface_colors call: bounds the six views' colour and depth buffers

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
        for n in ("avc_bake_atlas_grid", "avc_bake_texel_points", "avc_bake_vertex_normals"):
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


def encode_png(texture: np.ndarray) -> bytes:
    """The RGB uint8 [H,W,3] texture as PNG bytes (``cv2.imencode``, which takes BGR)."""
    import cv2 as cv
    ok, buf = cv.imencode(".png", np.ascontiguousarray(np.asarray(texture, dtype=np.uint8)[..., ::-1]))
    if not ok:
        raise RuntimeError("cv2.imencode('.png') failed")
    return buf.tobytes()
