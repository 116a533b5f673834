"""The tangent-space normal map of avatarclip_b200.bake in float64: corner tangents, texel frames, the zero-set snap
(bracket and bisection) on an SDF callable, the encode, and glTF's decode.  Semantics as avc_bake_corner_tangents ..
avc_bake_normal_encode in include/avc_b200.h; the atlas itself is oracle/bake.py."""
from __future__ import annotations

import numpy as np

from . import bake as B

K = 16                 # samples of the search segment
STEPS = 12             # bisection steps


def _unit(x):
    return x / np.linalg.norm(x, axis=-1, keepdims=True)


def tangent_against(t, n) -> np.ndarray:
    """[..., 3] t Gram-Schmidt'd against the unit n, normalised; the axis of n's smallest |component| instead when
    |o| <= 1e-6 |t|."""
    t, n = np.asarray(t, np.float64), np.asarray(n, np.float64)
    o = t - (t * n).sum(-1, keepdims=True) * n
    bad = ~(np.linalg.norm(o, axis=-1) > 1e-6 * np.linalg.norm(t, axis=-1))
    if bad.any():
        e = np.eye(3)[np.argmin(np.abs(n[bad]), axis=-1)]               # argmin takes the first of equals
        o[bad] = e - (e * n[bad]).sum(-1, keepdims=True) * n[bad]
    return _unit(o)


def corner_tangents(verts, faces, normals, uv) -> np.ndarray:
    """[F, 3, 4]: per corner dP/du Gram-Schmidt'd against the corner's normal, and w with w cross(N, T) along -dP/dv."""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    n = np.asarray(normals, np.float64)[f]                                 # [F, 3, 3]
    uv = np.asarray(uv, np.float64).reshape(-1, 3, 2)
    e1, e2 = v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]
    du1, dv1 = uv[:, 1, 0] - uv[:, 0, 0], uv[:, 1, 1] - uv[:, 0, 1]
    du2, dv2 = uv[:, 2, 0] - uv[:, 0, 0], uv[:, 2, 1] - uv[:, 0, 1]
    det = du1 * dv2 - du2 * dv1
    s = np.where(det < 0, -1.0, 1.0)[:, None]
    tf = s * (e1 * dv2[:, None] - e2 * dv1[:, None])
    bf = s * (e2 * du1[:, None] - e1 * du2[:, None])
    t = tangent_against(np.repeat(tf[:, None], 3, 1), n)
    w = np.where((det[:, None] != 0) & ((np.cross(n, t) * bf[:, None]).sum(-1) > 0), -1.0, 1.0)
    return np.concatenate([t, w[..., None]], -1)


def texel_bary(texels, F: int, T: int):
    """(owner [n], barycentrics [n, 3]) of texel indices, as avc_bake_texel_points takes them."""
    m, c = B.grid(F, T)
    own = B.texel_owner(F, T).reshape(-1)[texels]
    y, x = np.divmod(np.asarray(texels, np.int64), T)
    i, j = x % c, y % c
    return own, B.barycentric(i + 0.5, j + 0.5, c, i < j)


def texel_frames(faces, normals, tangents, T: int, texels) -> np.ndarray:
    """[n, 3, 3] rows T, B, N at used texels."""
    f = np.asarray(faces, np.int64)
    own, b = texel_bary(texels, f.shape[0], T)
    n = np.asarray(normals, np.float64)[f[own]]                              # [n, 3, 3]
    tg = np.asarray(tangents, np.float64)[own]                               # [n, 3, 4]
    N = (b[..., None] * n).sum(1)
    ln = np.linalg.norm(N, axis=-1, keepdims=True)
    N = np.where(ln > 0, N / np.where(ln > 0, ln, 1.0), np.array([0.0, 1.0, 0.0]))
    Tt = tangent_against((b[..., None] * tg[..., :3]).sum(1), N)
    w = np.where((b * tg[..., 3]).sum(1) >= 0, 1.0, -1.0)
    return np.stack([Tt, w[:, None] * np.cross(N, Tt), N], 1)


def offsets(D: float) -> np.ndarray:
    """[K] the sample offsets t_k = (2k - 15) D / 15."""
    return (2.0 * np.arange(K) - (K - 1)) * D / (K - 1)


def candidates(sdf) -> np.ndarray:
    """[n, 2K - 1] bool: position q = 2k is sample k with sdf exactly 0, q = 2k + 1 the interval [t_k, t_k+1] with a
    strict sign change."""
    s = np.asarray(sdf, np.float64)
    c = np.zeros((s.shape[0], 2 * K - 1), bool)
    c[:, 0::2] = s == 0
    c[:, 1::2] = ((s[:, :-1] < 0) & (s[:, 1:] > 0)) | ((s[:, :-1] > 0) & (s[:, 1:] < 0))
    return c


def bracket(sdf, D: float):
    """(lo [n], hi [n], state [n] int): the candidate nearest t = 0, the outside (+t) one on a tie."""
    s = np.asarray(sdf, np.float64)
    c = candidates(s)
    key = np.abs(np.arange(2 * K - 1) - (K - 1))
    score = np.where(c, 2 * key - (np.arange(2 * K - 1) > K - 1), 1 << 20)  # ties go to the larger q
    q = score.argmin(1)
    found = c[np.arange(s.shape[0]), q]
    t = offsets(D)
    k = q // 2
    odd = q % 2 == 1
    lo = np.where(found, t[k], 0.0)
    hi = np.where(found, np.where(odd, t[np.minimum(k + 1, K - 1)], t[k]), 0.0)
    state = np.where(~found, 0, np.where(odd & (s[np.arange(s.shape[0]), k] > 0), 2, 1))
    return lo, hi, state


def ties(sdf, bound: float) -> np.ndarray:
    """[n] bool: texels whose bracket a float32 evaluation may pick differently: a sample with |sdf| < bound, or two
    candidates at the same distance from t = 0."""
    s = np.asarray(sdf, np.float64)
    c = candidates(s)
    key = np.abs(np.arange(2 * K - 1) - (K - 1))
    best = np.where(c, key, 1 << 20).min(1)
    two = (c & (key == best[:, None])).sum(1) > 1
    return (np.abs(s) < bound).any(1) | two


def snap(points, N, D: float, sdf_fn, steps: int = STEPS):
    """The search on sdf_fn ([m, 3] float64 -> [m] float64): (lo, hi, state, snapped points [n, 3], sample sdf
    [n, K])."""
    p, N = np.asarray(points, np.float64), np.asarray(N, np.float64)
    t = offsets(D)
    s = sdf_fn((p[:, None, :] + t[None, :, None] * N[:, None, :]).reshape(-1, 3)).reshape(-1, K)
    lo, hi, state = bracket(s, D)
    for _ in range(steps):
        m = (lo + hi) * 0.5
        sm = sdf_fn(p + m[:, None] * N)
        live = state != 0
        zero = live & (sm == 0)
        same = live & ~zero & ((sm < 0) == (state == 1))
        other = live & ~zero & ~same
        lo = np.where(zero | same, m, lo)
        hi = np.where(zero | other, m, hi)
    return lo, hi, state, p + ((lo + hi) * 0.5)[:, None] * N, s


def encode(frames, grad, state):
    """(bytes [n, 3] uint8, flat [n] bool, back-facing [n] bool)."""
    fr, g = np.asarray(frames, np.float64), np.asarray(grad, np.float64)
    ln = np.linalg.norm(g, axis=-1)
    flat = (np.asarray(state) == 0) | ~(ln >= 1e-6)
    n = g / np.where(flat, 1.0, ln)[:, None]
    c = np.einsum("nij,nj->ni", fr, n)
    out = np.clip(np.rint(127.5 * c + 127.5), 0, 255).astype(np.uint8)
    out[flat] = (128, 128, 255)
    return out, flat, ~flat & (c[:, 2] <= 0)


def decode(rgb, T, Bt, N) -> np.ndarray:
    """glTF's normalTexture: (x, y, z) = 2 byte / 255 - 1, n = normalise(T x + B y + N z)."""
    x = 2.0 * np.asarray(rgb, np.float64) / 255.0 - 1.0
    return _unit(np.asarray(T) * x[..., :1] + np.asarray(Bt) * x[..., 1:2] + np.asarray(N) * x[..., 2:3])
