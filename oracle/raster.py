"""CPU oracle (test infrastructure, never on the product path): the template silhouette render of
``render_one_batch`` (AvatarGen/AppearanceGen/models/utils.py:108-125) and the host-side mask handling of
``gen_rays_silhouettes`` (models/dataset.py:252-275), restated in numpy.

PARITY UNPINNED for the rasteriser: the arithmetic lives in ``neural_renderer`` (requirements.txt:
``git+https://github.com/daniilidis-group/neural_renderer``, unpinned, CUDA-only build, not installable here); the
reference has no test or golden image at this boundary.  Restated from the package's published algorithm:
``Renderer(camera_mode='look')`` defaults -- image_size 256, anti_aliasing (render at 2x, 2 x 2 average pool),
viewing_angle 30 deg, near 0.1 / far 100, fill_back (both windings drawn, back faces culled => the camera-facing normal
lights the pixel), light_intensity_ambient 0.5 + directional 0.5 along (0, 1, 0), flat per-face lighting, white texture,
black background; ``look``: z = direction, x = normalize(cross(up, z)), y = normalize(cross(z, x));
``perspective``: x' = x / (z tan(angle)); pixel centre xi <-> (2 xi + 1 - is) / is, image row 0 at the top; depth by
barycentric interpolation of 1/z.  What CAN be pinned -- the dilation, canvas sizing, nearest resizes and the ray mask --
is pinned against dataset.py's own lines by oracle/pin_loss_stage.py.
"""
from __future__ import annotations

import numpy as np


def raster_template(verts, faces, eye, at, n=256, ss=2):
    """-> rgb [n, n, 3] float32 (already flipped like utils.py:124), mask [n, n] bool (rgb != 0)."""
    v = np.asarray(verts, dtype=np.float64).reshape(-1, 3)
    rot = np.stack([v[:, 0], v[:, 2], -v[:, 1]], 1)                      # utils.py:115-119
    eye, at = np.asarray(eye, dtype=np.float64), np.asarray(at, dtype=np.float64)
    z = (at - eye) / np.linalg.norm(at - eye)
    x = np.cross([0.0, 1.0, 0.0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    y /= np.linalg.norm(y)
    cam = (rot - eye) @ np.stack([x, y, z], 1)
    w = np.tan(np.deg2rad(30.0))
    px, py, pz = cam[:, 0] / cam[:, 2] / w, cam[:, 1] / cam[:, 2] / w, cam[:, 2]
    size = n * ss
    depth = np.full((size, size), np.inf)
    shade = np.zeros((size, size))
    for f in np.asarray(faces):
        a, b, c = f
        if pz[a] <= 0 or pz[b] <= 0 or pz[c] <= 0:
            continue
        xs, ys = px[[a, b, c]], py[[a, b, c]]
        xi0 = max(0, int(np.ceil((xs.min() * size + size - 1) / 2))); xi1 = min(size - 1, int(np.floor((xs.max() * size + size - 1) / 2)))
        yi0 = max(0, int(np.ceil((ys.min() * size + size - 1) / 2))); yi1 = min(size - 1, int(np.floor((ys.max() * size + size - 1) / 2)))
        if xi0 > xi1 or yi0 > yi1:
            continue
        det = (ys[1] - ys[2]) * (xs[0] - xs[2]) + (xs[2] - xs[1]) * (ys[0] - ys[2])
        if abs(det) < 1e-20:
            continue
        gx = (2.0 * np.arange(xi0, xi1 + 1) + 1 - size) / size
        gy = (2.0 * np.arange(yi0, yi1 + 1) + 1 - size) / size
        X, Y = np.meshgrid(gx, gy)
        w0 = ((ys[1] - ys[2]) * (X - xs[2]) + (xs[2] - xs[1]) * (Y - ys[2])) / det
        w1 = ((ys[2] - ys[0]) * (X - xs[2]) + (xs[0] - xs[2]) * (Y - ys[2])) / det
        w2 = 1 - w0 - w1
        inside = (w0 >= 0) & (w1 >= 0) & (w2 >= 0)
        zp = 1.0 / (w0 / pz[a] + w1 / pz[b] + w2 / pz[c])
        ok = inside & (zp > 0.1) & (zp < 100.0)
        if not ok.any():
            continue
        nrm = np.cross(rot[b] - rot[a], rot[c] - rot[a])
        nl = np.linalg.norm(nrm) + 1e-20
        s = 1.0 if nrm @ (eye - rot[a]) >= 0 else -1.0
        val = 0.5 + 0.5 * max(s * nrm[1] / nl, 0.0)
        rows = size - 1 - np.arange(yi0, yi1 + 1)
        sub_d = depth[rows[:, None], np.arange(xi0, xi1 + 1)[None, :]]
        upd = ok & (zp < sub_d)
        rr, cc = np.nonzero(upd)
        depth[rows[rr], xi0 + cc] = zp[rr, cc]
        shade[rows[rr], xi0 + cc] = val
    img = shade.reshape(n, ss, n, ss).mean(axis=(1, 3))[:, ::-1]
    rgb = np.repeat(img[:, :, None], 3, axis=2).astype(np.float32)
    return np.ascontiguousarray(rgb), rgb[..., 0] != 0


def dilate_and_canvas(mask, max_ray_num, iterations=10):
    """dataset.py:255-258: binary dilation with the 3 x 3 full structure, ``iterations`` times; canvas size."""
    m = np.asarray(mask).astype(bool)
    n = m.shape[0]
    for _ in range(iterations):
        p = np.pad(m, 1)
        out = np.zeros_like(m)
        for dy in range(3):
            for dx in range(3):
                out |= p[dy:dy + n, dx:dx + n]
        m = out
    ratio = m.sum() / float(n * n)
    W = min(n, int(np.sqrt(max_ray_num / ratio))) if m.sum() else n // 4
    return m, W


def nearest_resize(a, W):
    """F.interpolate(..., size=(W, W)) default (nearest): src = floor(dst * scale) with scale = n / W and the product
    both rounded to float32, as torch forms them: a float64 product floors differently at some sizes (33 -> 1023)."""
    n = a.shape[0]
    idx = np.minimum(np.floor(np.arange(W, dtype=np.float32) * (np.float32(n) / np.float32(W))).astype(np.int64), n - 1)
    return a[idx][:, idx]


def chessboard_blurred(H, W, length, sigma):
    """main.py:396-402 with torchvision's GaussianBlur(kernel_size=(5, 9), sigma) semantics (5 taps along x, 9 along y,
    reflect padding)."""
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    board = np.where(((yy // length) + (xx // length)) % 2 == 0, 0.8, 0.2)
    kx = np.exp(-0.5 * ((np.arange(5) - 2) / sigma) ** 2); kx /= kx.sum()
    ky = np.exp(-0.5 * ((np.arange(9) - 4) / sigma) ** 2); ky /= ky.sum()
    p = np.pad(board, ((4, 4), (2, 2)), mode="reflect")
    out = np.zeros((H, W))
    for j in range(9):
        for i in range(5):
            out += ky[j] * kx[i] * p[j:j + H, i:i + W]
    return out.astype(np.float32)
