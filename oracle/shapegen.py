"""CPU oracle (test infrastructure, never on the product path): AvatarGen/ShapeGen's shape search (main.py:93-123,
utils.py:9-35) restated in numpy / torch CPU fp64 -- the shape-VAE decode, neural_renderer's texture loading and
textured ``look_at`` render, the nearest resize + CLIP Normalize, and the codebook score -- plus the seeded synthetic
inputs the tests and oracle/pin_shapegen.py share.

PARITY UNPINNED for the texture loading and the textured rasteriser: their arithmetic lives in ``neural_renderer``
(requirements.txt, unpinned, CUDA-only build, not installable here), exactly as oracle/raster.py says for the template
render.  Restated from the package's published algorithm:
  * ``load_obj(..., load_texture=True, texture_size=R)``: per triangle an R x R x R colour cube, 1.0 unless the face's
    material has a ``map_Kd`` image; texel (i, j, k) is the bilinear sample at barycentric (i, j, k) / (i + j + k) of the
    face's UV triangle ((0, 0, 0): the first corner), UVs wrapped into [0, 1) (REPEAT), the image flipped vertically
    before sampling, pixel position uv * (size - 1), the +1 neighbours clamped to the last row / column;
  * ``Renderer(camera_mode='look_at')``: look_at() (z = normalize(at - eye), x = normalize(cross(up, z)),
    y = normalize(cross(z, x))), perspective x / (z tan 30 deg), the z-buffer of oracle/raster.py (pixel centres
    (2 i + 1 - is) / is, depth by barycentric 1/z, near 0.1 / far 100, faces with a vertex at z <= 0 skipped, image row
    0 at the top); fill_back draws both windings and culls back faces, so the lit copy is the one facing the eye:
    light = 0.5 + 0.5 relu(n . (0, 1, 0)), n = normalize((v0 - v1) x (v2 - v1)) oriented towards the eye, in the world
    frame; colour = light x trilinear sample of the cube at w_k (R - 1) z / z_k clamped to [0, R - 1 - 1e-5]; black
    background; 2 x 2 average pool.
What the reference's own code does around them (parse_prompt, the decode, the resize, the score, writeOBJ) is pinned
by oracle/pin_shapegen.py, which runs the unmodified main.py / utils.py with this rasteriser standing in for
neural_renderer.
"""
from __future__ import annotations

import gzip
import os

import numpy as np
import torch

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)       # main.py:102
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)        # main.py:103
LATENT = 16
HIDDEN = 8192
VAE_SEED = 7
CODEBOOK_SEED = 8
UV_SEED = 9
CLIP_SEED = 10
CODEBOOK_N = 48
CODEBOOK_WINNER = 29
NEUTRAL_TXT = "a 3d rendering of a person in unreal engine"
TARGET_TXT = "a tall strong man with broad shoulders:2"


# ---------------------------------------------------------------- decode
def vae_decode(z, W1, b1, W2, b2, v_template) -> np.ndarray:
    """main.py:67-68 in fp64: dec2(dec1(z)) + v_template -> [B, D]."""
    d = lambda t: np.asarray(torch.as_tensor(t).detach().cpu(), dtype=np.float64)
    h = d(z).reshape(-1, d(W1).shape[1]) @ d(W1).T + d(b1)
    return h @ d(W2).T + d(b2) + d(v_template).reshape(-1)


# ---------------------------------------------------------------- textures
def load_textures(image, face_uv, is_update, textures):
    """One material of neural_renderer's load_textures (module docstring), fp64: image [H,W,3] as stored (row 0 at
    the top), face_uv [F,3,2], is_update [F]; textures [F,R,R,R,3] (fp64) updated in place and returned."""
    img = np.asarray(image, dtype=np.float64)[::-1]
    H, W = img.shape[:2]
    uv = np.asarray(face_uv, dtype=np.float64)
    uv = uv - np.floor(uv)
    R = textures.shape[1]
    g = np.arange(R, dtype=np.float64) / (R - 1)
    d0, d1, d2 = np.meshgrid(g, g, g, indexing="ij")
    s = d0 + d1 + d2
    s = np.where(s > 0, s, 1.0)
    w = np.stack([d0 / s, d1 / s, d2 / s], -1).reshape(-1, 3)               # [R^3, 3]
    for f in np.nonzero(np.asarray(is_update))[0]:
        pos = w @ uv[f]                                                      # [R^3, 2]
        px, py = pos[:, 0] * (W - 1), pos[:, 1] * (H - 1)
        x0, y0 = px.astype(np.int64), py.astype(np.int64)
        x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
        wx1, wy1 = (px - x0)[:, None], (py - y0)[:, None]
        c = (img[y0, x0] * (1 - wx1) * (1 - wy1) + img[y1, x0] * (1 - wx1) * wy1 + img[y0, x1] * wx1 * (1 - wy1) +
             img[y1, x1] * wx1 * wy1)
        textures[f] = c.reshape(R, R, R, 3)
    return textures


def read_uv_obj(obj_fname):
    """The texture half of nr.load_obj: (face_uv [F,3,2] float32, materials [F], {material: map_Kd path})."""
    lines = open(obj_fname).read().splitlines()
    vt, tri, mats, mtls, mat = [], [], [], [], ""
    for line in lines:
        t = line.split()
        if not t:
            continue
        if t[0] == "vt":
            vt.append([float(x) for x in t[1:3]])
        elif t[0] == "usemtl":
            mat = t[1]
        elif t[0] == "mtllib":
            mtls.append(os.path.join(os.path.dirname(obj_fname), t[1]))
        elif t[0] == "f":
            ti = [int(c.split("/")[1]) for c in t[1:]]
            for k in range(len(ti) - 2):
                tri.append((ti[0], ti[k + 1], ti[k + 2]))
                mats.append(mat)
    images, name = {}, None
    for m in mtls:
        for line in open(m).read().splitlines():
            t = line.split()
            if len(t) >= 2 and t[0] == "newmtl":
                name = t[1]
            elif len(t) >= 2 and t[0] == "map_Kd":
                images[name] = os.path.join(os.path.dirname(obj_fname), t[1])
    vt = np.asarray(vt, dtype=np.float32)
    return vt[np.asarray(tri) - 1], mats, images


def read_png_rgb01(path) -> np.ndarray:
    import cv2 as cv
    img = cv.cvtColor(cv.imread(path, cv.IMREAD_COLOR), cv.COLOR_BGR2RGB)
    return img.astype(np.float32) / np.float32(255.0)


def load_obj_textures(obj_fname, texture_size=8) -> np.ndarray:
    """nr.load_obj(obj_fname, load_texture=True, texture_size)[2] in fp64: [F,R,R,R,3]."""
    face_uv, mats, images = read_uv_obj(obj_fname)
    R = texture_size
    tex = np.ones((face_uv.shape[0], R, R, R, 3))
    mats = np.asarray(mats)
    for name, path in images.items():
        load_textures(read_png_rgb01(path), face_uv, mats == name, tex)
    return tex


# ---------------------------------------------------------------- textured look_at render
def look_at_camera(eye, at=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0)):
    eye, at, up = (np.asarray(a, dtype=np.float64) for a in (eye, at, up))
    z = (at - eye) / np.linalg.norm(at - eye)
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    y /= np.linalg.norm(y)
    return eye, np.stack([x, y, z], 1)


def raster_textured(verts, faces, textures, eye, at=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0), n=256, ss=2):
    """The textured look_at render (module docstring) in fp64 -> rgb [n, n, 3] float64, row 0 at the top."""
    v = np.asarray(verts, dtype=np.float64).reshape(-1, 3)
    faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    tex = np.asarray(textures, dtype=np.float64)
    R = tex.shape[1]
    eye, rot = look_at_camera(eye, at, up)
    cam = (v - eye) @ rot
    w = np.tan(np.deg2rad(30.0))
    px, py, pz = cam[:, 0] / cam[:, 2] / w, cam[:, 1] / cam[:, 2] / w, cam[:, 2]
    size = n * ss
    depth = np.full((size, size), np.inf)
    fid = np.full((size, size), -1, dtype=np.int64)
    for fi, (a, b, c) in enumerate(faces):
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
        X, Y = np.meshgrid((2.0 * np.arange(xi0, xi1 + 1) + 1 - size) / size, (2.0 * np.arange(yi0, yi1 + 1) + 1 - size) / size)
        w0 = ((ys[1] - ys[2]) * (X - xs[2]) + (xs[2] - xs[1]) * (Y - ys[2])) / det
        w1 = ((ys[2] - ys[0]) * (X - xs[2]) + (xs[0] - xs[2]) * (Y - ys[2])) / det
        w2 = 1 - w0 - w1
        zp = 1.0 / (w0 / pz[a] + w1 / pz[b] + w2 / pz[c])
        ok = (w0 >= 0) & (w1 >= 0) & (w2 >= 0) & (zp > 0.1) & (zp < 100.0)
        rows = size - 1 - np.arange(yi0, yi1 + 1)
        cols = np.arange(xi0, xi1 + 1)
        sub = depth[rows[:, None], cols[None, :]]
        # ties keep the smaller face index, like the device's (depth, face) atomicMin
        rr, cc = np.nonzero(ok & (zp < sub))
        depth[rows[rr], cols[cc]] = zp[rr, cc]
        fid[rows[rr], cols[cc]] = fi
    rgb = np.zeros((size, size, 3))
    rr, cc = np.nonzero(fid >= 0)
    if rr.size:
        f = fid[rr, cc]
        i0, i1, i2 = faces[f, 0], faces[f, 1], faces[f, 2]
        a, b = v[i0] - v[i1], v[i2] - v[i1]
        nrm = np.cross(a, b)
        nl = np.maximum(np.linalg.norm(nrm, axis=1), 1e-5)
        s = np.where(np.einsum("ij,ij->i", nrm, eye - v[i1]) >= 0, 1.0, -1.0)
        light = 0.5 + 0.5 * np.maximum(s * nrm[:, 1] / nl, 0.0)
        X = (2.0 * cc + 1 - size) / size
        Y = (2.0 * (size - 1 - rr) + 1 - size) / size
        xa, ya, xb, yb, xc, yc = px[i0], py[i0], px[i1], py[i1], px[i2], py[i2]
        det = (yb - yc) * (xa - xc) + (xc - xb) * (ya - yc)
        w0 = ((yb - yc) * (X - xc) + (xc - xb) * (Y - yc)) / det
        w1 = ((yc - ya) * (X - xc) + (xa - xc) * (Y - yc)) / det
        w2 = 1 - w0 - w1
        zp = depth[rr, cc]
        wz = np.stack([w0 * zp / pz[i0], w1 * zp / pz[i1], w2 * zp / pz[i2]], 1)
        ti = np.clip(wz * (R - 1), 0.0, R - 1 - 1e-5)
        tb = ti.astype(np.int64)
        fr = ti - tb
        col = np.zeros((f.size, 3))
        for corner in range(8):
            hi = np.array([(corner >> k) & 1 for k in range(3)])
            wt = np.prod(np.where(hi[None, :] == 1, fr, 1 - fr), axis=1)
            idx = np.minimum(tb + hi[None, :], R - 1)
            col += wt[:, None] * tex[f, idx[:, 0], idx[:, 1], idx[:, 2]]
        rgb[rr, cc] = col * light[:, None]
    return rgb.reshape(n, ss, n, ss, 3).mean(axis=(1, 3))


# ---------------------------------------------------------------- CLIP preprocessing and the score
def clip_prep_nearest(images_b3hw, size=224) -> torch.Tensor:
    """main.py:101-103: F.interpolate(images, size) (nearest) then (x - mean) / std with float64 operands on a
    float32 tensor (each in-place step computed in fp64, rounded to fp32)."""
    x = torch.as_tensor(images_b3hw, dtype=torch.float32)
    n = x.shape[-1]
    idx = torch.clamp(torch.floor(torch.arange(size, dtype=torch.float32) * (np.float32(n) / np.float32(size))).long(),
                      max=n - 1)
    x = x[:, :, idx][:, :, :, idx]
    mean = torch.tensor(CLIP_MEAN, dtype=torch.float64).view(1, 3, 1, 1)
    std = torch.tensor(CLIP_STD, dtype=torch.float64).view(1, 3, 1, 1)
    x = (x.double() - mean).float()
    return (x.double() / std).float()


def codebook_cos(clip_codebook, image_emb, delta) -> np.ndarray:
    """main.py:106-107 in fp64 with F.normalize's max(|x|, 1e-12)."""
    Cb = np.asarray(torch.as_tensor(clip_codebook), dtype=np.float64)
    e = np.asarray(torch.as_tensor(image_emb), dtype=np.float64).reshape(-1)
    d = np.asarray(torch.as_tensor(delta), dtype=np.float64).reshape(-1)
    a = Cb - e
    a /= np.maximum(np.linalg.norm(a, axis=1, keepdims=True), 1e-12)
    return a @ (d / max(np.linalg.norm(d), 1e-12))


# ---------------------------------------------------------------- seeded synthetic inputs
def vae_state(v_template, seed: int = VAE_SEED) -> dict:
    """A full-size LinearVAE state dict (in_dim = 3 V, latent 16, hidden 8192) from ``seed``: the decoder is scaled so
    that decoded shapes stay within a few centimetres of the template; the encoder is never run."""
    D = int(np.asarray(v_template).size)
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, std: torch.randn(*s, generator=g) * std
    return {"enc1.weight": rn(HIDDEN, D, std=1e-3), "enc1.bias": rn(HIDDEN, std=1e-3),
            "enc2.weight": rn(2 * LATENT, HIDDEN, std=1e-3), "enc2.bias": rn(2 * LATENT, std=1e-3),
            "dec1.weight": rn(HIDDEN, LATENT, std=0.25), "dec1.bias": rn(HIDDEN, std=0.25),
            "dec2.weight": rn(D, HIDDEN, std=2e-4), "dec2.bias": rn(D, std=5e-3)}


def write_uv_obj(directory, v_template, faces, seed: int = UV_SEED) -> str:
    """``smpl_uv.obj`` stand-in: the template with one seeded UV triangle per face (some outside [0, 1), to exercise
    REPEAT), faces in three materials -- two with ``map_Kd`` images of different sizes and one without -- plus its
    ``.mtl`` and PNGs.  Returns the OBJ path."""
    import cv2 as cv
    rng = np.random.default_rng(seed)
    F = len(faces)
    os.makedirs(directory, exist_ok=True)
    for name, (h, w) in (("skin.png", (96, 128)), ("cloth.png", (40, 56))):
        yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
        img = np.stack([0.5 + 0.4 * np.sin(6 * xx + 2 * yy), 0.5 + 0.4 * np.cos(5 * yy), 0.3 + 0.6 * xx * yy], -1)
        img = img + rng.uniform(-0.08, 0.08, img.shape)
        cv.imwrite(os.path.join(directory, name), cv.cvtColor((np.clip(img, 0, 1) * 255).round().astype(np.uint8),
                                                              cv.COLOR_RGB2BGR))
    with open(os.path.join(directory, "smpl_uv.mtl"), "w") as fp:
        fp.write("newmtl skin\nKd 1 1 1\nmap_Kd skin.png\n\nnewmtl cloth\nmap_Kd cloth.png\n\nnewmtl bare\nKd 0.5 0.5 0.5\n")
    centre = rng.uniform(-0.4, 1.4, (F, 1, 2))
    vt = (centre + rng.uniform(-0.03, 0.03, (F, 3, 2))).reshape(-1, 2).astype(np.float32)
    mat = np.where(np.arange(F) < F // 2, 0, np.where(np.arange(F) < (9 * F) // 10, 1, 2))
    lines = ["mtllib smpl_uv.mtl"] + [f"v {x:.6f} {y:.6f} {z:.6f}" for x, y, z in np.asarray(v_template)]
    lines += [f"vt {float(u)!r} {float(t)!r}" for u, t in vt]
    names = ("skin", "cloth", "bare")
    last = None
    for i, (a, b, c) in enumerate(np.asarray(faces)):
        if mat[i] != last:
            lines.append(f"usemtl {names[mat[i]]}")
            last = mat[i]
        lines.append(f"f {a + 1}/{3 * i + 1} {b + 1}/{3 * i + 2} {c + 1}/{3 * i + 3}")
    path = os.path.join(directory, "smpl_uv.obj")
    with open(path, "w") as fp:
        fp.write("\n".join(lines) + "\n")
    return path


def write_bpe(path) -> str:
    """A merges file with the version header and no merges: every byte is one token (a stand-in for openai's
    ``bpe_simple_vocab_16e6.txt.gz``, whose vocabulary the random towers do not need)."""
    with gzip.open(path, "wt", encoding="utf-8") as f:
        f.write("#version: 0.2\n")
    return str(path)


def clip_states(seed: int = CLIP_SEED):
    """(visual, text) seeded random ViT-B/32 towers in the layout ``load_clip_model`` returns."""
    from oracle import clip_text as oct
    from oracle import clip_vit as ocv
    visual = {"visual." + k: v for k, v in ocv.random_vit_state(seed=seed).items()}
    return visual, oct.random_text_state(seed=seed + 1)


def make_codebook(image_emb, delta, seed: int = CODEBOOK_SEED, n: int = CODEBOOK_N, winner: int = CODEBOOK_WINNER):
    """A tensor-keyed codebook {latents [n,16]: embeddings [n,512]} built around the neutral image embedding e and
    the text direction: every entry is e + |e| u_i with u_i a random unit vector (cosine ~ +-0.15 with the direction),
    except entry ``winner``, whose u leans 0.6 along it -- the winning cosine beats the runner-up by far more than the
    fp16 towers can move it."""
    g = torch.Generator().manual_seed(seed)
    e = torch.as_tensor(image_emb, dtype=torch.float64).reshape(-1)
    d = torch.as_tensor(delta, dtype=torch.float64).reshape(-1)
    d = d / d.norm()
    u = torch.randn(n, e.numel(), generator=g, dtype=torch.float64)
    u = u - 0.5 * (u @ d).clamp(min=0)[:, None] * d        # pull the positive cosines down
    u = u / u.norm(dim=1, keepdim=True)
    r = torch.randn(e.numel(), generator=g, dtype=torch.float64)
    r = r - (r @ d) * d
    u[winner] = 0.6 * d + 0.8 * r / r.norm()
    emb = (e + e.norm() * u).float()
    latents = torch.randn(n, LATENT, generator=g)
    return {latents: emb}
