"""Render generated avatars to video on the GPU: a turntable of the coloured mesh, or the avatar performing a motion.

``iter_motion_frames`` rigs the PLY ``Runner.validate_mesh`` exports exactly as ``drive.generate_animation`` does
(``drive.rig_mesh``: the rotation into SMPL's frame, ``cleanup_mesh``, the nearest template vertex, inverse LBS), skins
it through the motion chunk by chunk (``avc_lbs_frames``) and renders each chunk in one launch per stage
(``avc_video_render``); ``iter_turntable_frames`` renders the mesh itself, rotated into the same frame, from a camera
orbiting it.  Both yield [n][n][3] uint8 RGB frames on the host; ``write_video`` encodes them into an MP4.

The renderer is smooth-shaded: per-vertex colours and normals interpolated perspective-correctly, a headlight
(0.25 ambient + 0.75 diffuse), supersampled.  Cameras work in drive's frame: z up, the avatar in its stand pose facing
-y.  The camera starts on the -y side looking at the avatar's front, at a fixed 30 degree field of view and a distance
that fits the bounding sphere of every rendered frame's vertices with a margin.

    python -m avatarclip_b200.video --mesh exp/.../meshes/00029500.ply --out turntable.mp4
    python -m avatarclip_b200.video --mesh exp/.../meshes/00029500.ply --motion action.npy --smpl smpl.npz \\
        --stand_pose ShapeGen/output/stand_pose.npy --out avatar.mp4
"""
from __future__ import annotations

import argparse
import ctypes as C
import math
import os
import sys
from typing import Iterator, NamedTuple, Optional

import numpy as np
import torch

from . import _lib, drive

FOV_DEGREES = 30.0
MARGIN = 1.1                    # the bounding sphere fills 1 / MARGIN of the field of view
BACKGROUND = (255, 255, 255)
_CHUNK_BYTES = 256 << 20        # device bytes per chunk of frames (skinned vertices, render workspace, images)

_bound = None


def _L():
    global _bound
    L = _lib.lib()
    if _bound is None:
        vp, i32, i64, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t
        L.avc_video_adjacency_workspace_bytes.argtypes = [i32, C.POINTER(sz)]
        L.avc_video_adjacency.argtypes = [vp, i32, i32, vp, vp, vp, sz, vp]
        L.avc_video_render_workspace_bytes.argtypes = [i32, i32, i32, i32, i32, C.POINTER(sz)]
        L.avc_video_render.argtypes = [vp, i64, vp, vp, vp, vp, i32, i32, vp, i32, i32, i32, vp, vp, vp, vp, sz, vp]
        for n in ("avc_video_adjacency_workspace_bytes", "avc_video_adjacency", "avc_video_render_workspace_bytes",
                  "avc_video_render"):
            getattr(L, n).restype = C.c_int
        _bound = L
    return L


# ---------------------------------------------------------------- kernels
class Adjacency(NamedTuple):
    """The vertex -> incident-face lists of a mesh (CSR): offsets [V+1], vf [3F] int32 on the device."""
    offsets: torch.Tensor
    vf: torch.Tensor


def adjacency(faces: torch.Tensor, V: int) -> Adjacency:
    """``avc_video_adjacency``: each vertex's faces in ascending face order."""
    device = drive._cuda(faces.device)
    faces = faces.to(torch.int32).contiguous()
    L = _L()
    need = C.c_size_t()
    _lib.check(L.avc_video_adjacency_workspace_bytes(V, C.byref(need)), "avc_video_adjacency_workspace_bytes")
    ws = torch.empty(need.value, dtype=torch.uint8, device=device)
    offsets = torch.empty(V + 1, dtype=torch.int32, device=device)
    vf = torch.empty(max(1, 3 * faces.shape[0]), dtype=torch.int32, device=device)
    _lib.check(L.avc_video_adjacency(_lib.ptr(faces), V, faces.shape[0], _lib.ptr(offsets), _lib.ptr(vf), _lib.ptr(ws),
                                     ws.numel(), _lib.stream_ptr()), "avc_video_adjacency")
    return Adjacency(offsets, vf)


def render_workspace_bytes(V: int, F: int, n_frames: int, image_size: int, supersample: int) -> int:
    need = C.c_size_t()
    _lib.check(_L().avc_video_render_workspace_bytes(V, F, n_frames, image_size, supersample, C.byref(need)),
               "avc_video_render_workspace_bytes")
    return need.value


def render(verts: torch.Tensor, faces: torch.Tensor, adj: Adjacency, colors: Optional[torch.Tensor],
           cameras: np.ndarray, image_size: int, supersample: int, background=BACKGROUND,
           out: Optional[torch.Tensor] = None, workspace: Optional[torch.Tensor] = None,
           face_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``avc_video_render`` of ``len(cameras)`` frames.  ``verts`` is [frames, V, 3], or [V, 3] shared by every frame;
    ``colors`` [V, 3] uint8 on the device or None (grey); ``cameras`` [frames, 13] (world-to-camera [R | t] row-major,
    then the focal length in output pixels).  Returns [frames, n, n, 3] uint8 on the device; ``face_out``, when given,
    receives the winning face of every sample, [frames, n * supersample, n * supersample] int32 (-1: none)."""
    device = drive._cuda(verts.device)
    for t in (faces, colors):
        if t is not None:
            drive._cuda(t.device)
    cams = np.ascontiguousarray(cameras, dtype=np.float32).reshape(-1, 13)
    n_frames = cams.shape[0]
    V, F = verts.shape[-2], faces.shape[0]
    stride = 0 if verts.dim() == 2 else V * 3
    need = render_workspace_bytes(V, F, n_frames, image_size, supersample)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=device)
    if out is None:
        out = torch.empty(n_frames, image_size, image_size, 3, dtype=torch.uint8, device=device)
    bg = (C.c_uint8 * 3)(*background)
    _lib.check(_L().avc_video_render(_lib.ptr(verts), stride, _lib.ptr(faces), _lib.ptr(adj.offsets),
                                     _lib.ptr(adj.vf), _lib.ptr(colors), V, F, cams.ctypes.data_as(C.c_void_p),
                                     n_frames, image_size, supersample, bg, _lib.ptr(out), _lib.ptr(face_out),
                                     _lib.ptr(workspace),
                                     workspace.numel(), _lib.stream_ptr()), "avc_video_render")
    return out


# ---------------------------------------------------------------- cameras
def focal_length(image_size: int) -> float:
    return 0.5 * image_size / math.tan(math.radians(FOV_DEGREES) / 2)


def orbit_cameras(center, radius: float, n_frames: int, image_size: int, degrees: float = 360.0) -> np.ndarray:
    """[n_frames, 13] cameras looking at ``center`` from a distance that fits a sphere of ``radius`` inside the field of
    view with the margin; frame i is turned by ``degrees * i / n_frames`` about +z, frame 0 looks along +y with +z up."""
    c = np.asarray(center, dtype=np.float64).reshape(3)
    d = max(float(radius), 1e-6) * MARGIN / math.sin(math.radians(FOV_DEGREES) / 2)
    out = np.empty((n_frames, 13), dtype=np.float32)
    for i in range(n_frames):
        phi = math.radians(degrees) * i / n_frames
        cp, sp = math.cos(phi), math.sin(phi)
        R = np.array([[cp, sp, 0.0], [0.0, 0.0, -1.0], [-sp, cp, 0.0]])      # rows: camera x right, y down, z forward
        eye = c + d * np.array([sp, -cp, 0.0])
        out[i, :12] = np.concatenate([R, (-R @ eye)[:, None]], 1).reshape(-1)
        out[i, 12] = focal_length(image_size)
    return out


def _bounding_sphere(lo: torch.Tensor, hi: torch.Tensor):
    lo, hi = lo.double().cpu().numpy(), hi.double().cpu().numpy()
    return (lo + hi) / 2, float(np.linalg.norm(hi - lo)) / 2


# ---------------------------------------------------------------- frames
def _check_size(image_size: int, supersample: int):
    if not 1 <= image_size <= 4096 or not 1 <= supersample <= 4:
        raise ValueError(f"image_size must be in [1, 4096] and supersample in [1, 4], got {image_size}, {supersample}")


def _read_mesh(mesh_ply: str, device) -> drive.Mesh:
    mesh = drive.read_ply(mesh_ply, device)
    if mesh.triangles.shape[0] == 0:
        raise ValueError(f"{mesh_ply}: the PLY holds no triangles")
    return mesh


def _chunk_frames(V: int, F: int, image_size: int, supersample: int, frames: int, frames_per_chunk, skinned: bool):
    if frames_per_chunk:
        return max(1, min(frames, frames_per_chunk))
    per = render_workspace_bytes(V, F, 1, image_size, supersample) + 2 * image_size * image_size * 3
    return max(1, min(frames, _CHUNK_BYTES // (per + (12 * V if skinned else 0))))


def _pipeline(produce, frames: int, chunk: int, image_size: int, device) -> Iterator[np.ndarray]:
    """``produce(f0, n, out)`` renders frames [f0, f0 + n) into ``out`` on the current stream.  Chunk k renders and
    copies to pinned memory while the caller consumes chunk k-1; buffer pair k % 2 is free again because chunk k-2 was
    consumed in the previous iteration."""
    shape = (chunk, image_size, image_size, 3)
    dev = [torch.empty(shape, dtype=torch.uint8, device=device) for _ in range(2)]
    host = [torch.empty(shape, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
    done = [torch.cuda.Event() for _ in range(2)]
    pending = None
    for k, f0 in enumerate(range(0, frames, chunk)):
        b, n = k % 2, min(chunk, frames - f0)
        produce(f0, n, dev[b][:n])
        host[b][:n].copy_(dev[b][:n], non_blocking=True)
        done[b].record()
        if pending is not None:
            pb, pn = pending
            done[pb].synchronize()
            for i in range(pn):
                yield host[pb][i].numpy().copy()
        pending = (b, n)
    pb, pn = pending
    done[pb].synchronize()
    for i in range(pn):
        yield host[pb][i].numpy().copy()


class MotionRig(NamedTuple):
    """What the motion path skins: the rig of ``drive.rig_mesh``, the motion's joint transforms A [frames, 24, 12] and
    the SMPL tensors on the device."""
    rig: drive.Rig
    A: torch.Tensor
    smpl: dict


def motion_rig(mesh_ply: str, motion_npy: str, smpl, stand_pose_npy: str, device="cuda") -> MotionRig:
    device = drive._cuda(device)
    s = drive.smpl_tensors(smpl, device)
    A = drive.motion_transforms(s, motion_npy)
    return MotionRig(drive.rig_mesh(_read_mesh(mesh_ply, device), s, stand_pose_npy), A, s)


def skin(m: MotionRig, f0: int, n: int, out: torch.Tensor) -> torch.Tensor:
    """Frames [f0, f0 + n) of the motion into ``out`` [n, V, 3]: the payload ``generate_animation`` writes to the PC2."""
    return drive._lbs_frames(m.rig.tpose, m.rig.nearest, m.smpl["lbs_weights"], m.A, f0, n, out)


def iter_motion_frames(mesh_ply: str, motion_npy: str, smpl, stand_pose_npy: str, *, image_size: int = 512,
                       supersample: int = 2, orbit_degrees: float = 0.0, frames_per_chunk: Optional[int] = None,
                       device="cuda") -> Iterator[np.ndarray]:
    """The avatar performing ``motion_npy`` (drive.py's read_pose_my: the global orientation fixed to (pi/2, 0, 0)),
    one [n][n][3] uint8 frame per motion frame; ``orbit_degrees`` turns the camera about +z over the motion."""
    _check_size(image_size, supersample)
    m = motion_rig(mesh_ply, motion_npy, smpl, stand_pose_npy, device)
    mesh = m.rig.mesh
    device = mesh.vertices.device
    V, F, frames = mesh.vertices.shape[0], mesh.triangles.shape[0], m.A.shape[0]
    if F == 0:
        raise ValueError(f"{mesh_ply}: the largest piece of the mesh holds no triangles")
    adj = adjacency(mesh.triangles, V)
    colors = None if mesh.vertex_colors is None else torch.from_numpy(np.ascontiguousarray(mesh.vertex_colors)).to(device)
    chunk = _chunk_frames(V, F, image_size, supersample, frames, frames_per_chunk, True)
    verts = torch.empty(chunk, V, 3, dtype=torch.float32, device=device)
    lo = torch.full((3,), math.inf, device=device)
    hi = torch.full((3,), -math.inf, device=device)
    for f0 in range(0, frames, chunk):              # bounds of every frame: one skinning pass before the render pass
        n = min(chunk, frames - f0)
        v = skin(m, f0, n, verts[:n]).reshape(-1, 3)
        lo, hi = torch.minimum(lo, v.amin(0)), torch.maximum(hi, v.amax(0))
    cams = orbit_cameras(*_bounding_sphere(lo, hi), frames, image_size, orbit_degrees)
    ws = torch.empty(render_workspace_bytes(V, F, chunk, image_size, supersample), dtype=torch.uint8, device=device)

    def produce(f0, n, out):
        render(skin(m, f0, n, verts[:n]), mesh.triangles, adj, colors, cams[f0:f0 + n], image_size, supersample,
               out=out, workspace=ws)
    return _pipeline(produce, frames, chunk, image_size, device)


def iter_turntable_frames(mesh_ply: str, *, n_frames: int = 120, image_size: int = 512, supersample: int = 2,
                          frames_per_chunk: Optional[int] = None, device="cuda") -> Iterator[np.ndarray]:
    """The mesh as exported (rotated into drive's frame, neither cleaned nor rigged) from a camera orbiting 360 degrees
    about +z, one [n][n][3] uint8 frame per step."""
    _check_size(image_size, supersample)
    if n_frames < 1:
        raise ValueError(f"n_frames must be >= 1, got {n_frames}")
    device = drive._cuda(device)
    mesh = _read_mesh(mesh_ply, device)
    v = mesh.vertices
    verts = torch.stack([v[:, 0], -v[:, 2], v[:, 1]], 1).contiguous()          # drive.NEUS_TO_SMPL
    V, F = verts.shape[0], mesh.triangles.shape[0]
    adj = adjacency(mesh.triangles, V)
    colors = None if mesh.vertex_colors is None else torch.from_numpy(np.ascontiguousarray(mesh.vertex_colors)).to(device)
    cams = orbit_cameras(*_bounding_sphere(verts.amin(0), verts.amax(0)), n_frames, image_size)
    chunk = _chunk_frames(V, F, image_size, supersample, n_frames, frames_per_chunk, False)
    ws = torch.empty(render_workspace_bytes(V, F, chunk, image_size, supersample), dtype=torch.uint8, device=device)

    def produce(f0, n, out):
        render(verts, mesh.triangles, adj, colors, cams[f0:f0 + n], image_size, supersample, out=out, workspace=ws)
    return _pipeline(produce, n_frames, chunk, image_size, device)


def write_video(frames, path: str, fps: float = drive.PC2_SAMPLE_RATE) -> int:
    """Encode [n][n][3] uint8 RGB frames into an MP4 (OpenCV, fourcc mp4v); returns the number of frames written."""
    import cv2 as cv
    if not fps > 0:
        raise ValueError(f"fps must be > 0, got {fps}")
    writer, count = None, 0
    try:
        for fr in frames:
            if writer is None:
                h, w = fr.shape[:2]
                writer = cv.VideoWriter(path, cv.VideoWriter_fourcc(*"mp4v"), float(fps), (w, h))
                if not writer.isOpened():
                    raise OSError(f"{path}: OpenCV cannot open an mp4v writer")
            writer.write(cv.cvtColor(fr, cv.COLOR_RGB2BGR))
            count += 1
    finally:
        if writer is not None:
            writer.release()
    return count


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(
        prog="python -m avatarclip_b200.video",
        description="Render a generated avatar mesh to an MP4: with --motion, the avatar rigged as "
                    "avatarclip_b200.drive rigs it and performing the motion; without, a 360 degree turntable.",
        epilog="The SMPL .npz is the one avatarclip_b200.drive reads (python -m avatarclip_b200.drive --help).")
    p.add_argument("--mesh", required=True, help="PLY written by --mode validate_mesh")
    p.add_argument("--out", required=True, help="the .mp4 to write")
    p.add_argument("--motion", default=None, help=".npy of shape [frames, >= 72] (SMPL axis-angle per frame)")
    p.add_argument("--smpl", default=None, help=".npz with the SMPL tensors (with --motion)")
    p.add_argument("--stand_pose", default=None, help="ShapeGen/output/stand_pose.npy (with --motion)")
    p.add_argument("--orbit_degrees", type=float, default=0.0, help="camera turn about the up axis over the motion")
    p.add_argument("--frames", type=int, default=None, help="turntable frames (default 120)")
    p.add_argument("--image_size", type=int, default=512)
    p.add_argument("--supersample", type=int, default=2)
    p.add_argument("--fps", type=float, default=drive.PC2_SAMPLE_RATE)
    p.add_argument("--frames_per_chunk", type=int, default=None, help="frames rendered per device chunk")
    p.add_argument("--device", default="cuda")
    return p


def main(argv=None) -> int:
    parser = build_parser()
    a = parser.parse_args(argv)
    if not 1 <= a.image_size <= 4096:
        parser.error("--image_size must be in [1, 4096]")
    if not 1 <= a.supersample <= 4:
        parser.error("--supersample must be in [1, 4]")
    if not a.fps > 0:
        parser.error("--fps must be > 0")
    if a.frames_per_chunk is not None and a.frames_per_chunk < 1:
        parser.error("--frames_per_chunk must be >= 1")
    if a.motion is None:
        for flag, val in (("--smpl", a.smpl), ("--stand_pose", a.stand_pose)):
            if val is not None:
                parser.error(f"{flag} is only used with --motion")
        if a.orbit_degrees:
            parser.error("--orbit_degrees is only used with --motion (a turntable turns 360 degrees)")
        if a.frames is not None and a.frames < 1:
            parser.error("--frames must be >= 1")
    else:
        if a.frames is not None:
            parser.error("--frames sets the turntable length; a motion renders each of its frames")
        for flag, val in (("--smpl", a.smpl), ("--stand_pose", a.stand_pose)):
            if val is None:
                parser.error(f"--motion needs {flag}")
    for flag, path in (("--mesh", a.mesh), ("--motion", a.motion), ("--smpl", a.smpl), ("--stand_pose", a.stand_pose)):
        if path is not None and not os.path.isfile(path):
            parser.error(f"{flag}: no such file: {path}")
    if a.motion is None:
        frames = iter_turntable_frames(a.mesh, n_frames=a.frames or 120, image_size=a.image_size,
                                       supersample=a.supersample, frames_per_chunk=a.frames_per_chunk, device=a.device)
    else:
        try:
            smpl = drive.load_smpl_npz(a.smpl)
        except (ValueError, OSError) as e:
            parser.error(f"--smpl: {e}")
        frames = iter_motion_frames(a.mesh, a.motion, smpl, a.stand_pose, image_size=a.image_size,
                                    supersample=a.supersample, orbit_degrees=a.orbit_degrees,
                                    frames_per_chunk=a.frames_per_chunk, device=a.device)
    n = write_video(frames, a.out, a.fps)
    print(f"{a.out}: {n} frames, {a.image_size}x{a.image_size}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
