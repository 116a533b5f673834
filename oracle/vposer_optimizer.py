"""CPU oracle (test infrastructure, never on the product path): VPoser 2.x's decode as torch fp64 autograd, so that its
gradient is the reference's -- the gradient of AvatarAnimate's VPoserOptimizer with respect to its latent.

PARITY UNPINNED, as for oracle/animate.py's numpy ``vposer_decode`` (whose forward this equals): ``human_body_prior``
and the torchgeometry it calls are neither vendored nor installed, so both are restated from their published
algorithms.  The restatement follows torchgeometry's formulation literally -- ``rotation_matrix_to_quaternion`` builds
all four candidate quaternions on the transposed matrix and blends them with masks (eps 1e-6), and
``quaternion_to_angle_axis`` selects its atan2 and its k with ``torch.where`` -- so that autograd gives the gradient the
reference's autograd gives: only the selected branch carries gradient, through its 0.5 / sqrt(t) included; F.normalize's
clamp at 1e-12 passes none where it is active; LeakyReLU(0.01) on each pre-activation; Dropout is the identity in eval.
At an exact identity rotation (sin theta = 0) torch's backward is NaN (sqrt's backward at 0).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def rot6d_to_matrix(x: torch.Tensor) -> torch.Tensor:
    """ContinousRotReprDecoder: [N, 6] -> [N, 3, 3], R = [b1 b2 b3] as columns."""
    m = x.reshape(-1, 3, 2)
    b1 = F.normalize(m[:, :, 0], dim=1)
    dot = torch.sum(b1 * m[:, :, 1], dim=1, keepdim=True)
    b2 = F.normalize(m[:, :, 1] - dot * b1, dim=-1)
    b3 = torch.cross(b1, b2, dim=1)
    return torch.stack([b1, b2, b3], dim=-1)


def branches(R: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """Which of rotation_matrix_to_quaternion's four masked branches each [N, 3, 3] takes (0..3)."""
    m = R.transpose(1, 2)
    d2, d0_d1, d0_nd1 = m[:, 2, 2] < eps, m[:, 0, 0] > m[:, 1, 1], m[:, 0, 0] < -m[:, 1, 1]
    return torch.where(d2, torch.where(d0_d1, 0, 1), torch.where(d0_nd1, 2, 3))


def rotation_matrix_to_quaternion(R: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """torchgeometry's masked formulation on rmat_t = R^T: [N, 3, 3] -> [N, 4] (w, x, y, z)."""
    m = R.transpose(1, 2)
    mask_d2 = m[:, 2, 2] < eps
    mask_d0_d1 = m[:, 0, 0] > m[:, 1, 1]
    mask_d0_nd1 = m[:, 0, 0] < -m[:, 1, 1]
    t0 = 1 + m[:, 0, 0] - m[:, 1, 1] - m[:, 2, 2]
    q0 = torch.stack([m[:, 1, 2] - m[:, 2, 1], t0, m[:, 0, 1] + m[:, 1, 0], m[:, 2, 0] + m[:, 0, 2]], -1)
    t1 = 1 - m[:, 0, 0] + m[:, 1, 1] - m[:, 2, 2]
    q1 = torch.stack([m[:, 2, 0] - m[:, 0, 2], m[:, 0, 1] + m[:, 1, 0], t1, m[:, 1, 2] + m[:, 2, 1]], -1)
    t2 = 1 - m[:, 0, 0] - m[:, 1, 1] + m[:, 2, 2]
    q2 = torch.stack([m[:, 0, 1] - m[:, 1, 0], m[:, 2, 0] + m[:, 0, 2], m[:, 1, 2] + m[:, 2, 1], t2], -1)
    t3 = 1 + m[:, 0, 0] + m[:, 1, 1] + m[:, 2, 2]
    q3 = torch.stack([t3, m[:, 1, 2] - m[:, 2, 1], m[:, 2, 0] - m[:, 0, 2], m[:, 0, 1] - m[:, 1, 0]], -1)
    rep = lambda t: t.repeat(4, 1).t()
    c0 = (mask_d2 & mask_d0_d1).view(-1, 1).type_as(q0)
    c1 = (mask_d2 & ~mask_d0_d1).view(-1, 1).type_as(q1)
    c2 = (~mask_d2 & mask_d0_nd1).view(-1, 1).type_as(q2)
    c3 = (~mask_d2 & ~mask_d0_nd1).view(-1, 1).type_as(q3)
    q = q0 * c0 + q1 * c1 + q2 * c2 + q3 * c3
    q = q / torch.sqrt(rep(t0) * c0 + rep(t1) * c1 + rep(t2) * c2 + rep(t3) * c3)
    return q * 0.5


def quaternion_to_angle_axis(q: torch.Tensor) -> torch.Tensor:
    """torchgeometry's quaternion_to_angle_axis: [N, 4] -> [N, 3]."""
    q1, q2, q3 = q[..., 1], q[..., 2], q[..., 3]
    s2 = q1 * q1 + q2 * q2 + q3 * q3
    s = torch.sqrt(s2)
    co = q[..., 0]
    two_theta = 2.0 * torch.where(co < 0.0, torch.atan2(-s, -co), torch.atan2(s, co))
    k = torch.where(s2 > 0.0, two_theta / s, 2.0 * torch.ones_like(s))
    return torch.stack([q1 * k, q2 * k, q3 * k], -1)


def atan2_negative(R: torch.Tensor) -> torch.Tensor:
    """Whether quaternion_to_angle_axis takes its atan2(-s, -q0) branch (q0 < 0) for each [N, 3, 3]."""
    return rotation_matrix_to_quaternion(R)[:, 0] < 0


def decoder_rotations(z: torch.Tensor, sd: dict) -> torch.Tensor:
    """decoder_net then ContinousRotReprDecoder: the rotation matrices [B * n_joints, 3, 3] in z's dtype."""
    w = lambda k: torch.as_tensor(sd[f"decoder_net.{k}"]).to(z.dtype)
    h = F.leaky_relu(z @ w("0.weight").T + w("0.bias"), 0.01)
    h = F.leaky_relu(h @ w("3.weight").T + w("3.bias"), 0.01)
    return rot6d_to_matrix((h @ w("5.weight").T + w("5.bias")).reshape(-1, 6))


def decode(z: torch.Tensor, sd: dict) -> torch.Tensor:
    """VPoser.decode(z)['pose_body'] [B, n_joints, 3] in z's dtype, differentiable in z (and the weights)."""
    R = decoder_rotations(z, sd)
    return quaternion_to_angle_axis(rotation_matrix_to_quaternion(R)).reshape(z.shape[0], -1, 3)


class VPoserDecoder(torch.nn.Module):
    """What ``load_model(vposer_path, model_code=VPoser, ...)`` returns, as far as VPoserOptimizer uses it: ``decode(z)``
    -> {'pose_body': [B, n_joints, 3]} in fp32, computed in fp64 by ``decode`` with gradient to z."""

    def __init__(self, sd: dict):
        super().__init__()
        self.sd = {k: torch.as_tensor(v).double() for k, v in sd.items()}

    def decode(self, z: torch.Tensor) -> dict:
        return {"pose_body": decode(z.double(), self.sd).float()}


def axis_angle_matrix(axis, angle: float) -> torch.Tensor:
    """Rodrigues: the fp64 rotation by angle about axis (normalised)."""
    a = torch.as_tensor(axis, dtype=torch.float64)
    a = a / a.norm()
    K = torch.tensor([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]], dtype=torch.float64)
    return torch.eye(3, dtype=torch.float64) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K


# rotations whose matrices take each of rotation_matrix_to_quaternion's branches (0, 0, 1, 1, 2, 2, 3) and, for the
# near-pi ones, both signs of q0 (both of quaternion_to_angle_axis's atan2 branches), all clear of every branch boundary
STEER = (((1.0, 0.1, -0.1), 2.6), ((1.0, -0.1, 0.1), -2.6), ((0.1, 1.0, 0.1), 2.6), ((-0.1, 1.0, 0.1), -2.6),
         ((0.1, -0.1, 1.0), 2.6), ((0.1, 0.1, 1.0), -2.6), ((0.3, -0.5, 0.8), 0.7))


def steered_state(seed: int = 31, latent: int = 32, hidden: int = 512, n_joints: int = 21) -> dict:
    """decoder_net weights whose joint j decodes near STEER[j % 7]: decoder_net.5.bias holds that rotation's 6D
    encoding (its first two columns, the [3, 2] matrix row-major) and decoder_net.5.weight is small, so every row of a
    unit-normal latent keeps each joint on its rotation's branches."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, std: torch.randn(*s, generator=g) * std
    bias = torch.stack([axis_angle_matrix(*STEER[j % len(STEER)])[:, :2].reshape(6) for j in range(n_joints)])
    return {"decoder_net.0.weight": rn(hidden, latent, std=0.3), "decoder_net.0.bias": rn(hidden, std=0.1),
            "decoder_net.3.weight": rn(hidden, hidden, std=0.06), "decoder_net.3.bias": rn(hidden, std=0.1),
            "decoder_net.5.weight": rn(6 * n_joints, hidden, std=0.002), "decoder_net.5.bias": bias.reshape(-1).float()}
