"""Camera matrices exactly as ExAvatar builds them for the rasteriser.

Device-agnostic restatement of /root/reference/avatar/common/utils/transforms.py:38-70
(`get_view_matrix`, `get_proj_matrix`, `get_fov`), which hard-code `.cuda()` and therefore cannot
run on a CPU test box.  Semantics kept on purpose:
  * the principal point is accepted and IGNORED (transforms.py:66-70 uses focal and image shape only),
  * znear/zfar enter only the (unused-by-the-rasteriser) third row of the projection,
  * tan(fov/2) is evaluated in Python float64 (math.tan) and stored as fp32 (transforms.py:47-48,57-58).
"""
from __future__ import annotations

import math

import torch


def get_fov(focal, princpt, img_shape):
    """transforms.py:66-70.  Returns tensor([fov_x, fov_y]) (fp32) on focal's device."""
    fov_x = 2 * torch.atan(img_shape[1] / (2 * focal[0]))
    fov_y = 2 * torch.atan(img_shape[0] / (2 * focal[1]))
    return torch.stack([fov_x.float().reshape(()), fov_y.float().reshape(())]).to(focal.device)


def get_view_matrix(R, t):
    """transforms.py:38-41.  4x4 [R t; 0 0 0 1]."""
    Rt = torch.cat((R, t.view(3, 1)), 1)
    bottom = torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=torch.float32, device=R.device)
    return torch.cat((Rt, bottom))


def get_proj_matrix(focal, princpt, img_shape, z_near, z_far, z_sign):
    """transforms.py:43-64.  OpenGL-style perspective with a centred principal point."""
    fov = get_fov(focal, princpt, img_shape)
    tan_half_y = math.tan(float(fov[1]) / 2)
    tan_half_x = math.tan(float(fov[0]) / 2)
    top = tan_half_y * z_near
    bottom = -top
    right = tan_half_x * z_near
    left = -right
    z_sign = 1.0
    m = torch.zeros(4, 4, dtype=torch.float32)
    m[0, 0] = 2.0 * z_near / (right - left)
    m[1, 1] = 2.0 * z_near / (top - bottom)
    m[0, 2] = (right + left) / (right - left)
    m[1, 2] = (top + bottom) / (top - bottom)
    m[3, 2] = z_sign
    m[2, 2] = z_sign * z_far / (z_far - z_near)
    m[2, 3] = -(z_far * z_near) / (z_far - z_near)
    return m.to(focal.device)


def _inv3(R: torch.Tensor) -> torch.Tensor:
    """3x3 inverse by cofactors: a handful of elementwise kernels, no cuSOLVER call -- capturable in a CUDA graph
    (`torch.inverse`, which the reference uses at module.py:556, synchronises)."""
    a, b, c, d, e, f, g, h, i = R.reshape(9).unbind()
    adj = torch.stack((e * i - f * h, c * h - b * i, b * f - c * e,
                       f * g - d * i, a * i - c * g, c * d - a * f,
                       d * h - e * g, b * g - a * h, a * e - b * d)).reshape(3, 3)
    return adj / (a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g))


def look_at_cam_param(yaw_deg: float, img_shape, focal_ratio: float = 1.465, target_z: float = 4.24, device="cpu"):
    """Synthetic camera orbiting the subject (SURVEY section 8d: fx = fy = 1.465*H, subject at z = 4.24 m)."""
    H, W = img_shape
    a = math.radians(yaw_deg)
    # rotate the world about the vertical axis through the subject centre
    Ry = torch.tensor([[math.cos(a), 0.0, math.sin(a)], [0.0, 1.0, 0.0], [-math.sin(a), 0.0, math.cos(a)]],
                      dtype=torch.float32)
    c = torch.tensor([0.0, 0.0, target_z])
    t = c - Ry @ c
    f = focal_ratio * H
    return {
        "R": Ry.to(device), "t": t.to(device),
        "focal": torch.tensor([f, f], dtype=torch.float32, device=device),
        "princpt": torch.tensor([W / 2.0, H / 2.0], dtype=torch.float32, device=device),
    }
