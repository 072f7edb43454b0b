"""`scene_assets` -- ExAvatar's `SceneGaussian.forward` (avatar/common/nets/module.py:253-272) as one sync-free CUDA op.

Every frame ExAvatar turns the scene's stored parameters into the asset dict the renders read: sigmoid opacity, exp
scale, the quaternion of pytorch3d's `matrix_to_quaternion(rotation_6d_to_matrix(rotation))`, the SH coefficients
`cat(feature_dc, feature_rest)` and, for the reference's own renderer, the colour `eval_sh` gives them seen from the
camera.  In PyTorch that is dozens of elementwise kernels each way, and `eval_sh`'s asserts and `if deg > k` on the
float `active_sh_degree` buffer plus `torch.inverse(R)` read the device from the host.  `scene_assets` computes the same
dict in one forward and one backward launch (csrc/scene_assets.cu); the degree is read on the device, so the op can sit
in a CUDA graph that replays across ExAvatar's SH schedule.

    assets = scene_assets(mean, opacity, scale, rotation, feature_dc, feature_rest, active_sh_degree)  # shs mode
    TrainingFrameRenderer(..., sh_coeffs=16)(assets, human, refined, cam, bg)
    assets = scene_assets(..., active_sh_degree_buffer, cam_param)                                   # rgb mode
    GaussianRenderer()(assets, img_shape, cam_param)

`scene_assets_reference` restates the reference lines in device-agnostic torch (float64 or float32) for tests and
measurements; the product path never calls it.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib as L
from .camera import _inv3
from .sh import sh_to_rgb
from .smplx_rig import matrix_to_quaternion, rotation_6d_to_matrix

MAX_COEFFS = 16  # B2R_SCENE_MAX_COEFFS: a CTA stages 3 M floats per Gaussian through shared memory


def _rows(t: torch.Tensor, row_len: int):
    """(tensor, row stride in floats): rows of `row_len` contiguous floats read in place, or a contiguous copy."""
    inner_ok = t.shape[1] == 1 or t.stride(1) == 3
    if t.stride(2) == 1 and inner_ok and (t.shape[0] <= 1 or t.stride(0) >= row_len):
        return t, max(int(t.stride(0)), row_len)
    return t.contiguous(), row_len


def _struct(P, M, mean, logit, log_scale, rot6d, dc, dc_stride, rest, rest_stride, deg, R, t) -> "L.B2RSceneAssets":
    s = L.B2RSceneAssets(P=P, M=M, dc_stride=dc_stride, rest_stride=rest_stride)
    s.mean, s.opacity_logit, s.log_scale, s.rotation6d = L.ptr(mean), L.ptr(logit), L.ptr(log_scale), L.ptr(rot6d)
    s.feature_dc, s.feature_rest, s.active_sh_degree = L.ptr(dc), L.ptr(rest), L.ptr(deg)
    s.cam_R, s.cam_t = L.ptr(R), L.ptr(t)
    return s


class _SceneAssets(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mean, logit, log_scale, rot6d, feature_dc, feature_rest, deg, R, t):
        dev = logit.device
        P, M = logit.shape[0], 1 + feature_rest.shape[1]
        rgb = R is not None
        dc, dc_stride = _rows(feature_dc.detach(), 3)
        rest, rest_stride = _rows(feature_rest.detach(), 3 * (M - 1))
        ins = [x.detach().contiguous() if x is not None else None for x in (mean, logit, log_scale, rot6d)]
        f = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)  # noqa: E731
        opacity, scale, rotation = f(P, 1), f(P, 3), f(P, 4)
        color = f(P, 3) if rgb else f(P, M, 3)
        st = _struct(P, M, *ins, dc, dc_stride, rest, rest_stride, deg, R, t)
        L.run("b2r_scene_assets_forward", dev, C.byref(st), L.ptr(opacity), L.ptr(scale), L.ptr(rotation), L.ptr(color))
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(*ins, dc, rest, deg, R, t, opacity, scale)
        ctx.meta = (P, M, dc_stride, rest_stride, logit.shape, feature_dc.shape, feature_rest.shape)
        return opacity, scale, rotation, color

    @staticmethod
    def backward(ctx, g_opacity, g_scale, g_rotation, g_color):
        mean, logit, log_scale, rot6d, dc, rest, deg, R, t, opacity, scale = ctx.saved_tensors
        P, M, dc_stride, rest_stride, logit_shape, dc_shape, rest_shape = ctx.meta
        dev = logit.device
        up = [None if g is None else g.to(torch.float32).contiguous() for g in (g_opacity, g_scale, g_rotation, g_color)]
        f = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)  # noqa: E731
        d_logit, d_log_scale, d_rot6d = f(*logit_shape), f(P, 3), f(P, 6)
        d_dc, d_rest = f(*dc_shape), f(*rest_shape)
        d_mean = f(P, 3) if R is not None else None
        gs = L.B2RSceneAssetsGrads(*[L.ptr(x) for x in (opacity, scale, *up, d_logit, d_log_scale, d_rot6d, d_dc,
                                                        d_rest, d_mean)])
        st = _struct(P, M, mean, logit, log_scale, rot6d, dc, dc_stride, rest, rest_stride, deg, R, t)
        L.run("b2r_scene_assets_backward", dev, C.byref(st), C.byref(gs))
        return d_mean, d_logit, d_log_scale, d_rot6d, d_dc, d_rest, None, None, None


def _check(name, t, shape, dev):
    L.cuda("scene_assets", name, t, dev)
    L.float32("scene_assets", name, t)
    if shape is not None and tuple(t.shape) != shape:
        raise ValueError(f"scene_assets: `{name}` must be {shape}, got {tuple(t.shape)}")


def scene_assets(mean, opacity_logit, log_scale, rotation6d, feature_dc, feature_rest, active_sh_degree,
                 cam_param: Optional[dict] = None) -> dict:
    """SceneGaussian.forward's asset dict from the scene's float32 CUDA parameters: mean (P,3), opacity_logit (P,1),
    log_scale (P,3), rotation6d (P,6), feature_dc (P,1,3) and feature_rest (P,M-1,3), 1 <= M <= 16.  Views such as
    init_from_point_cloud's slices of one (P,M,3) tensor are read through their strides.

    cam_param None (shs mode): {mean_3d, opacity, scale, rotation, shs (P,M,3), sh_degree}, what
    `TrainingFrameRenderer(sh_coeffs=M)` takes; `sh_degree` is `active_sh_degree` as given (the renderer reads it as a
    host int).  Otherwise (rgb mode): {mean_3d, opacity, scale, rotation, rgb (P,3)}, what `GaussianRenderer`, the
    five-call drop-in and the test-mode forward take, with `active_sh_degree` ExAvatar's (1,) float CUDA buffer read on
    the device and cam_param's R (3,3) and t (3) on the same device; the camera gets no gradient.  A buffer degree
    outside 0..3, or one needing more than M coefficients, gives NaN colours.  `mean_3d` is `mean` itself.  Gradients
    reach every parameter (mean through the view direction in rgb mode, as well as through mean_3d)."""
    dev = mean.device if isinstance(mean, torch.Tensor) else None
    _check("mean", mean, None, dev)
    P = mean.shape[0]
    if mean.dim() != 2 or mean.shape[1] != 3:
        raise ValueError(f"scene_assets: `mean` must be (P,3), got {tuple(mean.shape)}")
    if not isinstance(feature_rest, torch.Tensor) or feature_rest.dim() != 3:
        raise ValueError("scene_assets: `feature_rest` must be a (P,M-1,3) tensor")
    M = 1 + feature_rest.shape[1]
    if not 1 <= M <= MAX_COEFFS:
        raise ValueError(f"scene_assets: {M} SH coefficients; the op takes 1 <= M <= {MAX_COEFFS}")
    for name, t, shape in (("opacity_logit", opacity_logit, (P, 1)), ("log_scale", log_scale, (P, 3)),
                           ("rotation6d", rotation6d, (P, 6)), ("feature_dc", feature_dc, (P, 1, 3)),
                           ("feature_rest", feature_rest, (P, M - 1, 3))):
        _check(name, t, shape, dev)
    assets = {"mean_3d": mean}
    if cam_param is None:
        opacity, scale, rotation, shs = _SceneAssets.apply(None, opacity_logit, log_scale, rotation6d, feature_dc,
                                                           feature_rest, None, None, None)
        assets.update(opacity=opacity, scale=scale, rotation=rotation, shs=shs, sh_degree=active_sh_degree)
        return assets
    _check("active_sh_degree", active_sh_degree, None, dev)
    if active_sh_degree.numel() != 1:
        raise ValueError("scene_assets: `active_sh_degree` must be a one-element float32 CUDA buffer")
    R, t = cam_param["R"], cam_param["t"]
    for name, x in (("cam_param['R']", R), ("cam_param['t']", t)):
        L.cuda("scene_assets", name, x, dev)
    if tuple(R.shape) != (3, 3) or t.numel() != 3:
        raise ValueError(f"scene_assets: cam_param R must be (3,3) and t have 3 elements, got {tuple(R.shape)}, "
                         f"{tuple(t.shape)}")
    R = R.detach().to(torch.float32).contiguous()
    t = t.detach().to(torch.float32).reshape(3).contiguous()
    opacity, scale, rotation, rgb = _SceneAssets.apply(mean, opacity_logit, log_scale, rotation6d, feature_dc,
                                                       feature_rest, active_sh_degree.detach(), R, t)
    assets.update(opacity=opacity, scale=scale, rotation=rotation, rgb=rgb)
    return assets


def scene_assets_reference(mean, opacity_logit, log_scale, rotation6d, feature_dc, feature_rest, active_sh_degree,
                           cam_param: Optional[dict] = None) -> dict:
    """module.py:253-272 restated in device-agnostic torch, differentiable, in the inputs' dtype: pytorch3d's two
    conversions as smplx_rig restates them, campos = -R^-1 t by cofactors, and eval_sh with ExAvatar's comparisons of
    the degree (deg > 0, > 1, > 2; 0 <= deg <= 3 and (deg + 1)^2 <= M asserted).  Reads the degree on the host."""
    sh = torch.cat((feature_dc, feature_rest), 1)
    assets = {"mean_3d": mean, "opacity": torch.sigmoid(opacity_logit), "scale": torch.exp(log_scale),
              "rotation": matrix_to_quaternion(rotation_6d_to_matrix(rotation6d))}
    if cam_param is None:
        assets.update(shs=sh, sh_degree=active_sh_degree)
        return assets
    deg = float(active_sh_degree.reshape(-1)[0]) if isinstance(active_sh_degree, torch.Tensor) else float(active_sh_degree)
    if not (0 <= deg <= 3 and (deg + 1) ** 2 <= sh.shape[1]):
        raise ValueError(f"scene_assets_reference: degree {deg} with {sh.shape[1]} coefficients")
    level = sum(deg > k for k in (0, 1, 2))
    if (level + 1) ** 2 > sh.shape[1]:
        raise ValueError(f"scene_assets_reference: degree {deg} reads {(level + 1) ** 2} coefficients")
    R = cam_param["R"].to(device=mean.device, dtype=mean.dtype)
    t = cam_param["t"].to(device=mean.device, dtype=mean.dtype)
    cam_pos = torch.matmul(_inv3(R), -t.reshape(3, 1)).view(1, 3)
    assets["rgb"] = sh_to_rgb(level, sh, mean, cam_pos)
    return assets
