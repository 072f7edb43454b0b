"""Host-side mirror of ExAvatar's render boundary.

`GaussianRenderer.forward` restates /root/reference/avatar/common/nets/module.py:592-647 (the only
caller of the rasteriser) without its hard-coded `.cuda()` calls, so the same code drives the GPU
rasteriser on a GPU box and the CPU oracle in tests.  Argument meaning, the settings tuple
(module.py:609-622), the dummy `mean_2d` leaf (module.py:626-629) and the returned dict
(module.py:642-647) are the reference's.

`render_settings` additionally caches the per-camera setup: the reference rebuilds the matrices with
~8 host<->device syncs per call (SURVEY section 8a row a1); a caller that renders five asset sets with one
camera (avatar/main/model.py:130-162) can build the settings once and reuse them.
"""
from __future__ import annotations

import torch
from torch import nn

from . import _lib as L
from .camera import get_fov, get_proj_matrix, get_view_matrix
from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer
from .sh import sh_to_rgb


# Camera setup of CUDA-resident camera parameters.  The reference evaluates module.py:604-613 on the device: ~35 tiny
# kernels and five device->host synchronisations per render (float(torch.tan(.)), math.tan(float(.)), .inverse()), i.e.
# the host waits for everything the GPU still has queued, five times per render, 25 times per training frame.  The
# arithmetic is 16 floats of input, so this mirror fetches them with ONE packed copy, evaluates the same functions of
# camera.py on the CPU (where they are pinned bit for bit on the reference's own output, tests/test_golden.py) and
# uploads the three results with one packed copy.  The five renders of a frame share the camera (model.py:130-162):
# results are cached per camera -- the entry keeps the caller's tensors alive, so a storage address can never be seen
# with different contents, and an in-place update bumps the version and misses.
_CAM_CACHE = {}
_CAM_CACHE_MAX = 8


def _device_camera(img_shape, cam_param):
    keys = ("R", "t", "focal", "princpt")
    ts = [cam_param[k] for k in keys]
    key = tuple((t.data_ptr(), t._version, tuple(t.shape), t.dtype) for t in ts) + (int(img_shape[0]), int(img_shape[1]))
    hit = _CAM_CACHE.get(key)
    if hit is not None:
        return hit[1]
    dev = ts[0].device
    packed = torch.cat([t.reshape(-1).float() for t in ts]).cpu()  # one kernel, one copy, one synchronisation
    host = {"R": packed[0:9].view(3, 3), "t": packed[9:12], "focal": packed[12:14], "princpt": packed[14:16]}
    fov = get_fov(host["focal"], host["princpt"], img_shape)
    view = get_view_matrix(host["R"], host["t"]).permute(1, 0)
    proj = get_proj_matrix(host["focal"], host["princpt"], img_shape, 0.01, 100, 1.0).permute(1, 0)
    full = torch.mm(view, proj)
    campos = view.inverse()[3, :3]
    up = torch.cat((view.reshape(-1), full.reshape(-1), campos.reshape(-1))).to(dev)
    out = (up[0:16].view(4, 4), up[16:32].view(4, 4), up[32:35], float(torch.tan(fov[0] / 2)), float(torch.tan(fov[1] / 2)))
    if len(_CAM_CACHE) >= _CAM_CACHE_MAX:
        _CAM_CACHE.pop(next(iter(_CAM_CACHE)))
    _CAM_CACHE[key] = (ts, out)  # `ts` held on purpose: pins the storage the key refers to
    return out


def device_render_settings(img_shape, cam_param, bg):
    """`render_settings` for a camera given as CUDA tensors, computed on the device: one `b2r_camera_setup` launch writes
    a fresh 37-float block view | full projection | campos | tan(fov_x/2) | tan(fov_y/2), and the returned settings'
    viewmatrix, projmatrix, campos and tanfovx / tanfovy (0-dim tensors) are views of it.  Nothing is read back, so a
    new camera every frame costs no host synchronisation, and `TrainingFrameRenderer(use_graph=True)` replays one
    captured frame for every camera.  The arithmetic is module.py:604-613's as the reference evaluates it on the device
    (include/b200raster.h); it is not bit-equal to `render_settings`, whose host mirror evaluates atan / tan with torch's
    CPU kernels.  R (3,3), t (3) and focal (2) are read as fp32; princpt is ignored, as in the reference."""
    R, t, focal = cam_param["R"], cam_param["t"], cam_param["focal"]
    if not (R.is_cuda and t.is_cuda and focal.is_cuda):
        raise RuntimeError("device_render_settings: cam_param R, t and focal must be CUDA tensors (use render_settings "
                           "for a CPU camera)")
    dev = R.device
    R, t, focal = (x.to(dev, torch.float32).contiguous() for x in (R.reshape(9), t.reshape(3), focal.reshape(2)))
    H, W = int(img_shape[0]), int(img_shape[1])
    block = torch.empty(37, dtype=torch.float32, device=dev)
    L.run("b2r_camera_setup", dev, R.data_ptr(), t.data_ptr(), focal.data_ptr(), W, H, block.data_ptr())
    return GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=block[35], tanfovy=block[36], bg=bg,
                                         scale_modifier=1.0, viewmatrix=block[0:16].view(4, 4),
                                         projmatrix=block[16:32].view(4, 4), sh_degree=0, campos=block[32:35],
                                         prefiltered=False, debug=False)


def render_settings(img_shape, cam_param, bg, settings_cls=GaussianRasterizationSettings):
    """module.py:604-622: fov, transposed view / full-projection matrices, camera position, settings tuple."""
    if cam_param["R"].is_cuda:
        view_matrix, full_proj_matrix, cam_pos, tanx, tany = _device_camera(img_shape, cam_param)
        return settings_cls(image_height=img_shape[0], image_width=img_shape[1], tanfovx=tanx, tanfovy=tany, bg=bg,
                            scale_modifier=1.0, viewmatrix=view_matrix, projmatrix=full_proj_matrix, sh_degree=0,
                            campos=cam_pos, prefiltered=False, debug=False)
    fov = get_fov(cam_param["focal"], cam_param["princpt"], img_shape)
    view_matrix = get_view_matrix(cam_param["R"], cam_param["t"]).permute(1, 0)
    proj_matrix = get_proj_matrix(cam_param["focal"], cam_param["princpt"], img_shape, 0.01, 100, 1.0).permute(1, 0)
    full_proj_matrix = torch.mm(view_matrix, proj_matrix)
    cam_pos = view_matrix.inverse()[3, :3]
    return settings_cls(
        image_height=img_shape[0],
        image_width=img_shape[1],
        tanfovx=float(torch.tan(fov[0] / 2)),
        tanfovy=float(torch.tan(fov[1] / 2)),
        bg=bg,
        scale_modifier=1.0,
        viewmatrix=view_matrix,
        projmatrix=full_proj_matrix,
        sh_degree=0,  # colours are precomputed by the caller (module.py:618)
        campos=cam_pos,
        prefiltered=False,
        debug=False,
    )


class GaussianRenderer(nn.Module):
    """Same call as module.py:588-647; `rasterizer_cls` / `settings_cls` let tests substitute the CPU oracle."""

    def __init__(self, rasterizer_cls=GaussianRasterizer, settings_cls=GaussianRasterizationSettings):
        super().__init__()
        self.rasterizer_cls = rasterizer_cls
        self.settings_cls = settings_cls

    def forward(self, gaussian_assets, img_shape, cam_param, bg=None, raster_settings=None):
        mean_3d = gaussian_assets["mean_3d"]
        if bg is None:  # reference default: white (module.py:592)
            bg = torch.ones(3, dtype=torch.float32, device=mean_3d.device)
        if raster_settings is None:
            raster_settings = render_settings(img_shape, cam_param, bg, self.settings_cls)
        rasterizer = self.rasterizer_cls(raster_settings=raster_settings)

        # screen-space positions: a zero leaf whose .grad is read after backward (train.py:51, model.py:285)
        mean_2d = torch.zeros((mean_3d.shape[0], 3), dtype=torch.float32, device=mean_3d.device)
        mean_2d.requires_grad = True
        mean_2d.retain_grad()

        # Reference call: colours precomputed by the caller (module.py:635-636).  SURVEY.md section 8f-4: assets that carry
        # `shs` (P, M, 3) + `sh_degree` instead of `rgb` are coloured inside the projection kernel.
        shs = gaussian_assets.get("shs") if "rgb" not in gaussian_assets else None
        if shs is not None:
            rasterizer = self.rasterizer_cls(raster_settings=raster_settings._replace(sh_degree=int(gaussian_assets["sh_degree"])))

        render_img, radius, render_depthmap, render_mask = rasterizer(
            means3D=mean_3d,
            means2D=mean_2d,
            shs=shs,
            colors_precomp=None if shs is not None else gaussian_assets["rgb"],
            opacities=gaussian_assets["opacity"],
            scales=gaussian_assets["scale"],
            rotations=gaussian_assets["rotation"],
            cov3D_precomp=None)

        return {"img": render_img,
                "depthmap": render_depthmap,
                "mask": render_mask,
                "mean_2d": mean_2d,
                "is_vis": radius > 0,
                "radius": radius}


def scene_gaussian_assets(mean, opacity_logit, log_scale, rotation, feature_dc, feature_rest, active_sh_degree, cam_param,
                          in_kernel_sh: bool = False):
    """The asset dict `SceneGaussian.forward` hands to the renderer (module.py:253-272): sigmoid opacity, exp scale,
    SH coefficients `cat(feature_dc, feature_rest)` (P, 16, 3).  `rotation` is the activated quaternion (the reference
    derives it from a 6-D parametrisation with pytorch3d, which is outside this path).

    in_kernel_sh=False reproduces the reference: view direction, SH polynomial and clamp in PyTorch -> `rgb`.
    in_kernel_sh=True  (SURVEY.md section 8f-4) passes `shs` + `sh_degree` through; the rasteriser evaluates the same
    polynomial per Gaussian in its projection kernel and back-propagates to the coefficients and, through the view
    direction, to the mean -- no (P,16,3)->(P,3) PyTorch kernels, no (P,3) colour round trip through HBM."""
    sh = torch.cat((feature_dc, feature_rest), 1)
    assets = {"mean_3d": mean, "opacity": torch.sigmoid(opacity_logit), "scale": torch.exp(log_scale), "rotation": rotation}
    if in_kernel_sh:
        assets["shs"] = sh
        assets["sh_degree"] = int(active_sh_degree)
    else:
        cam_pos = torch.matmul(torch.inverse(cam_param["R"]), -cam_param["t"].view(3, 1)).view(1, 3)
        assets["rgb"] = sh_to_rgb(int(active_sh_degree), sh, mean, cam_pos.to(mean.dtype))
    return assets


def lbs_reference(xyz, skin_weights, joint_mats, trans, cam_R=None, cam_t=None, cam_R_inv=None):
    """Caller-side mirror of how `HumanGaussian.forward` poses its Gaussians -- `get_transform_mat_vertex`, `lbs` and the
    camera->world transform, op for op (module.py:413-422, 555-557); device-agnostic, differentiable.  This is the
    reference the skinning op `skinning.skin_gaussians` and `SkinnedGaussianRasterizer` (SURVEY section 8f-2) are
    compared against; the product path never calls it.
    `cam_R_inv` (optional) skips the `torch.inverse` call, e.g. inside a CUDA-graph capture."""
    P, J = skin_weights.shape
    tmv = torch.matmul(skin_weights, joint_mats.reshape(J, 16)).view(P, 4, 4)
    xyz1 = torch.cat((xyz, torch.ones_like(xyz[:, :1])), 1)
    posed = torch.bmm(tmv, xyz1[:, :, None]).view(P, 4)[:, :3] + trans.reshape(1, 3)
    if cam_R is not None or cam_R_inv is not None:
        Rinv = torch.inverse(cam_R) if cam_R_inv is None else cam_R_inv
        posed = torch.matmul(Rinv, (posed - cam_t.view(1, 3)).permute(1, 0)).permute(1, 0)
    return posed
