"""`GaussianRasterizationSettings` / `GaussianRasterizer` -- the Python surface ExAvatar imports.

Drop-in for `from diff_gaussian_rasterization_depth import GaussianRasterizationSettings, GaussianRasterizer`
(/root/reference/avatar/common/nets/module.py:11): same 12-field settings tuple in the order of the call site
(module.py:609-622), same keyword call (module.py:632-640), same 4-tuple `(color, radii, depth, alpha)` (module.py:632),
same argument-validation exceptions, gradients for the same eight tensor inputs.  The compute is the hand-written
sm_90a library behind include/b200raster.h, on the caller's current CUDA stream; PyTorch only owns memory, streams and
autograd.  Every call goes through one host: the compiled binding csrc_torch/b2r_torch.cpp (a C++ autograd Function
over the C ABI, built in-tree by build_ext.build()).  This module maps the public arguments onto it.

No CPU path exists here on purpose: CPU tensors, a missing libb200raster.so or a missing _b2r_torch.so raise.

Duplicate-capacity policy (the reference rasteriser stalls on a device->host copy of the duplicate count every
render, SURVEY.md section 2.3 row 3):
  * "exact": run the projection phase, learn the count from a pinned-host mirror the scan kernel writes (polling, no
    stream synchronise), size the lists exactly, run the render phase;
  * "speculative" (default once a count has been seen for this shape): enqueue BOTH phases with a capacity predicted
    from the previous render of the same (P, W, H); the poll then only confirms the prediction while the GPU is
    already compositing.  A misprediction re-runs the forward with the exact size -- outputs are never truncated;
  * fixed (`set_fixed_capacity`): every render gets the same capacity and nothing is polled, so the call is capturable
    in a CUDA graph; `overflowed()` reports afterwards whether a render needed more.
"""
from __future__ import annotations

import os
from typing import NamedTuple, Optional

import torch
from torch import nn

from . import _lib as L
from .skinning import skin_gaussians


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    # Python floats (the reference's signature), or 0-dim CUDA tensors (renderer.device_render_settings): those are read
    # by the kernels on the device and never converted on the host
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


CAPACITY_MODE = os.environ.get("B2R_CAPACITY_MODE", "speculative")  # or "exact"
CAPACITY_HEADROOM = 1.25
# Fixed-capacity mode: every render uses this many list entries, nothing is polled or synchronised, so the call is
# capturable in a CUDA graph (torch.cuda.graph) together with the caller's loss, backward and copies.  Overflow is
# not repaired on the fly in this mode: check `overflowed()` after the step (outputs are truncated, never corrupt).
FIXED_CAPACITY = None


def _f32c(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise RuntimeError(f"b200raster: `{name}` must be a CUDA tensor (got {t.device}); there is no CPU fallback")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def device_tanfov(settings) -> Optional[torch.Tensor]:
    """(2) fp32 CUDA tensor (tan(fov_x / 2), tan(fov_y / 2)) of settings whose tanfovx / tanfovy are 0-dim CUDA tensors,
    None for float settings.  Adjacent fp32 elements of one block (device_render_settings, the resident block of a
    captured frame) are used in place; other tensors are stacked on the device.  Nothing is read on the host."""
    tx, ty = settings.tanfovx, settings.tanfovy
    if not isinstance(tx, torch.Tensor) and not isinstance(ty, torch.Tensor):
        return None
    if not (isinstance(tx, torch.Tensor) and isinstance(ty, torch.Tensor)) or tx.numel() != 1 or ty.numel() != 1:
        raise TypeError("b200raster: tanfovx / tanfovy must both be floats or both be one-element tensors")
    if not (tx.is_cuda and ty.is_cuda):
        raise RuntimeError("b200raster: tensor tanfovx / tanfovy must be CUDA tensors; there is no CPU fallback")
    if (tx.dtype == ty.dtype == torch.float32 and tx.device == ty.device and ty.data_ptr() == tx.data_ptr() + 4
            and tx.untyped_storage().data_ptr() == ty.untyped_storage().data_ptr()):
        return tx.as_strided((2,), (1,))
    return torch.stack((tx.reshape(()), ty.reshape(()))).float()


def _make_scene(settings: GaussianRasterizationSettings, means3D, shs, colors, opac, scales, rots, cov, flags):
    dev = means3D.device
    tanfov = device_tanfov(settings)
    keep = {
        "tanfov": None if tanfov is None else tanfov.to(dev),
        "bg": _f32c(settings.bg.to(dev), "bg"),
        "view": _f32c(settings.viewmatrix.to(dev), "viewmatrix"),
        "proj": _f32c(settings.projmatrix.to(dev), "projmatrix"),
        "campos": _f32c(settings.campos.to(dev), "campos"),
        "means3D": means3D, "shs": shs, "colors": colors, "opac": opac, "scales": scales, "rots": rots, "cov": cov,
    }
    sc = L.B2RScene()
    sc.P = means3D.shape[0]
    sc.width = int(settings.image_width)
    sc.height = int(settings.image_height)
    sc.sh_degree = int(settings.sh_degree)
    sc.sh_coeffs = 0 if shs is None or shs.numel() == 0 else int(shs.shape[1])
    sc.flags = flags
    sc.scale_modifier = float(settings.scale_modifier)
    if tanfov is None:
        sc.tanfovx = float(settings.tanfovx)
        sc.tanfovy = float(settings.tanfovy)
    sc.tanfov = L.ptr(keep["tanfov"])
    sc.bg = L.ptr(keep["bg"])
    sc.viewmatrix = L.ptr(keep["view"])
    sc.projmatrix = L.ptr(keep["proj"])
    sc.campos = L.ptr(keep["campos"])
    sc.means3D = L.ptr(means3D)
    sc.shs = L.ptr(shs)
    sc.colors_precomp = L.ptr(colors)
    sc.opacities = L.ptr(opac)
    sc.scales = L.ptr(scales)
    sc.rotations = L.ptr(rots)
    sc.cov3D_precomp = L.ptr(cov)
    return sc, keep


_EXT = None


def _compiled_binding():
    """The compiled binding of the call (csrc_torch/b2r_torch.cpp, built by build_ext.build()), loaded once.  Raises if
    it is absent -- the public call has no other host and never falls back to CPU code."""
    global _EXT
    if _EXT is None:
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_b2r_torch.so")
        if not os.path.exists(path):
            raise RuntimeError(f"b200raster: {path} not found. Build it with `python -m exavatar_release_b200.build_ext`. "
                               "There is no CPU fallback.")
        import importlib.util
        L.load()  # libb200raster.so first: the extension links against it
        spec = importlib.util.spec_from_file_location("_b2r_torch", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        if mod.abi_version() != L.ABI_VERSION:
            raise RuntimeError("b200raster: _b2r_torch.so was built against another ABI version; rebuild it")
        _EXT = mod
    return _EXT


def set_fixed_capacity(cap: Optional[int]) -> None:
    """None restores the adaptive (polling) policy."""
    global FIXED_CAPACITY
    FIXED_CAPACITY = None if cap is None else int(cap)
    _compiled_binding().clear_recent()


def overflowed() -> bool:
    """Deferred check for fixed-capacity mode: did any of the 64 most recent renders need more list entries than it was
    given?  Copies their status blocks to the host (synchronises)."""
    return any(L.read_status(b)["overflow"] for b in _compiled_binding().recent_contexts())


def last_duplicate_count(device: torch.device, P: int, W: int, H: int) -> int:
    """Duplicate count of the most recent adaptive-capacity render of this shape on `device`; KeyError when there was
    none.  Callers size fixed-capacity plans with it."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    n = _compiled_binding().get_predicted(idx, P, W, H)
    if n < 0:
        raise KeyError((P, W, H))
    return int(n)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
    st = raster_settings
    ext = _compiled_binding()
    tanfov = device_tanfov(st)
    tx, ty = (float(st.tanfovx), float(st.tanfovy)) if tanfov is None else (0.0, 0.0)
    try:
        return tuple(ext.rasterize(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                   int(st.image_height), int(st.image_width), tx, ty, st.bg,
                                   float(st.scale_modifier), st.viewmatrix, st.projmatrix, int(st.sh_degree), st.campos,
                                   CAPACITY_MODE == "speculative", CAPACITY_HEADROOM,
                                   -1 if FIXED_CAPACITY is None else FIXED_CAPACITY, bool(st.debug), tanfov))
    except Exception:
        if st.debug:  # reference behaviour with debug=True: dump the arguments, re-raise
            args = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
            torch.save(tuple(None if a is None or a.numel() == 0 else a.detach().float().cpu() for a in args),
                       "snapshot_fw.dump")
        raise


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        """bool (P): Gaussians in front of the near plane (z_view > 0.2).  Unused by ExAvatar; kept for API parity."""
        with torch.no_grad():
            p = _f32c(positions, "positions")
            view = _f32c(self.raster_settings.viewmatrix.to(p.device), "viewmatrix")
            present = torch.empty(p.shape[0], dtype=torch.uint8, device=p.device)
            L.run("b2r_mark_visible", p.device, p.shape[0], L.ptr(p), L.ptr(view), L.ptr(present))
            return present.bool()

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        raster_settings = self.raster_settings
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")
        if ((scales is None or rotations is None) and cov3D_precomp is None) or (
                (scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        empty = torch.empty(0, dtype=torch.float32, device=means3D.device)
        if shs is None:
            shs = empty
        if colors_precomp is None:
            colors_precomp = empty
        if scales is None:
            scales = empty
        if rotations is None:
            rotations = empty
        if cov3D_precomp is None:
            cov3D_precomp = empty
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                   raster_settings)


class SkinnedGaussianRasterizer(nn.Module):
    """`GaussianRasterizer` with ExAvatar's linear-blend skinning in front of it: replaces `get_transform_mat_vertex` +
    `lbs` + the camera->world transform (avatar/common/nets/module.py:413-422, 549-557) AND the rasteriser call
    (module.py:632-640) for the human Gaussians.

        color, radii, depth, alpha, posed = SkinnedGaussianRasterizer(settings)(
            xyz, skin_weights, joint_mats, trans, cam_R, cam_t, means2D, opacities, colors_precomp, scales, rotations)

    xyz (P,3) canonical positions; skin_weights (P,J) rows gathered per Gaussian (module.py:414); joint_mats (J,4,4);
    trans (3); cam_R (3,3) / cam_t (3) or None to stay in the posed frame (`is_world_coord=True`).  `posed` (P,3) is the
    world position ExAvatar's other modules read, a differentiable output.  The call is `skinning.skin_gaussians`
    followed by `GaussianRasterizer` on the posed positions: autograd adds a gradient arriving at `posed` to the
    render's own, and the skinning op's backward carries the sum to xyz, joint_mats and trans."""

    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def forward(self, xyz, skin_weights, joint_mats, trans, cam_R, cam_t, means2D, opacities, colors_precomp, scales,
                rotations):
        posed = skin_gaussians(xyz, None, skin_weights, None, joint_mats, trans, cam_R, cam_t)[0]
        color, radii, depth, alpha = GaussianRasterizer(self.raster_settings)(
            means3D=posed, means2D=means2D, opacities=opacities, colors_precomp=colors_precomp, scales=scales,
            rotations=rotations)
        return color, radii, depth, alpha, posed
