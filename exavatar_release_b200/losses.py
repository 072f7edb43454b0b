"""`l1_ssim` -- ExAvatar's photometric L1 + SSIM terms as one differentiable CUDA op that never syncs the host.

ExAvatar's loss block (avatar/main/model.py:196-215) calls `RGBLoss` six times and `SSIM` three times per frame
(avatar/common/nets/loss.py:11-74).  Each call with a box crops with `[int(x) for x in bbox[0]]`, four device->host
reads of a CUDA tensor, and each SSIM rebuilds its window and runs five grouped 11x11 convolutions.  `l1_ssim` returns
`(RGBLoss(...).mean(), SSIM(...).mean())` from two kernels forward and one backward (csrc/l1ssim.cu), reading the box
on the device, so the block can run behind the renderer without draining the stream and can be captured in a graph.

    l1, s = l1_ssim(scene_human_img, gt, bbox)             # rgb_human 0.8 * l1, ssim_human 0.2 * (1 - s)
    l1, s = l1_ssim(scene_img, gt, mask=1 - data['mask'])  # rgb_scene, ssim_scene
    l1, _ = l1_ssim(face_composite(scene_human_img, face), gt, bbox, ssim=False)  # rgb_face (compose.face_composite)
    l1, _ = l1_ssim(human_img, composite_target, bbox, ssim=False)  # rgb_human_rand_bg

`l1_ssim_reference` restates the same semantics in plain torch (float64 by default) for tests and measurements.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from . import _lib as L

C1 = 0.01 ** 2
C2 = 0.03 ** 2
WINDOW = 11
SIGMA = 1.5


def ssim_window() -> torch.Tensor:
    """The 11 fp32 taps of the SSIM window: exp(-(x - 5)^2 / (2 sigma^2)) rounded to fp32, over their fp32 sum (the
    values csrc/l1ssim.cu holds as constants)."""
    g = torch.tensor([math.exp(-(x - WINDOW // 2) ** 2 / float(2 * SIGMA ** 2)) for x in range(WINDOW)],
                     dtype=torch.float32)
    return g / g.sum()


def crop_box(bbox: Optional[torch.Tensor], W: int, H: int) -> Tuple[int, int, int, int]:
    """(x0, y0, x1, y1) of the crop [y0:y1, x0:x1] by the reference's integer rules: int() truncates, the clamped start
    is added to the width (a box with negative xmin moves right), the end is clamped to the image.  Reads `bbox` on the
    host; the op evaluates the same rules on the device."""
    if bbox is None:
        return 0, 0, W, H
    xmin, ymin, width, height = (int(v) for v in bbox.reshape(-1).tolist())
    x0, y0 = max(xmin, 0), max(ymin, 0)
    return x0, y0, max(min(x0 + width, W), x0), max(min(y0 + height, H), y0)


def _image_shape(name: str, t: torch.Tensor) -> Tuple[int, int]:
    if t.dim() == 4 and t.shape[0] != 1:
        raise ValueError(f"l1_ssim: `{name}` has batch size {t.shape[0]}; ExAvatar trains with one image per GPU and "
                         "only a batch of 1 is supported")
    if t.dim() not in (3, 4) or t.shape[-3] != 3:
        raise ValueError(f"l1_ssim: `{name}` must be (3,H,W) or (1,3,H,W), got {tuple(t.shape)}")
    return int(t.shape[-2]), int(t.shape[-1])


class _L1Ssim(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, target, bbox, mask, with_ssim):
        dev = img.device
        H, W = img.shape[-2:]
        x = img.detach().reshape(3, H, W).contiguous()
        y = target.detach().reshape(3, H, W).contiguous()
        m = None if mask is None else mask.detach().reshape(H, W).contiguous()
        b = None if bbox is None else bbox.detach().reshape(4).to(torch.float32).contiguous()
        nbytes = L.load().b2r_l1ssim_scratch_bytes(W, H)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty(2, dtype=torch.float32, device=dev)  # out[1] is written (and returned) only with SSIM
        L.run("b2r_l1ssim_forward", dev, W, H, L.ptr(x), L.ptr(y), L.ptr(m), L.ptr(b), int(with_ssim), L.ptr(out),
              L.ptr(scratch), nbytes)
        ctx.save_for_backward(x, y, m, b, scratch)
        ctx.with_ssim = with_ssim
        ctx.img_shape = img.shape
        return out

    @staticmethod
    def backward(ctx, dout):
        if not ctx.needs_input_grad[0]:
            return None, None, None, None, None
        x, y, m, b, scratch = ctx.saved_tensors
        dev = x.device
        H, W = x.shape[-2:]
        g = dout.to(torch.float32).contiguous()
        dimg = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        L.run("b2r_l1ssim_backward", dev, W, H, L.ptr(x), L.ptr(y), L.ptr(m), L.ptr(b), int(ctx.with_ssim), L.ptr(g),
              L.ptr(dimg), L.ptr(scratch), scratch.numel())
        return dimg.reshape(ctx.img_shape), None, None, None, None


def l1_ssim(img: torch.Tensor, target: torch.Tensor, bbox: Optional[torch.Tensor] = None,
            mask: Optional[torch.Tensor] = None, ssim: bool = True) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """ExAvatar's `RGBLoss(img, target, bbox).mean()` and `SSIM(img, target, bbox, mask).mean()` as two 0-dim tensors.

    img, target  (3,H,W) or (1,3,H,W) fp32 CUDA tensors; only a batch of 1.
    bbox         CUDA float tensor (4,) or (1,4): xmin, ymin, width, height, read ON THE DEVICE.  The crop is
                 [y0:y1, x0:x1] with x0 = max(trunc(xmin), 0), x1 = min(x0 + trunc(width), W) (the clamped x0: a box
                 with negative xmin moves right rather than being clipped), likewise for y.  None: the whole image.
    mask         (H,W), (1,H,W) or (1,1,H,W), values >= 0, multiplies BOTH images before anything else (as
                 `SSIM(mask=)`); for m >= 0 the L1 of the masked images is also `RGBLoss(...) * m` averaged.
    ssim         False skips the SSIM kernels and returns (l1, None).

    SSIM: 11-tap Gaussian window (sigma 1.5, fp32 taps) applied to the crop with zero padding 5 at the CROP's border,
    C1 = 0.01^2, C2 = 0.03^2, sigma^2 = E[x^2] - mu^2, the map averaged over 3 h w; the L1 is mean |x - y| over the same
    crop.  Gradients reach `img` only (exactly zero outside the crop and where mask = 0); `target` or `mask` requiring
    grad raises ValueError rather than dropping that gradient.

    An empty crop returns NaN for both means and a zero gradient.  (The reference disagrees with itself there:
    `RGBLoss(...).mean()` is NaN, while `SSIM` raises inside F.conv2d because the 10-pixel padded input is smaller than
    the window.  Any crop of one pixel or more is valid in both.)

    Neither forward nor backward synchronises with the host, both can be captured in a CUDA graph, and the reductions
    run in a fixed order: two runs give bit-identical results.  CUDA tensors only: there is no CPU fallback.
    """
    for name, v in (("img", img), ("target", target), ("bbox", bbox), ("mask", mask)):
        if v is not None:
            L.cuda("l1_ssim", name, v)
    H, W = _image_shape("img", img)
    if _image_shape("target", target) != (H, W):
        raise ValueError(f"l1_ssim: target {tuple(target.shape)} does not match img {tuple(img.shape)}")
    for name, v in (("img", img), ("target", target), ("mask", mask)):
        if v is not None:
            L.float32("l1_ssim", name, v)
    if mask is not None and (mask.dim() not in (2, 3, 4) or tuple(mask.shape[-2:]) != (H, W) or mask.numel() != H * W):
        raise ValueError(f"l1_ssim: mask must be (H,W), (1,H,W) or (1,1,H,W) with H,W = {H},{W}, "
                         f"got {tuple(mask.shape)}")
    if bbox is not None and (tuple(bbox.shape) not in ((4,), (1, 4)) or not bbox.is_floating_point()):
        raise ValueError(f"l1_ssim: bbox must be a float tensor of shape (4,) or (1,4), got {bbox.dtype} "
                         f"{tuple(bbox.shape)}")
    for name, v in (("target", target), ("mask", mask)):
        if v is not None and v.requires_grad:
            raise ValueError(f"l1_ssim: `{name}` requires grad, but the op returns a gradient for `img` only")
    L.same_device("l1_ssim", (img, target, bbox, mask))
    out = _L1Ssim.apply(img, target, bbox, mask, bool(ssim))
    return (out[0], out[1]) if ssim else (out[0], None)


def l1_ssim_reference(img: torch.Tensor, target: torch.Tensor, bbox: Optional[torch.Tensor] = None,
                      mask: Optional[torch.Tensor] = None, ssim: bool = True, dtype: torch.dtype = torch.float64
                      ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """`l1_ssim` restated in plain torch from its formulas, computed in `dtype` (float64 by default); device-agnostic
    and differentiable.  Reads `bbox` on the host.  The reference the op is tested against; the product never calls it.
    An empty crop gives NaN for both means (the SSIM term without evaluating the window)."""
    H, W = int(img.shape[-2]), int(img.shape[-1])
    x = img.reshape(1, 3, H, W).to(dtype)
    y = target.reshape(1, 3, H, W).to(dtype)
    if mask is not None:
        m = mask.reshape(1, 1, H, W).to(dtype)
        x, y = x * m, y * m
    x0, y0, x1, y1 = crop_box(bbox, W, H)
    x, y = x[:, :, y0:y1, x0:x1], y[:, :, y0:y1, x0:x1]
    l1 = (x - y).abs().mean()
    if not ssim:
        return l1, None
    if x.numel() == 0:
        return l1, torch.full((), float("nan"), dtype=dtype, device=img.device)
    w = ssim_window().to(device=img.device, dtype=dtype)
    win = (w[:, None] * w[None, :]).expand(3, 1, WINDOW, WINDOW)
    conv = lambda t: F.conv2d(t, win, padding=WINDOW // 2, groups=3)  # noqa: E731
    mx, my = conv(x), conv(y)
    sxx, syy, sxy = conv(x * x) - mx * mx, conv(y * y) - my * my, conv(x * y) - mx * my
    smap = ((2 * mx * my + C1) * (2 * sxy + C2)) / ((mx * mx + my * my + C1) * (sxx + syy + C2))
    return l1, smap.mean()
