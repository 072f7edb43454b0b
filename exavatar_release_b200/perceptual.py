"""`LPIPS` -- ExAvatar's LPIPS-VGG perceptual terms as one differentiable CUDA op that never syncs the host.

ExAvatar's loss block (avatar/main/model.py:199, :206) calls `nets.loss.LPIPS` (avatar/common/nets/loss.py:77-95) on
the combined render and on the refined one, each against `data['img']` with the same box.  Each call crops with
`[int(x) for x in bbox[0]]` (four device->host reads) and runs lpips.LPIPS(net='vgg') on a crop whose shape changes
every frame, so nothing after it can share a CUDA graph.  `LPIPS` computes both terms in one call
(csrc/lpips.cu): the box is read on the device, every grid is sized from the image, the target's VGG pass runs once,
and the convolutions are TF32 implicit GEMMs on the tensor cores -- the arithmetic torch's default cuDNN convolutions
already use for ExAvatar's fp32 LPIPS.

    op = LPIPS.from_lpips(lpips.LPIPS(net='vgg').cuda())
    lp = op(torch.cat((scene_human_img, scene_human_img_refined)), data['img'], bbox)   # (2,1,1,1)

`lpips_reference` restates the same semantics in plain torch (float64 by default) for tests and measurements.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from . import _lib as L
from .losses import crop_box

SHIFT = (-.030, -.088, -.188)  # lpips ScalingLayer
SCALE = (.458, .448, .450)
EPS = 1e-10                    # lpips normalize_tensor
SLICES = ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))  # torchvision vgg16().features -> relu1_2 ... relu5_3
CHANNELS = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)  # output channels of the 13 convs
TAP_CHANNELS = (64, 128, 256, 512, 512)
MIN_CROP = 16  # the fourth pool's output is empty below this


def _vgg_convs(vgg_features) -> List[torch.nn.Conv2d]:
    mods = list(vgg_features)[:SLICES[-1][1]]
    convs = [m for m in mods if isinstance(m, torch.nn.Conv2d)]
    if len(convs) != 13:
        raise ValueError(f"lpips: expected the 13 convolutions of vgg16().features[0:30], found {len(convs)}")
    for k, (m, co) in enumerate(zip(convs, CHANNELS)):
        ci = 3 if k == 0 else CHANNELS[k - 1]
        if tuple(m.weight.shape) != (co, ci, 3, 3) or m.bias is None or m.padding != (1, 1) or m.stride != (1, 1):
            raise ValueError(f"lpips: conv {k} must be a 3x3 stride-1 padding-1 conv {ci}->{co} with a bias, got {m}")
    return convs


def _lin_vectors(lin_weights: Sequence[torch.Tensor], channels: Sequence[int], prefix: str) -> List[torch.Tensor]:
    """The (1,C,1,1) weights of lpips's lin layers as C-vectors, one per tap of `channels`."""
    if len(lin_weights) != len(channels):
        raise ValueError(f"{prefix}: expected {len(channels)} lin weights, got {len(lin_weights)}")
    out = []
    for k, (w, c) in enumerate(zip(lin_weights, channels)):
        if w.numel() != c:
            raise ValueError(f"{prefix}: lin weight {k} must be (1,{c},1,1), got {tuple(w.shape)}")
        out.append(w.detach().reshape(c))
    return out


def _lpips_modules(m, features: str, n: int, prefix: str) -> Tuple[torch.nn.Sequential, List[torch.Tensor]]:
    """The first `n` modules of the backbone's `features` held by an lpips.LPIPS instance's `m.net.slice1..5` (which
    keep torchvision's child indices), and its lin weights `m.lin{k}.model[-1].weight`."""
    mods = {}
    for k in range(1, 6):
        for name, mod in getattr(m.net, f"slice{k}").named_children():
            mods[int(name)] = mod
    if sorted(mods) != list(range(n)):
        raise ValueError(f"{prefix}: m.net.slice1..5 must hold {features}[0:{n}], got indices {sorted(mods)}")
    return torch.nn.Sequential(*(mods[i] for i in range(n))), [getattr(m, f"lin{k}").model[-1].weight for k in range(5)]


def _image_shape(name: str, t: torch.Tensor, batch: bool) -> Tuple[int, int]:
    if t.dim() == 4 and not batch and t.shape[0] != 1:
        raise ValueError(f"lpips: `{name}` has batch size {t.shape[0]}; the target is one image")
    if t.dim() not in (3, 4) or t.shape[-3] != 3:
        raise ValueError(f"lpips: `{name}` must be (3,H,W) or (N,3,H,W), got {tuple(t.shape)}")
    return int(t.shape[-2]), int(t.shape[-1])


class _Lpips(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, op, target, bbox):
        lib = L.load()
        dev = img.device
        H, W = img.shape[-2:]
        x = img.detach().reshape(-1, 3, H, W).contiguous()
        N = x.shape[0]
        y = target.detach().reshape(3, H, W).contiguous()
        b = None if bbox is None else bbox.detach().reshape(4).to(torch.float32).contiguous()
        p = op._args(W, H, N, x, y, b)
        n_saved, n_scratch = lib.b2r_lpips_saved_bytes(W, H, N), lib.b2r_lpips_scratch_bytes(W, H)
        saved = torch.empty(n_saved, dtype=torch.uint8, device=dev)
        scratch = torch.empty(n_scratch, dtype=torch.uint8, device=dev)
        out = torch.empty(N, dtype=torch.float32, device=dev)
        L.run("b2r_lpips_forward", dev, C.byref(p), L.ptr(out), L.ptr(saved), n_saved, L.ptr(scratch), n_scratch)
        ctx.save_for_backward(x, y, b, saved)
        ctx.op = op
        ctx.img_shape = img.shape
        return out.reshape(N, 1, 1, 1)

    @staticmethod
    def backward(ctx, dout):
        if not ctx.needs_input_grad[0]:
            return None, None, None, None
        x, y, b, saved = ctx.saved_tensors
        dev = x.device
        N, _, H, W = x.shape
        g = dout.reshape(N).to(torch.float32).contiguous()
        dimg = torch.empty((N, 3, H, W), dtype=torch.float32, device=dev)
        n_scratch = L.load().b2r_lpips_scratch_bytes(W, H)
        scratch = torch.empty(n_scratch, dtype=torch.uint8, device=dev)
        p = ctx.op._args(W, H, N, x, y, b)
        L.run("b2r_lpips_backward", dev, C.byref(p), L.ptr(saved), saved.numel(), L.ptr(g), L.ptr(dimg), L.ptr(scratch),
              n_scratch)
        return dimg.reshape(ctx.img_shape), None, None, None


class LPIPS:
    """ExAvatar's `nets.loss.LPIPS` (lpips.LPIPS(net='vgg'), version 0.1, eval mode) as one CUDA op.

    vgg_features  torchvision-layout `vgg16().features` (at least its first 30 modules; the 13 convs are read)
    lin_weights   the five (1,C,1,1) weights of lpips's lin layers, tap order relu1_2 ... relu5_3
    device        where the op's copies of the weights live

    The weights are snapshotted once into the kernels' layouts (later changes to the modules are not seen):
    (3,3,C_in,C_out) for the forward, flipped in both taps and (3,3,C_out,C_in) for the input gradient.

    Divergence: the gradient goes to the images only.  ExAvatar's lin weights receive a `.grad` that no optimiser reads
    (its VGG weights are frozen); the op gives them none.
    """

    def __init__(self, vgg_features, lin_weights: Sequence[torch.Tensor], device):
        convs = _vgg_convs(vgg_features)
        lins = _lin_vectors(lin_weights, TAP_CHANNELS, "lpips")
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError(f"lpips: device must be a CUDA device (got {dev}); there is no CPU fallback")
        f32 = dict(device=dev, dtype=torch.float32)
        w = [m.weight.detach().to(**f32) for m in convs]
        self.w_fwd = [w[0].contiguous()] + [t.permute(2, 3, 1, 0).contiguous() for t in w[1:]]
        self.w_bwd = [t.flip(2, 3).permute(2, 3, 0, 1).contiguous() for t in w[1:]]
        self.bias = [m.bias.detach().to(**f32).contiguous() for m in convs]
        self.lin = [t.to(**f32).contiguous() for t in lins]
        self.device = dev

    @classmethod
    def from_lpips(cls, m) -> "LPIPS":
        """From an `lpips.LPIPS(net='vgg')` instance: the convs of `m.net.slice1..5` (which keep torchvision's child
        indices) and the weights `m.lin{k}.model[-1].weight`, on the device of those weights."""
        features, lins = _lpips_modules(m, "vgg16().features", SLICES[-1][1], "lpips")
        return cls(features, lins, lins[0].device)

    def _args(self, W, H, N, x, y, b) -> L.B2RLpips:
        p = L.B2RLpips(width=W, height=H, n_images=N, img=L.ptr(x), target=L.ptr(y), bbox=L.ptr(b))
        p.w_fwd[0] = L.ptr(self.w_fwd[0])
        for k in range(1, 13):
            p.w_fwd[k] = L.ptr(self.w_fwd[k])
            p.w_bwd[k] = L.ptr(self.w_bwd[k - 1])
        for k in range(13):
            p.bias[k] = L.ptr(self.bias[k])
        for k in range(5):
            p.lin[k] = L.ptr(self.lin[k])
        return p

    def __call__(self, img_out: torch.Tensor, img_target: torch.Tensor,
                 bbox: Optional[torch.Tensor] = None) -> torch.Tensor:
        """ExAvatar's `LPIPS(img_out[n:n+1], img_target, bbox)` for every image n, as an (N,1,1,1) fp32 tensor.

        img_out     (3,H,W) or (N,3,H,W) fp32 CUDA tensor; N = 2 is ExAvatar's pair of renders
        img_target  (3,H,W) or (1,3,H,W): one target for all N (its VGG pass runs once per call)
        bbox        CUDA float tensor (4,) or (1,4): xmin, ymin, width, height, read ON THE DEVICE by `l1_ssim`'s crop
                    rules (`losses.crop_box`).  None: the whole image.  H, W >= 16.

        Gradients reach `img_out` only: exactly zero outside the crop.  `img_target` requiring grad raises ValueError.
        A crop narrower or shorter than 16 px returns NaN and a zero gradient (the reference raises there: its fourth
        pool is empty; raising would need a host sync).  A tapped pixel whose channels are all 0 has a NaN gradient at
        the head, as torch's autograd through sqrt(0) has; the ReLU below it drops it, as in torch.

        Neither forward nor backward synchronises with the host, both can be captured in a CUDA graph (a replay may
        carry a box of another size), and every reduction runs in a fixed order: two runs give bit-identical results.
        """
        for name, v in (("img_out", img_out), ("img_target", img_target), ("bbox", bbox)):
            if v is not None:
                L.cuda("lpips", name, v)
        H, W = _image_shape("img_out", img_out, True)
        if _image_shape("img_target", img_target, False) != (H, W):
            raise ValueError(f"lpips: img_target {tuple(img_target.shape)} does not match img_out "
                             f"{tuple(img_out.shape)}")
        if H < MIN_CROP or W < MIN_CROP:
            raise ValueError(f"lpips: images must be at least {MIN_CROP}x{MIN_CROP}, got {H}x{W}")
        for name, v in (("img_out", img_out), ("img_target", img_target)):
            L.float32("lpips", name, v)
        if bbox is not None and (tuple(bbox.shape) not in ((4,), (1, 4)) or not bbox.is_floating_point()):
            raise ValueError(f"lpips: bbox must be a float tensor of shape (4,) or (1,4), got {bbox.dtype} "
                             f"{tuple(bbox.shape)}")
        if img_target.requires_grad:
            raise ValueError("lpips: `img_target` requires grad, but the op returns a gradient for `img_out` only")
        L.same_device("lpips", (img_out, img_target, bbox), self.device)
        return _Lpips.apply(img_out, self, img_target, bbox)


def vgg_taps_reference(x: torch.Tensor, vgg_features, dtype: torch.dtype = torch.float64) -> List[torch.Tensor]:
    """relu1_2, relu2_2, relu3_3, relu4_3, relu5_3 of `x` (N,3,h,w) through the 13 convs of `vgg_features`, restated
    with torch.nn.functional in `dtype`: 3x3 convs with zero padding 1, ReLU, 2x2 stride-2 floor max pools."""
    convs = iter(_vgg_convs(vgg_features))
    taps = []
    x = x.to(dtype)
    for t, (a, b) in enumerate(SLICES):
        if t > 0:
            x = F.max_pool2d(x, 2, 2)
        for _ in range((b - a - (1 if t > 0 else 0)) // 2):
            m = next(convs)
            x = F.relu(F.conv2d(x, m.weight.to(device=x.device, dtype=dtype), m.bias.to(device=x.device, dtype=dtype),
                                padding=1))
        taps.append(x)
    return taps


def lpips_reference(img_out: torch.Tensor, img_target: torch.Tensor, bbox: Optional[torch.Tensor], vgg_features,
                    lin_weights: Sequence[torch.Tensor], dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """`LPIPS.__call__` restated in plain torch in `dtype` (float64 by default); device-agnostic and differentiable
    (the target too).  Reads `bbox` on the host.  Raises where the reference does: a crop under 16 px.  The reference
    the op is tested against; the product never calls it."""
    H, W = int(img_out.shape[-2]), int(img_out.shape[-1])
    x0, y0, x1, y1 = crop_box(bbox, W, H)
    dev = img_out.device
    # lpips holds the ScalingLayer constants as fp32 buffers
    shift = torch.tensor(SHIFT, dtype=torch.float32).to(device=dev, dtype=dtype)[None, :, None, None]
    scale = torch.tensor(SCALE, dtype=torch.float32).to(device=dev, dtype=dtype)[None, :, None, None]

    def taps(t):
        t = t.reshape(-1, 3, H, W)[:, :, y0:y1, x0:x1].to(dtype) * 2 - 1
        fs = vgg_taps_reference((t - shift) / scale, vgg_features, dtype)
        return [f / (torch.sqrt(torch.sum(f ** 2, dim=1, keepdim=True)) + EPS) for f in fs]

    fa, fb = taps(img_out), taps(img_target)
    val = 0
    for a, b, w in zip(fa, fb, _lin_vectors(lin_weights, TAP_CHANNELS, "lpips")):
        lin = F.conv2d((a - b) ** 2, w.to(device=dev, dtype=dtype).reshape(1, -1, 1, 1))
        val = val + lin.mean([2, 3], keepdim=True)
    return val
