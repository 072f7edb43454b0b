"""`NeumanScores` -- the test-set scores of ExAvatar's NeuMan protocol (PSNR, SSIM, LPIPS-AlexNet) in one CUDA op that
never syncs the host.

ExAvatar's `avatar/tools/eval_neuman.py` reads back the PNGs test.py wrote (`cv2.imwrite` of `img * 255`), paints the
background white with the segmentation (`x * mask + 1 * (1 - mask)`, unless `--include_bkg`), and scores each frame with
torchmetrics' PeakSignalNoiseRatio(data_range=1), StructuralSimilarityIndexMeasure(data_range=1) and
LearnedPerceptualImagePatchSimilarity(net_type='alex') on `x * 2 - 1`, reading every score back on the host.
`NeumanScores` computes the same three scores from the renders in memory (csrc/metrics.cu): the PNG's 8-bit round trip
is restated exactly, SSIM's window sums run in fp64, and the AlexNet convolutions are TF32 implicit GEMMs on the tensor
cores -- the arithmetic torch's default cuDNN convolutions use for the reference's fp32 LPIPS.

    op = NeumanScores.from_lpips(lpips.LPIPS(net='alex').cuda())
    scores = op(render, target, mask)          # (N,3): psnr, ssim, lpips per frame

`neuman_scores_reference` and `alex_taps_reference` restate the semantics in plain torch (float64 by default) for tests
and measurements; the op never calls them.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import torch
import torch.nn.functional as F

from . import _lib as L
from .perceptual import EPS, SCALE, SHIFT, _lin_vectors, _lpips_modules

# torchvision alexnet().features[0:12]: (child index, C_in, C_out, kernel, stride, padding) of the five convs
ALEX_CONVS = ((0, 3, 64, 11, 4, 2), (3, 64, 192, 5, 1, 2), (6, 192, 384, 3, 1, 1), (8, 384, 256, 3, 1, 1),
              (10, 256, 256, 3, 1, 1))
ALEX_SLICES = ((0, 2), (2, 5), (5, 8), (8, 10), (10, 12))  # lpips' slice1..5: relu1 ... relu5
TAP_CHANNELS = (64, 192, 384, 256, 256)
MIN_SIZE = 31  # the second max pool is empty below this
SSIM_C1, SSIM_C2 = 0.01 ** 2, 0.03 ** 2
# torchmetrics' 1D SSIM window as `gaussian_window` builds it on a CUDA device (eval_neuman scores CUDA tensors), bit
# for bit; the CPU build differs by up to 8 ulps, which moves SSIM by up to ~4e-5 through the cancellation in
# E[x^2] - mu^2.  csrc/metrics.cu holds the same values.
SSIM_WINDOW = tuple(float.fromhex(v) for v in (
    "0x1.0d956p-10", "0x1.f1fdfcp-8", "0x1.26eb18p-5", "0x1.bff1p-4", "0x1.b43c4p-3", "0x1.106562p-2",
    "0x1.b43c4p-3", "0x1.bff1p-4", "0x1.26eb18p-5", "0x1.f1fdfcp-8", "0x1.0d956p-10"))


def _alex_convs(features) -> List[torch.nn.Conv2d]:
    mods = list(features)
    if len(mods) < ALEX_SLICES[-1][1]:
        raise ValueError(f"neuman: expected alexnet().features[0:12], got {len(mods)} modules")
    convs = []
    for k, (i, ci, co, ks, s, p) in enumerate(ALEX_CONVS):
        m = mods[i]
        if (not isinstance(m, torch.nn.Conv2d) or tuple(m.weight.shape) != (co, ci, ks, ks) or m.bias is None
                or m.stride != (s, s) or m.padding != (p, p) or m.dilation != (1, 1) or m.groups != 1):
            raise ValueError(f"neuman: module {i} must be a {ks}x{ks} stride-{s} padding-{p} conv {ci}->{co} with a "
                             f"bias, got {m}")
        convs.append(m)
    for i in (2, 5):
        m = mods[i]
        if not isinstance(m, torch.nn.MaxPool2d) or m.kernel_size not in (3, (3, 3)) or m.stride not in (2, (2, 2)) \
                or m.padding not in (0, (0, 0)) or m.ceil_mode:
            raise ValueError(f"neuman: module {i} must be a 3x3 stride-2 floor max pool, got {m}")
    return convs


def gaussian_window(device=None) -> torch.Tensor:
    """torchmetrics' 1D SSIM window (11 taps, sigma 1.5) in fp32: exp(-(d / 1.5)^2 / 2) over d = -5..5, divided by its
    sum, built on `device` (SSIM_WINDOW holds the CUDA build)."""
    d = torch.arange(-5.0, 6.0, 1.0, dtype=torch.float32, device=device)
    g = torch.exp(-torch.pow(d / 1.5, 2) / 2)
    return g / g.sum()


def png_round_trip(x: torch.Tensor) -> torch.Tensor:
    """fp32 `x` through `cv2.imwrite(path, x * 255)` and `cv2.imread(path) / 255.` read back as fp32: v = fl(x 255);
    u8 = 0 where v is NaN or |v| >= 2^31 (cvRound's out-of-range result saturates to 0), else clamp(rint(v), 0, 255)
    with ties to even; then u8 / 255 in double, rounded to fp32.  The identity on the 256 codes n / 255."""
    v = x.to(torch.float32) * 255
    bad = torch.isnan(v) | (v.abs() >= 2.0 ** 31)
    u8 = torch.where(bad, torch.zeros_like(v), torch.round(v).clamp(0, 255)).to(torch.uint8)  # -0 becomes 0
    return (u8.to(torch.float64) / 255.0).to(torch.float32)


def composite(q: torch.Tensor, mask: Optional[torch.Tensor]) -> torch.Tensor:
    """eval_neuman's white background in fp32: q * mask + (1 - mask), two rounded elementwise ops; None keeps q."""
    return q if mask is None else q * mask + (1 - mask)


def alex_taps_reference(x: torch.Tensor, alex_features, dtype: torch.dtype = torch.float64) -> List[torch.Tensor]:
    """relu1 ... relu5 of `x` (N,3,h,w) through the convs of `alex_features`, restated with torch.nn.functional in
    `dtype`: the conv shapes of ALEX_CONVS, ReLU after each, 3x3 stride-2 floor max pools after relu1 and relu2."""
    taps = []
    x = x.to(dtype)
    for k, (m, (_, _, _, _, s, p)) in enumerate(zip(_alex_convs(alex_features), ALEX_CONVS)):
        if k in (1, 2):
            x = F.max_pool2d(x, 3, 2)
        x = F.relu(F.conv2d(x, m.weight.to(device=x.device, dtype=dtype), m.bias.to(device=x.device, dtype=dtype),
                            stride=s, padding=p))
        taps.append(x)
    return taps


@torch.no_grad()
def neuman_scores_reference(render: torch.Tensor, target: torch.Tensor, mask: Optional[torch.Tensor], alex_features,
                            lin_weights: Sequence[torch.Tensor], dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """`NeumanScores.__call__` restated in plain torch: the round trip and the composite in fp32 (their definition),
    then PSNR, SSIM and LPIPS-AlexNet in `dtype` (float64 by default).  Device-agnostic; (N,3) in `dtype`.  SSIM's 2D
    window is the outer product of SSIM_WINDOW taken in `dtype` (torchmetrics rounds its entries to fp32), and
    only the (H-10) x (W-10) centres torchmetrics keeps are computed.  The reference the op is tested against; the
    product never calls it."""
    H, W = int(render.shape[-2]), int(render.shape[-1])
    dev = render.device
    m = None if mask is None else mask.reshape(-1, mask.shape[-3], H, W).to(torch.float32)
    x = composite(png_round_trip(render.reshape(-1, 3, H, W)), m).to(dtype)
    y = composite(png_round_trip(target.reshape(-1, 3, H, W)), m).to(dtype)
    psnr = 10 * torch.log10(1 / ((x - y) ** 2).mean((1, 2, 3)))

    g = torch.tensor(SSIM_WINDOW, dtype=dtype, device=dev)
    win = (g[:, None] * g[None, :]).expand(3, 1, 11, 11)
    f = lambda t: F.conv2d(t, win, groups=3)  # noqa: E731 -- valid centres only
    mx, my = f(x), f(y)
    vx = (f(x * x) - mx * mx).clamp_min(0)
    vy = (f(y * y) - my * my).clamp_min(0)
    cxy = f(x * y) - mx * my
    s = ((2 * mx * my + SSIM_C1) * (2 * cxy + SSIM_C2)) / ((mx * mx + my * my + SSIM_C1) * (vx + vy + SSIM_C2))
    ssim = s.mean((1, 2, 3))

    # lpips holds the ScalingLayer constants as fp32 buffers
    shift = torch.tensor(SHIFT, dtype=torch.float32).to(device=dev, dtype=dtype)[None, :, None, None]
    scale = torch.tensor(SCALE, dtype=torch.float32).to(device=dev, dtype=dtype)[None, :, None, None]

    def taps(t):
        fs = alex_taps_reference(((t * 2 - 1) - shift) / scale, alex_features, dtype)
        return [v / (torch.sqrt(torch.sum(v ** 2, dim=1, keepdim=True)) + EPS) for v in fs]

    lp = 0
    for a, b, w in zip(taps(x), taps(y), _lin_vectors(lin_weights, TAP_CHANNELS, "neuman")):
        lp = lp + (w.to(device=dev, dtype=dtype).reshape(1, -1, 1, 1) * (a - b) ** 2).sum(1).mean((1, 2))
    return torch.stack((psnr, ssim, lp), 1)


class NeumanScores:
    """eval_neuman.py's per-frame PSNR, SSIM and LPIPS-AlexNet (lpips version 0.1, eval mode) as one CUDA op.

    alex_features  torchvision-layout `alexnet().features` (at least its first 12 modules; the 5 convs are read)
    lin_weights    the five (1,C,1,1) weights of lpips's lin layers, tap order relu1 ... relu5
    device         where the op's copies of the weights live

    The weights are snapshotted once into the kernels' layouts (later changes to the modules are not seen): per conv
    (K, C_out) with rows (ky, kx, ci), conv 1's input padded to 4 channels, the rows padded with zeros to a multiple
    of 32 (include/b200raster.h B2RNeumanScores).
    """

    def __init__(self, alex_features, lin_weights: Sequence[torch.Tensor], device):
        convs = _alex_convs(alex_features)
        lins = _lin_vectors(lin_weights, TAP_CHANNELS, "neuman")
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError(f"neuman: device must be a CUDA device (got {dev}); there is no CPU fallback")
        f32 = dict(device=dev, dtype=torch.float32)
        self.w, self.bias = [], []
        for m in convs:
            w = m.weight.detach().to(**f32).permute(2, 3, 1, 0)  # (ky, kx, ci, co)
            if w.shape[2] == 3:
                w = F.pad(w, (0, 0, 0, 1))
            w = w.reshape(-1, w.shape[-1])
            self.w.append(F.pad(w, (0, 0, 0, -w.shape[0] % 32)).contiguous())
            self.bias.append(m.bias.detach().to(**f32).contiguous())
        self.lin = [t.to(**f32).contiguous() for t in lins]
        self.device = dev

    @classmethod
    def from_lpips(cls, m) -> "NeumanScores":
        """From an `lpips.LPIPS(net='alex')` instance, or the `.net` of torchmetrics'
        LearnedPerceptualImagePatchSimilarity(net_type='alex'): the convs of `m.net.slice1..5` (which keep
        torchvision's child indices) and the weights `m.lin{k}.model[-1].weight`, on the device of those weights."""
        features, lins = _lpips_modules(m, "alexnet().features", ALEX_SLICES[-1][1], "neuman")
        return cls(features, lins, lins[0].device)

    def _args(self, W, H, N, x, y, m, mc) -> L.B2RNeumanScores:
        p = L.B2RNeumanScores(width=W, height=H, n_images=N, mask_channels=mc, render=L.ptr(x), target=L.ptr(y),
                              mask=L.ptr(m))
        for k in range(5):
            p.w[k], p.bias[k], p.lin[k] = L.ptr(self.w[k]), L.ptr(self.bias[k]), L.ptr(self.lin[k])
        return p

    def __call__(self, render: torch.Tensor, target: torch.Tensor,
                 mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """eval_neuman's [psnr, ssim, lpips] of every frame, as an (N,3) fp32 CUDA tensor.

        render  (3,H,W) or (N,3,H,W) fp32 CUDA tensor, nominally in [0,1] (test.py's scene_human_img_refined_composed)
        target  the same shape: each frame's own ground truth
        mask    None (eval's --include_bkg), or (1,H,W) / (3,H,W) -- (N,1,H,W) / (N,3,H,W) with batched frames -- fp32,
                1 = human (eval's 1 - seg / 255); the background of both images is painted white with it
        H, W >= 31.

        Both images go through the PNG's 8-bit round trip first (`png_round_trip`), so a target read from an 8-bit PNG
        passes unchanged.  Identical frames give psnr +inf, ssim 1 and lpips 0.  No gradient; nothing is read back on
        the host, the call can be captured in a CUDA graph, and every reduction runs in a fixed order: two calls give
        bit-identical scores.  The caller averages the rows, as eval_neuman averages the frames.
        """
        for name, v in (("render", render), ("target", target), ("mask", mask)):
            if v is not None:
                L.cuda("neuman", name, v)
                L.float32("neuman", name, v)
        if render.dim() not in (3, 4) or render.shape[-3] != 3:
            raise ValueError(f"neuman: render must be (3,H,W) or (N,3,H,W), got {tuple(render.shape)}")
        if target.shape != render.shape:
            raise ValueError(f"neuman: target {tuple(target.shape)} does not match render {tuple(render.shape)}")
        H, W = int(render.shape[-2]), int(render.shape[-1])
        N = 1 if render.dim() == 3 else int(render.shape[0])
        if H < MIN_SIZE or W < MIN_SIZE:
            raise ValueError(f"neuman: images must be at least {MIN_SIZE}x{MIN_SIZE}, got {H}x{W}")
        mc = 0
        if mask is not None:
            mc = int(mask.shape[-3]) if mask.dim() == render.dim() else 0
            if mc not in (1, 3) or mask.shape[:-3] != render.shape[:-3] or mask.shape[-2:] != render.shape[-2:]:
                raise ValueError(f"neuman: mask must be {tuple(render.shape[:-3])} x (1 or 3,H,W) to match render "
                                 f"{tuple(render.shape)}, got {tuple(mask.shape)}")
        L.same_device("neuman", (render, target, mask), self.device)
        x = render.detach().contiguous()
        y = target.detach().contiguous()
        m = None if mask is None else mask.detach().contiguous()
        n_scratch = L.load().b2r_neuman_scratch_bytes(W, H, N)
        scratch = torch.empty(n_scratch, dtype=torch.uint8, device=self.device)
        out = torch.empty((N, 3), dtype=torch.float32, device=self.device)
        p = self._args(W, H, N, x, y, m, mc)
        L.run("b2r_neuman_scores", self.device, C.byref(p), L.ptr(out), L.ptr(scratch), n_scratch)
        return out
