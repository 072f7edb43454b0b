"""Generates tests/golden/loss.npz from the original ExAvatar_RELEASE's own loss classes.

    python tests/golden/make_loss_golden.py /path/to/ExAvatar_RELEASE

`RGBLoss` and `SSIM` (avatar/common/nets/loss.py:11-74) are executed verbatim, class sources only: the module itself
imports lpips and pytorch3d.  `.cuda()` is patched to the identity.  The cases are the boxes, mask and
random-background target of avatar/main/model.py:196-215 on a 512x512 and a 136x200 image pair.  Each case stores both
means, and the gradient of the weighted loss with respect to the image at a seeded sample of elements plus its
abs-sum and non-zero count; each image pair stores the sums of its pixels.

The images are not stored.  `loss_images` builds them from integer arithmetic only (a hashed coarse grid, bilinearly
interpolated, plus hashed noise, and a soft elliptic mask), so the tests rebuild the same uint8 pixels on any machine
and the fixture stays a few tens of kilobytes.
"""
import ast
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))

# (name, image pair, bbox or None, term): "l1_ssim" = rgb + ssim with a box (rgb_human, ssim_human), "l1" = rgb alone
# (rgb_face), "rand_bg" = rgb with the target composited over a random background through the mask
# (rgb_human_rand_bg), "scene" = rgb * (1 - mask) and ssim with mask = 1 - mask, no box (rgb_scene, ssim_scene)
LOSS_CASES = [
    ("neg_xy", "big", (-20.7, -8.3, 300.9, 280.4), "l1_ssim"),      # negative xmin / ymin: shifted, not clipped
    ("past_edge", "big", (400.5, 380.2, 200.0, 250.0), "l1_ssim"),  # past the right and bottom edges
    ("c4_box", "big", (102.4, 60.8, 307.5, 396.2), "l1_ssim"),      # ~60 % of the image
    ("frac", "small", (13.6, 7.9, 150.3, 101.8), "l1_ssim"),        # fractional coordinates
    ("narrow", "small", (50.2, 40.9, 7.5, 60.3), "l1_ssim"),        # 7 px wide: narrower than the 11-tap window
    ("one_px", "small", (30.0, 20.0, 1.9, 1.2), "l1_ssim"),         # a single pixel
    ("face_l1", "big", (102.4, 60.8, 307.5, 396.2), "l1"),
    ("rand_bg", "small", (10.2, 5.5, 120.7, 90.1), "rand_bg"),
    ("scene", "big", None, "scene"),
]
SIZES = {"big": (512, 512), "small": (136, 200)}
BG = (0.25, 0.6, 0.85)  # the random background of the rand_bg case
SAMPLES = 256           # gradient elements stored per case: this many non-zero ones plus this many anywhere

_M32 = 0xFFFFFFFF


def _hash(*keys):
    """32-bit integer hash of broadcastable int64 tensors: every intermediate stays below 2**63, so it is exact."""
    h = torch.zeros((), dtype=torch.int64)
    for k, p in zip(keys, (0x9E3779B1, 0x85EBCA77, 0xC2B2AE3D)):
        h = (h ^ ((k * p) & _M32)) & _M32
        h = ((h ^ (h >> 15)) * 0x5BD1E995) & _M32
    return h ^ (h >> 13)


def loss_images(H, W):
    """(img, target, mask) as uint8 tensors (3,H,W), (3,H,W), (1,H,W), from integer arithmetic only."""
    y = torch.arange(H, dtype=torch.int64)[None, :, None]
    x = torch.arange(W, dtype=torch.int64)[None, None, :]
    c = torch.arange(3, dtype=torch.int64)[:, None, None]
    gy, fy, gx, fx = y // 8, y % 8, x // 8, x % 8
    v = lambda i, j: _hash(i, j, c) & 255  # noqa: E731  -- a random value every 8 pixels
    target = ((8 - fx) * (8 - fy) * v(gy, gx) + fx * (8 - fy) * v(gy, gx + 1) + (8 - fx) * fy * v(gy + 1, gx)
              + fx * fy * v(gy + 1, gx + 1)) // 64
    img = (target + _hash(y, x, c + 7) % 41 - 20).clamp(0, 255)
    # 1.5 - 2 ((x/a)^2 + (y/1.3b)^2) on [-1,1]^2, clamped to [0,1]: 1 inside, a soft edge, 0 in the corners
    dx, dy = 2 * x[0] - (W - 1), 2 * y[0] - (H - 1)
    num = 169 * dx * dx * H * H + 100 * dy * dy * W * W
    den = 169 * W * W * H * H
    mask = ((3 * den - 4 * num) * 255 // (2 * den)).clamp(0, 255)
    return img.to(torch.uint8), target.to(torch.uint8), mask[None].to(torch.uint8)


def load_loss_classes(ref_root):
    torch.Tensor.cuda = lambda self, *a, **k: self
    path = os.path.join(ref_root, "avatar", "common", "nets", "loss.py")
    src = open(path).read()
    ns = {"torch": torch, "nn": torch.nn, "F": torch.nn.functional, "math": math, "np": np}
    for cls in (n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name in ("RGBLoss", "SSIM")):
        exec(compile(ast.get_source_segment(src, cls), path, "exec"), ns)
    return ns["RGBLoss"](), ns["SSIM"]()


def main(ref_root):
    rgb_loss, ssim = load_loss_classes(ref_root)
    g = torch.Generator().manual_seed(11)
    pairs = {k: loss_images(*hw) for k, hw in SIZES.items()}
    bg = torch.tensor(BG)
    out = {f"{k}_pixel_sums": np.array([int(t.long().sum()) for t in v], np.int64) for k, v in pairs.items()}
    for name, key, box, term in LOSS_CASES:
        img8, tgt8, m8 = pairs[key]
        x = (img8.float() / 255)[None].requires_grad_()
        y = (tgt8.float() / 255)[None]
        m = (m8.float() / 255)[None]
        bbox = None if box is None else torch.tensor([box], dtype=torch.float32)
        s = torch.tensor(float("nan"))
        if term == "scene":
            l1 = (rgb_loss(x, y) * (1 - m)).mean()
            s = ssim(x, y, mask=1 - m).mean()
        elif term == "rand_bg":
            l1 = rgb_loss(x, y, bbox=bbox, mask=m, bg=bg[None]).mean()
        else:
            l1 = rgb_loss(x, y, bbox=bbox).mean()
            if term == "l1_ssim":
                s = ssim(x, y, bbox=bbox).mean()
        loss = 0.8 * l1 + 0.2 * (1 - s) if term in ("l1_ssim", "scene") else l1
        loss.backward()
        grad = x.grad[0].reshape(-1)
        nz = torch.nonzero(grad).reshape(-1)
        idx = torch.cat((nz[torch.randperm(nz.numel(), generator=g)[:SAMPLES]],
                         torch.randperm(grad.numel(), generator=g)[:SAMPLES])).unique()
        out.update({f"{name}_l1": l1.detach().numpy(), f"{name}_ssim": s.detach().numpy(),
                    f"{name}_grad_idx": idx.numpy().astype(np.int32), f"{name}_grad_val": grad[idx].numpy(),
                    f"{name}_grad_abs_sum": grad.abs().sum().numpy(), f"{name}_grad_nonzero": np.array(nz.numel())})
    np.savez_compressed(os.path.join(HERE, "loss.npz"), **out)
    print("wrote loss.npz")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
