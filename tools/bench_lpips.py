"""ExAvatar's LPIPS-VGG terms (avatar/main/model.py:199, :206) the way ExAvatar runs them vs. `perceptual.LPIPS`.

  python tools/bench_lpips.py [--iters 10] [--rounds 5] [--frames 10] [--json out.json]

C4 size (512 x 512, a box of 60 % of the image as tools/bench_l1_ssim.py uses), forward + backward of both terms per
frame, with the weights of tests/golden/make_lpips_golden.py (the real VGG weights need a download; the cost does not
depend on their values).  Arms:
  1. exavatar:  two calls of nets.loss.LPIPS restated -- crop by int() of the box (four device->host reads each), x*2-1,
                lpips's ScalingLayer and torchvision's vgg16().features on cuDNN with torch's default TF32 convolutions,
                the render and the target through VGG in each call -- and one backward;
  2. op:        `LPIPS` on the pair (N = 2, one target pass), eager;
  3. op_graph:  arm 2 captured once in a CUDA graph and replayed;
  4. frame_*:   C4 training frames/s of tools/c4_frame.py's frame (rig op, networks, skinning, the five renders,
                l1_ssim, regularisers) with 0.2 x the two LPIPS terms of scene_human / scene_human_refined added: none,
                arm 1's form, or the op.
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Per-kernel
device time per call comes from a separate torch.profiler run, and achieved TFLOP/s from the FLOPs of the layer shapes
(2 x MACs; a backward counts the input gradient only, the same MACs as the forward minus conv1_1's, which neither side's
backward runs as a GEMM) over that device time, against the 495 TFLOP/s dense TF32 data-sheet figure.  Prints the card
name and power limit with the numbers.
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, graph_replay, host_syncs, kernel_events, stats  # noqa: E402
from c4_frame import BOX, FrameArm, frames_per_second  # noqa: E402
from exavatar_release_b200.perceptual import LPIPS, SCALE, SHIFT, SLICES  # noqa: E402

H = W = 512
TF32_PEAK = 495e12


def vgg_macs(h, w):
    """(forward MACs through relu5_3, conv1_1's share) of one image of h x w."""
    chans = [(3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512),
             (512, 512), (512, 512), (512, 512), (512, 512)]
    level = (0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4)
    macs = [9 * ci * co * (h >> lv) * (w >> lv) for (ci, co), lv in zip(chans, level)]
    return sum(macs), macs[0]


class ExAvatarLpips(torch.nn.Module):
    """nets.loss.LPIPS over lpips.LPIPS(net='vgg'): the crop by int(), then lpips's forward on cuDNN."""

    def __init__(self, features, lins, dev):
        super().__init__()
        # lpips freezes the VGG weights; its lin weights take a gradient (no optimiser reads it)
        self.features = features.to(dev).eval().requires_grad_(False)
        self.lins = [w.to(dev).requires_grad_() for w in lins]
        self.shift = torch.tensor(SHIFT, device=dev)[None, :, None, None]
        self.scale = torch.tensor(SCALE, device=dev)[None, :, None, None]

    def taps(self, x):
        out = []
        for a, b in SLICES:
            x = self.features[a:b](x)
            out.append(x)
        return out

    def forward(self, img_out, img_target, bbox):
        img_h, img_w = img_out.shape[-2:]
        xmin, ymin, width, height = [int(x) for x in bbox[0]]
        xmin, ymin = max(xmin, 0), max(ymin, 0)
        xmax, ymax = min(xmin + width, img_w), min(ymin + height, img_h)
        a = img_out[:, :, ymin:ymax, xmin:xmax] * 2 - 1
        b = img_target[:, :, ymin:ymax, xmin:xmax] * 2 - 1
        fa, fb = self.taps((a - self.shift) / self.scale), self.taps((b - self.shift) / self.scale)
        val = 0
        for x, y, w in zip(fa, fb, self.lins):
            x = x / (torch.sqrt(torch.sum(x ** 2, dim=1, keepdim=True)) + 1e-10)
            y = y / (torch.sqrt(torch.sum(y ** 2, dim=1, keepdim=True)) + 1e-10)
            val = val + F.conv2d((x - y) ** 2, w).mean([2, 3], keepdim=True)
        return val


def main():
    a = arg_parser(__doc__, iters=10, frames=10).parse_args()
    dev = cuda_device("bench_lpips")
    from make_lpips_golden import lpips_weights
    feats, lins = lpips_weights()
    op = LPIPS(feats, lins, dev)
    ref = ExAvatarLpips(feats, lins, dev)
    g = torch.Generator().manual_seed(21)
    base = F.interpolate(torch.rand(1, 3, 32, 32, generator=g), size=(H, W), mode="bilinear")[0]
    pair = torch.stack([(base + 0.05 * torch.randn(3, H, W, generator=g)).clamp(0, 1) for _ in range(2)]).to(dev)
    gt = base.to(dev)
    bbox = torch.tensor([BOX], device=dev)

    def run_exavatar(x=None):
        x = pair.clone().requires_grad_() if x is None else x
        for w in ref.lins:
            w.grad = None
        loss = 0.2 * ref(x[0:1], gt[None], bbox) + 0.2 * ref(x[1:2], gt[None], bbox)
        loss.sum().backward()
        return x

    def run_op(x=None):
        x = pair.clone().requires_grad_() if x is None else x
        (0.2 * op(x, gt, bbox)).sum().backward()
        return x

    xe, xo = run_exavatar(), run_op()
    torch.cuda.synchronize()
    agree = {"grad_max_abs_diff": float((xe.grad - xo.grad).abs().max()), "grad_max_abs": float(xe.grad.abs().max())}

    xg = pair.clone().requires_grad_()

    def run_op_xg():
        xg.grad = None
        run_op(xg)

    arms = {"exavatar": run_exavatar, "op": run_op, "op_graph": graph_replay(run_op_xg, 2)}
    times = alternate(arms, a.iters, a.rounds, 1)
    syncs = {k: host_syncs(arms[k]) for k in ("exavatar", "op")}

    x0, y0 = int(BOX[0]), int(BOX[1])
    cw, ch = min(x0 + int(BOX[2]), W) - x0, min(y0 + int(BOX[3]), H) - y0
    fwd, c11 = vgg_macs(ch, cw)
    flops = {"exavatar": 2 * (4 * fwd + 2 * (fwd - c11)), "op": 2 * (3 * fwd + 2 * (fwd - c11))}
    flops["op_graph"] = flops["op"]
    prof = {}
    for k, fn in arms.items():
        ev, prof[k] = kernel_events(fn)
        per = {}
        for e in ev:
            n = e.name if len(e.name) <= 90 else e.name[:87] + "..."
            per.setdefault(n, [0.0, 0])
            per[n][0] += e.device_time / 1e3
            per[n][1] += 1
        dms = prof[k]["device_ms"]
        prof[k].update(tflops=flops[k] / (dms * 1e-3) / 1e12, share_of_tf32_peak=flops[k] / (dms * 1e-3) / TF32_PEAK,
                       kernels_ms={n: round(v[0], 4) for n, v in sorted(per.items(), key=lambda kv: -kv[1][0])[:12]})

    def lp_exavatar(o, target):
        return sum(0.2 * ref(o[r]["img"][None], target[None], bbox).sum()
                   for r in ("scene_human", "scene_human_refined"))

    def lp_op(o, target):
        return 0.2 * op(torch.stack((o["scene_human"]["img"], o["scene_human_refined"]["img"])), target, bbox).sum()

    frames = frames_per_second(a, dev, {"lpips_none": FrameArm(loss=lambda o, t: 0.0),
                                        "lpips_exavatar": FrameArm(loss=lp_exavatar), "lpips_op": FrameArm(loss=lp_op)})
    res = {"card": card(), "size": [H, W], "crop": [ch, cw], "gflop_per_frame": {k: v / 1e9 for k, v in flops.items()},
           "lpips_ms": {k: stats(v, 1e3) for k, v in times.items()},
           "host_syncs_per_call": syncs, "profile": prof, "exavatar_vs_op": agree, "frames_per_s": frames}
    emit(res, a.json)


if __name__ == "__main__":
    main()
