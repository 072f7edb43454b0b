"""ExAvatar's NeuMan test-set scores (avatar/tools/eval_neuman.py) the way the script computes them vs. `NeumanScores`.

  python tools/bench_neuman_scores.py [--iters 10] [--rounds 5] [--json out.json]

One frame (N = 1) at 512 x 512 and at 1080 x 1920, with a 1-channel mask, AlexNet weights from a seed (the pretrained
weights need a download; the cost does not depend on their values).  Arms:
  1. eval:      eval_neuman's scoring restated in torch from the images in memory (no PNG files): the white-background
                composite, PSNR, torchmetrics' SSIM (reflect pad, depthwise F.conv2d of the 11x11 window) and
                torchvision's AlexNet plus the lin heads on cuDNN with torch's default TF32 convolutions, each score
                read back on the host as the script does;
  2. op:        `NeumanScores`, eager;
  3. op_graph:  arm 2 captured once in a CUDA graph and replayed.
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Per-kernel
device time comes from a separate torch.profiler run, and the trunk's achieved TF32 TFLOP/s from the FLOPs of the layer
shapes (2 x MACs of both images' five convs) over the conv kernels' device time, against the 495 TFLOP/s dense TF32
data-sheet figure.  Prints the card name and power limit with the numbers.
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, graph_replay, host_syncs, kernel_events, stats  # noqa: E402
from exavatar_release_b200.metrics import ALEX_CONVS, ALEX_SLICES, NeumanScores, gaussian_window  # noqa: E402
from exavatar_release_b200.perceptual import SCALE, SHIFT  # noqa: E402

SIZES = ((512, 512), (1080, 1920))
TF32_PEAK = 495e12


def trunk_flops(h, w):
    """2 x MACs of the five AlexNet convs of one h x w image."""
    flops = 0
    for k, (_, ci, co, ks, s, p) in enumerate(ALEX_CONVS):
        if k in (1, 2):
            h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
        h, w = (h + 2 * p - ks) // s + 1, (w + 2 * p - ks) // s + 1
        flops += 2 * h * w * co * ci * ks * ks
    return flops


class EvalScores:
    """eval_neuman.py's scoring of one frame in torch: torchmetrics' PSNR / SSIM and lpips' AlexNet LPIPS."""

    def __init__(self, feats, lins, dev):
        self.feats = feats.to(dev).eval().requires_grad_(False)
        self.lins = [w.to(dev) for w in lins]
        self.shift = torch.tensor(SHIFT, device=dev)[None, :, None, None]
        self.scale = torch.tensor(SCALE, device=dev)[None, :, None, None]
        g = gaussian_window(dev)
        self.win = (g[:, None] @ g[None, :]).expand(3, 1, 11, 11).contiguous()

    def ssim(self, x, y):
        xs = F.pad(torch.cat((x, y, x * x, y * y, x * y)), (5, 5, 5, 5), mode="reflect")
        o = F.conv2d(xs, self.win, groups=3)
        mx, my, exx, eyy, exy = o.split(x.shape[0])
        vx, vy, cxy = (exx - mx * mx).clamp_min(0), (eyy - my * my).clamp_min(0), exy - mx * my
        s = ((2 * mx * my + 0.01 ** 2) * (2 * cxy + 0.03 ** 2)) / ((mx * mx + my * my + 0.01 ** 2) * (vx + vy + 0.03 ** 2))
        return s[..., 5:-5, 5:-5].mean()

    def lpips(self, x, y):
        h = (torch.cat((x, y)) * 2 - 1 - self.shift) / self.scale
        val = 0
        for (a, b), w in zip(ALEX_SLICES, self.lins):
            h = self.feats[a:b](h)
            n = h / (torch.sqrt((h * h).sum(1, keepdim=True)) + 1e-10)
            val = val + F.conv2d((n[:1] - n[1:]) ** 2, w).mean()
        return val

    def __call__(self, render, target, mask):
        with torch.no_grad():
            x, y = render * mask + (1 - mask), target * mask + (1 - mask)
            psnr = 10 * torch.log10(1 / ((x - y) ** 2).mean())
            return [float(psnr), float(self.ssim(x, y)), float(self.lpips(x, y))]  # the script's host reads


def main():
    args = arg_parser(__doc__, iters=10).parse_args()
    dev = cuda_device("bench_neuman_scores")
    torch.backends.cudnn.benchmark = False
    torch.manual_seed(0)
    import torchvision
    feats = torchvision.models.alexnet(weights=None).features
    lins = [torch.rand(1, c, 1, 1) * 0.2 for c in (64, 192, 384, 256, 256)]
    op = NeumanScores(feats, lins, dev)
    ev = EvalScores(feats, lins, dev)
    result = {"card": card(), "sizes": {}}
    for H, W in SIZES:
        g = torch.Generator(device=dev).manual_seed(H)
        render = torch.rand(1, 3, H, W, device=dev, generator=g)
        target = (torch.rand(1, 3, H, W, device=dev, generator=g) * 255).round() / 255
        mask = (torch.rand(1, 1, H, W, device=dev, generator=g) > 0.3).float()
        rq = (render * 255).round().clamp(0, 255) / 255  # eval reads back the PNG test.py wrote
        arms = {"eval": lambda: ev(rq, target, mask), "op": lambda: op(render, target, mask),
                "op_graph": graph_replay(lambda: op(render, target, mask), 3)}
        times = alternate(arms, args.iters, args.rounds, warmup=3)
        ref = ev(rq, target, mask)
        got = op(render, target, mask)[0].tolist()
        ev_k, ev_sum = kernel_events(lambda: ev(rq, target, mask))
        op_k, op_sum = kernel_events(lambda: op(render, target, mask))
        per = {}
        for e in op_k:
            per.setdefault(e.name.split("(")[0].replace("void ", "").replace("b2r::", ""), []).append(e.device_time)
        conv_ms = sum(sum(v) for k, v in per.items() if "nm_conv" in k) / 1e3
        flops = 2 * trunk_flops(H, W)
        result["sizes"][f"{H}x{W}"] = {
            "ms_per_frame": {k: stats(v, 1e3, 3) for k, v in times.items()},
            "device_ms": {"eval": round(ev_sum["device_ms"], 3), "op": round(op_sum["device_ms"], 3)},
            "launches": {"eval": ev_sum["launches"], "op": op_sum["launches"]},
            "host_syncs": {"eval": host_syncs(lambda: ev(rq, target, mask)),
                           "op": host_syncs(lambda: op(render, target, mask))},
            "op_kernels_us": {k: round(sum(v), 1) for k, v in sorted(per.items(), key=lambda kv: -sum(kv[1]))},
            "trunk_gflop": round(flops / 1e9, 2),
            "trunk_tflops": round(flops / (conv_ms * 1e-3) / 1e12, 1) if conv_ms else None,
            "trunk_share_of_tf32_peak": round(flops / (conv_ms * 1e-3) / TF32_PEAK, 3) if conv_ms else None,
            "scores": {"eval_tf32": [round(v, 5) for v in ref], "op": [round(v, 5) for v in got]},
        }
    emit(result, args.json)


if __name__ == "__main__":
    main()
