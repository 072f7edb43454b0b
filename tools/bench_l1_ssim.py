"""ExAvatar's photometric loss block (avatar/main/model.py:196-215 without LPIPS): PyTorch ops vs. `losses.l1_ssim`.

  python tools/bench_l1_ssim.py [--workload C4] [--iters 50] [--frames 30] [--rounds 5] [--json out.json]

The block at C4 size (512x512, a box of ~60 % of the image): rgb + ssim of both combined renders, the two face
composites (L1 only), the two random-background terms (L1 only), rgb + ssim of the scene with the mask; forward +
backward into the five renders.  Arms:
  1. ops:        restated in PyTorch the way loss.py runs it -- `int()` of each box coordinate (four device->host reads
                 per cropped call), the window built and uploaded per SSIM call, grouped 11x11 F.conv2d;
  2. op:         the same terms through `l1_ssim`, eager;
  3. op_graph:   arm 2 captured once in a CUDA graph and replayed;
  4. frame_*:    C4 training frames/s, `TrainingFrameRenderer(use_graph=True)` forward + backward with no loss block,
                 then followed by the block of arm 1, then of arm 2.
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Kernel
times come from a separate torch.profiler run.  Prints the card name and power limit with the numbers.
"""
import argparse
import json
import math
import os
import statistics
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_frame_sh import card  # noqa: E402
from exavatar_release_b200 import TrainingFrameRenderer  # noqa: E402
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.losses import l1_ssim  # noqa: E402
from exavatar_release_b200.plan import RENDERS  # noqa: E402
from exavatar_release_b200.synthetic import WORKLOADS, make_population_assets  # noqa: E402


# ---- arm 1: the loss terms as loss.py evaluates them (host-side int() crops, a fresh window per SSIM call) ----------
def _crop(a, b, bbox):
    H, W = a.shape[2:]
    xmin, ymin, width, height = [int(v) for v in bbox[0]]  # four device->host reads
    xmin, ymin = max(xmin, 0), max(ymin, 0)
    xmax, ymax = min(xmin + width, W), min(ymin + height, H)
    return a[:, :, ymin:ymax, xmin:xmax], b[:, :, ymin:ymax, xmin:xmax]


def ops_rgb(out, target, bbox=None, mask=None, bg=None):
    if mask is not None and bg is not None:
        target = target * mask + (1 - mask) * bg[:, :, None, None]
    if bbox is not None:
        out, target = _crop(out, target, bbox)
    return torch.abs(out - target)


def ops_ssim(out, target, bbox=None, mask=None):
    if mask is not None:
        out, target = out * mask, target * mask
    if bbox is not None:
        out, target = _crop(out, target, bbox)
    g = torch.tensor([math.exp(-(x - 5) ** 2 / 4.5) for x in range(11)], dtype=torch.float32).to(out.device)
    g = (g / g.sum())[:, None]
    win = torch.mm(g, g.t())[None, None].repeat(3, 1, 1, 1)
    conv = lambda t: F.conv2d(t, win, padding=5, groups=3)  # noqa: E731
    m1, m2 = conv(out), conv(target)
    s11, s22, s12 = conv(out * out) - m1 ** 2, conv(target * target) - m2 ** 2, conv(out * target) - m1 * m2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    return ((2 * m1 * m2 + C1) * (2 * s12 + C2)) / ((m1 ** 2 + m2 ** 2 + C1) * (s11 + s22 + C2))


def block_ops(img, d):
    gt, bbox, mask, bg = d["img"], d["bbox"], d["mask"], d["bg"]
    loss = 0.0
    for r, (face, is_face) in zip(("scene_human", "scene_human_refined"), d["faces"]):
        x = img[r][None]
        loss = loss + ops_rgb(x, gt, bbox=bbox).mean() * 0.8 + (1 - ops_ssim(x, gt, bbox=bbox)).mean() * 0.2
        loss = loss + ops_rgb(x * (1 - is_face) + face * is_face, gt, bbox=bbox).mean() * 0.8
    for r in ("human", "human_refined"):
        loss = loss + ops_rgb(img[r][None], gt, bbox=bbox, mask=mask, bg=bg[None]).mean()
    x = img["scene"][None]
    loss = loss + (ops_rgb(x, gt) * (1 - mask)).mean() * 0.8 + (1 - ops_ssim(x, gt, mask=1 - mask)).mean() * 0.2
    return loss


def block_op(img, d):
    gt, bbox, mask, bg = d["img"][0], d["bbox"], d["mask"][0], d["bg"]
    loss = 0.0
    for r, (face, is_face) in zip(("scene_human", "scene_human_refined"), d["faces"]):
        x = img[r]
        l1, s = l1_ssim(x, gt, bbox)
        loss = loss + 0.8 * l1 + 0.2 * (1 - s)
        loss = loss + 0.8 * l1_ssim(x * (1 - is_face[0]) + face[0] * is_face[0], gt, bbox, ssim=False)[0]
    tgt = gt * mask + (1 - mask) * bg[:, None, None]
    for r in ("human", "human_refined"):
        loss = loss + l1_ssim(img[r], tgt, bbox, ssim=False)[0]
    l1, s = l1_ssim(img["scene"], gt, mask=1 - mask)
    return loss + 0.8 * l1 + 0.2 * (1 - s)


BLOCKS = {"ops": block_ops, "op": block_op}


def make_data(H, W, dev):
    g = torch.Generator().manual_seed(0)
    gt = F.interpolate(torch.rand(1, 3, H // 16, W // 16, generator=g), size=(H, W), mode="bilinear")
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1, 1, W), indexing="ij")
    mask = (1.5 - 2.0 * (xx ** 2 + (yy / 1.3) ** 2)).clamp(0, 1)[None, None]
    faces = []
    for _ in range(2):
        is_face = torch.zeros(1, 1, H, W)
        is_face[..., H // 5:H // 3, W // 3:W * 2 // 3] = 1.0
        faces.append((torch.rand(1, 3, H, W, generator=g).to(dev), is_face.to(dev)))
    # ~60 % of the image: 0.7 W x 0.85 H
    bbox = torch.tensor([[0.15 * W + 0.3, 0.08 * H + 0.6, 0.7 * W + 0.2, 0.85 * H + 0.9]])
    return {"img": gt.to(dev), "mask": mask.to(dev), "bbox": bbox.to(dev), "bg": torch.rand(3, generator=g).to(dev),
            "faces": faces}


def timed(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n


def stats(v, scale=1.0, nd=3):
    return {"median": round(statistics.median(v) * scale, nd), "min": round(min(v) * scale, nd),
            "max": round(max(v) * scale, nd)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C4")
    ap.add_argument("--iters", type=int, default=50, help="block calls per timed window")
    ap.add_argument("--frames", type=int, default=30, help="training frames per timed window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile-iters", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_l1_ssim: needs a CUDA device (no CPU timing)")
    dev = torch.device("cuda:0")
    wl = WORKLOADS[a.workload]
    H, W = wl.height, wl.width
    d = make_data(H, W, dev)
    g = torch.Generator().manual_seed(1)
    renders = {r: torch.rand(3, H, W, generator=g).to(dev).requires_grad_() for r in RENDERS}
    leaves = list(renders.values())
    result = {"workload": wl.name, "H": H, "W": W, "card": card(), "block_ms": {}, "frame_fps": {}, "kernels": {}}

    def step(name):
        for t in leaves:
            t.grad = None
        BLOCKS[name](renders, d).backward()

    # arm 3: forward + backward of the op block captured once
    static_in = {r: t.detach().clone().requires_grad_() for r, t in renders.items()}

    def graph_body():
        return torch.autograd.grad(block_op(static_in, d), list(static_in.values()))

    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(3):
            graph_body()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        graph_body()

    arms = {"ops": lambda: step("ops"), "op": lambda: step("op"), "op_graph": graph.replay}
    for fn in arms.values():
        for _ in range(5):
            fn()
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():
            times[k].append(timed(fn, a.iters))
    result["block_ms"] = {k: stats(v, 1e3) for k, v in times.items()}

    # kernel times of one block call (fwd + bwd), profiler run of its own
    from torch.profiler import ProfilerActivity, profile
    for k in ("ops", "op"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_iters):
                arms[k]()
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" and e.device_time_total > 0:
                per[e.key] = (e.device_time_total / a.profile_iters, e.count / a.profile_iters)
        top = sorted(per.items(), key=lambda kv: -kv[1][0])
        result["kernels"][k] = {"device_us_per_block": round(sum(v[0] for v in per.values()), 1),
                                "launches_per_block": round(sum(v[1] for v in per.values()), 1),
                                "top": {n[:90]: [round(v[0], 1), v[1]] for n, v in top[:8]}}

    # arm 4: training frames/s, TrainingFrameRenderer(use_graph=True) then no block / the ops block / the op block
    scene, human, refined = make_population_assets(a.workload, seed=0, device=dev)
    Ps, Ph = scene["mean_3d"].shape[0], human["mean_3d"].shape[0]
    lv = [{k: v.detach().clone().requires_grad_() for k, v in x.items()} for x in (scene, human, refined)]
    fleaves = [t for x in lv for t in x.values()]
    cams = [look_at_cam_param(y, (H, W), device=dev) for y in (-8.0, -3.0, 2.0, 7.0)]
    bg_r = torch.tensor([0.3, 0.7, 0.2], device=dev)
    fr = TrainingFrameRenderer(Ps, Ph, (H, W), dev, {"A": 8_000_000, "B": 8_000_000}, use_graph=True)

    def frame(block, i):
        out = fr(lv[0], lv[1], lv[2], cams[i % len(cams)], bg_r)
        img = {r: out[r]["img"] for r in RENDERS}
        loss = sum((img[r] * 1e-3).sum() for r in RENDERS) if block is None else BLOCKS[block](img, d)
        loss.backward()
        for t in fleaves:
            t.grad = None

    farms = {"frame_only": None, "frame_ops": "ops", "frame_op": "op"}
    for b in farms.values():
        for i in range(5):
            frame(b, i)
    fps = {k: [] for k in farms}
    for _ in range(a.rounds):
        for k, b in farms.items():
            fps[k].append(1.0 / timed(lambda: [frame(b, i) for i in range(a.frames)], 1) * a.frames)
    assert not fr.overflowed()
    result["frame_fps"] = {k: stats(v, 1.0, 1) for k, v in fps.items()}
    print(json.dumps(result))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
