"""SURVEY.md section 8f-2 outside the render: posing both human Gaussian sets, ExAvatar's ops vs `skin_gaussians`.

  python tools/bench_skin_pair.py [--workload C4] [--iters 50] [--frames 30] [--rounds 5] [--json out.json]

ExAvatar poses `mean_3d` and `mean_3d_refined` with one rig (avatar/common/nets/module.py:549-557).  At the workload's
human size (C4: P = 167 000, J = 55, a 4-sparse (P,55) weight table read through a row index):
  (a) ops:   skinning_weight[rows] gather, (P,55)x(55,16) matmul, one bmm per set, camera->world per set
             (`renderer.lbs_reference`; torch.inverse eagerly, the cofactor inverse under a CUDA graph, where
             torch.inverse cannot be captured), forward + autograd backward into xyz, xyz_refined, joint_mats, trans;
  (b) fused: `skinning.skin_gaussians`, the same forward + backward.
Timed eager and as a captured CUDA graph (CUDA events around --iters calls), arms alternated window by window, median
(min-max) over --rounds windows.  Then one C4 training frame (five renders, forward + backward) with each posing path
in front of `TrainingFrameRenderer(use_graph=True)`, frames/s the same way.  Then a torch.profiler run of its own for
the device time of each skinning kernel.  Prints the card name and power limit with the numbers.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_frame_sh import card  # noqa: E402
from exavatar_release_b200 import TrainingFrameRenderer  # noqa: E402
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.plan import RENDERS  # noqa: E402
from exavatar_release_b200.rasterizer import _inv3  # noqa: E402
from exavatar_release_b200.renderer import lbs_reference  # noqa: E402
from exavatar_release_b200.skinning import skin_gaussians  # noqa: E402
from exavatar_release_b200.synthetic import WORKLOADS, make_grad_image, make_population_assets  # noqa: E402

J = 55
ARMS = ("a_ops", "b_fused")


def rig(P, dev, seed=5):
    """4-sparse weights summing to one, small joint rotations / translations; rows: random, own row for the first 12 %."""
    g = torch.Generator().manual_seed(seed)
    w = torch.zeros(P, J)
    idx = torch.rand(P, J, generator=g).topk(4, dim=1).indices
    val = torch.rand(P, 4, generator=g) + 0.05
    w.scatter_(1, idx, val / val.sum(1, keepdim=True))
    A = torch.eye(4).repeat(J, 1, 1)
    ang = 0.15 * torch.rand(J, generator=g)
    A[:, 0, 0], A[:, 0, 1], A[:, 1, 0], A[:, 1, 1] = torch.cos(ang), -torch.sin(ang), torch.sin(ang), torch.cos(ang)
    A[:, :3, 3] = 0.02 * torch.randn(J, 3, generator=g)
    rows = torch.randint(0, P, (P,), generator=g)
    n_self = P * 12 // 100
    rows[:n_self] = torch.arange(n_self)
    return w.to(dev), rows.to(dev), A.to(dev), torch.tensor([0.01, -0.02, 0.03], device=dev)


def pose(arm, x, xr, W, rows, A, tr, R, t, capturable):
    if arm == "b_fused":
        return skin_gaussians(x, xr, W, rows, A, tr, R, t)
    w = W[rows]  # the (P,55) gather of ExAvatar (module.py:414)
    Rinv = _inv3(R) if capturable else None  # torch.inverse synchronises and cannot be captured
    return (lbs_reference(x, w, A, tr, R, t, cam_R_inv=Rinv), lbs_reference(xr, w, A, tr, R, t, cam_R_inv=Rinv))


def stats(v):
    return {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C4")
    ap.add_argument("--iters", type=int, default=50, help="pose fwd+bwd calls per timed window")
    ap.add_argument("--frames", type=int, default=30, help="training frames per timed window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_skin_pair: needs a CUDA device (no CPU timing)")
    dev = torch.device("cuda:0")
    wl = WORKLOADS[a.workload]
    H, W_img = wl.height, wl.width
    scene, human, refined = make_population_assets(a.workload, seed=0, device=dev)
    P = human["mean_3d"].shape[0]
    Ps = scene["mean_3d"].shape[0]
    W, rows, A0, tr0 = rig(P, dev)
    cam = look_at_cam_param(-6.0, (H, W_img), device=dev)
    R, t = cam["R"], cam["t"]
    x0 = (human["mean_3d"] @ R.t() + t.view(1, 3)).contiguous()
    xr0 = (refined["mean_3d"] @ R.t() + t.view(1, 3)).contiguous()
    gen = torch.Generator().manual_seed(3)
    gp, gq = torch.randn(P, 3, generator=gen).to(dev), torch.randn(P, 3, generator=gen).to(dev)
    lv = {k: v.clone().requires_grad_() for k, v in (("x", x0), ("xr", xr0), ("A", A0), ("tr", tr0))}
    result = {"workload": wl.name, "P": P, "J": J, "card": card(), "pose_fwd_bwd_ms": {}, "frame_fps": {},
              "kernel_us": {}}

    def pose_step(arm, capturable=False):
        posed, posed_r = pose(arm, lv["x"], lv["xr"], W, rows, lv["A"], lv["tr"], R, t, capturable)
        loss = (posed * gp).sum() + (posed_r * gq).sum()
        return torch.autograd.grad(loss, (lv["x"], lv["xr"], lv["A"], lv["tr"]))

    # ---- pose forward + backward: eager and CUDA graph ----
    graphs = {}
    for arm in ARMS:
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(3):
                pose_step(arm, capturable=True)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize()
        graphs[arm] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[arm]):
            pose_step(arm, capturable=True)
    runners = {"eager": lambda arm: pose_step(arm), "graph": lambda arm: graphs[arm].replay()}
    for mode, run in runners.items():
        for arm in ARMS:
            for _ in range(5):
                run(arm)
        times = {arm: [] for arm in ARMS}
        for _ in range(a.rounds):
            for arm in ARMS:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(a.iters):
                    run(arm)
                e1.record()
                torch.cuda.synchronize()
                times[arm].append(e0.elapsed_time(e1) / a.iters)
        result["pose_fwd_bwd_ms"][mode] = {arm: stats(v) for arm, v in times.items()}
    del graphs

    # ---- device time per kernel (profiler run of its own) ----
    from torch.profiler import ProfilerActivity, profile
    n_prof = 20
    for arm in ARMS:
        for _ in range(3):
            pose_step(arm)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n_prof):
                pose_step(arm)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            dt = getattr(ev, "device_time_total", None)
            if dt is None:
                dt = ev.cuda_time_total
            if dt > 0:
                per[ev.key] = dt / n_prof
        top = dict(sorted(per.items(), key=lambda kv: -kv[1])[:8])
        result["kernel_us"][arm] = {"top_per_call": {k[:80]: round(v, 2) for k, v in top.items()}}
        if arm == "b_fused":
            result["kernel_us"][arm]["skin_kernels"] = {k: round(v, 2) for k, v in per.items() if "skin_" in k}

    # ---- one C4 training frame with each posing path in front of TrainingFrameRenderer(use_graph=True) ----
    bg_r = torch.tensor([0.3, 0.7, 0.2], device=dev)
    g5 = {r: make_grad_image(a.workload, 10 + j, device=dev) for j, r in enumerate(RENDERS)}
    cams = [look_at_cam_param(y, (H, W_img), device=dev) for y in (-8.0, -3.0, 2.0, 7.0)]
    caps = {"A": 8_000_000, "B": 8_000_000}
    frs = {arm: TrainingFrameRenderer(Ps, P, (H, W_img), dev, caps, use_graph=True) for arm in ARMS}
    sc_leaves = {k: v.detach().clone().requires_grad_() for k, v in scene.items()}
    h_leaves = {k: v.detach().clone().requires_grad_() for k, v in human.items() if k != "mean_3d"}
    r_leaves = {k: v.detach().clone().requires_grad_() for k, v in refined.items() if k != "mean_3d"}
    leaves = list(lv.values()) + list(sc_leaves.values()) + list(h_leaves.values()) + list(r_leaves.values())

    def frame(arm, i):
        c = cams[i % len(cams)]
        posed, posed_r = pose(arm, lv["x"], lv["xr"], W, rows, lv["A"], lv["tr"], R, t, capturable=False)
        out = frs[arm](sc_leaves, dict(h_leaves, mean_3d=posed), dict(r_leaves, mean_3d=posed_r), c, bg_r)
        sum((out[r]["img"] * g5[r]).sum() for r in RENDERS).backward()
        for x in leaves:
            x.grad = None

    for arm in ARMS:
        for i in range(5):
            frame(arm, i)
    torch.cuda.synchronize()
    fps = {arm: [] for arm in ARMS}
    for _ in range(a.rounds):
        for arm in ARMS:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(a.frames):
                frame(arm, i)
            torch.cuda.synchronize()
            fps[arm].append(a.frames / (time.perf_counter() - t0))
    assert not any(f.overflowed() for f in frs.values())
    result["frame_fps"]["use_graph"] = {arm: stats(v) for arm, v in fps.items()}
    print(json.dumps(result))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
