"""Runs a few forward(+backward) frames of a workload through FramePlan (no CUDA graph) -- the target for ncu.

  ncu --set full -k regex:composite -s 18 -c 2 -o gpurun_out/prof python tools/profile_frame.py --workload C2 --frames 3
Also prints the tile-list statistics the design discussion in DESIGN.md relies on.
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from exavatar_release_b200 import rasterizer as RZ  # noqa: E402
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.plan import FramePlan, grad_bucket  # noqa: E402
from exavatar_release_b200.renderer import render_settings  # noqa: E402
from exavatar_release_b200.synthetic import WORKLOADS, make_assets, make_grad_image  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C2")
    ap.add_argument("--frames", type=int, default=3)
    ap.add_argument("--stats", action="store_true")
    a = ap.parse_args()
    wl = WORKLOADS[a.workload]
    dev = torch.device("cuda:0")
    P, H, W = wl.n_avatar + wl.n_scene, wl.height, wl.width
    M = (wl.sh_degree + 1) ** 2 if wl.sh_degree > 0 else 0
    assets = make_assets(a.workload, seed=0, device=dev)
    bg = torch.ones(3, device=dev)
    st = render_settings((H, W), look_at_cam_param(5.0, (H, W), device=dev), bg)
    if M:
        st = st._replace(sh_degree=wl.sh_degree)
    gi = make_grad_image(a.workload, 0, device=dev)
    plan = FramePlan(P, W, H, 40_000_000 if a.workload in ("C3", "C5") else 12_000_000, dev, sh_coeffs=M)
    sc = plan.scene(0, st, assets)
    _, views = grad_bucket(P, dev, M)
    for f in range(a.frames):
        plan.forward(sc)
        if wl.backward:
            plan.backward(sc, gi, views)
    torch.cuda.synchronize()
    s = plan.status()
    print("status", s)
    if a.stats:
        ctx = plan.read_ctx()
        r, nc = ctx["ranges"], ctx["n_contrib"]
        n = (r[:, 1] - r[:, 0]).astype(np.int64)
        print("tiles", len(r), "D", n.sum(), "max", n.max(), "mean", n.mean(), "pct50/90/99", np.percentile(n, [50, 90, 99]))
        print("tiles with n>2048:", (n > 2048).sum(), " n>1024:", (n > 1024).sum(), " n>256:", (n > 256).sum(), " n==0:", (n == 0).sum())
        tmax = nc.reshape(H // 16, 16, W // 16, 16).max(axis=(1, 3)).reshape(-1) if H % 16 == 0 and W % 16 == 0 else None
        if tmax is not None:
            print("n_contrib tile-max: sum", tmax.sum(), "max", tmax.max(), " mean pixel n_contrib", nc.mean())
            top = np.argsort(-n)[:8]
            print("longest tiles:", [(int(t), int(n[t]), int(tmax[t])) for t in top])


if __name__ == "__main__":
    main()
