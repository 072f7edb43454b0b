"""K6 (`project_bwd_kernel`, `b2r_backward_project`) on its own, at the two pass shapes of a C4 training frame.

  python tools/bench_project_bwd.py [--iters 200] [--rounds 5] [--label new] [--check-dir DIR]

One C4 scene (297 k Gaussians: 167 k human + 130 k scene, 512x512) is projected, binned and composited once; its
backward composite fills the gradient scratch.  Then K6 alone, as `MergedFivePlan` launches it:
  pass_A  all rows, accumulate, densification statistics on the first P_SCENE rows, scratch clear;
  pass_B  first_row = P_SCENE (the detached scene prefix of the refined pass), accumulate, scratch clear.
The scratch clear leaves the scratch zero after the first launch; the kernel's work does not depend on its values.
CUDA events around --iters launches after a warm-up, median (min-max) over --rounds windows.

Algorithmic bytes per launch (what the kernel must move, each byte once), with V the visible rows of [first_row, P):
  (P - first_row) * 16                      aux records (radius decides visibility)
  + V * (48 + 4 + 12 + 12 + 16)             scratch row, clamp bits, means3D, scales, rotations
  + V * 17 * 4 * (2 if accumulate else 1)   the 17 output floats (read and written when accumulating)
  + V * 48                                  scratch clear
  + V_scene * 3 * 4 * 2                     densification sums (read and written) on the scene rows
Culled rows of an accumulating launch are not touched.  The fraction is against the H100 SXM data sheet's 3.35 TB/s.

_lib.py loads one library per process: to compare two builds, run this script once per build (B2R_LIB=<path>) and
alternate the runs.  Prints one JSON line per run with the card's name, power limit and SM clock read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import HBM_BYTES_PER_S, card, cuda_device  # noqa: E402
from exavatar_release_b200 import _lib as L  # noqa: E402
from exavatar_release_b200 import rasterizer as rz  # noqa: E402
from exavatar_release_b200.plan import FramePlan  # noqa: E402
from exavatar_release_b200.synthetic import WORKLOADS, make_assets, make_grad_image  # noqa: E402
from util import workload_settings  # noqa: E402

WIDTHS = {"means3D": 3, "means2D": 3, "colors": 3, "opacities": 1, "scales": 3, "rotations": 4}


def algorithmic_bytes(rows, vis, vis_scene, accumulate):
    return rows * 16 + vis * (48 + 4 + 12 + 12 + 16) + vis * 17 * 4 * (2 if accumulate else 1) + vis * 48 + vis_scene * 24


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--label", default=os.environ.get("B2R_LIB", "tree").replace("/", "_"))
    ap.add_argument("--check-dir", default=None,
                    help="the first run saves the gradient scratch here, later runs load it; every run saves the outputs "
                         "of one writing launch per pass as <label>_<pass>.pt")
    a = ap.parse_args()
    dev = cuda_device("bench_project_bwd")
    wl = WORKLOADS["C4"]
    P, Ps = wl.n_avatar + wl.n_scene, wl.n_scene
    assets = {k: v.to(dev) for k, v in make_assets("C4", seed=0).items()}
    assert assets["mean_3d"].shape[0] == P
    st = workload_settings("C4", yaw=4.0, device=dev, settings_cls=rz.GaussianRasterizationSettings)
    plan = FramePlan(P, wl.width, wl.height, 40_000_000, dev)
    sc = plan.scene(0, st, assets)
    plan.forward(sc)
    g_color = make_grad_image("C4", 1).to(dev).contiguous()
    stream = torch.cuda.current_stream(dev).cuda_stream
    args = L.B2RBackwardArgs(g_color.data_ptr(), None, None)
    L.check(plan.lib.b2r_backward_composite(C.byref(sc), C.byref(plan.ws), None, C.byref(args), plan.bwd_scratch.data_ptr(),
                                            plan.bwd_bytes, stream), "b2r_backward_composite")
    torch.cuda.synchronize()
    assert plan.status()["overflow"] == 0
    visible = plan.radii > 0
    if a.check_dir:  # same scratch for every build: the backward composite's float atomics do not sum in a fixed order
        os.makedirs(a.check_dir, exist_ok=True)
        path = os.path.join(a.check_dir, "scratch.pt")
        if os.path.exists(path):
            plan.bwd_scratch.copy_(torch.load(path).to(dev))
        else:
            torch.save(plan.bwd_scratch.cpu(), path)
        scratch0 = plan.bwd_scratch.clone()  # the timed launches of a pass clear it
    result = {"label": a.label, "workload": wl.name, "P": P, "P_scene": Ps, "passes": {}}
    for name, first_row in (("pass_A", 0), ("pass_B", Ps)):
        rows = P - first_row
        g = {k: torch.zeros(rows, w, device=dev) for k, w in WIDTHS.items()}
        dens = {k: torch.zeros(rows, device=dev) for k in ("grad_accum", "count", "radius_max")} if first_row == 0 else None
        ka = L.B2RBackwardArgs(None, None, None, g["means3D"].data_ptr(), g["means2D"].data_ptr(), None,
                               g["colors"].data_ptr(), g["opacities"].data_ptr(), g["scales"].data_ptr(),
                               g["rotations"].data_ptr(), None)
        ka.flags = L.B2R_BWD_ACCUMULATE | L.B2R_BWD_SCRATCH_ZEROED
        ka.first_row = first_row
        if dens is not None:
            ka.densify_grad_accum, ka.densify_count = dens["grad_accum"].data_ptr(), dens["count"].data_ptr()
            ka.densify_radius_max, ka.densify_rows = dens["radius_max"].data_ptr(), Ps

        def launch():
            L.check(plan.lib.b2r_backward_project(C.byref(sc), C.byref(plan.ws), C.byref(ka), plan.bwd_scratch.data_ptr(),
                                                  plan.bwd_bytes, stream), "b2r_backward_project")

        if a.check_dir:  # one writing launch that keeps the scratch: the outputs, to compare builds bit for bit
            flags = ka.flags
            ka.flags = 0
            plan.bwd_scratch.copy_(scratch0)
            launch()
            torch.cuda.synchronize()
            ka.flags = flags
            torch.save({k: v.cpu() for k, v in {**g, **(dens or {})}.items()},
                       os.path.join(a.check_dir, f"{a.label}_{name}.pt"))
        for _ in range(20):
            launch()
        torch.cuda.synchronize()
        times = []
        for _ in range(a.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                launch()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) * 1e3 / a.iters)
        vis = int(visible[first_row:].sum())
        vis_scene = int(visible[:Ps].sum()) if dens is not None else 0
        nbytes = algorithmic_bytes(rows, vis, vis_scene, True)
        us = statistics.median(times)
        result["passes"][name] = {"first_row": first_row, "rows": rows, "visible": vis, "us_per_launch": round(us, 2),
                                  "us_min": round(min(times), 2), "us_max": round(max(times), 2),
                                  "algorithmic_bytes": nbytes, "GBps": round(nbytes / us / 1e3, 1),
                                  "frac_of_3.35TBps": round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)}
    result["card"] = card()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
