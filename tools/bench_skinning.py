"""SURVEY.md section 8f-2 measurement: ExAvatar's human path (skinning + rasteriser, forward + backward), its ops vs ours.

  python tools/bench_skinning.py [--workload C4]
Unfused = `lbs_reference` (the reference's five PyTorch ops, module.py:413-422, 555-557) + GaussianRasterizer;
fused = SkinnedGaussianRasterizer (the skinning op `skin_gaussians`, then GaussianRasterizer).  Public autograd API, fixed-capacity mode, CUDA events, L2 flushed between iterations.
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import cuda_device, graph_replay  # noqa: E402
from exavatar_release_b200 import rasterizer as RZ  # noqa: E402
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.renderer import lbs_reference, render_settings  # noqa: E402
from exavatar_release_b200.synthetic import WORKLOADS, make_grad_image, make_population_assets  # noqa: E402
from test_fused_skinning import _rig  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C4")
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    wl = WORKLOADS[a.workload]
    dev = cuda_device("bench_skinning")
    H, W = wl.height, wl.width
    _, human, _ = make_population_assets(a.workload, seed=0, device=dev)
    P, J = human["mean_3d"].shape[0], 55
    cam = look_at_cam_param(7.0, (H, W), device=dev)
    st = render_settings((H, W), cam, torch.tensor([0.2, 0.4, 0.9], device=dev))
    w, A, trans = _rig(P, J, torch.float32, dev)
    xyz0 = human["mean_3d"] @ cam["R"].t() + cam["t"].view(1, 3)
    gi = make_grad_image(a.workload, 2).to(dev)
    Rinv = torch.inverse(cam["R"])  # outside the timed / captured region for both paths
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def leaves():
        return {"xyz": xyz0.clone().requires_grad_(), "A": A.clone().requires_grad_(), "trans": trans.clone().requires_grad_(),
                "scale": human["scale"].clone().requires_grad_(), "rgb": human["rgb"].clone().requires_grad_(),
                "opacity": human["opacity"].clone().requires_grad_()}

    def unfused(lv):
        posed = lbs_reference(lv["xyz"], w, lv["A"], lv["trans"], None, cam["t"], cam_R_inv=Rinv)
        m2 = torch.zeros(P, 3, device=dev, requires_grad=True)
        img = RZ.GaussianRasterizer(st)(means3D=posed, means2D=m2, opacities=lv["opacity"], colors_precomp=lv["rgb"],
                                        scales=lv["scale"], rotations=human["rotation"])[0]
        (img * gi).sum().backward()

    def fused(lv):
        m2 = torch.zeros(P, 3, device=dev, requires_grad=True)
        img = RZ.SkinnedGaussianRasterizer(st)(lv["xyz"], w, lv["A"], lv["trans"], cam["R"], cam["t"], m2, lv["opacity"],
                                               lv["rgb"], lv["scale"], human["rotation"])[0]
        (img * gi).sum().backward()

    # learn the duplicate count, then fixed capacity (no polling) for both paths
    with torch.no_grad():
        RZ.GaussianRasterizer(st)(means3D=human["mean_3d"], means2D=torch.zeros(P, 3, device=dev), opacities=human["opacity"],
                                  colors_precomp=human["rgb"], scales=human["scale"], rotations=human["rotation"])
    cap = int(RZ.last_duplicate_count(dev, P, W, H) * 1.3) + 4096
    RZ.set_fixed_capacity(cap)
    out, out_graph = {}, {}
    for name, fn in (("unfused", unfused), ("fused", fused)):
        lv = leaves()
        for _ in range(5):
            fn(lv)
        torch.cuda.synchronize()

        def event_ms(run):
            ms = 0.0
            for _ in range(a.iters):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run()
                e1.record()
                torch.cuda.synchronize()
                ms += e0.elapsed_time(e1)
            return ms / a.iters

        def eager():
            for v in lv.values():
                v.grad = None
            fn(lv)

        out[name] = event_ms(eager)
        # the same work captured in a CUDA graph: removes the host cost of the extra PyTorch launches from the picture.
        # Fresh leaves: the gradient-accumulation nodes of the eager ones belong to the default stream, which a capture
        # may not wait on.
        lv = leaves()
        replay = graph_replay(eager, 1)
        replay()
        torch.cuda.synchronize()
        out_graph[name] = event_ms(replay)
    assert not RZ.overflowed()
    print(f"{a.workload}: human population P={P}, J={J}, {W}x{H}; forward+backward through the public API")
    for tag, o in (("eager", out), ("CUDA graph", out_graph)):
        print(f"  [{tag}] unfused (5 PyTorch skinning ops + rasteriser): {o['unfused'] * 1e3:8.1f} us")
        print(f"  [{tag}] fused   (SkinnedGaussianRasterizer)          : {o['fused'] * 1e3:8.1f} us   ({o['unfused'] / o['fused']:.2f}x)")


if __name__ == "__main__":
    main()
