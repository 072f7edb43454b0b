"""ExAvatar's scene Gaussian assets (SceneGaussian.forward, avatar/common/nets/module.py:253-272) the way ExAvatar
computes them vs. `scene_assets`.

  python tools/bench_scene_assets.py [--iters 20] [--rounds 5] [--frames 10] [--json out.json]

C4 size (130 000 scene Gaussians, M = 16, degree 3, rgb mode as ExAvatar renders), forward + backward of a seeded
weighted sum of the four outputs.  Arms:
  1. exavatar:  SceneGaussian.forward's work and host reads as ExAvatar pays them, built from this project's
                restatements (`exavatar_form`): pytorch3d's two conversions, torch.inverse(R), and the reads of the float
                active_sh_degree buffer that ExAvatar's eval_sh makes;
  2. op:        `scene_assets`, eager;
  3. op_graph:  arm 2 captured once in a CUDA graph and replayed;
  4. frame_*:   C4 training frames/s of tools/bench_lpips.py's frame (tools/c4_frame.py's frame -- rig op, networks,
                skinning, the five renders, l1_ssim, regularisers -- plus the two LPIPS terms as the op) with the
                scene's assets built every frame by arm 1's form or by the op.
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Host
syncs per call are counted with torch's sync debug mode ("warn").  Device time per
kernel comes from a separate torch.profiler run, and each scene_assets kernel's achieved bandwidth from the fp32 words
it must move over that time.  Prints the card name and power limit with the numbers.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, graph_replay, host_syncs, kernel_events, stats  # noqa: E402
from c4_frame import BOX, FrameArm, frames_per_second  # noqa: E402
from exavatar_release_b200 import scene_assets  # noqa: E402
from exavatar_release_b200.scene_assets import scene_assets_reference  # noqa: E402
from exavatar_release_b200.sh import sh_to_rgb  # noqa: E402

P, M = 130000, 16


def exavatar_form(mean, opacity, scale, rotation, feature_dc, feature_rest, active_sh_degree, cam_param):
    """Arm 1: SceneGaussian.forward's work and host reads as ExAvatar pays them, from this project's restatements.
    The activations, pytorch3d's two conversions and the packed coefficients come from `scene_assets_reference`, the
    colour from `sh.sh_to_rgb`.  Around them sit the reads of the (1,) float degree buffer that ExAvatar's eval_sh
    makes: two range checks, the coefficient-count check, and one comparison per degree level reached, up to three.
    The camera position goes through `torch.inverse(R)`."""
    out = scene_assets_reference(mean, opacity, scale, rotation, feature_dc, feature_rest, active_sh_degree)
    sh = out.pop("shs")
    del out["sh_degree"]
    deg = active_sh_degree
    if not bool(deg <= 4) or not bool(deg >= 0):
        raise ValueError("degree out of range")
    if not bool(sh.shape[1] >= (deg + 1) ** 2):
        raise ValueError("too few SH coefficients for the degree")
    level = 0
    while level < 3 and bool(deg > level):
        level += 1
    cam_pos = torch.matmul(torch.inverse(cam_param["R"]), -cam_param["t"].view(3, 1)).view(1, 3)
    out["rgb"] = sh_to_rgb(level, sh, mean, cam_pos)
    return out


def params(dev, scene=None, seed=0):
    g = torch.Generator().manual_seed(seed)
    n = P if scene is None else scene["mean_3d"].shape[0]
    p = {"mean": torch.randn(n, 3, generator=g) if scene is None else scene["mean_3d"].cpu(),
         "opacity": 2 * torch.randn(n, 1, generator=g) if scene is None else
         torch.logit(scene["opacity"].cpu().clamp(1e-4, 1 - 1e-4)),
         "scale": -4 + torch.randn(n, 3, generator=g) if scene is None else torch.log(scene["scale"].cpu()),
         "rotation": torch.randn(n, 6, generator=g)}
    base = torch.cat([torch.randn(n, 1, 3, generator=g), 0.3 * torch.randn(n, M - 1, 3, generator=g)], 1).to(dev)
    p = {k: v.to(dev).requires_grad_() for k, v in p.items()}
    base.requires_grad_()
    return p, base  # feature_dc / feature_rest: views of one (P,16,3) tensor, as init_from_point_cloud registers them


def main():
    a = arg_parser(__doc__, iters=20, frames=10).parse_args()
    dev = cuda_device("bench_scene_assets")
    from exavatar_release_b200.camera import look_at_cam_param
    cam = look_at_cam_param(8.0, (512, 512), device=dev)
    deg = torch.full((1,), 3.0, device=dev)  # ExAvatar's active_sh_degree buffer
    p, base = params(dev)
    g = torch.Generator().manual_seed(1)
    w = [torch.randn(s, generator=g).to(dev) for s in ((P, 1), (P, 3), (P, 4), (P, 3))]

    def loss(out):
        return sum((out[k] * wk).sum() for k, wk in zip(("opacity", "scale", "rotation", "rgb"), w))

    def args():
        return (p["mean"], p["opacity"], p["scale"], p["rotation"], base[:, :1], base[:, 1:], deg, cam)

    def clear():
        for t in (*p.values(), base):
            t.grad = None

    def run_exavatar():
        clear()
        loss(exavatar_form(*args())).backward()

    def run_op():
        clear()
        loss(scene_assets(*args())).backward()

    run_exavatar()
    ge = [t.grad.clone() for t in (*p.values(), base)]
    run_op()
    go = [t.grad.clone() for t in (*p.values(), base)]
    torch.cuda.synchronize()
    agree = {k: float((x - y).abs().max() / y.abs().max()) for k, x, y in zip((*p, "sh"), go, ge)}

    arms = {"exavatar": run_exavatar, "op": run_op, "op_graph": graph_replay(run_op, 2)}
    times = alternate(arms, a.iters, a.rounds, 1)
    syncs = {k: host_syncs(arms[k]) for k in ("exavatar", "op")}

    # fp32 words each kernel must move per Gaussian: the forward reads 6 + 1 + 3 + 3 + 48 and writes 1 + 3 + 4 + 3;
    # the backward reads 6 + 4 + 1 + 1 + 3 + 3 + 3 + 3 + 48 and writes 1 + 3 + 6 + 48 + 3
    words = {"scene_assets_fwd": 61 + 11, "scene_assets_bwd": 72 + 61}
    prof = {}
    for k, fn in arms.items():
        ev, prof[k] = kernel_events(fn)
        for name, nw in words.items():
            ms = sum(e.device_time for e in ev if name in e.name) / 1e3
            if ms > 0:
                prof[k][name] = {"ms": ms, "TBps": 4 * nw * P / (ms * 1e-3) / 1e12}

    # the frame of tools/bench_lpips.py: tools/c4_frame.py's frame with ExAvatar's two LPIPS terms as the op
    from make_lpips_golden import lpips_weights
    from exavatar_release_b200.perceptual import LPIPS
    lp = LPIPS(*lpips_weights(), dev)
    bbox = torch.tensor([BOX], device=dev)

    def lpips_terms(o, target):
        return 0.2 * lp(torch.stack((o["scene_human"]["img"], o["scene_human_refined"]["img"])), target, bbox).sum()

    def scene_arm(form):
        leaves = {}

        def build(scene, cam_):
            if not leaves:
                leaves["p"] = params(dev, scene, seed=2)
            sp, sb = leaves["p"]
            for t in (*sp.values(), sb):
                t.grad = None
            return form(sp["mean"], sp["opacity"], sp["scale"], sp["rotation"], sb[:, :1], sb[:, 1:], deg, cam_)
        return FrameArm(scene=build, loss=lpips_terms)

    frames = frames_per_second(a, dev, {"scene_exavatar": scene_arm(exavatar_form), "scene_op": scene_arm(scene_assets)})
    res = {"card": card(), "P": P, "M": M, "degree": 3,
           "scene_ms": {k: stats(v, 1e3) for k, v in times.items()},
           "host_syncs_per_call": syncs, "profile": prof, "op_vs_exavatar_grad_rel": agree, "frames_per_s": frames}
    emit(res, a.json)


if __name__ == "__main__":
    main()
