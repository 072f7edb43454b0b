"""ExAvatar's human-Gaussian networks (avatar/common/nets/module.py:424-457 extract_tri_feature and the four
make_linear_layers(use_gn=True) stacks): PyTorch modules vs. `human_nets.TriplaneFeatures` + `human_nets.gn_mlp`.

  python tools/bench_human_nets.py [--iters 10] [--rounds 5] [--json out.json]

Workload: C4 size, P = 167 618 rows, two (3,32,128,128) triplanes, the four stacks with ExAvatar's shapes (geo_net and
geo_offset_net with a 3 + 1 head each, rgb_net and rgb_offset_net with a final Linear to 3; the pose block 126 wide,
the normal 3 wide).  One step = triplane features + all four stacks forward, then one backward of a weighted sum of
the outputs to both triplanes and every parameter.  Arms:
  1. torch:     the modules in fp32 with torch defaults (TF32 off for matmul), F.grid_sample, the face overwrite and
                the `.repeat(P, 1)` pose block as the reference writes them;
  2. op:        TriplaneFeatures + gn_mlp, eager;
  3. op_graph:  arm 2 captured once in a CUDA graph and replayed;
  4. frame_*:   C4 training frames/s of the whole human chain -- triplane, the three stacks, offsets, nearest_rows,
                skin_gaussians, VertexNormals, rgb_offset_net -- in front of `TrainingFrameRenderer(use_graph=True)`,
                then ExAvatar's L1 + SSIM terms (`l1_ssim`) of the five renders and the backward, with the networks as
                the torch modules (frame_torch) or as the ops (frame_op), on the synthetic human mesh.
Arms alternate window by window in one process (host clock around N steps + device sync): median (min-max).  Kernel
times come from a separate torch.profiler run of arm 2.  Achieved TFLOP/s counts the stacks' multiply-adds in
ExAvatar's form (pose unfolded) and with the pose folded; 3xTF32 issues three tensor-core MMAs per counted product, so
the tensor cores do three times the counted work.  Prints the card name and power limit with the numbers.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_frame_sh import card  # noqa: E402
from exavatar_release_b200 import TrainingFrameRenderer  # noqa: E402
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.geometry import VertexNormals, nearest_rows  # noqa: E402
from exavatar_release_b200.human_nets import TriplaneFeatures, gn_mlp  # noqa: E402
from exavatar_release_b200.losses import l1_ssim  # noqa: E402
from exavatar_release_b200.plan import RENDERS  # noqa: E402
from exavatar_release_b200.skinning import skin_gaussians  # noqa: E402
from exavatar_release_b200.synthetic import WORKLOADS, Workload, make_human_mesh, make_population_assets  # noqa: E402

P = 167618
TRI, POSE, NORMAL = 96, 126, 3


def stack(k_in, heads=None, final=None):
    mods = []
    for k in (k_in, 128, 128):
        mods += [nn.Linear(k, 128), nn.GroupNorm(4, 128), nn.ReLU(inplace=True)]
    if final:
        mods.append(nn.Linear(128, final))
    return nn.Sequential(*mods).cuda(), [nn.Sequential(nn.Linear(128, h)).cuda() for h in (heads or [])]


def macs_per_row(folded):
    first = {"geo": TRI, "geo_offset": TRI + (0 if folded else POSE), "rgb": TRI,
             "rgb_offset": TRI + NORMAL + (0 if folded else POSE)}
    heads = {"geo": 4, "geo_offset": 4, "rgb": 3, "rgb_offset": 3}
    return sum(k * 128 + 2 * 128 * 128 + 128 * heads[n] for n, k in first.items())


def stats(v, scale=1.0, nd=3):
    return {"median": round(statistics.median(v) * scale, nd), "min": round(min(v) * scale, nd),
            "max": round(max(v) * scale, nd)}


def frames_per_second(args, dev, nets, tp, tpf, pose):
    """C4 training frames/s of the human chain in front of TrainingFrameRenderer(use_graph=True), per network arm."""
    m = make_human_mesh()
    P = m["verts"].shape[0]
    c4 = WORKLOADS["C4"]
    H, W = c4.height, c4.width
    wl = Workload("C4 with the synthetic mesh's Gaussians", H, W, P, c4.n_scene, 0, True)
    scene, human, _ = make_population_assets(wl, seed=0, device=dev)
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    R, tc = cam["R"], cam["t"]
    to_cam = lambda v: (v.to(dev) @ R.t() + tc.view(1, 3)).contiguous()  # noqa: E731
    canon, targets, sm = to_cam(m["queries"]), to_cam(m["targets"]), m["self_map"].to(dev)
    verts = m["verts"].to(dev)
    is_face = verts[:, 1] > 0.6
    tri_op = TriplaneFeatures(verts, is_face)
    grid = tri_op.grid
    vn = VertexNormals(m["faces"], P, flip=m["flip"].to(dev))
    g = torch.Generator().manual_seed(5)
    table = torch.zeros(P, 55)
    table.scatter_(1, torch.rand(P, 55, generator=g).topk(4, dim=1).indices, torch.full((P, 4), 0.25))
    table = table.to(dev)
    A = torch.eye(4).repeat(55, 1, 1).to(dev)
    A[:, :3, 3] = 0.01 * torch.randn(55, 3, generator=g).to(dev)
    A.requires_grad_()
    tr = torch.zeros(3, device=dev, requires_grad=True)
    lv = {k: v.detach().clone().requires_grad_() for k, v in scene.items()}
    bg = torch.tensor([0.3, 0.7, 0.2], device=dev)
    target = torch.rand((3, H, W), generator=torch.Generator(device=dev).manual_seed(6), device=dev)
    fr = TrainingFrameRenderer(scene["mean_3d"].shape[0], P, (H, W), dev, {"A": 8_000_000, "B": 8_000_000},
                               use_graph=True)
    leaves = [tp, tpf, A, tr, *lv.values()] + [p for t, hs in nets.values() for mm in [t, *hs] for p in mm.parameters()]

    def torch_tri():
        def sample(planes, gg):
            return torch.cat([F.grid_sample(planes[p, None], gg[None, :, None, p, :], align_corners=False)[0, :, :, 0]
                              for p in range(3)]).permute(1, 0)
        tri = sample(tp, grid)
        tri[is_face] = sample(tpf, grid[is_face])
        return tri

    def torch_net(k, ins):
        t, hs = nets[k]
        x = torch.cat([v if v.dim() == 2 else v.view(1, -1).repeat(P, 1).detach() for v in ins], 1)
        f = t(x)
        return torch.cat([h(f) for h in hs], 1) if hs else f

    def frame(which):
        if which == "op":
            tri = tri_op(tp, tpf)
            net = lambda k, ins: gn_mlp(ins, *nets[k])  # noqa: E731
        else:
            tri = torch_tri()
            net = torch_net
        geo, geo_off, rgb = net("geo", [tri]), net("geo_offset", [tri, pose]), net("rgb", [tri])
        mean_3d = canon + 0.01 * geo[:, :3]
        mean_3d_r = mean_3d + 0.005 * geo_off[:, :3]
        rows = nearest_rows(mean_3d.detach(), targets, sm)
        posed, posed_r = skin_gaussians(mean_3d, mean_3d_r, table, rows, A, tr, R, tc)
        rgb_off = net("rgb_offset", [tri, pose, vn(posed_r)])
        hv = dict(human, mean_3d=posed, scale=human["scale"] * torch.exp(0.1 * geo[:, 3:]),
                  rgb=(torch.tanh(rgb) + 1) / 2)
        rv = dict(human, mean_3d=posed_r, scale=human["scale"] * torch.exp(0.1 * (geo[:, 3:] + geo_off[:, 3:])),
                  rgb=(torch.tanh(rgb + rgb_off) + 1) / 2)
        out = fr(lv, hv, rv, cam, bg)
        loss = 0
        for r in RENDERS:
            l1, ss = l1_ssim(out[r]["img"], target)
            loss = loss + 0.8 * l1 + 0.2 * (1 - ss)
        loss.backward()
        for v in leaves:
            v.grad = None

    arms = ("torch", "op")
    for k in arms:
        for _ in range(3):
            frame(k)
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k in arms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.frames):
                frame(k)
            torch.cuda.synchronize()
            times[k].append(args.frames / (time.perf_counter() - t0))
    if fr.overflowed():
        raise SystemExit("bench_human_nets: a render overflowed its list capacity")
    return {f"frame_{k}": stats(v, 1.0, 1) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=10, help="training frames per timed window")
    ap.add_argument("--json", default=None)
    ap.add_argument("--trace-dir", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_human_nets: needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    g = torch.Generator(device=dev).manual_seed(0)
    pos = (torch.rand((P, 3), generator=g, device=dev) - 0.5) * torch.tensor([0.9, 1.9, 0.4], device=dev)
    is_face = pos[:, 1] > 0.72
    tri_op = TriplaneFeatures(pos, is_face)
    grid = tri_op.grid
    tp = nn.Parameter(torch.randn((3, 32, 128, 128), device=dev) * 0.1)
    tpf = nn.Parameter(torch.randn((3, 32, 128, 128), device=dev) * 0.1)
    nets = {"geo": stack(TRI, [3, 1]), "geo_offset": stack(TRI + POSE, [3, 1]), "rgb": stack(TRI, None, 3),
            "rgb_offset": stack(TRI + POSE + NORMAL, None, 3)}
    pose = torch.randn(POSE, device=dev)
    normal = F.normalize(torch.randn((P, 3), device=dev), dim=1)
    w_out = {k: torch.randn((P, 4 if k.startswith("geo") else 3), device=dev) for k in nets}
    params = [tp, tpf] + [p for t, hs in nets.values() for m in [t, *hs] for p in m.parameters()]

    def torch_step():
        def sample(planes, gg):
            return torch.cat([F.grid_sample(planes[p, None], gg[None, :, None, p, :], align_corners=False)[0, :, :, 0]
                              for p in range(3)]).permute(1, 0)
        tri = sample(tp, grid)
        tri[is_face] = sample(tpf, grid[is_face])
        posep = pose.view(1, POSE).repeat(P, 1)
        feats = {"geo": tri, "geo_offset": torch.cat((tri, posep.detach()), 1), "rgb": tri,
                 "rgb_offset": torch.cat((tri, posep.detach(), normal.detach()), 1)}
        loss = 0
        for k, (t, hs) in nets.items():
            f = t(feats[k])
            out = torch.cat([h(f) for h in hs], 1) if hs else f
            loss = loss + (out * w_out[k]).sum()
        loss.backward()

    def op_step():
        tri = tri_op(tp, tpf)
        ins = {"geo": [tri], "geo_offset": [tri, pose], "rgb": [tri], "rgb_offset": [tri, pose, normal]}
        loss = 0
        for k, (t, hs) in nets.items():
            loss = loss + (gn_mlp(ins[k], t, hs) * w_out[k]).sum()
        loss.backward()

    def zero():
        for p in params:
            p.grad = None

    # warm-up and capture
    for _ in range(3):
        zero(); torch_step()  # noqa: E702
        zero(); op_step()  # noqa: E702
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            zero()
            op_step()
    torch.cuda.current_stream().wait_stream(s)
    zero()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        op_step()
    graph.replay()
    torch.cuda.synchronize()

    arms = {"torch": lambda: (zero(), torch_step()), "op": lambda: (zero(), op_step()), "op_graph": graph.replay}
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.iters):
                fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) / args.iters)
    res = {"card": card(), "P": P, "step_ms": {k: stats(v, 1e3) for k, v in times.items()}}
    for folded in (False, True):
        flop = 3 * 2 * macs_per_row(folded) * P  # forward + backward (dX and dW)
        key = "tflops_folded" if folded else "tflops_exavatar_form"
        res[key] = {k: round(flop / statistics.median(v) / 1e12, 1) for k, v in times.items()}
    res["flop_per_step"] = {"exavatar_form": 3 * 2 * macs_per_row(False) * P, "folded": 3 * 2 * macs_per_row(True) * P}
    res["note"] = ("3xTF32 issues three tensor-core MMAs per counted product; H100 SXM data sheet: 495 TFLOP/s TF32 "
                   "dense, 67 TFLOP/s FP32")

    # per-kernel device times of arm 2 (separate profiled run)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            zero()
            op_step()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.count:
            kern[e.key] = round(e.device_time_total / 3 / 1e3, 4)  # ms per step
    res["kernels_ms_per_step"] = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:16])
    if args.trace_dir:
        os.makedirs(args.trace_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.trace_dir, "human_nets_trace.json"))
    res["frame_fps"] = frames_per_second(args, dev, nets, tp, tpf, pose)
    print(json.dumps(res, indent=1))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
