"""ExAvatar's regulariser block (avatar/main/model.py:217-257) in PyTorch ops vs. `HumanRegularizers`.

  python tools/bench_human_regs.py [--iters 20] [--rounds 5] [--frames 10] [--json out.json]

The block at C4 size (the synthetic 167 618-vertex mesh with make_regs_labels' labels), forward + backward.  Arms:
  1. ops:       the block restated the way ExAvatar runs it -- five weight columns rebuilt with boolean-mask assignments,
                three normal evaluations each uploading the face table from pageable memory, boolean row selections,
                the two host reads of ArmRGBReg and its dense lower x upper matrices with topk, twice.  pytorch3d cannot
                be installed offline, so its `Meshes` normals are replaced by geometry.vertex_normals_reference on the
                device: pytorch3d's own normal kernel is not timed;
  2. op:        `HumanRegularizers`, eager;
  3. op_graph:  arm 2 captured once in a CUDA graph and replayed;
  4. frame_*:   C4 training frames/s of the f-7 human chain (triplane, the GroupNorm stacks as ops, offsets,
                nearest_rows, skin_gaussians, VertexNormals) in front of `TrainingFrameRenderer(use_graph=True)`, then
                `l1_ssim` of the five renders, then the regularisers and the backward: without the block
                (frame_no_regs), with the block of arm 1 (frame_regs_ops) and with the op (frame_regs_op).
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Host
syncs per block are counted under torch.cuda.set_sync_debug_mode("warn"); device time and launch count per block come
from a separate torch.profiler run.  Prints the card name and power limit with the numbers.
"""
import argparse
import json
import math
import os
import statistics
import sys
import time
import warnings

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_frame_sh import card  # noqa: E402
from bench_human_nets import stack  # noqa: E402
from exavatar_release_b200 import HumanRegularizers, TrainingFrameRenderer  # noqa: E402
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.geometry import VertexNormals, nearest_rows, vertex_normals_reference  # noqa: E402
from exavatar_release_b200.human_nets import TriplaneFeatures, gn_mlp  # noqa: E402
from exavatar_release_b200.losses import l1_ssim  # noqa: E402
from exavatar_release_b200.plan import RENDERS  # noqa: E402
from exavatar_release_b200.regularizers import KEYS  # noqa: E402
from exavatar_release_b200.skinning import skin_gaussians  # noqa: E402
from exavatar_release_b200.synthetic import (WORKLOADS, Workload, make_human_mesh, make_population_assets,  # noqa: E402
                                             make_regs_labels)

# SMPL-X's joint names as the golden generator read them from the reference
JOINTS = [str(n) for n in np.load(os.path.join(ROOT, "tests", "golden", "regs.npz"))["joints_name"]]

INPUTS = ("mean_offset", "mean_offset_offset", "scale_offset", "scale", "scale_refined", "rgb", "rgb_refined",
          "joint_offset")


def block_ops(d, x):
    """model.py:217-257 with loss.py's classes, restated in torch ops on the device (batch 1)."""
    P = d["P"]
    mnp = d["mesh"]
    mo, moo, so = x["mean_offset"][None], x["mean_offset_offset"][None], x["scale_offset"][None]
    s, sr, rgb, rgbr = x["scale"][None], x["scale_refined"][None], x["rgb"][None], x["rgb_refined"][None]
    r, l, f, e, c = (d[k] for k in ("is_rhand", "is_lhand", "is_face", "is_face_expr", "is_cavity"))

    def normals():  # Meshes(verts, torch.LongTensor(face_upsampled).cuda()).verts_normals_packed()
        faces = torch.LongTensor(d["faces_np"]).cuda()
        return vertex_normals_reference(mnp, faces, dtype=torch.float32)

    def lap(v):
        return v + (v[:, d["nbr"]] * d["nbr_w"][None, :, :, None]).sum(2)

    def hand_mean(o):
        is_hand = (r + l) > 0
        with torch.no_grad():
            n = normals().reshape(1, P, 3)
        return torch.clamp(torch.sum(n * F.normalize(o, p=2, dim=2), 2)[:, is_hand], min=0)

    def hand_rgb(v):
        return (v[:, r, :] - v[:, r, :].mean(1)[:, None, :].detach()) ** 2 + \
               (v[:, l, :] - v[:, l, :].mean(1)[:, None, :].detach()) ** 2

    def arm_rgb(up, lo, v):
        mu, ml = mnp[up, :], mnp[lo, :]
        dist_x = torch.abs(ml[:, None, 0] - mu[None, :, 0])
        mask = (dist_x < 0.01).float()
        valid = int(torch.min(mask.sum(1)))
        dist = torch.sqrt(torch.sum((ml[:, None, :] - mu[None, :, :]) ** 2, 2))
        dist = dist * mask + 9999 * (1 - mask)
        k = min(50, valid)
        idxs = torch.topk(dist, k=k, dim=1, largest=False, sorted=False)[1]
        ui = torch.arange(P).long().cuda()[up][idxs].view(-1)
        return (v[:, lo, :] - v[:, ui, :].view(1, int(lo.sum()), k, 3).mean(2).detach()) ** 2

    loss = {}
    w = torch.ones((1, P, 1)).float().cuda() * 10
    w[:, r, :] = 1000
    w[:, l, :] = 1000
    w[:, f, :] = 1
    w[:, e, :] = 10
    loss["gaussian_mean_reg"] = (mo ** 2 + moo ** 2) * w
    loss["gaussian_mean_hand_reg"] = hand_mean(mo) + hand_mean(moo)
    w = torch.ones((1, P, 1)).float().cuda()
    w[:, r, :] = 1000
    w[:, l, :] = 1000
    w[:, e, :] = 10
    w[:, c, :] = 0
    loss["gaussian_scale_reg"] = (s ** 2 + so ** 2) * w
    w = torch.ones((1, P, 1)).float().cuda()
    w[:, e, :] = 50
    w[:, c, :] = 0.1
    base = mnp[None].detach()
    loss["lap_mean"] = ((lap(base + mo) - lap(base)) ** 2 + (lap(base + mo + moo) - lap(base)) ** 2) * 100000 * w
    w = torch.ones((1, P, 1)).float().cuda() * 10
    w[:, r, :] = 10
    w[:, l, :] = 10
    w[:, e, :] = 0
    loss["lap_scale"] = (lap(s) ** 2 + lap(sr) ** 2) * 100000 * w
    w = torch.ones((1, P, 1)).float().cuda() * 0.1
    w[:, r, :] = 100
    w[:, l, :] = 100
    loss["lap_rgb"] = (lap(rgb) ** 2 + lap(rgbr) ** 2) * w
    loss["hand_rgb_reg"] = (hand_rgb(rgb) + hand_rgb(rgbr)) * 0.01
    n = normals().detach()  # smpl_x.get_arm
    up = d["is_arm"] * (n[:, 1] > math.cos(math.pi / 3))
    lo = d["is_arm"] * (n[:, 1] <= math.cos(math.pi / 3))
    loss["arm_rgb_reg"] = (arm_rgb(up, lo, rgb) + arm_rgb(up, lo, rgbr)) * 0.1
    jw = torch.ones((55, 3)).float().cuda()
    jw[d["hand_joints"], :] = 10
    jo = x["joint_offset"]
    loss["joint_offset_reg"] = (jo - d["joint_target"].cuda()) ** 2 * jw
    ri, li = [], []
    for j in range(55):  # JointOffsetSymmetricReg rebuilds its Python lists every call
        if d["names"][j][:2] == "R_":
            ri.append(j)
            li.append(d["names"].index("L_" + d["names"][j][2:]))
    loss["joint_offset_sym_reg"] = torch.abs(jo[ri, 0] + jo[li, 0]) + torch.abs(jo[ri, 1] - jo[li, 1]) + \
        torch.abs(jo[ri, 2] - jo[li, 2])
    return {k: v.mean() for k, v in loss.items()}


def setup(dev):
    from exavatar_release_b200.regularizers import laplacian_table
    m = make_human_mesh()
    P = m["verts"].shape[0]
    lab = make_regs_labels(m)
    names = JOINTS
    hand = [i for i, n in enumerate(names) if n[2:].split("_")[0] in ("Index", "Middle", "Pinky", "Ring", "Thumb")]
    right = [j for j in range(55) if names[j][:2] == "R_"]
    left = [names.index("L_" + names[j][2:]) for j in right]
    g = torch.Generator().manual_seed(1)
    target = 1e-2 * torch.randn(55, 3, generator=g)
    nbr, nbr_w = laplacian_table(m["faces"].numpy(), P)
    d = {"P": P, "mesh": m["verts"].to(dev), "m": m, "faces_np": m["faces"].numpy(), "names": names, "hand_joints": hand,
         "joint_target": target, "nbr": torch.from_numpy(nbr).to(dev), "nbr_w": torch.from_numpy(nbr_w).to(dev),
         **{k: v.to(dev) for k, v in lab.items()}}
    regs = HumanRegularizers(m["faces"], P, device=dev, **{k: v.to(dev) for k, v in lab.items()},
                             joint_offset_target=target, hand_joints=hand, sym_pairs=(right, left))
    x = {"mean_offset": 1e-3 * torch.randn(P, 3, generator=g), "mean_offset_offset": 5e-4 * torch.randn(P, 3, generator=g),
         "scale_offset": 1e-2 * torch.randn(P, 1, generator=g),
         "scale": torch.exp(-5.5 + 0.3 * torch.randn(P, 3, generator=g)),
         "scale_refined": torch.exp(-5.5 + 0.3 * torch.randn(P, 3, generator=g)),
         "rgb": torch.rand(P, 3, generator=g), "rgb_refined": torch.rand(P, 3, generator=g),
         "joint_offset": 1e-2 * torch.randn(55, 3, generator=g)}
    x = {k: v.to(dev).requires_grad_() for k, v in x.items()}
    return d, regs, x


def frames_per_second(a, dev, d, regs):
    """C4 training frames/s: the f-7 human chain, TrainingFrameRenderer(use_graph=True), l1_ssim of the five renders,
    then no regulariser block, the block in PyTorch ops, or the op; one backward per frame."""
    m, P = d["m"], d["P"]
    c4 = WORKLOADS["C4"]
    H, W = c4.height, c4.width
    wl = Workload("C4 with the synthetic mesh's Gaussians", H, W, P, c4.n_scene, 0, True)
    scene, human, _ = make_population_assets(wl, seed=0, device=dev)
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    R, tc = cam["R"], cam["t"]
    to_cam = lambda v: (v.to(dev) @ R.t() + tc.view(1, 3)).contiguous()  # noqa: E731
    canon, targets, sm = to_cam(m["queries"]), to_cam(m["targets"]), m["self_map"].to(dev)
    verts = d["mesh"]
    tri = TriplaneFeatures(verts, verts[:, 1] > 0.6)
    vn = VertexNormals(m["faces"], P, flip=m["flip"].to(dev))
    torch.manual_seed(3)
    nets = {"geo": stack(96, [3, 1]), "geo_offset": stack(96 + 126, [3, 1]), "rgb": stack(96, None, 3),
            "rgb_offset": stack(96 + 126 + 3, None, 3)}
    g = torch.Generator().manual_seed(5)
    tp = (0.3 * torch.randn((3, 32, 128, 128), generator=g)).to(dev).requires_grad_()
    tpf = (0.3 * torch.randn((3, 32, 128, 128), generator=g)).to(dev).requires_grad_()
    pose = (0.5 * torch.randn(126, generator=g)).to(dev)
    table = torch.zeros(P, 55)
    table.scatter_(1, torch.rand(P, 55, generator=g).topk(4, dim=1).indices, torch.full((P, 4), 0.25))
    table = table.to(dev)
    A = torch.eye(4).repeat(55, 1, 1).to(dev)
    A[:, :3, 3] = 0.01 * torch.randn(55, 3, generator=g).to(dev)
    A.requires_grad_()
    tr = torch.zeros(3, device=dev, requires_grad=True)
    jo = (1e-2 * torch.randn(55, 3, generator=g)).to(dev).requires_grad_()
    lv = {k: v.detach().clone().requires_grad_() for k, v in scene.items()}
    bg = torch.tensor([0.3, 0.7, 0.2], device=dev)
    target = torch.rand((3, H, W), generator=torch.Generator(device=dev).manual_seed(6), device=dev)
    fr = TrainingFrameRenderer(scene["mean_3d"].shape[0], P, (H, W), dev, {"A": 8_000_000, "B": 8_000_000},
                               use_graph=True)
    leaves = [tp, tpf, A, tr, jo, *lv.values()] + [p for t, hs in nets.values() for mm in [t, *hs]
                                                   for p in mm.parameters()]

    def frame(which):
        f = tri(tp, tpf)
        net = lambda k, ins: gn_mlp(ins, *nets[k])  # noqa: E731
        geo, geo_off, rgb = net("geo", [f]), net("geo_offset", [f, pose]), net("rgb", [f])
        mean_3d = canon + 0.01 * geo[:, :3]
        mean_3d_r = mean_3d + 0.005 * geo_off[:, :3]
        rows = nearest_rows(mean_3d.detach(), targets, sm)
        posed, posed_r = skin_gaussians(mean_3d, mean_3d_r, table, rows, A, tr, R, tc)
        rgb_off = net("rgb_offset", [f, pose, vn(posed_r)])
        x = {"mean_offset": 0.01 * geo[:, :3], "mean_offset_offset": 0.005 * geo_off[:, :3],
             "scale_offset": 0.1 * geo_off[:, 3:], "scale": human["scale"] * torch.exp(0.1 * geo[:, 3:]),
             "scale_refined": human["scale"] * torch.exp(0.1 * (geo[:, 3:] + geo_off[:, 3:])),
             "rgb": (torch.tanh(rgb) + 1) / 2, "rgb_refined": (torch.tanh(rgb + rgb_off) + 1) / 2, "joint_offset": jo}
        hv = dict(human, mean_3d=posed, scale=x["scale"], rgb=x["rgb"])
        rv = dict(human, mean_3d=posed_r, scale=x["scale_refined"], rgb=x["rgb_refined"])
        out = fr(lv, hv, rv, cam, bg)
        loss = 0
        for r in RENDERS:
            l1, ss = l1_ssim(out[r]["img"], target)
            loss = loss + 0.8 * l1 + 0.2 * (1 - ss)
        if which == "regs_ops":
            loss = loss + sum(block_ops(d, x).values())
        elif which == "regs_op":
            loss = loss + sum(regs(verts, *[x[k] for k in INPUTS]).values())
        loss.backward()
        for v in leaves:
            v.grad = None

    arms = ("no_regs", "regs_ops", "regs_op")
    for k in arms:
        for _ in range(3):
            frame(k)
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k in arms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.frames):
                frame(k)
            torch.cuda.synchronize()
            times[k].append(a.frames / (time.perf_counter() - t0))
    if fr.overflowed():
        raise SystemExit("bench_human_regs: a render overflowed its list capacity")
    return {f"frame_{k}": {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="block calls per timed window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=10, help="training frames per timed window")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_human_regs: needs a CUDA device (there is no CPU measurement)")
    dev = torch.device("cuda:0")
    d, regs, x = setup(dev)

    def run_ops():
        sum(block_ops(d, x).values()).backward()

    def run_op(xs=x):
        sum(regs(d["mesh"], *[xs[k] for k in INPUTS]).values()).backward()

    with torch.no_grad():
        ref = block_ops(d, x)
        mine = regs(d["mesh"], *[x[k] for k in INPUTS])
        agree = {k: [float(ref[k]), float(mine[k])] for k in KEYS}

    # the graph arm owns its leaves, so no autograd node of the eager arms is kept alive into the capture
    xg = {k: v.detach().clone().requires_grad_() for k, v in x.items()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            run_op(xg)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run_op(xg)
    arms = {"ops": run_ops, "op": run_op, "op_graph": graph.replay}
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(a.iters):
                fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t) / a.iters * 1e3)

    syncs = {}
    for k in ("ops", "op"):
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                arms[k]()
            finally:
                torch.cuda.set_sync_debug_mode(0)
        syncs[k] = sum("synchroniz" in str(m.message).lower() for m in w)

    prof = {}
    from torch.profiler import ProfilerActivity, profile
    for k, fn in arms.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            fn()
            torch.cuda.synchronize()
        ev = [e for e in p.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name
              and "Memset" not in e.name]
        prof[k] = {"device_ms": sum(e.device_time for e in ev) / 1e3, "launches": len(ev)}

    res = {"card": card(), "P": d["P"],
           "block_ms": {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()},
           "host_syncs_per_block": syncs, "profile": prof, "values_ops_vs_op": agree,
           "frames_per_s": frames_per_second(a, dev, d, regs)}
    print(json.dumps(res, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
