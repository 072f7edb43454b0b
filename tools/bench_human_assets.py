"""ExAvatar's per-frame pose decode (SMPLXParamDict.forward, module.py:673-684) and HumanGaussian's code around its
networks (module.py:524-539, 561-565, model.py:92-96) the way ExAvatar computes them vs. `decode_smplx_pose` and
`HumanAssets`.

  python tools/bench_human_assets.py [--iters 20] [--rounds 5] [--frames 10] [--json out.json]

C4 size (P = 167 618, 55 joints), warm-up clamp on, forward + backward of a seeded weighted sum of the axis-angle pose
and every asset output.  Arms:
  1. exavatar:  pytorch3d's matrix_to_axis_angle(rotation_6d_to_matrix(p)) per pose key as this project restates it
                (its boolean-mask indexings read the device from the host), then the torch lines around the networks
                in ExAvatar's fp32 operations, with line 564's per-frame matrix_to_quaternion of P identity matrices;
  2. op:        `decode_smplx_pose` + `HumanAssets.geometry` / `.colors`, eager;
  3. op_graph:  arm 2 captured once in a CUDA graph and replayed;
  4. frame_*:   C4 training frames/s of tools/bench_smplx_rig.py's frame with the rig's pose decoded every frame from
                the frame's 6D parameters by arm 1's route (frame_decode_exavatar) or by the op (frame_decode_op).
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Host
syncs per call are counted with torch's sync debug mode ("warn"); device time and launches per call come from a
separate torch.profiler run.  Prints the card name and power limit with the numbers.
"""
import argparse
import json
import os
import statistics
import sys
import time
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_frame_sh import card  # noqa: E402
from exavatar_release_b200 import HumanAssets, decode_smplx_pose  # noqa: E402
from exavatar_release_b200.human_assets import (POSE_KEYS, POSE_ROWS, constant_rotation_reference,  # noqa: E402
                                                decode_smplx_pose_reference, human_colors_reference,
                                                human_geometry_reference)
from exavatar_release_b200.smplx_rig import axis_angle_to_matrix, matrix_to_rotation_6d  # noqa: E402

P = 167618


def pose_params(dev, seed=0):
    """One frame's 6D parameters as ExAvatar stores them: (6,) for root / jaw / eyes, (n,6) otherwise."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, n in zip(POSE_KEYS, POSE_ROWS):
        p = matrix_to_rotation_6d(axis_angle_to_matrix(0.3 * torch.randn(n, 3, generator=g)))
        out[k] = (p[0] if n == 1 else p).to(dev).requires_grad_()
    return out


def exavatar_form(params, mesh, pose_offset, expr_offset, geo, geo_offset, rgb, rgb_offset, mask):
    """Arm 1: the reference's route, from this project's restatements, in fp32 on the device."""
    sp = decode_smplx_pose_reference(params)
    a = human_geometry_reference(mesh, pose_offset, expr_offset, geo, geo_offset, mask, warmup=True)
    a["rgb"], a["rgb_refined"] = human_colors_reference(rgb, rgb_offset)
    a["rotation"] = constant_rotation_reference(mesh.shape[0], torch.float32, mesh.device)
    a["opacity"] = torch.ones((mesh.shape[0], 1), device=mesh.device)
    return sp["full_pose"], a


def op_form(ha, params, mesh, pose_offset, expr_offset, geo, geo_offset, rgb, rgb_offset):
    sp = decode_smplx_pose(params)
    a = ha.geometry(mesh, pose_offset, expr_offset, geo, geo_offset, warmup=True)
    a["rgb"], a["rgb_refined"] = ha.colors(rgb, rgb_offset)
    return sp["full_pose"], a


KEYS = ("mean_3d", "mean_3d_refined", "scale", "scale_refined", "mean_offset_offset", "scale_wo_clamp",
        "scale_refined_wo_clamp", "rgb", "rgb_refined")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="calls per timed window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=10, help="training frames per timed window")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_human_assets: needs a CUDA device (there is no CPU measurement)")
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(1)
    mask = torch.zeros(P, dtype=torch.bool)
    mask[torch.randperm(P, generator=g)[:P // 3]] = True
    mask = mask.to(dev)
    ha = HumanAssets(mask, torch.zeros_like(mask), torch.zeros_like(mask))
    r = lambda *s: torch.randn(*s, generator=g).to(dev)  # noqa: E731
    ins = [r(P, 3), 0.01 * r(P, 3) * mask[:, None], 0.01 * r(P, 3),
           torch.cat([0.01 * r(P, 3), -6.9 + 0.5 * r(P, 1)], 1), torch.cat([0.005 * r(P, 3), 0.3 * r(P, 1)], 1),
           r(P, 3), 0.2 * r(P, 3)]
    ins = [t.requires_grad_() for t in ins]
    ins[1].requires_grad_(False)  # the rig's pose offset carries no gradient
    params = pose_params(dev)
    w = [r(P, 3) for _ in KEYS]
    wp = r(55, 3)

    def loss(full_pose, assets):
        return (full_pose * wp).sum() + sum((assets[k] * wk).sum() for k, wk in zip(KEYS, w))

    def run_exavatar(ps=params, xs=ins):
        loss(*exavatar_form(ps, *xs, mask)).backward()

    def run_op(ps=params, xs=ins):
        loss(*op_form(ha, ps, *xs)).backward()

    with torch.no_grad():
        fe, ae = exavatar_form(params, *ins, mask)
        fo, ao = op_form(ha, params, *ins)
        agree = {"full_pose_max_abs_diff": float((fe - fo).abs().max()),
                 "assets_bit_identical": all(torch.equal(ae[k], ao[k]) for k in KEYS),
                 "rotation_equal": bool(torch.equal(ae["rotation"], ha.rotation))}

    pg = {k: v.detach().clone().requires_grad_() for k, v in params.items()}
    xg = [t.detach().clone().requires_grad_(t.requires_grad) for t in ins]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            run_op(pg, xg)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run_op(pg, xg)
    arms = {"exavatar": run_exavatar, "op": run_op, "op_graph": graph.replay}
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
    for k in ("exavatar", "op"):
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                arms[k]()
            finally:
                torch.cuda.set_sync_debug_mode(0)
        syncs[k] = sum("synchroniz" in str(m.message).lower() for m in caught)

    prof = {}
    from torch.profiler import ProfilerActivity, profile
    for k, fn in arms.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            fn()
            torch.cuda.synchronize()
        ev = [e for e in p.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name
              and "Memset" not in e.name]
        prof[k] = {"device_ms": sum(e.device_time for e in ev) / 1e3, "launches": len(ev),
                   "kernels": sorted({e.name for e in ev if "human" in e.name or "decode_pose" in e.name})}

    from bench_smplx_rig import frames_per_second
    fp = pose_params(dev, seed=2)

    def decode(form):
        def fn():
            for v in fp.values():
                v.grad = None
            return decode_smplx_pose_reference(fp)["full_pose"] if form == "exavatar" else \
                decode_smplx_pose(fp)["full_pose"]
        return fn

    res = {"card": card(), "P": P, "joints": 55,
           "ms_per_call": {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()},
           "host_syncs_per_call": syncs, "profile": prof, "exavatar_vs_op": agree,
           "frames_per_s": frames_per_second(a, dev, poses={"decode_exavatar": decode("exavatar"),
                                                            "decode_op": decode("op")})}
    print(json.dumps(res, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
