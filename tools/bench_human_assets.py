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
  4. frame_*:   C4 training frames/s of tools/c4_frame.py's frame with the rig's pose decoded every frame from
                the frame's 6D parameters by arm 1's route (frame_decode_exavatar) or by the op (frame_decode_op).
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Host
syncs per call are counted with torch's sync debug mode ("warn"); device time and launches per call come from a
separate torch.profiler run.  Prints the card name and power limit with the numbers.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, graph_replay, host_syncs, kernel_events, stats  # noqa: E402
from c4_frame import FrameArm, frames_per_second  # noqa: E402
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
    a = arg_parser(__doc__, iters=20, frames=10).parse_args()
    dev = cuda_device("bench_human_assets")
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
    arms = {"exavatar": run_exavatar, "op": run_op, "op_graph": graph_replay(lambda: run_op(pg, xg), 2)}
    times = alternate(arms, a.iters, a.rounds, 1)
    syncs = {k: host_syncs(arms[k]) for k in ("exavatar", "op")}

    prof = {}
    for k, fn in arms.items():
        ev, prof[k] = kernel_events(fn)
        prof[k]["kernels"] = sorted({e.name for e in ev if "human" in e.name or "decode_pose" in e.name})

    fp = pose_params(dev, seed=2)

    def decode_arm(decode):
        def pose_rig(rig, d, x):
            for v in fp.values():
                v.grad = None
            return rig(x[0], x[1], decode(fp)["full_pose"], x[3])
        return FrameArm(rig=pose_rig)

    res = {"card": card(), "P": P, "joints": 55,
           "ms_per_call": {k: stats(v, 1e3) for k, v in times.items()},
           "host_syncs_per_call": syncs, "profile": prof, "exavatar_vs_op": agree,
           "frames_per_s": frames_per_second(a, dev, {"decode_exavatar": decode_arm(decode_smplx_pose_reference),
                                                      "decode_op": decode_arm(decode_smplx_pose)})}
    emit(res, a.json)


if __name__ == "__main__":
    main()
