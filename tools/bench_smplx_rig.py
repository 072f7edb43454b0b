"""ExAvatar's SMPL-X rig (avatar/common/nets/module.py:517-518, 533, 537, 549) in PyTorch ops vs. `SmplxRig`.

  python tools/bench_smplx_rig.py [--iters 20] [--rounds 5] [--json out.json]

The rig at C4 size (make_smplx_model on make_human_mesh: V = 10 478, P = 167 618, 55 joints, 100 shape and 50
expression coefficients), forward + backward of a seeded weighted sum of mesh_neutral_pose, joint_mats and expr_offset.
Arms:
  1. ops:       the rig the way ExAvatar runs it, in fp32 torch ops on the device: two body-model forwards (the 大 pose
                with the jaw at zero and the zero pose; shapedirs and expr_dirs concatenated per call, batch_rodrigues,
                the posedirs product, the Python FK loop of 4x4 matmuls, LBS of every vertex), the two-level
                subdivision of the mesh with its edge tables uploaded from the host each call (pytorch3d rebuilds them
                from the uploaded face table; pytorch3d cannot be installed offline), torch.inverse and the rotation
                conversions of the inverse-neutral chain and its FK loop, the frame's FK loop and bmm, the upsampled
                pose_dirs product (9 x 54 x 3P fp32, 977 MB) and mask, and the (P,3,50) broadcast-sum of expr.  The
                SMPL-X layer's landmarks and extra joints are omitted: ExAvatar discards them;
  2. op:        `SmplxRig`, eager;
  3. op_graph:  arm 2 captured once in a CUDA graph and replayed;
  4. frame_*:   C4 training frames/s of tools/c4_frame.py's frame with the rig of arm 1 (frame_rig_ops) or the op
                eager (frame_rig_op) in front.
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Host
syncs per call are counted with torch's sync debug mode ("warn"); device time and launch count per call come from a
separate torch.profiler run.  Prints the card name and power limit with the numbers.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, graph_replay, host_syncs, kernel_events, stats  # noqa: E402
from c4_frame import FrameArm, frames_per_second, rig_ops, setup  # noqa: E402


def main():
    a = arg_parser(__doc__, iters=20, frames=10).parse_args()
    dev = cuda_device("bench_smplx_rig")
    rig, d, x, w = setup(dev)

    def loss(out):
        return (out[0] * w[0]).sum() + (out[2] * w[1]).sum() + (out[4] * w[2]).sum()

    def run_ops(xs=x):
        loss(rig_ops(d, *xs)).backward()

    def run_op(xs=x):
        loss(rig(*xs)).backward()

    with torch.no_grad():
        ref, mine = rig_ops(d, *x), rig(*x)
        names = ("mesh_neutral_pose", "mesh_neutral_pose_wo_upsample", "joint_mats", "pose_offset", "expr_offset",
                 "pose_6d")
        agree = {n: {"max_abs_diff": float((r - o).abs().max()), "max_abs": float(r.abs().max())}
                 for n, r, o in zip(names, ref, mine)}

    xg = [t.detach().clone().requires_grad_() for t in x]
    arms = {"ops": run_ops, "op": run_op, "op_graph": graph_replay(lambda: run_op(xg), 2)}
    times = alternate(arms, a.iters, a.rounds, 1)
    res = {"card": card(), "V": d["V"], "P": d["P"], "J": d["J"],
           "rig_ms": {k: stats(v, 1e3) for k, v in times.items()},
           "host_syncs_per_call": {k: host_syncs(arms[k]) for k in ("ops", "op")},
           "profile": {k: kernel_events(fn)[1] for k, fn in arms.items()}, "ops_vs_op": agree,
           "frames_per_s": frames_per_second(a, dev, {"rig_ops": FrameArm(rig=lambda r, d, x: rig_ops(d, *x)),
                                                      "rig_op": FrameArm()})}
    emit(res, a.json)


if __name__ == "__main__":
    main()
