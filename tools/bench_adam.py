"""ExAvatar's optimizer step (avatar/common/base.py:83-85, train.py:57) with torch.optim.Adam vs. `optim.Adam`.

  python tools/bench_adam.py [--steps 20] [--rounds 5] [--frames 1 100 1000] [--json out.json]

Workload: ExAvatar's group layout at C4 size -- the six scene groups at P_scene = 130 000 with SH degree 3, the two
(3,32,128,128) triplanes and the eight network groups sized as in tools/bench_human_nets.py, shape_param and
joint_offset, and N_frames SMPL-X frames of nine groups each; every step one frame (in turn) has gradients and the
others' are None, as with batch_size = 1.  Arms, alternated window by window in one process:
  1. foreach: torch.optim.Adam(eps=1e-15), ExAvatar's default;
  2. fused:   torch.optim.Adam(eps=1e-15, fused=True), for context only: a different formulation, so after the run its
              largest difference from arm 1 is reported rather than assumed zero; it refuses the strided feature
              views, so this arm gets contiguous copies of them;
  3. op:      optim.Adam(eps=1e-15); after the run it must equal arm 1 bit for bit.
The two feature groups are views of one (P,16,3) tensor, as SceneGaussian.init_from_point_cloud makes them.
Per arm: the host wall time of step() (the call alone), the step time to a device synchronise (the window's step() calls
plus the wait for the sync at its end; the gradient assignment between steps is not timed), and from a separate torch.profiler run the device time and launches per step.  For the op also its
algorithmic bytes (28 B per element: p, g, m, v read, p, m, v written), achieved bandwidth and share of 3.35 TB/s (the
H100 SXM data sheet's HBM3 figure).  Prints the card name and power limit with the numbers.
"""
import os
import sys
import time

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import HBM_BYTES_PER_S, arg_parser, card, cuda_device, emit, stats  # noqa: E402
from exavatar_release_b200.optim import Adam  # noqa: E402

FRAME_PARAMS = {"root_pose": (6,), "body_pose": (21, 6), "jaw_pose": (6,), "leye_pose": (6,), "reye_pose": (6,),
                "lhand_pose": (15, 6), "rhand_pose": (15, 6), "expr": (50,), "trans": (3,)}


def trunk(k_in, final=None):
    shapes = []
    for k in (k_in, 128, 128):
        shapes += [(128, k), (128,), (128,), (128,)]  # Linear weight, bias; GroupNorm weight, bias
    return shapes + ([(final, 128), (final,)] if final else [])


def layout(n_scene, n_frames):
    """(name, [shape], lr) of ExAvatar's groups: module.py:143-148 (scene), 322-333 (human), 666-671 (SMPL-X)."""
    P = n_scene
    groups = [("mean_scene", [(P, 3)], 4e-4), ("feature_dc_scene", [(P, 1, 3)], 2.5e-3),
              ("feature_rest_scene", [(P, 15, 3)], 2.5e-3 / 20), ("opacity_scene", [(P, 1)], 0.05),
              ("scale_scene", [(P, 3)], 5e-3), ("rotation_scene", [(P, 4)], 1e-3),
              ("triplane_human", [(3, 32, 128, 128)], 1e-3), ("triplane_face_human", [(3, 32, 128, 128)], 1e-3),
              ("geo_net_human", trunk(96), 1e-3), ("mean_offset_net_human", [(3, 128), (3,)], 1e-3),
              ("scale_net_human", [(1, 128), (1,)], 1e-3), ("geo_offset_net_human", trunk(96 + 126), 1e-3),
              ("mean_offset_offset_net_human", [(3, 128), (3,)], 1e-3),
              ("scale_offset_net_human", [(1, 128), (1,)], 1e-3), ("rgb_net_human", trunk(96, 3), 1e-3),
              ("rgb_offset_net_human", trunk(96 + 126 + 3, 3), 1e-3), ("shape_param_human", [(100,)], 1e-3),
              ("joint_offset_human", [(55, 3)], 1e-3)]
    return groups + [(f"smplx_{k}_{f}", [s], 1e-3) for f in range(n_frames) for k, s in FRAME_PARAMS.items()]


class Arm:
    def __init__(self, kind, spec, values, grads, n_frames):
        # same sizes and strides as `values`: the two feature groups stay views of one (P,16,3) tensor, except for
        # torch's fused kernel, which refuses params whose layout differs from their grads'
        like = (lambda v: v.clone(memory_format=torch.contiguous_format)) if kind == "fused" else (
            lambda v: torch.empty_strided(v.shape, v.stride(), device=v.device).copy_(v))
        groups = [{"params": [nn.Parameter(like(v)) for v in vs], "name": name, "lr": lr}
                  for (name, _, lr), vs in zip(spec, values)]
        if kind == "op":
            self.opt = Adam(groups, lr=0.0, eps=1e-15)
        else:
            # fused=False would select torch's single-tensor path, not ExAvatar's default foreach one
            self.opt = torch.optim.Adam(groups, lr=0.0, eps=1e-15, **({"fused": True} if kind == "fused" else {}))
        self.grads, self.n_frames, self.i = grads, n_frames, 0
        # the SMPL-X frame of each group; None: a group that has a gradient every step
        self.frame_of = [gr["name"].rsplit("_", 1)[-1] if gr["name"].startswith("smplx") else None
                         for gr in self.opt.param_groups]

    def set_grads(self):
        f = str(self.i % self.n_frames)
        for gr, fr, gs in zip(self.opt.param_groups, self.frame_of, self.grads):
            on = fr is None or fr == f
            for p, g in zip(gr["params"], gs):
                p.grad = g if on else None
        self.i += 1

    def elems_with_grad(self):
        return sum(p.numel() for gr in self.opt.param_groups for p in gr["params"] if p.grad is not None)


def run(n_frames, a, dev):
    spec = layout(a.scene, n_frames)
    gen = torch.Generator(device=dev).manual_seed(0)
    values = [[0.1 * torch.randn(s, device=dev, generator=gen) for s in shapes] for _, shapes, _ in spec]
    # SceneGaussian.init_from_point_cloud (module.py:106-107): feature_dc and feature_rest are views of one tensor
    feature = 0.1 * torch.randn((a.scene, 16, 3), device=dev, generator=gen)
    values[1], values[2] = [feature[:, 0:1, :]], [feature[:, 1:, :]]
    grads = [[torch.randn(s, device=dev, generator=gen) for s in shapes] for _, shapes, _ in spec]
    arms = {k: Arm(k, spec, values, grads, n_frames) for k in ("foreach", "fused", "op")}
    for arm in arms.values():
        for _ in range(3):
            arm.set_grads()
            arm.opt.step()
    torch.cuda.synchronize()
    host = {k: [] for k in arms}
    step_ms = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, arm in arms.items():
            torch.cuda.synchronize()
            h = 0.0
            for _ in range(a.steps):
                arm.set_grads()  # not timed: a walk over every group that belongs to the harness, not to the step
                t1 = time.perf_counter()
                arm.opt.step()
                h += time.perf_counter() - t1
            t1 = time.perf_counter()
            torch.cuda.synchronize()
            step_ms[k].append((h + time.perf_counter() - t1) / a.steps * 1e3)
            host[k].append(h / a.steps * 1e3)
    torch.cuda.synchronize()

    def pdiff(x, y):
        return max(float((p - q).abs().max()) for gx, gy in zip(x.opt.param_groups, y.opt.param_groups)
                   for p, q in zip(gx["params"], gy["params"]) if p.numel())

    def pequal(x, y):
        return all(torch.equal(p.view(torch.int32), q.view(torch.int32))
                   for gx, gy in zip(x.opt.param_groups, y.opt.param_groups) for p, q in zip(gx["params"], gy["params"]))

    agree = {"op_bitwise_equal_foreach": pequal(arms["op"], arms["foreach"]),
             "fused_max_abs_diff_vs_foreach": pdiff(arms["fused"], arms["foreach"])}

    from torch.profiler import ProfilerActivity, profile
    prof = {}
    for k, arm in arms.items():
        arm.set_grads()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            arm.opt.step()
            torch.cuda.synchronize()
        ev = [e for e in p.events() if e.device_type.name == "CUDA"]
        kern = [e for e in ev if "Memcpy" not in e.name and "Memset" not in e.name]
        prof[k] = {"device_ms": sum(e.device_time for e in kern) / 1e3, "launches": len(kern),
                   "copies": len(ev) - len(kern)}
        if k == "op":
            elems = arm.elems_with_grad()
            kms = sum(e.device_time for e in kern if "adam_step_kernel" in e.name) / 1e3
            nbytes = 28 * elems
            prof[k].update(elements=elems, algorithmic_bytes=nbytes, kernel_ms=kms,
                           achieved_TBps=nbytes / (kms * 1e-3) / 1e12 if kms else None,
                           share_of_hbm=nbytes / (kms * 1e-3) / HBM_BYTES_PER_S if kms else None)
    return {"groups": len(spec), "host_step_ms": {k: stats(v) for k, v in host.items()},
            "step_to_sync_ms": {k: stats(v) for k, v in step_ms.items()}, "profile": prof, "agreement": agree}


def main():
    ap = arg_parser(__doc__, iters=None)
    ap.add_argument("--steps", type=int, default=20, help="optimizer steps per timed window")
    ap.add_argument("--scene", type=int, default=130_000)
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 100, 1000], help="SMPL-X frames in the layout")
    a = ap.parse_args()
    dev = cuda_device("bench_adam")
    res = {"card": card(), "scene": a.scene, "by_frames": {n: run(n, a, dev) for n in a.frames}}
    emit(res, a.json)


if __name__ == "__main__":
    main()
