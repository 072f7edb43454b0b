"""animate_view_rot.py's video loop on a trained avatar: the scripts' structure with the repo's ops vs. AvatarAnimator.

  python tools/bench_animator.py [--frames 16] [--rounds 3] [--json out.json] [--profile-dir DIR]

The C4 human (tools/c4_frame.py's SyntheticAvatar: the synthetic SMPL-X rig, P = 167 618 Gaussians, all four GroupNorm
stacks and the triplanes seeded) drives a motion folder of --frames frames written once per size, at 512 x 512 and 1080 x 1920
(portrait: H = 1920, W = 1080).  Every arm goes from the motion to each frame's uint8 (H, 3W, 3) panel on the host,
orbit camera on (animate_view_rot.py; k = 16), in the rasteriser's fixed-capacity mode:
  1. script:  the scripts' structure with the repo's ops -- per frame, the two JSON files and the PNG read on the host
              and uploaded, HumanGaussian's forward through the ops (SyntheticAvatar.full_chain: rig, triplane, all
              four stacks, both sets posed, nearest_rows, VertexNormals, colours), then f-19's ops arm (body_mesh with
              joints, OrbitCamera, orbit_points x 2, device_render_settings, GaussianRasterizer, ShadedMeshRenderer,
              animation_panel) and the panel's copy to the host;
  2. eager:   AvatarAnimator(use_graph=False).frames() over a MotionTable built once;
  3. graph:   AvatarAnimator(use_graph=True, in_flight=2).frames().
Arms alternate pass by pass over the whole motion in one process (host clock around each pass, device synchronised at
both ends): median (min-max) frames/s.  The MotionTable build is timed once per size, outside the arms.  A separate
torch.profiler pass of the eager animator gives each kernel's share of the device time, the mesh panel's (mr_* and the
mesh's vertex normals) among them.  Prints the card name and power limit read in the same run.
"""
import json
import os
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, kernel_events, stats  # noqa: E402
from c4_frame import SyntheticAvatar  # noqa: E402
from exavatar_release_b200 import MotionTable  # noqa: E402
from exavatar_release_b200.animation import OrbitCamera  # noqa: E402
from exavatar_release_b200.human_assets import POSE_KEYS  # noqa: E402
from exavatar_release_b200.rasterizer import set_fixed_capacity  # noqa: E402

SIZES = ((512, 512), (1920, 1080))  # (H, W)
CAPACITY = 1 << 23


class ScriptArm:
    """One pass of animate_view_rot.py's loop in its structure, the repo's ops in place of ExAvatar's modules."""

    def __init__(self, av, root, n, H, W, dev):
        self.av, self.root, self.n, self.H, self.W, self.dev = av, root, n, H, W, dev

    @torch.no_grad()
    def frame(self, i, orbit):
        with open(os.path.join(self.root, "cam_params", f"{i}.json")) as f:
            cam = {k: torch.FloatTensor(v).cuda() for k, v in json.load(f).items()}
        with open(os.path.join(self.root, "smplx_optimized", "smplx_params_smoothed", f"{i}.json")) as f:
            sp = {k: torch.FloatTensor(v).cuda().view(-1) for k, v in json.load(f).items()}
        img = torch.from_numpy(cv2.imread(os.path.join(self.root, "frames", f"{i}.png"))).to(self.dev)
        fr = {"pose": torch.cat([sp[k] for k in POSE_KEYS]).view(-1, 3), "expr": sp["expr"], "trans": sp["trans"],
              "cam": cam, "frame": img}
        return self.av.full_chain(fr, i, (self.H, self.W), orbit)["panel"].cpu().numpy()

    def __call__(self):
        orbit = OrbitCamera(16, self.n, self.dev)
        return [self.frame(i, orbit) for i in range(self.n)]


def main():
    ap = arg_parser(__doc__, iters=None, rounds=3, frames=16)
    ap.add_argument("--profile-dir", default=None, help="also write the profiled pass's kernel table here")
    args = ap.parse_args()
    dev = cuda_device("bench_animator")
    result = {"card": card(), "frames_per_motion": args.frames, "sizes": {}}
    av = SyntheticAvatar(dev)
    set_fixed_capacity(CAPACITY)
    try:
        for H, W in SIZES:
            with tempfile.TemporaryDirectory() as root:
                av.write_motion(root, range(args.frames), H, W)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                motion = MotionTable.from_folder(root, dev)
                torch.cuda.synchronize()
                build_s = time.perf_counter() - t0
                script = ScriptArm(av, root, args.frames, H, W, dev)
                eager = av.animator(motion, orbit=True, capacity=CAPACITY, use_graph=False)
                graph = av.animator(motion, orbit=True, capacity=CAPACITY, in_flight=2)
                runs = {"script": script,
                        "eager": lambda: [p.copy() for _, p in eager.frames()],
                        "graph": lambda: [p.copy() for _, p in graph.frames()]}
                outs = {k: fn() for k, fn in runs.items()}
                same = {k: all(np.array_equal(a, b) for a, b in zip(outs[k], outs["eager"])) for k in outs}
                times = alternate(runs, 1, args.rounds, 1)
                ev, tot = kernel_events(runs["eager"])
                by = {}
                for e in ev:
                    by[e.name] = by.get(e.name, 0.0) + e.device_time / 1e3
                total = sum(by.values())
                mesh = sum(v for k, v in by.items() if "::mr_" in k or "vertex_normals" in k)
                top = sorted(by.items(), key=lambda kv: -kv[1])[:12]
                result["sizes"][f"{H}x{W}"] = {
                    "P": av.rig.P,
                    "frames_per_s": {k: stats([args.frames / s for s in v], 1.0, 2) for k, v in times.items()},
                    "panels_equal_to_eager": same,
                    "motion_table_build_s": round(build_s, 2), "motion_table_mb": round(motion.nbytes / 1e6, 1),
                    "eager_device_ms_per_frame": round(tot["device_ms"] / args.frames, 3),
                    "eager_launches_per_frame": round(tot["launches"] / args.frames, 1),
                    "mesh_panel_share_of_device_time": round(mesh / total, 3),
                    "top_kernels_share": {k[:60]: round(v / total, 3) for k, v in top},
                }
                if args.profile_dir:
                    os.makedirs(args.profile_dir, exist_ok=True)
                    with open(os.path.join(args.profile_dir, f"animator_kernels_{H}x{W}.json"), "w") as f:
                        json.dump({k: v / args.frames for k, v in sorted(by.items(), key=lambda kv: -kv[1])}, f,
                                  indent=1)
                del eager, graph, motion
    finally:
        set_fixed_capacity(None)
    emit(result, args.json)


if __name__ == "__main__":
    main()
