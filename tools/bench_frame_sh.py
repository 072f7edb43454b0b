"""SURVEY.md section 8f-4 inside the merged training frame: caller-side vs in-kernel SH colour of the scene Gaussians.

  python tools/bench_frame_sh.py [--workload C4] [--frames 30] [--rounds 5] [--json out.json]

One ExAvatar training frame (avatar/main/model.py:117-162: five renders, forward + backward into every parameter) through
`TrainingFrameRenderer`, scene of BASELINE configs[3] with degree-3 SH coefficients (synthetic.make_scene_sh_params):
  (a) caller-side colour: `scene_gaussian_assets(in_kernel_sh=False)` -- view direction, SH polynomial, clamp in PyTorch
      with autograd -- feeding `rgb` to the renderer;
  (b) in-kernel colour:   `scene_gaussian_assets(in_kernel_sh=True)` feeding `shs` + `sh_degree` (sh_coeffs=16).
Both arms include the activations of `SceneGaussian.forward` (sigmoid, exp, cat of the SH features).  Frames/s, eager
and use_graph=True, arms alternated round by round in one process (host clock around N frames + device sync).  Then the
in-library CUDA-event profiler (profiling run of its own) gives K1 (project) and K6 (project_bwd) per merged pass.
Prints the card name and power limit with the numbers.
"""
import ctypes as C
import os
import statistics
import sys
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, stats  # noqa: E402
from exavatar_release_b200 import TrainingFrameRenderer  # noqa: E402
from exavatar_release_b200 import _lib as L  # noqa: E402
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.plan import RENDERS, MergedFivePlan  # noqa: E402
from exavatar_release_b200.renderer import render_settings, scene_gaussian_assets  # noqa: E402
from exavatar_release_b200.sh import sh_to_rgb  # noqa: E402
from exavatar_release_b200.synthetic import WORKLOADS, make_grad_image, make_population_assets, make_scene_sh_params  # noqa: E402

ARMS = {"a_caller_rgb": False, "b_in_kernel_sh": True}
L_NUM = 9  # B2R_NUM_KERNELS: kernel ids 0 project (K1) ... 7 project_bwd (K6)


def main():
    ap = arg_parser(__doc__, iters=None, frames=30)
    ap.add_argument("--workload", default="C4")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile-frames", type=int, default=10)
    a = ap.parse_args()
    dev = cuda_device("bench_frame_sh")
    lib = L.load()
    wl = WORKLOADS[a.workload]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets(a.workload, seed=0, device=dev)
    p = make_scene_sh_params(scene, 3, seed=0)
    Ps, Ph = scene["mean_3d"].shape[0], human["mean_3d"].shape[0]
    deg = 3
    cams = [look_at_cam_param(y, (H, W), device=dev) for y in (-8.0, -3.0, 2.0, 7.0)]
    bg_r = torch.tensor([0.3, 0.7, 0.2], device=dev)
    g5 = {r: make_grad_image(a.workload, 10 + j, device=dev) for j, r in enumerate(RENDERS)}
    lv = {"scene": {k: v.detach().clone().requires_grad_() for k, v in p.items()},
          "human": {k: v.detach().clone().requires_grad_() for k, v in human.items()},
          "refined": {k: v.detach().clone().requires_grad_() for k, v in refined.items()}}
    leaves = [t for d in lv.values() for t in d.values()]

    # duplicate capacities from one generous frame (same lists in both arms: colour does not enter binning)
    probe = MergedFivePlan(Ps, Ph, W, H, None, dev)
    probe.set_scene(scene)
    need = {"A": 0, "B": 0}
    for cam in cams:
        st_w = render_settings((H, W), cam, torch.ones(3, device=dev))
        probe.frame(None, st_w, st_w._replace(bg=bg_r), scene, human, refined, g5, accumulate=False)
        torch.cuda.synchronize()
        need = {k: max(need[k], v) for k, v in probe.dups().items()}
    del probe
    torch.cuda.empty_cache()
    caps = {k: int(v * 1.1) + 4096 for k, v in need.items()}

    def step(fr, sh, cam):
        s = lv["scene"]
        assets = scene_gaussian_assets(s["mean"], s["opacity_logit"], s["log_scale"], s["rotation"], s["feature_dc"],
                                       s["feature_rest"], deg, cam, in_kernel_sh=sh)
        out = fr(assets, lv["human"], lv["refined"], cam, bg_r)
        sum((out[r]["img"] * g5[r]).sum() for r in RENDERS).backward()
        for t in leaves:
            t.grad = None

    def window(fr, sh):
        for i in range(a.frames):
            step(fr, sh, cams[i % len(cams)])

    result = {"workload": wl.name, "sh_degree": deg, "P_scene": Ps, "P_human": Ph, "caps": caps, "card": card(),
              "fps": {}, "kernel_ms": {}}
    for mode, use_graph in (("eager", False), ("graph", True)):
        frs = {arm: TrainingFrameRenderer(Ps, Ph, (H, W), dev, caps, use_graph=use_graph, sh_coeffs=16 if sh else 0)
               for arm, sh in ARMS.items()}
        for arm, sh in ARMS.items():
            for i in range(a.warmup):
                step(frs[arm], sh, cams[i % len(cams)])
        # one call per window: each window walks the cameras from the first
        windows = alternate({arm: partial(window, frs[arm], sh) for arm, sh in ARMS.items()}, 1, a.rounds, 0)
        assert not any(f.overflowed() for f in frs.values())
        result["fps"][mode] = {arm: stats([a.frames / s for s in v], nd=1) for arm, v in windows.items()}
        del frs
        torch.cuda.empty_cache()

    # K1 / K6 per merged pass: serial frames on MergedFivePlan with the in-library profiler, read after every stage
    ms, cnt = (C.c_double * L_NUM)(), (C.c_uint64 * L_NUM)()
    shs = torch.cat((p["feature_dc"], p["feature_rest"]), 1).contiguous()
    for arm, sh in ARMS.items():
        plan = MergedFivePlan(Ps, Ph, W, H, caps, dev, sh_coeffs=16 if sh else 0)
        acc = {}

        def probe_fn(label):
            torch.cuda.synchronize()
            lib.b2r_profile_read(ms, cnt, 1)
            pk, stage = label.split(":")[0], label.split(":")[-1]
            for kid, kname in ((0, "K1_project"), (7, "K6_project_bwd")):
                if cnt[kid] and stage in ("bin", "project_bwd"):
                    acc.setdefault(f"{pk}:{kname}", []).append(ms[kid] / cnt[kid])

        for i in range(a.profile_frames + 2):
            cam = cams[i % len(cams)]
            st_w = render_settings((H, W), cam, torch.ones(3, device=dev))
            if sh:
                sc = dict(scene, shs=shs, sh_degree=deg)
                del sc["rgb"]
            else:
                sc = dict(scene, rgb=sh_to_rgb(deg, shs, scene["mean_3d"], st_w.campos))
            plan.set_scene(sc)
            if i == 2:  # two unprofiled warm-up frames
                lib.b2r_profile_enable(1)
                lib.b2r_profile_read(ms, cnt, 1)
            plan.frame(None, st_w, st_w._replace(bg=bg_r), sc, human, refined, g5, accumulate=False, serial=True,
                       probe=probe_fn if i >= 2 else None)
        torch.cuda.synchronize()
        lib.b2r_profile_enable(0)
        result["kernel_ms"][arm] = {k: round(statistics.median(v), 4) for k, v in sorted(acc.items())}
        del plan
        torch.cuda.empty_cache()
    emit(result, a.json)


if __name__ == "__main__":
    main()
