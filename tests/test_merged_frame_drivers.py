"""`MergedFivePlan` drives one training frame three ways: `frame()` with its passes and views on parallel streams,
`frame(serial=True, probe=...)` with everything on the caller's stream and a probe after every stage (bench.py and
tools/five_breakdown.py read per-view kernel times there), and `forward_frame()` + `backward_frame()` (fused.py).  All
three must compute the same frame: bit-equal images, and gradients equal up to the order of the backward's float sums.
"""
import pytest
import torch

from exavatar_release_b200.synthetic import WORKLOADS, make_grad_image, make_population_assets
from util import dev  # noqa: F401

pytestmark = pytest.mark.gpu

# bench.py parses these labels and reads per-view counter deltas between them
PROBE_LABELS = ["A:bin", "A:scene:fwd", "A:scene:bwd", "A:human:fwd", "A:human:bwd", "A:scene_human:fwd",
                "A:scene_human:bwd", "A:project_bwd",
                "B:bin", "B:human_refined:fwd", "B:human_refined:bwd", "B:scene_human_refined:fwd",
                "B:scene_human_refined:bwd", "B:project_bwd"]


def test_serial_split_and_concurrent_frames_agree(dev):
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.plan import RENDERS, MergedFivePlan
    from exavatar_release_b200.renderer import render_settings
    wl = WORKLOADS["T1"]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets("T1", seed=0, device=dev)
    Ps, Ph = scene["mean_3d"].shape[0], human["mean_3d"].shape[0]
    bg_w, bg_r = torch.ones(3, device=dev), torch.tensor([0.3, 0.7, 0.2], device=dev)
    cams = [look_at_cam_param(y, (H, W), device=dev) for y in (-8.0, 11.0)]
    settings = [(render_settings((H, W), c, bg_w), render_settings((H, W), c, bg_r)) for c in cams]
    gcol = [{r: make_grad_image("T1", 10 * f + j).to(dev) for j, r in enumerate(RENDERS)} for f in range(len(cams))]

    def run(one_frame):
        """Two frames (the second accumulates) on a fresh plan; its images of the last frame and its gradients."""
        plan = MergedFivePlan(Ps, Ph, W, H, None, dev)
        plan.set_scene(scene)
        for f, (st_w, st_r) in enumerate(settings):
            one_frame(plan, f, st_w, st_r)
        torch.cuda.synchronize()
        assert not plan.overflowed()
        imgs = {pk: [[t.clone() for t in img] + [plan.passes[pk].radii.clone()] for img in plan.passes[pk].img]
                for pk in plan.VIEWS}
        grads = {w: {k: v.clone() for k, v in plan.grads(w).items()} for w in ("scene", "human", "human_refined")}
        return imgs, grads

    unused = []
    ref = run(lambda p, f, st_w, st_r: p.frame(f, st_w, st_r, scene, human, refined, gcol[f], accumulate=f > 0,
                                               probe=unused.append))
    assert unused == []  # the probe is a serial-mode hook

    labels = []

    def serial(p, f, st_w, st_r):
        labels.clear()
        p.frame(f, st_w, st_r, scene, human, refined, gcol[f], accumulate=f > 0, serial=True, probe=labels.append)

    def split(p, f, st_w, st_r):
        p.forward_frame(f, st_w, st_r, scene, human, refined)
        p.backward_frame(gcol[f], p.views_A, p.views_B, accumulate=f > 0)

    for tag, (imgs, grads) in (("serial", run(serial)), ("split", run(split))):
        for pk, views in ref[0].items():
            for v, tensors in enumerate(views):
                for x, y in zip(imgs[pk][v], tensors):
                    assert torch.equal(x, y), (tag, pk, v)
        for which, named in ref[1].items():
            for k, y in named.items():
                x = grads[which][k]
                assert torch.allclose(x, y, rtol=1e-4, atol=1e-5 * float(y.abs().max()) + 1e-12), (tag, which, k)
    assert labels == PROBE_LABELS
