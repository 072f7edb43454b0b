"""The refined pass of `MergedFivePlan` (pass B, cat(scene, human_refined)) as a SPLIT pass: it projects, scatters and sorts
only the refined rows and builds a list only in the tiles they reach, as the merge of pass A's list of the tile filtered
to scene ids with its own sorted entries on the (depth_bits, id) key (b2r_forward_project_split / b2r_forward_bin_split).

CPU: a numpy restatement of that filter + merge against the joint sort.  GPU: the split pass against the whole pass
(MergedFivePlan.SPLIT = False) at full C4 size -- lists, images, alpha and radii bit-equal, gradients within the tolerance of
the backward's reordered float sums."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

SEG, CHUNK = 512, 2048  # the composites' segment cut and the sort's chunk length (common.cuh)


def joint_sort(depth_bits, ids):
    """Order of the per-tile sort: ascending depth bits, ties by ascending id."""
    return ids[np.lexsort((ids, depth_bits))]


def split_merge(base_list, depth_of, split, own_sorted):
    """Restates split_merge_kernel: filter the base list to ids < split (order kept), then place every entry at its index
    in its own sequence plus the number of entries of the other sequence below it on the 64-bit (depth_bits, id) key."""
    scene = base_list[base_list < split]
    key = lambda ids: (depth_of[ids].astype(np.uint64) << np.uint64(32)) | ids.astype(np.uint64)
    ko, ks = key(own_sorted), key(scene)
    assert np.all(ks[1:] > ks[:-1])  # filtering keeps the base order
    out = np.empty(ko.size + ks.size, dtype=np.int64)
    out[np.arange(ko.size) + np.searchsorted(ks, ko)] = own_sorted
    out[np.arange(ks.size) + np.searchsorted(ko, ks)] = scene
    return out


@pytest.mark.parametrize("n_scene,n_human,n_own,depth_levels", [
    (300, 200, 150, 10**6),      # short list
    (40, 30, 0, 10**6),          # a tile the refined rows do not reach: the split pass leaves it empty
    (0, 20, 90, 10**6),          # refined entries only
    (700, 500, 400, 7),          # few distinct depths: bit-identical depths across the two populations
    (2600, 1900, 2300, 50),      # long lists across the 2048-entry chunk and the 512-entry segment cuts
])
def test_filter_and_merge_equal_the_joint_sort(n_scene, n_human, n_own, depth_levels):
    rng = np.random.default_rng(n_scene * 7 + n_own)
    Ps = 5000
    P = Ps + 4000
    depth = rng.integers(0x3E000000, 0x3E000000 + depth_levels, size=P, dtype=np.int64).astype(np.uint32)
    scene_ids = rng.choice(Ps, n_scene, replace=False)
    human_ids = Ps + rng.choice(P - Ps, n_human, replace=False)   # pass A's human rows
    own_ids = Ps + rng.choice(P - Ps, n_own, replace=False)       # pass B's refined rows (same numbering)
    base = joint_sort(depth[np.r_[scene_ids, human_ids]], np.r_[scene_ids, human_ids])
    expect = joint_sort(depth[np.r_[scene_ids, own_ids]], np.r_[scene_ids, own_ids])
    own_sorted = joint_sort(depth[own_ids], own_ids)
    if n_own == 0:  # no refined entry: the split pass builds no list there (the views skip the tile)
        assert not np.any(expect >= Ps)
        return
    got = split_merge(base, depth, Ps, own_sorted)
    assert np.array_equal(got, expect)
    n = got.size
    if n >= CHUNK:  # the tile is cut into sort chunks and composite segments exactly as the whole pass cuts it
        assert math.ceil(n / CHUNK) >= 2 and math.ceil(n / SEG) >= 5
    if depth_levels < 100:  # equal depths do occur across the populations
        d = depth[expect]
        eq = np.flatnonzero(d[1:] == d[:-1])
        assert np.any((expect[eq] < Ps) != (expect[eq + 1] < Ps))


# ------------------------------------------------------------------ GPU ------------------------------------------------

def _plan_classes():
    from exavatar_release_b200.plan import MergedFivePlan

    class FullPass(MergedFivePlan):
        SPLIT = False

    class SplitPass(MergedFivePlan):
        SPLIT = True

    return SplitPass, FullPass


def _pitched_rolled(cam, pitch_deg, roll_deg):
    """The camera turned about its own x (pitch) and z (roll) axes, centre unchanged."""
    p, r = math.radians(pitch_deg), math.radians(roll_deg)
    dev = cam["R"].device
    Rx = torch.tensor([[1, 0, 0], [0, math.cos(p), -math.sin(p)], [0, math.sin(p), math.cos(p)]], dtype=torch.float32)
    Rz = torch.tensor([[math.cos(r), -math.sin(r), 0], [math.sin(r), math.cos(r), 0], [0, 0, 1]], dtype=torch.float32)
    Q = (Rz @ Rx).to(dev)
    return dict(cam, R=Q @ cam["R"], t=(Q @ cam["t"].reshape(3, 1)).reshape(cam["t"].shape))


def _lists(plan):
    """Per-tile id lists of pass B (numpy), from its ranges and dup_ids."""
    ps = plan.passes["B"]
    lib = plan.lib
    ptr = lib.b2r_ctx_ranges(C.byref(ps.ws), plan.P, plan.W, plan.H)
    off = ptr - ps.ctx_buf.data_ptr()
    tiles = ((plan.W + 15) // 16) * ((plan.H + 15) // 16)
    ranges = ps.ctx_buf[off:off + 8 * tiles].view(torch.int32).view(tiles, 2).cpu().numpy()
    ids = ps.ids.cpu().numpy()
    return [ids[a:b] for a, b in ranges]


def _close(x, y, what):
    """Gradients: the backward composites add with float atomics in no fixed order, so every run -- pass A's, which the
    split pass does not change, included -- differs from the next in the last bits.  Every entry agrees to rtol 1e-3 /
    atol 1e-4 of the tensor's largest entry, except at most three, and those within 5e-3 of it (parity.compare's bound
    for its few allowed entries): a gradient summed from large terms of both signs keeps their rounding.  At C4 with the
    pitched and rolled SH cameras one such entry exists -- the rotation gradient of a needle-shaped scene Gaussian
    (scales 0.27 x 0.011 x 0.005), whose conic gradient sums squared pixel offsets of up to its length -- and two runs
    of the SAME plan differ there by up to 3e-4 of the largest entry (H100)."""
    scale = float(y.abs().max()) + 1e-12
    d = (x - y).abs()
    over = int((d > 1e-3 * y.abs() + 1e-4 * scale).sum())
    err = float(d.max())
    assert over <= 3 and err <= 5e-3 * scale, (what, over, err, scale)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["rgb", "sh_pitched_rolled"])
def test_split_refined_pass_equals_the_whole_pass_c4(dev, mode):
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.plan import RENDERS
    from exavatar_release_b200.renderer import render_settings
    from exavatar_release_b200.synthetic import WORKLOADS, make_grad_image, make_population_assets
    wl = WORKLOADS["C4"]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets("C4", seed=0, device=dev)
    Ps, Ph = scene["mean_3d"].shape[0], human["mean_3d"].shape[0]
    sh = mode.startswith("sh")
    M = 16 if sh else 0
    if sh:
        g = torch.Generator(device="cpu").manual_seed(3)
        scene = {k: v for k, v in scene.items() if k != "rgb"}
        scene["shs"] = (0.3 * torch.randn(Ps, M, 3, generator=g)).to(dev)
        scene["sh_degree"] = 3
    bg_w, bg_r = torch.ones(3, device=dev), torch.tensor([0.3, 0.7, 0.2], device=dev)
    cams = [look_at_cam_param(y, (H, W), device=dev) for y in (-12.0, 9.0)]
    if mode == "sh_pitched_rolled":
        cams = [_pitched_rolled(c, 14.0, -21.0) for c in cams]
    settings = [(render_settings((H, W), c, bg_w), render_settings((H, W), c, bg_r)) for c in cams]
    gcol = [{r: make_grad_image("C4", 10 * f + j).to(dev) for j, r in enumerate(RENDERS)} for f in range(len(cams))]
    Split, Full = _plan_classes()
    out = {}
    for cls in (Full, Split):
        plan = cls(Ps, Ph, W, H, None, dev, sh_coeffs=M)
        plan.set_scene(scene)
        for f, (st_w, st_r) in enumerate(settings):
            plan.frame(f, st_w, st_r, scene, human, refined, gcol[f], accumulate=f > 0)
        torch.cuda.synchronize()
        assert not plan.overflowed()
        out[cls.SPLIT] = dict(
            imgs={r: [t.clone() for t in plan.render_outputs(r)[:2]] for r in RENDERS},
            radii=[plan.passes[k].radii.clone() for k in ("A", "B")],
            grads={w: {k: v.clone() for k, v in plan.grads(w).items()} for w in ("scene", "human", "human_refined")},
            lists=_lists(plan), dups=plan.dups(), consumed=plan.consumed())
        del plan
    full, split = out[False], out[True]
    for r in RENDERS:
        for x, y in zip(split["imgs"][r], full["imgs"][r]):
            assert torch.equal(x, y), r
    for x, y in zip(split["radii"], full["radii"]):
        assert torch.equal(x, y)
    n_lists = 0
    for a, b in zip(split["lists"], full["lists"]):
        if a.size:
            assert np.array_equal(a, b)
            n_lists += 1
        else:
            assert not np.any(b >= Ps)  # a tile without refined entries: the views skip it in both passes
    assert n_lists > 0
    assert split["dups"]["A"] == full["dups"]["A"] and split["dups"]["B"] < full["dups"]["B"]
    assert split["consumed"] == full["consumed"]
    for which, named in full["grads"].items():
        for k, y in named.items():
            _close(split["grads"][which][k], y, (which, k))


@pytest.mark.gpu
def test_split_refined_pass_reports_an_overflow(dev):
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.plan import RENDERS
    from exavatar_release_b200.renderer import render_settings
    from exavatar_release_b200.synthetic import WORKLOADS, make_grad_image, make_population_assets
    wl = WORKLOADS["C4"]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets("C4", seed=0, device=dev)
    Ps, Ph = scene["mean_3d"].shape[0], human["mean_3d"].shape[0]
    cam = look_at_cam_param(4.0, (H, W), device=dev)
    st_w = render_settings((H, W), cam, torch.ones(3, device=dev))
    st_r = render_settings((H, W), cam, torch.tensor([0.3, 0.7, 0.2], device=dev))
    gcol = {r: make_grad_image("C4", j).to(dev) for j, r in enumerate(RENDERS)}
    Split, _ = _plan_classes()
    ok = Split(Ps, Ph, W, H, None, dev)
    ok.set_scene(scene)
    ok.frame(0, st_w, st_r, scene, human, refined, gcol, accumulate=False)
    torch.cuda.synchronize()
    need = ok.dups()["B"]
    del ok
    small = Split(Ps, Ph, W, H, {"A": 8_000_000, "B": need // 3}, dev)
    small.set_scene(scene)
    small.frame(0, st_w, st_r, scene, human, refined, gcol, accumulate=False)
    torch.cuda.synchronize()
    st = small.passes["B"].status()
    assert st["overflow"] == 1 and st["num_dups"] == need and small.overflowed()
    assert not small.passes["A"].status()["overflow"]


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True])
def test_training_frame_renderer_split_equals_full(dev, use_graph):
    """fused.TrainingFrameRenderer, eager and graph-captured, on the split refined pass and on the whole one."""
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.fused import TrainingFrameRenderer
    from exavatar_release_b200.plan import RENDERS
    from exavatar_release_b200.synthetic import WORKLOADS, make_population_assets
    wl = WORKLOADS["C4"]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets("C4", seed=0, device=dev)
    Ps, Ph = scene["mean_3d"].shape[0], human["mean_3d"].shape[0]
    bg_r = torch.tensor([0.3, 0.7, 0.2], device=dev)
    res = {}
    for split in (False, True):
        fr = TrainingFrameRenderer(Ps, Ph, (H, W), dev, {"A": 8_000_000, "B": 8_000_000}, use_graph=use_graph)
        fr.plan.SPLIT = split
        leaves = [{k: v.detach().clone().requires_grad_() for k, v in x.items()} for x in (scene, human, refined)]
        for yaw in (-7.0, 5.0):
            outs = fr(*leaves, look_at_cam_param(yaw, (H, W), device=dev), bg_r)
            loss = sum((outs[r]["img"] * (0.5 + 0.1 * j)).sum() for j, r in enumerate(RENDERS))
            loss.backward()
        torch.cuda.synchronize()
        res[split] = ({r: outs[r]["img"].detach().clone() for r in RENDERS},
                      [{k: v.grad.clone() for k, v in lv.items()} for lv in leaves])
    for r in RENDERS:
        assert torch.equal(res[True][0][r], res[False][0][r]), r
    for gs, gf in zip(res[True][1], res[False][1]):
        for k, y in gf.items():
            _close(gs[k], y, k)
