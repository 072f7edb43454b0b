"""`optim.Adam` (csrc/adam.cu): ExAvatar's optimizer step in one launch, bit-identical to torch.optim.Adam's default
foreach path.  CPU: the C ABI's segment layout and argument checks, the constructor's refusals and the host scalar
table against torch's _multi_tensor_adam expressions.  GPU: side by side with torch.optim.Adam(eps=1e-15) on
ExAvatar's group layout, bit for bit after every step (NaN compared by bit pattern), through optimizer surgery, state
dicts of either class, odd shapes and alignments, pipelined steps, and with no sync and one launch per step."""
import copy
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

from util import header_defines, no_host_sync
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.optim import Adam
from exavatar_release_b200.rasterizer import _compiled_binding

# ExAvatar's learning rates (avatar/main/config.py): lr, smplx_param_lr (both stages), the scene's
POSITION_LR = (1.6e-4, 1.6e-6)
LRS = (1e-3, 1e-4, 2.5e-3, 2.5e-3 / 20, 0.05, 5e-3, 1e-3, 1.6e-4 * 2.5, 0.0)


# ---------------------------------------------------------------------------------------------------------- CPU tests

def test_segment_layout_matches_header():
    lib = L.load()
    assert C.sizeof(L.B2RAdamSegment) == 88
    chunk = int(header_defines()["B2R_ADAM_CHUNK"])
    assert lib.b2r_adam_chunk_elems() == chunk and chunk % 4 == 0


def test_adam_step_rejects_bad_arguments():
    lib = L.load()
    fake = 0x1000  # never dereferenced: every call below fails on the host
    assert lib.b2r_adam_step(None, -1, 0, None) == -1         # negative segment count
    assert lib.b2r_adam_step(None, 1, 1, None) == -1          # null table with segments
    assert lib.b2r_adam_step(fake, 1, -1, None) == -1         # negative chunk count
    assert lib.b2r_adam_step(fake, 1, 1 << 31, None) == -1    # more CTAs than grid.x holds
    assert lib.b2r_adam_step(None, 0, 1, None) == -1          # chunks without segments
    assert lib.b2r_adam_step(fake, -5, 1, None) == -1
    assert lib.b2r_adam_step(None, 0, 0, None) == 0           # nothing to do: no launch
    assert lib.b2r_adam_step(fake, 3, 0, None) == 0           # only empty tensors: no launch


@pytest.mark.parametrize("kw", [dict(weight_decay=0.01), dict(amsgrad=True), dict(maximize=True)])
def test_unsupported_options_raise(kw):
    (name,) = kw
    with pytest.raises(ValueError, match=name):  # the option's own refusal, checked before the parameters
        Adam([torch.zeros(3)], lr=0.0, eps=1e-15, **kw)


@pytest.mark.parametrize("p", [torch.zeros(3), torch.zeros(3, dtype=torch.float64), torch.zeros(3, dtype=torch.float16)])
def test_non_cuda_or_non_fp32_params_raise(p):
    with pytest.raises(ValueError, match="float32 CUDA"):
        Adam([p], lr=0.0, eps=1e-15)
    with pytest.raises(ValueError, match="float32 CUDA"):
        Adam([{"params": [p], "name": "x", "lr": 1e-3}], lr=0.0, eps=1e-15)


def test_param_row_layouts():
    """ExAvatar's scene features are views of one (P,16,3) tensor (module.py:106-107): rows of 3 and of 45 floats,
    48 apart.  Contiguous tensors are one row; a transpose has no row layout."""
    rl = _compiled_binding().adam_row_layout
    feature = torch.zeros(7, 16, 3)
    assert not feature[:, 0:1, :].is_contiguous() and not feature[:, 1:, :].is_contiguous()
    assert tuple(rl(feature[:, 0:1, :])) == (True, 3, 48)
    assert tuple(rl(feature[:, 1:, :])) == (True, 45, 48)
    assert tuple(rl(torch.zeros(5, 3))) == (True, 15, 15)
    assert tuple(rl(torch.zeros(4, 6)[:, 1:4])) == (True, 3, 6)
    assert tuple(rl(torch.zeros(2, 4, 6)[:, :, :3])) == (True, 3, 6)  # the outer stride is 4 rows
    assert tuple(rl(torch.zeros(2, 4, 6)[:, :3, :3]))[0] is False  # two row strides
    assert tuple(rl(torch.zeros(4, 4).t()))[0] is False


def torch_scalars(lr, beta1, beta2, eps, step):
    """torch/optim/adam.py _multi_tensor_adam (capturable=False), restated: the lerp weight, beta2, addcmul value,
    bias_correction2_sqrt, eps and step_size the foreach ops receive, each a Python float that the ops' scalar
    arguments round to fp32."""
    bias_correction1 = 1 - beta1 ** step
    bias_correction2 = 1 - beta2 ** step
    step_size = (lr / bias_correction1) * -1
    bias_correction2_sqrt = bias_correction2 ** 0.5
    return [np.float32(x) for x in (1 - beta1, beta2, 1 - beta2, bias_correction2_sqrt, eps, step_size)]


def test_host_scalars_are_torch_rounded_once():
    steps = np.concatenate([np.arange(1, 201), np.unique(np.geomspace(200, 1e4, 300).astype(np.int64)), [10 ** 4]])
    sched = [math.exp(math.log(POSITION_LR[0]) * (1 - t) + math.log(POSITION_LR[1]) * t) for t in (0.0, 0.37, 1.0)]
    scalars = _compiled_binding().adam_scalars
    for lr in (*LRS, *sched):
        for betas in ((0.9, 0.999), (0.8, 0.99), (0.6, 0.0)):
            for s in steps:
                step = float(np.float32(s))  # the value of the CPU float32 step tensor
                want = torch_scalars(lr, *betas, 1e-15, step)
                got = [np.float32(x) for x in scalars(lr, *betas, 1e-15, step)]
                assert [x.tobytes() for x in got] == [x.tobytes() for x in want], (lr, betas, s)


# ---------------------------------------------------------------------------------------------------------- GPU tests

FRAME_PARAMS = {"root_pose": (6,), "body_pose": (21, 6), "jaw_pose": (6,), "leye_pose": (6,), "reye_pose": (6,),
                "lhand_pose": (15, 6), "rhand_pose": (15, 6), "expr": (50,), "trans": (3,)}


def trunk(k_in, final=None):
    shapes = []
    for k in (k_in, 128, 128):
        shapes += [(128, k), (128,), (128,), (128,)]  # Linear weight, bias; GroupNorm weight, bias
    return shapes + ([(final, 128), (final,)] if final else [])


def exavatar_layout(n_scene, n_frames, dev, seed=0):
    """ExAvatar's optimizer groups (module.py:143-148, 322-333, 666-671) as (name, [Parameter], lr) at the given scene
    size, with the human's tensors at C4 size (tools/bench_human_nets.py) and n_frames SMPL-X frames."""
    g = torch.Generator(device=dev).manual_seed(seed)
    mk = lambda s: nn.Parameter(0.1 * torch.randn(s, generator=g, device=dev))  # noqa: E731
    P = n_scene
    groups = [("mean_scene", [(P, 3)], POSITION_LR[0] * 2.5), ("feature_dc_scene", ["dc"], 2.5e-3),
              ("feature_rest_scene", ["rest"], 2.5e-3 / 20), ("opacity_scene", [(P, 1)], 0.05),
              ("scale_scene", [(P, 3)], 5e-3), ("rotation_scene", [(P, 4)], 1e-3),
              ("triplane_human", [(3, 32, 128, 128)], 1e-3), ("triplane_face_human", [(3, 32, 128, 128)], 1e-3),
              ("geo_net_human", trunk(96), 1e-3), ("mean_offset_net_human", [(3, 128), (3,)], 1e-3),
              ("scale_net_human", [(1, 128), (1,)], 1e-3), ("geo_offset_net_human", trunk(96 + 126), 1e-3),
              ("mean_offset_offset_net_human", [(3, 128), (3,)], 1e-3),
              ("scale_offset_net_human", [(1, 128), (1,)], 1e-3), ("rgb_net_human", trunk(96, 3), 1e-3),
              ("rgb_offset_net_human", trunk(96 + 126 + 3, 3), 1e-3), ("shape_param_human", [(100,)], 1e-3),
              ("joint_offset_human", [(55, 3)], 1e-3)]
    groups += [(f"smplx_{k}_{f}", [s], 1e-3) for f in range(n_frames) for k, s in FRAME_PARAMS.items()]
    # SceneGaussian.init_from_point_cloud (module.py:106-107): both feature groups are views of one (P,16,3) tensor
    feature = 0.1 * torch.randn((P, 16, 3), generator=g, device=dev)
    views = {"dc": nn.Parameter(feature[:, 0:1, :]), "rest": nn.Parameter(feature[:, 1:, :])}
    return [{"params": [views[s] if isinstance(s, str) else mk(s) for s in shapes], "name": name, "lr": lr}
            for name, shapes, lr in groups]


def twin(groups):
    """The same groups with fresh Parameters holding the same values: one set for torch.optim.Adam, one for Adam."""
    return [dict(gr, params=[same_layout(p) for p in gr["params"]]) for gr in groups]


def same_layout(p):
    """A new Parameter with p's values, sizes and strides (clone() would make a strided view contiguous)."""
    return nn.Parameter(torch.empty_strided(p.shape, p.stride(), device=p.device).copy_(p.detach()))


def wild_grad(p, gen):
    """Magnitudes 1e-30 ... 1e10, both signs, about one exact zero in eight."""
    mag = torch.pow(10.0, torch.empty(p.shape, device=p.device).uniform_(-30, 10, generator=gen))
    sign = torch.where(torch.rand(p.shape, device=p.device, generator=gen) < 0.5, -1.0, 1.0)
    zero = torch.rand(p.shape, device=p.device, generator=gen) < 0.125
    return torch.where(zero, 0.0, sign * mag)


def expon_lr(step, lr_init, lr_final, max_steps):
    """ExAvatar's scene-mean schedule (base.py:20-53 with no delay): log-linear from lr_init at 0 to lr_final at
    max_steps, clamped outside."""
    t = min(max(step / max_steps, 0.0), 1.0)
    return float(np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t))


def set_lr(opt, itr, tot_itr, base_lr=1e-3, smplx_lr=1e-3):
    """ExAvatar's set_lr (base.py:94-108): the scene mean follows expon_lr, human and SMPL-X groups drop to 1/10 past
    75 % of the run and to 1/100 past 95 %; the other scene groups keep their rate."""
    for gr in opt.param_groups:
        if gr["name"] == "mean_scene":
            gr["lr"] = expon_lr(itr, POSITION_LR[0] * 2.5, POSITION_LR[1] * 2.5, tot_itr)
        elif "human" in gr["name"] or "smplx" in gr["name"]:
            lr = base_lr if "human" in gr["name"] else smplx_lr
            if 0.75 * tot_itr < itr <= 0.95 * tot_itr:
                gr["lr"] = lr / 10
            elif itr > 0.95 * tot_itr:
                gr["lr"] = lr / 100


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.detach().view(torch.int32), b.detach().view(torch.int32))


def assert_same(ref, mine, where=""):
    assert len(ref.param_groups) == len(mine.param_groups)
    for gr, gm in zip(ref.param_groups, mine.param_groups):
        for pr, pm in zip(gr["params"], gm["params"]):
            assert bits_equal(pr, pm), f"{where} {gr['name']}: param"
            sr, sm = ref.state.get(pr, {}), mine.state.get(pm, {})
            assert sr.keys() == sm.keys(), f"{where} {gr['name']}: state keys"
            if sr:
                assert sm["step"].device.type == "cpu" and sm["step"].dtype == torch.float32 and sm["step"].dim() == 0
                assert sr["step"].item() == sm["step"].item(), f"{where} {gr['name']}: step"
                for k in ("exp_avg", "exp_avg_sq"):
                    assert sm[k].device == pm.device and sm[k].dtype == pm.dtype
                    assert bits_equal(sr[k], sm[k]), f"{where} {gr['name']}: {k}"


def set_grads(ref, mine, gen, frame=None, n_frames=None, wild=True):
    """Identical gradients on both optimizers' params; with `frame`, only that SMPL-X frame's groups get one."""
    for gr, gm in zip(ref.param_groups, mine.param_groups):
        on = not gr["name"].startswith("smplx") or frame is None or gr["name"].endswith(f"_{frame}")
        for pr, pm in zip(gr["params"], gm["params"]):
            if not on:
                pr.grad = pm.grad = None
                continue
            gval = wild_grad(pr, gen) if wild else torch.randn(pr.shape, device=pr.device, generator=gen)
            pr.grad, pm.grad = gval, gval.clone()


def pair(groups):
    return torch.optim.Adam(twin(groups), lr=0.0, eps=1e-15), Adam(twin(groups), lr=0.0, eps=1e-15)


@pytest.mark.gpu
def test_whole_layout_60_steps_bitwise():
    dev = torch.device("cuda")
    n_frames, tot = 4, 60
    ref, mine = pair(exavatar_layout(130_000, n_frames, dev))
    views = [gr["params"][0] for gr in mine.param_groups if gr["name"] in ("feature_dc_scene", "feature_rest_scene")]
    assert len(views) == 2 and not any(v.is_contiguous() for v in views)  # strided, as init_from_point_cloud makes them
    gen = torch.Generator(device=dev).manual_seed(1)
    for itr in range(tot):
        set_lr(ref, itr, tot)
        set_lr(mine, itr, tot)
        set_grads(ref, mine, gen, frame=itr % n_frames)
        ref.step()
        mine.step()
        assert_same(ref, mine, f"step {itr}")
    lrs = {gr["name"]: gr["lr"] for gr in mine.param_groups}
    assert lrs["shape_param_human"] == 1e-3 / 100 and lrs["mean_scene"] < POSITION_LR[0] * 2.5


def cat_rows(opt, new):
    """Densification's surgery (module.py:17-36 behaviour): append rows with zero moments, keeping step."""
    out = {}
    for gr in opt.param_groups:
        if gr["name"] not in new:
            continue
        old = gr["params"][0]
        st = opt.state.pop(old, None)
        p = nn.Parameter(torch.cat((old.detach(), new[gr["name"]])))
        if st is not None:
            st["exp_avg"] = torch.cat((st["exp_avg"], torch.zeros_like(new[gr["name"]])))
            st["exp_avg_sq"] = torch.cat((st["exp_avg_sq"], torch.zeros_like(new[gr["name"]])))
            opt.state[p] = st
        gr["params"][0] = out[gr["name"]] = p
    return out


def prune_rows(opt, names, keep):
    """Pruning's surgery (module.py:38-56 behaviour): keep the masked rows of param and moments."""
    for gr in opt.param_groups:
        if gr["name"] not in names:
            continue
        old = gr["params"][0]
        st = opt.state.pop(old, None)
        p = nn.Parameter(old.detach()[keep])
        if st is not None:
            st["exp_avg"], st["exp_avg_sq"] = st["exp_avg"][keep], st["exp_avg_sq"][keep]
            opt.state[p] = st
        gr["params"][0] = p


def replace_param(opt, name, value):
    """The opacity reset's surgery (module.py:58-72 behaviour): a new tensor with zero moments, keeping step."""
    for gr in opt.param_groups:
        if gr["name"] == name:
            st = opt.state.pop(gr["params"][0], None)
            p = nn.Parameter(value.clone())
            if st is not None:
                st["exp_avg"], st["exp_avg_sq"] = torch.zeros_like(p), torch.zeros_like(p)
                opt.state[p] = st
            gr["params"][0] = p


SCENE = ("mean_scene", "feature_dc_scene", "feature_rest_scene", "opacity_scene", "scale_scene", "rotation_scene")


@pytest.mark.gpu
def test_surgery_midrun():
    dev = torch.device("cuda")
    ref, mine = pair(exavatar_layout(20_000, 2, dev, seed=2))
    gen = torch.Generator(device=dev).manual_seed(3)

    def run(k):
        for i in range(k):
            set_grads(ref, mine, gen, frame=i % 2)
            ref.step()
            mine.step()
            assert_same(ref, mine, "after surgery")

    run(5)
    tails = {}
    for gr in ref.param_groups:
        if gr["name"] in SCENE:
            p = gr["params"][0]
            tails[gr["name"]] = torch.randn((1001, *p.shape[1:]), device=dev, generator=gen)
    cat_rows(ref, tails)
    cat_rows(mine, {k: v.clone() for k, v in tails.items()})  # 21 001 rows: odd, unaligned tails
    assert next(g for g in mine.param_groups if g["name"] == "opacity_scene")["params"][0].shape[0] == 21_001
    run(5)
    keep = torch.rand(21_001, device=dev, generator=gen) > 0.3
    prune_rows(ref, SCENE, keep)
    prune_rows(mine, SCENE, keep)
    run(5)
    op = next(g for g in ref.param_groups if g["name"] == "opacity_scene")["params"][0]
    fresh = torch.full_like(op, -2.19)
    replace_param(ref, "opacity_scene", fresh)
    replace_param(mine, "opacity_scene", fresh)
    run(5)


@pytest.mark.gpu
@pytest.mark.parametrize("direction", ["torch_to_op", "op_to_torch"])
def test_state_dict_round_trips(direction):
    dev = torch.device("cuda")
    groups = exavatar_layout(5_000, 2, dev, seed=4)
    ref, mine = pair(groups)
    gen = torch.Generator(device=dev).manual_seed(5)
    for i in range(4):
        set_grads(ref, mine, gen, frame=i % 2)
        ref.step()
        mine.step()
    # continue from the other class's state: a fresh twin of each set of params, loaded from the other optimizer
    src = ref if direction == "torch_to_op" else mine
    sd = src.state_dict()
    a_groups = [dict(gr, params=[same_layout(p) for p in g2["params"]]) for gr, g2 in zip(groups, src.param_groups)]
    b_groups = [dict(gr, params=[same_layout(p) for p in g2["params"]]) for gr, g2 in zip(groups, src.param_groups)]
    ref2 = torch.optim.Adam(a_groups, lr=0.0, eps=1e-15)
    mine2 = Adam(b_groups, lr=0.0, eps=1e-15)
    # a copy per load, as from a checkpoint file: state_dict() hands out the live 'step' tensors, and loading keeps them
    ref2.load_state_dict(copy.deepcopy(sd))
    mine2.load_state_dict(copy.deepcopy(sd))
    assert_same(ref2, mine2, "loaded")
    for i in range(4):
        set_grads(ref2, mine2, gen, frame=i % 2)
        ref2.step()
        mine2.step()
        assert_same(ref2, mine2, f"{direction} step {i}")


@pytest.mark.gpu
def test_odd_shapes_unaligned_views_and_nonfinite_grads():
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(6)
    store_r = torch.randn(1 + 4 * 40_000 + 7, device=dev, generator=gen)
    store_m = store_r.clone()
    shapes = [(0,), (1,), (3,), (5,), (16_385,), (3, 5)]

    def params(store):
        ps = [nn.Parameter(torch.randn(s, device=dev, generator=torch.Generator(device=dev).manual_seed(i)))
              for i, s in enumerate(shapes)]
        # views from a storage offset of 1 float (4 bytes): no segment pointer is 16-byte aligned
        v = store[1:1 + 4 * 40_000].view(40_000, 4)
        ps.append(nn.Parameter(v))
        return ps

    ref = torch.optim.Adam([{"params": params(store_r), "name": "odd", "lr": 1e-2}], lr=0.0, eps=1e-15)
    mine = Adam([{"params": params(store_m), "name": "odd", "lr": 1e-2}], lr=0.0, eps=1e-15)
    assert mine.param_groups[0]["params"][-1].data_ptr() % 16 == 4
    for i in range(6):
        for pr, pm in zip(ref.param_groups[0]["params"], mine.param_groups[0]["params"]):
            gval = wild_grad(pr, gen)
            if gval.numel() > 4 and i in (2, 4):  # NaN and +-inf grads, then finite again: both propagate the same
                gval.view(-1)[:4] = torch.tensor([float("nan"), float("inf"), -float("inf"), 0.0], device=dev)
            pr.grad, pm.grad = gval, gval.clone()
        ref.step()
        mine.step()
        assert_same(ref, mine, f"odd step {i}")
    assert mine.state[mine.param_groups[0]["params"][0]]["step"].item() == 6  # numel 0: the step still advances
    assert torch.isnan(mine.param_groups[0]["params"][-2]).any()


@pytest.mark.gpu
def test_pipelined_steps_without_sync():
    dev = torch.device("cuda")
    ref, mine = pair(exavatar_layout(50_000, 3, dev, seed=7))
    gen = torch.Generator(device=dev).manual_seed(8)
    grads = []
    for i in range(20):  # every step's gradients made up front, so the loop below only enqueues
        set_grads(ref, mine, gen, frame=i % 3, wild=False)
        grads.append([[p.grad for p in gr["params"]] for gr in mine.param_groups])
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)  # hold the stream (~0.1 s) so that all 20 copies and launches are queued behind it
    for i in range(20):
        for gr in mine.param_groups:
            gr["lr"] = 1e-3 * (1 + i)  # a new lr every step: a staging buffer reused too early shows here
        for gr, gs in zip(mine.param_groups, grads[i]):
            for p, g in zip(gr["params"], gs):
                p.grad = g
        mine.step()
    for i in range(20):
        for gr in ref.param_groups:
            gr["lr"] = 1e-3 * (1 + i)
        for gr, gs in zip(ref.param_groups, grads[i]):
            for p, g in zip(gr["params"], gs):
                p.grad = None if g is None else g.clone()
        ref.step()
    torch.cuda.synchronize()
    assert_same(ref, mine, "pipelined")


@pytest.mark.gpu
def test_no_sync_and_one_launch_per_step_with_1000_frames():
    dev = torch.device("cuda")
    lib = L.load()
    groups = exavatar_layout(130_000, 1000, dev, seed=9)
    mine = Adam(groups, lr=0.0, eps=1e-15)
    assert len(mine.param_groups) == 18 + 9 * 1000
    gen = torch.Generator(device=dev).manual_seed(10)
    for i in range(3):
        for gr in mine.param_groups:
            on = not gr["name"].startswith("smplx") or gr["name"].endswith(f"_{i}")
            for p in gr["params"]:
                p.grad = torch.randn(p.shape, device=dev, generator=gen) if on else None
        torch.cuda.synchronize()
        n0 = lib.b2r_launch_count()
        with no_host_sync():
            mine.step()
        assert lib.b2r_launch_count() == n0 + 1
    for gr in mine.param_groups:
        for p in gr["params"]:
            p.grad = None
    n0 = lib.b2r_launch_count()
    mine.step()
    assert lib.b2r_launch_count() == n0
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_cuda_only_refusals():
    dev = torch.device("cuda")
    with pytest.raises(ValueError, match="rows of contiguous floats"):
        Adam([torch.zeros(4, 4, device=dev).t()], lr=0.0)  # a transpose: no row layout
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="more than one device"):
            Adam([torch.zeros(3, device="cuda:0"), torch.zeros(3, device="cuda:1")], lr=0.0)
    p = nn.Parameter(torch.zeros(3, device=dev))
    opt = Adam([p], lr=1e-3)
    p.grad = torch.zeros(3, device=dev).to_sparse()
    with pytest.raises(ValueError, match="sparse"):
        opt.step()


@pytest.mark.gpu
def test_deepcopy_and_pickle_keep_stepping():
    import pickle
    dev = torch.device("cuda")
    ref, mine = pair(exavatar_layout(1_000, 1, dev, seed=11))
    gen = torch.Generator(device=dev).manual_seed(12)
    set_grads(ref, mine, gen, frame=0, wild=False)
    ref.step()
    mine.step()
    for clone in (copy.deepcopy, lambda o: pickle.loads(pickle.dumps(o))):
        r2, m2 = clone(ref), clone(mine)
        set_grads(r2, m2, gen, frame=0, wild=False)
        r2.step()
        m2.step()
        assert_same(r2, m2, "copied optimizer")
