"""A whole training iteration as one CUDA graph per key (`IterationGraph`), and the two pieces under it: Adam's
frame-row groups and its step split into `stage()` + `launch()`.  CPU: the frame-row refusals.  GPU: frame-row Adam
bit-identical to torch.optim.Adam over ExAvatar's per-frame groups (tests/test_adam.py's layout and set_lr, restated
here) over a frame sequence with repeats; a captured `launch()` replayed 60 times with a new lr each step,
bit-identical to eager `step()`, without a host sync; and a reduced iteration through IterationGraph, bit-identical to
the same chain run eagerly and to the per-frame ParameterDict route, through a key change and optimizer surgery."""
import contextlib
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from exavatar_release_b200 import _lib as L
from exavatar_release_b200.human_assets import POSE_KEYS, POSE_ROWS, SmplxParamTable, decode_smplx_pose
from exavatar_release_b200.iteration import IterationGraph
from exavatar_release_b200.losses import l1_ssim
from exavatar_release_b200.optim import Adam, StaleLayoutError
from util import no_host_sync

POSITION_LR = (1.6e-4, 1.6e-6)
FRAME_PARAMS = {"root_pose": (6,), "body_pose": (21, 6), "jaw_pose": (6,), "leye_pose": (6,), "reye_pose": (6,),
                "lhand_pose": (15, 6), "rhand_pose": (15, 6), "expr": (50,), "trans": (3,)}


def expon_lr(step, lr_init, lr_final, max_steps):
    """ExAvatar's scene-mean schedule (base.py:20-53 with no delay)."""
    t = min(max(step / max_steps, 0.0), 1.0)
    return float(np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t))


def set_lr(opt, itr, tot_itr, base_lr=1e-3, smplx_lr=1e-3):
    """ExAvatar's set_lr (base.py:94-108)."""
    for gr in opt.param_groups:
        if gr["name"] == "mean_scene":
            gr["lr"] = expon_lr(itr, POSITION_LR[0] * 2.5, POSITION_LR[1] * 2.5, tot_itr)
        elif "human" in gr["name"] or "smplx" in gr["name"]:
            lr = base_lr if "human" in gr["name"] else smplx_lr
            if 0.75 * tot_itr < itr <= 0.95 * tot_itr:
                gr["lr"] = lr / 10
            elif itr > 0.95 * tot_itr:
                gr["lr"] = lr / 100


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def shared_groups(P, dev, seed):
    """ExAvatar's scene and human groups at a small size: (name, [Parameter], lr); the two feature groups are views
    of one (P,16,3) tensor, as SceneGaussian.init_from_point_cloud makes them."""
    g = torch.Generator(device=dev).manual_seed(seed)
    mk = lambda s: nn.Parameter(0.1 * torch.randn(s, generator=g, device=dev))  # noqa: E731
    feature = 0.1 * torch.randn((P, 16, 3), generator=g, device=dev)
    return [("mean_scene", [mk((P, 3))], POSITION_LR[0] * 2.5),
            ("feature_dc_scene", [nn.Parameter(feature[:, 0:1, :])], 2.5e-3),
            ("feature_rest_scene", [nn.Parameter(feature[:, 1:, :])], 2.5e-3 / 20),
            ("opacity_scene", [mk((P, 1))], 0.05), ("geo_net_human", [mk((128, 96)), mk((128,))], 1e-3),
            ("shape_param_human", [mk((100,))], 1e-3), ("joint_offset_human", [mk((55, 3))], 1e-3)]


def same_layout(p):
    return nn.Parameter(torch.empty_strided(p.shape, p.stride(), device=p.device).copy_(p.detach()))


def frame_values(F, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return [{k: 0.1 * torch.randn(s, generator=g, device=dev) for k, s in FRAME_PARAMS.items()} for _ in range(F)]


def per_frame_groups(frames):
    """module.py:666-671: nine groups per frame, named smplx_<key>_<frame>."""
    return [{"params": [nn.Parameter(v.clone())], "name": f"smplx_{k}_{f}", "lr": 1e-3}
            for f, d in enumerate(frames) for k, v in d.items()]


def table_of(frames):
    pose = torch.stack([torch.cat([d[k].reshape(-1, 6) for k in POSE_KEYS]) for d in frames]).contiguous()
    expr = torch.stack([d["expr"] for d in frames]).contiguous()
    trans = torch.stack([d["trans"] for d in frames]).contiguous()
    return SmplxParamTable(pose.requires_grad_(), expr.requires_grad_(), trans.requires_grad_())


def frame_rows(table, i):
    """Frame i of the table split into FRAME_PARAMS' nine tensors: views without autograd history (a view of a leaf
    with history would keep its AccumulateGrad node, and the stream it was made on, alive into the next capture)."""
    pose, expr, trans = (t.detach() for t in table)
    out, r0 = {}, 0
    for k, n in zip(POSE_KEYS, POSE_ROWS):
        out[k] = pose[i, r0:r0 + n].reshape(FRAME_PARAMS[k])
        r0 += n
    out["expr"], out["trans"] = expr[i], trans[i]
    return out


# ---------------------------------------------------------------------------------------------------------- CPU tests

def test_frame_row_group_refusals():
    """The frame-row checks of the host walk run before any device check, state creation or count."""
    from exavatar_release_b200.optim import _chunk
    from exavatar_release_b200.rasterizer import _compiled_binding
    stage = _compiled_binding().adam_stage
    p = torch.zeros(4, 3, requires_grad=True)
    p.grad = torch.ones(4, 3)
    group = {"params": [p], "frame_rows": True, "lr": 1e-3, "betas": (0.9, 0.999), "eps": 1e-15}
    state = {}
    with pytest.raises(ValueError, match="only with `rows`"):
        stage([group], state, 0, _chunk(), None, None, None)
    for bad in (-1, 4):
        with pytest.raises(ValueError, match="outside"):
            stage([group], state, 0, _chunk(), bad, None, None)
    q = torch.zeros(4, 6, requires_grad=True)
    q.grad = torch.ones(4, 6)
    view = q.detach()[:, :3]
    view.grad = torch.ones(4, 3)
    with pytest.raises(ValueError, match="frame-row parameter must be contiguous"):
        stage([dict(group, params=[view])], state, 0, _chunk(), 1, None, None)
    assert not state
    with pytest.raises(ValueError, match="float32 CUDA"):
        Adam([{"params": [torch.zeros(4, 3)], "frame_rows": True}], lr=0.0)


# ---------------------------------------------------------------------------------------------------------- GPU tests

@pytest.mark.gpu
def test_frame_row_refusals_on_the_device():
    dev = torch.device("cuda")
    with pytest.raises(ValueError, match="frame-row"):
        Adam([{"params": [nn.Parameter(torch.zeros(4, 6, device=dev)[:, :3])], "frame_rows": True}], lr=0.0)
    p = nn.Parameter(torch.zeros(4, 3, device=dev))
    opt = Adam([{"params": [p], "frame_rows": True}], lr=1e-3)
    p.grad = torch.ones_like(p)
    with pytest.raises(ValueError, match="rows"):
        opt.step()
    for bad in (-1, 4):
        with pytest.raises(ValueError, match="outside"):
            opt.step(rows=bad)
    assert not opt.state  # nothing was counted or created by a refused step
    opt.step(rows=2)
    assert opt.state[p]["step"].tolist() == [0, 0, 1, 0]


@pytest.mark.gpu
def test_step_without_gradients_launches_nothing():
    """An optimizer that has never staged a table and whose params have no gradient: step() does nothing."""
    lib = L.load()
    p = nn.Parameter(torch.zeros(5, 3, device="cuda"))
    opt = Adam([p], lr=1e-3)
    n0 = lib.b2r_launch_count()
    opt.step()
    assert lib.b2r_launch_count() == n0 and not opt.state
    assert torch.equal(p, torch.zeros_like(p))


@pytest.mark.gpu
def test_frame_rows_match_per_frame_groups_60_steps():
    dev = torch.device("cuda")
    F, tot = 9, 60
    shared = shared_groups(5_003, dev, seed=0)
    frames = frame_values(F, dev, seed=1)
    ref_groups = [{"params": [same_layout(p) for p in ps], "name": n, "lr": lr} for n, ps, lr in shared]
    ref = torch.optim.Adam(ref_groups + per_frame_groups(frames), lr=0.0, eps=1e-15)
    table = table_of(frames)
    mine_groups = [{"params": [same_layout(p) for p in ps], "name": n, "lr": lr} for n, ps, lr in shared]
    mine = Adam(mine_groups + [{"params": table.parameters(), "name": "smplx", "lr": 1e-3, "frame_rows": True}],
                lr=0.0, eps=1e-15)
    init = [t.detach().clone() for t in table.parameters()]
    rng = np.random.default_rng(2)
    seq = [int(x) for x in rng.integers(0, F - 2, tot)]  # repeats, and frames F-2, F-1 never visited
    seq[5] = seq[4]
    gen = torch.Generator(device=dev).manual_seed(3)
    ref_frames = [ref.param_groups[len(shared) + 9 * f: len(shared) + 9 * f + 9] for f in range(F)]
    n = len(shared)
    for itr, f in enumerate(seq):
        set_lr(ref, itr, tot)
        set_lr(mine, itr, tot)
        for gr, gm in zip(ref.param_groups[:n], mine.param_groups[:n]):
            for pr, pm in zip(gr["params"], gm["params"]):
                pr.grad = torch.randn(pr.shape, device=dev, generator=gen)
                pm.grad = pr.grad.clone()
        for gr in ref.param_groups[n:]:
            gr["params"][0].grad = None
        for t in table.parameters():
            t.grad = torch.zeros_like(t)
        gm = frame_rows([t.grad for t in table.parameters()], f)
        for gr in ref_frames[f]:
            k = gr["name"][len("smplx_"):gr["name"].rindex("_")]
            gr["params"][0].grad = torch.randn(FRAME_PARAMS[k], device=dev, generator=gen)
            gm[k].copy_(gr["params"][0].grad)
        ref.step()
        mine.step(rows=f)
        for gr, gm_ in zip(ref.param_groups[:n], mine.param_groups[:n]):
            for pr, pm in zip(gr["params"], gm_["params"]):
                assert same(pr, pm), (itr, gr["name"])
                for k in ("exp_avg", "exp_avg_sq"):
                    assert same(ref.state[pr][k], mine.state[pm][k]), (itr, gr["name"], k)
    st = [mine.state[t] for t in table.parameters()]
    for f in range(F):
        rows = frame_rows(table.parameters(), f)
        moments = {k: frame_rows([s[k] for s in st], f) for k in ("exp_avg", "exp_avg_sq")}
        for gr in ref_frames[f]:
            k = gr["name"][len("smplx_"):gr["name"].rindex("_")]
            pr = gr["params"][0]
            assert same(pr, rows[k]), (f, k)
            sr = ref.state.get(pr)
            if sr is None:  # never visited: untouched, bit for bit
                assert f not in seq
                for s in st:
                    assert s["step"][f].item() == 0
                assert same(rows[k], frame_rows(init, f)[k])
                assert not moments["exp_avg"][k].any() and not moments["exp_avg_sq"][k].any()
                continue
            assert sr["step"].item() == seq.count(f)
            for s in st:
                assert s["step"][f].item() == seq.count(f)
            for m in ("exp_avg", "exp_avg_sq"):
                assert same(sr[m], moments[m][k]), (f, k, m)
    # state_dict round trip
    sd = mine.state_dict()
    other = Adam([{"params": [same_layout(p) for p in gr["params"]], **{k: v for k, v in gr.items() if k != "params"}}
                  for gr in mine.param_groups], lr=0.0, eps=1e-15)
    other.load_state_dict(sd)
    for pa, pb in zip([p for g in mine.param_groups for p in g["params"]],
                      [p for g in other.param_groups for p in g["params"]]):
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert same(mine.state[pa][k], other.state[pb][k])
    assert other.param_groups[-1]["frame_rows"] is True


@pytest.mark.gpu
def test_captured_launch_replays_match_eager_steps():
    dev = torch.device("cuda")
    lib = L.load()
    F = 6
    shared = shared_groups(20_011, dev, seed=4)
    frames = frame_values(F, dev, seed=5)

    def build():
        t = table_of(frames)
        groups = [{"params": [same_layout(p) for p in ps], "name": n, "lr": lr} for n, ps, lr in shared]
        return Adam(groups + [{"params": t.parameters(), "name": "smplx", "lr": 1e-3, "frame_rows": True}],
                    lr=0.0, eps=1e-15)

    eager, graphed = build(), build()
    params = lambda o: [p for g in o.param_groups for p in g["params"]]  # noqa: E731
    for p in params(graphed):  # the gradients the graph's launch reads, at fixed addresses
        p.grad = torch.zeros_like(p)
    gen = torch.Generator(device=dev).manual_seed(6)
    rng = np.random.default_rng(7)
    g = None
    for i in range(60):
        slot = int(rng.integers(0, F))
        for o in (eager, graphed):
            for k, gr in enumerate(o.param_groups):
                gr["lr"] = 1e-3 * (1 + i) / (1 + k)
        new = [torch.randn(p.shape, device=dev, generator=gen) for p in params(eager)]
        for p, gv in zip(params(eager), new):
            p.grad = gv
        for p, gv in zip(params(graphed), new):
            p.grad.copy_(gv)
        eager.step(rows=slot)
        if g is None:
            graphed.stage(rows=slot)
            g = torch.cuda.CUDAGraph()
            n0 = lib.b2r_launch_count()
            with torch.cuda.graph(g):
                graphed.launch()
            assert lib.b2r_launch_count() == n0 + 1  # one Adam launch in the graph
            g.replay()
        else:
            n0 = lib.b2r_launch_count()
            with no_host_sync():
                graphed.stage(rows=slot)
                g.replay()
            assert lib.b2r_launch_count() == n0
        for pa, pb in zip(params(eager), params(graphed)):
            assert same(pa, pb), i
            for k in ("step", "exp_avg", "exp_avg_sq"):
                assert same(eager.state[pa][k], graphed.state[pb][k]), (i, k)
    # another set of params with gradients: reported, nothing counted
    params(graphed)[0].grad = None
    steps = [graphed.state[p]["step"].clone() for p in params(graphed)[1:]]
    with pytest.raises(StaleLayoutError):
        graphed.stage(rows=0)
    assert all(torch.equal(s, graphed.state[p]["step"]) for s, p in zip(steps, params(graphed)[1:]))
    graphed.release_graph()
    graphed.stage(rows=0)


# The training iteration at reduced size (tools/bench_iteration_graph.py's Chain: SMPL-X decode, the synthetic SMPL-X
# rig, networks, HumanAssets, skinning, TrainingFrameRenderer(use_graph=False), l1_ssim of the five renders and
# HumanRegularizers, with densification statistics) in three forms that must agree bit for bit.

def _chain_module():
    import importlib
    import sys
    tools = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools")
    if tools not in sys.path:
        sys.path.insert(0, tools)
    return importlib.import_module("bench_iteration_graph")


def _close(a, b, bound, where):
    """Equal NaN positions, and the other entries within `bound` (the synthetic fixture's face triplane takes NaN
    gradients in some rows, in every form alike)."""
    a, b = a.detach(), b.detach()
    assert a.shape == b.shape, where
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), (where, "NaN positions")
    d = (a[~na] - b[~nb]).abs().max().item() if (~na).any() else 0.0
    assert d <= bound, (where, d, bound)


@torch.no_grad()
def _sync_from(src, dst, n_shared, F):
    """dst's parameters, Adam state and densification buffers set to src's, in place (the tensors keep their
    addresses): each iteration below starts every form from the same state."""
    for gs, gd in zip(src.opt.param_groups[:n_shared], dst.opt.param_groups[:n_shared]):
        ps, pd_ = gs["params"][0], gd["params"][0]
        pd_.copy_(ps)
        ss, sd = src.opt.state.get(ps), dst.opt.state.get(pd_)
        if ss is not None:
            for k in ("step", "exp_avg", "exp_avg_sq"):
                sd[k].copy_(ss[k])
    tparams = src.table.parameters()
    tstate = [src.opt.state.get(t) for t in tparams]
    if dst.form == "table":
        for ts, td, st in zip(tparams, dst.table.parameters(), tstate):
            td.copy_(ts)
            if st is not None:
                for k in ("step", "exp_avg", "exp_avg_sq"):
                    dst.opt.state[td][k].copy_(st[k])
    else:
        for f in range(F):
            rows = frame_rows(tparams, f)
            for k, pa in dst.pd[str(f)].items():
                pa.copy_(rows[k].reshape(pa.shape))
                if tstate[0] is not None and tstate[0]["step"][f] > 0:
                    mom = {m: frame_rows([st[m] for st in tstate], f)[k].reshape(pa.shape)
                           for m in ("exp_avg", "exp_avg_sq")}
                    dst.opt.state[pa] = {"step": tstate[0]["step"][f].clone(), **{m: v.clone() for m, v in mom.items()}}
    for k, v in src.fr.densify.items():
        dst.fr.densify[k].copy_(v)


@pytest.mark.gpu
def test_iteration_graph_matches_eager_and_per_frame_route():
    """The full chain in three forms: per-frame ParameterDicts + decode_smplx_pose + per-frame groups (a), the table
    + frame-row Adam eager (b), and the table through IterationGraph (c).  The renderer's backward composite adds each
    Gaussian's gradient with float atomics (DESIGN.md f-15), so two runs of one frame differ in the last bits of the
    scene and human gradients and of grad_accum, whatever the form.  So every iteration starts a and b from c's
    state, and what does not pass through that backward is checked bit for bit: the loss terms, the visibility
    counts and radii of the densification statistics, every step count, and that the other frames' rows and state
    stay untouched.  What does: grad_accum to 1e-5 of its max (f-15's bound), the moments to 1e-4 of their max, and
    each parameter to twice its group's lr -- the most one Adam step can move it."""
    bm = _chain_module()
    dev = torch.device("cuda")
    F, H, W, NS = 4, 64, 96, 3000
    seq = [2, 0, 2, 3, 1, 1, 3, 0, 2, 3, 3, 0, 1]
    warm = [i < 5 for i in range(len(seq))]  # the key changes at iteration 5
    surgery_at = 9
    a = bm.Chain(dev, "frames", F, H, W, NS, use_graph=False, capacity=400_000)
    b = bm.Chain(dev, "table", F, H, W, NS, use_graph=False, capacity=400_000)
    c = bm.Chain(dev, "table", F, H, W, NS, use_graph=False, capacity=400_000)
    inputs = bm.make_inputs(dev, H, W)
    it, run = c.graph(inputs[0])
    lib = L.load()
    n_shared = len(a.opt.param_groups) - 9 * F
    for itr, f in enumerate(seq):
        x = inputs[itr % len(inputs)]
        if itr == surgery_at:
            rows = {k: v.detach()[:17].clone() for k, v in c.scene.items()}
            for ch in (a, b, c):
                ch.append_scene({k: v.clone() for k, v in rows.items()})
            with pytest.raises(StaleLayoutError, match="invalidate"):  # the graph of this key holds the old tensors
                for p in c.scene.values():
                    p.grad = torch.zeros_like(p)
                run(f, x, warm[itr])
            it.invalidate()
        if itr > 0:
            _sync_from(c, a, n_shared, F)
            _sync_from(c, b, n_shared, F)
        others = [t.detach().clone() for t in c.table.parameters()]
        for ch in (a, b, c):
            bm.set_lr(ch.opt, itr, len(seq))
        ta = a.eager(f, x, warm[itr])
        tb = b.eager(f, x, warm[itr])
        replay = warm[itr] in it._graphs
        n0 = lib.b2r_launch_count()
        with no_host_sync() if replay else contextlib.nullcontext():
            tc = run(f, x, warm[itr])
        if replay:
            assert lib.b2r_launch_count() == n0  # the whole iteration replayed: no host launch
        assert ta.keys() == tb.keys() == tc.keys()
        for k in ta:
            assert same(ta[k], tb[k]) and same(tb[k], tc[k]), (itr, k)
        for k in ("count", "radius_max"):
            assert same(a.fr.densify[k], b.fr.densify[k]) and same(b.fr.densify[k], c.fr.densify[k]), (itr, k)
        ga = c.fr.densify["grad_accum"]
        for ch in (a, b):
            _close(ch.fr.densify["grad_accum"], ga, 1e-5 * ga.nan_to_num().abs().max().item(), (itr, "grad_accum"))
        for gb, gc in zip(b.opt.param_groups, c.opt.param_groups):
            for pb, pc in zip(gb["params"], gc["params"]):
                _close(pb, pc, 2 * gc["lr"], (itr, gc["name"]))
                sb, sc = b.opt.state[pb], c.opt.state[pc]
                assert same(sb["step"], sc["step"]), (itr, gc["name"])
                for m in ("exp_avg", "exp_avg_sq"):
                    _close(sb[m], sc[m], 1e-4 * sc[m].nan_to_num().abs().max().item(), (itr, gc["name"], m))
        for ga_, gc in zip(a.opt.param_groups[:n_shared], c.opt.param_groups[:n_shared]):
            _close(ga_["params"][0], gc["params"][0], 2 * gc["lr"], (itr, gc["name"]))
        rows_c = frame_rows(c.table.parameters(), f)
        for k, pa in a.pd[str(f)].items():
            _close(pa, rows_c[k].reshape(pa.shape), 2e-3, (itr, k))
            assert a.opt.state[pa]["step"].item() == c.opt.state[c.table.pose]["step"][f].item()
        for t, before in zip(c.table.parameters(), others):  # the other frames' rows: untouched
            keep = torch.ones(t.shape[0], dtype=torch.bool, device=dev)
            keep[f] = False
            assert same(t.detach()[keep], before[keep]), (itr, "other rows")
    assert set(it._graphs) == {False}  # recaptured after the surgery; the warm-up key ended before it
    assert float(c.fr.densify["count"].sum()) > 0


# A reduced training iteration: the SMPL-X table, a scene image and a scene point set, an L1 + SSIM term, pose /
# expression / translation terms and the Adam step.

SH, SW, NP = 48, 64, 3001


def make_model(dev, F, seed=8):
    g = torch.Generator(device=dev).manual_seed(seed)
    frames = frame_values(F, dev, seed + 1)
    scene = {"img": nn.Parameter(torch.rand((3, SH, SW), generator=g, device=dev)),
             "mean": nn.Parameter(torch.randn((NP, 3), generator=g, device=dev))}
    return frames, scene


def chain(sp, scene, inputs, warm):
    """One iteration's loss terms from the frame's decoded parameters `sp` and the static inputs."""
    img = scene["img"] * inputs["bg"].view(3, 1, 1) + 0.01 * sp["trans"].sum()
    if warm:
        img = torch.clamp(img, max=0.9)
    l1, ss = l1_ssim(img, inputs["img"], inputs["bbox"])
    mean_term = ((scene["mean"] - inputs["R"].sum()) ** 2).mean()
    return {"l1": 0.8 * l1, "ssim": 0.2 * (1 - ss), "pose": (sp["full_pose"] ** 2).mean(),
            "expr": 0.1 * (sp["expr"] ** 2).mean(), "mean": mean_term}


def groups_of(scene, smplx):
    return [{"params": [scene["img"]], "name": "img_scene", "lr": 1e-2},
            {"params": [scene["mean"]], "name": "mean_scene", "lr": 1e-3}] + smplx


def iteration_inputs(dev, itr):
    g = torch.Generator(device=dev).manual_seed(100 + itr)
    return {"img": torch.rand((3, SH, SW), generator=g, device=dev),
            "bbox": torch.tensor([3.0 + itr, 2.0, 40.0, 30.0], device=dev),
            "R": torch.randn((3, 3), generator=g, device=dev), "bg": torch.rand(3, generator=g, device=dev)}


def surgery(opt, scene, dev):
    """Densification's optimizer surgery (module.py:17-36): append rows to the scene mean with zero moments."""
    gr = next(g for g in opt.param_groups if g["name"] == "mean_scene")
    old = gr["params"][0]
    st = opt.state.pop(old)
    p = nn.Parameter(torch.cat((old.detach(), torch.full((17, 3), 0.5, device=dev))))
    st["exp_avg"] = torch.cat((st["exp_avg"], torch.zeros((17, 3), device=dev)))
    st["exp_avg_sq"] = torch.cat((st["exp_avg_sq"], torch.zeros((17, 3), device=dev)))
    opt.state[p] = st
    gr["params"][0] = scene["mean"] = p


@pytest.mark.gpu
def test_iteration_graph_bit_identical_without_the_renderer():
    """Every op of this chain has a fixed-order backward, so here all three forms agree bit for bit over every
    iteration: parameters, Adam state and loss terms."""
    dev = torch.device("cuda")
    F, tot = 5, 14
    seq = [2, 0, 2, 4, 1, 1, 3, 0, 2, 4, 3, 0, 1, 2]
    warm = [i < 5 for i in range(tot)]  # the key changes at iteration 5
    surgery_at = 9

    # (a) the per-frame route: ParameterDicts, decode_smplx_pose, per-frame groups of torch.optim.Adam
    frames, scene_a = make_model(dev, F)
    pd = nn.ParameterDict({str(f): nn.ParameterDict({k: nn.Parameter(v.clone()) for k, v in d.items()})
                           for f, d in enumerate(frames)})
    smplx_a = [{"params": [pd[str(f)][k]], "name": f"smplx_{k}_{f}", "lr": 1e-3} for f in range(F) for k in FRAME_PARAMS]
    opt_a = torch.optim.Adam(groups_of(scene_a, smplx_a), lr=0.0, eps=1e-15)
    # (b) the table and frame-row Adam, eager; (c) the same through IterationGraph
    runs = {}
    for name in ("b", "c"):
        frames_, scene = make_model(dev, F)
        table = table_of(frames_)
        opt = Adam(groups_of(scene, [{"params": table.parameters(), "name": "smplx", "lr": 1e-3,
                                      "frame_rows": True}]), lr=0.0, eps=1e-15)
        runs[name] = (table, scene, opt)
    table_c, scene_c, opt_c = runs["c"]
    cur = {"warm": True}

    def step_fn(inputs, slot):
        losses = chain(table_c(slot), scene_c, inputs, cur["warm"])
        sum(losses.values()).backward()
        return losses

    it = IterationGraph(step_fn, opt_c, iteration_inputs(dev, 0))
    lib = L.load()
    for itr, f in enumerate(seq):
        inputs = iteration_inputs(dev, itr)
        if itr == surgery_at:
            surgery(opt_a, scene_a, dev)
            surgery(runs["b"][2], runs["b"][1], dev)
            surgery(opt_c, scene_c, dev)
            with pytest.raises(StaleLayoutError, match="invalidate"):  # the graph for this key holds the old mean
                opt_c.param_groups[1]["params"][0].grad = torch.zeros_like(scene_c["mean"])
                it.run(inputs, f, key=warm[itr])
            it.invalidate()
        for o in (opt_a, runs["b"][2], opt_c):
            set_lr(o, itr, tot)
        # (a)
        opt_a.zero_grad(set_to_none=True)
        la = chain(decode_smplx_pose(pd[str(f)]), scene_a, inputs, warm[itr])
        sum(la.values()).backward()
        opt_a.step()
        # (b)
        table_b, scene_b, opt_b = runs["b"]
        opt_b.zero_grad(set_to_none=True)
        lb = chain(table_b(f), scene_b, inputs, warm[itr])
        sum(lb.values()).backward()
        opt_b.step(rows=f)
        # (c)
        cur["warm"] = warm[itr]
        replay = warm[itr] in it._graphs
        n0 = lib.b2r_launch_count()
        with no_host_sync() if replay else contextlib.nullcontext():
            lc = it.run(inputs, f, key=warm[itr])
        if replay:
            assert lib.b2r_launch_count() == n0  # a replay: no host launch
        for k in la:
            assert same(la[k], lb[k]) and same(lb[k], lc[k]), (itr, k)
        assert same(scene_a["img"], scene_b["img"]) and same(scene_b["img"], scene_c["img"]), itr
        assert same(scene_a["mean"], scene_b["mean"]) and same(scene_b["mean"], scene_c["mean"]), itr
        for tb, tc in zip(table_b.parameters(), table_c.parameters()):
            assert same(tb, tc), itr
            for k in ("step", "exp_avg", "exp_avg_sq"):
                assert same(opt_b.state[tb][k], opt_c.state[tc][k]), (itr, k)
        rows = frame_rows(table_b.parameters(), f)
        for k in FRAME_PARAMS:
            pa = pd[str(f)][k]
            assert same(pa, rows[k]), (itr, k)
            sa = opt_a.state[pa]
            for m in ("exp_avg", "exp_avg_sq"):
                assert same(sa[m], frame_rows([opt_b.state[t][m] for t in table_b.parameters()], f)[k]), (itr, k, m)
    assert set(it._graphs) == {False}  # recaptured after the surgery; the warm-up key ended before it
