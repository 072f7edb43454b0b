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
  4. frame_*:   C4 training frames/s of tools/bench_human_regs.py's frame (the f-7 human chain with the networks as
                ops, nearest_rows, skin_gaussians, VertexNormals, `TrainingFrameRenderer(use_graph=True)`, `l1_ssim` of
                the five renders and the regularisers as the op, one backward per frame) with the real rig in front
                instead of a fixed mesh and a random joint_mats leaf: the rig of arm 1 (frame_rig_ops) or the op eager
                (frame_rig_op).  The rig's pose_6d feeds the pose-conditioned stacks, its meshes and offsets build
                mean_3d / mean_3d_refined as module.py:528-539 does, and the template is placed in the frame
                skin_gaussians poses in, so the human is in view.
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Host
syncs per call are counted under torch.cuda.set_sync_debug_mode("warn"); device time and launch count per call come from
a separate torch.profiler run.  Prints the card name and power limit with the numbers.
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
from exavatar_release_b200.smplx_rig import (SmplxRig, axis_angle_to_matrix, batch_rodrigues,  # noqa: E402
                                             matrix_to_axis_angle, matrix_to_rotation_6d, rigid_transform, upsample)
from exavatar_release_b200.synthetic import make_human_mesh, make_smplx_model  # noqa: E402


def setup(dev, model=None):
    model = make_smplx_model(make_human_mesh()) if model is None else model
    rig = SmplxRig(**model, device=dev)
    m = rig.model
    f = lambda t: t.to(dev, torch.float32)  # noqa: E731
    d = {k: f(m[k]) for k in ("v_template", "face_offset", "shapedirs", "expr_dirs", "posedirs", "J_regressor",
                              "lbs_weights", "pose_mean", "neutral_body_pose")}
    d.update(V=m["V"], P=m["P"], J=m["J"], NE=m["NE"], n_body=m["n_body"], parents=m["parents"].tolist(),
             sub1=m["sub1"], sub2=m["sub2"], mask=m["mask"].to(dev)[:, None].float())
    V, P = d["V"], d["P"]
    # HumanGaussian.init's upsampled tables (module.py:297-306)
    d["pose_dirs"] = upsample(d["posedirs"].t().reshape(V, -1), d["sub1"], d["sub2"]).reshape(P * 3, -1).t().contiguous()
    d["expr_dirs_up"] = upsample(d["expr_dirs"].reshape(V, -1), d["sub1"], d["sub2"]).view(P, 3, -1)
    g = torch.Generator().manual_seed(0)
    J = d["J"]
    x = [torch.randn(m["NB"], generator=g), 0.01 * torch.randn(J, 3, generator=g), 0.3 * torch.randn(J, 3, generator=g),
         torch.randn(m["NE"], generator=g)]
    x = [t.to(dev).requires_grad_() for t in x]
    w = [torch.randn(s, generator=g).to(dev) for s in ((P, 3), (J, 4, 4), (P, 3))]
    return rig, d, x, w


def body_forward(d, beta, jo, full_pose):
    """smplx_layer(...) with face_offset and joint_offset (body_models.py SMPLX.forward + lbs.lbs), landmarks omitted."""
    V, J = d["V"], d["J"]
    comps = torch.cat([beta, torch.zeros(d["NE"], device=beta.device)])
    dirs = torch.cat([d["shapedirs"], d["expr_dirs"]], -1)
    vs = (d["v_template"] + d["face_offset"]) + torch.einsum("l,mkl->mk", comps, dirs)
    w = torch.ones(J, 1, device=beta.device)
    w[0] = 0  # smpl_x.get_joint_offset
    Jr = d["J_regressor"] @ vs + jo * w
    rot = batch_rodrigues(full_pose.view(-1, 3))
    eye = torch.eye(3, device=beta.device)
    v_posed = vs + ((rot[1:] - eye).view(1, -1) @ d["posedirs"]).view(V, 3)
    posed, A = rigid_transform(rot, Jr, d["parents"])
    T = (d["lbs_weights"] @ A.view(J, 16)).view(V, 4, 4)
    verts = (T @ torch.cat([v_posed, torch.ones_like(v_posed[:, :1])], 1)[:, :, None])[:, :3, 0]
    return verts, posed


def rig_ops(d, beta, jo, pose, expr):
    dev, J, nb = beta.device, d["J"], d["n_body"]
    zero = torch.zeros(1, 3, device=dev)
    neutral = torch.zeros(J, 3, device=dev)
    neutral[1:1 + nb] = d["neutral_body_pose"]
    mesh_wo, jnp = body_forward(d, beta, jo, neutral.view(-1) + d["pose_mean"])
    mesh = upsample(mesh_wo, d["sub1"], d["sub2"])  # edge tables uploaded per call
    inv = torch.cat([zero, matrix_to_axis_angle(torch.inverse(axis_angle_to_matrix(d["neutral_body_pose"]))),
                     matrix_to_axis_angle(torch.inverse(axis_angle_to_matrix(zero))), torch.zeros(J - nb - 2, 3, device=dev)])
    _, A_inv = rigid_transform(axis_angle_to_matrix(inv), jnp, d["parents"])
    _, jzp = body_forward(d, beta, jo, d["pose_mean"])
    _, A_f = rigid_transform(axis_angle_to_matrix(pose), jzp, d["parents"])
    joint_mats = torch.bmm(A_f, A_inv)
    feat = (axis_angle_to_matrix(pose[1:]) - torch.eye(3, device=dev)).view(1, -1)
    pose_offset = (feat.detach() @ d["pose_dirs"]).view(d["P"], 3) * d["mask"]
    expr_offset = (expr[None, None, :] * d["expr_dirs_up"]).sum(2)
    pose_6d = matrix_to_rotation_6d(axis_angle_to_matrix(pose[1:1 + nb])).view(-1).detach()
    return mesh, mesh_wo.detach(), joint_mats, pose_offset, expr_offset, pose_6d


def frames_per_second(a, dev, extras=None, scenes=None, poses=None, meshes=None):
    """Arm 4.  `extras` (name -> fn(renders, target) -> loss term): instead of the two rig arms, one arm per entry, each
    with the rig op and that term added to the frame's loss (tools/bench_lpips.py).  `scenes` (name -> fn(scene, cam)
    -> scene asset dict, given the population's activated assets and the camera): one arm per entry, each with the rig
    op and the scene's assets built by that function every frame (tools/bench_scene_assets.py).  `poses` (name -> fn()
    -> (J,3) axis-angle pose): one arm per entry, each with the rig op fed the pose that function decodes every frame
    from the frame's 6D parameters (tools/bench_human_assets.py).  `meshes` (name -> fn(rig, shape_param, joint_offset,
    full_pose, expr, trans, cam_R, cam_t) -> (V,3) mesh or None): one arm per entry, each with the rig op and the
    frame's SMPL-X body mesh of get_smplx_outputs computed by that function every frame, its result unused as in
    ExAvatar's training step (tools/bench_smplx_body.py)."""
    from bench_human_nets import stack
    from bench_human_regs import INPUTS as REG_INPUTS
    from bench_human_regs import setup as regs_setup
    from exavatar_release_b200 import TrainingFrameRenderer
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.geometry import VertexNormals, nearest_rows
    from exavatar_release_b200.human_nets import TriplaneFeatures, gn_mlp
    from exavatar_release_b200.losses import l1_ssim
    from exavatar_release_b200.plan import RENDERS
    from exavatar_release_b200.skinning import skin_gaussians
    from exavatar_release_b200.synthetic import WORKLOADS, Workload, make_population_assets
    dr, regs, _ = regs_setup(dev)
    m, P = dr["m"], dr["P"]
    c4 = WORKLOADS["C4"]
    H, W = c4.height, c4.width
    wl = Workload("C4 with the synthetic mesh's Gaussians", H, W, P, c4.n_scene, 0, True)
    scene, human, _ = make_population_assets(wl, seed=0, device=dev)
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    R, tc = cam["R"], cam["t"]
    to_cam = lambda x: (x.double() @ R.cpu().double().t() + tc.cpu().double().view(1, 3)).float()  # noqa: E731
    rig, d, x, _ = setup(dev, make_smplx_model(dict(m, targets=to_cam(m["targets"]))))
    trans = torch.zeros(3, device=dev, requires_grad=True)
    skw = upsample(d["lbs_weights"], d["sub1"], d["sub2"]).contiguous()
    sm, mask = m["self_map"].to(dev), d["mask"]
    verts = dr["mesh"]
    tri = TriplaneFeatures(verts, verts[:, 1] > 0.6)
    vn = VertexNormals(m["faces"], P, flip=m["flip"].to(dev))
    torch.manual_seed(3)
    nets = {"geo": stack(96, [3, 1]), "geo_offset": stack(96 + 126, [3, 1]), "rgb": stack(96, None, 3),
            "rgb_offset": stack(96 + 126 + 3, None, 3)}
    g = torch.Generator().manual_seed(5)
    tp = (0.3 * torch.randn((3, 32, 128, 128), generator=g)).to(dev).requires_grad_()
    tpf = (0.3 * torch.randn((3, 32, 128, 128), generator=g)).to(dev).requires_grad_()
    lv = {k: v.detach().clone().requires_grad_() for k, v in scene.items()}
    bg = torch.tensor([0.3, 0.7, 0.2], device=dev)
    target = torch.rand((3, H, W), generator=torch.Generator(device=dev).manual_seed(6), device=dev)
    fr = TrainingFrameRenderer(scene["mean_3d"].shape[0], P, (H, W), dev, {"A": 8_000_000, "B": 8_000_000},
                               use_graph=True)
    leaves = [tp, tpf, trans, *x, *lv.values()] + [p for t, hs in nets.values() for mm in [t, *hs]
                                                   for p in mm.parameters()]

    def frame(which):
        if poses is not None:
            out = rig(x[0], x[1], poses[which](), x[3])
        else:
            out = rig_ops(d, *x) if which == "rig_ops" else rig(*x)
        if meshes is not None:
            meshes[which](rig, *x, trans, R, tc)
        mesh, mesh_wo, joint_mats, pose_offset, expr_offset, pose = out
        f = tri(tp, tpf)
        net = lambda k, ins: gn_mlp(ins, *nets[k])  # noqa: E731
        geo, geo_off, rgb = net("geo", [f]), net("geo_offset", [f, pose]), net("rgb", [f])
        mean_3d = mesh + 0.01 * geo[:, :3]
        mean_3d_r = mean_3d + 0.005 * geo_off[:, :3] * (1 - mask) + pose_offset
        mean_3d, mean_3d_r = mean_3d + expr_offset, mean_3d_r + expr_offset
        rows = nearest_rows(mean_3d.detach(), mesh_wo.contiguous(), sm)
        posed, posed_r = skin_gaussians(mean_3d, mean_3d_r, skw, rows, joint_mats, trans, R, tc)
        rgb_off = net("rgb_offset", [f, pose, vn(posed_r)])
        y = {"mean_offset": 0.01 * geo[:, :3], "mean_offset_offset": 0.005 * geo_off[:, :3],
             "scale_offset": 0.1 * geo_off[:, 3:], "scale": human["scale"] * torch.exp(0.1 * geo[:, 3:]),
             "scale_refined": human["scale"] * torch.exp(0.1 * (geo[:, 3:] + geo_off[:, 3:])),
             "rgb": (torch.tanh(rgb) + 1) / 2, "rgb_refined": (torch.tanh(rgb + rgb_off) + 1) / 2, "joint_offset": x[1]}
        hv = dict(human, mean_3d=posed, scale=y["scale"], rgb=y["rgb"])
        rv = dict(human, mean_3d=posed_r, scale=y["scale_refined"], rgb=y["rgb_refined"])
        o = fr(lv if scenes is None else scenes[which](scene, cam), hv, rv, cam, bg)
        loss = 0
        for r in RENDERS:
            l1, ss = l1_ssim(o[r]["img"], target)
            loss = loss + 0.8 * l1 + 0.2 * (1 - ss)
        loss = loss + sum(regs(mesh.detach(), *[y[k] for k in REG_INPUTS]).values())
        if extras is not None:
            loss = loss + extras[which](o, target)
        loss.backward()
        for v in leaves:
            v.grad = None

    arms = (tuple(scenes) if scenes is not None else tuple(poses) if poses is not None else
            tuple(meshes) if meshes is not None else ("rig_ops", "rig_op") if extras is None else tuple(extras))
    for k in arms:
        for _ in range(3):
            frame(k)
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k in arms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.frames):
                frame(k)
            torch.cuda.synchronize()
            times[k].append(a.frames / (time.perf_counter() - t0))
    if fr.overflowed():
        raise SystemExit("bench_smplx_rig: a render overflowed its list capacity")
    return {f"frame_{k}": {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="rig calls per timed window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=10, help="training frames per timed window")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_smplx_rig: needs a CUDA device (there is no CPU measurement)")
    dev = torch.device("cuda:0")
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
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            run_op(xg)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run_op(xg)
    arms = {"ops": run_ops, "op": run_op, "op_graph": graph.replay}
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
    for k in ("ops", "op"):
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
        prof[k] = {"device_ms": sum(e.device_time for e in ev) / 1e3, "launches": len(ev)}

    res = {"card": card(), "V": d["V"], "P": d["P"], "J": d["J"],
           "rig_ms": {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()},
           "host_syncs_per_call": syncs, "profile": prof, "ops_vs_op": agree,
           "frames_per_s": frames_per_second(a, dev)}
    print(json.dumps(res, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
