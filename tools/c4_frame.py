"""The C4 training frame the op benchmarks time their ops in, and the SMPL-X rig fixtures it is built from.

The frame is tools/bench_human_regs.py's frame (the f-7 human chain with the networks as ops, nearest_rows,
skin_gaussians, VertexNormals, `TrainingFrameRenderer(use_graph=True)`, `l1_ssim` of the five renders and the
regularisers as the op, one backward per frame) with the real SMPL-X rig in front instead of a fixed mesh and a random
joint_mats leaf.  The rig's pose_6d feeds the pose-conditioned stacks, its meshes and offsets build mean_3d /
mean_3d_refined as module.py:528-539 does, and the template is placed in the frame skin_gaussians poses in, so the
human is in view.  Each benchmark arm replaces some of the frame's stages with a `FrameArm`.
"""
import os
import sys
from functools import partial
from typing import Callable, NamedTuple, Optional

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, stats  # noqa: E402
from bench_human_nets import stack  # noqa: E402
from bench_human_regs import INPUTS as REG_INPUTS  # noqa: E402
from bench_human_regs import setup as regs_setup  # noqa: E402
from exavatar_release_b200 import TrainingFrameRenderer  # noqa: E402
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.geometry import VertexNormals, nearest_rows  # noqa: E402
from exavatar_release_b200.human_nets import TriplaneFeatures, gn_mlp  # noqa: E402
from exavatar_release_b200.losses import l1_ssim  # noqa: E402
from exavatar_release_b200.plan import RENDERS  # noqa: E402
from exavatar_release_b200.skinning import skin_gaussians  # noqa: E402
from exavatar_release_b200.smplx_rig import (SmplxRig, axis_angle_to_matrix, batch_rodrigues,  # noqa: E402
                                             matrix_to_axis_angle, matrix_to_rotation_6d, rigid_transform, upsample)
from exavatar_release_b200.synthetic import WORKLOADS, Workload, make_human_mesh, make_population_assets  # noqa: E402
from exavatar_release_b200.synthetic import make_smplx_model  # noqa: E402

BOX = (102.4, 60.8, 307.5, 396.2)  # the LPIPS crop box: ~60 % of a 512 x 512 image (tools/bench_l1_ssim.py)


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


class FrameArm(NamedTuple):
    """The stages one arm of the frame replaces; a stage left None runs the frame's default."""
    rig: Optional[Callable] = None    # (rig, d, x) -> the rig's six outputs; default rig(*x)
    scene: Optional[Callable] = None  # (scene, cam) -> the scene's asset dict; default the scene leaves
    mesh: Optional[Callable] = None   # (rig, shape_param, joint_offset, full_pose, expr, trans, cam_R, cam_t), unused
    loss: Optional[Callable] = None   # (renders, target) -> a term added to the frame's loss; default none
    camera: Optional[Callable] = None  # (img_shape, cam, bg) -> the renderer's raster settings; default render_settings


def frames_per_second(a, dev, arms, use_graph=True):
    """C4 training frames/s of each arm (name -> FrameArm), arms alternated window by window: {"frame_<name>": stats}."""
    frame, fr = make_frame(dev, use_graph)
    times = alternate({k: partial(frame, arm) for k, arm in arms.items()}, a.frames, a.rounds, 3)
    if fr.overflowed():
        raise SystemExit("c4_frame: a render overflowed its list capacity")
    return {f"frame_{k}": stats([1 / s for s in v]) for k, v in times.items()}


def make_frame(dev, use_graph=True):
    """(frame, renderer): `frame(arm)` runs one C4 training frame, forward and backward, with the stages of `arm`
    (a FrameArm); `renderer` is its TrainingFrameRenderer."""
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
                               use_graph=use_graph)
    white = torch.ones(3, device=dev)
    leaves = [tp, tpf, trans, *x, *lv.values()] + [p for t, hs in nets.values() for mm in [t, *hs]
                                                   for p in mm.parameters()]

    def frame(arm):
        out = arm.rig(rig, d, x) if arm.rig else rig(*x)
        if arm.mesh:
            arm.mesh(rig, *x, trans, R, tc)
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
        st = arm.camera((H, W), cam, white) if arm.camera else None
        o = fr(arm.scene(scene, cam) if arm.scene else lv, hv, rv, cam, bg, raster_settings=st)
        loss = 0
        for r in RENDERS:
            l1, ss = l1_ssim(o[r]["img"], target)
            loss = loss + 0.8 * l1 + 0.2 * (1 - ss)
        loss = loss + sum(regs(mesh.detach(), *[y[k] for k in REG_INPUTS]).values())
        if arm.loss:
            loss = loss + arm.loss(o, target)
        loss.backward()
        for v in leaves:
            v.grad = None

    return frame, fr
