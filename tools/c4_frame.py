"""The C4 training frame the op benchmarks time their ops in, and the SMPL-X rig fixtures it is built from.

The frame is tools/bench_human_regs.py's frame (the f-7 human chain with the networks as ops, nearest_rows,
skin_gaussians, VertexNormals, `TrainingFrameRenderer(use_graph=True)`, `l1_ssim` of the five renders and the
regularisers as the op, one backward per frame) with the real SMPL-X rig in front instead of a fixed mesh and a random
joint_mats leaf.  The rig's pose_6d feeds the pose-conditioned stacks, its meshes and offsets build mean_3d /
mean_3d_refined as module.py:528-539 does, and the template is placed in the frame skin_gaussians poses in, so the
human is in view.  Each benchmark arm replaces some of the frame's stages with a `FrameArm`.

`SyntheticAvatar` is the same human as a trained avatar for the animation path: what `AvatarAnimator` takes, a motion
folder of it (`write_motion`), and the full forward and video frame through the ops that the animator must reproduce.
For the test pass it also builds a test split's tables, scene and face inputs (`test_setup`), the `AvatarTester` over
them, and `test_chain`, Model.forward(mode='test') eagerly through the ops, which the tester must reproduce.
"""
import json
import math
import os
import sys
from functools import partial
from typing import Callable, NamedTuple, Optional

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, stats  # noqa: E402
from bench_human_nets import stack  # noqa: E402
from bench_human_regs import INPUTS as REG_INPUTS  # noqa: E402
from bench_human_regs import setup as regs_setup  # noqa: E402
from exavatar_release_b200 import TrainingFrameRenderer  # noqa: E402
from exavatar_release_b200.animation import animation_panel, orbit_points  # noqa: E402
from exavatar_release_b200.human_assets import POSE_KEYS, POSE_ROWS, HumanAssets  # noqa: E402
from exavatar_release_b200.mesh_render import ShadedMeshRenderer  # noqa: E402
from exavatar_release_b200.rasterizer import GaussianRasterizer  # noqa: E402
from exavatar_release_b200.renderer import device_render_settings  # noqa: E402
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


def write_motion_frame(root, idx, smplx, cam, img):
    """One frame of a motion folder in the layout ExAvatar's animation scripts read: the SMPL-X parameters and the
    camera as JSON, the source frame as a PNG."""
    for sub, d in (("smplx_optimized/smplx_params_smoothed", smplx), ("cam_params", cam)):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
        with open(os.path.join(root, sub, f"{idx}.json"), "w") as f:
            json.dump(d, f)
    os.makedirs(os.path.join(root, "frames"), exist_ok=True)
    if not cv2.imwrite(os.path.join(root, "frames", f"{idx}.png"), img):
        raise OSError(f"cannot write frame {idx}'s PNG under {root}")


class SyntheticAvatar:
    """A trained HumanGaussian of C4 size on the synthetic SMPL-X rig, seeded: rig, triplanes, all four GroupNorm
    stacks (the offset heads scaled so the Gaussians stay on the body), upsampled skinning weights, masks and the mesh
    renderer -- what AvatarAnimator takes, and the full forward it must reproduce."""

    def __init__(self, dev):
        hm = make_human_mesh()
        model = make_smplx_model(hm)
        self.rig, d, x, _ = setup(dev, model)
        self.beta, self.jo, self.pose, self.expr = (t.detach() for t in x)
        P = self.rig.P
        self.skw = upsample(d["lbs_weights"], d["sub1"], d["sub2"]).contiguous()
        self.self_map = hm["self_map"].to(dev)
        verts = hm["verts"].to(dev)
        self.tri = TriplaneFeatures(verts, verts[:, 1] > 0.6)
        self.ha = HumanAssets(model["is_rhand"], model["is_lhand"], model["is_face_expr"], device=dev)
        self.vn = VertexNormals(hm["faces"], P, flip=hm["flip"].to(dev))
        self.mesh_r = ShadedMeshRenderer(hm["base_faces"], self.rig.V, device=dev)
        torch.manual_seed(3)
        self.nets = {"geo": stack(96, [3, 1]), "geo_offset": stack(96 + 126, [3, 1]), "rgb": stack(96, None, 3),
                     "rgb_offset": stack(96 + 126 + 3, None, 3)}
        with torch.no_grad():
            for k in ("geo", "geo_offset"):
                mo, sc = self.nets[k][1]
                mo[0].weight.mul_(1e-3)
                mo[0].bias.zero_()
                sc[0].weight.mul_(1e-2)
                sc[0].bias.fill_(math.log(0.004) if k == "geo" else 0.0)
        g = torch.Generator().manual_seed(5)
        self.tp = (0.3 * torch.randn((3, 32, 128, 128), generator=g)).to(dev)
        self.tpf = (0.3 * torch.randn((3, 32, 128, 128), generator=g)).to(dev)

    def animator(self, motion, **kw):
        from exavatar_release_b200 import AvatarAnimator
        return AvatarAnimator(motion, self.rig, self.tri, self.ha, self.mesh_r, triplane=self.tp,
                              triplane_face=self.tpf, geo_net=self.nets["geo"], rgb_net=self.nets["rgb"],
                              shape_param=self.beta, joint_offset=self.jo, skinning_weight=self.skw,
                              self_map=self.self_map, **kw)

    def write_motion(self, root, frame_idx, H, W, near=None):
        """A motion folder of len(frame_idx) poses, expressions, translations, cameras near the identity and random
        H x W frames; position `near` has its body 1.5 m closer to the camera."""
        for i, idx in enumerate(frame_idx):
            g = torch.Generator().manual_seed(40 + i)
            pose = (self.pose.cpu() + 0.1 * torch.randn(self.pose.shape, generator=g)).reshape(-1)
            smplx, r0 = {}, 0
            for k, n in zip(POSE_KEYS, POSE_ROWS):
                smplx[k] = pose[3 * r0:3 * (r0 + n)].tolist()
                r0 += n
            smplx["expr"] = (self.expr.cpu() + 0.5 * torch.randn(self.expr.shape, generator=g)).tolist()
            trans = 0.03 * torch.randn(3, generator=g)
            if i == near:
                trans[2] -= 1.5
            smplx["trans"] = trans.tolist()
            a = 0.1 * torch.randn(2, generator=g).double()
            Ry = torch.tensor([[math.cos(a[1]), 0.0, math.sin(a[1])], [0.0, 1.0, 0.0],
                               [-math.sin(a[1]), 0.0, math.cos(a[1])]], dtype=torch.float64)
            Rx = torch.tensor([[1.0, 0.0, 0.0], [0.0, math.cos(a[0]), -math.sin(a[0])],
                               [0.0, math.sin(a[0]), math.cos(a[0])]], dtype=torch.float64)
            cam = {"R": (Rx @ Ry).tolist(), "t": (0.05 * torch.randn(3, generator=g)).tolist(),
                   "focal": [1.2 * H, 1.2 * H], "princpt": [W / 2, H / 2]}
            img = np.random.default_rng(i).integers(0, 256, (H, W, 3), dtype=np.uint8)
            write_motion_frame(root, idx, smplx, cam, img)

    @torch.no_grad()
    def full_chain(self, fr, i, image_shape, orbit=None):
        """Video frame i (its position) as HumanGaussian.forward and the scripts compute it, through the existing ops:
        the rig, the triplane, all four stacks, both sets posed, the refined one's normals and colours computed and
        discarded, then the render, the body mesh (with `orbit`, an OrbitCamera: its camera and orbit_points), the mesh
        panel and the video panel.  `fr` holds pose (55,3), expr, trans, cam and frame (H,W,3) uint8 CUDA tensors."""
        pose, expr, trans, cam = fr["pose"], fr["expr"], fr["trans"], fr["cam"]
        out = self.rig(self.beta, self.jo, pose, expr)
        f = self.tri(self.tp, self.tpf)
        net = lambda k, ins: gn_mlp(ins, *self.nets[k])  # noqa: E731
        geo, geo_off, rgb = net("geo", [f]), net("geo_offset", [f, out.pose_6d]), net("rgb", [f])
        ga = self.ha.geometry(out.mesh_neutral_pose, out.pose_offset, out.expr_offset, geo, geo_off)
        rows = nearest_rows(ga["mean_3d"], out.mesh_neutral_pose_wo_upsample.contiguous(), self.self_map)
        posed, posed_r = skin_gaussians(ga["mean_3d"], ga["mean_3d_refined"], self.skw, rows, out.joint_mats, trans,
                                        cam["R"], cam["t"])
        rgb_c, _ = self.ha.colors(rgb, net("rgb_offset", [f, out.pose_6d, self.vn(posed_r)]))
        body = (self.beta, self.jo, pose, expr, trans)
        if orbit is not None:
            mesh, joints = self.rig.body_mesh(*body, cam["R"], cam["t"], joints=True)
            render_cam = orbit(cam, joints[0], i)
            mesh = orbit_points(mesh, orbit, view=True)
            posed = orbit_points(posed, orbit)
        else:
            mesh = self.rig.body_mesh(*body)
            render_cam = cam
        dev = posed.device
        render = GaussianRasterizer(device_render_settings(image_shape, render_cam, torch.ones(3, device=dev)))(
            means3D=posed, means2D=torch.zeros_like(posed), opacities=self.ha.opacity, colors_precomp=rgb_c,
            scales=ga["scale"], rotations=self.ha.rotation)[0]
        mesh_panel = self.mesh_r(mesh, cam, torch.full((*image_shape, 3), 255.0, device=dev))
        return {"mean_3d": posed, "scale": ga["scale"], "rgb": rgb_c, "render": render, "mesh_panel": mesh_panel,
                "panel": animation_panel(fr["frame"], mesh_panel, render)}

    def test_setup(self, root, frame_idx, H, W, capacity, n_scene=None, slots=None):
        """A test split of len(frame_idx) frames at H x W written under `root` (segmentations/%05d.png) and read into
        the device tables, the C4 scene, the face render's inputs and a TrainingFrameRenderer(use_graph=False) of
        `capacity` list entries per pass.  The SMPL-X table has the slots `slots` (default the split's frames in
        reverse order plus one frame that is not in the split), so table rows and slots differ."""
        from exavatar_release_b200 import FaceMeshRenderer, FrameTable, SegmentationTable, SmplxParamTable
        from exavatar_release_b200.synthetic import make_face_mesh
        dev = self.beta.device
        n_scene = WORKLOADS["C4"].n_scene if n_scene is None else n_scene
        slots = [str(f) for f in reversed(frame_idx)] + ["777777"] if slots is None else slots
        params, imgs, cams = {}, [], []
        for key in slots:
            g = torch.Generator().manual_seed(1000 + int(key) % 9973)
            pose = self.pose.cpu() + 0.1 * torch.randn(self.pose.shape, generator=g)
            six = matrix_to_rotation_6d(axis_angle_to_matrix(pose.to(torch.float64))).to(torch.float32)
            d, r0 = {}, 0
            for k, n in zip(POSE_KEYS, POSE_ROWS):
                d[k] = six[r0:r0 + n].reshape(6) if n == 1 else six[r0:r0 + n].clone()
                r0 += n
            d["expr"] = self.expr.cpu() + 0.5 * torch.randn(self.expr.shape, generator=g)
            d["trans"] = 0.03 * torch.randn(3, generator=g)
            params[key] = {k: v.to(dev) for k, v in d.items()}
        for i, idx in enumerate(frame_idx):
            g = torch.Generator().manual_seed(40 + i)
            a = 0.1 * torch.randn(2, generator=g).double()
            Ry = torch.tensor([[math.cos(a[1]), 0.0, math.sin(a[1])], [0.0, 1.0, 0.0],
                               [-math.sin(a[1]), 0.0, math.cos(a[1])]], dtype=torch.float64)
            Rx = torch.tensor([[1.0, 0.0, 0.0], [0.0, math.cos(a[0]), -math.sin(a[0])],
                               [0.0, math.sin(a[0]), math.cos(a[0])]], dtype=torch.float64)
            cams.append({"R": (Rx @ Ry).float().numpy(), "t": (0.05 * torch.randn(3, generator=g)).numpy(),
                         "focal": np.array([1.2 * H, 1.2 * H], np.float32),
                         "princpt": np.array([W / 2, H / 2], np.float32)})
            imgs.append(np.random.default_rng(i).integers(0, 256, (H, W, 3), dtype=np.uint8))
            write_segmentation(root, idx, H, W, seed=100 + i)
        table = SmplxParamTable.from_param_dict(params)
        frames = FrameTable.from_dataset(TestSplit(frame_idx, imgs, cams), dev, slots=table.frames, workers=0)
        masks = SegmentationTable.from_folder(root, frames, dev)
        scene = _test_scene(dev, n_scene)
        fm = make_face_mesh()
        face_r = FaceMeshRenderer(fm["vertex_uv"], fm["face_uv"], fm["faces"], fm["vertex_idx"].shape[0], device=dev)
        renderer = TrainingFrameRenderer(n_scene, self.rig.P, (H, W), dev, {"A": capacity, "B": capacity})
        return TestSetup(frames, table, masks, scene, torch.tensor([3.0], device=dev), face_r,
                         fm["texture"].to(dev)[None].contiguous(), fm["vertex_idx"].to(dev), renderer)

    def tester(self, s, **kw):
        """An AvatarTester of this avatar over the TestSetup `s` (keyword arguments: scorer, masks, png, ...)."""
        from exavatar_release_b200 import AvatarTester
        return AvatarTester(s.frames, s.params, self.rig, self.tri, self.ha, self.vn, s.face_renderer, s.renderer,
                            triplane=self.tp, triplane_face=self.tpf, geo_net=self.nets["geo"],
                            geo_offset_net=self.nets["geo_offset"], rgb_net=self.nets["rgb"],
                            rgb_offset_net=self.nets["rgb_offset"], shape_param=self.beta, joint_offset=self.jo,
                            skinning_weight=self.skw, self_map=self.self_map, scene=s.scene,
                            active_sh_degree=s.sh_degree, face_uvmap=s.face_uvmap, face_vertex_idx=s.face_vertex_idx,
                            **kw)

    @torch.no_grad()
    def test_chain(self, s, slot, png=True):
        """Model.forward(mode='test') of the frame in host slot `slot` of TestSetup `s`, eagerly through the ops with
        the tables read by host slot: the frame, its SMPL-X parameters, the rig, the triplane, all four stacks,
        geometry without the warm-up clamp, both sets posed, normals and colours, the scene in rgb mode with the
        frame's camera, the device camera, the five renders with bg_human = ones, the two face renders and
        test_outputs.  Returns test_outputs' dict plus "gt" (1,3,H,W)."""
        from exavatar_release_b200 import scene_assets, test_outputs
        data = s.frames(slot)
        cam = {k: v[0] for k, v in data["cam_param"].items()}
        sp = s.params(slot)
        out = self.rig(self.beta, self.jo, sp["full_pose"], sp["expr"])
        f = self.tri(self.tp, self.tpf)
        net = lambda k, ins: gn_mlp(ins, *self.nets[k])  # noqa: E731
        geo, geo_off, rgb = net("geo", [f]), net("geo_offset", [f, out.pose_6d]), net("rgb", [f])
        ga = self.ha.geometry(out.mesh_neutral_pose, out.pose_offset, out.expr_offset, geo, geo_off, warmup=False)
        rows = nearest_rows(ga["mean_3d"], out.mesh_neutral_pose_wo_upsample.contiguous(), self.self_map)
        posed, posed_r = skin_gaussians(ga["mean_3d"], ga["mean_3d_refined"], self.skw, rows, out.joint_mats,
                                        sp["trans"], cam["R"], cam["t"])
        rgb_c, rgb_r = self.ha.colors(rgb, net("rgb_offset", [f, out.pose_6d, self.vn(posed_r)]))
        human = dict(mean_3d=posed, opacity=self.ha.opacity, scale=ga["scale"], rotation=self.ha.rotation, rgb=rgb_c)
        refined = dict(mean_3d=posed_r, opacity=self.ha.opacity, scale=ga["scale_refined"], rotation=self.ha.rotation,
                       rgb=rgb_r)
        sc = s.scene
        scene = scene_assets(sc["mean"], sc["opacity_logit"], sc["log_scale"], sc["rotation6d"], sc["feature_dc"],
                             sc["feature_rest"], s.sh_degree, cam)
        shape = (s.frames.height, s.frames.width)
        ones = torch.ones(3, device=posed.device)
        renders = s.renderer(scene, human, refined, cam, ones, raster_settings=device_render_settings(shape, cam, ones))
        face = s.face_renderer(s.face_uvmap, posed[None, s.face_vertex_idx, :], cam, shape)
        face_r = s.face_renderer(s.face_uvmap, posed_r[None, s.face_vertex_idx, :], cam, shape)
        res = test_outputs(renders, face, face_r, gt=data["img"], png=png)
        res["gt"] = data["img"]
        return res


class TestSplit:
    """An ExAvatar-shaped test split held in memory, for `FrameTable.from_dataset`: `frame_idx_list` and dataset[i]'s
    dict of img (3,H,W) k / 255, mask, bbox and the frame's camera."""

    def __init__(self, frame_idx, imgs, cams):
        self.frame_idx_list = list(frame_idx)
        self.imgs, self.cams = imgs, cams

    def __len__(self):
        return len(self.frame_idx_list)

    def __getitem__(self, i):
        img = self.imgs[i]  # (H, W, 3) RGB bytes
        H, W = img.shape[:2]
        return {"img": torch.from_numpy(img.transpose(2, 0, 1).astype(np.float32)) / 255.,
                "mask": torch.ones((1, H, W), dtype=torch.float32),
                "bbox": np.array([0, 0, W, H], np.float32), "cam_param": self.cams[i],
                "frame_idx": self.frame_idx_list[i]}


class TestSetup(NamedTuple):
    """What `AvatarTester` takes besides the avatar: the split's tables, the scene and the face render's inputs."""
    frames: object  # FrameTable
    params: object  # SmplxParamTable
    masks: object   # SegmentationTable
    scene: dict     # scene_assets' raw parameters (tester.SCENE_KEYS)
    sh_degree: torch.Tensor
    face_renderer: object
    face_uvmap: torch.Tensor
    face_vertex_idx: torch.Tensor
    renderer: object


def write_segmentation(root, idx, H, W, seed):
    """segmentations/%05d.png in `root`: 0 on a box around the body, 255 elsewhere, and a matte-like edge noise that
    differs between the three channels (so a channel swap changes eval's mask)."""
    rng = np.random.default_rng(seed)
    seg = np.full((H, W, 3), 255, np.uint8)
    seg[H // 8:7 * H // 8, W // 4:3 * W // 4] = 0
    noisy = rng.random((H, W)) < 0.1
    seg[noisy] = rng.integers(0, 256, (int(noisy.sum()), 3), dtype=np.uint8)
    os.makedirs(os.path.join(root, "segmentations"), exist_ok=True)
    if not cv2.imwrite(os.path.join(root, "segmentations", "%05d.png" % idx), seg):
        raise OSError(f"cannot write frame {idx}'s segmentation under {root}")
    return seg


def _test_scene(dev, n, seed=11, sh_degree=3):
    """A seeded scene in front of the test cameras, as SceneGaussian stores it: scene_assets' raw parameters."""
    c4 = WORKLOADS["C4"]
    scene, _, _ = make_population_assets(Workload("C4 scene", c4.height, c4.width, 0, n, 0, True), seed=seed)
    g = torch.Generator().manual_seed(seed)
    M = (sh_degree + 1) ** 2
    p = {"mean": scene["mean_3d"], "opacity_logit": torch.logit(scene["opacity"].clamp(1e-4, 1 - 1e-4)),
         "log_scale": torch.log(scene["scale"]), "rotation6d": torch.randn(n, 6, generator=g),
         "feature_dc": ((scene["rgb"] - 0.5) / 0.28209479177387814).reshape(n, 1, 3),
         "feature_rest": 0.3 * torch.randn(n, M - 1, 3, generator=g)}
    return {k: v.to(dev).contiguous() for k, v in p.items()}
