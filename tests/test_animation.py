"""The animation ops on the device (exavatar_release_b200/animation.py, csrc/animate.cu, b2r_smplx_body_joints):
the orbit camera against pytorch3d's look-at restated on the CPU and in float64, the recentring against torch's fp32
expression, the panel against animate.py's numpy bytes, the body's joints against the float64 layer, no host sync, one
CUDA graph for the whole video frame, and an 8-frame animate_view_rot loop against its script form."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

from util import ROOT  # noqa: F401  (path setup)
from util import capture, no_host_sync
from util import dev  # noqa: F401
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.animation import (OrbitCamera, animation_panel, animation_panel_reference,
                                             look_at_view_transform_reference, orbit_points, orbit_reference)

EPS = 2.0 ** -23


def _camera(seed, dev, shape=None):
    """A frame camera near the identity; with shape (H, W), focal 1.2 H and the principal point at the centre."""
    g = torch.Generator().manual_seed(seed)
    a = 0.2 * torch.randn(2, generator=g).double()
    Ry = torch.tensor([[math.cos(a[1]), 0.0, math.sin(a[1])], [0.0, 1.0, 0.0], [-math.sin(a[1]), 0.0, math.cos(a[1])]],
                      dtype=torch.float64)
    Rx = torch.tensor([[1.0, 0.0, 0.0], [0.0, math.cos(a[0]), -math.sin(a[0])], [0.0, math.sin(a[0]), math.cos(a[0])]],
                      dtype=torch.float64)
    focal, princpt = (1100.0, 1080.0), (250.0, 262.0)
    if shape is not None:
        focal, princpt = (1.2 * shape[0], 1.2 * shape[0]), (shape[1] / 2, shape[0] / 2)
    return {"R": (Rx @ Ry).float().to(dev), "t": (0.1 * torch.randn(3, generator=g)).to(dev),
            "focal": torch.tensor(focal, device=dev), "princpt": torch.tensor(princpt, device=dev)}


def _azim(k, i, n):
    return float(np.float32(math.pi + math.pi * k * i / n))


def _look_at64(dist, elev, azim, at):
    """look_at_view_transform + inverse in float64 from the op's fp32 anchors and fp32 azim."""
    d, e, a = float(dist), float(elev), azim
    at = at.double().cpu()
    C_ = torch.tensor([d * math.cos(e) * math.sin(a), d * math.sin(e), d * math.cos(e) * math.cos(a)],
                      dtype=torch.float64) + at
    n = lambda v: v / max(float(v.norm()), 1e-5)  # noqa: E731
    z = n(at - C_)
    x = n(torch.linalg.cross(torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64), z))
    y = n(torch.linalg.cross(z, x))
    if bool((x.abs() <= 5e-3).all()):
        x = n(torch.linalg.cross(y, z))
    Rp = torch.stack([x, y, z], 1)
    return torch.inverse(Rp), -(Rp.T @ C_), C_


def _check_frame(orbit, cam_rot, k, i, n, worst):
    at, elev, dist = orbit.at.cpu(), orbit.elev.cpu(), orbit.dist.cpu()
    R, T = look_at_view_transform_reference(dist=dist, elev=elev, azim=math.pi + math.pi * k * i / n, degrees=False,
                                            at=at[None], up=((0, 1, 0),))
    R = torch.inverse(R)[0]
    Rop, top = cam_rot["R"].cpu(), cam_rot["t"].cpu()
    R64, t64, C64 = _look_at64(dist, elev, _azim(k, i, n), at)
    scale = float(C64.norm())
    worst["R_ulps"] = max(worst["R_ulps"], float((Rop - R).abs().max()) / EPS)
    worst["t_ulps"] = max(worst["t_ulps"], float((top - T[0]).abs().max()) / (EPS * scale))
    worst["R64"] = max(worst["R64"], float((Rop.double() - R64).abs().max()))
    worst["t64"] = max(worst["t64"], float((top.double() - t64).abs().max()) / scale)


def _assert_worst(worst, tag):
    print(f"{tag}: R {worst['R_ulps']:.1f} ulps, t {worst['t_ulps']:.1f} ulps of |C| from the CPU reference; "
          f"R {worst['R64']:.2e}, t {worst['t64']:.2e} relative from float64")
    assert worst["R_ulps"] <= 8 and worst["t_ulps"] <= 8
    assert worst["R64"] <= 1e-6 and worst["t64"] <= 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_orbit_camera_anchor_mode(dev, seed):
    n, k = 97, 16
    cam0 = _camera(seed, dev)
    root0 = torch.tensor([0.05, 0.25, 3.9], device=dev) + 0.1 * torch.randn(3, generator=torch.Generator().manual_seed(
        seed)).to(dev)
    orbit = OrbitCamera(k, n, dev)
    orbit.anchor(cam0, root0)
    anchors = {}
    mesh = root0[None].cpu() + torch.zeros(2, 3)
    cpu = {kk: v.cpu() for kk, v in cam0.items()}
    ref = orbit_reference(cpu, mesh, root0.cpu(), 0, n, anchors, k=k)
    for name, a, b in (("at", orbit.at, anchors["at_point"]), ("elev", orbit.elev, anchors["elev"]),
                       ("dist", orbit.dist, anchors["dist"])):
        d = float((a.cpu() - b).abs().max()) / (EPS * max(1.0, float(b.abs().max())))
        print(f"anchor {name}: {d:.1f} ulps from the script's CPU lines")
        assert d <= 8, name
    worst = dict(R_ulps=0.0, t_ulps=0.0, R64=0.0, t64=0.0)
    idx = torch.zeros(1, dtype=torch.int32, device=dev)
    for i in list(range(n)) + [1000, 4321, 99999]:
        cam = _camera(seed * 1000 + i + 1, dev) if i else cam0
        root = root0 + 0.05 * (i % 7) if i else root0
        idx.fill_(i)
        cam_rot = orbit(cam, root, idx)
        _check_frame(orbit, cam_rot, k, i, n, worst)
        rw = torch.matmul(torch.inverse(cam["R"].cpu()), root.cpu() - cam["t"].cpu())
        assert float((orbit.root_world.cpu() - rw).abs().max()) <= 8 * EPS * float(rw.abs().max())
        if i == 0:
            assert torch.allclose(cam_rot["R"].cpu(), ref["cam_param_rot"]["R"], atol=1e-6)
            assert torch.allclose(cam_rot["t"].cpu(), ref["cam_param_rot"]["t"], atol=1e-5)
    _assert_worst(worst, f"anchor seed {seed}")
    # frame 0 re-anchors from its own camera, as the script's `if i == 0`
    orbit2 = OrbitCamera(k, n, dev)
    orbit2(cam0, root0, 0)
    orbit(cam0, root0, 0)
    assert torch.equal(orbit2.state, orbit.state)


@pytest.mark.gpu
def test_orbit_camera_fixed_anchors(dev):
    """get_neutral_pose.py:76-82: k = 2, 50 views, elev = -pi/6 and at / dist from the host."""
    n, k = 50, 2
    orbit = OrbitCamera(k, n, dev)
    at = torch.tensor([0.02, 0.31, 3.05], device=dev)
    orbit.fixed(at, -math.pi / 6, torch.tensor(3.0513, device=dev))
    assert float(orbit.elev) == float(np.float32(-math.pi / 6))
    cam = _camera(4, dev)
    worst = dict(R_ulps=0.0, t_ulps=0.0, R64=0.0, t64=0.0)
    for i in range(n):
        cam_rot = orbit(cam, None, i)
        _check_frame(orbit, cam_rot, k, i, n, worst)
        assert torch.equal(orbit.root_world, at) and cam_rot["focal"] is cam["focal"]
    _assert_worst(worst, "fixed")


@pytest.mark.gpu
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_orbit_camera_vertical_replacement_branch(dev, sign):
    n, k = 16, 16
    orbit = OrbitCamera(k, n, dev)
    orbit.fixed(torch.tensor([0.0, 0.3, 0.0]), sign * math.pi / 2, 3.0)
    worst = dict(R_ulps=0.0, t_ulps=0.0, R64=0.0, t64=0.0)
    for i in range(n):
        cam_rot = orbit(_camera(0, dev), None, i)
        R, _ = look_at_view_transform_reference(dist=3.0, elev=sign * math.pi / 2, azim=math.pi + math.pi * k * i / n,
                                                degrees=False, at=((0.0, 0.3, 0.0),))
        assert abs(float(R[0, 1, 0])) < 0.1  # the replacement x axis lies in the horizontal plane
        _check_frame(orbit, cam_rot, k, i, n, worst)
    print(f"vertical {sign}: {worst}")
    assert worst["R_ulps"] <= 64 and worst["R64"] <= 1e-5 and worst["t64"] <= 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("n_pts", [1, 1000, 167_618])
def test_orbit_points(dev, n_pts):
    orbit = OrbitCamera(16, 8, dev)
    cam = _camera(7, dev)
    root = torch.tensor([0.1, 0.2, 4.0], device=dev)
    orbit(cam, root, 0)
    orbit(_camera(8, dev), root + 0.1, 3)
    g = torch.Generator(device=dev).manual_seed(n_pts)
    p = torch.randn(n_pts, 3, device=dev, generator=g) + torch.tensor([0.0, 0.0, 4.0], device=dev)
    rw, at = orbit.root_world.clone(), orbit.at.clone()
    q = orbit_points(p, orbit)
    ref = p.clone()
    ref[:, [0, 2]] = ref[:, [0, 2]] - rw[None, [0, 2]] + at[None, [0, 2]]
    assert torch.equal(q.view(torch.int32), ref.view(torch.int32))
    v = orbit_points(p, orbit, view=True)
    R, t = orbit.state[5:14].view(3, 3), orbit.state[14:17]
    vref = torch.matmul(R, ref.permute(1, 0)).permute(1, 0) + t.view(1, 3)
    err = float((v - vref).abs().max()) / float(vref.abs().max())
    print(f"orbit_points view: max |op - torch.matmul| / max |x| = {err:.2e}")
    assert err <= 4 * EPS


def _panel_inputs(H, W, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    frame = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, device=dev, generator=g)
    mesh = torch.rand(H, W, 3, device=dev, generator=g) * 255.999
    render = torch.rand(3, H, W, device=dev, generator=g) * 1.0039  # x 255 reaches 255.99
    mesh.view(-1)[:4] = torch.tensor([0.0, 255.0, 254.99998, 1.0 - 2 ** -24], device=dev)
    render.view(-1)[:3] = torch.tensor([1.0, 1.0 / 255, 2.0 / 255], device=dev)
    return frame, mesh, render


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(31, 37), (512, 512), (1920, 1080)])
def test_panel_is_the_scripts_bytes(dev, H, W):
    frame, mesh, render = _panel_inputs(H, W, dev, H)
    out = animation_panel(frame, mesh, render[None])
    ref = animation_panel_reference(frame, mesh, render)
    assert out.shape == (H, 3 * W, 3) and out.dtype == torch.uint8
    assert np.array_equal(out.cpu().numpy(), ref)
    # every byte written: a 0xFF-prefilled buffer and a zero-filled one give the same bytes
    p = L.B2RAnimationPanel(width=W, height=H, frame=L.ptr(frame), mesh_panel=L.ptr(mesh), render=L.ptr(render))
    for fill in (255, 0):
        buf = torch.full((H, 3 * W, 3), fill, dtype=torch.uint8, device=dev)
        L.run("b2r_animation_panel", dev, C.byref(p), L.ptr(buf))
        assert torch.equal(buf, out), fill


@pytest.mark.gpu
def test_panel_saturates_outside_the_byte_range(dev):
    H, W = 4, 8
    frame = torch.zeros(H, W, 3, dtype=torch.uint8, device=dev)
    vals = torch.tensor([-1.0, -0.5, -0.0, float("nan"), 255.5, 256.0, 1e9, float("inf"), -float("inf"), 0.99],
                        device=dev)
    mesh = vals.repeat(H * W * 3 // vals.numel() + 1)[:H * W * 3].reshape(H, W, 3).contiguous()
    out = animation_panel(frame, mesh, torch.zeros(3, H, W, device=dev))[:, W:2 * W].reshape(-1).cpu()
    m = mesh.reshape(-1).cpu()
    want = torch.where(torch.isnan(m), 0.0, m.clamp(0, 255)).trunc().to(torch.uint8)
    assert torch.equal(out, want)


def _body(dev):
    from exavatar_release_b200.smplx_rig import SmplxRig
    from exavatar_release_b200.synthetic import make_human_mesh, make_smplx_model
    mesh = make_human_mesh()
    model = make_smplx_model(mesh)
    rig = SmplxRig(**model, device=dev)
    return rig, mesh["base_faces"]


def _body_inputs(rig, dev, seed):
    g = torch.Generator().manual_seed(seed)
    ins = [torch.randn(rig.NB, generator=g), 0.01 * torch.randn(rig.J, 3, generator=g),
           0.2 * torch.randn(rig.J, 3, generator=g), torch.randn(rig.NE, generator=g),
           torch.tensor([0.02, -0.05, 0.1]) + 0.05 * torch.randn(3, generator=g)]
    return [t.to(dev) for t in ins]


@pytest.mark.gpu
def test_body_mesh_joints(dev):
    from exavatar_release_b200.smplx_rig import smplx_body_reference
    rig, _ = _body(dev)
    ins = _body_inputs(rig, dev, 3)
    cam = _camera(3, dev)
    for c in ((), (cam["R"], cam["t"])):
        mesh = rig.body_mesh(*ins, *c)
        mesh2, joints = rig.body_mesh(*ins, *c, joints=True)
        assert torch.equal(mesh.view(torch.int32), mesh2.view(torch.int32))
        assert joints.shape == (rig.J, 3) and not joints.requires_grad
        ref_mesh, ref_j = smplx_body_reference(rig.model, *ins, *c, joints=True)
        assert torch.allclose(mesh.double(), ref_mesh, atol=2e-6)
        err = float((joints.double() - ref_j).abs().max())
        print(f"joints (camera {bool(c)}): max |op - float64| = {err:.2e}")
        assert err <= 2e-6
        if c:
            assert torch.equal(joints, rig.body_mesh(*ins, joints=True)[1])  # camera coordinates either way
    # the gradient of the mesh is unchanged by the joints
    leaves = [t.clone().requires_grad_() for t in ins]
    w = torch.randn(rig.V, 3, device=dev)
    (rig.body_mesh(*leaves) * w).sum().backward()
    g0 = [t.grad.clone() for t in leaves]
    for t in leaves:
        t.grad = None
    (rig.body_mesh(*leaves, joints=True)[0] * w).sum().backward()
    assert all(torch.equal(a, t.grad) for a, t in zip(g0, leaves))


def _gaussians(mesh_world, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    P = 4 * mesh_world.shape[0]
    rows = torch.arange(P, device=dev) % mesh_world.shape[0]
    rot = torch.zeros(P, 4, device=dev)
    rot[:, 0] = 1
    return {"mean_3d": mesh_world[rows] + 0.01 * torch.randn(P, 3, device=dev, generator=g),
            "scale": 0.004 + 0.006 * torch.rand(P, 3, device=dev, generator=g), "rotation": rot,
            "opacity": 0.2 + 0.7 * torch.rand(P, 1, device=dev, generator=g),
            "rgb": torch.rand(P, 3, device=dev, generator=g)}


def _render(assets, mean_3d, shape, cam_rot, bg):
    from exavatar_release_b200 import GaussianRasterizer
    from exavatar_release_b200.renderer import device_render_settings
    st = device_render_settings(shape, cam_rot, bg)
    m2d = torch.zeros_like(mean_3d)
    return GaussianRasterizer(st)(means3D=mean_3d, means2D=m2d, opacities=assets["opacity"], colors_precomp=assets["rgb"],
                                  scales=assets["scale"], rotations=assets["rotation"])[0]


def _op_frame(rig, mesh_r, orbit, assets, ins, cam, frame_u8, index, bkg, bg):
    """One animate_view_rot video frame from the ops: body mesh and joints, orbit camera, recentred mesh and
    Gaussians, render, mesh panel and the uint8 frame."""
    H, W = frame_u8.shape[:2]
    with torch.no_grad():
        mesh, joints = rig.body_mesh(*ins, cam["R"], cam["t"], joints=True)
        cam_rot = orbit(cam, joints[0], index)
        mesh_cam = orbit_points(mesh, orbit, view=True)
        mean_3d = orbit_points(assets["mean_3d"], orbit)
        render = _render(assets, mean_3d, (H, W), cam_rot, bg)
        return animation_panel(frame_u8, mesh_r(mesh_cam, cam, bkg), render)


@pytest.mark.gpu
def test_no_host_sync(dev):
    from exavatar_release_b200.mesh_render import ShadedMeshRenderer
    from exavatar_release_b200.rasterizer import set_fixed_capacity
    rig, faces = _body(dev)
    mesh_r = ShadedMeshRenderer(faces, rig.V, device=dev)
    H, W = 96, 128
    ins, cam = _body_inputs(rig, dev, 1), _camera(1, dev, (H, W))
    assets = _gaussians(rig.body_mesh(*ins, cam["R"], cam["t"]).detach(), dev, 1)
    frame_u8, _, _ = _panel_inputs(H, W, dev, 1)
    bkg, bg = torch.full((H, W, 3), 255.0, device=dev), torch.ones(3, device=dev)
    orbit = OrbitCamera(16, 8, dev)
    index = torch.zeros(1, dtype=torch.int32, device=dev)
    set_fixed_capacity(1 << 21)
    try:
        _op_frame(rig, mesh_r, orbit, assets, ins, cam, frame_u8, index, bkg, bg)
        with no_host_sync():
            _op_frame(rig, mesh_r, orbit, assets, ins, cam, frame_u8, index, bkg, bg)
    finally:
        set_fixed_capacity(None)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_one_graph_holds_the_video_frame(dev):
    from exavatar_release_b200.mesh_render import ShadedMeshRenderer
    from exavatar_release_b200.rasterizer import overflowed, set_fixed_capacity
    rig, faces = _body(dev)
    mesh_r = ShadedMeshRenderer(faces, rig.V, device=dev)
    H, W = 192, 256
    ins, cam = _body_inputs(rig, dev, 2), _camera(2, dev, (H, W))
    assets = _gaussians(rig.body_mesh(*ins, cam["R"], cam["t"]).detach(), dev, 2)
    frame_u8, _, _ = _panel_inputs(H, W, dev, 2)
    bkg, bg = torch.full((H, W, 3), 255.0, device=dev), torch.ones(3, device=dev)
    orbit = OrbitCamera(16, 8, dev)
    index = torch.zeros(1, dtype=torch.int32, device=dev)
    set_fixed_capacity(1 << 21)
    try:
        run = lambda: _op_frame(rig, mesh_r, orbit, assets, ins, cam, frame_u8, index, bkg, bg)  # noqa: E731
        first = run()  # frame 0: anchors
        graph, static = capture(run, 1)
        eager_orbit = OrbitCamera(16, 8, dev)
        graph.replay()  # frame 0 again: the same bytes
        torch.cuda.synchronize()
        assert torch.equal(static, first)
        e_index = torch.zeros(1, dtype=torch.int32, device=dev)
        _op_frame(rig, mesh_r, eager_orbit, assets, ins, cam, frame_u8, e_index, bkg, bg)
        for i in (1, 5):
            new_ins, new_cam = _body_inputs(rig, dev, 10 + i), _camera(10 + i, dev, (H, W))
            new_frame, _, _ = _panel_inputs(H, W, dev, 10 + i)
            with torch.no_grad():
                for a, b in zip(ins, new_ins):
                    a.copy_(b)
                for kk in ("R", "t"):
                    cam[kk].copy_(new_cam[kk])
                frame_u8.copy_(new_frame)
                index.fill_(i)
            graph.replay()
            torch.cuda.synchronize()
            replayed = static.clone()
            e_index.fill_(i)
            eager = _op_frame(rig, mesh_r, eager_orbit, assets, ins, cam, frame_u8, e_index, bkg, bg)
            torch.cuda.synchronize()
            assert torch.equal(replayed, eager), i
            assert torch.equal(replayed[:, :W], new_frame)
            assert not torch.equal(replayed, first)
        assert not overflowed()
    finally:
        set_fixed_capacity(None)


@pytest.mark.gpu
def test_eight_frame_loop_matches_the_script_form(dev):
    """animate_view_rot's loop over 8 frames on the synthetic C4 rig (tools/c4_frame.setup): the ops against the
    script's lines (orbit_reference: torch.inverse, the CPU look-at, indexed recentring; the layer's mesh and joints
    from body_mesh).  The cameras agree within fp32 tolerance; with both arms rendering through the op's camera the
    panels are the same bytes (the script arm converts on the host with numpy and concatenates)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from c4_frame import setup
    from exavatar_release_b200.mesh_render import ShadedMeshRenderer
    from exavatar_release_b200.synthetic import make_human_mesh, make_smplx_model
    hm = make_human_mesh()
    rig, _, x, _ = setup(dev, make_smplx_model(hm))
    mesh_r = ShadedMeshRenderer(hm["base_faces"], rig.V, device=dev)
    H, W, n = 160, 128, 8
    bkg, bg = torch.full((H, W, 3), 255.0, device=dev), torch.ones(3, device=dev)
    orbit = OrbitCamera(16, n, dev)
    anchors = {}
    beta, jo, pose, expr = (t.detach() for t in x)
    for i in range(n):
        g = torch.Generator().manual_seed(100 + i)
        ins = [beta, jo, pose + 0.05 * torch.randn(pose.shape, generator=g).to(dev), expr,
               (torch.tensor([0.0, 0.0, 0.1]) + 0.02 * torch.randn(3, generator=g)).to(dev)]
        cam = _camera(200 + i, dev, (H, W))
        frame_u8, _, _ = _panel_inputs(H, W, dev, 300 + i)
        with torch.no_grad():
            mesh_layer, joints = rig.body_mesh(*ins, joints=True)  # the layer's output.vertices / joints
            mesh_world, joints_w = rig.body_mesh(*ins, cam["R"], cam["t"], joints=True)
            assets = _gaussians(mesh_world, dev, i)
            # the ops
            cam_rot = orbit(cam, joints_w[0], i)
            mesh_cam = orbit_points(mesh_world, orbit, view=True)
            mean_3d = orbit_points(assets["mean_3d"], orbit)
            render = _render(assets, mean_3d, (H, W), cam_rot, bg)
            mesh_panel = mesh_r(mesh_cam, cam, bkg)
            panel = animation_panel(frame_u8, mesh_panel, render).cpu().numpy()
            # the script form
            ref = orbit_reference(cam, mesh_layer.clone(), joints[0], i, n, anchors, mean_3d=assets["mean_3d"])
            assert torch.allclose(cam_rot["R"], ref["cam_param_rot"]["R"], atol=2e-6), i
            assert torch.allclose(cam_rot["t"], ref["cam_param_rot"]["t"], atol=2e-6 * float(ref["cam_param_rot"]["t"].norm())), i
            assert torch.allclose(mean_3d, ref["mean_3d"], atol=4e-6), i
            assert torch.allclose(mesh_cam, ref["mesh"], atol=1e-5), i
            img = frame_u8.cpu().numpy()
            mesh_render = mesh_panel.cpu().numpy().astype(np.uint8)
            render_ = (render.cpu().numpy().transpose(1, 2, 0)[:, :, ::-1] * 255).copy().astype(np.uint8)
            out = np.concatenate((img, mesh_render, render_), 1).astype(np.uint8)
        assert np.array_equal(panel, out), i
        assert (render_ < 255).any() and (mesh_render < 255).any()  # the body is in view
