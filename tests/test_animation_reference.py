"""CPU checks of the animation ops' restatements (exavatar_release_b200/animation.py) and of their C ABI's validation:
pytorch3d's look-at transform by its properties, the scripts' lines as written, the panel's numpy expressions, cv2's
text on the device panel, and the new entry points' error codes."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import ROOT  # noqa: F401  (path setup)
from exavatar_release_b200 import _lib as L
from exavatar_release_b200 import animation as AN  # the module: pytest would collect its test_* names
from exavatar_release_b200.animation import (animation_panel_reference, look_at_view_transform_reference,
                                             orbit_reference)

FAKE = 0x1000  # never dereferenced: validation fails before any launch


def _views(n, seed):
    g = torch.Generator().manual_seed(seed)
    dist = 0.5 + 5 * torch.rand(n, generator=g)
    elev = (torch.rand(n, generator=g) - 0.5) * 3.0   # within (-pi/2, pi/2)
    azim = (torch.rand(n, generator=g) - 0.5) * 40.0  # several turns, as animate_view_rot's k = 16 reaches
    at = torch.randn(n, 3, generator=g)
    return dist, elev, azim, at


@pytest.mark.parametrize("seed", [0, 1])
def test_look_at_reference_properties(seed):
    dist, elev, azim, at = _views(64, seed)
    for i in range(64):
        R, T = look_at_view_transform_reference(dist=dist[i], elev=elev[i], azim=float(azim[i]), degrees=False,
                                                at=at[i][None], up=((0, 1, 0),))
        assert R.shape == (1, 3, 3) and T.shape == (1, 3) and R.dtype == T.dtype == torch.float32
        R, T = R[0].double(), T[0].double()
        assert torch.allclose(R.T @ R, torch.eye(3, dtype=torch.float64), atol=1e-6)  # orthonormal
        e, a, d = float(elev[i]), float(np.float32(azim[i])), float(dist[i])
        C_ = torch.tensor([d * math.cos(e) * math.sin(a), d * math.sin(e), d * math.cos(e) * math.cos(a)],
                          dtype=torch.float64) + at[i].double()
        v = R.T @ (at[i].double() - C_)  # the look direction is the camera's +z
        assert torch.allclose(v, torch.tensor([0.0, 0.0, d], dtype=torch.float64), atol=1e-5 * (1 + d))
        assert torch.allclose(T, -(R.T @ C_), atol=1e-5 * (1 + float(C_.norm())))
        assert float(R[:, 0][1]) == 0.0  # x = n(up x z) has no y component


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_look_at_reference_vertical_takes_the_replacement_branch(sign):
    at = torch.tensor([[0.0, 0.3, 0.0]])
    for azim in (math.pi, 2.0, math.pi + 0.7):
        R, T = look_at_view_transform_reference(dist=3.0, elev=sign * math.pi / 2, azim=azim, degrees=False, at=at)
        dist, elev, az = (torch.tensor([v], dtype=torch.float32) for v in (3.0, sign * math.pi / 2, azim))
        C_ = torch.stack([dist * torch.cos(elev) * torch.sin(az), dist * torch.sin(elev),
                          dist * torch.cos(elev) * torch.cos(az)], 1) + at
        z = F.normalize(at - C_, eps=1e-5)
        x = F.normalize(torch.cross(torch.tensor([[0.0, 1.0, 0.0]]), z, dim=1), eps=1e-5)
        y = F.normalize(torch.cross(z, x, dim=1), eps=1e-5)
        assert bool((x.abs() <= 5e-3).all())  # the first x axis is degenerate ...
        assert torch.equal(R[0, :, 0], F.normalize(torch.cross(y, z, dim=1), eps=1e-5)[0])  # ... and replaced
        assert torch.equal(R[0, :, 1], y[0]) and torch.equal(R[0, :, 2], z[0])
        assert abs(float(torch.linalg.det(R[0].double())) - 1.0) < 1e-3


def _frame_inputs(seed, V=40):
    g = torch.Generator().manual_seed(seed)
    a = 0.3 * torch.randn(3, generator=g)
    Rc = torch.tensor([[math.cos(a[1]), 0.0, math.sin(a[1])], [0.0, 1.0, 0.0], [-math.sin(a[1]), 0.0, math.cos(a[1])]])
    Rx = torch.tensor([[1.0, 0.0, 0.0], [0.0, math.cos(a[0]), -math.sin(a[0])], [0.0, math.sin(a[0]), math.cos(a[0])]])
    cam = {"R": (Rx @ Rc).float(), "t": torch.tensor([0.1, -0.2, 0.3]) + 0.1 * torch.randn(3, generator=g),
           "focal": torch.tensor([1500.0, 1500.0]), "princpt": torch.tensor([256.0, 256.0])}
    root = torch.tensor([0.05, 0.2, 3.5]) + 0.1 * torch.randn(3, generator=g)
    mesh = root + 0.3 * torch.randn(V, 3, generator=g)
    mean_3d = torch.randn(3 * V, 3, generator=g)
    return cam, mesh, root, mean_3d


def _script_frame(cam_param, output_vertices, root_joint_cam, i, frame_idx_list, st, mean_3d):
    """animate_view_rot.py:79-97,103 verbatim, with look_at_view_transform from the restatement."""
    look_at_view_transform = look_at_view_transform_reference
    mesh = output_vertices
    mesh = torch.matmul(torch.inverse(cam_param['R']), (mesh - cam_param['t'].view(-1,3)).permute(1,0)).permute(1,0) # camera coordinate -> world coordinate  # noqa: E231,E501
    root_joint_world = torch.matmul(torch.inverse(cam_param['R']), root_joint_cam - cam_param['t']) # camera coordinate -> world coordinate  # noqa: E261,E501
    azim = math.pi + math.pi*16*i/len(frame_idx_list) # azim angle of the camera  # noqa: E226,E261
    if i == 0:
        st["at_point_orig"] = root_joint_world.clone()
        st["at_point"] = root_joint_world # world coordinate  # noqa: E261
        cam_pos = torch.matmul(torch.inverse(cam_param['R']), -cam_param['t'].view(3,1)).view(3) # get camera position (world coordinate system)  # noqa: E231,E261,E501
        at_point_cam = root_joint_cam # camera coordinate  # noqa: E261
        st["elev"] = torch.arctan(torch.abs(at_point_cam[1])/torch.abs(at_point_cam[2])) # elev angle of the camera  # noqa: E226,E261,E501
        st["dist"] = torch.sqrt(torch.sum((cam_pos - st["at_point"])**2)) # distance between camera and mesh  # noqa: E226,E261,E501
    at_point_orig, at_point, elev, dist = st["at_point_orig"], st["at_point"], st["elev"], st["dist"]
    mesh[:,[0,2]] = mesh[:,[0,2]] - root_joint_world[None,[0,2]] + at_point_orig[None,[0,2]]  # noqa: E231
    R, t = look_at_view_transform(dist=dist, elev=elev, azim=azim, degrees=False, at=at_point[None,:], up=((0,1,0),))  # noqa: E231,E501
    R = torch.inverse(R)
    cam_param_rot = {'R': R[0], 't': t[0], 'focal': cam_param['focal'], 'princpt': cam_param['princpt']}
    mesh = torch.matmul(cam_param_rot['R'], mesh.permute(1,0)).permute(1,0) + cam_param_rot['t'].view(1,3) # world coordinate -> camera coordinate  # noqa: E231,E261,E501
    mean_3d = mean_3d.clone()
    mean_3d[:,[0,2]] = mean_3d[:,[0,2]] - root_joint_world[None,[0,2]] + at_point_orig[None,[0,2]]  # noqa: E231
    return cam_param_rot, mesh, mean_3d, root_joint_world


@pytest.mark.parametrize("seed", [0, 3])
def test_orbit_reference_is_the_script_as_written(seed):
    frames = list(range(6))
    st, anchors = {}, {}
    for i in frames:
        cam, mesh, root, mean_3d = _frame_inputs(seed * 100 + i)
        cr, m, g, rw = _script_frame(cam, mesh.clone(), root, i, frames, st, mean_3d)
        out = orbit_reference(cam, mesh.clone(), root, i, len(frames), anchors, mean_3d=mean_3d)
        assert torch.equal(out["cam_param_rot"]["R"], cr["R"]) and torch.equal(out["cam_param_rot"]["t"], cr["t"])
        assert torch.equal(out["mesh"], m) and torch.equal(out["mean_3d"], g) and torch.equal(out["root_joint_world"], rw)
        for k in ("at_point_orig", "at_point", "elev", "dist"):
            assert torch.equal(anchors[k], st[k]), (i, k)


def _panel_inputs(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    frame = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=g)
    mesh = torch.rand(H, W, 3, generator=g) * 255.99
    mesh[0, :3] = torch.tensor([0.0, 255.0, 254.99998])
    render = torch.rand(3, H, W, generator=g) * 1.0039
    render[:, 0, 0] = torch.tensor([0.0, 1.0, 1.0 / 255])
    return frame, mesh, render


@pytest.mark.parametrize("H,W", [(31, 37), (64, 48)])
def test_panel_reference_is_animate_py(H, W):
    frame, mesh, render = _panel_inputs(H, W, H)
    img = frame.numpy()
    mesh_render = mesh.numpy().astype(np.uint8)
    human_render = {"img": render}
    render_ = (human_render['img'].cpu().numpy().transpose(1,2,0)[:,:,::-1]*255).copy().astype(np.uint8)  # noqa: E231,E226,E501
    out = np.concatenate((img, mesh_render, render_),1).astype(np.uint8)  # noqa: E231
    ref = animation_panel_reference(frame, mesh, render)
    assert ref.dtype == np.uint8 and ref.shape == (H, 3 * W, 3)
    assert np.array_equal(ref, out)
    assert np.array_equal(animation_panel_reference(frame, mesh, render[None]), out)


def _put_panel_text(img, mesh_render, render):
    cv2 = pytest.importorskip("cv2")
    font_size = 1.5
    thick = 3
    cv2.putText(img, 'image', (int(1/3*img.shape[1]), int(0.05*img.shape[0])), cv2.FONT_HERSHEY_SIMPLEX, font_size, [51,51,255], thick, 2)  # noqa: E226,E231,E501
    cv2.putText(mesh_render, 'rendered SMPL-X mesh', (int(1/5*mesh_render.shape[1]), int(0.05*mesh_render.shape[0])), cv2.FONT_HERSHEY_SIMPLEX, font_size, [51,51,255], thick, 2)  # noqa: E226,E231,E501
    cv2.putText(render, 'render', (int(1/3*render.shape[1]), int(0.05*render.shape[0])), cv2.FONT_HERSHEY_SIMPLEX, font_size, [51,51,255], thick, 2)  # noqa: E226,E231,E501


def _put_frame_number(out, frame_idx):
    cv2 = pytest.importorskip("cv2")
    return cv2.putText(out, str(frame_idx), (int(out.shape[1]*0.05), int(out.shape[0]*0.05)), cv2.FONT_HERSHEY_SIMPLEX, 1.0, (0,0,255), 2, 2)  # noqa: E226,E231,E501


@pytest.mark.parametrize("H,W", [(64, 80), (512, 512), (1920, 1080)])
def test_put_text_on_column_views_of_the_panel_is_the_scripts_order(H, W):
    """The script writes text on each panel, concatenates, then writes the frame number.  The ops give the concatenated
    panel, so the text goes on its three column views in place (cv2 accepts the strided views; no copy is needed) and
    then on the whole: the same bytes."""
    frame, mesh, render = _panel_inputs(H, W, 7)
    img = frame.numpy().copy()
    mesh_render = mesh.numpy().astype(np.uint8)
    render_ = (render.numpy().transpose(1, 2, 0)[:, :, ::-1] * 255).copy().astype(np.uint8)
    _put_panel_text(img, mesh_render, render_)
    script = _put_frame_number(np.concatenate((img, mesh_render, render_), 1).astype(np.uint8), 123)
    panel = animation_panel_reference(frame, mesh, render)
    before = panel.copy()
    _put_panel_text(panel[:, :W], panel[:, W:2 * W], panel[:, 2 * W:])
    ours = _put_frame_number(panel, 123)
    assert not np.array_equal(ours, before)
    assert np.array_equal(ours, script)


# ---------------------------------------------------------------------------------------------------------------------
# C ABI and Python validation (no device needed: every call fails before a launch)
# ---------------------------------------------------------------------------------------------------------------------

def test_struct_sizes():
    lib = L.load()
    assert C.sizeof(L.B2ROrbitCamera) == 56
    assert C.sizeof(L.B2RAnimationPanel) == 40
    assert lib.b2r_abi_version() == L.ABI_VERSION == 4


def test_orbit_camera_validation():
    lib = L.load()
    good = dict(k=16, n_frames=8, anchor=1, cam_R=FAKE, cam_t=FAKE, root_cam=FAKE, index=FAKE, state=FAKE)
    call = lambda p: lib.b2r_orbit_camera(C.byref(p) if p is not None else None, None)  # noqa: E731
    assert call(None) == -1
    for bad in ({"k": 0}, {"k": -1}, {"n_frames": 0}, {"n_frames": -5}, {"anchor": 3}, {"anchor": -1},
                {"index": None}, {"state": None}, {"cam_R": None}, {"cam_t": None}, {"root_cam": None},
                {"anchor": 2, "cam_R": None, "cam_t": None, "root_cam": None},
                {"anchor": 0, "root_cam": None}):
        assert call(L.B2ROrbitCamera(**{**good, **bad})) == -1, bad
    assert lib.b2r_launch_count() == 0


def test_orbit_points_and_panel_validation():
    lib = L.load()
    pts = lambda n=4, p=FAKE, s=FAKE, o=FAKE: lib.b2r_orbit_points(n, p, s, 1, o, None)  # noqa: E731
    for kw in ({"n": 0}, {"n": -1}, {"p": None}, {"s": None}, {"o": None}):
        assert pts(**kw) == -1, kw
    good = dict(width=8, height=4, frame=FAKE, mesh_panel=FAKE, render=FAKE)
    pan = lambda p, out=FAKE: lib.b2r_animation_panel(C.byref(p) if p is not None else None, out, None)  # noqa: E731
    assert pan(None) == -1
    assert pan(L.B2RAnimationPanel(**good), out=None) == -1
    for bad in ({"width": 0}, {"height": -2}, {"frame": None}, {"mesh_panel": None}, {"render": None},
                {"width": 1 << 16, "height": 1 << 15}):
        assert pan(L.B2RAnimationPanel(**{**good, **bad})) == -1, bad
    assert lib.b2r_launch_count() == 0


def test_body_joints_validation():
    lib = L.load()
    rig = L.B2RRig(V=10, V1=20, P=40, J=5, NB=3, NE=2, n_body=1)
    for n, _ in L.B2RRig._fields_[8:]:
        setattr(rig, n, FAKE)
    good = dict(rig=rig, pose_mean=FAKE, shape_param=FAKE, joint_offset=FAKE, full_pose=FAKE, expr=FAKE, trans=FAKE)
    need = lib.b2r_smplx_body_scratch_bytes(10, 5)
    call = lambda b, s=FAKE, n=need, j=FAKE: lib.b2r_smplx_body_joints(  # noqa: E731
        C.byref(b) if b is not None else None, s, n, j, None)
    assert call(None) == -1
    b = L.B2RSmplxBody(**good)
    assert call(b, j=None) == -1
    assert call(b, s=None) == -1
    assert call(b, n=need - 1) == lib.b2r_smplx_body_forward(C.byref(b), FAKE, FAKE, need - 1, None) != 0
    for field in ("trans", "pose_mean", "full_pose"):
        assert call(L.B2RSmplxBody(**{**good, field: None})) == -1, field
    assert call(L.B2RSmplxBody(**good, cam_R=FAKE)) == -1  # cam_R without cam_t
    assert lib.b2r_launch_count() == 0


def test_python_checks_without_a_device():
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        AN.OrbitCamera(16, 8, "cpu")
    with pytest.raises(ValueError, match="k"):
        AN.OrbitCamera(0, 8, "cuda")
    with pytest.raises(ValueError, match="n_frames"):
        AN.OrbitCamera(16, True, "cuda")
    frame, mesh, render = _panel_inputs(8, 8, 0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        AN.animation_panel(frame, mesh, render)
