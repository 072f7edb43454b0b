"""The per-frame host work of ExAvatar's animation scripts as sync-free CUDA ops (csrc/animate.cu): the orbit camera of
animate_view_rot.py and get_neutral_pose.py, the recentred avatar, and the three-panel video frame of animate.py and
animate_view_rot.py.

animate_view_rot.py:65-117 inverts the frame's camera three times with `torch.inverse` (each a host sync), builds its
orbit camera with pytorch3d's `look_at_view_transform` on the CPU, recentres the posed Gaussians and mesh with indexed
assignments and converts the render on the host (a 25 MB fp32 read-back at 1080x1920, then numpy's transpose, flip,
scale and cast).  With these ops a frame goes from the SMPL-X parameters and the source frame's bytes to one uint8
panel and one copy to the host; at a fixed render shape the whole frame can be captured as one CUDA graph:

    orbit = OrbitCamera(16, len(frame_idx_list), "cuda")           # once; anchors come from the frame with index 0
    mesh, joints = rig.body_mesh(*body_inputs, cam_R, cam_t, joints=True)    # world mesh, camera-space joints
    cam_rot = orbit(cam_param, joints[0], index)                   # index: a (1,) int32 CUDA tensor (or an int)
    mesh_cam = orbit_points(mesh, orbit, view=True)                # :92 and :97
    human_asset["mean_3d"] = orbit_points(human_asset["mean_3d"], orbit)     # :103
    render = GaussianRasterizer(device_render_settings(shape, cam_rot, bg))(...)[0]
    panel = animation_panel(frame_u8, mesh_renderer(mesh_cam, cam_param, bkg), render)   # (H, 3W, 3) uint8 BGR

`look_at_view_transform_reference`, `orbit_reference` and `animation_panel_reference` restate pytorch3d's function and
the scripts' lines in torch fp32 and numpy; the tests compare the ops with them and the ops never call them.  pytorch3d
is not a dependency of this project, so its look-at semantics are restated from its source (pytorch3d/renderer/
cameras.py: look_at_view_transform, look_at_rotation, camera_position_from_spherical_angles; common/datatypes.py:
format_tensor, convert_to_tensors_and_broadcast) and not pinned against it by a test.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib as L

# the state block of b2r_orbit_camera (include/b200raster.h)
_AT, _ELEV, _DIST, _R, _T, _ROOT = slice(0, 3), 3, 4, slice(5, 14), slice(14, 17), slice(17, 20)


def _count(fn: str, name: str, v) -> int:
    if isinstance(v, bool) or not isinstance(v, numbers.Integral) or not 1 <= int(v) < 2 ** 31:
        raise ValueError(f"{fn}: `{name}` must be an integer in [1, 2^31), got {v!r}")
    return int(v)


def _vec(fn: str, name: str, t, n: int, device) -> torch.Tensor:
    L.cuda(fn, name, t, device)
    L.float32(fn, name, t)
    if t.numel() != n:
        raise ValueError(f"{fn}: `{name}` must have {n} elements, got {tuple(t.shape)}")
    return t.detach().reshape(n).contiguous()


class OrbitCamera:
    """The orbit camera of animate_view_rot.py:79-95 (k = 16) and get_neutral_pose.py:76-82 (k = 2) on the device:
    pytorch3d's `look_at_view_transform(dist, elev, azim, degrees=False, at, up=((0,1,0),))` for
    azim = pi + pi k i / n_frames, followed by the scripts' `R = torch.inverse(R)`, in one single-thread launch per frame
    (b2r_orbit_camera; include/b200raster.h has the arithmetic).

    The anchors at, elev and dist live in a device state block.  By default (animate_view_rot) a call whose frame
    index is 0 sets them from its own camera and root joint first, as the script's `if i == 0` does, so one captured
    graph serves every frame including the first.  `.anchor(cam_param, root_cam)` sets them from a given frame now;
    `.fixed(at, elev, dist)` writes them from the host (get_neutral_pose) and turns the frame-0 anchoring off.
    Calls of one camera run on one stream.
    """

    def __init__(self, k: int, n_frames: int, device=None):
        fn = "OrbitCamera"
        self.k = _count(fn, "k", k)
        self.n_frames = _count(fn, "n_frames", n_frames)
        device = torch.device(device if device is not None else "cuda")
        if device.type != "cuda":
            raise RuntimeError(f"{fn}: device must be CUDA (got {device}); there is no CPU fallback")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = device
        self.state = torch.full((L.ORBIT_STATE,), float("nan"), dtype=torch.float32, device=device)
        self._index = torch.zeros(1, dtype=torch.int32, device=device)
        self._zero = torch.zeros(1, dtype=torch.int32, device=device)
        self._anchor_mode = 1

    # views of the state block: the anchors, and the latest frame's render camera and root joint in world coordinates
    at = property(lambda self: self.state[_AT])
    elev = property(lambda self: self.state[_ELEV])
    dist = property(lambda self: self.state[_DIST])
    root_world = property(lambda self: self.state[_ROOT])

    def _launch(self, cam_param, root_cam, index, anchor: int) -> None:
        fn = "OrbitCamera"
        p = L.B2ROrbitCamera(k=self.k, n_frames=self.n_frames, anchor=anchor, index=L.ptr(index),
                             state=L.ptr(self.state))
        keep = ()
        if root_cam is not None:
            keep = (_vec(fn, "cam_param['R']", cam_param["R"], 9, self.device),
                    _vec(fn, "cam_param['t']", cam_param["t"], 3, self.device),
                    _vec(fn, "root_cam", root_cam, 3, self.device))
            p.cam_R, p.cam_t, p.root_cam = (L.ptr(t) for t in keep)
        L.run("b2r_orbit_camera", self.device, C.byref(p))

    def anchor(self, cam_param: Dict[str, torch.Tensor], root_cam: torch.Tensor) -> None:
        """Sets at, elev and dist from this camera and root joint (camera coordinates) as animate_view_rot.py:85-91
        does on frame 0, and keeps the frame-0 anchoring on.  No host sync."""
        self._launch(cam_param, root_cam, self._zero, 2)
        self._anchor_mode = 1

    def fixed(self, at, elev, dist) -> None:
        """Writes the anchors from the caller: at (3), elev (radians) and dist, as tensors or numbers, stored as fp32
        (as look_at_view_transform's format_tensor stores them).  Frame-0 anchoring is off afterwards."""
        vals = [torch.as_tensor(v, dtype=torch.float32).detach().reshape(n).to(self.device)
                for v, n in ((at, 3), (elev, 1), (dist, 1))]
        self.state[:5].copy_(torch.cat(vals))
        self._anchor_mode = 0

    def __call__(self, cam_param: Dict[str, torch.Tensor], root_cam: Optional[torch.Tensor],
                 index) -> Dict[str, torch.Tensor]:
        """The render camera of frame `index`: {"R" (3,3), "t" (3), "focal", "princpt"} -- R and t are views of the
        state block, rewritten by the next call (clone them to keep a frame's camera); focal and princpt are the
        caller's.  `renderer.device_render_settings` takes the dict unchanged.

        cam_param   the frame's camera (R (3,3), t (3) fp32 CUDA); its R and t are read only with root_cam
        root_cam    (3) the root joint in that camera's coordinates (`body_mesh(..., joints=True)[1][0]`), or None
                    for fixed anchors: then `root_world` is `at` and no recentring is meant
        index       the frame index i: a one-element integer CUDA tensor (read on the device, so a captured graph
                    replays every frame), or a Python int (written into the camera's own index tensor)
        """
        fn = "OrbitCamera"
        if root_cam is None and self._anchor_mode:
            raise ValueError(f"{fn}: root_cam is needed unless the anchors are fixed (.fixed)")
        if isinstance(index, torch.Tensor):
            L.cuda(fn, "index", index, self.device)
            if index.numel() != 1 or index.dtype.is_floating_point or index.dtype == torch.bool:
                raise ValueError(f"{fn}: `index` must be a one-element integer tensor, got {index.dtype} "
                                 f"{tuple(index.shape)}")
            idx = index.reshape(1).to(torch.int32).contiguous()
        elif isinstance(index, numbers.Integral) and not isinstance(index, bool) and 0 <= int(index) < 2 ** 31:
            idx = self._index.fill_(int(index))
        else:
            raise ValueError(f"{fn}: `index` must be a CUDA integer tensor or an int in [0, 2^31), got {index!r}")
        self._launch(cam_param, root_cam, idx, self._anchor_mode)
        return {"R": self.state[_R].view(3, 3), "t": self.state[_T], "focal": cam_param["focal"],
                "princpt": cam_param["princpt"]}


def orbit_points(points: torch.Tensor, orbit: OrbitCamera, view: bool = False) -> torch.Tensor:
    """animate_view_rot.py:92 / :103 on a new (n,3) fp32 array: columns 0 and 2 become fl(fl(p - root_world) + at)
    with the orbit camera's latest frame, column 1 is copied; with `view`, the result is then moved into that frame's
    render camera, R p + t (:97, the mesh panel).  points (n,3) fp32 CUDA (the posed Gaussians' mean_3d, or the world
    mesh of `body_mesh`).  One launch, no host sync; no gradient."""
    fn = "orbit_points"
    L.cuda(fn, "points", points, orbit.device)
    L.float32(fn, "points", points)
    if points.dim() != 2 or points.shape[1] != 3 or not 1 <= points.shape[0] < 2 ** 31:
        raise ValueError(f"{fn}: `points` must be (n,3) with n >= 1, got {tuple(points.shape)}")
    x = points.detach().contiguous()
    out = torch.empty_like(x)
    L.run("b2r_orbit_points", orbit.device, x.shape[0], L.ptr(x), L.ptr(orbit.state), int(bool(view)), L.ptr(out))
    return out


def animation_panel(frame_u8: torch.Tensor, mesh_panel: torch.Tensor, render: torch.Tensor) -> torch.Tensor:
    """The (H, 3W, 3) uint8 BGR video frame of animate.py:86,94 and animate_view_rot.py:107,115 before the text, in one
    launch: the source frame, trunc(mesh_panel), and trunc(render[::-1] * 255) side by side.

    frame_u8    (H,W,3) uint8 CUDA: the source frame's BGR bytes (cv2.imread's layout)
    mesh_panel  (H,W,3) fp32 CUDA: `ShadedMeshRenderer`'s output (render_mesh's float image, 0-255)
    render      (3,H,W) or (1,3,H,W) fp32 CUDA: the Gaussian render's RGB image in [0, 1]

    trunc is numpy's astype(np.uint8) on [0, 256): toward zero; values outside saturate (NaN gives 0), where numpy
    leaves them undefined.  The caller adds the text after its one copy to the host (cv2.putText on column views
    of the panel writes the script's bytes)."""
    fn = "animation_panel"
    L.cuda(fn, "frame_u8", frame_u8)
    if frame_u8.dtype != torch.uint8 or frame_u8.dim() != 3 or frame_u8.shape[2] != 3:
        raise ValueError(f"{fn}: `frame_u8` must be uint8 (H,W,3), got {frame_u8.dtype} {tuple(frame_u8.shape)}")
    H, W = int(frame_u8.shape[0]), int(frame_u8.shape[1])
    if H < 1 or W < 1 or H * W >= 2 ** 31:
        raise ValueError(f"{fn}: bad image size {(H, W)}")
    for name, t, shape in (("mesh_panel", mesh_panel, (H, W, 3)), ("render", render, (3, H, W))):
        L.cuda(fn, name, t)
        L.float32(fn, name, t)
        if tuple(t.shape[-3:]) != shape or t.dim() not in (3, 4) or (t.dim() == 4 and t.shape[0] != 1):
            raise ValueError(f"{fn}: `{name}` must be {shape}, got {tuple(t.shape)}")
    L.same_device(fn, (frame_u8, mesh_panel, render))
    f, m, r = (t.detach().contiguous() for t in (frame_u8, mesh_panel, render.reshape(3, H, W)))
    out = torch.empty((H, 3 * W, 3), dtype=torch.uint8, device=f.device)
    p = L.B2RAnimationPanel(width=W, height=H, frame=L.ptr(f), mesh_panel=L.ptr(m), render=L.ptr(r))
    L.run("b2r_animation_panel", f.device, C.byref(p), L.ptr(out))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# References (tests and measurements; the ops never call them)
# ---------------------------------------------------------------------------------------------------------------------

def _format_tensor(x, device) -> torch.Tensor:
    """pytorch3d's format_tensor: a number becomes a float32 tensor, a tensor keeps its dtype; moved to `device`."""
    t = x if torch.is_tensor(x) else torch.tensor(x, dtype=torch.float32, device=device)
    if t.dim() == 0:
        t = t.view(1)
    return t.to(device=device)


def _broadcast(*args, device):
    """pytorch3d's convert_to_tensors_and_broadcast."""
    ts = [_format_tensor(a, device) for a in args]
    n = max(t.shape[0] for t in ts)
    return [t.expand(n, *t.shape[1:]) if t.shape[0] == 1 else t for t in ts]


def look_at_view_transform_reference(dist=1.0, elev=0.0, azim=0.0, degrees: bool = True, at=((0, 0, 0),),
                                     up=((0, 1, 0),), device="cpu"):
    """pytorch3d's look_at_view_transform (eye=None) restated in torch with its defaults: every argument is moved to
    `device` (the CPU unless given, which is where the scripts run it), R (N,3,3) has columns x, y, z of the look-at
    frame and T (N,3) = -R^T C."""
    dist, elev, azim, at, up = _broadcast(dist, elev, azim, at, up, device=device)
    # camera_position_from_spherical_angles
    dist_, elev_, azim_ = _broadcast(dist, elev, azim, device=device)
    if degrees:
        elev_ = math.pi / 180.0 * elev_
        azim_ = math.pi / 180.0 * azim_
    x = dist_ * torch.cos(elev_) * torch.sin(azim_)
    y = dist_ * torch.sin(elev_)
    z = dist_ * torch.cos(elev_) * torch.cos(azim_)
    C_ = torch.stack([x, y, z], dim=1).view(-1, 3) + at
    # look_at_rotation
    cam, at_, up_ = _broadcast(C_, at, up, device=device)
    z_axis = F.normalize(at_ - cam, eps=1e-5)
    x_axis = F.normalize(torch.cross(up_, z_axis, dim=1), eps=1e-5)
    y_axis = F.normalize(torch.cross(z_axis, x_axis, dim=1), eps=1e-5)
    is_close = torch.isclose(x_axis, torch.tensor(0.0), atol=5e-3).all(dim=1, keepdim=True)
    if is_close.any():
        replacement = F.normalize(torch.cross(y_axis, z_axis, dim=1), eps=1e-5)
        x_axis = torch.where(is_close, replacement, x_axis)
    R = torch.cat((x_axis[:, None, :], y_axis[:, None, :], z_axis[:, None, :]), dim=1).transpose(1, 2)
    T = -torch.bmm(R.transpose(1, 2), C_[:, :, None])[:, :, 0]
    return R, T


def orbit_reference(cam_param: Dict[str, torch.Tensor], mesh: torch.Tensor, root_joint_cam: torch.Tensor, i: int,
                    n_frames: int, anchors: dict, mean_3d: Optional[torch.Tensor] = None, k: int = 16) -> dict:
    """animate_view_rot.py:79-97 and :103 as written, with torch.inverse, for frame i: `mesh` (V,3) and
    `root_joint_cam` (3) are the layer's outputs in camera coordinates, `anchors` a dict the caller keeps across
    frames (frame 0 fills it), `mean_3d` the posed Gaussians (recentred on a copy).  Returns cam_param_rot, the mesh in
    the render camera, the recentred mean_3d and root_joint_world."""
    mesh = torch.matmul(torch.inverse(cam_param['R']), (mesh - cam_param['t'].view(-1, 3)).permute(1, 0)).permute(1, 0)
    root_joint_world = torch.matmul(torch.inverse(cam_param['R']), root_joint_cam - cam_param['t'])
    azim = math.pi + math.pi * k * i / n_frames
    if i == 0:
        anchors["at_point_orig"] = root_joint_world.clone()
        anchors["at_point"] = root_joint_world
        cam_pos = torch.matmul(torch.inverse(cam_param['R']), -cam_param['t'].view(3, 1)).view(3)
        at_point_cam = root_joint_cam
        anchors["elev"] = torch.arctan(torch.abs(at_point_cam[1]) / torch.abs(at_point_cam[2]))
        anchors["dist"] = torch.sqrt(torch.sum((cam_pos - anchors["at_point"]) ** 2))
    at_point_orig = anchors["at_point_orig"]
    mesh[:, [0, 2]] = mesh[:, [0, 2]] - root_joint_world[None, [0, 2]] + at_point_orig[None, [0, 2]]
    R, t = look_at_view_transform_reference(dist=anchors["dist"], elev=anchors["elev"], azim=azim, degrees=False,
                                            at=anchors["at_point"][None, :], up=((0, 1, 0),))
    R = torch.inverse(R)
    dev = cam_param['R'].device
    cam_param_rot = {'R': R[0].to(dev), 't': t[0].to(dev), 'focal': cam_param['focal'],
                     'princpt': cam_param['princpt']}
    mesh = torch.matmul(cam_param_rot['R'], mesh.permute(1, 0)).permute(1, 0) + cam_param_rot['t'].view(1, 3)
    out = {"cam_param_rot": cam_param_rot, "mesh": mesh, "root_joint_world": root_joint_world}
    if mean_3d is not None:
        mean_3d = mean_3d.clone()
        mean_3d[:, [0, 2]] = mean_3d[:, [0, 2]] - root_joint_world[None, [0, 2]] + at_point_orig[None, [0, 2]]
        out["mean_3d"] = mean_3d
    return out


def animation_panel_reference(frame_u8, mesh_panel, render) -> np.ndarray:
    """animate.py:86,94's numpy expressions without the text: the (H, 3W, 3) uint8 frame of the source frame,
    render_mesh(...).astype(np.uint8) and (render.transpose(1,2,0)[:,:,::-1]*255).copy().astype(np.uint8)."""
    as_np = lambda t: t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)  # noqa: E731
    img = as_np(frame_u8)
    mesh_render = as_np(mesh_panel).astype(np.uint8)
    r = as_np(render)
    r = r.reshape(r.shape[-3:])
    render_u8 = (r.transpose(1, 2, 0)[:, :, ::-1] * 255).copy().astype(np.uint8)
    return np.concatenate((img, mesh_render, render_u8), 1).astype(np.uint8)
