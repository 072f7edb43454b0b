"""A trained avatar animated on the device: ExAvatar's animate.py and animate_view_rot.py video loop as one table and
one CUDA graph replay per video frame.

Each frame of the scripts reads two JSON files and a PNG, runs `HumanGaussian.forward` in PyTorch (the SMPL-X rig, the
triplane, four GroupNorm MLP stacks, pytorch3d's brute-force knn) and renders through the polling path, then keeps
only `human_asset` (animate.py:65-66, animate_view_rot.py:102-104).  For a trained avatar that set depends on the frame
only through the rig and the camera: mesh_neutral_pose, tri_feat, geo_net -> mean_offset / scale and rgb_net -> rgb
are constants, and geo_offset_net / rgb_offset_net feed only the refined set the scripts discard.  So a video frame
needs no network:

    motion = MotionTable.from_folder(motion_path, "cuda")        # every frame's parameters, camera and bytes, once
    animator = AvatarAnimator(motion, rig, tri, assets, mesh_renderer, triplane=..., ...)   # constants, once
    for frame_idx, panel in animator.frames():                    # (H, 3W, 3) uint8 BGR, before the text
        ... cv2.putText on panel[:, :W], panel[:, W:2W], panel[:, 2W:] and panel; video_out.write(panel)

Per frame the device runs the existing ops: `SmplxRig` (joint transforms, expr_offset), the asset sum in
`HumanAssets.geometry`'s fp32 order, `nearest_rows`, `skin_gaussians` on one set, `device_render_settings` +
`GaussianRasterizer`'s call (`rasterize_gaussians`) with a per-call fixed capacity, `SmplxRig.body_mesh`,
`ShadedMeshRenderer` and `animation_panel` (with `OrbitCamera` and `orbit_points` for animate_view_rot.py).  The frame is picked by a device slot with tensor indexing,
so one captured graph serves the whole sequence.
"""
from __future__ import annotations

import ctypes as C
import glob
import json
import os
from collections import deque
from typing import Iterator, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib as L
from . import rasterizer as _rz
from .animation import OrbitCamera, animation_panel, orbit_points
from .geometry import nearest_rows
from .human_assets import POSE_KEYS, POSE_ROWS
from .human_nets import gn_mlp
from .renderer import device_render_settings
from .skinning import skin_gaussians

# the nine keys of smplx_optimized/smplx_params_smoothed/{idx}.json and the four of cam_params/{idx}.json with their
# lengths after `.view(-1)`; expr's length is the first frame's
SMPLX_KEYS = POSE_KEYS + ("expr", "trans")
SMPLX_LENGTHS = dict(zip(POSE_KEYS, (3 * n for n in POSE_ROWS)), trans=3)
CAM_LENGTHS = {"R": 9, "t": 3, "focal": 2, "princpt": 2}
# the list capacity taken from the first frame's duplicate count when the caller gives none: the motion moves the
# body, so later frames can need more than the first
CAPACITY_FROM_FIRST = 2.0
_STATUS_BYTES = C.sizeof(L.B2RStatus)


def _floats(v, what: str, n: Optional[int]) -> torch.Tensor:
    """The scripts' `torch.FloatTensor(v).view(-1)`, refused unless v is a list of n numbers after flattening."""
    if not isinstance(v, list):
        raise ValueError(f"MotionTable: {what} must be a list of numbers, got {type(v).__name__}")
    try:
        t = torch.FloatTensor(v).view(-1)
    except (TypeError, ValueError, RuntimeError) as e:
        raise ValueError(f"MotionTable: {what} is not a list of numbers ({e})") from None
    if n is not None and t.numel() != n:
        raise ValueError(f"MotionTable: {what} has {t.numel()} values, expected {n}")
    return t


def _json(path: str) -> dict:
    if not os.path.isfile(path):
        raise ValueError(f"MotionTable: missing {path}")
    with open(path) as f:
        d = json.load(f)
    if not isinstance(d, dict):
        raise ValueError(f"MotionTable: {path} does not hold a JSON object")
    return d


def read_motion(motion_path: str) -> dict:
    """The host half of `MotionTable.from_folder`: every file of a motion folder read once and checked, nothing
    uploaded.  Frames come in the scripts' order, `sorted(int(name[:-5]))` of smplx_optimized/smplx_params_smoothed/
    *.json.  Returns CPU arrays: frame_idx (F,) int64, pose (F,55,3), expr (F,NE), trans (F,3), R (F,3,3), t (F,3),
    focal (F,2), princpt (F,2) float32 with the bits of `torch.FloatTensor(v).view(-1)`, and frames (F,H,W,3) uint8,
    the BGR bytes of `cv2.imread`.

    Raises ValueError on a missing file or key, a file name that is not an integer, a value of the wrong length, and a
    frame whose size differs from frame 0's (the scripts size the VideoWriter from frame 0; cv2 silently drops frames
    of another size)."""
    import cv2
    root = os.path.join(motion_path, "smplx_optimized", "smplx_params_smoothed")
    names = [os.path.basename(p)[:-5] for p in glob.glob(os.path.join(root, "*.json"))]
    if not names:
        raise ValueError(f"MotionTable: no SMPL-X parameter files in {root}")
    try:
        frame_idx = sorted(int(s) for s in names)
    except ValueError:
        raise ValueError(f"MotionTable: a file name in {root} is not an integer frame index") from None
    if len(set(frame_idx)) != len(frame_idx):
        raise ValueError(f"MotionTable: two files in {root} name the same frame index")
    cols = {k: [] for k in ("pose", "expr", "trans", "R", "t", "focal", "princpt")}
    frames = []
    n_expr = None
    for idx in frame_idx:
        p = _json(os.path.join(root, f"{idx}.json"))
        missing = [k for k in SMPLX_KEYS if k not in p]
        if missing:
            raise ValueError(f"MotionTable: frame {idx}'s SMPL-X parameters lack {missing}")
        v = {k: _floats(p[k], f"frame {idx}'s `{k}`", SMPLX_LENGTHS.get(k, n_expr)) for k in SMPLX_KEYS}
        n_expr = v["expr"].numel() if n_expr is None else n_expr
        cols["pose"].append(torch.cat([v[k] for k in POSE_KEYS]).view(-1, 3))
        cols["expr"].append(v["expr"])
        cols["trans"].append(v["trans"])
        c = _json(os.path.join(motion_path, "cam_params", f"{idx}.json"))
        missing = [k for k in CAM_LENGTHS if k not in c]
        if missing:
            raise ValueError(f"MotionTable: frame {idx}'s camera lacks {missing}")
        for k, n in CAM_LENGTHS.items():
            cols[k].append(_floats(c[k], f"frame {idx}'s camera `{k}`", n))
        png = os.path.join(motion_path, "frames", f"{idx}.png")
        img = cv2.imread(png) if os.path.isfile(png) else None
        if img is None:
            raise ValueError(f"MotionTable: missing or unreadable {png}")
        if frames and img.shape != frames[0].shape:
            raise ValueError(f"MotionTable: frame {idx} is {img.shape[1]}x{img.shape[0]}, frame {frame_idx[0]} is "
                             f"{frames[0].shape[1]}x{frames[0].shape[0]}")
        frames.append(img)
    out = {k: torch.stack(v) for k, v in cols.items()}
    out["R"] = out["R"].view(-1, 3, 3)
    out["frame_idx"] = torch.tensor(frame_idx, dtype=torch.int64)
    out["frames"] = frames
    return out


class MotionTable:
    """A driving motion on one CUDA device, built once, read by a device slot (the frame's position in the motion):

        pose     (F,55,3)   axis-angle in `cat_full_pose` order, as SmplxRig and body_mesh take it
        expr     (F,NE), trans (F,3)
        R (F,3,3), t (F,3), focal (F,2), princpt (F,2)   the frame's camera (cam_params/{idx}.json)
        frames   (F,H,W,3)  uint8, the source frames' BGR bytes
        frame_idx           the frame indices in motion order (host ints)

    `table(slot)` gathers one frame with plain tensor indexing; a (1,) integer CUDA slot is read on the device, so the
    gather can be captured in a CUDA graph."""

    def __init__(self, frame_idx: Sequence[int], pose, expr, trans, R, t, focal, princpt, frames):
        F = len(frame_idx)
        self.frame_idx = [int(i) for i in frame_idx]
        self.pose, self.expr, self.trans, self.R, self.t, self.focal, self.princpt, self.frames = (
            pose, expr, trans, R, t, focal, princpt, frames)
        self.device = pose.device
        for name, x, shape in (("pose", pose, (F, 55, 3)), ("trans", trans, (F, 3)), ("R", R, (F, 3, 3)),
                               ("t", t, (F, 3)), ("focal", focal, (F, 2)), ("princpt", princpt, (F, 2))):
            L.cuda("MotionTable", name, x, self.device)
            L.float32("MotionTable", name, x)
            if tuple(x.shape) != shape:
                raise ValueError(f"MotionTable: `{name}` must be {shape}, got {tuple(x.shape)}")
        L.cuda("MotionTable", "expr", expr, self.device)
        L.cuda("MotionTable", "frames", frames, self.device)
        if expr.dim() != 2 or expr.shape[0] != F or frames.dtype != torch.uint8 or frames.dim() != 4 or \
                frames.shape[0] != F or frames.shape[3] != 3:
            raise ValueError(f"MotionTable: expr must be ({F}, NE) and frames ({F}, H, W, 3) uint8")
        self.n_frames = F
        self.image_shape = (int(frames.shape[1]), int(frames.shape[2]))

    @classmethod
    def from_folder(cls, motion_path: str, device=None) -> "MotionTable":
        """The table of a motion folder as animate.py reads it (`read_motion`, which checks every file before anything
        is uploaded), uploaded frame by frame into one device array."""
        host = read_motion(motion_path)
        device = torch.device(device if device is not None else "cuda")
        if device.type != "cuda":
            raise RuntimeError(f"MotionTable: device must be CUDA (got {device}); there is no CPU fallback")
        frames = host.pop("frames")
        pixels = torch.empty((len(frames), *frames[0].shape), dtype=torch.uint8, device=device)
        for i, img in enumerate(frames):
            pixels[i].copy_(torch.from_numpy(img))
        d = {k: v.to(device) for k, v in host.items() if k != "frame_idx"}
        return cls(host["frame_idx"].tolist(), d["pose"], d["expr"], d["trans"], d["R"], d["t"], d["focal"],
                   d["princpt"], pixels)

    @property
    def nbytes(self) -> int:
        """Device bytes of the table (the source frames take H·W·3 each)."""
        return sum(x.numel() * x.element_size() for x in (self.pose, self.expr, self.trans, self.R, self.t,
                                                         self.focal, self.princpt, self.frames))

    def __call__(self, slot) -> dict:
        """Frame `slot`'s rows: pose (55,3), expr (NE), trans (3), cam {R (3,3), t, focal, princpt} and frame (H,W,3).
        `slot` is a host int (range-checked, IndexError) or a (1,) integer CUDA tensor read on the device (no host
        sync).  A device slot is not checked: it must lie in [0, F), as torch's indexing asserts on the device."""
        if isinstance(slot, torch.Tensor):
            L.cuda("MotionTable", "slot", slot, self.device)
            row = lambda x: x.index_select(0, slot.reshape(1))[0]  # noqa: E731
        else:
            if not 0 <= int(slot) < self.n_frames:
                raise IndexError(f"MotionTable: slot {slot} outside [0, {self.n_frames})")
            row = lambda x: x[int(slot)]  # noqa: E731
        return {"pose": row(self.pose), "expr": row(self.expr), "trans": row(self.trans),
                "cam": {k: row(getattr(self, k)) for k in CAM_LENGTHS}, "frame": row(self.frames)}


class AvatarAnimator:
    """A trained ExAvatar avatar and a `MotionTable` turned into the scripts' video panels.

    rig, tri, assets, mesh_renderer  the ops' setup objects: `SmplxRig`, `TriplaneFeatures`, `HumanAssets` and
                      `ShadedMeshRenderer(smpl_x.face, smpl_x.vertex_num)`
    triplane, triplane_face           HumanGaussian.triplane / triplane_face
    geo_net, rgb_net  the pose-free stacks as (trunk, heads) for `gn_mlp`: (geo_net, [mean_offset_net, scale_net]) and
                      (rgb_net, None)
    shape_param, joint_offset         HumanGaussian.shape_param and joint_offset (raw, as the scripts pass them)
    skinning_weight   (P,J) HumanGaussian.skinning_weight, the upsampled lbs weights
    self_map          (P,) is_rhand | is_lhand | is_face: the Gaussians that keep their own vertex's weights
    orbit             False: animate.py (the frame's camera); True: animate_view_rot.py (OrbitCamera(16, F) with the
                      frame's position as its index, anchored on frame 0, Gaussians and mesh recentred)
    capacity          the renderer's list entries per frame; None renders the first frame with the adaptive policy
                      and then takes CAPACITY_FROM_FIRST times its duplicate count + 4096
    use_graph         frame 0 runs eagerly, the next frame is captured, every later frame is one replay
    in_flight         pinned host buffers in the ring `frames()` yields from (>= 1)

    The constant assets (mesh_neutral_pose and its base vertices, tri_feat, mean_offset, scale, rgb, opacity,
    rotation) are computed once here, under no_grad, through the same ops as the full forward, so their bits are the
    full chain's; shape_param, joint_offset, skinning_weight and self_map are copied.  Later changes to the modules or
    tensors are not seen: build a new animator to pick them up."""

    def __init__(self, motion: MotionTable, rig, tri, assets, mesh_renderer, *, triplane, triplane_face, geo_net,
                 rgb_net, shape_param, joint_offset, skinning_weight, self_map, orbit: bool = False,
                 capacity: Optional[int] = None, use_graph: bool = True, in_flight: int = 2):
        fn = "AvatarAnimator"
        if isinstance(in_flight, bool) or not isinstance(in_flight, int) or in_flight < 1:
            raise ValueError(f"{fn}: in_flight must be an int >= 1, got {in_flight!r}")
        if capacity is not None and (isinstance(capacity, bool) or not isinstance(capacity, int) or capacity < 1):
            raise ValueError(f"{fn}: capacity must be a positive int or None, got {capacity!r}")
        dev = motion.device
        P = rig.P
        if skinning_weight.shape[0] != P or self_map.numel() != P or assets.P != P or tri.P != P:
            raise ValueError(f"{fn}: the rig has {P} Gaussians; skinning_weight, self_map, the assets and the "
                             "triplane table must match")
        self.motion, self.rig, self.mesh_renderer = motion, rig, mesh_renderer
        self.device, self.P = dev, P
        self.shape_param = shape_param.detach().reshape(-1).clone()
        self.joint_offset = joint_offset.detach().clone()
        self.skinning_weight = skinning_weight.detach().to(torch.float32).clone()
        self.self_map = self_map.detach().reshape(-1).to(device=dev, dtype=torch.bool).clone()
        with torch.no_grad():
            m0 = motion(0)
            out = rig(self.shape_param, self.joint_offset, m0["pose"], m0["expr"])
            self.mesh_neutral_pose = out.mesh_neutral_pose
            self.mesh_wo_upsample = out.mesh_neutral_pose_wo_upsample.contiguous()
            tri_feat = tri(triplane.detach(), triplane_face.detach())
            geo = gn_mlp([tri_feat], *geo_net)
            rgb = gn_mlp([tri_feat], *rgb_net)
            z3 = torch.zeros((P, 3), dtype=torch.float32, device=dev)
            z4 = torch.zeros((P, 4), dtype=torch.float32, device=dev)
            ga = assets.geometry(self.mesh_neutral_pose, z3, z3, geo, z4)
            # geometry's mean_3d is fl(fl(mesh + mean_offset) + expr_offset); with a zero expr_offset it is the
            # first sum, to which a frame adds its own expr_offset in the same order
            self.mean_3d_neutral = ga["mean_3d"]
            self.scale = ga["scale"]
            self.rgb = assets.colors(rgb, z3)[0]
        self.opacity, self.rotation = assets.opacity, assets.rotation
        self._means2d = torch.zeros((P, 3), dtype=torch.float32, device=dev)
        self._empty = torch.empty(0, dtype=torch.float32, device=dev)
        self._status = torch.zeros(_STATUS_BYTES, dtype=torch.uint8, device=dev)  # the render's own status block
        H, W = motion.image_shape
        self.bg = torch.ones(3, dtype=torch.float32, device=dev)  # GaussianRenderer's default background
        self.bkg = torch.full((H, W, 3), 255.0, dtype=torch.float32, device=dev)  # render_mesh's white background
        self.orbit = OrbitCamera(16, motion.n_frames, dev) if orbit else None
        self.capacity = capacity
        self.use_graph = bool(use_graph)
        self.in_flight = in_flight
        self._slot = torch.zeros(1, dtype=torch.int32, device=dev)
        self._ring = torch.empty((in_flight, H, 3 * W, 3), dtype=torch.uint8, pin_memory=True)
        self._ring_status = torch.empty((in_flight, _STATUS_BYTES), dtype=torch.uint8, pin_memory=True)
        self._events = [torch.cuda.Event() for _ in range(in_flight)]
        self._graph = None
        self._static = None
        self._ran = False

    @torch.no_grad()
    def _device_frame(self, slot: torch.Tensor) -> dict:
        """One video frame on the device, every input read through `slot` (the frame's position)."""
        fr = self.motion(slot)
        pose, expr, trans, cam = fr["pose"], fr["expr"], fr["trans"], fr["cam"]
        out = self.rig(self.shape_param, self.joint_offset, pose, expr)
        mean_3d = self.mean_3d_neutral + out.expr_offset
        rows = nearest_rows(mean_3d, self.mesh_wo_upsample, self.self_map)
        posed, _ = skin_gaussians(mean_3d, None, self.skinning_weight, rows, out.joint_mats, trans, cam["R"], cam["t"])
        body = (self.shape_param, self.joint_offset, pose, expr, trans)
        if self.orbit is not None:
            mesh, joints = self.rig.body_mesh(*body, cam["R"], cam["t"], joints=True)
            render_cam = self.orbit(cam, joints[0], slot)
            mesh = orbit_points(mesh, self.orbit, view=True)
            posed = orbit_points(posed, self.orbit)
        else:
            mesh = self.rig.body_mesh(*body)
            render_cam = cam
        settings = device_render_settings(self.motion.image_shape, render_cam, self.bg)
        render = _rz.rasterize_gaussians(posed, self._means2d, self._empty, self.rgb, self.opacity, self.scale,
                                         self.rotation, self._empty, settings, capacity=self.capacity,
                                         status=self._status)[0]
        mesh_panel = self.mesh_renderer(mesh, cam, self.bkg)
        return {"mean_3d": posed, "mesh": mesh, "camera": render_cam, "render": render, "mesh_panel": mesh_panel,
                "panel": animation_panel(fr["frame"], mesh_panel, render), "status": self._status}

    def _eager(self, i: int) -> dict:
        self._slot.fill_(i)
        out = self._device_frame(self._slot)
        if self.capacity is None:  # this frame rendered with the adaptive policy, which sized its lists exactly
            H, W = self.motion.image_shape
            self.capacity = int(CAPACITY_FROM_FIRST * _rz.last_duplicate_count(self.device, self.P, W, H)) + 4096
        self._ran = True
        return out

    def frame(self, i: int) -> dict:
        """Frame i of the motion (its position), eagerly: the posed (and, in orbit mode, recentred) Gaussians
        `mean_3d` (P,3), the body `mesh` in the render camera, the render `camera`, `render` (3,H,W), `mesh_panel`
        (H,W,3) fp32 and `panel` (H,3W,3) uint8 on the device.  The orbit camera's anchors come from position 0."""
        if not 0 <= int(i) < self.motion.n_frames:
            raise IndexError(f"AvatarAnimator: frame {i} outside [0, {self.motion.n_frames})")
        out = self._eager(int(i))
        out.pop("status")
        return out

    def _submit(self, i: int, k: int) -> None:
        if not self.use_graph or not self._ran:
            out = self._eager(i)
        else:
            if self._graph is None:
                self._slot.fill_(i)
                self._graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self._graph):
                    self._static = self._device_frame(self._slot)
            self._slot.fill_(i)
            self._graph.replay()
            out = self._static
        self._ring[k].copy_(out["panel"], non_blocking=True)
        self._ring_status[k].copy_(out["status"], non_blocking=True)
        self._events[k].record()

    def _collect(self, i: int, k: int) -> Tuple[int, np.ndarray]:
        self._events[k].synchronize()
        st = L.B2RStatus.from_buffer_copy(self._ring_status[k].numpy().tobytes())
        if st.overflow:
            raise RuntimeError(f"AvatarAnimator: frame {self.motion.frame_idx[i]} (position {i}) needed "
                               f"{st.num_dups} render list entries, the capacity is {st.dup_capacity}; its render is "
                               "truncated (pass a larger `capacity`)")
        return self.motion.frame_idx[i], self._ring[k].numpy()

    def frames(self) -> Iterator[Tuple[int, np.ndarray]]:
        """(frame_idx, panel) for every frame in motion order: panel is the (H, 3W, 3) uint8 BGR array of the scripts'
        `np.concatenate((img, mesh_render, render), 1)` before the text, a view of one of `in_flight` pinned buffers.
        The buffer stays the caller's until the next iteration; up to `in_flight` frames are queued on the device
        meanwhile.  A frame whose render overflowed the list capacity raises RuntimeError when it is collected."""
        n = self.in_flight
        pending = deque()
        for i in range(self.motion.n_frames):
            if len(pending) == n:
                yield self._collect(*pending.popleft())
            k = i % n
            self._submit(i, k)
            pending.append((i, k))
        while pending:
            yield self._collect(*pending.popleft())
