"""ExAvatar's per-frame SMPL-X pose decode and HumanGaussian's asset code around its networks as sync-free CUDA ops.

`decode_smplx_pose` is `SMPLXParamDict.forward` (avatar/common/nets/module.py:673-684) for one frame: pytorch3d's
`matrix_to_axis_angle(rotation_6d_to_matrix(p))` of the seven 6D pose parameters in one launch each way
(csrc/smplx_pose.cu).  In PyTorch that route is hundreds of kernels, and `_sqrt_positive_part`'s and the candidate
pick's boolean-mask indexings read the device from the host three times per parameter.  The op writes the (55,3) pose
in `cat_full_pose` order once; the seven per-key tensors are views of it.

`HumanAssets` holds HumanGaussian's hand / face mask, its constant identity rotation and unit opacity, built once, and
computes the code around the networks (module.py:524-539, 561 and model.py:92-96) in two ops (csrc/human_assets.cu):
`geometry` (means, scales, the masked mean_offset_offset, the warm-up clamp) and `colors` (the two tanh colours, after
skinning).  Every forward output is bit-identical to ExAvatar's fp32 torch expressions.

    smplx_param = decode_smplx_pose(smplx_params[frame])           # the frame's ParameterDict (6D poses)
    rig_out = rig(shape_param, joint_offset, smplx_param['full_pose'], smplx_param['expr'])
    ha = HumanAssets(is_rhand, is_lhand, is_face_expr)             # once, next to HumanGaussian
    geo_a = ha.geometry(rig_out.mesh_neutral_pose, rig_out.pose_offset, rig_out.expr_offset, geo, geo_offset,
                        warmup=cfg.is_warmup)
    rgb, rgb_refined = ha.colors(rgb, rgb_offset)

`decode_smplx_pose_reference`, `human_geometry_reference` and `human_colors_reference` restate the reference lines in
device-agnostic torch (float64 or float32) for tests and measurements; the product path never calls them.
"""
from __future__ import annotations

import ctypes as C
import numbers

import torch

from . import _lib as L
from .smplx_rig import matrix_to_axis_angle, matrix_to_quaternion, rotation_6d_to_matrix

# SMPLXParamDict's pose keys in cat_full_pose order and their rows in SMPL-X (root, 21 body, jaw, eyes, 15 per hand)
POSE_KEYS = ("root_pose", "body_pose", "jaw_pose", "leye_pose", "reye_pose", "lhand_pose", "rhand_pose")
POSE_ROWS = (1, 21, 1, 1, 1, 15, 15)
WARMUP_SCALE_MAX = 0.001  # model.py:94


class _DecodePose(torch.autograd.Function):
    @staticmethod
    def forward(ctx, *params):
        dev = params[0].device
        rows = [p.detach().reshape(-1, 6).contiguous() for p in params]
        st = L.B2RSmplxPose()
        for k, r in enumerate(rows):
            st.param[k], st.rows[k] = L.ptr(r), r.shape[0]
        full = torch.empty((sum(POSE_ROWS), 3), dtype=torch.float32, device=dev)
        L.run("b2r_decode_pose_forward", dev, C.byref(st), L.ptr(full))
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(*rows)
        ctx.shapes = [p.shape for p in params]
        return full

    @staticmethod
    def backward(ctx, g_full):
        if g_full is None:
            return (None,) * len(POSE_KEYS)
        rows = ctx.saved_tensors
        dev = rows[0].device
        st, gs = L.B2RSmplxPose(), L.B2RSmplxPoseGrads()
        grads = [torch.empty_like(r) for r in rows]
        for k, (r, g) in enumerate(zip(rows, grads)):
            st.param[k], st.rows[k], gs.param[k] = L.ptr(r), r.shape[0], L.ptr(g)
        up = g_full.to(torch.float32).contiguous()
        L.run("b2r_decode_pose_backward", dev, C.byref(st), L.ptr(up), C.byref(gs))
        return tuple(g.reshape(s) for g, s in zip(grads, ctx.shapes))


def decode_smplx_pose(smplx_param) -> dict:
    """SMPLXParamDict.forward for one frame.  `smplx_param` maps the seven pose keys to ExAvatar's stored 6D
    parameters ((6,) or (n,6) float32 CUDA tensors, n = 1, 21, 1, 1, 1, 15, 15 rows in POSE_KEYS order), plus `expr`
    and `trans`.  Returns the reference's dict -- each pose key in axis-angle, (3,) or (n,3) as stored, `expr` and
    `trans` passed through -- plus `full_pose` (55,3) in cat_full_pose order, of which the seven pose entries are
    views (SmplxRig reads it without a torch.cat).  The shapes are checked on the host; nothing reads the device.
    Gradients reach every 6D parameter, finite at the identity."""
    params = [smplx_param[k] for k in POSE_KEYS]
    dev = params[0].device if isinstance(params[0], torch.Tensor) else None
    for k, p, n in zip(POSE_KEYS, params, POSE_ROWS):
        L.cuda("decode_smplx_pose", k, p, dev)
        L.float32("decode_smplx_pose", k, p)
        if not (tuple(p.shape) == (n, 6) or (n == 1 and tuple(p.shape) == (6,))):
            want = f"({n},6)" + (" or (6,)" if n == 1 else "")
            raise ValueError(f"decode_smplx_pose: `{k}` must be {want} (SMPL-X's 55-joint order), "
                             f"got {tuple(p.shape)}")
    full = _DecodePose.apply(*params)
    out, r0 = {}, 0
    for k, p, n in zip(POSE_KEYS, params, POSE_ROWS):
        out[k] = full[r0:r0 + n] if p.dim() == 2 else full[r0]
        r0 += n
    for k in ("expr", "trans"):
        if k in smplx_param:
            out[k] = smplx_param[k]
    out["full_pose"] = full
    return out


class _TableDecode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, table, slot_t, host_slot, pose, expr, trans):
        st = table._struct(slot_t, host_slot)
        dev = table.device
        full = torch.empty((table.n_joints, 3), dtype=torch.float32, device=dev)
        e = torch.empty((table.n_expr,), dtype=torch.float32, device=dev)
        t = torch.empty((3,), dtype=torch.float32, device=dev)
        L.run("b2r_param_table_forward", dev, C.byref(st), L.ptr(full), L.ptr(e), L.ptr(t))
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(*(x for x in (slot_t,) if x is not None))
        ctx.meta = (table, slot_t is not None, host_slot)
        return full, e, t

    @staticmethod
    def backward(ctx, g_full, g_expr, g_trans):
        table, on_device, host_slot = ctx.meta
        slot_t = ctx.saved_tensors[0] if on_device else None
        st = table._struct(slot_t, host_slot)
        up = [None if g is None else g.to(torch.float32).contiguous() for g in (g_full, g_expr, g_trans)]
        outs = [torch.empty_like(x) for x in (table.pose, table.expr, table.trans)]
        gs = L.B2RSmplxParamTableGrads(*[L.ptr(x) for x in (*up, *outs)])
        L.run("b2r_param_table_backward", table.device, C.byref(st), C.byref(gs))
        return (None, None, None, *outs)


class SmplxParamTable:
    """Every frame's SMPL-X parameters of SMPLXParamDict (module.py:654-684) in three fp32 CUDA leaves, one frame read
    by a slot on the device, so that one captured graph serves every frame:

        pose  (F, 55, 6)  ExAvatar's stored 6D values as they are, in POSE_KEYS / POSE_ROWS (cat_full_pose) order
        expr  (F, NE)
        trans (F, 3)

        table = SmplxParamTable.from_param_dict(smplx_params)   # SMPLXParamDict.smplx_params, frame key -> nine keys
        smplx_param = table(table.slot_of(frame_idx))           # decode_smplx_pose's dict for that frame
        table.write_to(smplx_params)                            # the rows back, e.g. before a checkpoint

    `table(slot)` is one launch each way and bit-identical to `decode_smplx_pose` on that frame's ParameterDict,
    forward and gradients.  The backward writes the whole (F, ...) gradients: the slot's rows, zeros elsewhere.  The
    slot is a host int (checked on the host) or a one-element int32 CUDA tensor read on the device; a device slot
    outside [0, F) reads and writes no frame's row: the outputs are NaN and the gradients zero."""

    def __init__(self, pose, expr, trans, frames=None, pose_shapes=None):
        """pose (F, 55, 6), expr (F, NE) and trans (F, 3) contiguous float32 tensors on one CUDA device, used as they
        are (leaves with requires_grad); `frames` the frame keys of the F slots in order (default "0" ... "F-1");
        `pose_shapes` the stored shape of each pose key, (6,) or (n,6) (default (6,) for the one-row keys, as
        SMPLXParamDict.init stores them)."""
        fn = "SmplxParamTable"
        for name, t in (("pose", pose), ("expr", expr), ("trans", trans)):
            L.cuda(fn, name, t, pose.device if isinstance(pose, torch.Tensor) else None)
            L.float32(fn, name, t)
            if not t.is_contiguous():
                raise ValueError(f"{fn}: `{name}` must be contiguous")
        J = sum(POSE_ROWS)
        F = pose.shape[0] if pose.dim() == 3 else -1
        if F < 1 or tuple(pose.shape[1:]) != (J, 6):
            raise ValueError(f"{fn}: `pose` must be (F, {J}, 6) with F >= 1, got {tuple(pose.shape)}")
        if expr.dim() != 2 or expr.shape[0] != F:
            raise ValueError(f"{fn}: `expr` must be ({F}, NE), got {tuple(expr.shape)}")
        if tuple(trans.shape) != (F, 3):
            raise ValueError(f"{fn}: `trans` must be ({F}, 3), got {tuple(trans.shape)}")
        if F >= 2 ** 31:
            raise ValueError(f"{fn}: at most 2^31 - 1 frames")
        frames = [str(f) for f in (range(F) if frames is None else frames)]
        if len(frames) != F or len(set(frames)) != F:
            raise ValueError(f"{fn}: `frames` must name the {F} slots once each")
        self.pose, self.expr, self.trans = pose, expr, trans
        self.device = pose.device
        self.n_frames, self.n_joints, self.n_expr = F, int(pose.shape[1]), int(expr.shape[1])
        self.frames = frames
        self._slot = {f: i for i, f in enumerate(frames)}
        self.pose_shapes = tuple((6,) if n == 1 else (n, 6) for n in POSE_ROWS) if pose_shapes is None else \
            tuple(tuple(s) for s in pose_shapes)
        for n, shp in zip(POSE_ROWS, self.pose_shapes):
            if not (shp == (n, 6) or (n == 1 and shp == (6,))):
                raise ValueError(f"{fn}: `pose_shapes` must be (n,6) or, for one row, (6,), got {shp}")

    @classmethod
    def from_param_dict(cls, smplx_params, device=None) -> "SmplxParamTable":
        """The table of `SMPLXParamDict.smplx_params` (frame key -> the seven 6D pose keys, (6,) or (n,6), plus expr
        and trans), slots in the dict's order, values copied bit for bit into new leaves (requires_grad=True)."""
        fn = "SmplxParamTable.from_param_dict"
        frames = list(smplx_params.keys())
        if not frames:
            raise ValueError(f"{fn}: no frames")
        poses, exprs, transs = [], [], []
        for f in frames:
            d = smplx_params[f]
            missing = [k for k in (*POSE_KEYS, "expr", "trans") if k not in d]
            if missing:
                raise ValueError(f"{fn}: frame {f!r} lacks {missing}")
            for k, n in zip(POSE_KEYS, POSE_ROWS):
                v, v0 = d[k], smplx_params[frames[0]][k]
                if not (tuple(v.shape) == (n, 6) or (n == 1 and tuple(v.shape) == (6,))):
                    want = f"({n},6)" + (" or (6,)" if n == 1 else "")
                    raise ValueError(f"{fn}: frame {f!r} `{k}` must be {want}, got {tuple(v.shape)}")
                if v.shape != v0.shape:
                    raise ValueError(f"{fn}: frame {f!r} stores `{k}` as {tuple(v.shape)}, the first frame as "
                                     f"{tuple(v0.shape)}")
            if d["expr"].dim() != 1 or tuple(d["trans"].shape) != (3,):
                raise ValueError(f"{fn}: frame {f!r} needs expr (NE,) and trans (3,), got "
                                 f"{tuple(d['expr'].shape)} and {tuple(d['trans'].shape)}")
            poses.append(torch.cat([d[k].detach().reshape(-1, 6) for k in POSE_KEYS]))
            exprs.append(d["expr"].detach())
            transs.append(d["trans"].detach())
        if len({e.shape[0] for e in exprs}) != 1:
            raise ValueError(f"{fn}: the frames' expr lengths differ")
        dev = torch.device(device) if device is not None else poses[0].device
        leaf = lambda xs: torch.stack(xs).to(device=dev, dtype=torch.float32).contiguous().requires_grad_()  # noqa: E731
        first = smplx_params[frames[0]]
        return cls(leaf(poses), leaf(exprs), leaf(transs), frames, [tuple(first[k].shape) for k in POSE_KEYS])

    @torch.no_grad()
    def write_to(self, smplx_params) -> None:
        """Copies every slot's rows back into `smplx_params` (the dict from_param_dict read), in place and bit for
        bit, each key keeping its stored shape."""
        for f, i in self._slot.items():
            d, r0 = smplx_params[f], 0
            for k, n in zip(POSE_KEYS, POSE_ROWS):
                d[k].copy_(self.pose[i, r0:r0 + n].reshape(d[k].shape))
                r0 += n
            d["expr"].copy_(self.expr[i])
            d["trans"].copy_(self.trans[i])

    def slot_of(self, frame_idx) -> int:
        """The slot of a frame: its key, or ExAvatar's int frame index (looked up as str(int(frame_idx)))."""
        key = frame_idx if isinstance(frame_idx, str) else str(int(frame_idx))
        if key not in self._slot:
            raise KeyError(f"SmplxParamTable: no frame {key!r}")
        return self._slot[key]

    def parameters(self):
        return [self.pose, self.expr, self.trans]

    def _struct(self, slot_t, host_slot: int = 0):
        return L.B2RSmplxParamTable(n_frames=self.n_frames, n_joints=self.n_joints, n_expr=self.n_expr,
                                    host_slot=host_slot, pose=L.ptr(self.pose), expr=L.ptr(self.expr),
                                    trans=L.ptr(self.trans), slot=L.ptr(slot_t))

    def __call__(self, slot) -> dict:
        """decode_smplx_pose's dict for the frame in `slot`: the seven pose keys in axis-angle as views of
        `full_pose` (J,3), plus `full_pose`, `expr` (NE) and `trans` (3), all fresh tensors."""
        fn = "SmplxParamTable"
        if isinstance(slot, torch.Tensor):
            L.cuda(fn, "slot", slot, self.device)
            if slot.dtype != torch.int32 or slot.numel() != 1 or not slot.is_contiguous():
                raise ValueError(f"{fn}: a tensor `slot` must be one contiguous int32 value, got {slot.dtype} "
                                 f"{tuple(slot.shape)}")
            full, expr, trans = _TableDecode.apply(self, slot, 0, self.pose, self.expr, self.trans)
        elif isinstance(slot, numbers.Integral) and not isinstance(slot, bool):
            if not 0 <= int(slot) < self.n_frames:
                raise IndexError(f"{fn}: slot {int(slot)} outside [0, {self.n_frames})")
            full, expr, trans = _TableDecode.apply(self, None, int(slot), self.pose, self.expr, self.trans)
        else:
            raise ValueError(f"{fn}: `slot` must be an int or a (1,) int32 CUDA tensor, got {type(slot).__name__}")
        out, r0 = {}, 0
        for k, n, shp in zip(POSE_KEYS, POSE_ROWS, self.pose_shapes):
            out[k] = full[r0:r0 + n] if len(shp) == 2 else full[r0]
            r0 += n
        out.update(expr=expr, trans=trans, full_pose=full)
        return out


def decode_smplx_pose_reference(smplx_param) -> dict:
    """module.py:677-683 restated in torch for one frame (pytorch3d's conversions as smplx_rig restates them), in the
    parameters' dtype and device, plus `full_pose` = cat_full_pose of the result."""
    out = {k: (matrix_to_axis_angle(rotation_6d_to_matrix(v)) if "pose" in k else v) for k, v in smplx_param.items()}
    out["full_pose"] = torch.cat([out[k].reshape(-1, 3) for k in POSE_KEYS])
    return out


def _rows4(t: torch.Tensor):
    """(tensor, row stride): (P,4) rows of 4 contiguous floats read in place, or a contiguous copy."""
    if t.stride(1) == 1 and (t.shape[0] <= 1 or t.stride(0) >= 4):
        return t, max(int(t.stride(0)), 4)
    return t.contiguous(), 4


class _Geometry(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ha, warmup, mesh, pose_offset, expr_offset, geo, geo_offset):
        dev = ha.device
        P = ha.P
        g4, gs = _rows4(geo.detach())
        o4, os_ = _rows4(geo_offset.detach())
        ins = [t.detach().contiguous() for t in (mesh, pose_offset, expr_offset)]
        st = L.B2RHumanAssets(P=P, warmup=int(warmup), geo_stride=gs, geo_offset_stride=os_)
        st.mesh, st.pose_offset, st.expr_offset = (L.ptr(t) for t in ins)
        st.geo, st.geo_offset, st.mask = L.ptr(g4), L.ptr(o4), L.ptr(ha.mask)
        outs = [torch.empty((P, 3), dtype=torch.float32, device=dev) for _ in range(7 if warmup else 5)]
        ptrs = [L.ptr(o) for o in outs] + [None, None] * (not warmup)
        L.run("b2r_human_geometry_forward", dev, C.byref(st), *ptrs)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(*ins, g4, o4)
        ctx.meta = (ha, st, geo.shape, geo_offset.shape)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        mesh, pose_offset, expr_offset, g4, o4 = ctx.saved_tensors
        ha, st, geo_shape, off_shape = ctx.meta
        dev = ha.device
        up = [None if g is None else g.to(torch.float32).contiguous() for g in grads]
        up += [None] * (7 - len(up))
        f = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)  # noqa: E731
        d_mesh, d_expr, d_geo, d_off = f(ha.P, 3), f(ha.P, 3), f(ha.P, 4), f(ha.P, 4)
        gs = L.B2RHumanAssetsGrads(*[L.ptr(x) for x in (*up, d_mesh, d_expr, d_geo, d_off)])
        L.run("b2r_human_geometry_backward", dev, C.byref(st), C.byref(gs))
        return None, None, d_mesh, None, d_expr, d_geo.reshape(geo_shape), d_off.reshape(off_shape)


class _Colors(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rgb, rgb_offset):
        dev = rgb.device
        x, o = rgb.detach().contiguous(), rgb_offset.detach().contiguous()
        P = x.shape[0]
        out, out_r = torch.empty_like(x), torch.empty_like(x)
        L.run("b2r_human_colors_forward", dev, P, L.ptr(x), L.ptr(o), L.ptr(out), L.ptr(out_r))
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(x, o)
        return out, out_r

    @staticmethod
    def backward(ctx, g, g_r):
        x, o = ctx.saved_tensors
        dev = x.device
        g, g_r = (None if t is None else t.to(torch.float32).contiguous() for t in (g, g_r))
        d_rgb, d_off = torch.empty_like(x), torch.empty_like(x)
        L.run("b2r_human_colors_backward", dev, x.shape[0], L.ptr(x), L.ptr(o), L.ptr(g), L.ptr(g_r), L.ptr(d_rgb),
              L.ptr(d_off))
        return d_rgb, d_off


class HumanAssets:
    """HumanGaussian's per-Gaussian tables for the two ops, built once (may synchronise): the hand / face mask
    (is_rhand | is_lhand | is_face_expr, module.py:489) as float 0 / 1, the constant identity `rotation` (P,4) and the
    unit `opacity` (P,1) of module.py:564-565.  `device` is where they live (CUDA)."""

    def __init__(self, is_rhand, is_lhand, is_face_expr, device=None):
        device = torch.device(device if device is not None else "cuda")
        if device.type != "cuda":
            raise RuntimeError(f"HumanAssets: device must be CUDA (got {device}); there is no CPU fallback")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        masks = [torch.as_tensor(m).detach().reshape(-1) for m in (is_rhand, is_lhand, is_face_expr)]
        if len({m.numel() for m in masks}) != 1:
            raise ValueError(f"HumanAssets: the three masks differ in length: {[m.numel() for m in masks]}")
        self.device = device
        self.P = masks[0].numel()
        self.mask = ((masks[0] != 0) | (masks[1] != 0) | (masks[2] != 0)).to(device=device, dtype=torch.float32)
        self.rotation = torch.zeros((self.P, 4), dtype=torch.float32, device=device)
        self.rotation[:, 0] = 1
        self.opacity = torch.ones((self.P, 1), dtype=torch.float32, device=device)

    def geometry(self, mesh_neutral_pose, pose_offset, expr_offset, geo, geo_offset, warmup: bool = False) -> dict:
        """module.py:524-539 and model.py:92-96 from the rig's mesh_neutral_pose, pose_offset (already masked) and
        expr_offset, (P,3), and the networks' geo (P,4) = mean_offset | scale and geo_offset (P,4) = mean_offset_offset
        | scale_offset, float32 CUDA tensors (geo / geo_offset may be column views of a wider tensor).  Returns
        mean_3d and mean_3d_refined (before skinning), scale and scale_refined (P,3), the masked mean_offset_offset
        (P,3), and the views mean_offset = geo[:, :3] and scale_offset = geo_offset[:, 3:] (ExAvatar's offsets).
        warmup=True clamps both scales to max=0.001 and adds scale_wo_clamp / scale_refined_wo_clamp.  Gradients reach
        the mesh, expr_offset, geo and geo_offset; pose_offset gets none (ExAvatar detaches the pose there)."""
        P, dev = self.P, self.device
        for name, t, shape in (("mesh_neutral_pose", mesh_neutral_pose, (P, 3)), ("pose_offset", pose_offset, (P, 3)),
                               ("expr_offset", expr_offset, (P, 3)), ("geo", geo, (P, 4)),
                               ("geo_offset", geo_offset, (P, 4))):
            L.cuda("HumanAssets.geometry", name, t, dev)
            L.float32("HumanAssets.geometry", name, t)
            if tuple(t.shape) != shape:
                raise ValueError(f"HumanAssets.geometry: `{name}` must be {shape}, got {tuple(t.shape)}")
        outs = _Geometry.apply(self, bool(warmup), mesh_neutral_pose, pose_offset, expr_offset, geo, geo_offset)
        names = ("mean_3d", "mean_3d_refined", "scale", "scale_refined", "mean_offset_offset", "scale_wo_clamp",
                 "scale_refined_wo_clamp")
        res = dict(zip(names, outs))
        res.update(mean_offset=geo[:, :3], scale_offset=geo_offset[:, 3:])
        return res

    def colors(self, rgb, rgb_offset):
        """module.py:561: ((tanh(rgb) + 1) / 2, (tanh(rgb + rgb_offset) + 1) / 2) from the (P,3) float32 CUDA network
        outputs; gradients reach both."""
        for name, t in (("rgb", rgb), ("rgb_offset", rgb_offset)):
            L.cuda("HumanAssets.colors", name, t, self.device)
            L.float32("HumanAssets.colors", name, t)
            if tuple(t.shape) != (self.P, 3):
                raise ValueError(f"HumanAssets.colors: `{name}` must be ({self.P}, 3), got {tuple(t.shape)}")
        return _Colors.apply(rgb, rgb_offset)


def human_geometry_reference(mesh_neutral_pose, pose_offset, expr_offset, geo, geo_offset, mask,
                             warmup: bool = False) -> dict:
    """module.py:524-539 (get_mean_offset_offset's :489-493 with the rig's already-masked pose offset) and
    model.py:92-96 in torch, in the inputs' dtype and ExAvatar's order of operations: in float32 on CUDA these are
    ExAvatar's own expressions.  `mask` (P,) is is_rhand | is_lhand | is_face_expr."""
    mean_offset, scale = geo[:, :3], geo[:, 3:]
    mean_offset_offset, scale_offset = geo_offset[:, :3], geo_offset[:, 3:]
    mean_3d = mesh_neutral_pose + mean_offset
    scale, scale_refined = torch.exp(scale).repeat(1, 3), torch.exp(scale + scale_offset).repeat(1, 3)
    m = (mask > 0)[:, None].to(geo.dtype)
    mean_offset_offset = mean_offset_offset * (1 - m)
    mean_3d_refined = mean_3d + (mean_offset_offset + pose_offset)
    res = {"mean_3d": mean_3d + expr_offset, "mean_3d_refined": mean_3d_refined + expr_offset, "scale": scale,
           "scale_refined": scale_refined, "mean_offset_offset": mean_offset_offset}
    if warmup:
        res["scale_wo_clamp"], res["scale_refined_wo_clamp"] = scale.clone(), scale_refined.clone()
        res["scale"] = torch.clamp(scale, max=WARMUP_SCALE_MAX)
        res["scale_refined"] = torch.clamp(scale_refined, max=WARMUP_SCALE_MAX)
    return res


def human_colors_reference(rgb, rgb_offset):
    """module.py:561 in torch."""
    return (torch.tanh(rgb) + 1) / 2, (torch.tanh(rgb + rgb_offset) + 1) / 2


def constant_rotation_reference(P: int, dtype=torch.float64, device=None):
    """module.py:564: the quaternion of P identity matrices, through matrix_to_quaternion."""
    return matrix_to_quaternion(torch.eye(3, dtype=dtype, device=device)[None].repeat(P, 1, 1))
