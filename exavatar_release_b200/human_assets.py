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

import torch

from . import _lib as L
from .rasterizer import _ptr
from .smplx_rig import matrix_to_axis_angle, matrix_to_quaternion, rotation_6d_to_matrix

# SMPLXParamDict's pose keys in cat_full_pose order and their rows in SMPL-X (root, 21 body, jaw, eyes, 15 per hand)
POSE_KEYS = ("root_pose", "body_pose", "jaw_pose", "leye_pose", "reye_pose", "lhand_pose", "rhand_pose")
POSE_ROWS = (1, 21, 1, 1, 1, 15, 15)
WARMUP_SCALE_MAX = 0.001  # model.py:94


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


class _DecodePose(torch.autograd.Function):
    @staticmethod
    def forward(ctx, *params):
        lib = L.load()
        dev = params[0].device
        rows = [p.detach().reshape(-1, 6).contiguous() for p in params]
        st = L.B2RSmplxPose()
        for k, r in enumerate(rows):
            st.param[k], st.rows[k] = _ptr(r), r.shape[0]
        full = torch.empty((sum(POSE_ROWS), 3), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.b2r_decode_pose_forward(C.byref(st), _ptr(full), _stream(dev)), "b2r_decode_pose_forward")
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
        lib = L.load()
        st, gs = L.B2RSmplxPose(), L.B2RSmplxPoseGrads()
        grads = [torch.empty_like(r) for r in rows]
        for k, (r, g) in enumerate(zip(rows, grads)):
            st.param[k], st.rows[k], gs.param[k] = _ptr(r), r.shape[0], _ptr(g)
        up = g_full.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            L.check(lib.b2r_decode_pose_backward(C.byref(st), _ptr(up), C.byref(gs), _stream(dev)),
                    "b2r_decode_pose_backward")
        return tuple(g.reshape(s) for g, s in zip(grads, ctx.shapes))


def _check_cuda(fn, name, t, dev):
    if not isinstance(t, torch.Tensor) or not t.is_cuda or (dev is not None and t.device != dev):
        raise RuntimeError(f"{fn}: `{name}` must be a CUDA tensor on {dev}; there is no CPU path")
    if t.dtype != torch.float32:
        raise ValueError(f"{fn}: `{name}` must be float32, got {t.dtype}")


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
        _check_cuda("decode_smplx_pose", k, p, dev)
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
        lib = L.load()
        dev = ha.device
        P = ha.P
        g4, gs = _rows4(geo.detach())
        o4, os_ = _rows4(geo_offset.detach())
        ins = [t.detach().contiguous() for t in (mesh, pose_offset, expr_offset)]
        st = L.B2RHumanAssets(P=P, warmup=int(warmup), geo_stride=gs, geo_offset_stride=os_)
        st.mesh, st.pose_offset, st.expr_offset = (_ptr(t) for t in ins)
        st.geo, st.geo_offset, st.mask = _ptr(g4), _ptr(o4), _ptr(ha.mask)
        outs = [torch.empty((P, 3), dtype=torch.float32, device=dev) for _ in range(7 if warmup else 5)]
        ptrs = [_ptr(o) for o in outs] + [None, None] * (not warmup)
        with torch.cuda.device(dev):
            L.check(lib.b2r_human_geometry_forward(C.byref(st), *ptrs, _stream(dev)), "b2r_human_geometry_forward")
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(*ins, g4, o4)
        ctx.meta = (ha, st, geo.shape, geo_offset.shape)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        mesh, pose_offset, expr_offset, g4, o4 = ctx.saved_tensors
        ha, st, geo_shape, off_shape = ctx.meta
        dev = ha.device
        lib = L.load()
        up = [None if g is None else g.to(torch.float32).contiguous() for g in grads]
        up += [None] * (7 - len(up))
        f = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)  # noqa: E731
        d_mesh, d_expr, d_geo, d_off = f(ha.P, 3), f(ha.P, 3), f(ha.P, 4), f(ha.P, 4)
        gs = L.B2RHumanAssetsGrads(*[_ptr(x) for x in (*up, d_mesh, d_expr, d_geo, d_off)])
        with torch.cuda.device(dev):
            L.check(lib.b2r_human_geometry_backward(C.byref(st), C.byref(gs), _stream(dev)),
                    "b2r_human_geometry_backward")
        return None, None, d_mesh, None, d_expr, d_geo.reshape(geo_shape), d_off.reshape(off_shape)


class _Colors(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rgb, rgb_offset):
        lib = L.load()
        dev = rgb.device
        x, o = rgb.detach().contiguous(), rgb_offset.detach().contiguous()
        P = x.shape[0]
        out, out_r = torch.empty_like(x), torch.empty_like(x)
        with torch.cuda.device(dev):
            L.check(lib.b2r_human_colors_forward(P, _ptr(x), _ptr(o), _ptr(out), _ptr(out_r), _stream(dev)),
                    "b2r_human_colors_forward")
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(x, o)
        return out, out_r

    @staticmethod
    def backward(ctx, g, g_r):
        x, o = ctx.saved_tensors
        dev = x.device
        lib = L.load()
        g, g_r = (None if t is None else t.to(torch.float32).contiguous() for t in (g, g_r))
        d_rgb, d_off = torch.empty_like(x), torch.empty_like(x)
        with torch.cuda.device(dev):
            L.check(lib.b2r_human_colors_backward(x.shape[0], _ptr(x), _ptr(o), _ptr(g), _ptr(g_r), _ptr(d_rgb),
                                                  _ptr(d_off), _stream(dev)), "b2r_human_colors_backward")
        return d_rgb, d_off


class HumanAssets:
    """HumanGaussian's per-Gaussian tables for the two ops, built once (may synchronise): the hand / face mask
    (is_rhand | is_lhand | is_face_expr, module.py:489) as float 0 / 1, the constant identity `rotation` (P,4) and the
    unit `opacity` (P,1) of module.py:564-565.  `device` is where they live (CUDA)."""

    def __init__(self, is_rhand, is_lhand, is_face_expr, device=None):
        device = torch.device(device if device is not None else "cuda")
        if device.type != "cuda":
            raise RuntimeError(f"HumanAssets: device must be CUDA (got {device}); there is no CPU path")
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
            _check_cuda("HumanAssets.geometry", name, t, dev)
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
            _check_cuda("HumanAssets.colors", name, t, self.device)
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
