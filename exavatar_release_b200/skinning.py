"""`skin_gaussians` -- ExAvatar's linear-blend skinning of both human Gaussian sets as one differentiable CUDA op.

`HumanGaussian.forward` poses `mean_3d` and `mean_3d_refined` with the same rig (avatar/common/nets/module.py:549-557):

    transform_mat_vertex = get_transform_mat_vertex(skinning_weight[nn_vertex_idxs], joint_mats)  # (P,55)x(55,16)
    mean_3d = lbs(mean_3d, transform_mat_vertex, trans)                                           # bmm + trans
    mean_3d = torch.matmul(torch.inverse(cam_R), (mean_3d - cam_t).permute(1, 0)).permute(1, 0)
    ... the same two lines again for mean_3d_refined

The posed positions feed the mesh normals and the colour network before anything is rendered, and face_mesh_renderer
reads them with gradient (avatar/main/model.py:172-173), so the skinning cannot live inside the render that consumes
those colours.  `skin_gaussians` replaces those lines: one kernel blends M_i = sum_j W[rows[i], j] A_j per Gaussian
(reading the (V,J) weight table through the row index, without the (P,55) gather) and applies it to both sets; the
backward recomputes M and reduces the joint-transform gradient deterministically (include/b200raster.h B2RSkin).

`rasterizer.SkinnedGaussianRasterizer` is this op followed by one render.  CUDA tensors only: there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from . import _lib as L
from .camera import _inv3


def _f32(t: torch.Tensor) -> torch.Tensor:
    """A contiguous float32 view or copy: the op converts other dtypes (`skin_gaussians` has checked the device)."""
    return t.to(torch.float32).contiguous()


def _skin_struct(P, weights, rows, joint_mats, trans, Rinv, t, xyz, xyz_r, posed, posed_r) -> L.B2RSkin:
    s = L.B2RSkin()
    s.P, s.J, s.V = P, int(weights.shape[1]), int(weights.shape[0])
    s.weights, s.rows, s.joint_mats, s.trans = L.ptr(weights), L.ptr(rows), L.ptr(joint_mats), L.ptr(trans)
    s.cam_Rinv, s.cam_t = L.ptr(Rinv), L.ptr(t)
    s.xyz[0], s.xyz[1] = L.ptr(xyz), L.ptr(xyz_r)
    s.posed[0], s.posed[1] = L.ptr(posed), L.ptr(posed_r)
    return s


class _SkinGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, xyz_refined, weights, rows, joint_mats, trans, cam_R, cam_t):
        dev = xyz.device
        P = int(xyz.shape[0])
        x0 = _f32(xyz)
        x1 = None if xyz_refined is None else _f32(xyz_refined)
        W = _f32(weights)
        r = None if rows is None else rows.reshape(-1).to(torch.int32).contiguous()
        A = _f32(joint_mats).reshape(-1, 16)
        tr = _f32(trans).reshape(3)
        Rinv = t = None
        if cam_R is not None:
            Rinv = _f32(_inv3(_f32(cam_R)))  # cofactors: no torch.inverse, no sync
            t = _f32(cam_t).reshape(3)
        posed = torch.empty((P, 3), dtype=torch.float32, device=dev)
        posed_r = None if x1 is None else torch.empty((P, 3), dtype=torch.float32, device=dev)
        s = _skin_struct(P, W, r, A, tr, Rinv, t, x0, x1, posed, posed_r)
        L.run("b2r_skin_forward", dev, C.byref(s))
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(x0, x1, W, r, A, tr, Rinv, t)
        ctx.shapes = (joint_mats.shape, trans.shape, xyz.shape, None if xyz_refined is None else xyz_refined.shape)
        return (posed, posed_r) if x1 is not None else posed

    @staticmethod
    def backward(ctx, *grads):
        x0, x1, W, r, A, tr, Rinv, t = ctx.saved_tensors
        g0 = grads[0]
        g1 = grads[1] if x1 is not None else None
        need = ctx.needs_input_grad
        if (g0 is None and g1 is None) or not (need[0] or need[1] or need[4] or need[5]):
            return (None,) * 8
        lib = L.load()
        dev = x0.device
        P, J = int(x0.shape[0]), int(W.shape[1])
        f = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
        gp = [None if g is None else _f32(g).reshape(P, 3) for g in (g0, g1)]
        d_xyz = [f(P, 3) if need[0] else None, f(P, 3) if (need[1] and x1 is not None) else None]
        d12 = f(J, 12) if (need[4] or need[5]) else None
        d_trans = f(3) if (need[4] or need[5]) else None
        sbytes = lib.b2r_skin_scratch_bytes(P, J)
        scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev) if d12 is not None else None
        s = _skin_struct(P, W, r, A, tr, Rinv, t, x0, x1, None, None)
        dposed = (C.c_void_p * 2)(L.ptr(gp[0]), L.ptr(gp[1]))
        dxyz = (C.c_void_p * 2)(L.ptr(d_xyz[0]), L.ptr(d_xyz[1]))
        L.run("b2r_skin_backward", dev, C.byref(s), dposed, dxyz, L.ptr(d12), L.ptr(d_trans), L.ptr(scratch),
              sbytes if scratch is not None else 0)
        js, ts, xs, xrs = ctx.shapes
        d_joint = None
        if need[4]:  # (J,4,4) with the last row zero, like the unfused ops' gradient
            d_joint = F.pad(d12.view(J, 3, 4), (0, 0, 0, 1)).reshape(js)
        return (None if d_xyz[0] is None else d_xyz[0].reshape(xs),
                None if d_xyz[1] is None else d_xyz[1].reshape(xrs),
                None, None, d_joint, d_trans.reshape(ts) if need[5] else None, None, None)


def skin_gaussians(xyz: torch.Tensor, xyz_refined: Optional[torch.Tensor], skinning_weight: torch.Tensor,
                   rows: Optional[torch.Tensor], joint_mats: torch.Tensor, trans: torch.Tensor,
                   cam_R: Optional[torch.Tensor] = None, cam_t: Optional[torch.Tensor] = None
                   ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Poses one or two (P,3) canonical Gaussian sets with one rig; returns (posed, posed_refined).

    xyz, xyz_refined  (P,3) canonical positions (`mean_3d`, `mean_3d_refined`); xyz_refined=None poses one set and
                      returns None in its place.
    skinning_weight   (V,J) weight table (`smplx_layer.skinning_weight` resampled to the Gaussians, J <= 64).
    rows              (P) integer row of the table per Gaussian (`nn_vertex_idxs`), or None for row i.
    joint_mats        (J,4,4) joint transforms; trans (3) root translation.
    cam_R, cam_t      (3,3), (3): camera->world after posing, world = R^-1 (posed - t); None stays in the posed frame.

    Gradients reach xyz, xyz_refined, joint_mats (rows [:, :3, :]; the last row gets zero) and trans.  Weights, rows
    and the camera get None: in ExAvatar they are registered buffers and data, not parameters.  Forward and backward
    are free of host synchronisation (R^-1 by cofactors, not torch.inverse), so a frame can be captured in a CUDA graph.
    """
    for name, v in (("xyz", xyz), ("xyz_refined", xyz_refined), ("skinning_weight", skinning_weight), ("rows", rows),
                    ("joint_mats", joint_mats), ("trans", trans), ("cam_R", cam_R), ("cam_t", cam_t)):
        if v is not None:
            L.cuda("skin_gaussians", name, v)
    if xyz.dim() != 2 or xyz.shape[1] != 3:
        raise ValueError(f"skin_gaussians: xyz must be (P,3), got {tuple(xyz.shape)}")
    P = xyz.shape[0]
    if xyz_refined is not None and tuple(xyz_refined.shape) != tuple(xyz.shape):
        raise ValueError(f"skin_gaussians: xyz_refined {tuple(xyz_refined.shape)} must match xyz {tuple(xyz.shape)}")
    if skinning_weight.dim() != 2:
        raise ValueError(f"skin_gaussians: skinning_weight must be (V,J), got {tuple(skinning_weight.shape)}")
    V, J = skinning_weight.shape
    if rows is None and V < P:
        raise ValueError(f"skin_gaussians: without `rows` the weight table needs one row per Gaussian ({V} < {P})")
    if rows is not None and rows.numel() != P:
        raise ValueError(f"skin_gaussians: rows has {rows.numel()} entries for {P} Gaussians")
    if joint_mats.numel() != 16 * J:
        raise ValueError(f"skin_gaussians: joint_mats must be ({J},4,4), got {tuple(joint_mats.shape)}")
    if (cam_R is None) != (cam_t is None):
        raise ValueError("skin_gaussians: cam_R and cam_t go together")
    out = _SkinGaussians.apply(xyz, xyz_refined, skinning_weight, rows, joint_mats, trans, cam_R, cam_t)
    return (out[0], out[1]) if xyz_refined is not None else (out, None)
