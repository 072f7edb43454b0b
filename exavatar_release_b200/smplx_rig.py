"""`SmplxRig` -- ExAvatar's SMPL-X rig as one differentiable CUDA op that never syncs the host.

Every frame, `HumanGaussian.forward` (avatar/common/nets/module.py:516-586) runs two full `smplx_layer` forwards (the
大 pose with identity information and the zero pose), subdivides the neutral mesh twice with pytorch3d (uploading the
face table each call), inverts the 大-pose rotations, walks two more kinematic chains in Python loops of 4x4 matmuls,
contracts the upsampled `pose_dirs` (a 977 MB fp32 table at P = 167 618) with the pose feature and broadcasts `expr`
over a (P,3,50) temporary.  `SmplxRig` builds the model's constant tables once and computes the same tensors in one
forward and one backward call (csrc/smplx_rig.cu), contracting the pose and expression offsets at the base vertex count
V before subdividing them (subdivision is linear, so the two routes agree in exact arithmetic; they differ in fp32
rounding only).

    rig = SmplxRig(**tables)                    # once, next to HumanGaussian
    out = rig(shape_param, joint_offset, cat_full_pose(smplx_param), smplx_param['expr'])
    out.mesh_neutral_pose, out.mesh_neutral_pose_wo_upsample, out.joint_mats, out.pose_offset, out.expr_offset,
    out.pose_6d

`smplx_rig_reference` restates those reference lines in torch (float64 or float32, ExAvatar's own route by default:
upsampled tables, Python FK loops, torch.inverse) for tests and measurements.

`rig.body_mesh(...)` is the frame's SMPL-X body mesh of `Model.get_smplx_outputs` (avatar/main/model.py:37-58, and
animate.py:81-82 without the camera) over the same tables, in one forward and one backward call; `smplx_body_reference`
restates it in torch.

    mesh = rig.body_mesh(shape_param, joint_offset, full_pose, expr, trans, cam_R, cam_t)   # (V,3)

pytorch3d's `axis_angle_to_matrix`, `matrix_to_axis_angle`, `matrix_to_rotation_6d` and `rotation_6d_to_matrix` (the
scene Gaussians' rotations, scene_assets.py) are restated here from
pytorch3d 0.7.5 (the quaternion route: axis_angle_to_quaternion with its small-angle branch |angle| < 1e-6, where
sin(angle/2)/angle is replaced by 0.5 - angle^2/48, then quaternion_to_matrix; matrix_to_quaternion with the
largest-denominator candidate and the 0.1 floor, then quaternion_to_axis_angle).  pytorch3d is not a dependency of
this project, so the restatement is not pinned against it by a test; the CUDA op's derivative of axis_angle_to_matrix
is pinned against torch autograd through this restatement.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import _lib as L
from .rasterizer import _ptr
from .synthetic import subdivide_edges

JMAX = 64       # joints: one thread per joint in the op's single-CTA kernels
COEFF_MAX = 128  # shape / expression coefficients: four per lane


# ----------------------------------------------------------------------------------------------------------------------
# pytorch3d 0.7.5 rotation conversions and smplx's batch_rodrigues / batch_rigid_transform, restated

def axis_angle_to_quaternion(axis_angle: torch.Tensor) -> torch.Tensor:
    angles = torch.norm(axis_angle, p=2, dim=-1, keepdim=True)
    half = angles * 0.5
    small = angles.abs() < 1e-6
    safe = torch.where(small, torch.ones_like(angles), angles)
    s = torch.where(small, 0.5 - angles * angles / 48, torch.sin(half) / safe)
    return torch.cat([torch.cos(half), axis_angle * s], dim=-1)


def quaternion_to_matrix(q: torch.Tensor) -> torch.Tensor:
    r, i, j, k = torch.unbind(q, -1)
    two_s = 2.0 / (q * q).sum(-1)
    o = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return o.reshape(q.shape[:-1] + (3, 3))


def axis_angle_to_matrix(axis_angle: torch.Tensor) -> torch.Tensor:
    return quaternion_to_matrix(axis_angle_to_quaternion(axis_angle))


def _sqrt_positive_part(x: torch.Tensor) -> torch.Tensor:
    ret = torch.zeros_like(x)
    pos = x > 0
    ret[pos] = torch.sqrt(x[pos])
    return ret


def matrix_to_quaternion(m: torch.Tensor) -> torch.Tensor:
    batch = m.shape[:-2]
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = torch.unbind(m.reshape(batch + (9,)), -1)
    q_abs = _sqrt_positive_part(torch.stack([1.0 + m00 + m11 + m22, 1.0 + m00 - m11 - m22, 1.0 - m00 + m11 - m22,
                                             1.0 - m00 - m11 + m22], -1))
    cand = torch.stack([torch.stack([q_abs[..., 0] ** 2, m21 - m12, m02 - m20, m10 - m01], -1),
                        torch.stack([m21 - m12, q_abs[..., 1] ** 2, m10 + m01, m02 + m20], -1),
                        torch.stack([m02 - m20, m10 + m01, q_abs[..., 2] ** 2, m12 + m21], -1),
                        torch.stack([m10 - m01, m20 + m02, m21 + m12, q_abs[..., 3] ** 2], -1)], -2)
    floor = torch.tensor(0.1, dtype=q_abs.dtype, device=q_abs.device)
    cand = cand / (2.0 * q_abs[..., None].max(floor))
    pick = torch.nn.functional.one_hot(q_abs.argmax(-1), num_classes=4) > 0.5
    q = cand[pick, :].reshape(batch + (4,))
    return torch.where(q[..., 0:1] < 0, -q, q)


def quaternion_to_axis_angle(q: torch.Tensor) -> torch.Tensor:
    norms = torch.norm(q[..., 1:], p=2, dim=-1, keepdim=True)
    half = torch.atan2(norms, q[..., :1])
    angles = 2 * half
    small = angles.abs() < 1e-6
    safe = torch.where(small, torch.ones_like(angles), angles)
    s = torch.where(small, 0.5 - angles * angles / 48, torch.sin(half) / safe)
    return q[..., 1:] / s


def matrix_to_axis_angle(m: torch.Tensor) -> torch.Tensor:
    return quaternion_to_axis_angle(matrix_to_quaternion(m))


def matrix_to_rotation_6d(m: torch.Tensor) -> torch.Tensor:
    return m[..., :2, :].clone().reshape(m.shape[:-2] + (6,))


def rotation_6d_to_matrix(d6: torch.Tensor) -> torch.Tensor:
    """Gram-Schmidt on the two 3-vectors of `d6`; the three orthonormal vectors are the matrix's ROWS."""
    a1, a2 = d6[..., :3], d6[..., 3:]
    b1 = torch.nn.functional.normalize(a1, dim=-1)
    b2 = a2 - (b1 * a2).sum(-1, keepdim=True) * b1
    b2 = torch.nn.functional.normalize(b2, dim=-1)
    b3 = torch.cross(b1, b2, dim=-1)
    return torch.stack((b1, b2, b3), dim=-2)


def batch_rodrigues(rot_vecs: torch.Tensor) -> torch.Tensor:
    """smplx lbs.batch_rodrigues: angle = |v + 1e-8|, I + sin K + (1 - cos) K^2."""
    angle = torch.norm(rot_vecs + 1e-8, dim=1, keepdim=True)
    d = rot_vecs / angle
    cos, sin = torch.cos(angle)[:, :, None], torch.sin(angle)[:, :, None]
    z = torch.zeros_like(d[:, :1])
    K = torch.cat([z, -d[:, 2:3], d[:, 1:2], d[:, 2:3], z, -d[:, 0:1], -d[:, 1:2], d[:, 0:1], z], 1).view(-1, 3, 3)
    eye = torch.eye(3, dtype=rot_vecs.dtype, device=rot_vecs.device)[None]
    return eye + sin * K + (1 - cos) * torch.bmm(K, K)


def rigid_transform(rot: torch.Tensor, joints: torch.Tensor, parents):
    """smplx lbs.batch_rigid_transform for one body: (J,3,3) rotations, (J,3) joints -> posed joints (J,3) and the rel
    transforms (J,4,4), by the same Python loop of 4x4 matmuls."""
    par = [int(p) for p in parents]
    rel = joints.clone()
    rel[1:] = joints[1:] - joints[par[1:]]
    Jn = rot.shape[0]
    bottom = torch.zeros((Jn, 1, 4), dtype=rot.dtype, device=rot.device)
    bottom[:, 0, 3] = 1
    T = torch.cat([torch.cat([rot, rel[:, :, None]], 2), bottom], 1)
    chain = [T[0]]
    for i in range(1, Jn):
        chain.append(chain[par[i]] @ T[i])
    G = torch.stack(chain)
    posed = G[:, :3, 3]
    jh = torch.cat([joints, torch.zeros_like(joints[:, :1])], 1)[:, :, None]
    return posed, G - torch.nn.functional.pad(G @ jh, [3, 0])


# ----------------------------------------------------------------------------------------------------------------------
# Two-level midpoint subdivision (smpl_x.upsample_mesh)

def subdivision_tables(faces, num_vertices: int):
    """The two levels of smpl_x's SubdivideMeshes: sub1 (V1-V,2) and sub2 (P-V1,2), the endpoints of the edge each new
    vertex halves (sorted unique edges, base vertices first), and V1, P."""
    f = np.asarray(faces, dtype=np.int64)
    sub1, f1 = subdivide_edges(f, num_vertices)
    V1 = num_vertices + len(sub1)
    sub2, _ = subdivide_edges(f1, V1)
    return sub1, sub2, V1, V1 + len(sub2)


def upsample(x: torch.Tensor, sub1, sub2) -> torch.Tensor:
    """(V,k) rows -> (P,k): each new row the mean of its edge's two rows, level by level (pytorch3d's feats path)."""
    s1, s2 = (torch.as_tensor(s, device=x.device) for s in (sub1, sub2))
    x1 = torch.cat([x, (x[s1[:, 0]] + x[s1[:, 1]]) * 0.5])
    return torch.cat([x1, (x1[s2[:, 0]] + x1[s2[:, 1]]) * 0.5])


def _upsample_transpose(sub1, sub2, V: int, V1: int, P: int):
    """The composed (P,V) subdivision matrix transposed as a CSR over V: offsets (V+1), rows ascending, weights."""
    c1 = np.concatenate([np.stack([np.arange(V)] * 2, 1), sub1])
    w1 = np.concatenate([np.tile([1.0, 0.0], (V, 1)), np.full((len(sub1), 2), 0.5)])
    c2 = np.concatenate([np.stack([np.arange(V1)] * 2, 1), sub2])
    w2 = np.concatenate([np.tile([1.0, 0.0], (V1, 1)), np.full((len(sub2), 2), 0.5)])
    rows = np.repeat(np.arange(P), 4)
    cols = c1[c2].reshape(-1)  # (p, a, b) -> c1[c2[p, a], b]
    w = (w2[:, :, None] * w1[c2]).reshape(-1)
    keep = w != 0
    key = cols[keep].astype(np.int64) * P + rows[keep]
    uk, inv = np.unique(key, return_inverse=True)
    ws = np.zeros(len(uk))
    np.add.at(ws, inv, w[keep])  # dyadic weights: exact
    col, row = uk // P, uk % P
    offs = np.zeros(V + 1, dtype=np.int64)
    offs[1:] = np.cumsum(np.bincount(col, minlength=V))
    return offs, row, ws


# ----------------------------------------------------------------------------------------------------------------------

class RigOutputs(NamedTuple):
    mesh_neutral_pose: torch.Tensor              # (P,3)  gradient to shape_param, joint_offset
    mesh_neutral_pose_wo_upsample: torch.Tensor  # (V,3)  no gradient (nearest_rows' targets)
    joint_mats: torch.Tensor                     # (J,4,4) gradient to full_pose, shape_param, joint_offset
    pose_offset: torch.Tensor                    # (P,3)  smplx_pose_offset * mask; no gradient (the pose is detached)
    expr_offset: torch.Tensor                    # (P,3)  gradient to expr
    pose_6d: torch.Tensor                        # (6 n_body,) no gradient (detached)


def cat_full_pose(smplx_param: dict) -> torch.Tensor:
    """ExAvatar's (J,3) axis-angle pose in the model's joint order (module.py:404)."""
    return torch.cat([smplx_param[k].reshape(-1, 3) for k in ("root_pose", "body_pose", "jaw_pose", "leye_pose",
                                                               "reye_pose", "lhand_pose", "rhand_pose")])


def _t(x, dtype=torch.float64) -> torch.Tensor:
    return torch.as_tensor(np.asarray(x.detach().cpu()) if isinstance(x, torch.Tensor) else np.asarray(x)).to(dtype)


class _Rig(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rig, shape_param, joint_offset, full_pose, expr):
        lib = L.load()
        dev = rig.device
        ins = [rig._input(t, n, name) for t, n, name in ((shape_param, rig.NB, "shape_param"),
                                                          (joint_offset, 3 * rig.J, "joint_offset"),
                                                          (full_pose, 3 * rig.J, "full_pose"),
                                                          (expr, rig.NE, "expr"))]
        f = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)  # noqa: E731
        outs = [f(rig.P, 3), f(rig.V, 3), f(rig.J, 4, 4), f(rig.P, 3), f(rig.P, 3), f(6 * rig.n_body)]
        scratch = torch.empty(rig.scratch_bytes, dtype=torch.uint8, device=dev)
        st = rig._struct(ins)
        with torch.cuda.device(dev):
            L.check(lib.b2r_rig_forward(C.byref(st), *[_ptr(o) for o in outs], _ptr(scratch), rig.scratch_bytes,
                                        torch.cuda.current_stream(dev).cuda_stream), "b2r_rig_forward")
        ctx.rig = rig
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(outs[1], outs[3], outs[5])
        ctx.save_for_backward(*ins, scratch)
        ctx.shapes = (shape_param.shape, joint_offset.shape, full_pose.shape, expr.shape)
        return tuple(outs)

    @staticmethod
    def backward(ctx, g_mesh, g_wo, g_jm, g_po, g_eo, g_6d):
        *ins, scratch = ctx.saved_tensors
        rig = ctx.rig
        dev = rig.device
        lib = L.load()
        grads = [torch.empty(n, dtype=torch.float32, device=dev) for n in (rig.NB, 3 * rig.J, 3 * rig.J, rig.NE)]
        gs = L.B2RRigGrads(*[_ptr(g) for g in grads])
        up = [None if g is None else g.to(torch.float32).contiguous() for g in (g_mesh, g_jm, g_eo)]
        st = rig._struct(ins)
        with torch.cuda.device(dev):
            L.check(lib.b2r_rig_backward(C.byref(st), *[_ptr(g) for g in up], C.byref(gs), _ptr(scratch),
                                         scratch.numel(), torch.cuda.current_stream(dev).cuda_stream),
                    "b2r_rig_backward")
        return (None, *[g.reshape(s) for g, s in zip(grads, ctx.shapes)])


class _Body(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rig, shape_param, joint_offset, full_pose, expr, trans, cam_R, cam_t):
        lib = L.load()
        dev = rig.device
        ins = [rig._input(t, n, name) for t, n, name in ((shape_param, rig.NB, "shape_param"),
                                                          (joint_offset, 3 * rig.J, "joint_offset"),
                                                          (full_pose, 3 * rig.J, "full_pose"),
                                                          (expr, rig.NE, "expr"), (trans, 3, "trans"))]
        if (cam_R is None) != (cam_t is None):
            raise ValueError("SmplxRig.body_mesh: give both cam_R and cam_t, or neither")
        cam = [] if cam_R is None else [rig._input(cam_R, 9, "cam_R"), rig._input(cam_t, 3, "cam_t")]
        mesh = torch.empty((rig.V, 3), dtype=torch.float32, device=dev)
        scratch = torch.empty(rig.body_scratch_bytes, dtype=torch.uint8, device=dev)
        st = rig._body_struct(ins, cam)
        with torch.cuda.device(dev):
            L.check(lib.b2r_smplx_body_forward(C.byref(st), _ptr(mesh), _ptr(scratch), rig.body_scratch_bytes,
                                               torch.cuda.current_stream(dev).cuda_stream), "b2r_smplx_body_forward")
        ctx.rig = rig
        ctx.n_cam = len(cam)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(*ins, *cam, scratch)
        ctx.shapes = (shape_param.shape, joint_offset.shape, full_pose.shape, expr.shape, trans.shape)
        return mesh

    @staticmethod
    def backward(ctx, g_mesh):
        *ins, scratch = ctx.saved_tensors
        ins, cam = ins[:5], ins[5:]
        rig = ctx.rig
        dev = rig.device
        lib = L.load()
        grads = [torch.empty(n, dtype=torch.float32, device=dev) for n in (rig.NB, 3 * rig.J, 3 * rig.J, rig.NE, 3)]
        gs = L.B2RSmplxBodyGrads(*[_ptr(g) for g in grads])
        up = None if g_mesh is None else g_mesh.to(torch.float32).contiguous()
        st = rig._body_struct(ins, cam)
        with torch.cuda.device(dev):
            L.check(lib.b2r_smplx_body_backward(C.byref(st), _ptr(up), C.byref(gs), _ptr(scratch), scratch.numel(),
                                                torch.cuda.current_stream(dev).cuda_stream), "b2r_smplx_body_backward")
        return (None, *[g.reshape(s) for g, s in zip(grads, ctx.shapes)], None, None)


class SmplxRig:
    """ExAvatar's SMPL-X rig (module.py:517-518, 533, 537, 549) as one sync-free CUDA op.

    From `smplx_layer`: v_template (V,3), shapedirs (V,3,NB) (the shape columns), expr_dirs (V,3,NE) after the FLAME
    override, posedirs (9 (J-1), 3V), J_regressor (J,V), parents (J,), lbs_weights (V,J), pose_mean (3J).  From
    `smpl_x`: face_offset (V,3), faces (F0,3) the base faces with the cavity faces (`smpl_x.face`), neutral_body_pose
    (n_body,3).  The (P,) masks is_rhand, is_lhand, is_face_expr of HumanGaussian.  `device` is where the tables live.

    Construction (may synchronise) builds, once: the two-level subdivision and its transpose, J_regressor as a per-joint
    CSR and its per-vertex transpose, the 大-pose rotations batch_rodrigues(full_pose + pose_mean) with the jaw at zero,
    the zero-pose rotations batch_rodrigues(pose_mean), the inverse-neutral rotations of module.py:361-366 (through the
    restated pytorch3d conversions), and the 大 pose's constant pose-corrective offsets (V,3), all in float64.

    A call takes shape_param (NB), joint_offset (J,3) before get_joint_offset (the op zeroes the root), full_pose (J,3)
    axis-angle in the model's order (`cat_full_pose`) and expr (NE), float32 CUDA tensors, and returns `RigOutputs`.
    Divergence from the reference: the pose and expression offsets are contracted at V and then subdivided (ExAvatar
    subdivides the tables and contracts at P); the joints and the four chains run in fp64.

    `body_mesh` is the frame's body mesh of get_smplx_outputs over the same tables (its own scratch per call).
    """

    def __init__(self, *, v_template, shapedirs, expr_dirs, posedirs, J_regressor, parents, lbs_weights, pose_mean,
                 face_offset, faces, neutral_body_pose, is_rhand, is_lhand, is_face_expr, device=None):
        device = torch.device(device if device is not None else "cuda")
        if device.type != "cuda":
            raise RuntimeError(f"SmplxRig: device must be CUDA (got {device}); there is no CPU path")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = device
        self.model = m = validate_model(v_template=v_template, shapedirs=shapedirs, expr_dirs=expr_dirs,
                                        posedirs=posedirs, J_regressor=J_regressor, parents=parents,
                                        lbs_weights=lbs_weights, pose_mean=pose_mean, face_offset=face_offset,
                                        faces=faces, neutral_body_pose=neutral_body_pose, is_rhand=is_rhand,
                                        is_lhand=is_lhand, is_face_expr=is_face_expr)
        self.V, self.V1, self.P, self.J = m["V"], m["V1"], m["P"], m["J"]
        self.NB, self.NE, self.n_body = m["NB"], m["NE"], m["n_body"]
        V, J = self.V, self.J
        dev = lambda t, dt: torch.as_tensor(t).to(device=device, dtype=dt).contiguous()  # noqa: E731
        self.template = dev(m["v_template"].float() + m["face_offset"].float(), torch.float32)  # one fp32 add
        self.shapedirs = dev(m["shapedirs"], torch.float32)
        self.expr_dirs = dev(m["expr_dirs"], torch.float32)
        self.posedirs_t = dev(m["posedirs"].reshape(-1, V, 3).permute(1, 2, 0), torch.float32)
        self.pose_offset0 = dev(m["pose_offset0"], torch.float32)
        self.lbs_weights = dev(m["lbs_weights"], torch.float32)
        jr = m["J_regressor"].numpy()
        rows, cols = np.nonzero(jr)  # row-major: per joint, vertices ascending
        self.jreg_offsets = dev(np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=J))]), torch.int32)
        self.jreg_cols = dev(cols, torch.int32)
        self.jreg_vals = dev(jr[rows, cols], torch.float32)
        tc, tr = np.nonzero(jr.T)    # per vertex, joints ascending
        self.jregT_offsets = dev(np.concatenate([[0], np.cumsum(np.bincount(tc, minlength=V))]), torch.int32)
        self.jregT_rows = dev(tr, torch.int32)
        self.jregT_vals = dev(jr.T[tc, tr], torch.float32)
        self.parents = dev(m["parents"], torch.int32)
        self.rot_neutral = dev(m["rot_neutral"].reshape(J, 9), torch.float64)
        self.rot_zero = dev(m["rot_zero"].reshape(J, 9), torch.float64)
        self.rot_inv = dev(m["rot_inv"].reshape(J, 9), torch.float64)
        self.sub1 = dev(m["sub1"], torch.int32)
        self.sub2 = dev(m["sub2"], torch.int32)
        offs, row, w = _upsample_transpose(m["sub1"], m["sub2"], V, self.V1, self.P)
        self.upT_offsets, self.upT_rows, self.upT_w = (dev(offs, torch.int32), dev(row, torch.int32),
                                                       dev(w, torch.float32))
        self.mask = dev(m["mask"], torch.uint8)
        self.pose_mean = dev(m["pose_mean"], torch.float32)  # body_mesh only
        self.scratch_bytes = int(L.load().b2r_rig_scratch_bytes(V, J, self.NB, self.NE))
        self.body_scratch_bytes = int(L.load().b2r_smplx_body_scratch_bytes(V, J))
        self._template = L.B2RRig(
            V=V, V1=self.V1, P=self.P, J=J, NB=self.NB, NE=self.NE, n_body=self.n_body,
            **{k: _ptr(getattr(self, a)) for k, a in (
                ("template_", "template"), ("shapedirs", "shapedirs"), ("expr_dirs", "expr_dirs"),
                ("posedirs_t", "posedirs_t"), ("pose_offset0", "pose_offset0"), ("lbs_weights", "lbs_weights"),
                ("jreg_offsets", "jreg_offsets"), ("jreg_cols", "jreg_cols"), ("jreg_vals", "jreg_vals"),
                ("jregT_offsets", "jregT_offsets"), ("jregT_rows", "jregT_rows"), ("jregT_vals", "jregT_vals"),
                ("parents", "parents"), ("rot_neutral", "rot_neutral"), ("rot_zero", "rot_zero"),
                ("rot_inv", "rot_inv"), ("sub1", "sub1"), ("sub2", "sub2"), ("upT_offsets", "upT_offsets"),
                ("upT_rows", "upT_rows"), ("upT_w", "upT_w"), ("mask", "mask"))})

    def _input(self, t: torch.Tensor, n: int, name: str) -> torch.Tensor:
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != self.device:
            raise RuntimeError(f"SmplxRig: `{name}` must be a CUDA tensor on {self.device}; there is no CPU path")
        if t.dtype != torch.float32 or t.numel() != n:
            raise ValueError(f"SmplxRig: `{name}` must be float32 with {n} elements, got {t.dtype} {tuple(t.shape)}")
        return t.detach().reshape(n).contiguous()

    def _struct(self, ins) -> "L.B2RRig":
        st = L.B2RRig.from_buffer_copy(self._template)
        st.shape_param, st.joint_offset, st.full_pose, st.expr = (_ptr(t) for t in ins)
        return st

    def __call__(self, shape_param, joint_offset, full_pose, expr) -> RigOutputs:
        return RigOutputs(*_Rig.apply(self, shape_param, joint_offset, full_pose, expr))

    def reference(self, *args, **kw) -> RigOutputs:
        """smplx_rig_reference with this rig's model."""
        return smplx_rig_reference(self.model, *args, **kw)

    def _body_struct(self, ins, cam) -> "L.B2RSmplxBody":
        st = L.B2RSmplxBody(rig=self._template, pose_mean=_ptr(self.pose_mean))
        st.shape_param, st.joint_offset, st.full_pose, st.expr, st.trans = (_ptr(t) for t in ins)
        if cam:
            st.cam_R, st.cam_t = (_ptr(t) for t in cam)
        return st

    def body_mesh(self, shape_param, joint_offset, full_pose, expr, trans, cam_R=None, cam_t=None) -> torch.Tensor:
        """The frame's SMPL-X body mesh (V,3) float32: ExAvatar's get_smplx_outputs (model.py:37-58), i.e. smplx's
        SMPLX.forward + lbs (body_models.py:1122-1300, lbs.py:155-250) with face_offset, the raw joint_offset and transl,
        then R^-1 (mesh - t) in world coordinates.  Without a camera the mesh stays in camera coordinates (animate.py).

        shape_param (NB), joint_offset (J,3) as given -- every row moves the joints, the root included (ExAvatar passes
        human_gaussian.joint_offset without get_joint_offset here) --, full_pose (J,3) in `cat_full_pose` order
        (`decode_smplx_pose(...)["full_pose"]` as is; the model's pose_mean is added), expr (NE), trans (3), and the
        optional cam_R (3,3) / cam_t (3): float32 CUDA tensors on the rig's device.  Gradients flow to the five inputs;
        the camera gets none.  The layer's landmarks, extra joints and `joints` output, which both callers discard, are
        not computed.  Divergence from the reference: v_shaped is (template + shapedirs . beta) + expr_dirs . expr in
        fp32 (smplx contracts the 150 coefficients in one einsum), the joints, rotations and chain run in fp64, and
        R^-1 is taken by cofactors instead of torch.inverse, so nothing synchronises the host."""
        return _Body.apply(self, shape_param, joint_offset, full_pose, expr, trans, cam_R, cam_t)


def validate_model(*, v_template, shapedirs, expr_dirs, posedirs, J_regressor, parents, lbs_weights, pose_mean,
                   face_offset, faces, neutral_body_pose, is_rhand, is_lhand, is_face_expr) -> dict:
    """Checks the model's tables on the host and returns them as float64 / int64 CPU tensors with the derived constants
    (subdivision tables, the three constant rotation sets, the 大 pose's corrective offsets, the offset mask)."""
    vt = _t(v_template).reshape(-1, 3)
    V = vt.shape[0]
    par = _t(parents, torch.int64).reshape(-1)
    J = par.numel()
    if not 2 <= J <= JMAX:
        raise ValueError(f"SmplxRig: {J} joints; the op takes 2 <= J <= {JMAX}")
    if int(par[0]) != -1 or any(not 0 <= int(par[i]) < i for i in range(1, J)):
        raise ValueError("SmplxRig: parents must be topological: parents[0] = -1 and 0 <= parents[i] < i")
    sd, ed = _t(shapedirs), _t(expr_dirs)
    if sd.dim() != 3 or sd.shape[:2] != (V, 3) or not 1 <= sd.shape[2] <= COEFF_MAX:
        raise ValueError(f"SmplxRig: shapedirs must be ({V},3,NB) with NB <= {COEFF_MAX}, got {tuple(sd.shape)}")
    if ed.dim() != 3 or ed.shape[:2] != (V, 3) or not 1 <= ed.shape[2] <= COEFF_MAX:
        raise ValueError(f"SmplxRig: expr_dirs must be ({V},3,NE) with NE <= {COEFF_MAX}, got {tuple(ed.shape)}")
    pd = _t(posedirs)
    if tuple(pd.shape) != (9 * (J - 1), 3 * V):
        raise ValueError(f"SmplxRig: posedirs must be ({9 * (J - 1)},{3 * V}), got {tuple(pd.shape)}")
    jr, W = _t(J_regressor), _t(lbs_weights)
    if tuple(jr.shape) != (J, V) or tuple(W.shape) != (V, J):
        raise ValueError(f"SmplxRig: J_regressor must be ({J},{V}) and lbs_weights ({V},{J})")
    pm = _t(pose_mean).reshape(-1)
    fo = _t(face_offset).reshape(-1, 3)
    if pm.numel() != 3 * J or fo.shape[0] != V:
        raise ValueError(f"SmplxRig: pose_mean must have {3 * J} entries and face_offset {V} rows")
    nbp = _t(neutral_body_pose).reshape(-1, 3)
    n_body = nbp.shape[0]
    if not 1 <= n_body <= J - 4:
        raise ValueError(f"SmplxRig: {n_body} body joints need 1 + n_body + 3 face joints <= J = {J}")
    f = np.asarray(faces.detach().cpu() if isinstance(faces, torch.Tensor) else faces, dtype=np.int64)
    if f.ndim != 2 or f.shape[1] != 3 or f.min() < 0 or f.max() >= V:
        raise ValueError(f"SmplxRig: faces must be (F,3) indices into {V} vertices")
    sub1, sub2, V1, P = subdivision_tables(f, V)
    masks = []
    for name, msk in (("is_rhand", is_rhand), ("is_lhand", is_lhand), ("is_face_expr", is_face_expr)):
        t = torch.as_tensor(msk).detach().cpu().reshape(-1)
        if t.numel() != P:
            raise ValueError(f"SmplxRig: `{name}` has {t.numel()} entries; the subdivided mesh has {P} vertices")
        masks.append(t != 0)
    # 大 pose with the jaw at zero (get_neutral_pose_human(jaw_zero_pose=True)); the zero pose; the inverse chain
    neutral = torch.zeros(J, 3, dtype=torch.float64)
    neutral[1:1 + n_body] = nbp
    rot_neutral = batch_rodrigues(neutral + pm.view(J, 3))
    rot_zero = batch_rodrigues(pm.view(J, 3))
    inv = torch.zeros(J, 3, dtype=torch.float64)
    inv[1:1 + n_body] = matrix_to_axis_angle(torch.inverse(axis_angle_to_matrix(nbp)))
    inv[1 + n_body] = matrix_to_axis_angle(torch.inverse(axis_angle_to_matrix(torch.zeros(1, 3, dtype=torch.float64))))[0]
    rot_inv = axis_angle_to_matrix(inv)
    eye = torch.eye(3, dtype=torch.float64)
    pose_offset0 = ((rot_neutral[1:] - eye).reshape(1, -1) @ pd).view(V, 3)
    return {"V": V, "V1": V1, "P": P, "J": J, "NB": sd.shape[2], "NE": ed.shape[2], "n_body": n_body,
            "v_template": vt, "face_offset": fo, "shapedirs": sd, "expr_dirs": ed, "posedirs": pd, "J_regressor": jr,
            "parents": par, "lbs_weights": W, "pose_mean": pm, "neutral_body_pose": nbp, "sub1": sub1, "sub2": sub2,
            "rot_neutral": rot_neutral, "rot_zero": rot_zero, "rot_inv": rot_inv, "pose_offset0": pose_offset0,
            "mask": masks[0] | masks[1] | masks[2]}


def smplx_rig_reference(model: dict, shape_param, joint_offset, full_pose, expr, *, dtype=torch.float64,
                        device=None, route: str = "upsample", cache: Optional[dict] = None) -> RigOutputs:
    """ExAvatar's rig lines restated in torch, differentiable in the four inputs.  `model` is validate_model's dict
    (SmplxRig.model).  route="upsample" is ExAvatar's: the base tables are subdivided to (P,3,9(J-1)) pose_dirs and
    (P,3,NE) expr_dirs and contracted there; route="contract" contracts at V and subdivides the result, as the op does.
    The constant rotation sets are the model's float64 ones, cast to `dtype`.  `cache` (a dict) keeps the upsampled
    tables between calls.  The product never calls this."""
    dev = torch.device(device) if device is not None else shape_param.device
    cv = lambda t: t.to(device=dev, dtype=dtype)  # noqa: E731
    V, J, P, n_body = model["V"], model["J"], model["P"], model["n_body"]
    par = model["parents"].tolist()
    beta, jo, pose, e = (cv(t).reshape(-1) for t in (shape_param, joint_offset, full_pose, expr))
    jo, pose = jo.view(J, 3), pose.view(J, 3)
    sub1, sub2 = model["sub1"], model["sub2"]
    tmpl = cv(model["v_template"]) + cv(model["face_offset"])
    vs = tmpl + torch.einsum("l,mkl->mk", beta, cv(model["shapedirs"]))
    w = torch.ones(J, 1, dtype=dtype, device=dev)
    w[0] = 0
    Jr = cv(model["J_regressor"]) @ vs + jo * w
    eye = torch.eye(3, dtype=dtype, device=dev)
    pd = cv(model["posedirs"])
    v_posed = vs + ((cv(model["rot_neutral"])[1:] - eye).reshape(1, -1) @ pd).view(V, 3)
    jnp, A_n = rigid_transform(cv(model["rot_neutral"]), Jr, par)
    T = (cv(model["lbs_weights"]) @ A_n.reshape(J, 16)).view(V, 4, 4)
    mesh_wo = (T @ torch.cat([v_posed, torch.ones_like(v_posed[:, :1])], 1)[:, :, None])[:, :3, 0]
    jzp, _ = rigid_transform(cv(model["rot_zero"]), Jr, par)
    _, A_inv = rigid_transform(cv(model["rot_inv"]), jnp, par)
    Rf = axis_angle_to_matrix(pose)
    _, A_f = rigid_transform(Rf, jzp, par)
    joint_mats = torch.bmm(A_f, A_inv)
    mesh = upsample(mesh_wo, sub1, sub2)
    feat = (Rf[1:] - eye).reshape(1, -1).detach()
    mask = model["mask"].to(dev)[:, None].to(dtype)
    ed = cv(model["expr_dirs"])
    if route == "upsample":
        key = (dtype, dev)
        tabs = cache.get(key) if cache is not None else None
        if tabs is None:
            pose_dirs = upsample(pd.t().reshape(V, -1), sub1, sub2).reshape(P * 3, -1).t()
            expr_dirs = upsample(ed.reshape(V, -1), sub1, sub2).view(P, 3, -1)
            tabs = (pose_dirs, expr_dirs)
            if cache is not None:
                cache[key] = tabs
        pose_dirs, expr_dirs = tabs
        pose_offset = (feat @ pose_dirs).view(P, 3) * mask
        expr_offset = (e[None, None, :] * expr_dirs).sum(2)
    elif route == "contract":
        pose_offset = upsample((feat @ pd).view(V, 3), sub1, sub2) * mask
        expr_offset = upsample(torch.einsum("n,vcn->vc", e, ed), sub1, sub2)
    else:
        raise ValueError(f"smplx_rig_reference: route must be 'upsample' or 'contract', got {route!r}")
    pose_6d = matrix_to_rotation_6d(Rf[1:1 + n_body]).reshape(-1).detach()
    return RigOutputs(mesh, mesh_wo.detach(), joint_mats, pose_offset, expr_offset, pose_6d)


def smplx_body_reference(model: dict, shape_param, joint_offset, full_pose, expr, trans, cam_R=None, cam_t=None, *,
                         dtype=torch.float64, device=None) -> torch.Tensor:
    """get_smplx_outputs (avatar/main/model.py:37-58) restated in torch, differentiable in the five inputs: smplx's
    SMPLX.forward + lbs for one frame with face_offset, the raw joint_offset and transl (body_models.py:1233 adds
    pose_mean; lbs.py:155-250 with smplx's batch_rodrigues and batch_rigid_transform), then torch.inverse(R) (mesh - t)
    when a camera is given.  `model` is validate_model's dict (SmplxRig.model); the tables are cast to `dtype`, so
    dtype=torch.float32 is ExAvatar's own fp32 route.  The product never calls this."""
    dev = torch.device(device) if device is not None else shape_param.device
    cv = lambda t: t.to(device=dev, dtype=dtype)  # noqa: E731
    V, J = model["V"], model["J"]
    beta, jo, pose, e, tr = (cv(t).reshape(-1) for t in (shape_param, joint_offset, full_pose, expr, trans))
    jo, pose = jo.view(J, 3), pose.view(J, 3)
    tmpl = cv(model["v_template"]) + cv(model["face_offset"])
    dirs = torch.cat([cv(model["shapedirs"]), cv(model["expr_dirs"])], dim=-1)
    v_shaped = tmpl + torch.einsum("l,mkl->mk", torch.cat([beta, e]), dirs)
    Jr = cv(model["J_regressor"]) @ v_shaped + jo
    rot = batch_rodrigues(pose + cv(model["pose_mean"]).view(J, 3))
    eye = torch.eye(3, dtype=dtype, device=dev)
    v_posed = v_shaped + ((rot[1:] - eye).reshape(1, -1) @ cv(model["posedirs"])).view(V, 3)
    _, A = rigid_transform(rot, Jr, model["parents"].tolist())
    T = (cv(model["lbs_weights"]) @ A.reshape(J, 16)).view(V, 4, 4)
    mesh = (T @ torch.cat([v_posed, torch.ones_like(v_posed[:, :1])], 1)[:, :, None])[:, :3, 0] + tr
    if cam_R is not None:
        mesh = torch.matmul(torch.inverse(cv(cam_R)), (mesh - cv(cam_t).view(1, 3)).permute(1, 0)).permute(1, 0)
    return mesh
