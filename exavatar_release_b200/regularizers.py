"""`HumanRegularizers` -- ExAvatar's per-frame human regularisers as one differentiable CUDA op that never syncs the host.

ExAvatar's regulariser block (avatar/main/model.py:217-257, with LaplacianReg, HandMeanReg, HandRGBReg, ArmRGBReg and
JointOffsetSymmetricReg of avatar/common/nets/loss.py:97-197 and smpl_x.get_arm) rebuilds five weight columns with
boolean-mask assignments, builds three pytorch3d `Meshes` (each uploading the 8 MB face table), selects rows with boolean
masks, reads two counts on the host and materialises dense lower-arm x upper-arm matrices twice.  Every one of those
synchronises the host.  `HumanRegularizers` builds the constant tables once and computes the ten terms in one forward
and one backward call (csrc/regularizers.cu): no sync, no upload, no allocation beyond the outputs and one scratch
buffer, capturable in a CUDA graph, and bit-identical from run to run.

    regs = HumanRegularizers(smpl_x.face_upsampled, smpl_x.vertex_num_upsampled, is_rhand=..., ..., sym_pairs=...)
    loss.update(regs(mesh_neutral_pose, mean_offset, mean_offset_offset, scale_offset, scale, scale_refined, rgb,
                     rgb_refined, joint_offset, scale_reg=scale_wo_clamp if cfg.is_warmup else None))

`human_regularizers_reference` restates the block in plain torch (float64 by default) for tests and measurements.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib as L
from .geometry import VertexNormals, vertex_normals_reference
from .rasterizer import _ptr

KEYS = ("gaussian_mean_reg", "gaussian_mean_hand_reg", "gaussian_scale_reg", "lap_mean", "lap_scale", "lap_rgb",
        "hand_rgb_reg", "arm_rgb_reg", "joint_offset_reg", "joint_offset_sym_reg")
NEIGHBOR_MAX = 10   # LaplacianReg.get_neighbor's neighbor_max_num
ARM_TOPK = 50       # ArmRGBReg's top_k cap
ARM_DIST_X = 0.01   # ArmRGBReg's dist_x_thr (compared against fp32 distances, so in effect 0.01f)


def laplacian_table(faces, num_vertices: int) -> Tuple[np.ndarray, np.ndarray]:
    """LaplacianReg.get_neighbor's table: the same set operations in the same order (so `list(adj[v])` iterates in the
    same order), the first 10 neighbours of that list, weights -1/n in float32, unused slots pointing at the vertex
    itself with weight 0.  Returns (idx (V,10) int64, w (V,10) float32)."""
    f = faces.tolist() if hasattr(faces, "tolist") else [list(r) for r in faces]
    adj = {i: set() for i in range(num_vertices)}
    for face in f:
        for idx in face:
            adj[idx] |= set(face) - set([idx])
    idx = np.tile(np.arange(num_vertices)[:, None], (1, NEIGHBOR_MAX))
    w = np.zeros((num_vertices, NEIGHBOR_MAX), dtype=np.float32)
    for v in range(num_vertices):
        n = min(len(adj[v]), NEIGHBOR_MAX)
        if n:
            idx[v, :n] = np.array(list(adj[v]))[:n]
            w[v, :n] = -1.0 / n
    return idx, w


def _mask(m, P: int, name: str) -> torch.Tensor:
    t = torch.as_tensor(m).detach().to("cpu").reshape(-1)
    if t.numel() != P:
        raise ValueError(f"HumanRegularizers: `{name}` must have {P} entries, got {t.numel()}")
    return t != 0


def weight_columns(P: int, is_rhand, is_lhand, is_face, is_face_expr, is_cavity) -> torch.Tensor:
    """The five per-vertex weight columns of model.py:217-247 (gaussian_mean_reg, gaussian_scale_reg, lap_mean, lap_scale,
    lap_rgb) as a (5,P) float32 CPU tensor, assigned in model.py's order: later assignments win."""
    r, l, f, e, c = (_mask(m, P, n) for m, n in ((is_rhand, "is_rhand"), (is_lhand, "is_lhand"), (is_face, "is_face"),
                                               (is_face_expr, "is_face_expr"), (is_cavity, "is_cavity")))
    w = torch.ones((5, P), dtype=torch.float32)
    w[0] *= 10
    w[0, r] = 1000
    w[0, l] = 1000
    w[0, f] = 1
    w[0, e] = 10
    w[1, r] = 1000
    w[1, l] = 1000
    w[1, e] = 10
    w[1, c] = 0
    w[2, e] = 50
    w[2, c] = 0.1
    w[3] *= 10
    w[3, r] = 10
    w[3, l] = 10
    w[3, e] = 0
    w[4] *= 0.1
    w[4, r] = 100
    w[4, l] = 100
    return w


def _rows(name: str, t: torch.Tensor, P: int, k: int) -> torch.Tensor:
    shape = tuple(t.shape)
    ok = shape in ((P, k), (1, P, k)) or (k == 1 and shape in ((P,), (1, P)))
    if not ok:
        raise ValueError(f"HumanRegularizers: `{name}` must be ({P},{k}) or (1,{P},{k}), got {shape}")
    if not t.is_cuda:
        raise RuntimeError(f"HumanRegularizers: `{name}` must be a CUDA tensor (got {t.device}); there is no CPU path")
    if t.dtype != torch.float32:
        raise ValueError(f"HumanRegularizers: `{name}` must be float32, got {t.dtype}")
    return t.detach().reshape(P * k).contiguous()


class _Regs(torch.autograd.Function):
    @staticmethod
    def forward(ctx, regs, mesh, mo, moo, so, s, sr, rgb, rgbr, jo, sreg):
        lib = L.load()
        P, dev = regs.num_vertices, regs.device
        ins = [_rows("mesh_neutral_pose", mesh, P, 3), _rows("mean_offset", mo, P, 3),
               _rows("mean_offset_offset", moo, P, 3), _rows("scale_offset", so, P, 1), _rows("scale", s, P, 3),
               _rows("scale_refined", sr, P, 3), _rows("rgb", rgb, P, 3), _rows("rgb_refined", rgbr, P, 3),
               _rows("joint_offset", jo, regs.num_joints, 3),
               None if sreg is None else _rows("scale_reg", sreg, P, 3)]
        if any(t is not None and t.device != dev for t in ins):
            raise ValueError(f"HumanRegularizers: every input must be on {dev}, where the tables live")
        st = regs._struct(ins)
        nbytes = regs.scratch_bytes
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty(len(KEYS), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.b2r_regs_forward(C.byref(st), _ptr(out), _ptr(scratch), nbytes,
                                         torch.cuda.current_stream(dev).cuda_stream), "b2r_regs_forward")
        ctx.regs = regs
        ctx.shapes = [t.shape for t in (mo, moo, so, s, sr, rgb, rgbr, jo)] + [None if sreg is None else sreg.shape]
        ctx.save_for_backward(*[t for t in ins if t is not None], scratch)
        ctx.has_sreg = sreg is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        saved = list(ctx.saved_tensors)
        scratch = saved.pop()
        ins = saved + ([] if ctx.has_sreg else [None])
        regs = ctx.regs
        dev = regs.device
        lib = L.load()
        g = dout.to(torch.float32).contiguous()
        grads = [torch.empty_like(t) for t in ins[1:9]] + [None if ins[9] is None else torch.empty_like(ins[9])]
        gs = L.B2RRegsGrads(**{k: _ptr(t) for k, t in zip(("mean_offset", "mean_offset_offset", "scale_offset", "scale",
                                                            "scale_refined", "rgb", "rgb_refined", "joint_offset",
                                                            "scale_reg"), grads)})
        st = regs._struct(ins)
        with torch.cuda.device(dev):
            L.check(lib.b2r_regs_backward(C.byref(st), _ptr(g), C.byref(gs), _ptr(scratch), scratch.numel(),
                                          torch.cuda.current_stream(dev).cuda_stream), "b2r_regs_backward")
        out = [None if t is None else t.reshape(shape) for t, shape in zip(grads, ctx.shapes)]
        return (None, None, *out)


class HumanRegularizers:
    """ExAvatar's regulariser block (avatar/main/model.py:217-257) as one sync-free CUDA op.

    faces          (F,3) integer array: smpl_x.face_upsampled.
    num_vertices   P = smpl_x.vertex_num_upsampled.
    is_rhand, is_lhand, is_face, is_face_expr, is_cavity   (P,) masks of HumanGaussian; is_rhand and is_lhand must
                   have equal counts (HandRGBReg broadcasts the two hands against each other).
    is_arm         (P,) mask: the vertices whose skinning_weight.argmax(1) is R_Shoulder, R_Elbow, L_Shoulder or L_Elbow
                   (the constant half of smpl_x.get_arm).
    joint_offset_target  (J,3): smpl_x.joint_offset.
    hand_joints    joint ids weighted 10 in joint_offset_reg (smpl_x.joint_part['lhand'] + ['rhand']).
    sym_pairs      (right_ids, left_ids): the joint pairs of JointOffsetSymmetricReg.
    device         where the tables live; defaults to is_rhand's device if CUDA, else the current CUDA device.

    Construction builds the tables once (it may synchronise): LaplacianReg's neighbour table by its own rule and its
    transpose, the five weight columns, the hand and arm rows, the joint tables, and a `VertexNormals` (no flip) whose
    kernel gives the normals of mesh_neutral_pose.

    A call returns {key: 0-dim float32} for KEYS, each the mean of the reference's map with its constant factor.
    Per-vertex inputs are (P,3) float32 CUDA tensors ((P,1) or (P,) for scale_offset), with an optional leading batch
    dimension of 1.  scale_reg (assets['scale_wo_clamp'] in the warm-up) replaces `scale` in gaussian_scale_reg.
    mesh_neutral_pose gets no gradient (the reference detaches it or uses it under no_grad); every other input does.
    Divergences from the reference: lap_mean takes the Laplacian of the offsets, lap(mnp + o) - lap(mnp) = lap(o), which
    equals the reference's difference in exact arithmetic without its fp32 cancellation; a tie at the k-th arm distance
    goes to the lowest vertex index (torch.topk leaves it unspecified); with no lower-arm row arm_rgb_reg is NaN, where
    the reference raises in torch.min of an empty tensor.
    """

    def __init__(self, faces, num_vertices: int, *, is_rhand, is_lhand, is_face, is_face_expr, is_cavity, is_arm,
                 joint_offset_target, hand_joints: Sequence[int], sym_pairs: Tuple[Sequence[int], Sequence[int]],
                 device=None):
        if device is None:
            device = is_rhand.device if isinstance(is_rhand, torch.Tensor) and is_rhand.is_cuda else \
                torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError(f"HumanRegularizers: device must be CUDA (got {device}); there is no CPU path")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        P = int(num_vertices)
        f = np.asarray(faces.detach().cpu() if isinstance(faces, torch.Tensor) else faces)
        self.normals = VertexNormals(f, P, flip=None, device=device)
        tab = make_tables(f, P, is_rhand=is_rhand, is_lhand=is_lhand, is_face=is_face, is_face_expr=is_face_expr,
                          is_cavity=is_cavity, is_arm=is_arm, joint_offset_target=joint_offset_target,
                          hand_joints=hand_joints, sym_pairs=sym_pairs)
        self.tables = tab  # CPU copies, for human_regularizers_reference
        dev = lambda t, dt: t.to(device=device, dtype=dt).contiguous()  # noqa: E731
        self.nbr_idx = dev(torch.from_numpy(tab["nbr_idx"]), torch.int32)
        self.nbr_w = dev(torch.from_numpy(tab["nbr_w"]), torch.float32)
        src = np.repeat(np.arange(P), NEIGHBOR_MAX)
        dst, w = tab["nbr_idx"].reshape(-1), tab["nbr_w"].reshape(-1)
        keep = w != 0
        order = np.argsort(dst[keep], kind="stable")  # entries come in (source, slot) order: sources stay ascending
        self.lapT_src = dev(torch.from_numpy(src[keep][order]), torch.int32)
        self.lapT_w = dev(torch.from_numpy(w[keep][order]), torch.float32)
        offs = np.zeros(P + 1, dtype=np.int64)
        offs[1:] = np.cumsum(np.bincount(dst[keep], minlength=P))
        self.lapT_offsets = dev(torch.from_numpy(offs), torch.int32)
        self.weights = dev(tab["weights"], torch.float32)
        self.hand = dev(tab["is_rhand"].to(torch.uint8) | (tab["is_lhand"].to(torch.uint8) << 1), torch.uint8)
        arm_idx = torch.nonzero(tab["is_arm"]).reshape(-1)
        slot = torch.full((P,), -1, dtype=torch.int64)
        slot[arm_idx] = torch.arange(arm_idx.numel())
        self.arm_idx = dev(arm_idx, torch.int32)
        self.arm_slot = dev(slot, torch.int32)
        self.joint_target = dev(tab["joint_target"], torch.float32)
        self.joint_weight = dev(tab["joint_weight"], torch.float32)
        self.sym_pairs = dev(tab["sym_pairs"], torch.int32)
        self.num_vertices, self.num_joints, self.device = P, int(tab["joint_target"].shape[0]), device
        self.n_arm = int(arm_idx.numel())
        self.scratch_bytes = int(L.load().b2r_regs_scratch_bytes(P, self.n_arm))
        self._template = L.B2RRegs(
            P=P, J=self.num_joints, n_arm=self.n_arm, n_pairs=int(self.sym_pairs.shape[0]),
            n_hand=int((tab["is_rhand"] | tab["is_lhand"]).sum()), n_rhand=int(tab["is_rhand"].sum()),
            faces=_ptr(self.normals.faces), vf_offsets=_ptr(self.normals.offsets), vf_entries=_ptr(self.normals.entries),
            nbr_idx=_ptr(self.nbr_idx), nbr_w=_ptr(self.nbr_w), lapT_offsets=_ptr(self.lapT_offsets),
            lapT_src=_ptr(self.lapT_src), lapT_w=_ptr(self.lapT_w), weights=_ptr(self.weights), hand=_ptr(self.hand),
            arm_idx=_ptr(self.arm_idx) if self.n_arm else None, arm_slot=_ptr(self.arm_slot),
            joint_target=_ptr(self.joint_target), joint_weight=_ptr(self.joint_weight), sym_pairs=_ptr(self.sym_pairs))

    def _struct(self, ins) -> "L.B2RRegs":
        st = L.B2RRegs.from_buffer_copy(self._template)
        for name, t in zip(("mesh", "mean_offset", "mean_offset_offset", "scale_offset", "scale", "scale_refined", "rgb",
                            "rgb_refined", "joint_offset", "scale_reg"), ins):
            setattr(st, name, _ptr(t))
        return st

    def __call__(self, mesh_neutral_pose, mean_offset, mean_offset_offset, scale_offset, scale, scale_refined, rgb,
                 rgb_refined, joint_offset, scale_reg: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        out = _Regs.apply(self, mesh_neutral_pose, mean_offset, mean_offset_offset, scale_offset, scale, scale_refined,
                          rgb, rgb_refined, joint_offset, scale_reg)
        return {k: out[i] for i, k in enumerate(KEYS)}

    def reference(self, *args, dtype: torch.dtype = torch.float64, **kw) -> Dict[str, torch.Tensor]:
        """human_regularizers_reference with this op's tables."""
        return human_regularizers_reference(self.normals.faces.cpu(), *args, tables=self.tables, dtype=dtype, **kw)


def make_tables(faces, P: int, *, is_rhand, is_lhand, is_face, is_face_expr, is_cavity, is_arm, joint_offset_target,
                hand_joints, sym_pairs, nbr: Optional[Tuple[np.ndarray, np.ndarray]] = None) -> dict:
    """The op's constant tables on the CPU (shared by HumanRegularizers and human_regularizers_reference)."""
    r, l = _mask(is_rhand, P, "is_rhand"), _mask(is_lhand, P, "is_lhand")
    if int(r.sum()) != int(l.sum()):
        raise ValueError(f"HumanRegularizers: is_rhand has {int(r.sum())} rows and is_lhand {int(l.sum())}; "
                         "HandRGBReg broadcasts the two hands against each other and needs equal counts")
    jt = torch.as_tensor(joint_offset_target).detach().to("cpu", torch.float64)  # the op uploads it as float32
    if jt.dim() != 2 or jt.shape[1] != 3 or not 1 <= jt.shape[0] <= 256:
        raise ValueError(f"HumanRegularizers: joint_offset_target must be (J,3) with 1 <= J <= 256, got {tuple(jt.shape)}")
    J = jt.shape[0]
    jw = torch.ones(J, dtype=torch.float32)
    hj = torch.as_tensor(list(hand_joints), dtype=torch.int64)
    right, left = (torch.as_tensor(list(x), dtype=torch.int64) for x in sym_pairs)
    for name, ids in (("hand_joints", hj), ("sym_pairs", right), ("sym_pairs", left)):
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= J):
            raise ValueError(f"HumanRegularizers: `{name}` holds joint ids outside [0, {J})")
    if right.numel() != left.numel() or right.numel() == 0:
        raise ValueError("HumanRegularizers: sym_pairs must be two equally long, non-empty lists of joint ids")
    jw[hj] = 10
    idx, w = laplacian_table(faces, P) if nbr is None else nbr
    return {"nbr_idx": idx, "nbr_w": w,
            "weights": weight_columns(P, r, l, is_face, is_face_expr, is_cavity),
            "is_rhand": r, "is_lhand": l, "is_arm": _mask(is_arm, P, "is_arm"), "joint_target": jt,
            "joint_weight": jw, "sym_pairs": torch.stack([right, left], 1)}


def arm_selection_reference(mesh: torch.Tensor, normals: torch.Tensor, is_arm: torch.Tensor, chunk: int = 1024):
    """smpl_x.get_arm's split and ArmRGBReg's neighbour selection in fp32 torch on the CPU: upper rows n_y > cos(pi/3),
    lower rows n_y <= cos(pi/3); per lower row the k = min(50, min_i c_i) upper rows of least fp32 distance
    sqrt((dx*dx + dy*dy) + dz*dz) among the c_i with |fl(l_x - u_x)| < 0.01, ties to the lowest vertex index.
    Returns (lower (n_lo,), sel (n_lo,k) vertex ids, k, tie (n_lo,) bool: the k-th and (k+1)-th distances are equal)."""
    m = mesh.detach().to("cpu", torch.float32).reshape(-1, 3)
    n = normals.detach().to("cpu", torch.float32).reshape(-1, 3)
    arm = is_arm.to("cpu").reshape(-1).bool()
    upper = torch.nonzero(arm & (n[:, 1] > math.cos(math.pi / 3))).reshape(-1)
    lower = torch.nonzero(arm & (n[:, 1] <= math.cos(math.pi / 3))).reshape(-1)
    mu, ml = m[upper], m[lower]
    dists, counts = [], []
    for a in range(0, lower.numel(), chunk):
        lo = ml[a:a + chunk]
        mask = torch.abs(lo[:, None, 0] - mu[None, :, 0]) < ARM_DIST_X
        d = lo[:, None, :] - mu[None, :, :]
        dist = torch.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])
        dists.append(torch.where(mask, dist, torch.full_like(dist, float("inf"))))
        counts.append(mask.sum(1))
    if lower.numel() == 0:
        return lower, torch.zeros((0, 0), dtype=torch.int64), 0, torch.zeros(0, dtype=torch.bool)
    dist = torch.cat(dists)
    k = min(ARM_TOPK, int(torch.cat(counts).min()))
    ds, order = torch.sort(dist, dim=1, stable=True)  # upper rows ascend by vertex id: stable = ties to the lowest id
    sel = upper[order[:, :k]]
    tie = torch.zeros(lower.numel(), dtype=torch.bool)
    if 0 < k < upper.numel():
        tie = (ds[:, k - 1] == ds[:, k]) & torch.isfinite(ds[:, k])
    return lower, sel, k, tie


def human_regularizers_reference(faces, mesh_neutral_pose, mean_offset, mean_offset_offset, scale_offset, scale,
                                 scale_refined, rgb, rgb_refined, joint_offset, *, scale_reg=None, tables=None,
                                 dtype: torch.dtype = torch.float64, **labels) -> Dict[str, torch.Tensor]:
    """`HumanRegularizers` restated in plain torch on the CPU, in `dtype` (float64 by default) and differentiable in every
    input but mesh_neutral_pose.  `tables` are make_tables' (or pass the constructor's keyword arguments as `labels`).
    HandMeanReg's normals are vertex_normals_reference in `dtype`; the arm split and selection are
    arm_selection_reference's, in fp32 like the reference's training run; the lap_mean differences are Laplacians of the
    offsets.  The product never calls this."""
    P = int(mesh_neutral_pose.shape[-2])
    if tables is None:
        tables = make_tables(faces, P, **labels)
    cpu = lambda t, k=3: t.to("cpu").reshape(P, k).to(dtype)  # noqa: E731
    mo, moo, s, sr, c, cr = (cpu(t) for t in (mean_offset, mean_offset_offset, scale, scale_refined, rgb, rgb_refined))
    so = cpu(scale_offset, 1)
    su = s if scale_reg is None else cpu(scale_reg)
    jo = joint_offset.to("cpu").reshape(-1, 3).to(dtype)
    mesh = mesh_neutral_pose.detach().to("cpu", torch.float32).reshape(P, 3)
    normal = vertex_normals_reference(mesh, faces, dtype=dtype)
    w = tables["weights"].to(dtype)
    nidx = torch.as_tensor(tables["nbr_idx"]).long()
    nw = torch.as_tensor(tables["nbr_w"]).to(dtype)
    lap = lambda x: x + (x[nidx] * nw[:, :, None]).sum(1)  # noqa: E731
    r, l = tables["is_rhand"], tables["is_lhand"]
    hand = r | l
    out = {}
    out["gaussian_mean_reg"] = ((mo ** 2 + moo ** 2) * w[0][:, None]).mean()
    hm = lambda o: torch.clamp((normal * F.normalize(o, p=2, dim=1)).sum(1)[hand], min=0)  # noqa: E731
    out["gaussian_mean_hand_reg"] = (hm(mo) + hm(moo)).mean()
    out["gaussian_scale_reg"] = ((su ** 2 + so ** 2) * w[1][:, None]).mean()
    out["lap_mean"] = ((lap(mo) ** 2 + lap(mo + moo) ** 2) * 100000 * w[2][:, None]).mean()
    out["lap_scale"] = ((lap(s) ** 2 + lap(sr) ** 2) * 100000 * w[3][:, None]).mean()
    out["lap_rgb"] = ((lap(c) ** 2 + lap(cr) ** 2) * w[4][:, None]).mean()
    hr = lambda x: (x[r] - x[r].mean(0).detach()) ** 2 + (x[l] - x[l].mean(0).detach()) ** 2  # noqa: E731
    out["hand_rgb_reg"] = (hr(c) + hr(cr)).mean() * 0.01
    lower, sel, k, _ = arm_selection_reference(mesh, vertex_normals_reference(mesh, faces, dtype=torch.float32),
                                               tables["is_arm"])
    if lower.numel() == 0:
        out["arm_rgb_reg"] = (c.sum() + cr.sum()) * float("nan")
    else:
        ar = lambda x: (x[lower] - x[sel.reshape(-1)].reshape(lower.numel(), k, 3).mean(1).detach()) ** 2  # noqa: E731
        out["arm_rgb_reg"] = (ar(c) + ar(cr)).mean() * 0.1
    jw = tables["joint_weight"].to(dtype)
    out["joint_offset_reg"] = ((jo - tables["joint_target"].to(dtype)) ** 2 * jw[:, None]).mean()
    ri, li = tables["sym_pairs"][:, 0], tables["sym_pairs"][:, 1]
    out["joint_offset_sym_reg"] = (torch.abs(jo[ri, 0] + jo[li, 0]) + torch.abs(jo[ri, 1] - jo[li, 1])
                                   + torch.abs(jo[ri, 2] - jo[li, 2])).mean()
    return out
