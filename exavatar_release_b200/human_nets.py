"""`TriplaneFeatures` and `gn_mlp` -- the networks of ExAvatar's `HumanGaussian.forward` as sync-free CUDA ops.

`HumanGaussian` (avatar/common/nets/module.py) samples two (3,32,128,128) triplanes at every upsampled vertex
(`extract_tri_feature`, 424-457) and runs four `make_linear_layers(..., use_gn=True)` stacks over the features
(layer.py:9-20): Linear -> GroupNorm(4, 128) -> ReLU three times, then a small head.

    tri = TriplaneFeatures(pos_enc_mesh, is_face)                        # once: sample positions are constants
    tri_feat = tri(self.triplane, self.triplane_face)                     # (P,96)
    geo = gn_mlp([tri_feat], self.geo_net, [self.mean_offset_net, self.scale_net])        # (P,4): mean offset, scale
    geo_off = gn_mlp([tri_feat, pose6d], self.geo_offset_net,
                     [self.mean_offset_offset_net, self.scale_offset_net])              # pose6d (126,) is folded
    rgb = gn_mlp([tri_feat], self.rgb_net)                                                # (P,3)
    rgb_off = gn_mlp([tri_feat, pose6d, normal], self.rgb_offset_net)                     # (P,3)

Both ops read the modules' own parameters on every call and return gradients to them, never synchronise the host, can
be captured in a CUDA graph and sum their gradients in a fixed order (bit-identical runs).  The kernels are
csrc/triplane.cu and csrc/gn_mlp.cu (3xTF32 on the tensor cores: fp32-accurate).  `tri_feature_reference`,
`gn_mlp_reference` and `human_nets_reference` restate the semantics in plain torch for tests.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from .rasterizer import _ptr

TRIPLANE_SHAPE_3D = 2.0       # cfg.triplane_shape_3d: the body triplane spans [-1, 1] m around the mean vertex
TRIPLANE_FACE_SHAPE_3D = 0.3  # cfg.triplane_face_shape_3d
HIDDEN = 128
GROUPS = 4
GN_EPS = 1e-5
MAX_ROW_INPUTS = 128
MAX_HEAD = 4


def _per_axis(v) -> Tuple[float, float, float]:
    if isinstance(v, (int, float)):
        return (float(v),) * 3
    v = tuple(float(a) for a in v)
    if len(v) != 3:
        raise ValueError(f"a 3-D triplane extent must be a number or 3 numbers, got {v}")
    return v


def triplane_grid(pos_enc_mesh: torch.Tensor, is_face: torch.Tensor, shape_3d=TRIPLANE_SHAPE_3D,
                  face_shape_3d=TRIPLANE_FACE_SHAPE_3D) -> torch.Tensor:
    """(P,3,2) grid_sample coordinates of every row on the xy, xz and yz planes, by extract_tri_feature's expressions
    in pos_enc_mesh's dtype: the body rows centred on the mean over ALL rows and divided by shape_3d / 2, the face rows
    on the mean over the face rows and divided by face_shape_3d / 2."""
    def grid(xyz, ext):
        xyz = xyz - torch.mean(xyz, 0)[None, :]
        x, y, z = (xyz[:, a] / (ext[a] / 2) for a in range(3))
        return torch.stack((torch.stack((x, y), 1), torch.stack((x, z), 1), torch.stack((y, z), 1)), 1)
    g = grid(pos_enc_mesh, _per_axis(shape_3d))
    face = is_face.bool()
    if bool(face.any()):
        g[face] = grid(pos_enc_mesh[face, :], _per_axis(face_shape_3d))
    return g


def bilinear_corners(grid: torch.Tensor, height: int, width: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """F.grid_sample's bilinear corners of (..., 2) coordinates (align_corners=False, zero padding), in its order
    nw, ne, sw, se: texel indices y * width + x as int32 (-1 outside the plane) and float32 weights.  The weights are
    evaluated in float64 from the given coordinates and rounded once."""
    g = grid.double()
    ix = ((g[..., 0] + 1) * width - 1) / 2
    iy = ((g[..., 1] + 1) * height - 1) / 2
    x0, y0 = torch.floor(ix), torch.floor(iy)
    x1, y1 = x0 + 1, y0 + 1
    w = torch.stack(((x1 - ix) * (y1 - iy), (ix - x0) * (y1 - iy), (x1 - ix) * (iy - y0), (ix - x0) * (iy - y0)), -1)
    xs = torch.stack((x0, x1, x0, x1), -1)
    ys = torch.stack((y0, y0, y1, y1), -1)
    ok = (xs >= 0) & (xs < width) & (ys >= 0) & (ys < height)
    idx = torch.where(ok, ys * width + xs, torch.full_like(xs, -1)).to(torch.int32)
    return idx, w.to(torch.float32)


def _plane_shape(name: str, t: torch.Tensor, fn: str) -> Tuple[int, int, int]:
    if not t.is_cuda:
        raise RuntimeError(f"{fn}: `{name}` must be a CUDA tensor (got {t.device}); there is no CPU path")
    if t.dim() != 4 or t.shape[0] != 3:
        raise ValueError(f"{fn}: `{name}` must be (3,C,H,W), got {tuple(t.shape)}")
    if t.dtype != torch.float32:
        raise ValueError(f"{fn}: `{name}` must be float32, got {t.dtype}")
    return int(t.shape[1]), int(t.shape[2]), int(t.shape[3])


class _Triplane(torch.autograd.Function):
    @staticmethod
    def forward(ctx, triplane, triplane_face, op):
        lib = L.load()
        dev = triplane.device
        Cc, H, W = triplane.shape[1:]
        t = triplane.detach().contiguous()
        tf = triplane_face.detach().contiguous()
        feat = torch.empty((op.P, 3 * Cc), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.b2r_triplane_forward(op.P, Cc, H, W, _ptr(t), _ptr(tf), _ptr(op.is_face), _ptr(op.corners),
                                             _ptr(op.weights), _ptr(feat), torch.cuda.current_stream(dev).cuda_stream),
                    "b2r_triplane_forward")
        ctx.op = op
        ctx.shape = tuple(triplane.shape)
        return feat

    @staticmethod
    def backward(ctx, dfeat):
        op = ctx.op
        lib = L.load()
        g = dfeat.to(torch.float32).contiguous()
        dev = g.device
        _, Cc, H, W = ctx.shape
        d = torch.empty(ctx.shape, dtype=torch.float32, device=dev)
        df = torch.empty(ctx.shape, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.b2r_triplane_backward(op.P, Cc, H, W, _ptr(g), _ptr(op.offsets), _ptr(op.rows),
                                              _ptr(op.entry_w), _ptr(d), _ptr(df),
                                              torch.cuda.current_stream(dev).cuda_stream), "b2r_triplane_backward")
        return d, df, None


class TriplaneFeatures:
    """HumanGaussian.extract_tri_feature for fixed sample positions.

        tri = TriplaneFeatures(pos_enc_mesh, is_face)        # once (may synchronise)
        tri_feat = tri(self.triplane, self.triplane_face)      # every frame: (P, 3C), columns xy | xz | yz

    pos_enc_mesh  (P,3) float32 CUDA, the buffer set in HumanGaussian.init() (never trained).
    is_face       (P,) bool / uint8 / 0-1 float: the rows read from the face triplane.
    shape_3d, face_shape_3d, plane_size: cfg.triplane_shape_3d (2), cfg.triplane_face_shape_3d (0.3) and the planes'
                  (H, W) (128, 128); the extents may be numbers or per-axis triples.

    Construction computes the sample coordinates with the reference's expressions (`triplane_grid`, in float32 as the
    reference does), every row's bilinear corners and weights per plane (`bilinear_corners`: F.grid_sample's
    align_corners=False and zero padding) and the texel -> (row, weight) CSR of the backward, rows ascending.  A call
    gathers (no float atomics): face rows read `triplane_face` only and give the body triplane no gradient (the
    reference overwrites them).  The backward returns dL/dtriplane and dL/dtriplane_face, bit-identical from run to run.
    No host synchronisation per call, CUDA-graph capturable.
    """

    def __init__(self, pos_enc_mesh: torch.Tensor, is_face: torch.Tensor, shape_3d=TRIPLANE_SHAPE_3D,
                 face_shape_3d=TRIPLANE_FACE_SHAPE_3D, plane_size: Tuple[int, int] = (128, 128)):
        fn = "TriplaneFeatures"
        if not pos_enc_mesh.is_cuda:
            raise RuntimeError(f"{fn}: pos_enc_mesh must be a CUDA tensor (got {pos_enc_mesh.device})")
        if pos_enc_mesh.dim() != 2 or pos_enc_mesh.shape[1] != 3 or pos_enc_mesh.dtype != torch.float32:
            raise ValueError(f"{fn}: pos_enc_mesh must be (P,3) float32, got {pos_enc_mesh.dtype} "
                             f"{tuple(pos_enc_mesh.shape)}")
        P = int(pos_enc_mesh.shape[0])
        dev = pos_enc_mesh.device
        if is_face.numel() != P:
            raise ValueError(f"{fn}: is_face must have {P} entries, got {tuple(is_face.shape)}")
        face = (is_face.reshape(-1).to(dev) != 0)
        H, W = (int(v) for v in plane_size)
        if P < 1 or H < 1 or W < 1:
            raise ValueError(f"{fn}: need at least one row and a non-empty plane")
        pos = pos_enc_mesh.detach()
        self.grid = triplane_grid(pos, face, shape_3d, face_shape_3d)                    # (P,3,2) float32
        corners, weights = bilinear_corners(self.grid, H, W)
        self.corners = corners.contiguous()                                               # (P,3,4) int32
        self.weights = weights.contiguous()                                               # (P,3,4) float32
        # CSR: key (s * 3 + p) * H * W + texel, s = 1 for face rows; a stable sort keeps the rows ascending per key
        s = face.to(torch.int64)[:, None, None]
        p = torch.arange(3, device=dev)[None, :, None]
        key = ((s * 3 + p) * (H * W) + corners.long()).reshape(-1)
        row = torch.arange(P, device=dev)[:, None, None].expand(P, 3, 4).reshape(-1)
        valid = corners.reshape(-1) >= 0
        key, row, w = key[valid], row[valid], weights.reshape(-1)[valid]
        order = torch.sort(key, stable=True).indices
        self.rows = row[order].to(torch.int32).contiguous()
        self.entry_w = w[order].contiguous()
        self.offsets = torch.zeros(6 * H * W + 1, dtype=torch.int32, device=dev)
        self.offsets[1:] = torch.cumsum(torch.bincount(key, minlength=6 * H * W), 0).to(torch.int32)
        self.is_face = face.to(torch.uint8).contiguous()
        self.P, self.plane_size, self.device = P, (H, W), dev

    def __call__(self, triplane: torch.Tensor, triplane_face: torch.Tensor) -> torch.Tensor:
        fn = "TriplaneFeatures"
        shp = _plane_shape("triplane", triplane, fn)
        if _plane_shape("triplane_face", triplane_face, fn) != shp:
            raise ValueError(f"{fn}: triplane {tuple(triplane.shape)} and triplane_face {tuple(triplane_face.shape)} "
                             "differ")
        if shp[1:] != self.plane_size:
            raise ValueError(f"{fn}: planes are {shp[1]}x{shp[2]}, the sample table was built for "
                             f"{self.plane_size[0]}x{self.plane_size[1]}")
        if triplane.device != self.device or triplane_face.device != self.device:
            raise ValueError(f"{fn}: the planes must be on {self.device}")
        return _Triplane.apply(triplane, triplane_face, self)


def tri_feature_reference(grid: torch.Tensor, is_face: torch.Tensor, triplane: torch.Tensor,
                          triplane_face: torch.Tensor) -> torch.Tensor:
    """extract_tri_feature restated with F.grid_sample (defaults: bilinear, align_corners=False, zero padding) at the
    (P,3,2) coordinates of `triplane_grid`, in the planes' dtype: all rows from `triplane`, then the face rows
    overwritten by their samples of `triplane_face`.  Differentiable; any device."""
    g = grid.to(triplane.dtype)

    def sample(planes, gg):
        return torch.cat([F.grid_sample(planes[p, None], gg[None, :, None, p, :], align_corners=False)[0, :, :, 0]
                          for p in range(3)]).permute(1, 0)
    feat = sample(triplane, g)
    face = is_face.reshape(-1).to(g.device) != 0
    feat = feat.clone()
    feat[face] = sample(triplane_face, g[face])
    return feat


# ---------------------------------------------------------------------------------------------------------------------
# gn_mlp
# ---------------------------------------------------------------------------------------------------------------------

def _head_linears(trunk: nn.Sequential, heads) -> Tuple[List[nn.Module], List[nn.Linear]]:
    mods = list(trunk)
    heads = list(heads) if heads is not None else []
    if len(mods) == 10 and not heads:           # rgb_net / rgb_offset_net: the final Linear is the head
        body, head_lins = mods[:9], [mods[9]]
    elif len(mods) == 9 and heads:              # geo_net / geo_offset_net + their head Sequentials
        body, head_lins = mods, []
        for h in heads:
            hm = list(h) if isinstance(h, nn.Sequential) else [h]
            if len(hm) != 1 or not isinstance(hm[0], nn.Linear):
                raise ValueError("gn_mlp: each head must be a single Linear (make_linear_layers([128, k], "
                                 f"relu_final=False)), got {h}")
            head_lins.append(hm[0])
    else:
        raise ValueError(f"gn_mlp: unsupported stack of {len(mods)} modules with {len(heads)} heads: expected three "
                         "Linear -> GroupNorm(4, 128) -> ReLU blocks and either separate heads or a final Linear")
    for l in range(3):
        lin, gn, relu = body[3 * l: 3 * l + 3]
        if not isinstance(lin, nn.Linear) or lin.out_features != HIDDEN or lin.bias is None:
            raise ValueError(f"gn_mlp: layer {l} must be Linear(., {HIDDEN}) with bias, got {lin}")
        if l > 0 and lin.in_features != HIDDEN:
            raise ValueError(f"gn_mlp: layer {l} must take {HIDDEN} inputs, got {lin.in_features}")
        if (not isinstance(gn, nn.GroupNorm) or gn.num_groups != GROUPS or gn.num_channels != HIDDEN or not gn.affine
                or gn.eps != GN_EPS):
            raise ValueError(f"gn_mlp: layer {l} must be followed by GroupNorm({GROUPS}, {HIDDEN}) with affine and eps "
                             f"{GN_EPS}, got {gn}")
        if not isinstance(relu, nn.ReLU):
            raise ValueError(f"gn_mlp: layer {l} GroupNorm must be followed by ReLU, got {relu}")
    for h in head_lins:
        if not isinstance(h, nn.Linear) or h.in_features != HIDDEN or h.bias is None:
            raise ValueError(f"gn_mlp: a head must be Linear({HIDDEN}, k) with bias, got {h}")
    if sum(h.out_features for h in head_lins) > MAX_HEAD:
        raise ValueError(f"gn_mlp: the heads give {sum(h.out_features for h in head_lins)} outputs; at most "
                         f"{MAX_HEAD} are supported")
    return body, head_lins


def _layout(inputs: Sequence[torch.Tensor], in_features: int):
    """(per-row block indices, constant block indices, per-row columns, constant columns) of the first layer."""
    row_blocks, const_blocks, row_cols, const_cols = [], [], [], []
    col = 0
    for i, t in enumerate(inputs):
        if not isinstance(t, torch.Tensor) or t.dim() not in (1, 2):
            raise ValueError(f"gn_mlp: input {i} must be a (P,k) or (k,) tensor")
        k = int(t.shape[-1])
        (row_blocks if t.dim() == 2 else const_blocks).append(i)
        (row_cols if t.dim() == 2 else const_cols).extend(range(col, col + k))
        col += k
    if col != in_features:
        raise ValueError(f"gn_mlp: the inputs have {col} columns, the first layer takes {in_features}")
    if not row_blocks:
        raise ValueError("gn_mlp: at least one input must be a per-row (P,k) block")
    if len(row_cols) > MAX_ROW_INPUTS:
        raise ValueError(f"gn_mlp: {len(row_cols)} per-row first-layer inputs; at most {MAX_ROW_INPUTS} are supported")
    return row_blocks, const_blocks, row_cols, const_cols


def _runs(cols: Sequence[int]) -> List[Tuple[int, int]]:
    """(start, length) of the maximal runs of consecutive column indices."""
    runs = []
    for c in cols:
        if runs and runs[-1][0] + runs[-1][1] == c:
            runs[-1] = (runs[-1][0], runs[-1][1] + 1)
        else:
            runs.append((c, 1))
    return runs


def _columns(w: torch.Tensor, cols: Sequence[int]) -> torch.Tensor:
    """w[:, cols] from slices (no index upload, so it can be captured in a CUDA graph)."""
    return torch.cat([w[:, s:s + n] for s, n in _runs(cols)], 1)


def _set_columns(w: torch.Tensor, cols: Sequence[int], v: torch.Tensor):
    o = 0
    for s, n in _runs(cols):
        w[:, s:s + n] = v[:, o:o + n]
        o += n


class _GnMlp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, spec, *tensors):
        n_in, n_heads, row_blocks, const_blocks, row_cols, const_cols, _ = spec
        inputs = tensors[:n_in]
        params = tensors[n_in:]
        w0, b0 = params[0], params[1]
        dev = w0.device
        P = int(inputs[row_blocks[0]].shape[0])
        x = (inputs[row_blocks[0]] if len(row_blocks) == 1 else torch.cat([inputs[i] for i in row_blocks], 1))
        x = x.detach().contiguous()
        w0r = _columns(w0.detach(), row_cols).contiguous()
        b0e = b0.detach()
        c = None
        if const_blocks:
            c = torch.cat([inputs[i].detach().reshape(-1) for i in const_blocks])
            b0e = b0e + _columns(w0.detach(), const_cols) @ c  # the constant block folded into the first bias
        b0e = b0e.contiguous()
        lay = [(w0r, b0e, params[2].detach().contiguous(), params[3].detach().contiguous())]
        for l in (1, 2):
            lay.append(tuple(p.detach().contiguous() for p in params[4 * l: 4 * l + 4]))
        hw = [params[12 + 2 * h].detach() for h in range(n_heads)]
        hb = [params[13 + 2 * h].detach() for h in range(n_heads)]
        wh = torch.cat(hw, 0).contiguous()
        bh = torch.cat(hb, 0).contiguous()
        H = int(wh.shape[0])
        m = L.B2RGnMlp(P=P, K=len(row_cols), H=H, x=_ptr(x), w_head=_ptr(wh), b_head=_ptr(bh))
        for l in range(3):
            m.w[l], m.b[l], m.gamma[l], m.beta[l] = (_ptr(t) for t in lay[l])
        out = torch.empty((P, H), dtype=torch.float32, device=dev)
        train = any(ctx.needs_input_grad)
        saved = torch.empty((3, P, HIDDEN), dtype=torch.float32, device=dev) if train else None
        lib = L.load()
        with torch.cuda.device(dev):
            L.check(lib.b2r_gn_mlp_forward(C.byref(m), _ptr(out), _ptr(saved),
                                           torch.cuda.current_stream(dev).cuda_stream), "b2r_gn_mlp_forward")
        if train:
            ctx.spec = spec
            ctx.keep = (x, lay, wh, bh, c)  # the struct's pointers stay valid while these live
            ctx.m = m
            ctx.head_widths = [int(t.shape[0]) for t in hw]
            ctx.in_features = int(w0.shape[1])
            ctx.save_for_backward(saved)
        return out

    @staticmethod
    def backward(ctx, dout):
        n_in, n_heads, row_blocks, const_blocks, row_cols, const_cols, row_widths = ctx.spec
        (saved,) = ctx.saved_tensors
        x, lay, wh, bh, c = ctx.keep
        m = ctx.m
        dev = saved.device
        P, K, H = m.P, m.K, m.H
        g = dout.to(torch.float32).contiguous()
        need_x = any(ctx.needs_input_grad[1 + i] for i in row_blocks)
        dx = torch.empty((P, K), dtype=torch.float32, device=dev) if need_x else None
        lib = L.load()
        grads = torch.empty(int(lib.b2r_gn_mlp_grads_count(K, H)), dtype=torch.float32, device=dev)
        nbytes = int(lib.b2r_gn_mlp_scratch_bytes(P))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.b2r_gn_mlp_backward(C.byref(m), _ptr(saved), _ptr(g), _ptr(dx), _ptr(grads), _ptr(scratch),
                                            nbytes, torch.cuda.current_stream(dev).cuda_stream), "b2r_gn_mlp_backward")
        o = 0

        def take(*shape):
            nonlocal o
            n = 1
            for s in shape:
                n *= s
            t = grads[o:o + n].view(*shape)
            o += n
            return t
        dw = [take(HIDDEN, K), take(HIDDEN, HIDDEN), take(HIDDEN, HIDDEN)]
        dgamma, dbeta, db = take(3, HIDDEN), take(3, HIDDEN), take(3, HIDDEN)
        dwh, dbh = take(H, HIDDEN), take(H)
        dw0 = torch.empty((HIDDEN, ctx.in_features), dtype=torch.float32, device=dev)
        _set_columns(dw0, row_cols, dw[0])
        if const_blocks:
            _set_columns(dw0, const_cols, torch.outer(db[0], c))  # (sum_rows dz_0) x c
        out_inputs = [None] * n_in
        if need_x:
            col = 0
            for i, k in zip(row_blocks, row_widths):
                if ctx.needs_input_grad[1 + i]:
                    out_inputs[i] = dx[:, col:col + k]
                col += k
        params = [dw0, db[0], dgamma[0], dbeta[0]]
        for l in (1, 2):
            params += [dw[l], db[l], dgamma[l], dbeta[l]]
        r = 0
        for w in ctx.head_widths:
            params += [dwh[r:r + w], dbh[r:r + w]]
            r += w
        return (None, *out_inputs, *params)


def gn_mlp(inputs: Sequence[torch.Tensor], trunk: nn.Sequential, heads: Optional[Sequence[nn.Module]] = None
           ) -> torch.Tensor:
    """One of HumanGaussian's GroupNorm MLP stacks; returns the pre-activation head output (P, H).

    inputs  the first layer's column blocks in order: a (P,k) float32 CUDA tensor is a per-row block, a 1-D tensor is
            the same for every row and is folded into the first layer's bias (its columns' weight gradient is
            (sum_rows dL/dz_0) x c).  geo_offset_net: [tri_feat, pose6d]; rgb_offset_net: [tri_feat, pose6d, normal].
            A constant block that requires grad raises ValueError (the reference detaches it).
    trunk   the caller's nn.Sequential from make_linear_layers(..., use_gn=True): three Linear(., 128) ->
            GroupNorm(4, 128) -> ReLU blocks, optionally followed by the final Linear(128, H) (rgb_net).
    heads   the head Sequentials (each one Linear(128, k)), concatenated in column order; None / [] when the trunk
            ends in its own Linear.

    Only ExAvatar's shapes: hidden width 128, GroupNorm(4, 128) with affine and eps 1e-5, three hidden layers, at most
    128 per-row inputs and 4 head outputs; anything else raises ValueError.  The modules' parameters are read on every
    call and receive gradients (optimizer param groups and state dicts are unchanged), as do the per-row blocks that
    require grad.  Forward and backward run on the tensor cores as 3xTF32 (fp32-accurate), with no host sync, and the
    parameter gradients are reduced in a fixed order (bit-identical runs).  The forward keeps the three pre-GroupNorm
    activations (3 x P x 128 fp32) for the backward when a gradient is needed.
    """
    body, head_lins = _head_linears(trunk, heads)
    inputs = list(inputs)
    row_blocks, const_blocks, row_cols, const_cols = _layout(inputs, body[0].in_features)
    for i in const_blocks:
        if inputs[i].requires_grad:
            raise ValueError(f"gn_mlp: the constant input {i} requires grad; detach it (the reference does)")
    P = int(inputs[row_blocks[0]].shape[0])
    params = []
    for l in range(3):
        params += [body[3 * l].weight, body[3 * l].bias, body[3 * l + 1].weight, body[3 * l + 1].bias]
    for h in head_lins:
        params += [h.weight, h.bias]
    dev = params[0].device
    for t in params + inputs:
        if not t.is_cuda:
            raise RuntimeError(f"gn_mlp: every tensor must be on a CUDA device (got {t.device}); there is no CPU path")
        if t.device != dev:
            raise ValueError(f"gn_mlp: tensors on {t.device} and {dev}")
        if t.dtype != torch.float32:
            raise ValueError(f"gn_mlp: every tensor must be float32, got {t.dtype}")
    for i in row_blocks:
        if int(inputs[i].shape[0]) != P:
            raise ValueError(f"gn_mlp: per-row input {i} has {inputs[i].shape[0]} rows, input {row_blocks[0]} has {P}")
    if P < 1:
        raise ValueError("gn_mlp: no rows")
    spec = (len(inputs), len(head_lins), tuple(row_blocks), tuple(const_blocks), tuple(row_cols), tuple(const_cols),
            tuple(int(inputs[i].shape[1]) for i in row_blocks))
    return _GnMlp.apply(spec, *inputs, *params)


def gn_mlp_reference(inputs: Sequence[torch.Tensor], trunk: nn.Sequential, heads: Optional[Sequence[nn.Module]] = None,
                     dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """`gn_mlp` restated in plain torch from the formulas, in `dtype` (float64 by default): the blocks concatenated
    (constant ones repeated over the rows) in column order, then per layer z = x W^T + b, GroupNorm over 4 groups of 32
    consecutive channels with the biased variance, z_hat = (z - mean) / sqrt(var + 1e-5), y = z_hat gamma + beta, ReLU,
    and the heads' outputs concatenated.  Differentiable with respect to the modules' parameters and the inputs."""
    body, head_lins = _head_linears(trunk, heads)
    P = next(int(t.shape[0]) for t in inputs if t.dim() == 2)
    x = torch.cat([(t if t.dim() == 2 else t.reshape(1, -1).expand(P, -1)).to(dtype) for t in inputs], 1)
    for l in range(3):
        lin, gn = body[3 * l], body[3 * l + 1]
        z = x @ lin.weight.to(dtype).t() + lin.bias.to(dtype)
        zg = z.reshape(P, GROUPS, HIDDEN // GROUPS)
        mean = zg.mean(-1, keepdim=True)
        var = ((zg - mean) ** 2).mean(-1, keepdim=True)
        zh = ((zg - mean) / torch.sqrt(var + GN_EPS)).reshape(P, HIDDEN)
        x = torch.relu(zh * gn.weight.to(dtype) + gn.bias.to(dtype))
    return torch.cat([x @ h.weight.to(dtype).t() + h.bias.to(dtype) for h in head_lins], 1)


def human_nets_reference(grid: torch.Tensor, is_face: torch.Tensor, triplane: torch.Tensor,
                         triplane_face: torch.Tensor, nets: Dict[str, nn.Module], pose6d: torch.Tensor,
                         normal: torch.Tensor, dtype: torch.dtype = torch.float64) -> Dict[str, torch.Tensor]:
    """The network part of HumanGaussian.forward restated in plain torch: the triplane features (`tri_feature_reference`)
    and the four stacks (`gn_mlp_reference`) as the reference wires them.  `nets` holds ExAvatar's module names.
    Returns tri_feat (P,96), geo (P,4) = mean_offset | scale, geo_offset (P,4) = mean_offset_offset | scale_offset,
    rgb (P,3) and rgb_offset (P,3), all pre-activation."""
    tri = tri_feature_reference(grid, is_face, triplane.to(dtype), triplane_face.to(dtype))
    return {
        "tri_feat": tri,
        "geo": gn_mlp_reference([tri], nets["geo_net"], [nets["mean_offset_net"], nets["scale_net"]], dtype),
        "geo_offset": gn_mlp_reference([tri, pose6d], nets["geo_offset_net"],
                                       [nets["mean_offset_offset_net"], nets["scale_offset_net"]], dtype),
        "rgb": gn_mlp_reference([tri], nets["rgb_net"], None, dtype),
        "rgb_offset": gn_mlp_reference([tri, pose6d, normal], nets["rgb_offset_net"], None, dtype),
    }
