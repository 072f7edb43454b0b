"""`nearest_rows` and `VertexNormals` -- the two per-frame mesh queries of ExAvatar's `HumanGaussian` as sync-free CUDA ops.

`HumanGaussian.forward` (avatar/common/nets/module.py) runs two pytorch3d calls every frame on the path that poses the
human Gaussians:

    nn_vertex_idxs = knn_points(mean_3d[None], mesh_neutral_pose_wo_upsample[None], K=1, return_nn=True).idx[0,:,0]
    nn_vertex_idxs[mask] = torch.arange(P).cuda()[mask]                                   # 541-546, mask -> nonzero
    normal = Meshes(verts=xyz[None], faces=torch.LongTensor(face_upsampled).cuda()[None]).verts_normals_packed()
    normal = normal * (1 - is_cavity) + (-normal) * is_cavity                             # 501-504, per-frame upload

`nearest_rows` returns the int32 rows `skinning.skin_gaussians(rows=...)` reads: an exact K=1 search over a uniform grid
built on the device per call (csrc/geometry.cu), with the self-map applied in the same kernel.  `VertexNormals` builds
a vertex -> face table once and computes the area-weighted normals with the flip in one gather kernel, with no float
atomics.  Neither synchronises the host, so `nearest_rows` -> `skin_gaussians` -> `VertexNormals` can be captured in a
CUDA graph.  `nearest_rows_reference` and `vertex_normals_reference` restate the semantics in plain torch for tests.
"""
from __future__ import annotations

from typing import Optional, Union

import numpy as np
import torch

from . import _lib as L

NORMAL_EPS = 1e-6  # F.normalize's eps


def _points(name: str, t: torch.Tensor, fn: str) -> torch.Tensor:
    L.cuda(fn, name, t)
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{fn}: `{name}` must be (N,3), got {tuple(t.shape)}")
    L.float32(fn, name, t)
    return t.detach().contiguous()


def _mask_u8(name: str, m: Optional[torch.Tensor], P: int, fn: str, device) -> Optional[torch.Tensor]:
    if m is None:
        return None
    L.cuda(fn, name, m)
    if m.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"{fn}: `{name}` must be bool or uint8, got {m.dtype}")
    if m.numel() != P or m.dim() != 1:
        raise ValueError(f"{fn}: `{name}` must be ({P},), got {tuple(m.shape)}")
    if m.device != device:
        raise ValueError(f"{fn}: `{name}` is on {m.device}, the points on {device}")
    return m.detach().contiguous().view(torch.uint8)


def nearest_rows(queries: torch.Tensor, targets: torch.Tensor, self_map: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Row of the nearest target for every query, as the (P,) int32 `rows` of `skin_gaussians`.

    queries   (P,3) float32 CUDA (`mean_3d`), targets (V,3) float32 CUDA (`mesh_neutral_pose_wo_upsample`), finite.
    self_map  (P,) bool / uint8 CUDA or None: where set, rows[i] = i and the query is not searched (ExAvatar's
              is_rhand | is_lhand | is_face, whose Gaussians keep their own vertex's skinning weights).

    Elsewhere rows[i] is the smallest j minimising dx*dx + dy*dy + dz*dz in fp32 (left to right, no fma): exactly
    torch.argmin over the full distance row, ties to the lowest index.  A query with a non-finite coordinate gets 0.
    No gradient (the rows are indices), no host synchronisation, CUDA-graph capturable.
    """
    fn = "nearest_rows"
    q = _points("queries", queries, fn)
    t = _points("targets", targets, fn)
    if q.device != t.device:
        raise ValueError(f"{fn}: queries on {q.device}, targets on {t.device}")
    P, V = int(q.shape[0]), int(t.shape[0])
    if V < 1 and P > 0:
        raise ValueError(f"{fn}: no targets to search")
    m = _mask_u8("self_map", self_map, P, fn, q.device)
    rows = torch.empty(P, dtype=torch.int32, device=q.device)
    nbytes = L.load().b2r_nearest_scratch_bytes(P, V)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=q.device)
    L.run("b2r_nearest_rows", q.device, P, L.ptr(q), V, L.ptr(t), L.ptr(m), L.ptr(rows), L.ptr(scratch), nbytes)
    return rows


def nearest_rows_reference(queries: torch.Tensor, targets: torch.Tensor, self_map: Optional[torch.Tensor] = None,
                           query_chunk: int = 2048, target_chunk: int = 4096) -> torch.Tensor:
    """`nearest_rows` restated in torch on any device: elementwise fp32 distances dx*dx + dy*dy + dz*dz per
    (query chunk, target chunk), argmin within the chunk (first minimum), chunks merged in index order with a strict `<`
    so the lowest index keeps a tie.  Non-finite queries get 0, self-mapped ones their own index.  (P,) int32."""
    q = queries.detach().float()
    t = targets.detach().float()
    P, V = q.shape[0], t.shape[0]
    rows = torch.zeros(P, dtype=torch.int64, device=q.device)
    for a in range(0, P, query_chunk):
        qa = q[a:a + query_chunk]
        best = torch.full((qa.shape[0],), float("inf"), device=q.device)
        arg = torch.zeros(qa.shape[0], dtype=torch.int64, device=q.device)
        for b in range(0, V, target_chunk):
            tb = t[b:b + target_chunk]
            dx = qa[:, 0, None] - tb[None, :, 0]
            dy = qa[:, 1, None] - tb[None, :, 1]
            dz = qa[:, 2, None] - tb[None, :, 2]
            d = dx * dx + dy * dy + dz * dz
            j = torch.argmin(d, dim=1)
            dj = d.gather(1, j[:, None])[:, 0]
            take = dj < best
            best = torch.where(take, dj, best)
            arg = torch.where(take, j + b, arg)
        rows[a:a + query_chunk] = arg
    rows[~torch.isfinite(q).all(dim=1)] = 0
    if self_map is not None:
        sm = self_map.to(q.device).bool()
        rows = torch.where(sm, torch.arange(P, device=q.device), rows)
    return rows.to(torch.int32)


class VertexNormals:
    """Area-weighted vertex normals of a fixed triangle list, with ExAvatar's cavity flip.

        normals = VertexNormals(smpl_x.face_upsampled, smpl_x.vertex_num_upsampled, flip=self.is_cavity)  # once
        normal = normals(xyz)                                                                          # per frame

    faces         (F,3) integer array or tensor, any device; uploaded once as int32 and range-checked.
    num_vertices  rows of `xyz`.
    flip          (num_vertices,) bool / uint8 / float 0-1 CUDA tensor or None: rows whose normal is negated.
    device        where the tables live; defaults to flip's device, else the current CUDA device.

    Construction builds the vertex -> face CSR (each vertex's incident faces in ascending order, one entry per corner)
    and may synchronise.  A call sums (x1 - x0) x (x2 - x0) over the entries in fp32, divides by max(|n|, 1e-6) (as
    F.normalize) and negates the flipped rows: one kernel, no float atomics (bit-identical runs), no host sync, no
    upload.  The result is a new (num_vertices,3) float32 tensor that does not require grad.
    """

    def __init__(self, faces: Union[np.ndarray, torch.Tensor], num_vertices: int,
                 flip: Optional[torch.Tensor] = None, device=None):
        f = torch.as_tensor(np.asarray(faces) if not isinstance(faces, torch.Tensor) else faces)
        if f.dim() != 2 or f.shape[1] != 3 or f.dtype.is_floating_point or f.dtype == torch.bool:
            raise ValueError(f"VertexNormals: faces must be an integer (F,3) array, got {f.dtype} {tuple(f.shape)}")
        if device is None:
            device = flip.device if flip is not None else torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError(f"VertexNormals: device must be CUDA (got {device}); there is no CPU fallback")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        num_vertices = int(num_vertices)
        if num_vertices < 0 or num_vertices >= 2 ** 31 - 1 or 3 * f.shape[0] >= 2 ** 31:
            raise ValueError(f"VertexNormals: {num_vertices} vertices / {f.shape[0]} faces do not fit int32 indices")
        f = f.to(device=device, dtype=torch.int64)
        if f.numel() and (int(f.min()) < 0 or int(f.max()) >= num_vertices):
            raise ValueError(f"VertexNormals: face indices must lie in [0, {num_vertices})")
        if flip is not None:
            L.cuda("VertexNormals", "flip", flip)
            if flip.numel() != num_vertices or flip.dim() != 1:
                raise ValueError(f"VertexNormals: flip must be ({num_vertices},), got {tuple(flip.shape)}")
            flip = (flip.to(device) != 0).to(torch.uint8).contiguous()
        corner = f.reshape(-1)
        order = torch.sort(corner, stable=True).indices  # corners are in face order: stable keeps faces ascending
        counts = torch.bincount(corner, minlength=num_vertices)
        self.offsets = torch.zeros(num_vertices + 1, dtype=torch.int32, device=device)
        self.offsets[1:] = torch.cumsum(counts, 0).to(torch.int32)
        self.entries = (order // 3).to(torch.int32).contiguous()
        self.faces = f.to(torch.int32).contiguous()
        self.flip = flip
        self.num_vertices = num_vertices
        self.device = device

    def __call__(self, xyz: torch.Tensor) -> torch.Tensor:
        fn = "VertexNormals"
        x = _points("xyz", xyz, fn)
        if x.shape[0] != self.num_vertices:
            raise ValueError(f"{fn}: xyz has {x.shape[0]} rows for a mesh of {self.num_vertices} vertices")
        if x.device != self.device:
            raise ValueError(f"{fn}: xyz is on {x.device}, the mesh tables on {self.device}")
        out = torch.empty((self.num_vertices, 3), dtype=torch.float32, device=x.device)
        L.run("b2r_vertex_normals", x.device, self.num_vertices, L.ptr(x), L.ptr(self.faces), L.ptr(self.offsets),
              L.ptr(self.entries), L.ptr(self.flip), L.ptr(out))
        return out


def vertex_normals_reference(xyz: torch.Tensor, faces: Union[np.ndarray, torch.Tensor],
                             flip: Optional[torch.Tensor] = None, dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """`VertexNormals` restated in torch (float64 by default) on xyz's device: the face cross products
    (x1 - x0) x (x2 - x0) added to each corner's vertex with index_add, divided by max(|n|, 1e-6), negated where `flip`
    is set."""
    x = xyz.detach().to(dtype)
    f = torch.as_tensor(np.asarray(faces) if not isinstance(faces, torch.Tensor) else faces).to(x.device).long()
    v0, v1, v2 = x[f[:, 0]], x[f[:, 1]], x[f[:, 2]]
    fn = torch.cross(v1 - v0, v2 - v0, dim=1)
    n = torch.zeros_like(x)
    for c in range(3):
        n.index_add_(0, f[:, c], fn)
    n = n / n.norm(dim=1, keepdim=True).clamp_min(NORMAL_EPS)
    if flip is not None:
        n = torch.where(flip.to(x.device).bool()[:, None], -n, n)
    return n
