"""`FaceMeshRenderer` -- ExAvatar's textured face render as one differentiable CUDA op that never syncs the host.

ExAvatar renders its FLAME face mesh twice per training frame (avatar/main/model.py:170-175):

    face_render = self.face_mesh_renderer(face_texture, human_asset['mean_3d'][None, smpl_x.face_vertex_idx, :],
                                          flame.face, cam_param_i, (img_height, img_width))   # and the refined set

`MeshRenderer` (avatar/common/nets/layer.py:23-68) builds a pytorch3d `Meshes`, `PerspectiveCameras` and
`MeshRasterizer` on every call and samples a `TexturesUV`; its output feeds loss['rgb_face'] / ['rgb_face_refined'] and
the gradient flows through the barycentric coordinates into `mean_3d`.  `FaceMeshRenderer` computes the same image from
four kernels forward and two backward (csrc/mesh_raster.cu): the camera is read on the device, nothing is uploaded
per call, the backward sums in a fixed order (bit-identical runs), and forward + backward can be captured in a CUDA
graph.  The semantics below are restated from pytorch3d's implementation; pytorch3d cannot be installed offline, so the
restatement has not been checked against pytorch3d itself.

  1. camera    p_c = R p + t (ExAvatar negates x and y; pytorch3d's screen-space camera and its screen -> NDC step undo
               that), so u = fx x_c / z_c + cx, v = fy y_c / z_c + cy, x_ndc = (W/2 - u) / s, y_ndc = (H/2 - v) / s,
               s = min(H, W) / 2; a corner's z is its view depth z_c.
  2. pixels    (row r, col c) sits at NDC (PixToNonSquareNdc(W-1-c, W, H), PixToNonSquareNdc(H-1-r, H, W)): the point
               u = c + 0.5, v = r + 0.5 (unlike the Gaussian rasteriser, which puts centres at integers and ignores the
               principal point).
  3. coverage  rasterize_meshes with blur_radius 0, faces_per_pixel 1, perspective_correct, no culling or clipping.  A
               face is skipped if max z < 0, |E(v0,v1,v2)| <= 1e-8 or a corner is not finite.  A pixel centre is covered
               if it lies in the face's closed NDC xy box (pytorch3d's CheckPointOutsideBoundingBox; it only matters for
               a face that straddles the camera plane), pz = b.z >= 0 and all three perspective-corrected b are > 0, with
               b0 = (E(p,v1,v2), E(p,v2,v0), E(p,v0,v1)) / (E(v2,v0,v1) + 1e-8) and
               b = (b0.x z1 z2, z0 b0.y z2, z0 z1 b0.z) / max(sum, 1e-8).  The least pz wins, ties to the lowest index.
  4. texture   TexturesUV: uv = sum_k b_k (a_k, 1 - b_k) over the corners' vertex_uv rows, the vertically flipped map
               sampled at 2 uv - 1 (bilinear, align_corners=True, padding_mode="border"): uv row (a, b) reads column
               a (Wt - 1), row b (Ht - 1) of the map as given.
  5. output    (1,C,H,W), -1 in every channel where no face covers the pixel (layer.py:67).
  6. gradient  to the mesh only, with the per-pixel face held fixed (the max(., 1e-8) inactive, zero beyond the texture
               border clamp, nothing from background pixels).

`face_render_reference` is the literal torch restatement of 1-6 (float32 or float64, any device) the tests compare
against; the product never calls it.

Shaded render
-------------
`ShadedMeshRenderer` draws the middle panel of every video frame of ExAvatar's animation scripts (animate.py:83,
animate_view_rot.py:98 -> `render_mesh`, avatar/common/utils/vis.py:73-109).  `render_mesh` uploads the face list,
builds pytorch3d's `Meshes`, `PerspectiveCameras`, `MeshRasterizer(bin_size=0)`, `PointLights`, `SoftPhongShader` and
`Materials` on every call, reads zbuf and the image back to the host and composites there.  The op runs the vertex
normals, the coverage pass above and one shading + composite kernel on the device.  Restated from pytorch3d's
implementation, which cannot be installed offline, so this restatement has not been checked against pytorch3d itself:

  1. camera    the mesh is in camera coordinates: R = I, t = 0, only focal and princpt are read; the image size is
               bkg's (H, W), which may be non-square.
  2. coverage  steps 1-3 above, unchanged (bin_size=0 changes pytorch3d's speed, not its result).
  3. normals   pytorch3d's verts_normals_packed of the xy-negated mesh equals D n, D = diag(-1, -1, 1), with n the
               area-weighted normals of the mesh as given (b2r_vertex_normals, no flip).  Divergence: that kernel's
               (x1 - x0) x (x2 - x0) summed per vertex in CSR order differs from pytorch3d's (v2 - v1) x (v0 - v1) and
               float index_add in rounding only.
  4. shading   SoftPhongShader with PointLights() (location (0, 1, 0), ambient 0.5, diffuse 0.3, specular 0.2),
               Materials(specular 0, shininess 0) and all-ones TexturesVertex.  With b the corrected barycentrics and
               each sum over the corners in order 0, 1, 2: P = sum b_k p_k, N = sum b_k n_k, texel = b0 + b1 + b2 (not
               1 in fp32, and kept), c = (0.5 + 0.3 relu(N/max(|N|,1e-6) . (L - P)/max(|L - P|,1e-6))) texel.  The
               kernel shades in ExAvatar's camera coordinates with L = (0, -1, 0): the dot product does not change
               under D.  The specular term is 0.2 pow(., 0) 0 = 0.
  5. blend     softmax_rgb_blend with one face per pixel (sigma = gamma = 1e-4, white background, znear 1, zfar 100)
               gives (p c + d) / (p + d) with p >= 0.5 and d = 1e-10 while pz < 99.8, i.e. c to within an fp32
               rounding; the op writes c.  Divergence: past depth ~99.8 pytorch3d fades the mesh towards white, which
               needs its signed edge distance; that branch is not restated.
  6. composite vis.py:105-108 in fp32, numpy's order: is_bkg = 1 where no face covers the pixel or pz <= 0,
               fg = c blend + (bkg / 255) (1 - blend), out = (fg (1 - is_bkg)) 255 + bkg is_bkg, with blend and
               (1 - blend), taken in double, rounded to fp32.  Background pixels are bkg bit for bit.

`shaded_mesh_reference` restates 1-6 in torch (float32 or float64) for the tests; the product never calls it.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers
from typing import Dict, Optional, Tuple, Union

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib as L
from .geometry import NORMAL_EPS, VertexNormals

EPS = 1e-8  # pytorch3d's kEpsilon


def _cam_tensors(cam_param: Dict[str, torch.Tensor], device, fn: str,
                 keys: Tuple[Tuple[str, int], ...] = (("R", 9), ("t", 3), ("focal", 2), ("princpt", 2))):
    out = []
    for k, n in keys:
        if k not in cam_param:
            raise ValueError(f"{fn}: cam_param has no `{k}`")
        v = cam_param[k]
        L.cuda(fn, f"cam_param['{k}']", v)
        if v.numel() != n:
            raise ValueError(f"{fn}: cam_param['{k}'] must hold {n} values (batch 1), got {tuple(v.shape)}")
        if v.device != device:
            raise ValueError(f"{fn}: cam_param['{k}'] is on {v.device}, the mesh tables on {device}")
        out.append(v.detach().reshape(n).to(torch.float32).contiguous())
    return out


class _FaceRender(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mesh, texture, R, t, focal, princpt, renderer, H, W):
        dev = mesh.device
        x = mesh.detach().reshape(-1, 3).contiguous()
        Cn = int(texture.shape[0])
        keys = renderer._keys_for(H * W)
        m = renderer._struct(x, texture, R, t, focal, princpt, H, W, keys)
        nbytes = L.load().b2r_mesh_render_scratch_bytes(renderer.num_faces)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        image = torch.empty((Cn, H, W), dtype=torch.float32, device=dev)
        p2f = torch.empty((H, W), dtype=torch.int32, device=dev)
        L.run("b2r_mesh_render_forward", dev, C.byref(m), L.ptr(image), L.ptr(p2f), L.ptr(scratch), nbytes)
        ctx.save_for_backward(x, texture, R, t, focal, princpt, p2f, scratch)
        ctx.renderer = renderer
        ctx.size = (H, W)
        ctx.mesh_shape = mesh.shape
        ctx.mark_non_differentiable(p2f)
        return image.unsqueeze(0), p2f

    @staticmethod
    def backward(ctx, gimg, _gp2f):
        if not ctx.needs_input_grad[0] or gimg is None:
            return (None,) * 9
        x, texture, R, t, focal, princpt, p2f, scratch = ctx.saved_tensors
        dev = x.device
        H, W = ctx.size
        r = ctx.renderer
        g = gimg.reshape(texture.shape[0], H, W).to(torch.float32).contiguous()
        dmesh = torch.empty((r.num_vertices, 3), dtype=torch.float32, device=dev)
        m = r._struct(x, texture, R, t, focal, princpt, H, W, None)
        L.run("b2r_mesh_render_backward", dev, C.byref(m), L.ptr(p2f), L.ptr(g), L.ptr(dmesh), L.ptr(scratch),
              scratch.numel())
        return (dmesh.reshape(ctx.mesh_shape),) + (None,) * 8


def _int_table(name: str, a, fn: str) -> torch.Tensor:
    t = torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a)
    if t.dim() != 2 or t.shape[1] != 3 or t.dtype.is_floating_point or t.dtype == torch.bool:
        raise ValueError(f"{fn}: {name} must be an integer (F,3) array, got {t.dtype} {tuple(t.shape)}")
    return t


class _CoverageTables:
    """What both mesh renderers hand to the coverage pass of csrc/mesh_raster.cu: the int32 face table and its CSR (a
    `VertexNormals` in `self.topology`), the sizes, and the per-pixel key buffer its calls leave clean."""

    def _keys_for(self, n: int) -> torch.Tensor:
        if self._keys is None or self._keys.numel() < n:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError(f"{type(self).__name__}: run one call at this output size before capturing a CUDA "
                                   "graph (the first call allocates the per-pixel key buffer)")
            self._keys = torch.full((n,), -1, dtype=torch.int64, device=self.device)  # all bits set = no face
        return self._keys

    def _struct(self, x, texture, R, t, focal, princpt, H, W, keys) -> L.B2RMeshRender:
        """texture None: the texture fields stay zero (the shaded render ignores them)."""
        m = L.B2RMeshRender()
        m.V, m.F, m.height, m.width = self.num_vertices, self.num_faces, H, W
        m.mesh, m.faces = L.ptr(x), L.ptr(self.topology.faces)
        if texture is not None:
            m.Vt, m.C = int(self.vertex_uv.shape[0]), int(texture.shape[0])
            m.tex_height, m.tex_width = int(texture.shape[1]), int(texture.shape[2])
            m.vertex_uv, m.face_uv, m.texture = L.ptr(self.vertex_uv), L.ptr(self.face_uv), L.ptr(texture)
        m.cam_R, m.cam_t, m.focal, m.princpt = L.ptr(R), L.ptr(t), L.ptr(focal), L.ptr(princpt)
        m.keys = L.ptr(keys)
        m.vf_offsets, m.vf_entries = L.ptr(self.topology.offsets), L.ptr(self.topology.entries)
        return m


class FaceMeshRenderer(_CoverageTables):
    """ExAvatar's `MeshRenderer(flame.vertex_uv, flame.face_uv)` + its call with `flame.face`, as a CUDA op.

        renderer = FaceMeshRenderer(flame.vertex_uv, flame.face_uv, flame.face, flame.vertex_num)     # once
        face_render = renderer(face_texture, mean_3d[None, face_vertex_idx], cam_param, (H, W))        # per render

    vertex_uv     (Vt,2) float array or tensor; face_uv (F,3) rows of it; faces (F,3) vertex indices in
                  [0, num_vertices).  Uploaded once as float32 / int32 and range-checked (construction may
                  synchronise); the vertex -> face table of the backward is `VertexNormals`'s.
    device        where the tables live; defaults to the current CUDA device.

    A call takes the reference's arguments: uvmap (1,C,Ht,Wt) or (C,Ht,Wt) float32 with C in 1..4 (RGB + mask in
    ExAvatar), mesh (1,V,3) or (V,3) float32 world positions, cam_param {R (3,3), t (3), focal (2), princpt (2)} with
    or without a leading batch of 1, render_shape (H, W).  It returns (1,C,H,W) float32 with -1 on the background
    (the module docstring has the semantics).  The gradient reaches `mesh` only; a `uvmap` that requires grad raises
    rather than dropping its gradient.  No host synchronisation and no upload per call; the camera is read on the
    device, so a captured CUDA graph replays with new mesh and camera contents.  The renderer keeps one per-pixel key
    buffer, which its calls leave clean: calls of one renderer must run on one stream, and the first call at an output
    size must not be inside a graph capture (it allocates the buffer).  `render` also returns the per-pixel face.
    """

    def __init__(self, vertex_uv: Union[np.ndarray, torch.Tensor], face_uv: Union[np.ndarray, torch.Tensor],
                 faces: Union[np.ndarray, torch.Tensor], num_vertices: int, device=None):
        fn = "FaceMeshRenderer"
        f = _int_table("faces", faces, fn)
        fu = _int_table("face_uv", face_uv, fn)
        if f.shape[0] != fu.shape[0]:
            raise ValueError(f"{fn}: faces has {f.shape[0]} rows, face_uv {fu.shape[0]}")
        vt = torch.as_tensor(np.asarray(vertex_uv) if not isinstance(vertex_uv, torch.Tensor) else vertex_uv)
        if vt.dim() != 2 or vt.shape[1] != 2 or not vt.dtype.is_floating_point:
            raise ValueError(f"{fn}: vertex_uv must be a float (Vt,2) array, got {vt.dtype} {tuple(vt.shape)}")
        if f.shape[0] >= 2 ** 29 or int(num_vertices) >= 2 ** 29:
            raise ValueError(f"{fn}: {f.shape[0]} faces / {num_vertices} vertices exceed the op's limits")
        self.topology = VertexNormals(f, num_vertices, device=device)  # faces range-checked, int32, + the CSR
        self.device = self.topology.device
        fu = fu.to(device=self.device, dtype=torch.int64)
        if fu.numel() and (int(fu.min()) < 0 or int(fu.max()) >= vt.shape[0]):
            raise ValueError(f"{fn}: face_uv indices must lie in [0, {vt.shape[0]})")
        self.face_uv = fu.to(torch.int32).contiguous()
        self.vertex_uv = vt.detach().to(device=self.device, dtype=torch.float32).contiguous()
        self.num_vertices = int(num_vertices)
        self.num_faces = int(f.shape[0])
        self._keys: Optional[torch.Tensor] = None

    def render(self, uvmap: torch.Tensor, mesh: torch.Tensor, cam_param: Dict[str, torch.Tensor],
               render_shape: Tuple[int, int]) -> Tuple[torch.Tensor, torch.Tensor]:
        """The image (1,C,H,W) and the per-pixel face (H,W) int32 (-1: background; no gradient)."""
        fn = "FaceMeshRenderer"
        for name, v in (("uvmap", uvmap), ("mesh", mesh)):
            L.cuda(fn, name, v)
        if uvmap.requires_grad:
            raise ValueError(f"{fn}: `uvmap` requires grad, but the op returns a gradient for `mesh` only")
        if uvmap.dim() == 4 and uvmap.shape[0] != 1 or mesh.dim() == 3 and mesh.shape[0] != 1:
            raise ValueError(f"{fn}: only a batch of 1 is supported (uvmap {tuple(uvmap.shape)}, mesh "
                             f"{tuple(mesh.shape)})")
        if uvmap.dim() not in (3, 4) or not 1 <= uvmap.shape[-3] <= 4:
            raise ValueError(f"{fn}: uvmap must be (1,C,Ht,Wt) or (C,Ht,Wt) with C in 1..4, got {tuple(uvmap.shape)}")
        if mesh.dim() not in (2, 3) or mesh.shape[-1] != 3 or mesh.shape[-2] != self.num_vertices:
            raise ValueError(f"{fn}: mesh must be (1,{self.num_vertices},3) or ({self.num_vertices},3), got "
                             f"{tuple(mesh.shape)}")
        for name, v in (("uvmap", uvmap), ("mesh", mesh)):
            L.float32(fn, name, v)
            if v.device != self.device:
                raise ValueError(f"{fn}: `{name}` is on {v.device}, the mesh tables on {self.device}")
        H, W = (int(s) for s in render_shape)
        if H < 1 or W < 1 or H * W >= 2 ** 31:
            raise ValueError(f"{fn}: bad render_shape {tuple(render_shape)}")
        R, t, focal, princpt = _cam_tensors(cam_param, self.device, fn)
        tex = uvmap.detach().reshape(uvmap.shape[-3:]).contiguous()
        return _FaceRender.apply(mesh, tex, R, t, focal, princpt, self, H, W)

    def __call__(self, uvmap: torch.Tensor, mesh: torch.Tensor, cam_param: Dict[str, torch.Tensor],
                 render_shape: Tuple[int, int]) -> torch.Tensor:
        return self.render(uvmap, mesh, cam_param, render_shape)[0]


class ShadedMeshRenderer(_CoverageTables):
    """The mesh panel of ExAvatar's animation scripts, `render_mesh(mesh, smpl_x.face, cam_param, bkg)`
    (avatar/common/utils/vis.py:73-109; animate.py:83, animate_view_rot.py:98), as a CUDA op.

        renderer = ShadedMeshRenderer(smpl_x.face, smpl_x.vertex_num)                 # once
        panel = renderer(mesh, cam_param, bkg, blend_ratio=1.0)                        # per video frame

    faces         (F,3) integer array or tensor of vertex indices in [0, num_vertices); uploaded once as int32 and
                  range-checked with its vertex -> face table (construction may synchronise).
    device        where the tables live; defaults to the current CUDA device.

    A call takes mesh (V,3) or (1,V,3) float32 in camera coordinates, cam_param with focal (2) and princpt (2) (other
    keys are ignored, as render_mesh ignores them), bkg (H,W,3) float32 in 0-255 (it sets the image size) and a finite
    blend_ratio.  It returns a new (H,W,3) float32 tensor, HWC like render_mesh's numpy result, with no gradient: the
    shaded mesh blended with bkg where a face covers the pixel, bkg bit for bit elsewhere (the module section
    "Shaded render" has the semantics).  Normals, coverage, shading and composite run in three kernels with no
    upload and no host synchronisation, so a captured CUDA graph replays with new mesh, focal, princpt and bkg
    contents.  As with `FaceMeshRenderer`, calls of one renderer run on one stream and the first call at an output size
    must not be inside a graph capture.
    """

    def __init__(self, faces: Union[np.ndarray, torch.Tensor], num_vertices: int, device=None):
        fn = "ShadedMeshRenderer"
        f = _int_table("faces", faces, fn)
        if f.shape[0] >= 2 ** 29 or int(num_vertices) >= 2 ** 29:
            raise ValueError(f"{fn}: {f.shape[0]} faces / {num_vertices} vertices exceed the op's limits")
        self.topology = VertexNormals(f, num_vertices, device=device)  # faces range-checked, int32, + the CSR
        self.device = self.topology.device
        self.num_vertices = int(num_vertices)
        self.num_faces = int(f.shape[0])
        self.R = torch.eye(3, dtype=torch.float32, device=self.device).reshape(9)  # PerspectiveCameras without R / T
        self.t = torch.zeros(3, dtype=torch.float32, device=self.device)
        self._keys: Optional[torch.Tensor] = None

    def __call__(self, mesh: torch.Tensor, cam_param: Dict[str, torch.Tensor], bkg: torch.Tensor,
                 blend_ratio: float = 1.0) -> torch.Tensor:
        fn = "ShadedMeshRenderer"
        for name, v in (("mesh", mesh), ("bkg", bkg)):
            L.cuda(fn, name, v)
        if mesh.dim() == 3 and mesh.shape[0] != 1:
            raise ValueError(f"{fn}: only a batch of 1 is supported (mesh {tuple(mesh.shape)})")
        if mesh.dim() not in (2, 3) or mesh.shape[-1] != 3 or mesh.shape[-2] != self.num_vertices:
            raise ValueError(f"{fn}: mesh must be (1,{self.num_vertices},3) or ({self.num_vertices},3), got "
                             f"{tuple(mesh.shape)}")
        if bkg.dim() != 3 or bkg.shape[2] != 3:
            raise ValueError(f"{fn}: bkg must be (H,W,3), got {tuple(bkg.shape)}")
        H, W = int(bkg.shape[0]), int(bkg.shape[1])
        if H < 1 or W < 1 or H * W >= 2 ** 31:
            raise ValueError(f"{fn}: bad image size {(H, W)}")
        for name, v in (("mesh", mesh), ("bkg", bkg)):
            L.float32(fn, name, v)
            if v.device != self.device:
                raise ValueError(f"{fn}: `{name}` is on {v.device}, the mesh tables on {self.device}")
        if isinstance(blend_ratio, bool) or not isinstance(blend_ratio, numbers.Real) or \
                not math.isfinite(blend_ratio):
            raise ValueError(f"{fn}: blend_ratio must be a finite number, got {blend_ratio!r}")
        focal, princpt = _cam_tensors(cam_param, self.device, fn, (("focal", 2), ("princpt", 2)))
        x = mesh.detach().reshape(-1, 3).contiguous()
        return self._shade(x, self.topology(x), focal, princpt, bkg.detach().contiguous(), float(blend_ratio))

    def _shade(self, x, normals, focal, princpt, bkg, blend_ratio: float) -> torch.Tensor:
        """b2r_mesh_shade_forward on checked, contiguous float32 tensors; `normals` (V,3) per vertex."""
        H, W = int(bkg.shape[0]), int(bkg.shape[1])
        m = self._struct(x, None, self.R, self.t, focal, princpt, H, W, self._keys_for(H * W))
        nbytes = L.load().b2r_mesh_render_scratch_bytes(self.num_faces)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        out = torch.empty((H, W, 3), dtype=torch.float32, device=self.device)
        # vis.py's `render * blend_ratio + bkg / 255 * (1 - blend_ratio)`: numpy rounds the Python floats blend_ratio
        # and (1 - blend_ratio), the latter taken in double, to float32; ctypes' c_float rounds the same way
        L.run("b2r_mesh_shade_forward", self.device, C.byref(m), L.ptr(normals), L.ptr(bkg), blend_ratio,
              1.0 - blend_ratio, L.ptr(out), L.ptr(scratch), nbytes)
        return out


# ---------------------------------------------------------------------------------------------------------------------
# The torch restatement
# ---------------------------------------------------------------------------------------------------------------------

def _div(a: torch.Tensor, b) -> torch.Tensor:
    """a / b as an elementwise IEEE division: a scalar divisor is expanded to a full tensor first, because torch turns
    division by a scalar into multiplication by its reciprocal (one more rounding than the kernel's division)."""
    b = torch.as_tensor(b, dtype=a.dtype, device=a.device)
    return a / torch.broadcast_to(b, torch.broadcast_shapes(a.shape, b.shape)).contiguous()


def _pix_ndc(n: int, other: int, dtype, device) -> torch.Tensor:
    """pytorch3d's PixToNonSquareNdc(n-1-i, n, other) for i = 0..n-1 (pixel centres along one axis)."""
    one = lambda v: torch.tensor(float(v), dtype=dtype, device=device)  # noqa: E731
    rng = one(2.0)
    if n > other:
        rng = _div(one(n) * rng, one(other))
    off = _div(rng, one(2.0))
    i = torch.arange(n - 1, -1, -1, dtype=dtype, device=device)
    return -off + _div(rng * i + off, one(n))


def _edge(px, py, ax, ay, bx, by):
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax)


def _ndc(mesh: torch.Tensor, cam: Dict[str, torch.Tensor], H: int, W: int):
    """Step 1 elementwise, in the kernel's operation order: (x_ndc, y_ndc, z) per vertex."""
    dt = mesh.dtype
    R = cam["R"].reshape(3, 3).to(device=mesh.device, dtype=dt)
    t = cam["t"].reshape(3).to(device=mesh.device, dtype=dt)
    f = cam["focal"].reshape(2).to(device=mesh.device, dtype=dt)
    c = cam["princpt"].reshape(2).to(device=mesh.device, dtype=dt)
    X, Y, Z = mesh[:, 0], mesh[:, 1], mesh[:, 2]
    xc = R[0, 0] * X + R[0, 1] * Y + R[0, 2] * Z + t[0]
    yc = R[1, 0] * X + R[1, 1] * Y + R[1, 2] * Z + t[1]
    zc = R[2, 0] * X + R[2, 1] * Y + R[2, 2] * Z + t[2]
    u = _div(f[0] * xc, zc) + c[0]
    v = _div(f[1] * yc, zc) + c[1]
    s = 0.5 * min(H, W)
    return _div(0.5 * W - u, s), _div(0.5 * H - v, s), zc


def _bary(px, py, x, y, z):
    """Screen barycentrics, their perspective correction and pz for (pixel, face) rows; x, y, z are (N,3)."""
    area = _edge(x[:, 2], y[:, 2], x[:, 0], y[:, 0], x[:, 1], y[:, 1]) + EPS
    w0 = _div(_edge(px, py, x[:, 1], y[:, 1], x[:, 2], y[:, 2]), area)
    w1 = _div(_edge(px, py, x[:, 2], y[:, 2], x[:, 0], y[:, 0]), area)
    w2 = _div(_edge(px, py, x[:, 0], y[:, 0], x[:, 1], y[:, 1]), area)
    z0, z1, z2 = z[:, 0], z[:, 1], z[:, 2]
    t0 = w0 * z1 * z2
    t1 = z0 * w1 * z2
    t2 = z0 * z1 * w2
    den = torch.clamp_min(t0 + t1 + t2, EPS)
    b = torch.stack([_div(t0, den), _div(t1, den), _div(t2, den)], 1)
    pz = b[:, 0] * z0 + b[:, 1] * z1 + b[:, 2] * z2
    return b, pz


def _pixel_faces(x, y, z, faces, H, W, chunk):
    """Step 3 without grad: the (H*W,) covering face of least pz, ties to the lowest index, -1 where none."""
    dev, dt = x.device, x.dtype
    fx, fy, fz = x[faces], y[faces], z[faces]  # (F,3)
    e = _edge(fx[:, 0], fy[:, 0], fx[:, 1], fy[:, 1], fx[:, 2], fy[:, 2])
    ok = torch.isfinite(fx).all(1) & torch.isfinite(fy).all(1) & torch.isfinite(fz).all(1)
    ok &= ~(fz.amax(1) < 0) & ~((e <= EPS) & (e >= -EPS))
    s = 0.5 * min(H, W)
    # conservative pixel box of the NDC box (u = n/2 - ndc * s, centre at index + 0.5), two pixels of margin
    xs, ys = fx.double().nan_to_num(), fy.double().nan_to_num()
    c0 = (0.5 * W - xs.amax(1) * s - 0.5).floor().sub(2).clamp(0, W).long()
    c1 = (0.5 * W - xs.amin(1) * s - 0.5).ceil().add(2).clamp(-1, W - 1).long()
    r0 = (0.5 * H - ys.amax(1) * s - 0.5).floor().sub(2).clamp(0, H).long()
    r1 = (0.5 * H - ys.amin(1) * s - 0.5).ceil().add(2).clamp(-1, H - 1).long()
    bw, bh = (c1 - c0 + 1).clamp_min(0), (r1 - r0 + 1).clamp_min(0)
    n = torch.where(ok, bw * bh, torch.zeros_like(bw))
    colx, rowy = _pix_ndc(W, H, dt, dev), _pix_ndc(H, W, dt, dev)
    best_z = torch.full((H * W,), float("inf"), dtype=dt, device=dev)
    pair_f, pair_p, pair_z = [], [], []
    fids = torch.nonzero(n > 0)[:, 0]
    counts = n[fids]
    start = 0
    while start < len(fids):  # faces in chunks of about `chunk` (face, pixel) pairs
        csum = torch.cumsum(counts[start:], 0)
        stop = start + max(1, int(torch.searchsorted(csum, torch.tensor(chunk, device=dev))))
        fid = fids[start:stop]
        cnt = counts[start:stop]
        f = torch.repeat_interleave(fid, cnt)
        k = torch.arange(len(f), device=dev) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
        col = c0[f] + k % bw[f]
        row = r0[f] + torch.div(k, bw[f], rounding_mode="floor")
        px, py = colx[col], rowy[row]
        inbox = (px <= fx[f].amax(1)) & (px >= fx[f].amin(1)) & (py <= fy[f].amax(1)) & (py >= fy[f].amin(1))
        b, pz = _bary(px, py, fx[f], fy[f], fz[f])
        cov = inbox & ~(pz < 0) & (b > 0).all(1)
        p = (row * W + col)[cov]
        pair_f.append(f[cov])
        pair_p.append(p)
        pair_z.append(pz[cov])
        best_z.scatter_reduce_(0, p, pz[cov], reduce="amin")
        start = stop
    p2f = torch.full((H * W,), torch.iinfo(torch.int64).max, dtype=torch.int64, device=dev)
    if pair_f:
        f, p, pz = torch.cat(pair_f), torch.cat(pair_p), torch.cat(pair_z)
        win = pz == best_z[p]
        p2f.scatter_reduce_(0, p[win], f[win], reduce="amin")
    return torch.where(p2f == torch.iinfo(torch.int64).max, -1, p2f)


def face_render_reference(uvmap: torch.Tensor, mesh: torch.Tensor, faces, vertex_uv, face_uv,
                          cam_param: Dict[str, torch.Tensor], render_shape: Tuple[int, int],
                          pix_to_face: Optional[torch.Tensor] = None, chunk: int = 1 << 22
                          ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Steps 1-6 of the module docstring restated in torch, computed in mesh's dtype (float32 or float64) on mesh's
    device; differentiable with respect to `mesh`.  Returns (image (1,C,H,W), pix_to_face (H,W) int64).

    The per-pixel face is found without grad: every face's (face, pixel) candidates over a conservative pixel box, the
    exact coverage test of step 3, then a scatter_reduce amin of pz per pixel and an amin of the face index among the
    candidates at that pz.  `pix_to_face` given: that map is used instead (the gradient with the face held fixed).
    Then b, uv, the flips and F.grid_sample are recomputed with autograd for the covered pixels.  The tests' reference;
    the product never calls it."""
    H, W = (int(s) for s in render_shape)
    dev, dt = mesh.device, mesh.dtype
    x3 = mesh.reshape(-1, 3)
    tex = uvmap.reshape(uvmap.shape[-3:]).to(device=dev, dtype=dt)
    Cn = tex.shape[0]
    fa = torch.as_tensor(np.asarray(faces) if not isinstance(faces, torch.Tensor) else faces).to(dev).long()
    fu = torch.as_tensor(np.asarray(face_uv) if not isinstance(face_uv, torch.Tensor) else face_uv).to(dev).long()
    vt = torch.as_tensor(np.asarray(vertex_uv) if not isinstance(vertex_uv, torch.Tensor) else vertex_uv)
    vt = vt.to(device=dev, dtype=dt)
    x, y, z = _ndc(x3, cam_param, H, W)
    if pix_to_face is None:
        with torch.no_grad():
            p2f = _pixel_faces(x.detach(), y.detach(), z.detach(), fa, H, W, chunk)
    else:
        p2f = pix_to_face.reshape(-1).to(device=dev, dtype=torch.int64)
    fg = torch.nonzero(p2f >= 0)[:, 0]
    f = p2f[fg]
    colx, rowy = _pix_ndc(W, H, dt, dev), _pix_ndc(H, W, dt, dev)
    px, py = colx[fg % W], rowy[torch.div(fg, W, rounding_mode="floor")]
    b, _ = _bary(px, py, x[fa[f]], y[fa[f]], z[fa[f]])
    uvk = torch.stack([vt[:, 0], 1 - vt[:, 1]], 1)[fu[f]]  # (N,3,2): MeshRenderer's flip of the rows
    uv = b[:, 0, None] * uvk[:, 0] + b[:, 1, None] * uvk[:, 1] + b[:, 2, None] * uvk[:, 2]
    grid = (uv * 2.0 - 1.0).view(1, 1, -1, 2)
    val = F.grid_sample(torch.flip(tex, [1])[None], grid, mode="bilinear", padding_mode="border",
                        align_corners=True)[0, :, 0]  # (C,N)
    img = torch.full((Cn, H * W), -1.0, dtype=dt, device=dev)
    img = img.index_put((torch.arange(Cn, device=dev)[:, None], fg[None]), val)
    return img.view(1, Cn, H, W), p2f.view(H, W)


def _shade_reference(mesh: torch.Tensor, faces, cam_param: Dict[str, torch.Tensor], H: int, W: int,
                     pix_to_face: Optional[torch.Tensor] = None, chunk: int = 1 << 22):
    """Steps 1-5 of "Shaded render" in mesh's dtype, without grad: (colour c (H,W,3), zbuf (H,W) with -1 where no face
    covers the pixel, pix_to_face (H,W) int64).  `pix_to_face` given: that map is used instead of step 2's."""
    dev, dt = mesh.device, mesh.dtype
    v = mesh.detach().reshape(-1, 3)
    fa = torch.as_tensor(np.asarray(faces) if not isinstance(faces, torch.Tensor) else faces).to(dev).long()
    cam = {"R": torch.eye(3, dtype=dt, device=dev), "t": torch.zeros(3, dtype=dt, device=dev),
           "focal": cam_param["focal"], "princpt": cam_param["princpt"]}
    x, y, z = _ndc(v, cam, H, W)
    if pix_to_face is None:
        p2f = _pixel_faces(x, y, z, fa, H, W, chunk)
    else:
        p2f = pix_to_face.reshape(-1).to(device=dev, dtype=torch.int64)
    fg = torch.nonzero(p2f >= 0)[:, 0]
    fc = fa[p2f[fg]]
    colx, rowy = _pix_ndc(W, H, dt, dev), _pix_ndc(H, W, dt, dev)
    b, pz = _bary(colx[fg % W], rowy[torch.div(fg, W, rounding_mode="floor")], x[fc], y[fc], z[fc])
    # pytorch3d renders the xy-negated mesh: verts_normals_packed, interpolate_face_attributes, _apply_lighting there
    vn = torch.stack([-v[:, 0], -v[:, 1], v[:, 2]], 1)
    v0, v1, v2 = vn[fa[:, 0]], vn[fa[:, 1]], vn[fa[:, 2]]
    fnorm = torch.cross(v2 - v1, v0 - v1, dim=1)
    n = torch.zeros_like(vn)
    for k in range(3):
        n = n.index_add(0, fa[:, k], fnorm)
    n = F.normalize(n, eps=NORMAL_EPS, dim=1)
    P = b[:, 0, None] * vn[fc[:, 0]] + b[:, 1, None] * vn[fc[:, 1]] + b[:, 2, None] * vn[fc[:, 2]]
    N = b[:, 0, None] * n[fc[:, 0]] + b[:, 1, None] * n[fc[:, 1]] + b[:, 2, None] * n[fc[:, 2]]
    texel = b[:, 0] + b[:, 1] + b[:, 2]
    light = torch.tensor([0.0, 1.0, 0.0], dtype=dt, device=dev)  # PointLights' default location
    angle = torch.relu((F.normalize(N, eps=NORMAL_EPS, dim=1) * F.normalize(light - P, eps=NORMAL_EPS, dim=1)).sum(1))
    c = torch.ones(H * W, dtype=dt, device=dev)  # softmax_rgb_blend's white background
    c[fg] = (0.5 + 0.3 * angle) * texel
    zbuf = torch.full((H * W,), -1.0, dtype=dt, device=dev)
    zbuf[fg] = pz
    return c.view(H, W, 1).expand(H, W, 3).contiguous(), zbuf.view(H, W), p2f.view(H, W)


def shaded_mesh_reference(mesh: torch.Tensor, faces, cam_param: Dict[str, torch.Tensor], bkg: torch.Tensor,
                          blend_ratio: float = 1.0, pix_to_face: Optional[torch.Tensor] = None, chunk: int = 1 << 22
                          ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Steps 1-6 of "Shaded render" restated in torch, computed in mesh's dtype (float32 or float64) on mesh's device:
    returns (out (H,W,3), pix_to_face (H,W) int64).  The normals are pytorch3d's form in the xy-negated frame
    ((v2 - v1) x (v0 - v1) added per corner with index_add, F.normalize), not the op's b2r_vertex_normals; the
    composite is vis.py's numpy expression with blend_ratio and (1 - blend_ratio) rounded to the dtype.
    `pix_to_face` given: that map is used instead of step 2's.  The tests' reference; the product never calls it."""
    dev, dt = mesh.device, mesh.dtype
    H, W = int(bkg.shape[0]), int(bkg.shape[1])
    c, zbuf, p2f = _shade_reference(mesh, faces, cam_param, H, W, pix_to_face, chunk)
    bk = bkg.to(device=dev, dtype=dt)
    is_bkg = (zbuf <= 0).to(dt)[:, :, None]
    beta = torch.tensor(float(blend_ratio), dtype=dt, device=dev)
    beta_c = torch.tensor(1.0 - float(blend_ratio), dtype=dt, device=dev)
    fg = c * beta + _div(bk, 255.0) * beta_c
    return (fg * (1 - is_bkg)) * 255 + bk * is_bkg, p2f
