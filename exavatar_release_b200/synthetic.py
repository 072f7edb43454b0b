"""Seeded synthetic Gaussian assets for parity tests and bench.py (no dataset / SMPL-X files offline).

Generator of SURVEY.md section 8(d).  Two populations:
  * "avatar": what `HumanGaussian.forward` emits (module.py:516-586): isotropic scale (module.py:532),
    identity quaternion (module.py:564), opacity == 1 (module.py:565), on a body-sized ellipsoid shell;
  * "scene": what `SceneGaussian.forward` emits (module.py:253-272): anisotropic, random rotation,
    sigmoid opacity, scattered through the view frustum.
Workloads follow BASELINE.json `configs` (C1..C5).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

SH_C0 = 0.28209479177387814


@dataclass(frozen=True)
class Workload:
    name: str
    height: int
    width: int
    n_avatar: int
    n_scene: int
    sh_degree: int  # 0 => colours precomputed (ExAvatar's real call, module.py:618,635-636)
    backward: bool


WORKLOADS = {
    # BASELINE.json configs[0..4]
    "C1": Workload("C1:256x256,10475 avatar splats,fwd", 256, 256, 10475, 0, 0, False),
    "C2": Workload("C2:512x512,100k splats (56k avatar+44k scene),fwd+bwd", 512, 512, 56000, 44000, 0, True),
    "C3": Workload("C3:1024x1024,300k splats,SH deg 3,fwd+bwd", 1024, 1024, 167000, 133000, 3, True),
    "C4": Workload("C4:512x512 train frame,167k avatar+130k scene,fwd+bwd", 512, 512, 167000, 130000, 0, True),
    "C5": Workload("C5:1920x1080,500k splats (167k avatar+333k scene),fwd", 1080, 1920, 167000, 333000, 0, False),
    # small cases for tests
    "T0": Workload("T0:64x64,300 splats", 64, 64, 150, 150, 0, True),
    "T1": Workload("T1:128x96,4k splats", 96, 128, 2000, 2000, 0, True),
    "T2": Workload("T2:200x136,6k splats,SH3", 136, 200, 3000, 3000, 3, True),
}


def _avatar(n, g, tiny_scale=False):
    # points on a 0.5 x 1.7 x 0.3 m ellipsoid shell centred 4.24 m in front of the camera
    u = torch.randn(n, 3, generator=g)
    u = u / u.norm(dim=1, keepdim=True)
    semi = torch.tensor([0.25, 0.85, 0.15])
    pos = u * semi
    normal = u / semi
    normal = normal / normal.norm(dim=1, keepdim=True)
    pos = pos + normal * (0.005 * torch.randn(n, 1, generator=g))
    pos[:, 2] += 4.24
    s = torch.exp(math.log(0.004) + 0.4 * torch.randn(n, 1, generator=g))
    if tiny_scale:  # warm-up clamp of model.py:90-97
        s = s.clamp(max=1e-3)
    scale = s.repeat(1, 3)
    rot = torch.tensor([[1.0, 0.0, 0.0, 0.0]]).repeat(n, 1)
    opacity = torch.ones(n, 1)
    rgb = torch.rand(n, 3, generator=g)
    return pos, scale, rot, opacity, rgb


def _scene(n, g, tan_half_x, tan_half_y):
    z = 2.0 + 10.0 * torch.rand(n, generator=g)
    x = (2 * torch.rand(n, generator=g) - 1) * 1.2 * tan_half_x * z
    y = (2 * torch.rand(n, generator=g) - 1) * 1.2 * tan_half_y * z
    pos = torch.stack([x, y, z], 1)
    scale = torch.exp(math.log(0.02) + 0.7 * torch.randn(n, 3, generator=g))
    q = torch.randn(n, 4, generator=g)
    rot = q / q.norm(dim=1, keepdim=True)
    opacity = torch.sigmoid(2.0 * torch.randn(n, 1, generator=g))
    rgb = torch.rand(n, 3, generator=g)
    return pos, scale, rot, opacity, rgb


def make_assets(workload, seed=0, device="cpu", focal_ratio=1.465, tiny_scale=False):
    """Returns the dict `GaussianRenderer.forward` consumes (module.py:594-598) plus `shs` when sh_degree > 0."""
    wl = WORKLOADS[workload] if isinstance(workload, str) else workload
    g = torch.Generator().manual_seed(seed)
    tan_x = wl.width / (2 * focal_ratio * wl.height)
    tan_y = 1.0 / (2 * focal_ratio)
    parts = []
    if wl.n_avatar:
        parts.append(_avatar(wl.n_avatar, g, tiny_scale))
    if wl.n_scene:
        parts.append(_scene(wl.n_scene, g, tan_x, tan_y))
    pos, scale, rot, opacity, rgb = (torch.cat([p[i] for p in parts]) for i in range(5))
    # interleave the populations so depth order is not the input order
    perm = torch.randperm(pos.shape[0], generator=g)
    assets = {
        "mean_3d": pos[perm].contiguous(), "scale": scale[perm].contiguous(), "rotation": rot[perm].contiguous(),
        "opacity": opacity[perm].contiguous(), "rgb": rgb[perm].contiguous(),
    }
    if wl.sh_degree > 0:
        m = (wl.sh_degree + 1) ** 2
        shs = 0.3 * torch.randn(pos.shape[0], m, 3, generator=g)
        shs[:, 0, :] = (assets["rgb"] - 0.5) / SH_C0  # RGB2SH, transforms.py:169-170
        assets["shs"] = shs.contiguous()
    return {k: v.to(device) for k, v in assets.items()}


def make_grad_image(workload, seed=0, device="cpu"):
    """Upstream gradient dL/dcolor ~ N(0,1), fixed per seed (SURVEY section 8d)."""
    wl = WORKLOADS[workload] if isinstance(workload, str) else workload
    g = torch.Generator().manual_seed(1000 + seed)
    return torch.randn(3, wl.height, wl.width, generator=g).to(device)


def make_population_assets(workload, seed=0, device="cpu", focal_ratio=1.465):
    """The two populations of a workload as separate asset dicts, for ExAvatar's five-render training frame
    (avatar/main/model.py:81-162): `scene` (SceneGaussian), `human` (HumanGaussian) and `human_refined` (the same
    anchors with the pose-dependent mean / scale / colour offsets applied, module.py:531-534,561-562)."""
    wl = WORKLOADS[workload] if isinstance(workload, str) else workload
    g = torch.Generator().manual_seed(seed)
    tan_x = wl.width / (2 * focal_ratio * wl.height)
    tan_y = 1.0 / (2 * focal_ratio)
    keys = ("mean_3d", "scale", "rotation", "opacity", "rgb")
    human = dict(zip(keys, (t.contiguous() for t in _avatar(wl.n_avatar, g))))
    scene = dict(zip(keys, (t.contiguous() for t in _scene(wl.n_scene, g, tan_x, tan_y))))
    refined = {k: v.clone() for k, v in human.items()}
    refined["mean_3d"] = human["mean_3d"] + 0.002 * torch.randn(wl.n_avatar, 3, generator=g)
    refined["scale"] = human["scale"] * torch.exp(0.1 * torch.randn(wl.n_avatar, 1, generator=g))
    refined["rgb"] = (human["rgb"] + 0.05 * torch.randn(wl.n_avatar, 3, generator=g)).clamp(0, 1)
    to = lambda d: {k: v.to(device) for k, v in d.items()}
    return to(scene), to(human), to(refined)


def _subdivide(verts, faces):
    """One midpoint subdivision (each triangle into four, no smoothing), the input vertices kept first -- the order
    ExAvatar's `lr_idx_to_hr_idx` relies on (module.py:511-514)."""
    e = np.sort(np.stack([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]], 1).reshape(-1, 2), axis=1)
    uniq, inv = np.unique(e, axis=0, return_inverse=True)
    mid = (len(verts) + inv.reshape(-1, 3)).astype(np.int64)  # new vertex of edge (a,b), (b,c), (c,a)
    ab, bc, ca = mid[:, 0], mid[:, 1], mid[:, 2]
    a, b, c = faces[:, 0], faces[:, 1], faces[:, 2]
    nf = np.stack([np.stack([a, ab, ca], 1), np.stack([b, bc, ab], 1), np.stack([c, ca, bc], 1),
                   np.stack([ab, bc, ca], 1)], 1).reshape(-1, 3)
    return np.concatenate([verts, 0.5 * (verts[uniq[:, 0]] + verts[uniq[:, 1]])]), nf


def make_human_mesh(seed=0, rings=97, segments=108):
    """A seeded stand-in for ExAvatar's SMPL-X meshes, for `geometry.nearest_rows` / `VertexNormals`.

    The base mesh is a latitude-longitude triangulation of the body-sized ellipsoid shell of `_avatar` (0.25 x 0.85 x
    0.15 m around (0, 0, 4.24), poles on the long axis): rings * segments + 2 = 10 478 vertices by default, like
    SMPL-X's 10 475.  A small dent on the front is the "cavity": its vertices are pushed inward and flagged in `flip`.
    Two midpoint subdivisions in numpy keep the base vertices first (like `smpl_x.face_upsampled`): 167 618 vertices,
    335 232 faces.  Returns float32 / int64 / bool CPU tensors:
        targets   (V,3)  the base vertices (`mesh_neutral_pose_wo_upsample`)
        verts     (P,3)  the subdivided vertices (`mesh_neutral_pose`)
        faces     (F,3)  the subdivided faces, outward winding
        queries   (P,3)  verts + N(0, 1 mm) offsets (`mean_3d`)
        self_map  (P,)   head cap and both flanks, about 30 % (is_rhand | is_lhand | is_face)
        flip      (P,)   the cavity's vertices (is_cavity)
    """
    th = np.pi * np.arange(1, rings + 1) / (rings + 1)
    ph = 2 * np.pi * np.arange(segments) / segments
    u = np.concatenate([[[0.0, 1.0, 0.0]],
                        np.stack([np.sin(th)[:, None] * np.cos(ph)[None], np.cos(th)[:, None] * np.ones_like(ph)[None],
                                  np.sin(th)[:, None] * np.sin(ph)[None]], -1).reshape(-1, 3),
                        [[0.0, -1.0, 0.0]]])
    ring = lambda i, j: 1 + i * segments + j % segments  # noqa: E731
    j = np.arange(segments)
    faces = [np.stack([np.zeros_like(j), ring(0, j + 1), ring(0, j)], 1)]
    for i in range(rings - 1):
        faces += [np.stack([ring(i, j), ring(i, j + 1), ring(i + 1, j)], 1),
                  np.stack([ring(i + 1, j), ring(i, j + 1), ring(i + 1, j + 1)], 1)]
    south = len(u) - 1
    faces.append(np.stack([np.full_like(j, south), ring(rings - 1, j), ring(rings - 1, j + 1)], 1))
    faces = np.concatenate(faces).astype(np.int64)
    semi = np.array([0.25, 0.85, 0.15])
    # the cavity: a smooth dent, 15 mm deep, 6 cm across, on the front of the "head"
    dent_dir = np.array([0.0, 0.6, -0.8])
    ang = np.arccos(np.clip(u @ dent_dir, -1, 1))
    r0 = 0.2
    depth = np.where(ang < r0, 0.015 * 0.5 * (1 + np.cos(np.pi * ang / r0)), 0.0)
    pos = u * semi * (1 - depth / 0.15)[:, None]
    pos[:, 2] += 4.24
    v0, v1, v2 = pos[faces[:, 0]], pos[faces[:, 1]], pos[faces[:, 2]]
    outward = (np.cross(v1 - v0, v2 - v0) * ((v0 + v1 + v2) / 3 - [0.0, 0.0, 4.24])).sum(1) > 0
    faces[~outward] = faces[~outward][:, [0, 2, 1]]
    V = len(pos)
    verts, fs = _subdivide(pos, faces)
    verts, fs = _subdivide(verts, fs)
    c = verts - [0.0, 0.0, 4.24]
    d = c / semi
    flip = np.arccos(np.clip((d / np.linalg.norm(d, axis=1, keepdims=True)) @ dent_dir, -1, 1)) < 0.8 * r0
    self_map = (c[:, 1] > 0.6) | (np.abs(c[:, 0]) > 0.23)
    g = np.random.default_rng(seed)
    queries = verts + 0.001 * g.standard_normal(verts.shape)
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))  # noqa: E731
    return {"targets": f32(verts[:V]), "verts": f32(verts), "faces": torch.from_numpy(fs), "queries": f32(queries),
            "self_map": torch.from_numpy(self_map), "flip": torch.from_numpy(flip)}


def make_face_mesh(seed=0, num_vertices=5023, tex_size=512):
    """A seeded stand-in for ExAvatar's FLAME face mesh and texture, for `mesh_render.FaceMeshRenderer`.

    The mesh is a cap on the upper front of `make_human_mesh`'s "head" (facing the synthetic camera, like a face): the
    `num_vertices` vertices (5 023 like FLAME) nearest the direction (0, 0.75, -0.66) of the shell's parameter sphere and
    the faces among them (about 10 k, outward winding; the cavity's dent lies inside).  Returns CPU tensors / arrays:
        vertex_idx  (V,)      int64 indices into make_human_mesh()["verts"] (stands in for smpl_x.face_vertex_idx)
        faces       (F,3)     int64 indices into vertex_idx (flame.face)
        vertex_uv   (Vt,2)    float32 planar layout (x, z of the cap) with a seam: the faces left of x = 0 use a
                              second copy of the layout moved 0.02 left, so Vt = 2 V and face_uv != faces
        face_uv     (F,3)     int64 rows of vertex_uv (flame.face_uv)
        texture     (4,T,T)   float32 RGB in [0, 1] plus a mask channel in {0, 1} (flame.texture + texture_mask)
    """
    m = make_human_mesh(seed)
    verts, faces = m["verts"].numpy().astype(np.float64), m["faces"].numpy()
    d = (verts - [0.0, 0.0, 4.24]) / [0.25, 0.85, 0.15]
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    order = np.argsort(-(d @ np.array([0.0, 0.75, -0.66])), kind="stable")
    idx = np.sort(order[:num_vertices])
    local = np.full(len(verts), -1, np.int64)
    local[idx] = np.arange(len(idx))
    fl = local[faces]
    fl = fl[(fl >= 0).all(1)]
    p = verts[idx]
    c = p - p.mean(0)
    ext = np.abs(c).max(0)
    uv = np.stack([0.5 + 0.45 * c[:, 0] / ext[0], 0.5 + 0.45 * c[:, 2] / ext[2]], 1)
    left = c[fl].mean(1)[:, 0] < 0
    vertex_uv = np.concatenate([uv, uv - [0.02, 0.0]]).astype(np.float32)
    face_uv = np.where(left[:, None], fl + len(idx), fl)
    g = torch.Generator().manual_seed(9000 + seed)
    low = torch.rand(1, 3, 16, 16, generator=g)
    rgb = torch.nn.functional.interpolate(low, size=(tex_size, tex_size), mode="bilinear", align_corners=True)[0]
    rgb = (rgb + 0.1 * torch.rand(3, tex_size, tex_size, generator=g)).clamp(0, 1)
    mask = torch.nn.functional.interpolate((torch.rand(1, 1, 8, 8, generator=g) > 0.3).float(),
                                           size=(tex_size, tex_size), mode="nearest")[0]
    return {"vertex_idx": torch.from_numpy(idx), "faces": torch.from_numpy(fl), "vertex_uv": torch.from_numpy(vertex_uv),
            "face_uv": torch.from_numpy(face_uv), "texture": torch.cat([rgb, mask]).contiguous()}


def make_scene_sh_params(scene, sh_degree=3, seed=0):
    """Pre-activation parameters of the scene population as `SceneGaussian` stores them (module.py:103-108): mean,
    opacity logit, log scale, rotation, `feature_dc` (P,1,3) = RGB2SH(rgb) and `feature_rest` (P,(d+1)^2-1,3) seeded
    N(0, 0.3^2) -- the inputs of `renderer.scene_gaussian_assets` for a degree-`sh_degree` SH scene."""
    g = torch.Generator().manual_seed(7000 + seed)
    n = scene["mean_3d"].shape[0]
    m = (sh_degree + 1) ** 2
    rest = 0.3 * torch.randn(n, m - 1, 3, generator=g)
    return {"mean": scene["mean_3d"], "opacity_logit": torch.logit(scene["opacity"].clamp(1e-4, 1 - 1e-4)),
            "log_scale": torch.log(scene["scale"]), "rotation": scene["rotation"],
            "feature_dc": ((scene["rgb"] - 0.5) / SH_C0).reshape(n, 1, 3).contiguous(),  # RGB2SH, transforms.py:169-170
            "feature_rest": rest.to(scene["mean_3d"].device)}
