"""The mesh panel of ExAvatar's animation scripts (animate.py:83, animate_view_rot.py:98 -> render_mesh,
avatar/common/utils/vis.py:73-109) as a sync-free CUDA op: `mesh_render.ShadedMeshRenderer` (b2r_mesh_shade_forward).

These tests pin
  * without a device: the C ABI (symbol, struct mirror, validation before any launch), closed-form answers of
    `shaded_mesh_reference` (a triangle facing the light, the light's side of a sphere, zero normals, the fp32 texel
    sum), the D n identity of pytorch3d's normals, vis.py's numpy composite for blend_ratio 1, 0.5 and 0, and the
    Python argument checks;
  * on the GPU, on the posed synthetic SMPL-X body at 512x512, in a close-up and in a 1080x1920 portrait frame: the
    per-pixel face and is_bkg identical to the float32 restatement, the background bit for bit, covered pixels within
    1e-3 (0-255 scale) of the float32 restatement and of float64 on all but 0.1 % of them, bit-identical runs, no host
    synchronisation, and a CUDA-graph replay with new mesh, focal and princpt equal to eager.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from util import ROOT  # noqa: F401  (path setup)
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.geometry import vertex_normals_reference
from exavatar_release_b200.mesh_render import (ShadedMeshRenderer, _ndc, _shade_reference, face_render_reference,
                                               shaded_mesh_reference)
from exavatar_release_b200.synthetic import make_human_mesh, make_smplx_model

FAKE = 0x1000  # never dereferenced: validation fails before any launch


def _cam(fx, fy, cx, cy, dtype=torch.float64, device="cpu"):
    return {"focal": torch.tensor([fx, fy], dtype=dtype, device=device),
            "princpt": torch.tensor([cx, cy], dtype=dtype, device=device)}


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the C ABI
# ---------------------------------------------------------------------------------------------------------------------

def test_symbol_and_struct_mirror():
    raw = C.CDLL(L.LIB_PATH)
    assert hasattr(raw, "b2r_mesh_shade_forward")
    assert "b2r_mesh_shade_forward" in {s[0] for s in L.SYMBOLS}


def _struct(**kw):
    # only the fields the shaded render reads; the texture fields stay zero / NULL
    m = L.B2RMeshRender(V=100, F=50, height=16, width=24)
    for k in ("mesh", "faces", "cam_R", "cam_t", "focal", "princpt", "keys"):
        setattr(m, k, FAKE)
    for k, v in kw.items():
        setattr(m, k, v)
    return m


def test_validation_without_touching_cuda():
    lib = L.load()
    n0 = lib.b2r_launch_count()
    need = lib.b2r_mesh_render_scratch_bytes(50)

    def shade(m, normals=FAKE, bkg=FAKE, blend=1.0, blend_c=0.0, out=FAKE, scratch=FAKE, nbytes=need):
        return lib.b2r_mesh_shade_forward(C.byref(m) if m is not None else None, normals, bkg, blend, blend_c, out,
                                          scratch, nbytes, None)

    bad = [{"V": -1}, {"F": -1}, {"V": 0}, {"height": 0}, {"width": -3}, {"width": 65536, "height": 32768},
           {"F": 1 << 29}]
    bad += [{k: None} for k in ("mesh", "faces", "cam_R", "cam_t", "focal", "princpt", "keys")]
    for kw in bad:
        assert shade(_struct(**kw)) == -1, kw
    assert shade(None) == -1
    for kw in ({"normals": None}, {"bkg": None}, {"out": None}, {"scratch": None}, {"blend": float("nan")},
               {"blend_c": float("inf")}, {"blend": float("-inf")}):
        assert shade(_struct(), **kw) == -1, kw
    # the texture fields are not read: with them NULL / zero, a valid struct gets as far as the workspace check
    assert shade(_struct(), nbytes=need - 1) == -2
    assert lib.b2r_launch_count() == n0  # nothing was launched by any of the above


# ---------------------------------------------------------------------------------------------------------------------
# CPU: closed forms of the restatement
# ---------------------------------------------------------------------------------------------------------------------

def _ray_plane(u, v, cam, q0, n):
    """Camera-frame point where the ray of image point (u, v) meets the plane through q0 with normal n."""
    fx, fy = (float(a) for a in cam["focal"])
    cx, cy = (float(a) for a in cam["princpt"])
    d = np.array([(u - cx) / fx, (v - cy) / fy, 1.0])
    return d * (n @ q0) / (n @ d)


@pytest.mark.parametrize("shape", [(24, 32), (32, 24)])
def test_triangle_facing_the_light_matches_the_closed_form(shape):
    H, W = shape
    cam = _cam(40.0, 44.0, W / 2 + 1.3, H / 2 - 0.7)
    n = np.array([0.0, -0.6, -0.8])  # towards the light (0, -1, 0) and the camera
    e1, e2 = np.array([1.0, 0.0, 0.0]), np.cross(n, [1.0, 0.0, 0.0])
    ctr, s = np.array([0.05, 0.1, 2.0]), 0.4
    tri = np.stack([ctr + s * (-e1 - e2), ctr + s * (e1 - e2), ctr + 1.5 * s * e2])  # (q1 - q0) x (q2 - q0) || n
    assert np.cross(tri[1] - tri[0], tri[2] - tri[0]) @ n > 0
    bkg = torch.full((H, W, 3), 7.0, dtype=torch.float64)
    out, p2f = shaded_mesh_reference(torch.from_numpy(tri), [[0, 1, 2]], cam, bkg)
    fg = p2f == 0
    assert int(fg.sum()) > 60
    L_ = np.array([0.0, -1.0, 0.0])
    for r, c in torch.nonzero(fg).tolist():
        q = _ray_plane(c + 0.5, r + 0.5, cam, tri[0], n)
        d = (L_ - q) / np.linalg.norm(L_ - q)
        want = (0.5 + 0.3 * max(0.0, float(n @ d))) * 255
        assert abs(float(out[r, c, 0]) - want) < 1e-9, (r, c)
        assert out[r, c, 0] == out[r, c, 1] == out[r, c, 2]
    assert float(out[fg][:, 0].min()) > 0.5 * 255 + 1  # the diffuse term is on
    assert torch.equal(out[~fg], bkg[~fg])


def _sphere(n_lat=24, n_lon=32, radius=0.5, centre=(0.0, 0.0, 3.0)):
    th = np.pi * np.arange(1, n_lat) / n_lat
    ph = 2 * np.pi * np.arange(n_lon) / n_lon
    v = [[0.0, 1.0, 0.0]]
    v += [[np.sin(t) * np.cos(p), np.cos(t), np.sin(t) * np.sin(p)] for t in th for p in ph]
    v.append([0.0, -1.0, 0.0])
    v = np.array(v) * radius + centre
    ring = lambda i, j: 1 + i * n_lon + j % n_lon  # noqa: E731
    f = [[0, ring(0, j + 1), ring(0, j)] for j in range(n_lon)]
    for i in range(n_lat - 2):
        for j in range(n_lon):
            f += [[ring(i, j), ring(i, j + 1), ring(i + 1, j)], [ring(i + 1, j), ring(i, j + 1), ring(i + 1, j + 1)]]
    f += [[len(v) - 1, ring(n_lat - 2, j), ring(n_lat - 2, j + 1)] for j in range(n_lon)]
    f = np.array(f)
    out = (np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]) * (v[f].mean(1) - centre)).sum(1) > 0
    f[~out] = f[~out][:, [0, 2, 1]]
    return torch.from_numpy(v), f


def test_the_top_of_a_sphere_is_brighter_than_its_bottom():
    v, f = _sphere()
    H = W = 48
    cam = _cam(80.0, 80.0, 24.0, 24.0)
    out, p2f = shaded_mesh_reference(v, f, cam, torch.zeros(H, W, 3, dtype=torch.float64))
    rows = torch.nonzero((p2f >= 0).any(1))[:, 0]
    top, bottom = int(rows.min()), int(rows.max())
    third = (bottom - top + 1) // 3
    mean = lambda a, b: float(out[a:b, :, 0][p2f[a:b] >= 0].mean())  # noqa: E731
    hi, lo = mean(top, top + third), mean(bottom + 1 - third, bottom + 1)
    print(f"sphere: mean top third {hi:.2f}, bottom third {lo:.2f} (0-255)")
    assert hi > lo + 20  # the light sits at image-up, y = -1 in camera coordinates
    assert lo >= 0.5 * 255 - 1e-9  # the ambient floor


def _two_sided_sheet(dtype):
    """One triangle listed with both windings: every vertex normal sums to exactly 0 (the coordinates are multiples of
    1/8, so each cross product is exact in either form and the two windings cancel).  Vertex 3 is in no face."""
    mesh = torch.tensor([[-0.5, -0.375, 2.0], [0.625, -0.25, 2.5], [-0.125, 0.5, 2.25], [9.0, 9.0, 9.0]], dtype=dtype)
    return mesh, np.array([[0, 1, 2], [0, 2, 1]])


def test_zero_normals_and_a_vertex_in_no_face_shade_to_half_the_texel():
    mesh, f = _two_sided_sheet(torch.float64)
    n = vertex_normals_reference(mesh, f)
    assert torch.equal(n, torch.zeros_like(n))  # the vertex in no face included
    cam = _cam(30.0, 30.0, 12.0, 10.0)
    c, zbuf, p2f = _shade_reference(mesh, f, cam, 20, 24)
    fg = p2f >= 0
    assert int(fg.sum()) > 60
    b_sum = 2 * c[..., 0][fg]  # c = 0.5 texel
    assert float((b_sum - 1).abs().max()) < 1e-12
    assert torch.equal(c[~fg], torch.ones_like(c[~fg]))
    assert bool((zbuf[~fg] == -1).all())


def test_the_texel_sum_is_kept_in_float32():
    mesh, f = _two_sided_sheet(torch.float32)
    cam = _cam(30.0, 30.0, 12.0, 10.0, dtype=torch.float32)
    out, p2f = shaded_mesh_reference(mesh, f, cam, torch.zeros(20, 24, 3))
    fg = p2f >= 0
    from exavatar_release_b200.mesh_render import _bary, _pix_ndc
    idx = torch.nonzero(fg.reshape(-1))[:, 0]
    x, y, z = _ndc(mesh, {"R": torch.eye(3), "t": torch.zeros(3), **cam}, 20, 24)
    fc = torch.as_tensor(f)[p2f.reshape(-1)[idx]]
    b, _ = _bary(_pix_ndc(24, 20, torch.float32, "cpu")[idx % 24], _pix_ndc(20, 24, torch.float32, "cpu")[idx // 24],
                 x[fc], y[fc], z[fc])
    texel = b[:, 0] + b[:, 1] + b[:, 2]
    assert bool((texel != 1).any())  # fp32 barycentrics do not sum to exactly 1
    want = (texel * 0.5) * 255
    assert torch.equal(out.reshape(-1, 3)[idx, 0], want)
    assert bool((out.reshape(-1, 3)[idx, 0] != 127.5).any())


def test_pytorch3d_normals_of_the_negated_mesh_are_D_n():
    m = make_human_mesh()
    v, f = m["targets"].double(), m["base_faces"]
    D = torch.tensor([-1.0, -1.0, 1.0], dtype=torch.float64)
    vn = v * D
    v0, v1, v2 = vn[f[:, 0]], vn[f[:, 1]], vn[f[:, 2]]
    fn = torch.cross(v2 - v1, v0 - v1, dim=1)  # pytorch3d's _compute_vertex_normals
    # negating x and y negates the cross products componentwise, exactly
    u0, u1, u2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    assert torch.equal(fn, torch.cross(u2 - u1, u0 - u1, dim=1) * D)
    n = torch.zeros_like(vn)
    for k in range(3):
        n = n.index_add(0, f[:, k], fn)
    n = torch.nn.functional.normalize(n, eps=1e-6, dim=1)
    err = float((n - D * vertex_normals_reference(v, f)).abs().max())
    print(f"pytorch3d-form normals vs D n: max abs {err:.2e}")
    assert err < 1e-12


@pytest.mark.parametrize("blend_ratio", [1.0, 0.5, 0.0, 0.3])
def test_composite_is_vis_py_in_numpy_and_the_background_passes_through(blend_ratio):
    v, f = _sphere(centre=(0.1, -0.05, 2.5))
    v = v.float()
    H, W = 40, 56
    cam = _cam(70.0, 75.0, 27.0, 21.0, dtype=torch.float32)
    g = torch.Generator().manual_seed(0)
    bkg = torch.rand(H, W, 3, generator=g) * 255
    bkg[0, 0] = torch.tensor([0.0, 255.0, 1e-30])
    out, p2f = shaded_mesh_reference(v, f, cam, bkg, blend_ratio)
    c, zbuf, p2f2 = _shade_reference(v, f, cam, H, W)
    assert torch.equal(p2f, p2f2)
    # vis.py:105-108 as numpy runs it on the host
    is_bkg = (zbuf <= 0).float().numpy()[:, :, None]
    render = c.numpy()
    b = bkg.numpy()
    fg = render * blend_ratio + b / 255 * (1 - blend_ratio)
    want = fg * (1 - is_bkg) * 255 + b * is_bkg
    assert want.dtype == np.float32
    assert np.array_equal(out.numpy(), want)
    bg = (p2f < 0).numpy()
    assert bg.sum() > 100 and (~bg).sum() > 100
    assert np.array_equal(out.numpy()[bg].view(np.uint32), b[bg].view(np.uint32))  # bit for bit


def test_argument_errors():
    with pytest.raises(RuntimeError, match="CUDA"):
        ShadedMeshRenderer(np.zeros((2, 3), np.int64), 4, device="cpu")
    with pytest.raises(ValueError, match="faces"):
        ShadedMeshRenderer(np.zeros((2, 4), np.int64), 4)
    r = ShadedMeshRenderer.__new__(ShadedMeshRenderer)  # the checks of a call run before anything touches a device
    r.num_vertices, r.num_faces, r.device = 5, 2, torch.device("meta")

    class _Cuda(torch.Tensor):
        @property
        def is_cuda(self):
            return True

    cu = lambda *s, dtype=torch.float32: torch.empty(*s, device="meta", dtype=dtype).as_subclass(_Cuda)  # noqa: E731
    cam = {"focal": cu(2), "princpt": cu(2)}
    with pytest.raises(RuntimeError, match="CUDA"):
        r(torch.zeros(5, 3), cam, cu(8, 8, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        r(cu(5, 3), cam, torch.zeros(8, 8, 3))
    cases = [((cu(2, 5, 3), cu(8, 8, 3), 1.0), "batch"), ((cu(6, 3), cu(8, 8, 3), 1.0), "mesh"),
             ((cu(5, 3), cu(8, 8, 4), 1.0), "bkg"), ((cu(5, 3), cu(8, 8), 1.0), "bkg"),
             ((cu(5, 3), cu(0, 8, 3), 1.0), "image size"),
             ((cu(5, 3, dtype=torch.float64), cu(8, 8, 3), 1.0), "float32"),
             ((cu(5, 3), cu(8, 8, 3, dtype=torch.float16), 1.0), "float32"),
             ((cu(5, 3), cu(8, 8, 3), float("nan")), "blend_ratio"), ((cu(5, 3), cu(8, 8, 3), float("inf")),
                                                                      "blend_ratio"),
             ((cu(5, 3), cu(8, 8, 3), cu(())), "blend_ratio"), ((cu(5, 3), cu(8, 8, 3), "1"), "blend_ratio")]
    for (mesh, bkg, blend), match in cases:
        with pytest.raises(ValueError, match=match):
            r(mesh, cam, bkg, blend)
    with pytest.raises(ValueError, match="focal"):
        r(cu(5, 3), {"princpt": cu(2)}, cu(8, 8, 3))
    with pytest.raises(RuntimeError, match="princpt"):
        r(cu(5, 3), {"focal": cu(2), "princpt": torch.zeros(2)}, cu(8, 8, 3))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def body(dev):
    """The synthetic SMPL-X body posed by SmplxRig.body_mesh in camera coordinates (animate.py:81-82), and its rig."""
    from exavatar_release_b200.smplx_rig import SmplxRig
    mesh = make_human_mesh()
    rig = SmplxRig(**make_smplx_model(mesh), device=dev)
    g = torch.Generator().manual_seed(11)
    ins = [torch.randn(rig.NB, generator=g), 0.01 * torch.randn(rig.J, 3, generator=g),
           0.1 * torch.randn(rig.J, 3, generator=g), torch.randn(rig.NE, generator=g)]
    ins = [t.to(dev) for t in ins]
    return {"rig": rig, "ins": ins, "faces": mesh["base_faces"]}


CASES = {
    # name: (trans, focal, princpt, (H, W))
    "body_512": ((0.02, -0.05, 0.0), (1100.0, 1080.0), (250.0, 262.0), (512, 512)),
    # the surface 0.1 m from the camera: faces far larger than MR_SMALL pixels, and faces across the camera plane
    "closeup": ((0.0, 0.03, -3.85), (500.0, 520.0), (270.0, 240.0), (512, 512)),
    "portrait_1080x1920": ((0.0, 0.03, 0.0), (3600.0, 3650.0), (545.0, 950.0), (1920, 1080)),
}


def _case(body, dev, name):
    trans, focal, princpt, shape = CASES[name]
    with torch.no_grad():
        mesh = body["rig"].body_mesh(*body["ins"], torch.tensor(trans, device=dev))
    cam = {"R": torch.eye(3, device=dev), "t": torch.zeros(3, device=dev),  # ignored, as render_mesh ignores them
           "focal": torch.tensor(focal, device=dev), "princpt": torch.tensor(princpt, device=dev)}
    bkg = torch.rand(shape + (3,), generator=torch.Generator().manual_seed(1)).to(dev) * 255
    return mesh, cam, bkg


def _op_faces(faces, mesh, cam, bkg, dev):
    """The op's per-pixel face, read through the op itself: the same triangles with unshared corners (vertex 3f + k is
    corner k of face f, so coverage is unchanged), and NaN normals on the faces whose index has bit j set turn exactly
    their pixels NaN.  One call per bit.  -1 where no face covers the pixel."""
    F_ = faces.shape[0]
    flat = ShadedMeshRenderer(np.arange(3 * F_).reshape(F_, 3), 3 * F_, device=dev)
    x = mesh[faces.to(dev).reshape(-1).long()].contiguous()
    focal, princpt = cam["focal"].float().contiguous(), cam["princpt"].float().contiguous()
    zero = torch.zeros(bkg.shape, device=dev)
    covered = None
    ids = torch.zeros(bkg.shape[:2], dtype=torch.int64, device=dev)
    fid = torch.arange(F_, device=dev)
    for j in range(-1, int(F_ - 1).bit_length()):
        nrm = torch.ones(F_, 3, 3, device=dev)
        nrm[(fid >> j) & 1 == 1 if j >= 0 else torch.ones(F_, dtype=torch.bool, device=dev)] = float("nan")
        nan = torch.isnan(flat._shade(x, nrm.reshape(-1, 3), focal, princpt, zero, 1.0)[..., 0])
        if j < 0:
            covered = nan  # every face NaN: the covered pixels
        else:
            ids |= nan.long() << j
    return torch.where(covered, ids, -1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_op_matches_the_restatement(dev, body, name):
    mesh, cam, bkg = _case(body, dev, name)
    faces = body["faces"]
    r = ShadedMeshRenderer(faces, mesh.shape[0], device=dev)
    out = r(mesh, cam, bkg)
    ref, ref_p2f = shaded_mesh_reference(mesh, faces, cam, bkg)
    p2f = _op_faces(faces, mesh, cam, bkg, dev)
    torch.cuda.synchronize()
    H, W = bkg.shape[:2]
    assert out.shape == (H, W, 3) and out.dtype == torch.float32 and not out.requires_grad
    covered = int((p2f >= 0).sum())
    print(f"{name}: {covered} covered pixels, {len(torch.unique(p2f[p2f >= 0]))} faces visible")
    assert covered > 5000
    assert torch.equal(p2f, ref_p2f)  # the per-pixel face
    _, zbuf, _ = _shade_reference(mesh, faces, cam, H, W, pix_to_face=ref_p2f)
    is_bkg = zbuf <= 0
    op_bkg = r(mesh, cam, torch.full_like(bkg, -1.0))[..., 0] == -1  # covered pixels give c 255 >= 0
    assert torch.equal(op_bkg, is_bkg)
    assert torch.equal(out[is_bkg].view(torch.int32), bkg[is_bkg].view(torch.int32))  # background bit for bit
    assert torch.equal(ref[is_bkg], bkg[is_bkg])
    # covered pixels against float64 on the op's faces.  The fp32 barycentrics of the coverage pass (pytorch3d's
    # arithmetic, which the op keeps) err by up to ~1e-4, and on the synthetic body, whose vertex normals turn sharply
    # from face to face, a few pixels move by more than 1e-3 for that reason alone: the float32 restatement shows the
    # same.  So the op is held to 1e-3 of float64 on all but 0.1 % of the covered pixels and to 1e-3 of the float32
    # restatement, which shares its barycentrics, everywhere.
    ref64, _ = shaded_mesh_reference(mesh.double(), faces, cam, bkg, pix_to_face=p2f)
    fg = ~is_bkg
    d64 = (out[fg].double() - ref64[fg]).abs()
    d32 = (out[fg] - ref[fg]).abs()
    r64 = (ref[fg].double() - ref64[fg]).abs()
    print(f"{name}: covered pixels max |op - float64| {float(d64.max()):.2e} ({int((d64 > 1e-3).sum())} of "
          f"{d64.numel()} values > 1e-3), max |float32 restatement - float64| {float(r64.max()):.2e}, "
          f"max |op - float32 restatement| {float(d32.max()):.2e} (0-255)")
    assert float(d32.max()) <= 1e-3
    assert int((d64 > 1e-3).sum()) <= 1e-3 * d64.numel()
    assert float(d64.max()) <= max(1e-3, 2 * float(r64.max()))
    if name == "closeup":
        x, y, z = _ndc(mesh.double(), {"R": torch.eye(3), "t": torch.zeros(3), **cam}, H, W)
        f = faces.to(dev).long()
        vis = torch.unique(p2f[p2f >= 0])
        s = 0.5 * min(H, W)
        area = ((x[f[vis]].amax(1) - x[f[vis]].amin(1)) * s) * ((y[f[vis]].amax(1) - y[f[vis]].amin(1)) * s)
        assert float(area.max()) > 4 * 32  # visible faces whose pixel box exceeds MR_SMALL
        zf = z[f]
        assert bool(((zf.amin(1) < 0) & (zf.amax(1) > 0)).any())  # faces across the camera plane


@pytest.mark.gpu
def test_two_calls_are_bit_identical_and_nothing_syncs(dev, body):
    mesh, cam, bkg = _case(body, dev, "closeup")
    r = ShadedMeshRenderer(body["faces"], mesh.shape[0], device=dev)
    a = r(mesh, cam, bkg, 0.6)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = r(mesh[None], cam, bkg, 0.6)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert bool((r._keys == -1).all())  # the key buffer is left clean


@pytest.mark.gpu
def test_the_texel_sum_is_kept_by_the_op(dev):
    mesh, f = _two_sided_sheet(torch.float32)
    cam = _cam(30.0, 30.0, 12.0, 10.0, dtype=torch.float32, device=dev)
    bkg = torch.zeros(20, 24, 3, device=dev)
    out = ShadedMeshRenderer(f, 4, device=dev)(mesh.to(dev), cam, bkg)
    ref, p2f = shaded_mesh_reference(mesh.to(dev), f, cam, bkg)
    assert torch.equal(out, ref)  # zero normals: c = 0.5 texel, bit for bit
    assert bool((out[p2f >= 0] != 127.5).any())


@pytest.mark.gpu
def test_captured_graph_replays_new_mesh_and_camera(dev, body):
    mesh, cam, bkg = _case(body, dev, "body_512")
    r = ShadedMeshRenderer(body["faces"], mesh.shape[0], device=dev)
    m = mesh.clone()
    focal, princpt = cam["focal"].clone(), cam["princpt"].clone()
    c = {"focal": focal, "princpt": princpt}
    r(m, c, bkg, 0.75)  # allocates the key buffer
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        r(m, c, bkg, 0.75)
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = r(m, c, bkg, 0.75)
    rig, ins = body["rig"], body["ins"]
    with torch.no_grad():
        pose = ins[2] + 0.05 * torch.randn(ins[2].shape, generator=torch.Generator().manual_seed(2)).to(dev)
        m.copy_(rig.body_mesh(ins[0], ins[1], pose, ins[3], torch.tensor([0.03, 0.0, 0.2], device=dev)))
        focal.copy_(torch.tensor([1000.0, 990.0], device=dev))
        princpt.copy_(torch.tensor([262.0, 249.0], device=dev))
    graph.replay()
    torch.cuda.synchronize()
    replayed = static.clone()
    eager = r(m, c, bkg, 0.75)
    torch.cuda.synchronize()
    assert torch.equal(replayed.view(torch.int32), eager.view(torch.int32))
    ref, _ = shaded_mesh_reference(m, body["faces"], c, bkg, 0.75)
    assert torch.equal(replayed == bkg, ref == bkg)  # the replay saw the new mesh and camera
    assert not torch.equal(replayed, r(mesh, cam, bkg, 0.75))


@pytest.mark.gpu
def test_face_render_is_unchanged_by_a_shaded_render(dev, body):
    """Both ops run mr_face_kernel on one device: a face render after a shaded render of another mesh equals one
    without it, and equals its float32 restatement."""
    from exavatar_release_b200.mesh_render import FaceMeshRenderer
    mesh, cam, bkg = _case(body, dev, "body_512")
    faces = body["faces"]
    vt, fu = np.full((1, 2), 0.5, np.float32), np.zeros((faces.shape[0], 3), np.int64)
    fr = FaceMeshRenderer(vt, fu, faces, mesh.shape[0], device=dev)
    tex = torch.rand(1, 3, 4, 4, generator=torch.Generator().manual_seed(3)).to(dev)
    full = dict(cam, R=cam["R"], t=cam["t"])
    a, pa = fr.render(tex, mesh, full, (512, 512))
    ShadedMeshRenderer(faces, mesh.shape[0], device=dev)(mesh * 1.01, cam, bkg)
    b, pb = fr.render(tex, mesh, full, (512, 512))
    _, pr = face_render_reference(tex, mesh, faces, vt, fu, full, (512, 512))
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(pa, pb) and torch.equal(pa.long(), pr)
