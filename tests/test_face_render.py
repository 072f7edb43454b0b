"""ExAvatar's face render (avatar/main/model.py:170-175 -> MeshRenderer, avatar/common/nets/layer.py:23-68) as a sync-free
CUDA op: `mesh_render.FaceMeshRenderer` (b2r_mesh_render_forward / b2r_mesh_render_backward).

These tests pin
  * without a device: the C ABI (symbols, struct mirror, validation before any launch), hand-derived answers of
    `face_render_reference` (pixel placement, barycentrics, edges, depth order, skip rules, the uv convention, the
    background), its float64 gradient against finite differences, the Python argument checks and the synthetic mesh;
  * on the GPU: the op against the float32 reference (identical per-pixel face, image within 2e-6) at C4 size, on a
    close-up and at 1920x1080, its gradient against float64, bit-identical runs, no host synchronisation, forward +
    backward in one CUDA graph, and the chain skin_gaussians -> face render -> face composite -> l1_ssim.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from util import capture, no_host_sync
from util import dev  # noqa: F401
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.mesh_render import FaceMeshRenderer, _bary, _ndc, _pix_ndc, face_render_reference
from exavatar_release_b200.synthetic import make_face_mesh, make_human_mesh

FAKE = 0x1000  # never dereferenced: validation fails before any launch


def _cam(fx, fy, cx, cy, R=None, t=None, dtype=torch.float32):
    return {"R": torch.eye(3, dtype=dtype) if R is None else R, "t": torch.zeros(3, dtype=dtype) if t is None else t,
            "focal": torch.tensor([fx, fy], dtype=dtype), "princpt": torch.tensor([cx, cy], dtype=dtype)}


def _at_pixel(u, v, z, cam):
    """Camera-frame point (R = I, t = 0) that projects to image point (u, v) at depth z."""
    fx, fy = (float(a) for a in cam["focal"])
    cx, cy = (float(a) for a in cam["princpt"])
    return [(u - cx) * z / fx, (v - cy) * z / fy, z]


def _uv_const(F):
    return np.full((1, 2), 0.5, np.float32), np.zeros((F, 3), np.int64)


def _render(mesh, faces, cam, shape, tex=None, vertex_uv=None, face_uv=None, dtype=torch.float64):
    faces = np.asarray(faces, np.int64)
    if vertex_uv is None:
        vertex_uv, face_uv = _uv_const(len(faces))
    if tex is None:
        tex = torch.ones(4, 4, 4)
    return face_render_reference(tex.to(dtype), torch.as_tensor(mesh, dtype=dtype), faces, vertex_uv, face_uv,
                                 {k: v.to(dtype) for k, v in cam.items()}, shape)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the C ABI
# ---------------------------------------------------------------------------------------------------------------------

def test_symbols_and_struct_mirror():
    lib = L.load()
    raw = C.CDLL(L.LIB_PATH)
    for name in ("b2r_mesh_render_scratch_bytes", "b2r_mesh_render_forward", "b2r_mesh_render_backward"):
        assert hasattr(raw, name), name
        assert name in {s[0] for s in L.SYMBOLS}, name
    assert lib.b2r_mesh_render_scratch_bytes(9558) >= 9558 * (64 + 36)
    assert lib.b2r_mesh_render_scratch_bytes(0) > 0


def _struct(**kw):
    m = L.B2RMeshRender(V=100, F=50, Vt=100, C=4, tex_height=8, tex_width=8, height=16, width=16)
    for k in ("mesh", "faces", "vertex_uv", "face_uv", "texture", "cam_R", "cam_t", "focal", "princpt", "keys",
              "vf_offsets", "vf_entries"):
        setattr(m, k, FAKE)
    for k, v in kw.items():
        setattr(m, k, v)
    return m


def test_validation_without_touching_cuda():
    lib = L.load()
    n0 = lib.b2r_launch_count()
    need = lib.b2r_mesh_render_scratch_bytes(50)

    def fwd(m, img=FAKE, p2f=FAKE, scratch=FAKE, nbytes=need):
        return lib.b2r_mesh_render_forward(C.byref(m), img, p2f, scratch, nbytes, None)

    def bwd(m, p2f=FAKE, g=FAKE, d=FAKE, scratch=FAKE, nbytes=need):
        return lib.b2r_mesh_render_backward(C.byref(m), p2f, g, d, scratch, nbytes, None)

    bad = [{"C": 0}, {"C": 5}, {"V": -1}, {"F": -1}, {"height": 0}, {"width": -3}, {"width": 65536, "height": 32768},
           {"tex_height": 0}, {"Vt": 0}, {"V": 0}]
    bad += [{k: None} for k in ("mesh", "faces", "vertex_uv", "face_uv", "texture", "cam_R", "cam_t", "focal",
                                "princpt")]
    for kw in bad:
        assert fwd(_struct(**kw)) == -1, kw
        assert bwd(_struct(**kw)) == -1, kw
    assert lib.b2r_mesh_render_forward(None, FAKE, FAKE, FAKE, need, None) == -1
    assert lib.b2r_mesh_render_backward(None, FAKE, FAKE, FAKE, FAKE, need, None) == -1
    for kw in ({"img": None}, {"p2f": None}, {"scratch": None}):
        assert fwd(_struct(), **kw) == -1, kw
    assert fwd(_struct(keys=None)) == -1
    for kw in ({"p2f": None}, {"g": None}, {"d": None}, {"scratch": None}):
        assert bwd(_struct(), **kw) == -1, kw
    for k in ("vf_offsets", "vf_entries"):
        assert bwd(_struct(**{k: None})) == -1, k
    assert fwd(_struct(), nbytes=need - 1) == -2
    assert bwd(_struct(), nbytes=need - 1) == -2
    assert lib.b2r_launch_count() == n0  # nothing was launched by any of the above


# ---------------------------------------------------------------------------------------------------------------------
# CPU: known answers of the restatement
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(24, 16), (16, 24)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_tiny_triangle_covers_exactly_its_pixel(shape, dtype):
    H, W = shape
    cam = _cam(30.0, 41.0, 7.3, 9.6)  # fx != fy, off-centre principal point
    for r, c in ((0, 0), (5, 3), (H - 1, W - 1), (11, 13)):
        u, v = c + 0.5, r + 0.5
        tri = [_at_pixel(u - 0.3, v - 0.2, 2.0, cam), _at_pixel(u + 0.3, v - 0.2, 2.0, cam),
               _at_pixel(u, v + 0.3, 2.0, cam)]
        img, p2f = _render(tri, [[0, 1, 2]], cam, (H, W), dtype=dtype)
        want = torch.full((H, W), -1, dtype=torch.int64)
        want[r, c] = 0
        assert torch.equal(p2f, want), (r, c)
        assert img.shape == (1, 4, H, W)


def test_pixel_centres_are_half_integers():
    for n, other in ((7, 9), (9, 7), (8, 8)):
        s = min(n, other) / 2
        got = _pix_ndc(n, other, torch.float64, "cpu")
        want = (n / 2 - (torch.arange(n, dtype=torch.float64) + 0.5)) / s
        assert torch.allclose(got, want, atol=1e-15)


def test_barycentrics_affine_and_perspective_correct():
    cam = _cam(50.0, 60.0, 16.0, 12.0)
    H, W = 24, 32
    # fronto-parallel: b equals the screen-space barycentrics of (u, v)
    uvs = [(3.0, 2.0), (28.0, 5.0), (10.0, 21.0)]
    tri = torch.tensor([_at_pixel(u, v, 3.0, cam) for u, v in uvs], dtype=torch.float64)
    x, y, z = _ndc(tri, cam, H, W)
    pts = torch.tensor([(12.5, 9.5), (8.5, 6.5), (20.5, 7.5)], dtype=torch.float64)
    colx, rowy = _pix_ndc(W, H, torch.float64, "cpu"), _pix_ndc(H, W, torch.float64, "cpu")
    px, py = colx[(pts[:, 0] - 0.5).long()], rowy[(pts[:, 1] - 0.5).long()]
    b, pz = _bary(px, py, x[None].expand(3, 3), y[None].expand(3, 3), z[None].expand(3, 3))
    A = torch.tensor([[u for u, _ in uvs], [v for _, v in uvs], [1.0, 1.0, 1.0]], dtype=torch.float64)
    want = torch.linalg.solve(A, torch.stack([pts[:, 0], pts[:, 1], torch.ones(3, dtype=torch.float64)]))
    assert torch.allclose(b, want.t(), atol=1e-7)
    assert torch.allclose(pz, torch.full((3,), 3.0, dtype=torch.float64), atol=1e-7)
    # slanted: b are the 3-D barycentrics of where the pixel's ray meets the triangle's plane
    P = torch.tensor([_at_pixel(3.0, 2.0, 2.0, cam), _at_pixel(28.0, 5.0, 5.0, cam), _at_pixel(10.0, 21.0, 3.5, cam)],
                     dtype=torch.float64)
    x, y, z = _ndc(P, cam, H, W)
    b, pz = _bary(px, py, x[None].expand(3, 3), y[None].expand(3, 3), z[None].expand(3, 3))
    n = torch.linalg.cross(P[1] - P[0], P[2] - P[0])
    for i in range(3):
        d = torch.tensor([(float(pts[i, 0]) - 16.0) / 50.0, (float(pts[i, 1]) - 12.0) / 60.0, 1.0],
                         dtype=torch.float64)
        q = d * (n @ P[0]) / (n @ d)  # ray-plane intersection
        bq = torch.linalg.solve(P.t(), q)  # q = sum b_k P_k (b sums to 1 as q lies in the plane)
        assert torch.allclose(b[i], bq, atol=1e-9), (b[i], bq)
        assert abs(float(pz[i]) - float(q[2])) < 1e-9


def test_centre_on_a_shared_edge_is_covered_by_neither():
    # fx = fy = 2, principal point at the centre, z = 1 on a 4x4 image: x_ndc = -x and y_ndc = -y exactly, and
    # column 1's centres sit at x_ndc = 0.25, on the shared vertical edge x = -0.25
    cam = _cam(2.0, 2.0, 2.0, 2.0)
    mesh = [[-0.25, -3.0, 1.0], [-0.25, 3.0, 1.0], [-3.0, 0.0, 1.0], [3.0, 0.0, 1.0]]
    for dtype in (torch.float32, torch.float64):
        _, p2f = _render(mesh, [[0, 1, 2], [0, 3, 1]], cam, (4, 4), dtype=dtype)
        assert (p2f[:, 1] == -1).all(), p2f
        assert (p2f[:, 0] == 0).all() and (p2f[:, 2:] == 1).all(), p2f  # u = 2x + 2: column c holds x = (c - 1.5) / 2


def test_nearest_face_wins_and_ties_go_to_the_lower_index():
    cam = _cam(20.0, 20.0, 8.0, 8.0)
    big = lambda z: [_at_pixel(-4, -4, z, cam), _at_pixel(30, -4, z, cam), _at_pixel(-4, 30, z, cam)]  # noqa: E731
    mesh = big(3.0) + big(2.0) + big(2.0)
    for faces, want in (([[0, 1, 2], [3, 4, 5]], 1), ([[3, 4, 5], [0, 1, 2]], 0), ([[6, 7, 8], [3, 4, 5]], 0),
                        ([[0, 1, 2], [6, 7, 8], [3, 4, 5]], 1)):
        _, p2f = _render(mesh, faces, cam, (16, 16))
        assert int((p2f >= 0).sum()) > 100
        assert (p2f[p2f >= 0] == want).all(), (faces, p2f)


def test_skip_rules():
    cam = _cam(20.0, 20.0, 8.0, 8.0)
    tri = lambda z: [_at_pixel(1, 1, z, cam), _at_pixel(15, 2, z, cam), _at_pixel(3, 14, z, cam)]  # noqa: E731
    # behind the camera: the same NDC triangle with every z negated
    behind = [[-x, -y, -z] for x, y, z in tri(2.0)]
    _, p2f = _render(behind, [[0, 1, 2]], cam, (16, 16))
    assert (p2f == -1).all()
    _, p2f = _render(tri(2.0), [[0, 1, 2]], cam, (16, 16))
    assert (p2f == 0).sum() > 40
    # zero area: three collinear corners
    _, p2f = _render([_at_pixel(1, 1, 2.0, cam), _at_pixel(8, 8, 2.0, cam), _at_pixel(15, 15, 2.0, cam)],
                     [[0, 1, 2]], cam, (16, 16))
    assert (p2f == -1).all()
    # a face that straddles the camera plane: pixels with positive barycentrics but pz < 0 stay uncovered
    # corners given in NDC; v0 (behind the camera) is extreme in neither x nor y, so part of the wedge beyond it, where
    # all three corrected barycentrics are positive and pz is negative, lies inside the face's NDC box
    H = W = 16
    at_ndc = lambda xn, yn, z: [(0.5 * W - xn * 8 - 8) * z / 20, (0.5 * H - yn * 8 - 8) * z / 20, z]  # noqa: E731
    mesh = torch.tensor([at_ndc(0.2, -0.4, -1.0), at_ndc(-0.9, -0.9, 2.0), at_ndc(0.9, 0.9, 3.0)], dtype=torch.float64)
    _, p2f = _render(mesh, [[0, 1, 2]], cam, (H, W))
    x, y, z = _ndc(mesh, cam, H, W)
    colx, rowy = _pix_ndc(W, H, torch.float64, "cpu"), _pix_ndc(H, W, torch.float64, "cpu")
    px, py = colx.repeat(H), rowy.repeat_interleave(W)
    b, pz = _bary(px, py, x[None].expand(H * W, 3), y[None].expand(H * W, 3), z[None].expand(H * W, 3))
    inbox = (px <= x.max()) & (px >= x.min()) & (py <= y.max()) & (py >= y.min())
    pos = inbox & (b > 0).all(1)
    assert bool((pos & (pz < 0)).any())  # the rule has something to reject here
    assert torch.equal(p2f.reshape(-1) == 0, pos & ~(pz < 0))


def test_uv_convention_and_border_clamp():
    Ht, Wt = 5, 9
    tex = torch.zeros(3, Ht, Wt, dtype=torch.float64)
    tex[0] = torch.arange(Wt, dtype=torch.float64)[None]      # column index
    tex[1] = torch.arange(Ht, dtype=torch.float64)[:, None]   # row index of the map as given
    tex[2] = 7.0
    cam = _cam(20.0, 20.0, 8.0, 8.0)
    tri = [_at_pixel(-4, -4, 2.0, cam), _at_pixel(30, -4, 2.0, cam), _at_pixel(-4, 30, 2.0, cam)]
    for (a, b), want in (((0.25, 0.5), (2.0, 2.0)), ((0.0, 0.0), (0.0, 0.0)), ((0.625, 0.75), (5.0, 3.0)),
                         ((1.3, -0.2), (8.0, 0.0)), ((-1.0, 2.0), (0.0, 4.0))):
        vt = np.array([[a, b]], np.float32)
        img, p2f = _render(tri, [[0, 1, 2]], cam, (16, 16), tex=tex, vertex_uv=vt, face_uv=np.zeros((1, 3), np.int64))
        fg = p2f == 0
        assert int(fg.sum()) > 100
        assert torch.allclose(img[0, 0][fg], torch.tensor(want[0], dtype=torch.float64), atol=1e-12), (a, b)
        assert torch.allclose(img[0, 1][fg], torch.tensor(want[1], dtype=torch.float64), atol=1e-12), (a, b)
        assert torch.allclose(img[0, 2][fg], torch.tensor(7.0, dtype=torch.float64), atol=1e-12)
        assert (img[0][:, ~fg] == -1).all()  # background: -1 in every channel


def _fd_scene(dtype=torch.float64):
    cam = _cam(40.0, 46.0, 13.0, 11.0)
    cam["R"] = torch.tensor([[0.96, -0.28, 0.0], [0.28, 0.96, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float64)
    cam["t"] = torch.tensor([0.05, -0.02, 0.1], dtype=torch.float64)
    mesh = torch.tensor([[-0.6, -0.5, 2.2], [0.7, -0.4, 2.9], [-0.2, 0.6, 2.5], [0.6, 0.7, 3.2]], dtype=torch.float64)
    faces = np.array([[0, 1, 2], [2, 1, 3]])
    vt = np.array([[0.1, 0.2], [0.9, 0.15], [0.2, 0.85], [0.8, 0.9], [0.5, 0.5]], np.float32)
    fu = np.array([[0, 1, 2], [2, 1, 4]])
    g = torch.Generator().manual_seed(0)
    tex = torch.rand(4, 12, 10, generator=g, dtype=torch.float64)
    return cam, mesh.to(dtype), faces, vt, fu, tex


def test_reference_gradient_matches_finite_differences():
    H, W = 20, 26
    cam, mesh, faces, vt, fu, tex = _fd_scene()
    img, p2f = face_render_reference(tex, mesh, faces, vt, fu, cam, (H, W))
    # pixels away from the edges and from texel-cell boundaries
    x, y, z = _ndc(mesh, cam, H, W)
    fg = torch.nonzero(p2f.reshape(-1) >= 0)[:, 0]
    f = p2f.reshape(-1)[fg]
    fa = torch.as_tensor(faces)
    colx, rowy = _pix_ndc(W, H, torch.float64, "cpu"), _pix_ndc(H, W, torch.float64, "cpu")
    b, _ = _bary(colx[fg % W], rowy[fg // W], x[fa[f]], y[fa[f]], z[fa[f]])
    uvk = torch.stack([torch.from_numpy(vt[:, 0]).double(), 1 - torch.from_numpy(vt[:, 1]).double()], 1)
    uv = (b[:, :, None] * uvk[torch.as_tensor(fu)[f]]).sum(1)
    tx, ty = uv[:, 0] * 9, uv[:, 1] * 11
    far = lambda t: ((t - t.round()).abs() > 0.05)  # noqa: E731
    keep = (b > 0.05).all(1) & far(tx) & far(ty) & (uv > 0).all(1) & (uv < 1).all(1)
    assert int(keep.sum()) > 40
    wgt = torch.zeros(4, H * W, dtype=torch.float64)
    wgt[:, fg[keep]] = torch.randn(4, int(keep.sum()), generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    wgt = wgt.view(1, 4, H, W)

    def loss(m):
        return (face_render_reference(tex, m, faces, vt, fu, cam, (H, W), pix_to_face=p2f)[0] * wgt).sum()

    m = mesh.clone().requires_grad_()
    loss(m).backward()
    fd = torch.zeros_like(mesh)
    eps = 1e-6
    for i in range(mesh.shape[0]):
        for j in range(3):
            d = torch.zeros_like(mesh)
            d[i, j] = eps
            fd[i, j] = (loss(mesh + d) - loss(mesh - d)) / (2 * eps)
    err = float((m.grad - fd).abs().max() / fd.abs().max())
    print(f"reference gradient vs central differences: max rel {err:.2e}")
    assert err < 1e-6


def test_argument_errors():
    with pytest.raises(RuntimeError, match="CUDA"):
        FaceMeshRenderer(np.zeros((1, 2), np.float32), np.zeros((2, 3), np.int64), np.zeros((2, 3), np.int64), 4,
                         device="cpu")
    with pytest.raises(ValueError, match="face_uv"):
        FaceMeshRenderer(np.zeros((1, 2), np.float32), np.zeros((3, 3), np.int64), np.zeros((2, 3), np.int64), 4)
    with pytest.raises(ValueError, match="vertex_uv"):
        FaceMeshRenderer(np.zeros((1, 3), np.float32), np.zeros((2, 3), np.int64), np.zeros((2, 3), np.int64), 4)
    r = FaceMeshRenderer.__new__(FaceMeshRenderer)  # the checks of a call run before anything touches a device
    r.num_vertices, r.num_faces, r.device = 5, 2, torch.device("meta")

    class _Cuda(torch.Tensor):
        @property
        def is_cuda(self):
            return True

    cu = lambda *s: torch.empty(*s, device="meta").as_subclass(_Cuda)  # noqa: E731
    cam = {"R": cu(3, 3), "t": cu(3), "focal": cu(2), "princpt": cu(2)}
    with pytest.raises(RuntimeError, match="CUDA"):
        r(torch.zeros(4, 8, 8), cu(5, 3), cam, (8, 8))
    with pytest.raises(RuntimeError, match="CUDA"):
        r(cu(4, 8, 8), torch.zeros(5, 3), cam, (8, 8))
    tex_grad = torch.empty(4, 8, 8, device="meta", requires_grad=True).as_subclass(_Cuda)
    cases = [((tex_grad, cu(5, 3)), "requires grad"), ((cu(2, 4, 8, 8), cu(5, 3)), "batch"),
             ((cu(4, 8, 8), cu(2, 5, 3)), "batch"), ((cu(5, 8, 8), cu(5, 3)), "C in 1..4"),
             ((cu(1, 0, 8, 8), cu(5, 3)), "C in 1..4"), ((cu(4, 8, 8), cu(6, 3)), "mesh")]
    for (uvmap, mesh), match in cases:
        with pytest.raises(ValueError, match=match):
            r(uvmap, mesh, cam, (8, 8))


def test_synthetic_face_mesh():
    m = make_face_mesh()
    V, Fn = m["vertex_idx"].shape[0], m["faces"].shape[0]
    assert V == 5023 and 9000 <= Fn <= 11000
    assert int(m["vertex_idx"].min()) >= 0 and int(m["vertex_idx"].max()) < make_human_mesh()["verts"].shape[0]
    assert len(torch.unique(m["vertex_idx"])) == V
    assert int(m["faces"].min()) >= 0 and int(m["faces"].max()) < V
    Vt = m["vertex_uv"].shape[0]
    assert Vt != V and int(m["face_uv"].min()) >= 0 and int(m["face_uv"].max()) < Vt
    assert not torch.equal(m["face_uv"], m["faces"])
    assert float(m["vertex_uv"].min()) >= 0.0 and float(m["vertex_uv"].max()) <= 1.0
    tex = m["texture"]
    assert tex.shape == (4, 512, 512) and set(torch.unique(tex[3]).tolist()) == {0.0, 1.0}
    assert float(tex[:3].min()) >= 0.0 and float(tex[:3].max()) <= 1.0


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def face():
    m = make_face_mesh()
    m["verts"] = make_human_mesh()["verts"][m["vertex_idx"]].contiguous()
    return m


def _closeup_cam(dev, face):
    # the face mesh's centre 0.4 m in front of the camera: large triangles; fx != fy, off-centre principal point
    c = face["verts"].double().mean(0)
    return {"R": torch.eye(3, device=dev), "t": (torch.tensor([0.0, 0.0, 0.4], dtype=torch.float64) - c).float().to(dev),
            "focal": torch.tensor([900.0, 1000.0], device=dev), "princpt": torch.tensor([270.0, 180.0], device=dev)}


def _case(name, dev, face):
    from exavatar_release_b200.camera import look_at_cam_param
    if name == "c4_identity":
        return look_at_cam_param(0.0, (512, 512), device=dev), (512, 512)
    if name == "c4_yawed":
        return look_at_cam_param(-25.0, (512, 512), device=dev), (512, 512)
    if name == "closeup":
        return _closeup_cam(dev, face), (384, 512)
    if name == "fullhd":
        cam = look_at_cam_param(15.0, (1080, 1920), device=dev)
        cam["princpt"] = torch.tensor([930.0, 560.0], device=dev)
        return cam, (1080, 1920)
    raise KeyError(name)


def _renderer(face, dev):
    return FaceMeshRenderer(face["vertex_uv"], face["face_uv"], face["faces"], face["verts"].shape[0], device=dev)


def _ulps_from_one(a):
    return (a.double() - 1.0).abs() / float(np.spacing(np.float32(1.0)) / 2)  # ulps just below 1 are 2^-24


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c4_identity", "c4_yawed", "closeup", "fullhd"])
def test_op_matches_the_float32_reference(dev, face, name):
    cam, shape = _case(name, dev, face)
    r = _renderer(face, dev)
    tex = face["texture"].to(dev)[None]
    mesh = face["verts"].to(dev)[None]
    img, p2f = r.render(tex, mesh, cam, shape)
    ref, ref_p2f = face_render_reference(tex, mesh, face["faces"], face["vertex_uv"], face["face_uv"], cam, shape)
    torch.cuda.synchronize()
    assert img.shape == (1, 4) + shape and p2f.dtype == torch.int32
    covered = int((p2f >= 0).sum())
    nf = len(torch.unique(p2f[p2f >= 0]))
    print(f"{name}: {covered} covered pixels, {nf} faces visible")
    assert covered > 1000
    assert torch.equal(p2f.long(), ref_p2f)
    fg = p2f >= 0
    assert (img[0][:, ~fg] == -1).all()
    err = float((img[0][:, fg] - ref[0][:, fg]).abs().max())
    print(f"{name}: image max |op - reference| {err:.2e}")
    assert err <= 2e-6
    a, b = img[0, 3][fg] == 1, ref[0, 3][fg] == 1
    diff = a != b
    near = (_ulps_from_one(img[0, 3][fg]) <= 2) | (_ulps_from_one(ref[0, 3][fg]) <= 2)
    assert not bool((diff & ~near).any())


def _smooth_pixels(face, cam, shape, p2f, margin=1e-3):
    """(H,W) mask of the covered pixels whose float64 texel coordinates are at least `margin` from a texel-cell
    boundary and inside the border: grid_sample's derivative jumps across a cell boundary, so a pixel whose fp32 and
    fp64 uv fall in different cells has two different (both correct) gradients."""
    H, W = shape
    dev = p2f.device
    m = face["verts"].to(dev).double()
    x, y, z = _ndc(m, cam, H, W)
    flat = p2f.reshape(-1).long()
    fg = torch.nonzero(flat >= 0)[:, 0]
    f = flat[fg]
    fa, fu = face["faces"].to(dev), face["face_uv"].to(dev)
    colx, rowy = _pix_ndc(W, H, torch.float64, dev), _pix_ndc(H, W, torch.float64, dev)
    b, _ = _bary(colx[fg % W], rowy[fg // W], x[fa[f]], y[fa[f]], z[fa[f]])
    vt = face["vertex_uv"].to(dev).double()
    uvk = torch.stack([vt[:, 0], 1 - vt[:, 1]], 1)[fu[f]]
    uv = (b[:, :, None] * uvk).sum(1)
    Ht, Wt = face["texture"].shape[1:]
    t = torch.stack([uv[:, 0] * (Wt - 1), uv[:, 1] * (Ht - 1)], 1)
    ok = ((t - t.round()).abs() > margin).all(1) & (t > 0).all(1) & (t[:, 0] < Wt - 1) & (t[:, 1] < Ht - 1)
    keep = torch.zeros(H * W, dtype=torch.bool, device=dev)
    keep[fg[ok]] = True
    return keep.view(H, W)


def _grad_check(dev, face, name):
    cam, shape = _case(name, dev, face)
    r = _renderer(face, dev)
    tex = face["texture"].to(dev)[None]
    g = torch.Generator().manual_seed(3)
    G = torch.randn((1, 4) + shape, generator=g).to(dev)
    with torch.no_grad():
        _, p2f0 = r.render(tex, face["verts"].to(dev)[None], cam, shape)
        G *= _smooth_pixels(face, cam, shape, p2f0)
    m = face["verts"].to(dev).clone().requires_grad_()
    img, p2f = r.render(tex, m[None], cam, shape)
    (img * G).sum().backward()
    m64 = face["verts"].to(dev).double().requires_grad_()
    ref, _ = face_render_reference(tex, m64, face["faces"], face["vertex_uv"], face["face_uv"], cam, shape,
                                   pix_to_face=p2f)
    (ref * G.double()).sum().backward()
    return m.grad.double(), m64.grad


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c4_yawed", "closeup"])
def test_gradient_matches_float64(dev, face, name):
    got, ref = _grad_check(dev, face, name)
    scale = float(ref.abs().max())
    err = float((got - ref).abs().max()) / scale
    print(f"{name}: dL/dmesh max |op - float64| / max |float64| = {err:.2e} (max |grad| {scale:.3e})")
    assert scale > 0
    assert err <= 2e-3


@pytest.mark.gpu
def test_two_runs_are_bit_identical_and_nothing_syncs(dev, face):
    cam, shape = _case("closeup", dev, face)
    r = _renderer(face, dev)
    tex = face["texture"].to(dev)[None]
    G = torch.randn((1, 4) + shape, generator=torch.Generator().manual_seed(4)).to(dev)

    verts = face["verts"].to(dev)

    def run():
        m = verts.clone().requires_grad_()
        img, p2f = r.render(tex, m[None], cam, shape)
        (img * G).sum().backward()
        return img.detach(), p2f, m.grad

    run()
    torch.cuda.synchronize()
    a = run()
    with no_host_sync():
        b = run()
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.gpu
def test_forward_backward_in_one_cuda_graph_equals_eager(dev, face):
    cam, shape = _case("c4_yawed", dev, face)
    r = _renderer(face, dev)
    tex = face["texture"].to(dev)[None]
    G = torch.randn((1, 4) + shape, generator=torch.Generator().manual_seed(5)).to(dev)
    mesh = face["verts"].to(dev).clone()
    cam = {k: v.clone() for k, v in cam.items()}

    def step():
        m = mesh.clone().requires_grad_()
        img, p2f = r.render(tex, m[None], cam, shape)
        (img * G).sum().backward()
        return img.detach(), p2f, m.grad

    graph, static = capture(step, 1)
    from exavatar_release_b200.camera import look_at_cam_param
    new = look_at_cam_param(-10.0, shape, device=dev)
    with torch.no_grad():
        mesh.add_(0.004 * torch.randn(mesh.shape, generator=torch.Generator().manual_seed(6)).to(dev))
        for k in cam:
            cam[k].copy_(new[k])
        cam["focal"].mul_(torch.tensor([1.1, 1.05], device=dev))
    graph.replay()
    torch.cuda.synchronize()
    replayed = [x.clone() for x in static]
    eager = step()
    torch.cuda.synchronize()
    for nm, a, b in zip(("image", "pix_to_face", "grad"), replayed, eager):
        assert torch.equal(a, b), nm
    _, ref_p2f = face_render_reference(tex, mesh, face["faces"], face["vertex_uv"], face["face_uv"], cam, shape)
    assert torch.equal(replayed[1].long(), ref_p2f)  # the replay saw the new mesh and camera


@pytest.mark.gpu
def test_skinning_face_render_composite_l1_chain(dev, face):
    """skin_gaussians -> mean_3d[face_idx] -> face render -> ExAvatar's face composite -> l1_ssim(ssim=False); the
    gradient at the canonical positions against the same chain through the float64 reference."""
    from exavatar_release_b200.losses import l1_ssim, l1_ssim_reference
    from exavatar_release_b200.skinning import skin_gaussians
    cam, shape = _case("c4_yawed", dev, face)
    H, W = shape
    human = make_human_mesh()["verts"].to(dev)
    P, J = human.shape[0], 4
    g = torch.Generator().manual_seed(8)
    table = torch.rand(P, J, generator=g)
    table = (table / table.sum(1, keepdim=True)).to(dev)
    A = torch.eye(4).repeat(J, 1, 1)
    A[:, :3, 3] = 0.003 * torch.randn(J, 3, generator=g)
    A = A.to(dev)
    tr = torch.zeros(3, device=dev)
    idx = face["vertex_idx"].to(dev)
    r = _renderer(face, dev)
    tex = face["texture"].to(dev)[None]
    scene_img = torch.rand(1, 3, H, W, generator=g).to(dev)
    gt = torch.rand(1, 3, H, W, generator=g).to(dev)
    bbox = torch.tensor([[0.0, 0.0, float(W), float(H)]], device=dev)

    def composite(fr, is_face):
        return scene_img.to(fr.dtype) * (1 - is_face) + fr[:, :3] * is_face

    xyz = human.clone().requires_grad_()
    posed, _ = skin_gaussians(xyz, None, table, None, A, tr)
    fr, p2f = r.render(tex, posed[idx][None], cam, shape)
    is_face = ((fr[:, :3] != -1) * (fr[:, 3:] == 1)).float().detach()
    is_face = is_face * _smooth_pixels(dict(face, verts=posed[idx].detach()), cam, shape, p2f)  # see _smooth_pixels
    assert float(is_face.sum()) > 300
    l1, _ = l1_ssim(composite(fr, is_face), gt, bbox, ssim=False)
    l1.backward()
    xyz64 = human.clone().requires_grad_()
    posed64, _ = skin_gaussians(xyz64, None, table, None, A, tr)
    fr64, _ = face_render_reference(tex, posed64[idx].double(), face["faces"], face["vertex_uv"], face["face_uv"],
                                    cam, shape, pix_to_face=p2f)
    l1r, _ = l1_ssim_reference(composite(fr64, is_face.double()), gt, bbox, ssim=False)
    l1r.backward()
    torch.cuda.synchronize()
    assert abs(float(l1) - float(l1r)) <= 1e-6
    ref = xyz64.grad.double()
    scale = float(ref.abs().max())
    err = float((xyz.grad.double() - ref).abs().max()) / scale
    print(f"chain: dL/dxyz max |op - reference| / max |reference| = {err:.2e}")
    assert scale > 0 and err <= 2e-3
    assert float(xyz.grad[~torch.isin(torch.arange(P, device=dev), idx)].abs().max()) == 0.0
