"""The nearest-vertex rows and posed-mesh normals of ExAvatar's `HumanGaussian` (avatar/common/nets/module.py:541-546,
501-504) as sync-free ops: `geometry.nearest_rows` / `geometry.VertexNormals` (b2r_nearest_rows / b2r_vertex_normals).

These tests pin
  * without a device: the C ABI (symbols, scratch size, validation before any launch), `nearest_rows_reference` against
    scipy's float64 k-d tree (differences only at fp32 near-ties), its tie / NaN rules, `vertex_normals_reference`
    against a per-face numpy loop, the synthetic mesh, and the Python argument checks;
  * on the GPU: `nearest_rows` bit-equal to the reference at C4 size and on adversarial sets, the normals against
    float64, bit-identical runs, no host synchronisation, the chain nearest_rows -> skin_gaussians -> VertexNormals in
    one CUDA graph, and a C4 `TrainingFrameRenderer` frame posed with the op's rows.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from util import workload_settings  # noqa: F401  (path setup)
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.geometry import (VertexNormals, nearest_rows, nearest_rows_reference,
                                            vertex_normals_reference)
from exavatar_release_b200.synthetic import make_human_mesh

FAKE = 0x1000  # never dereferenced: validation fails before any launch


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

def test_symbols_and_scratch_size():
    lib = L.load()
    raw = C.CDLL(L.LIB_PATH)
    for name in ("b2r_nearest_scratch_bytes", "b2r_nearest_rows", "b2r_vertex_normals"):
        assert hasattr(raw, name), name
        assert name in {s[0] for s in L.SYMBOLS}, name
    last = 0
    for V in (1, 100, 10475, 100000):
        n = lib.b2r_nearest_scratch_bytes(167000, V)
        assert n >= 16 * V and n > last, V  # the sorted targets alone are 16 B each
        assert n == lib.b2r_nearest_scratch_bytes(1, V)  # sized from V only
        last = n


def test_validation_without_touching_cuda():
    lib = L.load()
    n0 = lib.b2r_launch_count()
    need = lib.b2r_nearest_scratch_bytes(64, 100)

    def nn(P=64, q=FAKE, V=100, t=FAKE, rows=FAKE, scratch=FAKE, nbytes=need):
        return lib.b2r_nearest_rows(P, q, V, t, None, rows, scratch, nbytes, None)

    for kw in ({"P": -1}, {"V": -1}, {"V": 0}, {"q": None}, {"t": None}, {"rows": None}, {"scratch": None},
               {"V": 1 << 29}):
        assert nn(**kw) == -1, kw
    assert nn(nbytes=need - 1) == -2
    assert nn(P=0, q=None, V=0, t=None, rows=None, scratch=None, nbytes=0) == 0  # nothing to do

    def vn(P=64, x=FAKE, f=FAKE, o=FAKE, e=FAKE, out=FAKE):
        return lib.b2r_vertex_normals(P, x, f, o, e, None, out, None)

    for kw in ({"P": -1}, {"x": None}, {"f": None}, {"o": None}, {"e": None}, {"out": None}):
        assert vn(**kw) == -1, kw
    assert vn(P=0, x=None, f=None, o=None, e=None, out=None) == 0
    assert lib.b2r_launch_count() == n0  # nothing was launched by any of the above


def _near_tie_only(q, t, got, ref_idx, rel=1e-6):
    """Indices may differ only where the float64 distances of the two candidates are within a few fp32 ulps."""
    q, t = q.double(), t.double()
    diff = (got.long() != ref_idx.long()).nonzero()[:, 0]
    da = ((q[diff] - t[got.long()[diff]]) ** 2).sum(1)
    db = ((q[diff] - t[ref_idx.long()[diff]]) ** 2).sum(1)
    assert bool(((da - db).abs() <= rel * db + 1e-30).all()), float(((da - db).abs() / db).max())
    return len(diff)


def _kdtree_rows(q, t):
    from scipy.spatial import cKDTree
    return torch.from_numpy(cKDTree(t.double().numpy()).query(q.double().numpy(), k=1)[1].astype(np.int64))


def test_reference_matches_a_float64_kdtree_on_the_mesh():
    m = make_human_mesh()
    q = m["queries"][::5]  # every fifth query keeps the CPU time down; all of them run on the GPU
    ref = nearest_rows_reference(q, m["targets"])
    n = _near_tie_only(q, m["targets"], ref, _kdtree_rows(q, m["targets"]))
    print(f"{n} near-ties of {len(q)}")
    assert n <= 1e-3 * len(q)


@pytest.mark.parametrize("seed", [0, 1])
def test_reference_matches_a_float64_kdtree_on_random_clouds(seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.rand(3000, 3, generator=g) * torch.tensor([1.0, 2.0, 0.5]) - 0.3
    q = torch.randn(5000, 3, generator=g)
    ref = nearest_rows_reference(q, t, target_chunk=700)  # several target chunks: the strict-< merge
    _near_tie_only(q, t, ref, _kdtree_rows(q, t))


def test_reference_ties_nan_and_self_map():
    t = torch.tensor([[1.0, 0, 0], [0, 0, 0], [1.0, 0, 0], [-1.0, 0, 0], [0, 0, 0]])
    q = torch.tensor([[0.0, 0, 0], [1.0, 0, 0], [0.0, 5.0, 0], [float("nan"), 0, 0], [float("inf"), 0, 0],
                      [1e30, 0, 0], [0.5, 0, 0]])
    # duplicates -> the lower index; (0,5,0) is equidistant from 1 and 4 (duplicates) -> 1; NaN / inf -> 0;
    # 1e30 overflows every distance to inf -> 0; 0.5 is equidistant from 0, 1, 2, 4 -> 0
    assert nearest_rows_reference(q, t, target_chunk=2).tolist() == [1, 0, 1, 0, 0, 0, 0]
    sm = torch.tensor([0, 1, 0, 1, 0, 0, 1], dtype=torch.bool)
    assert nearest_rows_reference(q, t, sm, target_chunk=2).tolist() == [1, 1, 1, 3, 0, 0, 6]


def _normals_loop(x, faces, flip):
    n = np.zeros_like(x)
    for a, b, c in faces:
        fn = np.cross(x[b] - x[a], x[c] - x[a])
        n[a] += fn
        n[b] += fn
        n[c] += fn
    n = n / np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-6)
    n[flip] *= -1
    return n


def test_vertex_normals_reference_matches_a_per_face_loop():
    g = np.random.default_rng(3)
    x = g.standard_normal((40, 3))
    faces = g.integers(0, 38, (90, 3))  # vertices 38 and 39 are in no face
    faces[5] = [7, 7, 12]                # a degenerate face: zero normal, listed twice for vertex 7
    flip = g.random(40) < 0.3
    flip[39] = True
    ref = vertex_normals_reference(torch.from_numpy(x), faces, torch.from_numpy(flip))
    assert ref.dtype == torch.float64
    np.testing.assert_allclose(ref.numpy(), _normals_loop(x, faces, flip), atol=1e-14)
    assert float(ref[38:].abs().max()) == 0.0


def test_synthetic_mesh():
    m = make_human_mesh()
    V, P = m["targets"].shape[0], m["verts"].shape[0]
    assert (V, P, m["faces"].shape[0]) == (10478, 167618, 335232)
    assert torch.equal(m["verts"][:V], m["targets"])  # the base vertices come first
    assert 0.25 < float(m["self_map"].float().mean()) < 0.35
    assert 0 < int(m["flip"].sum()) < 0.01 * P
    # outward winding: every face normal points away from the centre, except inside the cavity's dent
    x = m["verts"].double()
    f = m["faces"]
    fn = torch.cross(x[f[:, 1]] - x[f[:, 0]], x[f[:, 2]] - x[f[:, 0]], dim=1)
    out = (fn * (x[f].mean(1) - torch.tensor([0.0, 0.0, 4.24], dtype=torch.float64))).sum(1) > 0
    assert float(out.double().mean()) > 0.995
    assert float((m["queries"] - m["verts"]).abs().max()) < 0.01


class _Cuda(torch.Tensor):  # CUDA-agnostic stand-ins for the shape checks: they fail before any launch
    @property
    def is_cuda(self):
        return True


def _cu(*shape, dtype=torch.float32):
    return torch.empty(*shape, device="meta", dtype=dtype).as_subclass(_Cuda)


def test_argument_errors():
    with pytest.raises(RuntimeError, match="CUDA"):
        nearest_rows(torch.zeros(4, 3), torch.zeros(5, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        VertexNormals(np.zeros((2, 3), np.int64), 4, device="cpu")
    cases = [
        ((_cu(4, 2), _cu(5, 3)), {}, "queries"),
        ((_cu(4, 3), _cu(5, 3, dtype=torch.float64)), {}, "float32"),
        ((_cu(4, 3), _cu(0, 3)), {}, "no targets"),
        ((_cu(4, 3), _cu(5, 3)), {"self_map": _cu(5, dtype=torch.bool)}, "self_map"),
        ((_cu(4, 3), _cu(5, 3)), {"self_map": _cu(4, dtype=torch.float32)}, "self_map"),
    ]
    for args, kw, match in cases:
        with pytest.raises(ValueError, match=match):
            nearest_rows(*args, **kw)
    for faces in (np.zeros((2, 4), np.int64), np.zeros((2, 3), np.float32)):
        with pytest.raises(ValueError, match="faces"):
            VertexNormals(faces, 4, device="meta")


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def mesh():
    return make_human_mesh()


def _adversarial(name):
    g = torch.Generator().manual_seed(11)
    if name == "one_point":
        return torch.full((500, 3), 0.25).add_(torch.tensor([0.0, 1.0, 4.0])), torch.randn(4000, 3, generator=g)
    if name == "plane":
        t = torch.rand(3000, 3, generator=g)
        t[:, 2] = 1.5
        return t, torch.rand(4000, 3, generator=g) * 1.4 - 0.2
    if name == "far":  # 1 km to 1e20: finite distances, then distances that overflow to inf for every target
        t = torch.rand(2000, 3, generator=g)
        far = torch.randn(4000, 3, generator=g)
        far = far / far.norm(dim=1, keepdim=True) * torch.logspace(3, 20, 4000)[:, None]
        return t, far
    if name == "duplicates":
        base = torch.rand(700, 3, generator=g)
        t = base[torch.randint(0, 700, (3000,), generator=g)]
        return t, torch.cat([t[:1500], torch.rand(2500, 3, generator=g)])
    if name == "lattice":  # integer lattice, queries on cell boundaries and midpoints: exact ties everywhere
        ax = torch.arange(12, dtype=torch.float32)
        t = torch.stack(torch.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
        t = t[torch.randperm(len(t), generator=g)]
        q = torch.randint(-4, 30, (6000, 3), generator=g).float() * 0.5
        return t, q
    if name == "one_target":
        return torch.tensor([[0.3, -0.2, 4.0]]), torch.randn(3000, 3, generator=g)
    raise KeyError(name)


@pytest.mark.gpu
@pytest.mark.parametrize("self_map", ["mesh", "all", "none"])
def test_c4_rows_bit_equal_the_reference(dev, mesh, self_map):
    q, t = mesh["queries"].to(dev), mesh["targets"].to(dev)
    P = q.shape[0]
    sm = {"mesh": mesh["self_map"].to(dev), "all": torch.ones(P, dtype=torch.bool, device=dev), "none": None}[self_map]
    rows = nearest_rows(q, t, sm)
    ref = nearest_rows_reference(q, t, sm)
    torch.cuda.synchronize()
    assert rows.dtype == torch.int32 and rows.shape == (P,)
    assert torch.equal(rows, ref)
    if self_map == "all":
        assert torch.equal(rows.long().cpu(), torch.arange(P))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["one_point", "plane", "far", "duplicates", "lattice", "one_target"])
def test_adversarial_rows_bit_equal_the_reference(dev, name):
    t, q = _adversarial(name)
    q = torch.cat([q, torch.tensor([[float("nan"), 0.0, 0.0], [0.0, float("inf"), 1.0]])])
    q, t = q.to(dev), t.to(dev)
    sm = (torch.arange(q.shape[0], device=dev) % 7 == 3)
    sm[-2:] = False
    for m in (None, sm):
        rows = nearest_rows(q, t, m)
        ref = nearest_rows_reference(q, t, m)
        torch.cuda.synchronize()
        bad = (rows != ref).nonzero()[:5, 0].tolist()
        assert not bad, [(i, int(rows[i]), int(ref[i])) for i in bad]
        assert int(rows[-2]) == 0 and int(rows[-1]) == 0  # non-finite queries


@pytest.mark.gpu
def test_normals_match_float64(dev, mesh):
    vn = VertexNormals(mesh["faces"].numpy(), mesh["verts"].shape[0], flip=mesh["flip"].to(dev))
    got = vn(mesh["verts"].to(dev))
    torch.cuda.synchronize()
    assert not got.requires_grad
    x = mesh["verts"].double()
    ref = vertex_normals_reference(x, mesh["faces"], mesh["flip"])
    f = mesh["faces"]
    raw = torch.zeros_like(x)
    fn = torch.cross(x[f[:, 1]] - x[f[:, 0]], x[f[:, 2]] - x[f[:, 0]], dim=1)
    for c in range(3):
        raw.index_add_(0, f[:, c], fn)
    keep = raw.norm(dim=1) >= 1e-6
    err = (got.cpu().double() - ref).abs().max(dim=1).values
    print(f"normals: max |d| {float(err[keep].max()):.2e}, {int((~keep).sum())} vertices with |n| < 1e-6 excluded")
    # the excluded ones are the thin triangle fans around the two poles of the latitude-longitude mesh (1.7 %)
    assert int((~keep).sum()) <= 0.02 * len(keep)
    assert float(err[keep].max()) <= 1e-6
    plain = VertexNormals(mesh["faces"], len(x), device=dev)(mesh["verts"].to(dev))
    fl = mesh["flip"].to(dev)
    assert torch.equal(got[fl], -plain[fl]) and torch.equal(got[~fl], plain[~fl])


@pytest.mark.gpu
def test_two_runs_are_bit_identical(dev, mesh):
    q, t, sm = mesh["queries"].to(dev), mesh["targets"].to(dev), mesh["self_map"].to(dev)
    vn = VertexNormals(mesh["faces"], mesh["verts"].shape[0], flip=mesh["flip"].to(dev))
    x = mesh["verts"].to(dev)
    a = (nearest_rows(q, t, sm), vn(x))
    b = (nearest_rows(q, t, sm), vn(x))
    torch.cuda.synchronize()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def _rig_for(P, dev):
    from test_fused_skinning import _rig
    return _rig(P, 55, torch.float32, dev)


def _chain(q, qr, t, sm, table, A, tr, R, tc, vn):
    from exavatar_release_b200.skinning import skin_gaussians
    rows = nearest_rows(q, t, sm)
    posed, posed_r = skin_gaussians(q, qr, table, rows, A, tr, R, tc)
    return rows, posed, posed_r, vn(posed_r)


@pytest.mark.gpu
def test_neither_op_syncs(dev, mesh):
    q, t, sm = mesh["queries"].to(dev), mesh["targets"].to(dev), mesh["self_map"].to(dev)
    vn = VertexNormals(mesh["faces"], mesh["verts"].shape[0], flip=mesh["flip"].to(dev))
    x = mesh["verts"].to(dev)
    nearest_rows(q, t, sm), vn(x)  # loads the library and warms the allocator
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        nearest_rows(q, t, sm)
        nearest_rows(q, t, None)
        vn(x)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_chain_in_one_cuda_graph_equals_eager(dev, mesh):
    """nearest_rows -> skin_gaussians -> VertexNormals captured once; a replay with new queries, targets and rig
    inputs copied in equals an eager run on them, bit for bit."""
    from exavatar_release_b200.camera import look_at_cam_param
    P = mesh["verts"].shape[0]
    table, A, tr = _rig_for(P, dev)
    cam = look_at_cam_param(-6.0, (512, 512), device=dev)
    R, tc = cam["R"], cam["t"]
    q = mesh["queries"].to(dev).clone()
    qr = (q + 0.002).contiguous()
    t = mesh["targets"].to(dev).clone()
    sm = mesh["self_map"].to(dev)
    vn = VertexNormals(mesh["faces"], P, flip=mesh["flip"].to(dev))
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        _chain(q, qr, t, sm, table, A, tr, R, tc, vn)
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = _chain(q, qr, t, sm, table, A, tr, R, tc, vn)
    g = torch.Generator().manual_seed(23)
    with torch.no_grad():
        t.mul_(1.03).add_(0.01)  # a new neutral mesh
        q.copy_(mesh["verts"].to(dev) * 1.03 + 0.01 + 0.003 * torch.randn(P, 3, generator=g).to(dev))
        qr.copy_(q + 0.001 * torch.randn(P, 3, generator=g).to(dev))
    graph.replay()
    torch.cuda.synchronize()
    replayed = [x.clone() for x in static]
    eager = _chain(q, qr, t, sm, table, A, tr, R, tc, vn)
    torch.cuda.synchronize()
    for name, a, b in zip(("rows", "posed", "posed_refined", "normals"), replayed, eager):
        assert torch.equal(a, b), name
    assert torch.equal(replayed[0], nearest_rows_reference(q, t, sm))  # the replay saw the new mesh


@pytest.mark.gpu
def test_c4_frame_posed_with_op_rows_equals_reference_rows(dev, mesh):
    from exavatar_release_b200 import TrainingFrameRenderer
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.plan import RENDERS
    from exavatar_release_b200.skinning import skin_gaussians
    from exavatar_release_b200.synthetic import WORKLOADS, Workload, make_population_assets
    c4 = WORKLOADS["C4"]
    P = mesh["verts"].shape[0]
    wl = Workload("C4 with the synthetic mesh's Gaussians", c4.height, c4.width, P, c4.n_scene, 0, True)
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets(wl, seed=0, device=dev)
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    R, tc = cam["R"], cam["t"]
    to_cam = lambda x: (x.to(dev) @ R.t() + tc.view(1, 3)).contiguous()  # noqa: E731  (the skinning's frame)
    q, t = to_cam(mesh["queries"]), to_cam(mesh["targets"])
    qr = to_cam(mesh["queries"] + 0.002)
    sm = mesh["self_map"].to(dev)
    table, A, tr = _rig_for(P, dev)
    rows_op = nearest_rows(q, t, sm)
    rows_ref = nearest_rows_reference(q, t, sm)
    assert torch.equal(rows_op, rows_ref)
    bg = torch.tensor([0.3, 0.7, 0.2], device=dev)
    fr = TrainingFrameRenderer(scene["mean_3d"].shape[0], P, (H, W), dev, {"A": 8_000_000, "B": 8_000_000})
    imgs = {}
    for arm, rows in (("op", rows_op), ("reference", rows_ref)):
        posed, posed_r = skin_gaussians(q, qr, table, rows, A, tr, R, tc)
        out = fr(scene, dict(human, mean_3d=posed), dict(refined, mean_3d=posed_r), cam, bg)
        torch.cuda.synchronize()
        assert not fr.overflowed()
        imgs[arm] = {r: out[r]["img"].detach().clone() for r in RENDERS}
    for r in RENDERS:
        assert float(imgs["op"][r].abs().max()) > 0.1, r
        assert torch.equal(imgs["op"][r], imgs["reference"][r]), r
