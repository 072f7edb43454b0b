"""The frame's SMPL-X body mesh of ExAvatar's get_smplx_outputs (avatar/main/model.py:37-58) as the sync-free CUDA op
`SmplxRig.body_mesh` (csrc/smplx_rig.cu, b2r_smplx_body_*).

These tests pin
  * without a device: `smplx_body_reference` against tests/golden/body.npz (written by the reference's own SMPLX layer
    and get_smplx_outputs), the restated batch_rodrigues against scipy and its |r + 1e-8| shift at and near r = 0, that
    the root row of joint_offset moves the mesh, and the C ABI's symbols and host-side argument checks;
  * on the GPU at C4 size (V = 10 478): the mesh in camera and world coordinates against float64 (within 1e-6 of its
    max), the gradients of a seeded loss against float64 autograd for random, zero, tiny and near-pi poses (within 2e-6
    of each gradient's max), bit-identical runs, no host sync, forward + backward replayed from one CUDA graph with new
    inputs, the mesh against the fp32 torch restatement of ExAvatar's route, and SmplxRig.__call__'s outputs unchanged
    by a body_mesh call.  The bounds are about 3x the worst errors measured on an H100 80GB HBM3 at 700 W (mesh 2.9e-7,
    gradients 5.7e-7).
"""
import ctypes as C
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

from util import workload_settings  # noqa: F401  (path setup)
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.smplx_rig import batch_rodrigues, smplx_body_reference, validate_model
from exavatar_release_b200.synthetic import make_human_mesh, make_smplx_model

FAKE = 0x1000  # never dereferenced: validation fails before any launch
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden_module():
    spec = importlib.util.spec_from_file_location("make_body_golden", os.path.join(G, "make_body_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _inputs(J, NB, NE, seed=0, scale=0.3, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    beta = torch.randn(NB, generator=g)
    jo = 0.01 * torch.randn(J, 3, generator=g)
    jo[0] += torch.tensor([0.02, -0.03, 0.01])  # the root row counts here
    pose = scale * torch.randn(J, 3, generator=g)
    expr = torch.randn(NE, generator=g)
    trans = torch.tensor([0.1, -0.2, 3.0]) + 0.05 * torch.randn(3, generator=g)
    return [t.to(device) for t in (beta, jo, pose, expr, trans)]


def _camera(device="cpu", dtype=torch.float32):
    a = torch.tensor([[0.3, -0.5, 0.2]], dtype=torch.float64)
    R = batch_rodrigues(a)[0]
    return R.to(device, dtype), torch.tensor([0.2, 0.1, -0.4], dtype=dtype, device=device)


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

def test_restatement_reproduces_the_reference_golden():
    """tests/golden/body.npz was written by the reference's own SMPLX layer and Model.get_smplx_outputs."""
    gm = _golden_module()
    gold = np.load(os.path.join(G, "body.npz"))
    _, model, ins, cam, w = gm.body_case()
    m = validate_model(**model)
    leaves = [ins["shape_param"].clone().requires_grad_(), ins["joint_offset"].clone().requires_grad_(),
              gm.full_pose(ins).clone().requires_grad_(), ins["expr"].clone().requires_grad_(),
              ins["trans"].clone().requires_grad_()]
    world = smplx_body_reference(m, *leaves, cam["R"], cam["t"])
    camera = smplx_body_reference(m, *leaves)
    for name, x in (("world", world), ("camera", camera)):
        ref = torch.from_numpy(gold[f"out:{name}"])
        assert x.shape == ref.shape, name
        torch.testing.assert_close(x.detach(), ref, rtol=0, atol=1e-12 * float(ref.abs().max()), msg=name)
    assert float((world - camera).detach().abs().max()) > 0.1  # the camera is not the identity
    ((world * w[0]).sum() + (camera * w[1]).sum()).backward()
    for name, leaf in zip(gm.GRADS, leaves):
        ref = torch.from_numpy(gold[f"grad:{name}"])
        assert float(ref.abs().max()) > 0, name
        torch.testing.assert_close(leaf.grad, ref, rtol=0, atol=1e-12 * float(ref.abs().max()), msg=name)
    assert float(ins["joint_offset"][0].abs().max()) > 0 and float(gold["grad:joint_offset"][0].__abs__().max()) > 0


def test_batch_rodrigues_matches_scipy_away_from_zero():
    from scipy.spatial.transform import Rotation
    g = np.random.default_rng(0)
    aa = g.standard_normal((128, 3))
    aa[:16] *= 1e-3 / np.linalg.norm(aa[:16], axis=1, keepdims=True)
    aa[16:24] *= (math.pi - 1e-4) / np.linalg.norm(aa[16:24], axis=1, keepdims=True)
    ours = batch_rodrigues(torch.from_numpy(aa)).numpy()
    # the shift makes |r / |r + 1e-8|| differ from 1 by up to sqrt(3) 1e-8 / |r|: sin(angle) times that stays < 2e-8
    np.testing.assert_allclose(ours, Rotation.from_rotvec(aa).as_matrix(), rtol=0, atol=2e-8)


def _rodrigues_literal(r):
    """smplx lbs.batch_rodrigues (lbs.py:329-345) for one vector, term by term in numpy float64."""
    angle = np.linalg.norm(r + 1e-8)
    d = r / angle
    K = np.array([[0, -d[2], d[1]], [d[2], 0, -d[0]], [-d[1], d[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def test_batch_rodrigues_shift_at_and_near_zero():
    cases = np.array([[0.0, 0.0, 0.0], [1e-9, -2e-9, 5e-10], [-1e-8, 3e-8, 0.0], [2e-6, 1e-6, -3e-6], [0.4, -0.1, 0.2]])
    ours = batch_rodrigues(torch.from_numpy(cases)).numpy()
    for r, R in zip(cases, ours):
        np.testing.assert_allclose(R, _rodrigues_literal(r), rtol=0, atol=1e-15)
    assert (ours[0] == np.eye(3)).all()  # angle = sqrt(3) 1e-8, d = 0: exactly I, not 0/0
    # without the shift the zero vector divides 0 by 0
    with np.errstate(invalid="ignore"):
        assert np.isnan(np.zeros(3) / np.linalg.norm(np.zeros(3))).all()
    # the Jacobian at 0 is finite: sin(angle) / angle ~ 1, so dR/dr_x is the generator [e_x]x
    r = torch.zeros(1, 3, dtype=torch.float64, requires_grad=True)
    jac = torch.autograd.functional.jacobian(lambda x: batch_rodrigues(x)[0], r)[:, :, 0, :]
    gen = torch.zeros(3, 3, 3, dtype=torch.float64)
    gen[2, 1, 0], gen[1, 2, 0], gen[0, 2, 1], gen[2, 0, 1], gen[1, 0, 2], gen[0, 1, 2] = 1, -1, 1, -1, 1, -1
    torch.testing.assert_close(jac, gen, rtol=0, atol=1e-14)


def test_root_joint_offset_moves_the_mesh():
    """get_smplx_outputs passes joint_offset raw (no get_joint_offset): its root row moves the joints and the mesh."""
    mesh = make_human_mesh(rings=7, segments=12)
    m = validate_model(**make_smplx_model(mesh))
    beta, jo, pose, expr, trans = (t.double() for t in _inputs(m["J"], m["NB"], m["NE"]))
    root = torch.zeros_like(jo)
    root[0] = torch.tensor([0.05, 0.0, -0.03], dtype=torch.float64)
    a = smplx_body_reference(m, beta, torch.zeros_like(jo), pose, expr, trans)
    b = smplx_body_reference(m, beta, root, pose, expr, trans)
    assert float((a - b).norm(dim=1).max()) > 1e-3


def _fake_rig(**kw):
    r = L.B2RRig(V=100, V1=300, P=900, J=55, NB=100, NE=50, n_body=21)
    for name, _ in L.B2RRig._fields_[8:]:
        setattr(r, name, FAKE)
    for k, v in kw.items():
        setattr(r, k, v)
    return r


def _fake_body(rig=None, **kw):
    b = L.B2RSmplxBody(rig=rig if rig is not None else _fake_rig())
    for name in ("pose_mean", "shape_param", "joint_offset", "full_pose", "expr", "trans", "cam_R", "cam_t"):
        setattr(b, name, FAKE)
    for k, v in kw.items():
        setattr(b, k, v)
    return b


def test_cabi_symbols_and_argument_checks():
    lib = L.load()
    raw = C.CDLL(L.LIB_PATH)
    for name in ("b2r_smplx_body_scratch_bytes", "b2r_smplx_body_forward", "b2r_smplx_body_backward"):
        assert hasattr(raw, name) and name in {s[0] for s in L.SYMBOLS}, name
    assert C.sizeof(L.B2RSmplxBody) == C.sizeof(L.B2RRig) + 8 * 8
    assert C.sizeof(L.B2RSmplxBodyGrads) == 8 * 5
    nb = lib.b2r_smplx_body_scratch_bytes(100, 55)
    assert nb > lib.b2r_smplx_body_scratch_bytes(10, 55) > 0
    grads = L.B2RSmplxBodyGrads(FAKE, FAKE, FAKE, FAKE, FAKE)

    def fwd(b, mesh=FAKE, scratch=FAKE, n=nb):
        return lib.b2r_smplx_body_forward(C.byref(b), mesh, scratch, n, None)

    def bwd(b, g=grads, scratch=FAKE, n=nb):
        return lib.b2r_smplx_body_backward(C.byref(b), None, C.byref(g), scratch, n, None)

    bad = [_fake_body(_fake_rig(**kw)) for kw in ({"J": 65}, {"NB": 129}, {"NE": 0}, {"V": 0}, {"parents": None},
                                                  {"posedirs_t": None}, {"jreg_vals": None}, {"jregT_rows": None})]
    bad += [_fake_body(**{k: None}) for k in ("pose_mean", "shape_param", "joint_offset", "full_pose", "expr", "trans",
                                              "cam_R", "cam_t")]
    for b in bad:
        assert fwd(b) == -1 and bwd(b) == -1
    ok = _fake_body()
    assert fwd(ok, mesh=None) == -1 and fwd(ok, scratch=None) == -1 and bwd(ok, scratch=None) == -1
    assert fwd(ok, n=nb - 1) == -2 and bwd(ok, n=nb - 1) == -2
    assert fwd(_fake_body(cam_R=None, cam_t=None), n=nb - 1) == -2  # no camera is valid: it reaches the size check
    for i in range(5):
        g = L.B2RSmplxBodyGrads(*[None if k == i else FAKE for k in range(5)])
        assert bwd(ok, g=g) == -1, i


def test_host_side_checks():
    from exavatar_release_b200.smplx_rig import SmplxRig
    with pytest.raises(RuntimeError, match="CUDA"):
        SmplxRig(**make_smplx_model(make_human_mesh(rings=7, segments=12)), device="cpu")


# ---------------------------------------------------------------------------------------------------------------------
# GPU (H100, C4 size)
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def c4():
    from exavatar_release_b200.smplx_rig import SmplxRig
    return SmplxRig(**make_smplx_model(make_human_mesh()), device="cuda")


def _leaves(ins, dtype=torch.float32):
    return [t.detach().to("cuda", dtype).requires_grad_(True) for t in ins]


def _weights(rig, seed=3):
    return torch.randn((rig.V, 3), generator=torch.Generator().manual_seed(seed)).cuda()


def _err(a, b):
    return float((a.double() - b.double()).abs().max()) / max(float(b.abs().max()), 1e-30)


def _close(a, b, rel, name):
    err = _err(a, b)
    print(f"{name}: max error {err:.3e} of max")
    assert err <= rel, f"{name}: max error {err:.3e} x max vs {rel:.0e}"


@pytest.mark.gpu
@pytest.mark.parametrize("world", [False, True])
def test_mesh_against_float64(c4, world):
    rig = c4
    assert (rig.V, rig.J) == (10478, 55)
    ins = _inputs(rig.J, rig.NB, rig.NE, device="cuda")
    cam = _camera("cuda") if world else (None, None)
    out = rig.body_mesh(*ins, *cam)
    ref = smplx_body_reference(rig.model, *[t.double() for t in ins], *[None if c is None else c.double() for c in cam])
    assert out.shape == (rig.V, 3) and out.dtype == torch.float32
    _close(out, ref, 1e-6, "world" if world else "camera")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["random", "zero", "tiny", "near_pi"])
def test_gradients_against_float64_autograd(c4, case):
    rig = c4
    beta, jo, pose, expr, trans = _inputs(rig.J, rig.NB, rig.NE, seed=1)
    if case == "zero":
        pose = torch.zeros_like(pose)
    elif case == "tiny":
        pose = 1e-8 * torch.randn(pose.shape, generator=torch.Generator().manual_seed(2))
    elif case == "near_pi":
        pose = pose / pose.norm(dim=1, keepdim=True) * (math.pi - 1e-4)
    ins = [beta, jo, pose, expr, trans]
    w = _weights(rig)
    R, t = _camera("cuda")
    a = _leaves(ins)
    (rig.body_mesh(*a, R, t) * w).sum().backward()
    b = _leaves(ins, torch.float64)
    (smplx_body_reference(rig.model, *b, R.double(), t.double()) * w.double()).sum().backward()
    for name, x, y in zip(("shape_param", "joint_offset", "full_pose", "expr", "trans"), a, b):
        assert bool(torch.isfinite(x.grad).all()), name
        assert float(y.grad.abs().max()) > 0, name
        _close(x.grad, y.grad, 2e-6, f"{case} d{name}")
    if case in ("random", "near_pi"):
        # the root row moves the mesh through the root's rotation about it: with an identity root (the zero pose) a
        # root offset shifts every joint alike and the rel transforms cancel it, so its gradient is then exactly 0
        assert float(a[1].grad[0].abs().max()) > 0


def _run(rig, ins, cam, w):
    a = _leaves(ins)
    mesh = rig.body_mesh(*a, *cam)
    (mesh * w).sum().backward()
    return [mesh.detach().clone()] + [x.grad.clone() for x in a]


@pytest.mark.gpu
def test_runs_are_bit_identical(c4):
    rig = c4
    ins = _inputs(rig.J, rig.NB, rig.NE, seed=5)
    w = _weights(rig)
    cam = _camera("cuda")
    r1, r2 = _run(rig, ins, cam, w), _run(rig, ins, cam, w)
    for x, y in zip(r1, r2):
        assert torch.equal(x, y)


@pytest.mark.gpu
def test_no_host_sync(c4):
    rig = c4
    w = _weights(rig)
    cam = _camera("cuda")
    a = _leaves(_inputs(rig.J, rig.NB, rig.NE, seed=6))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        (rig.body_mesh(*a, *cam) * w).sum().backward()
        (rig.body_mesh(*a) * w).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_cuda_graph_replay_equals_eager(c4):
    rig = c4
    w = _weights(rig)
    cam = _camera("cuda")
    leaves = [t.cuda().requires_grad_(True) for t in _inputs(rig.J, rig.NB, rig.NE, seed=7)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):  # warm-up on the capture stream
            for x in leaves:
                x.grad = None
            (rig.body_mesh(*leaves, *cam) * w).sum().backward()
    torch.cuda.current_stream().wait_stream(s)
    for x in leaves:
        x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = rig.body_mesh(*leaves, *cam)
        (out * w).sum().backward()
    for seed in (8, 9):
        new = _inputs(rig.J, rig.NB, rig.NE, seed=seed, device="cuda")
        with torch.no_grad():
            for x, n in zip(leaves, new):
                x.copy_(n)
        graph.replay()
        torch.cuda.synchronize()
        eager = _run(rig, new, cam, w)
        for x, y in zip([out] + [x.grad for x in leaves], eager):
            assert torch.equal(x, y)


@pytest.mark.gpu
def test_mesh_against_the_fp32_restatement_of_exavatars_route(c4):
    """ExAvatar's own fp32 route (one 150-coefficient einsum, the Python FK loop, torch.inverse) and the op round
    differently; both stay within 1e-6 of the float64 mesh's max (measured on an H100: 3.9e-7 and 2.9e-7), and they
    agree within 1e-6 of it (measured: 3.2e-7)."""
    rig = c4
    ins = _inputs(rig.J, rig.NB, rig.NE, seed=10, device="cuda")
    R, t = _camera("cuda")
    out = rig.body_mesh(*ins, R, t)
    ref32 = smplx_body_reference(rig.model, *ins, R, t, dtype=torch.float32)
    ref64 = smplx_body_reference(rig.model, *[x.double() for x in ins], R.double(), t.double())
    _close(ref32, ref64, 1e-6, "fp32 restatement vs float64")
    _close(out, ref32, 1e-6, "op vs fp32 restatement")


@pytest.mark.gpu
def test_rig_outputs_unchanged_by_a_body_mesh_call(c4):
    rig = c4
    beta, jo, pose, expr, trans = _inputs(rig.J, rig.NB, rig.NE, seed=11, device="cuda")
    before = [x.clone() for x in rig(beta, jo, pose, expr)]
    rig.body_mesh(beta, jo, pose, expr, trans, *_camera("cuda"))
    after = rig(beta, jo, pose, expr)
    for x, y in zip(before, after):
        assert torch.equal(x, y)
