"""ExAvatar's SMPL-X rig (avatar/common/nets/module.py:517-518, 533, 537, 549) as the sync-free CUDA op `SmplxRig`
(csrc/smplx_rig.cu, b2r_rig_*).

These tests pin
  * without a device: `smplx_rig_reference` against tests/golden/rig.npz (written by the reference's own SMPL-X layer,
    lbs and module.py lines), the restated pytorch3d axis_angle_to_matrix against scipy, the matrix_to_axis_angle round trip,
    the two-level subdivision against make_human_mesh's, "contract at V then subdivide" against ExAvatar's "subdivide
    the tables then contract" in float64, the restatement's chains (the frame's pose equal to the 大 pose undoes the
    inverse-neutral chain), and the host and C ABI argument checks;
  * on the GPU at C4 size (P = 167 618): every output against float64 through ExAvatar's own route, the gradients of a
    seeded loss against float64 autograd, exact zeros, zero / tiny / near-pi poses, bit-identical runs, no host sync,
    forward + backward replayed from one CUDA graph with new inputs, NaN (not a fault) for non-topological parents through
    the C ABI, and the rig in front of nearest_rows, skin_gaussians, TrainingFrameRenderer and l1_ssim.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from util import assert_close, capture, golden_generator, no_host_sync
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.smplx_rig import (axis_angle_to_matrix, matrix_to_axis_angle, smplx_rig_reference,
                                             subdivision_tables, upsample, validate_model)
from exavatar_release_b200.synthetic import make_human_mesh, make_smplx_model

FAKE = 0x1000  # never dereferenced: validation fails before any launch
P_C4 = 167618
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _small():
    mesh = make_human_mesh(rings=7, segments=12)
    return mesh, make_smplx_model(mesh)


def _inputs(J, NB, NE, seed=0, scale=0.3, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    beta = torch.randn(NB, generator=g)
    jo = 0.01 * torch.randn(J, 3, generator=g)
    pose = scale * torch.randn(J, 3, generator=g)
    expr = torch.randn(NE, generator=g)
    return [t.to(device) for t in (beta, jo, pose, expr)]


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

def test_restatement_reproduces_the_reference_golden():
    """tests/golden/rig.npz was written by the reference's own SMPL-X layer, lbs and module.py lines."""
    gm = golden_generator("make_rig_golden")
    gold = np.load(os.path.join(G, "rig.npz"))
    _, model, ins, w = gm.rig_case()
    m = validate_model(**model)
    leaves = [ins["shape_param"].clone().requires_grad_(), ins["joint_offset"].clone().requires_grad_(),
              gm.full_pose(ins).clone().requires_grad_(), ins["expr"].clone().requires_grad_()]
    out = smplx_rig_reference(m, *leaves)
    for name in gm.OUTPUTS:
        ref = torch.from_numpy(gold[f"out:{name}"])
        x = getattr(out, name).detach()
        assert x.shape == ref.shape, name
        torch.testing.assert_close(x, ref, rtol=0, atol=1e-12 * max(1.0, float(ref.abs().max())), msg=name)
    ((out.mesh_neutral_pose * w[0]).sum() + (out.joint_mats * w[1]).sum() + (out.expr_offset * w[2]).sum()).backward()
    for name, leaf in zip(gm.GRADS, leaves):
        ref = torch.from_numpy(gold[f"grad:{name}"])
        assert float(ref.abs().max()) > 0, name
        torch.testing.assert_close(leaf.grad, ref, rtol=0, atol=1e-12 * max(1.0, float(ref.abs().max())), msg=name)


def test_axis_angle_to_matrix_matches_scipy():
    from scipy.spatial.transform import Rotation
    g = np.random.default_rng(0)
    axes = g.standard_normal((5, 3))
    axes /= np.linalg.norm(axes, axis=1, keepdims=True)
    cases = [np.zeros(3)] + [a * t for a in axes for t in (1e-7, math.pi - 1e-6, 3 * math.pi)]
    cases += list(g.standard_normal((64, 3)))
    aa = np.stack(cases)
    ours = axis_angle_to_matrix(torch.from_numpy(aa)).numpy()
    np.testing.assert_allclose(ours, Rotation.from_rotvec(aa).as_matrix(), rtol=0, atol=1e-12)


def test_matrix_to_axis_angle_round_trip():
    g = torch.Generator().manual_seed(1)
    aa = torch.randn(256, 3, generator=g, dtype=torch.float64)
    aa[:8] = aa[:8] / aa[:8].norm(dim=1, keepdim=True) * (math.pi - 1e-3)  # near pi: the other quaternion branches
    aa[8] = 0
    R = axis_angle_to_matrix(aa)
    back = matrix_to_axis_angle(R)
    torch.testing.assert_close(axis_angle_to_matrix(back), R, rtol=0, atol=1e-12)
    inside = aa.norm(dim=1) < math.pi - 1e-2
    torch.testing.assert_close(back[inside], aa[inside], rtol=0, atol=1e-12)


def test_subdivision_is_make_human_meshs():
    for kw in ({}, {"rings": 7, "segments": 12}):
        mesh = make_human_mesh(**kw)
        V = mesh["targets"].shape[0]
        sub1, sub2, V1, P = subdivision_tables(mesh["base_faces"].numpy(), V)
        assert P == mesh["verts"].shape[0]
        if not kw:
            assert (V, P) == (10478, P_C4)
        up = upsample(mesh["targets"].double(), sub1, sub2)
        # make_human_mesh subdivides the float64 base and rounds after: the same vertices in the same order, within one
        # fp32 ulp at |z| ~ 4.24 (4.8e-7); neighbouring vertices are millimetres apart
        torch.testing.assert_close(up, mesh["verts"].double(), rtol=0, atol=5e-7)


def test_contract_at_V_equals_exavatars_route_in_float64():
    mesh, model = _small()
    m = validate_model(**model)
    ins = [t.double() for t in _inputs(m["J"], m["NB"], m["NE"])]
    a = smplx_rig_reference(m, *ins, route="upsample")
    b = smplx_rig_reference(m, *ins, route="contract")
    for name in ("pose_offset", "expr_offset"):
        x, y = getattr(a, name), getattr(b, name)
        assert float(x.abs().max()) > 1e-3
        torch.testing.assert_close(x, y, rtol=0, atol=1e-12 * float(x.abs().max()), msg=name)


def test_reference_frame_at_the_neutral_pose_undoes_the_inverse_chain():
    # with no hand mean, the frame's chain at the 大 pose (jaw at zero) maps the zero-pose joints where the
    # inverse-neutral chain took them from: joint_mats = I
    mesh, model = _small()
    model = dict(model, pose_mean=torch.zeros_like(model["pose_mean"]))
    m = validate_model(**model)
    beta, jo, _, expr = (t.double() for t in _inputs(m["J"], m["NB"], m["NE"]))
    pose = torch.zeros(m["J"], 3, dtype=torch.float64)
    pose[1:1 + m["n_body"]] = m["neutral_body_pose"]
    out = smplx_rig_reference(m, beta, jo, pose, expr)
    torch.testing.assert_close(out.joint_mats, torch.eye(4, dtype=torch.float64).expand(m["J"], 4, 4), rtol=0,
                               atol=1e-12)


def test_host_validation_rejects_bad_models():
    mesh, model = _small()
    bad = list(model["parents"])
    bad[5], bad[6] = 6, 3
    with pytest.raises(ValueError, match="topological"):
        validate_model(**dict(model, parents=torch.tensor(bad)))
    J, V = 65, model["v_template"].shape[0]
    with pytest.raises(ValueError, match="joints"):
        validate_model(**dict(model, parents=torch.tensor([-1] + list(range(J - 1))),
                              J_regressor=torch.zeros(J, V), lbs_weights=torch.zeros(V, J)))
    with pytest.raises(ValueError, match="is_lhand"):
        validate_model(**dict(model, is_lhand=model["is_lhand"][:-1]))
    with pytest.raises(ValueError, match="posedirs"):
        validate_model(**dict(model, posedirs=model["posedirs"][:-9]))


def _fake_rig(**kw):
    r = L.B2RRig(V=100, V1=300, P=900, J=55, NB=100, NE=50, n_body=21)
    for name, _ in L.B2RRig._fields_[8:]:
        setattr(r, name, FAKE)
    for k, v in kw.items():
        setattr(r, k, v)
    return r


def test_cabi_symbols_and_argument_checks():
    lib = L.load()
    raw = C.CDLL(L.LIB_PATH)
    for name in ("b2r_rig_scratch_bytes", "b2r_rig_forward", "b2r_rig_backward"):
        assert hasattr(raw, name) and name in {s[0] for s in L.SYMBOLS}, name
    assert C.sizeof(L.B2RRig) == 32 + 8 * 26
    assert C.sizeof(L.B2RRigGrads) == 8 * 4
    nb = lib.b2r_rig_scratch_bytes(100, 55, 100, 50)
    assert nb > 0
    outs = [FAKE] * 6
    grads = L.B2RRigGrads(FAKE, FAKE, FAKE, FAKE)

    def fwd(r, scratch=FAKE, n=nb):
        return lib.b2r_rig_forward(C.byref(r), *outs, scratch, n, None)

    for kw in ({"J": 65}, {"J": 24}, {"NB": 129}, {"NE": 0}, {"V1": 99}, {"P": 299}, {"parents": None},
               {"mask": None}, {"full_pose": None}, {"rot_inv": None}, {"upT_w": None}):
        assert fwd(_fake_rig(**kw)) == -1, kw
        assert lib.b2r_rig_backward(C.byref(_fake_rig(**kw)), None, None, None, C.byref(grads), FAKE, nb, None) == -1
    assert fwd(_fake_rig(), scratch=None) == -1
    assert fwd(_fake_rig(), n=nb - 1) == -2
    assert lib.b2r_rig_backward(C.byref(_fake_rig()), None, None, None, C.byref(L.B2RRigGrads(FAKE, None, FAKE, FAKE)),
                                FAKE, nb, None) == -1


# ---------------------------------------------------------------------------------------------------------------------
# GPU (H100, C4 size)
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def c4():
    from exavatar_release_b200.smplx_rig import SmplxRig
    mesh = make_human_mesh()
    model = make_smplx_model(mesh)
    rig = SmplxRig(**model, device="cuda")
    return rig, {}


def _ref(rig, cache, ins, dtype=torch.float64):
    return rig.reference(*ins, dtype=dtype, device="cuda", cache=cache)


def _loss_weights(rig, seed=3):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g).cuda() for s in ((rig.P, 3), (rig.J, 4, 4), (rig.P, 3))]


def _loss(out, w, use=(True, True, True)):
    terms = [(out.mesh_neutral_pose * w[0]).sum(), (out.joint_mats * w[1]).sum(), (out.expr_offset * w[2]).sum()]
    return sum(t for t, u in zip(terms, use) if u)


def _leaves(ins, dtype=torch.float32):
    return [t.detach().to("cuda", dtype).requires_grad_(True) for t in ins]


@pytest.mark.gpu
def test_outputs_against_float64(c4):
    rig, cache = c4
    assert (rig.V, rig.P, rig.J) == (10478, P_C4, 55)
    ins = _inputs(rig.J, rig.NB, rig.NE, device="cuda")
    out = rig(*ins)
    ref = _ref(rig, cache, ins)
    for name in ("mesh_neutral_pose", "mesh_neutral_pose_wo_upsample", "joint_mats"):
        assert_close(getattr(out, name), getattr(ref, name), 1e-6, name)
    # the offsets are fp32 contractions of 486 and 50 signed terms (ExAvatar's own form rounds the same way)
    for name in ("pose_offset", "expr_offset"):
        assert_close(getattr(out, name), getattr(ref, name), 1e-5, name)
    assert float((out.pose_6d.double() - ref.pose_6d).abs().max()) <= 1e-6
    outside = ~rig.mask.bool()
    assert int(outside.sum()) > 0 and bool((out.pose_offset[outside] == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["random", "zero", "tiny", "near_pi"])
def test_gradients_against_float64_autograd(c4, case):
    rig, cache = c4
    beta, jo, pose, expr = _inputs(rig.J, rig.NB, rig.NE, seed=1)
    if case == "zero":
        pose = torch.zeros_like(pose)
    elif case == "tiny":
        pose = 1e-8 * torch.randn(pose.shape, generator=torch.Generator().manual_seed(2))
    elif case == "near_pi":
        pose = pose / pose.norm(dim=1, keepdim=True) * (math.pi - 1e-4)
    ins = [beta, jo, pose, expr]
    w = _loss_weights(rig)
    a = _leaves(ins)
    _loss(rig(*a), w).backward()
    b = _leaves(ins, torch.float64)
    _loss(_ref(rig, cache, b), [x.double() for x in w]).backward()
    for name, x, y in zip(("shape_param", "joint_offset", "full_pose", "expr"), a, b):
        assert bool(torch.isfinite(x.grad).all()), name
        assert_close(x.grad, y.grad, 1e-5, f"{case} d{name}")
    assert bool((a[1].grad[0] == 0).all())  # get_joint_offset zeroes the root


@pytest.mark.gpu
def test_pose_gradient_is_exactly_zero_without_joint_mats(c4):
    rig, _ = c4
    a = _leaves(_inputs(rig.J, rig.NB, rig.NE, seed=4))
    w = _loss_weights(rig)
    _loss(rig(*a), w, use=(True, False, False)).backward()
    assert bool((a[2].grad == 0).all())
    assert bool((a[3].grad == 0).all())
    assert float(a[0].grad.abs().max()) > 0 and float(a[1].grad.abs().max()) > 0


def _run(rig, ins, w):
    a = _leaves(ins)
    out = rig(*a)
    _loss(out, w).backward()
    return [t.clone() for t in out] + [x.grad.clone() for x in a]


@pytest.mark.gpu
def test_runs_are_bit_identical(c4):
    rig, _ = c4
    ins = _inputs(rig.J, rig.NB, rig.NE, seed=5)
    w = _loss_weights(rig)
    r1, r2 = _run(rig, ins, w), _run(rig, ins, w)
    for x, y in zip(r1, r2):
        assert torch.equal(x, y)


@pytest.mark.gpu
def test_no_host_sync(c4):
    rig, _ = c4
    ins = _inputs(rig.J, rig.NB, rig.NE, seed=6)
    w = _loss_weights(rig)
    a = _leaves(ins)
    with no_host_sync():
        _loss(rig(*a), w).backward()


@pytest.mark.gpu
def test_cuda_graph_replay_equals_eager(c4):
    rig, _ = c4
    w = _loss_weights(rig)
    static = [t.cuda() for t in _inputs(rig.J, rig.NB, rig.NE, seed=7)]
    leaves = [t.clone().requires_grad_(True) for t in static]

    def step():
        out = rig(*leaves)
        _loss(out, w).backward()
        return out

    def no_grads():
        for x in leaves:
            x.grad = None

    graph, out = capture(step, 2, reset=no_grads)
    for seed in (8, 9):
        new = _inputs(rig.J, rig.NB, rig.NE, seed=seed, device="cuda")
        with torch.no_grad():
            for x, n in zip(leaves, new):
                x.copy_(n)
        graph.replay()
        torch.cuda.synchronize()
        eager = _run(rig, new, w)
        for x, y in zip([t for t in out] + [x.grad for x in leaves], eager):
            assert torch.equal(x, y)


@pytest.mark.gpu
def test_non_topological_parents_give_nan_on_the_device(c4):
    """The C ABI cannot check `parents` on the host (a device pointer): the chain kernels find it and write NaN."""
    from exavatar_release_b200._lib import ptr as _ptr
    rig, _ = c4
    lib = L.load()
    ins = [rig._input(t, n, k) for t, n, k in zip(_inputs(rig.J, rig.NB, rig.NE, seed=13, device="cuda"),
                                                  (rig.NB, 3 * rig.J, 3 * rig.J, rig.NE), ("b", "j", "p", "e"))]
    bad = rig.parents.clone()
    bad[7] = 9
    st = rig._struct(ins)
    st.parents = _ptr(bad)
    f = lambda *s: torch.empty(s, dtype=torch.float32, device="cuda")  # noqa: E731
    outs = [f(rig.P, 3), f(rig.V, 3), f(rig.J, 4, 4), f(rig.P, 3), f(rig.P, 3), f(6 * rig.n_body)]
    scratch = torch.empty(rig.scratch_bytes, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    assert lib.b2r_rig_forward(C.byref(st), *[_ptr(o) for o in outs], _ptr(scratch), rig.scratch_bytes, stream) == 0
    grads = [f(n) for n in (rig.NB, 3 * rig.J, 3 * rig.J, rig.NE)]
    gjm = torch.ones(rig.J, 4, 4, device="cuda")
    assert lib.b2r_rig_backward(C.byref(st), None, _ptr(gjm), None, C.byref(L.B2RRigGrads(*[_ptr(g) for g in grads])),
                                _ptr(scratch), rig.scratch_bytes, stream) == 0
    torch.cuda.synchronize()
    assert bool(torch.isnan(outs[0]).all()) and bool(torch.isnan(outs[1]).all())
    assert bool(torch.isnan(outs[2][:, :3]).all())  # the constant last row (0, 0, 0, 1) stays
    assert bool(torch.isfinite(outs[4]).all()) and bool(torch.isfinite(outs[5]).all())
    assert bool(torch.isnan(grads[1][3:]).all()) and bool(torch.isnan(grads[2]).all())


@pytest.mark.gpu
def test_human_chain_through_the_renderer_against_the_fp32_restatement():
    """The rig in front of the human chain of a C4 frame: mean_3d / mean_3d_refined as module.py:528-539 builds them,
    nearest_rows against mesh_neutral_pose_wo_upsample, skin_gaussians with joint_mats and trans,
    TrainingFrameRenderer, l1_ssim of the five renders.  The op against the same chain with the rig as the fp32
    restatement (ExAvatar's route): the rows equal except at fp32 near-ties of the nearest-vertex distance, the loss and
    the gradients of shape_param, joint_offset, the pose, expr and trans within 1e-4 of their max plus what the
    renderer alone makes of fp32-sized position changes (below).  The two arms' mean_3d
    differ in fp32 rounding (a few 1e-7 m), so a query whose two nearest base vertices are that close to equidistant
    may pick either; such rows are checked to be ties and the restatement's chain is skinned with the op's rows, so the
    gradient comparison measures the rig, not the argmin."""
    from exavatar_release_b200 import SmplxRig, TrainingFrameRenderer
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.geometry import nearest_rows
    from exavatar_release_b200.losses import l1_ssim
    from exavatar_release_b200.plan import RENDERS
    from exavatar_release_b200.skinning import skin_gaussians
    from exavatar_release_b200.synthetic import WORKLOADS, Workload, make_population_assets, make_regs_labels
    dev = torch.device("cuda:0")
    c4 = WORKLOADS["C4"]
    H, W = c4.height, c4.width
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    R, tc = cam["R"], cam["t"]
    mesh = make_human_mesh()
    # the rig works in the posed frame skin_gaussians takes cam_R / cam_t from: the template there
    to_cam = lambda x: (x.double() @ R.cpu().double().t() + tc.cpu().double().view(1, 3)).float()  # noqa: E731
    model = make_smplx_model(dict(mesh, targets=to_cam(mesh["targets"])))
    rig = SmplxRig(**model, device=dev)
    P, J = rig.P, rig.J
    m = rig.model
    skinning_weight = upsample(m["lbs_weights"], m["sub1"], m["sub2"]).float().to(dev)  # init's upsampled weights
    labels = make_regs_labels(mesh)
    self_map = (labels["is_rhand"] | labels["is_lhand"] | labels["is_face"]).to(dev)
    mask = rig.mask.float()[:, None]
    wl = Workload("C4 with the synthetic mesh's Gaussians", H, W, P, c4.n_scene, 0, True)
    scene, human, refined = make_population_assets(wl, seed=0, device=dev)
    g = torch.Generator().manual_seed(11)
    mean_offset = (1e-3 * torch.randn(P, 3, generator=g)).to(dev)
    mean_offset_offset = (1e-3 * torch.randn(P, 3, generator=g)).to(dev)
    trans = 0.01 * torch.randn(3, generator=g)
    ins = _inputs(J, rig.NB, rig.NE, seed=12, scale=0.1) + [trans]
    target = torch.rand((3, H, W), generator=torch.Generator(device=dev).manual_seed(6), device=dev)
    bg = torch.tensor([0.3, 0.7, 0.2], device=dev)
    fr = TrainingFrameRenderer(scene["mean_3d"].shape[0], P, (H, W), dev, {"A": 8_000_000, "B": 8_000_000})
    cache, res, outs = {}, {}, {}
    # "perturbed": the op's chain with the canonical positions moved by 2e-7 m of seeded noise, the size of the two
    # arms' fp32 difference -- how far the renderer alone moves the gradients for such a change
    noise = (2e-7 * torch.randn(P, 3, generator=torch.Generator().manual_seed(14))).to(dev)
    for arm in ("op", "restatement", "perturbed"):
        leaves = _leaves(ins)
        out = rig.reference(*leaves[:4], dtype=torch.float32, device=dev, cache=cache) if arm == "restatement" \
            else rig(*leaves[:4])
        for t in (out.mesh_neutral_pose, out.joint_mats, out.expr_offset):
            t.retain_grad()
        outs[arm] = out
        mean_3d = out.mesh_neutral_pose + mean_offset + (noise if arm == "perturbed" else 0)  # module.py:528
        mean_3d_refined = mean_3d + mean_offset_offset * (1 - mask) + out.pose_offset  # 533-534
        mean_3d, mean_3d_refined = mean_3d + out.expr_offset, mean_3d_refined + out.expr_offset  # 537-539
        targets = out.mesh_neutral_pose_wo_upsample.contiguous()
        own_rows = nearest_rows(mean_3d.detach(), targets, self_map)
        rows = own_rows if arm == "op" else res["op"][1]
        posed, posed_r = skin_gaussians(mean_3d, mean_3d_refined, skinning_weight, rows, out.joint_mats, leaves[4],
                                        R, tc)
        o = fr(scene, dict(human, mean_3d=posed), dict(refined, mean_3d=posed_r), cam, bg)
        loss = 0
        for r in RENDERS:
            l1, ss = l1_ssim(o[r]["img"], target)
            loss = loss + 0.8 * l1 + 0.2 * (1 - ss)
        loss.backward()
        torch.cuda.synchronize()
        assert not fr.overflowed()
        res[arm] = (float(loss.detach()), own_rows.clone(), [x.grad.detach().clone() for x in leaves],
                    mean_3d.detach().double(), targets.detach().double())
    (lo, ro, go, qo, _), (lt, rt, gt, qt, tt) = res["op"], res["restatement"]
    gp = res["perturbed"][2]
    assert float((qo - qt).abs().max()) < 2e-6
    diff = torch.nonzero(ro != rt).reshape(-1)
    assert diff.numel() <= 1e-3 * P, diff.numel()
    if diff.numel():
        da = (qt[diff] - tt[ro[diff].long()]).norm(dim=1)
        db = (qt[diff] - tt[rt[diff].long()]).norm(dim=1)
        assert float((da - db).abs().max()) <= 1e-5, float((da - db).abs().max())  # ties within 10 um
    assert abs(lo - lt) <= 1e-4 * abs(lt), (lo, lt)
    # Split the difference of the two chains into the rig's share and the renderer's.  The gradients each chain sent
    # into its rig outputs (mesh_neutral_pose, joint_mats, expr_offset) differ, because the renders of positions that
    # differ in fp32 rounding differ; pulled back through float64, that difference bounds what the renderer
    # contributes.  The rig's share: the op chain's upstream gradients pulled back through the op stay within 1e-5 of
    # float64, and through the fp32 restatement within its own distance from float64.
    ups = {k: [o.mesh_neutral_pose.grad, o.joint_mats.grad, o.expr_offset.grad] for k, o in outs.items()
           if k != "perturbed"}

    def pull(fn, dtype, up):
        leaves = _leaves(ins[:4], dtype)
        o = fn(leaves)
        sum((t * u.to(dtype)).sum() for t, u in zip((o.mesh_neutral_pose, o.joint_mats, o.expr_offset), up)).backward()
        return [x.grad.double() for x in leaves]

    p_op = pull(lambda a: rig(*a), torch.float32, ups["op"])
    p32 = pull(lambda a: rig.reference(*a, dtype=torch.float32, device=dev, cache=cache), torch.float32, ups["op"])
    cache.clear()
    ref64 = lambda a: rig.reference(*a, dtype=torch.float64, device=dev, cache=cache)  # noqa: E731
    p64 = pull(ref64, torch.float64, ups["op"])
    p64_rt = pull(ref64, torch.float64, ups["restatement"])
    names = ("shape_param", "joint_offset", "full_pose", "expr", "trans")
    for i, (name, a, b) in enumerate(zip(names, go, gt)):
        scale = float(b.abs().max())
        err = float((a - b).abs().max())
        slack = 3 * float((gp[i] - a).abs().max())  # the renderer's sensitivity, measured on the op's chain
        if i < 4:
            s64 = float(p64[i].abs().max())
            assert float((p_op[i] - p64[i]).abs().max()) <= 1e-5 * s64, name
            slack = max(slack, float((p64[i] - p64_rt[i]).abs().max())) + float((p32[i] - p64[i]).abs().max())
        assert scale > 0 and err <= 1e-4 * scale + slack, (name, err, scale, slack)
