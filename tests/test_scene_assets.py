"""ExAvatar's scene Gaussian assets (avatar/common/nets/module.py:253-272, SceneGaussian.forward) as the sync-free CUDA
op `scene_assets` (csrc/scene_assets.cu, b2r_scene_assets_*).

These tests pin
  * without a device: `scene_assets_reference` against tests/golden/scene.npz (written by the reference's own
    SceneGaussian.forward and eval_sh) at degrees 0..3, the restated rotation_6d_to_matrix (orthonormal, det +1) and
    matrix_to_quaternion (round trip through quaternion_to_matrix, ties of q_abs included), and the C ABI's symbols,
    struct sizes and argument checks;
  * on the GPU at C4 size (130 000 scene Gaussians, M = 16) and a small case: every output and the gradients of a
    seeded loss against float64, exact zeros above the degree, strided feature views, torch's extremes of sigmoid /
    exp and clamp_min's mask at equality, degenerate 6D rows, bit-identical runs, no host sync, one CUDA graph replayed
    across new inputs and degrees, NaN for a bad device degree, the host checks, and the op in front of
    TrainingFrameRenderer (shs mode) and GaussianRenderer (rgb mode).
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
from exavatar_release_b200.scene_assets import scene_assets_reference
from exavatar_release_b200.smplx_rig import (axis_angle_to_matrix, matrix_to_quaternion, quaternion_to_matrix,
                                             rotation_6d_to_matrix)

FAKE = 0x1000  # never dereferenced: validation fails before any launch
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
P_C4 = 130000


def _golden_module():
    spec = importlib.util.spec_from_file_location("make_scene_golden", os.path.join(G, "make_scene_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_restatement_reproduces_the_reference_golden(deg):
    gm = _golden_module()
    gold = np.load(os.path.join(G, "scene.npz"))
    params, cam, w = gm.scene_case()
    leaves = {k: v.clone().requires_grad_() for k, v in params.items()}
    out = scene_assets_reference(leaves["mean"], leaves["opacity"], leaves["scale"], leaves["rotation"],
                                 leaves["feature_dc"], leaves["feature_rest"], torch.tensor([float(deg)]), cam)
    for name in gm.OUTPUTS:
        ref = torch.from_numpy(gold[f"d{deg}:out:{name}"])
        torch.testing.assert_close(out[name].detach(), ref, rtol=0, atol=1e-12 * max(1.0, float(ref.abs().max())))
    sum((out[k] * wk).sum() for k, wk in zip(gm.OUTPUTS, w)).backward()
    for name in gm.PARAMS:
        ref = torch.from_numpy(gold[f"d{deg}:grad:{name}"])
        g = leaves[name].grad if leaves[name].grad is not None else torch.zeros_like(ref)
        torch.testing.assert_close(g, ref, rtol=0, atol=1e-12 * max(1.0, float(ref.abs().max())), msg=name)
    assert float(torch.from_numpy(gold[f"d{deg}:grad:feature_rest"]).abs().max()) > 0 or deg == 0


def test_rotation_6d_to_matrix_is_a_rotation():
    g = torch.Generator().manual_seed(3)
    d6 = torch.randn(4096, 6, generator=g, dtype=torch.float64)
    m = rotation_6d_to_matrix(d6)
    eye = torch.eye(3, dtype=torch.float64).expand(4096, 3, 3)
    torch.testing.assert_close(m @ m.transpose(1, 2), eye, rtol=0, atol=1e-12)
    torch.testing.assert_close(torch.linalg.det(m), torch.ones(4096, dtype=torch.float64), rtol=0, atol=1e-12)
    # the first row is a1's direction, the second lies in the plane of a1 and a2
    torch.testing.assert_close(m[:, 0], d6[:, :3] / d6[:, :3].norm(dim=1, keepdim=True), rtol=0, atol=1e-12)


def test_matrix_to_quaternion_round_trip():
    g = torch.Generator().manual_seed(5)
    aa = torch.randn(2048, 3, generator=g, dtype=torch.float64)
    half = [torch.zeros(1, 3, dtype=torch.float64)]  # the identity
    for ax in torch.eye(3, dtype=torch.float64):  # 180-degree turns about each axis
        half.append(math.pi * ax[None])
    # near-ties of q_abs: 180-degree turns about the diagonals of two axes (two equal q_abs), and just off them
    for axis in ((1.0, 1.0, 0.0), (1.0, 0.0, 1.0), (0.0, 1.0, 1.0), (1.0, 1.0, 1.0)):
        a = torch.tensor([axis], dtype=torch.float64)
        a = a / a.norm()
        for eps in (0.0, 1e-9, -1e-9, 1e-6):
            half.append((math.pi + eps) * a)
            half.append(math.pi * (a + eps * torch.tensor([[1.0, -2.0, 0.5]], dtype=torch.float64)))
    aa = torch.cat([aa] + half)
    R = axis_angle_to_matrix(aa)
    q = matrix_to_quaternion(R)
    torch.testing.assert_close(quaternion_to_matrix(q), R, rtol=0, atol=1e-12)
    assert bool((q[:, 0] >= 0).all())
    torch.testing.assert_close(q.norm(dim=1), torch.ones(len(q), dtype=torch.float64), rtol=0, atol=1e-12)


def _fake(**kw):
    s = L.B2RSceneAssets(P=1000, M=16, dc_stride=48, rest_stride=48)
    for name, _ in L.B2RSceneAssets._fields_[4:]:
        setattr(s, name, FAKE)
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def test_cabi_symbols_struct_sizes_and_argument_checks():
    lib = L.load()
    raw = C.CDLL(L.LIB_PATH)
    for name in ("b2r_scene_assets_forward", "b2r_scene_assets_backward"):
        assert hasattr(raw, name) and name in {s[0] for s in L.SYMBOLS}, name
    assert lib.b2r_sizeof(17) == C.sizeof(L.B2RSceneAssets) == 8 + 16 + 8 * 9
    assert lib.b2r_sizeof(18) == C.sizeof(L.B2RSceneAssetsGrads) == 8 * 12
    launches = lib.b2r_launch_count()
    outs = [FAKE] * 4

    def fwd(s, o=outs):
        return lib.b2r_scene_assets_forward(C.byref(s), *o, None)

    grads = L.B2RSceneAssetsGrads(*([FAKE] * 12))

    def bwd(s, g=grads):
        return lib.b2r_scene_assets_backward(C.byref(s), C.byref(g), None)

    for kw in ({"P": -1}, {"M": 0}, {"M": 17}, {"dc_stride": 2}, {"rest_stride": 44}, {"opacity_logit": None},
               {"log_scale": None}, {"rotation6d": None}, {"feature_dc": None}, {"feature_rest": None},
               {"cam_t": None}, {"mean": None}, {"active_sh_degree": None}):
        assert fwd(_fake(**kw)) == -1, kw
        assert bwd(_fake(**kw)) == -1, kw
    assert lib.b2r_scene_assets_forward(None, *outs, None) == -1
    assert fwd(_fake(), [FAKE, None, FAKE, FAKE]) == -1
    assert lib.b2r_scene_assets_backward(C.byref(_fake()), None, None) == -1
    for field in ("opacity", "scale", "dL_dlogit", "dL_dlog_scale", "dL_drotation6d", "dL_dfeature_dc",
                  "dL_dfeature_rest", "dL_dmean"):
        g = L.B2RSceneAssetsGrads(*([FAKE] * 12))
        setattr(g, field, None)
        assert bwd(_fake(), g) == -1, field
    # shs mode: no camera, no mean, no degree; d mean must then be absent
    shs = _fake(cam_R=None, cam_t=None, mean=None, active_sh_degree=None)
    assert bwd(shs) == -1
    assert lib.b2r_launch_count() == launches


def test_cabi_accepts_an_empty_scene_without_launching():
    lib = L.load()
    launches = lib.b2r_launch_count()
    s = L.B2RSceneAssets(P=0, M=16)
    assert lib.b2r_scene_assets_forward(C.byref(s), None, None, None, None, None) == 0
    assert lib.b2r_scene_assets_backward(C.byref(s), C.byref(L.B2RSceneAssetsGrads()), None) == 0
    assert lib.b2r_launch_count() == launches


def test_host_refuses_cpu_tensors():
    from exavatar_release_b200 import scene_assets
    z = lambda *s: torch.zeros(s)  # noqa: E731
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        scene_assets(z(4, 3), z(4, 1), z(4, 3), z(4, 6), z(4, 1, 3), z(4, 15, 3), 3)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

def _params(P, M=16, seed=0, device="cuda"):
    """Seeded float32 scene parameters; the first rows of the 6D rotation are the identity and 180-degree turns."""
    g = torch.Generator().manual_seed(100 + seed)
    rot = torch.randn(P, 6, generator=g)
    special = torch.tensor([[1.0, 0, 0, 0, 1, 0], [1.0, 0, 0, 0, -1, 0], [-1.0, 0, 0, 0, 1, 0], [-1.0, 0, 0, 0, -1, 0],
                            [1.0, 1.0, 0, -1.0, 1.0, 0], [0, 1.0, 1.0, 0, -1.0, 1.0]])
    rot[:min(P, len(special))] = special[:P]
    p = {"mean": torch.randn(P, 3, generator=g) * torch.tensor([1.5, 1.0, 1.5]),
         "opacity_logit": 2 * torch.randn(P, 1, generator=g),
         "log_scale": -4 + torch.randn(P, 3, generator=g),
         "rotation6d": rot,
         "feature_dc": torch.randn(P, 1, 3, generator=g),
         "feature_rest": 0.3 * torch.randn(P, M - 1, 3, generator=g)}
    return {k: v.to(device) for k, v in p.items()}


KEYS = ("mean", "opacity_logit", "log_scale", "rotation6d", "feature_dc", "feature_rest")


def _cam(device="cuda", yaw=10.0):
    from exavatar_release_b200.camera import look_at_cam_param
    return look_at_cam_param(yaw, (512, 512), device=device)


def _weights(P, seed=9):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g).cuda() for s in ((P, 1), (P, 3), (P, 4), (P, 3), (P, 3, 3))]


def _loss(out, w, rgb, q_by_matrix):
    """opacity, scale, the quaternion (through R(q) on the rows in q_by_matrix: sign-free) and the colour."""
    q = out["rotation"]
    keep = (~q_by_matrix).to(q.dtype)[:, None]
    loss = (out["opacity"] * w[0]).sum() + (out["scale"] * w[1]).sum() + (q * w[2] * keep).sum()
    loss = loss + (quaternion_to_matrix(q) * w[4] * (1 - keep)[:, :, None]).sum()
    if rgb:
        loss = loss + (out["rgb"] * w[3]).sum()
    else:
        loss = loss + (out["shs"][:, :4] * w[3][:, None, :]).sum() + (out["shs"][:, 4:] * 0.5).sum()
    return loss


def _close(a, b, rel, name):
    scale = float(b.detach().abs().max())
    err = float((a.double() - b.double()).abs().max())
    assert err <= rel * max(scale, 1e-30), f"{name}: max error {err:.3e} vs {rel:.0e} x max {scale:.3e}"


def _deg(d):
    return torch.tensor([float(d)], device="cuda")


@pytest.fixture(scope="module")
def cases():
    return {"c4": _params(P_C4), "small": _params(37, seed=1)}


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["c4", "small"])
@pytest.mark.parametrize("mode", ["shs", 0, 1, 2, 3])
def test_outputs_and_gradients_against_float64(cases, case, mode):
    from exavatar_release_b200 import scene_assets
    p = cases[case]
    P = p["mean"].shape[0]
    rgb = mode != "shs"
    cam = _cam() if rgb else None
    deg = _deg(mode if rgb else 3)
    leaves = {k: v.clone().requires_grad_() for k, v in p.items()}
    out = scene_assets(*[leaves[k] for k in KEYS], deg if rgb else 3, cam)
    l64 = {k: v.double().requires_grad_() for k, v in p.items()}
    cam64 = None if cam is None else {k: v.double() for k, v in cam.items()}
    ref = scene_assets_reference(*[l64[k] for k in KEYS], deg.double(), cam64)
    for name in ("opacity", "scale") + (("rgb",) if rgb else ("shs",)):
        _close(out[name], ref[name], 1e-6, name)
    assert out["mean_3d"] is leaves["mean"]
    # quaternion: where the f64 pick wins clearly and q0 is away from 0, q itself; elsewhere R(q), and q up to sign
    m64 = rotation_6d_to_matrix(l64["rotation6d"].detach())
    t = torch.stack([1 + m64[:, 0, 0] + m64[:, 1, 1] + m64[:, 2, 2], 1 + m64[:, 0, 0] - m64[:, 1, 1] - m64[:, 2, 2],
                     1 - m64[:, 0, 0] + m64[:, 1, 1] - m64[:, 2, 2], 1 - m64[:, 0, 0] - m64[:, 1, 1] + m64[:, 2, 2]], 1)
    qa = t.clamp_min(0).sqrt().sort(dim=1, descending=True).values
    q64, q32 = ref["rotation"].detach(), out["rotation"].detach().double()
    # the op evaluates the rotation in fp64 and rounds once, so even rows with a1 nearly parallel to a2 (where
    # Gram-Schmidt magnifies rounding by about 1 / sin(a1, a2)) are held to the flat bound
    clear = (qa[:, 0] - qa[:, 1] > 1e-5) & (q64[:, 0].abs() > 1e-6)
    assert float((q32[clear] - q64[clear]).abs().max()) <= 1e-6
    near0 = q64[:, 0].abs() < 1e-6
    assert int(near0.sum()) >= 3  # the 180-degree rows
    _close(quaternion_to_matrix(q32), quaternion_to_matrix(q64), 1e-6, "R(q)")
    sign = torch.where((q32 * q64).sum(1, keepdim=True) < 0, -1.0, 1.0).double()
    assert float((q32 * sign - q64).abs().max()) <= 1e-6
    # gradients of a seeded loss
    w = _weights(P)
    _loss(out, w, rgb, near0).backward()
    _loss(ref, [x.double() for x in w], rgb, near0).backward()
    for k in KEYS:
        a = leaves[k].grad
        if k == "mean" and (not rgb or mode == 0):
            assert a is None or bool((a == 0).all())  # the direction is not read at degree 0
            continue
        assert a is not None and bool(torch.isfinite(a).all()), k
        b = l64[k].grad
        if float(b.abs().max()) == 0:  # the coefficients above degree 0
            assert bool((a == 0).all()), k
            continue
        _close(a, b, 1e-5, f"{case}/{mode} d{k}")
    if rgb:
        nb = (mode + 1) ** 2
        assert bool((leaves["feature_rest"].grad[:, nb - 1:] == 0).all())  # exact zeros above the degree
        if mode > 0:
            assert float(leaves["feature_rest"].grad[:, :nb - 1].abs().max()) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("rgb", [False, True])
def test_strided_feature_views_equal_contiguous_copies(rgb):
    from exavatar_release_b200 import scene_assets
    p = _params(1000, seed=2)
    base = torch.cat([p["feature_dc"], p["feature_rest"]], 1)  # (P,16,3): init_from_point_cloud's layout
    w = _weights(1000)
    res = []
    for strided in (True, False):
        b = base.clone().requires_grad_()
        dc, rest = (b[:, :1], b[:, 1:]) if strided else (b[:, :1].detach().clone().requires_grad_(),
                                                           b[:, 1:].detach().clone().requires_grad_())
        leaves = {k: p[k].clone().requires_grad_() for k in ("mean", "opacity_logit", "log_scale", "rotation6d")}
        out = scene_assets(leaves["mean"], leaves["opacity_logit"], leaves["log_scale"], leaves["rotation6d"], dc, rest,
                           _deg(3) if rgb else 3, _cam() if rgb else None)
        _loss(out, w, rgb, torch.zeros(1000, dtype=torch.bool, device="cuda")).backward()
        gsh = b.grad if strided else torch.cat([dc.grad, rest.grad], 1)
        res.append([out["opacity"], out["scale"], out["rotation"], out["rgb" if rgb else "shs"], gsh] +
                   [leaves[k].grad if leaves[k].grad is not None else torch.zeros(1) for k in leaves])
    for x, y in zip(*res):
        assert torch.equal(x, y)
    # a view whose rows do not hold contiguous (k, c) blocks is copied, with the same result
    b = base.transpose(1, 2).contiguous().transpose(1, 2).requires_grad_()
    out = scene_assets(p["mean"], p["opacity_logit"], p["log_scale"], p["rotation6d"], b[:, :1], b[:, 1:],
                       _deg(3) if rgb else 3, _cam() if rgb else None)
    assert torch.equal(out["rgb" if rgb else "shs"], res[1][3])


@pytest.mark.gpu
def test_extreme_logits_and_log_scales_give_what_torch_gives():
    from exavatar_release_b200 import scene_assets
    vals = torch.tensor([-1e4, -104.0, -88.8, -30.0, -1e-8, 0.0, 1e-8, 15.0, 17.0, 88.0, 88.8, 100.0, 1e4,
                         float("inf"), -float("inf"), float("nan")], device="cuda")
    P = vals.numel()
    p = _params(P, seed=3)
    logit = vals[:, None].clone().requires_grad_()
    ls = vals[:, None].repeat(1, 3).clone().requires_grad_()
    out = scene_assets(p["mean"], logit, ls, p["rotation6d"], p["feature_dc"], p["feature_rest"], 3)
    g = torch.Generator().manual_seed(4)
    go, gs = torch.randn(P, 1, generator=g).cuda(), torch.randn(P, 3, generator=g).cuda()
    ((out["opacity"] * go).sum() + (out["scale"] * gs).sum()).backward()
    lt, lst = vals[:, None].clone().requires_grad_(), vals[:, None].repeat(1, 3).clone().requires_grad_()
    o_t, s_t = torch.sigmoid(lt), torch.exp(lst)
    ((o_t * go).sum() + (s_t * gs).sum()).backward()
    torch.testing.assert_close(out["opacity"], o_t, rtol=2e-7, atol=0, equal_nan=True)
    torch.testing.assert_close(out["scale"], s_t, rtol=2e-7, atol=0, equal_nan=True)
    torch.testing.assert_close(logit.grad, lt.grad, rtol=1e-6, atol=0, equal_nan=True)
    torch.testing.assert_close(ls.grad, lst.grad, rtol=1e-6, atol=0, equal_nan=True)
    ext = vals.abs() >= 88.8
    assert torch.equal(out["opacity"][ext].isnan(), o_t[ext].isnan())
    fin = ext & ~vals.isnan()
    assert torch.equal(out["opacity"][fin], o_t[fin]) and torch.equal(out["scale"][fin], s_t[fin])


@pytest.mark.gpu
def test_clamp_min_passes_the_gradient_at_equality():
    """At degree 0, rgb = clamp_min(C0 dc + 0.5, 0): a dc with fl(C0 dc) = -0.5 exactly puts the sum on the clamp."""
    from exavatar_release_b200 import scene_assets
    c0 = np.float32(0.28209479177387814)
    x = np.float32(-0.5) / c0
    cands = [np.nextafter(x, np.float32(-1)), x, np.nextafter(x, np.float32(1))]
    dc = next(float(c) for c in cands if np.float32(c0 * np.float32(c)) + np.float32(0.5) == 0)
    p = _params(4, seed=5)
    fdc = p["feature_dc"].clone()
    fdc[:, 0, :] = dc
    fdc[3, 0, 2] = dc * 1.001  # below the clamp: zero gradient
    leaf = fdc.clone().requires_grad_()
    out = scene_assets(p["mean"], p["opacity_logit"], p["log_scale"], p["rotation6d"], leaf, p["feature_rest"],
                       _deg(0), _cam())
    assert bool((out["rgb"] == 0).all())
    gw = torch.ones(4, 3, device="cuda")
    (out["rgb"] * gw).sum().backward()
    ref = fdc.clone().requires_grad_()
    r = scene_assets_reference(p["mean"], p["opacity_logit"], p["log_scale"], p["rotation6d"], ref, p["feature_rest"],
                               _deg(0), _cam())
    assert bool((r["rgb"] == 0).all())
    (r["rgb"] * gw).sum().backward()
    assert torch.equal(leaf.grad, ref.grad)
    assert float(leaf.grad[0, 0, 0]) == float(np.float32(c0)) and float(leaf.grad[3, 0, 2]) == 0.0


@pytest.mark.gpu
def test_degenerate_6d_rows_give_a_finite_forward():
    from exavatar_release_b200 import scene_assets
    p = _params(6, seed=6)
    p["rotation6d"] = torch.tensor([[0.0, 0, 0, 0.3, -1.0, 2.0], [1.0, 2.0, 3.0, 2.0, 4.0, 6.0],
                                    [1.0, 2.0, 3.0, -0.5, -1.0, -1.5], [0.0, 0, 0, 0, 0, 0],
                                    [1e-30, 0, 0, 0, 1e-30, 0], [3.0, 0, 0, 1.0, 0, 0]], device="cuda")
    for rgb in (False, True):
        out = scene_assets(*[p[k] for k in KEYS], _deg(3) if rgb else 3, _cam() if rgb else None)
        for k in ("opacity", "scale", "rotation", "rgb" if rgb else "shs"):
            assert bool(torch.isfinite(out[k]).all()), k


def _run(p, w, rgb, deg):
    from exavatar_release_b200 import scene_assets
    leaves = {k: v.clone().requires_grad_() for k, v in p.items()}
    out = scene_assets(*[leaves[k] for k in KEYS], deg if rgb else 3, _cam() if rgb else None)
    _loss(out, w, rgb, torch.zeros(p["mean"].shape[0], dtype=torch.bool, device="cuda")).backward()
    return [out[k].detach().clone() for k in ("opacity", "scale", "rotation", "rgb" if rgb else "shs")] + \
        [leaves[k].grad.clone() for k in KEYS if leaves[k].grad is not None]


@pytest.mark.gpu
@pytest.mark.parametrize("rgb", [False, True])
def test_runs_are_bit_identical(cases, rgb):
    p = cases["c4"]
    w = _weights(P_C4)
    a, b = _run(p, w, rgb, _deg(3)), _run(p, w, rgb, _deg(3))
    assert len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
def test_no_host_sync(cases):
    from exavatar_release_b200 import scene_assets
    p = cases["c4"]
    w = _weights(P_C4)
    cam, deg = _cam(), _deg(2)
    leaves = {k: v.clone().requires_grad_() for k, v in p.items()}
    mask = torch.zeros(P_C4, dtype=torch.bool, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for c in (cam, None):
            out = scene_assets(*[leaves[k] for k in KEYS], deg if c is not None else 2, c)
            _loss(out, w, c is not None, mask).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_cuda_graph_replay_across_inputs_and_degrees_equals_eager(cases):
    from exavatar_release_b200 import scene_assets
    p = cases["small"]
    P = p["mean"].shape[0]
    w = _weights(P)
    cam = _cam()
    deg = _deg(1)
    mask = torch.zeros(P, dtype=torch.bool, device="cuda")
    leaves = {k: v.clone().requires_grad_() for k, v in p.items()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            for x in leaves.values():
                x.grad = None
            _loss(scene_assets(*[leaves[k] for k in KEYS], deg, cam), w, True, mask).backward()
    torch.cuda.current_stream().wait_stream(s)
    for x in leaves.values():
        x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = scene_assets(*[leaves[k] for k in KEYS], deg, cam)
        _loss(out, w, True, mask).backward()
    for seed, d in ((11, 3.0), (12, 0.0), (13, 2.0)):
        new = _params(P, seed=seed)
        with torch.no_grad():
            for k in KEYS:
                leaves[k].copy_(new[k])
            deg.fill_(d)
        graph.replay()
        torch.cuda.synchronize()
        eager = _run(new, w, True, _deg(d))
        got = [out[k] for k in ("opacity", "scale", "rotation", "rgb")] + [leaves[k].grad for k in KEYS]
        assert len(got) == len(eager)
        for x, y in zip(got, eager):
            assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [4.0, -1.0, float("nan"), 3.0])
def test_a_bad_device_degree_gives_nan_not_a_fault(bad):
    from exavatar_release_b200 import scene_assets
    M = 9 if bad == 3.0 else 16  # degree 3 needs 16 coefficients
    p = _params(300, M=M, seed=7)
    leaves = {k: v.clone().requires_grad_() for k, v in p.items()}
    out = scene_assets(*[leaves[k] for k in KEYS], _deg(bad), _cam())
    (out["rgb"].nan_to_num(0).sum() + out["opacity"].sum() + out["rotation"].sum()).backward()
    torch.cuda.synchronize()
    assert bool(out["rgb"].isnan().all())
    assert bool(torch.isfinite(out["opacity"]).all()) and bool(torch.isfinite(out["rotation"]).all())
    assert bool(leaves["feature_rest"].grad.isnan().all()) and bool(leaves["mean"].grad.isnan().all())
    assert bool(torch.isfinite(leaves["rotation6d"].grad).all())


@pytest.mark.gpu
def test_host_argument_checks():
    from exavatar_release_b200 import scene_assets
    p = _params(10, seed=8)
    a = [p[k] for k in KEYS]
    cam = _cam()
    with pytest.raises(ValueError, match="1 <= M <= 16"):
        scene_assets(*a[:5], torch.zeros(10, 16, 3, device="cuda"), 3)
    with pytest.raises(ValueError, match="float32"):
        scene_assets(a[0], a[1].double(), *a[2:], 3)
    with pytest.raises(ValueError, match="rotation6d"):
        scene_assets(*a[:3], a[3][:, :4], *a[4:], 3)
    with pytest.raises(ValueError, match="feature_dc"):
        scene_assets(*a[:4], torch.zeros(10, 2, 3, device="cuda"), a[5], 3)
    with pytest.raises(ValueError, match="\\(P,3\\)"):
        scene_assets(a[0][:, :2], *a[1:], 3)
    with pytest.raises(RuntimeError, match="active_sh_degree"):
        scene_assets(*a, torch.tensor([3.0]), cam)
    with pytest.raises(ValueError, match="one-element"):
        scene_assets(*a, torch.zeros(2, device="cuda"), cam)
    with pytest.raises(ValueError, match="R must be"):
        scene_assets(*a, _deg(3), {"R": cam["R"][:2], "t": cam["t"]})
    with pytest.raises(RuntimeError, match="cam_param"):
        scene_assets(*a, _deg(3), {"R": cam["R"].cpu(), "t": cam["t"]})
    # M = 1: no feature_rest rows
    out = scene_assets(*a[:5], torch.zeros(10, 0, 3, device="cuda"), _deg(0), cam)
    ref = scene_assets_reference(*a[:5], torch.zeros(10, 0, 3, device="cuda"), _deg(0), cam)
    _close(out["rgb"], ref["rgb"], 1e-6, "M=1 rgb")


@pytest.mark.gpu
def test_training_frame_renderer_fed_the_op_equals_the_fp32_restatement():
    """C4: TrainingFrameRenderer(sh_coeffs=16) fed scene_assets (shs mode) against the same renderer fed the fp32
    restatement.  Images within 1e-4 max, gradients at the raw scene parameters within 1e-4 max with the renderer's
    threshold outliers bounded as tests/parity.py bounds them."""
    from parity import compare
    from exavatar_release_b200 import TrainingFrameRenderer, scene_assets
    from exavatar_release_b200.plan import RENDERS
    from exavatar_release_b200.synthetic import WORKLOADS, make_grad_image, make_population_assets
    dev = torch.device("cuda:0")
    wl = WORKLOADS["C4"]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets("C4", seed=0, device=dev)
    p = _params(scene["mean_3d"].shape[0], seed=9)
    p["mean"] = scene["mean_3d"]
    p["opacity_logit"] = torch.logit(scene["opacity"].clamp(1e-4, 1 - 1e-4))
    p["log_scale"] = torch.log(scene["scale"])
    cam = _cam(yaw=7.0)
    bg = torch.tensor([0.3, 0.7, 0.2], device=dev)
    gcol = {r: make_grad_image("C4", 90 + j, device=dev) for j, r in enumerate(RENDERS)}
    fr = TrainingFrameRenderer(p["mean"].shape[0], human["mean_3d"].shape[0], (H, W), dev,
                               {"A": 8_000_000, "B": 8_000_000}, sh_coeffs=16)
    res = {}
    for arm, fn in (("op", scene_assets), ("restatement", scene_assets_reference)):
        leaves = {k: v.detach().clone().requires_grad_() for k, v in p.items()}
        assets = fn(*[leaves[k] for k in KEYS], 3)
        hs = {k: v.detach().clone() for k, v in human.items()}
        rs = {k: v.detach().clone() for k, v in refined.items()}
        out = fr(assets, hs, rs, cam, bg)
        sum((out[r]["img"] * gcol[r]).sum() for r in RENDERS).backward()
        torch.cuda.synchronize()
        assert not fr.overflowed()
        res[arm] = ({r: out[r]["img"].detach().clone() for r in RENDERS}, {k: v.grad.clone() for k, v in leaves.items()})
    (io, go), (it, gt) = res["op"], res["restatement"]
    for r in RENDERS:
        compare("scene_assets/frame", f"img:{r}", io[r].cpu().numpy(), it[r].cpu().numpy(), kind="image")
    for k in KEYS:
        assert float(gt[k].abs().max()) > 0, k
        compare("scene_assets/frame", f"d{k}", go[k].cpu().numpy(), gt[k].cpu().numpy())


@pytest.mark.gpu
def test_gaussian_renderer_fed_the_op_in_rgb_mode_equals_the_fp32_restatement():
    from parity import compare
    from exavatar_release_b200 import GaussianRenderer, scene_assets
    from exavatar_release_b200.synthetic import make_grad_image, make_population_assets
    dev = torch.device("cuda:0")
    scene, _, _ = make_population_assets("C4", seed=1, device=dev)
    p = _params(scene["mean_3d"].shape[0], seed=10)
    p["mean"] = scene["mean_3d"]
    p["opacity_logit"] = torch.logit(scene["opacity"].clamp(1e-4, 1 - 1e-4))
    p["log_scale"] = torch.log(scene["scale"])
    cam = _cam(yaw=-5.0)
    gi = make_grad_image("C4", 95, device=dev)
    res = {}
    for arm, fn in (("op", scene_assets), ("restatement", scene_assets_reference)):
        leaves = {k: v.detach().clone().requires_grad_() for k, v in p.items()}
        assets = fn(*[leaves[k] for k in KEYS], _deg(3), cam)
        out = GaussianRenderer()(assets, (512, 512), cam)
        (out["img"] * gi).sum().backward()
        torch.cuda.synchronize()
        res[arm] = (out["img"].detach().clone(), {k: v.grad.clone() for k, v in leaves.items()})
    (io, go), (it, gt) = res["op"], res["restatement"]
    compare("scene_assets/rgb", "img", io.cpu().numpy(), it.cpu().numpy(), kind="image")
    for k in KEYS:
        assert float(gt[k].abs().max()) > 0, k
        compare("scene_assets/rgb", f"d{k}", go[k].cpu().numpy(), gt[k].cpu().numpy())
