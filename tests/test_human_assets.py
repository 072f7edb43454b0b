"""ExAvatar's SMPL-X pose decode (SMPLXParamDict.forward, module.py:673-684) and HumanGaussian's geometry and colour code
around its networks (module.py:524-539, 561-565, model.py:92-96) as the sync-free CUDA ops `decode_smplx_pose` and
`HumanAssets` (csrc/smplx_pose.cu, csrc/human_assets.cu).

These tests pin
  * without a device: the float64 restatements against tests/golden/human_assets.npz (written by the reference's own
    lines), and the C ABI's symbols, struct sizes and argument checks;
  * on the GPU: the decode at every fixture row and the geometry / colours at C4 size (P = 167 618) against float64,
    outputs and gradients; the geometry and colour forwards bit-identical to ExAvatar's fp32 torch expressions;
    bit-identical runs; no host sync through decode -> SmplxRig -> geometry -> nearest_rows -> skin_gaussians ->
    colours, forward and backward; a CUDA graph replayed after in-place parameter updates; strided geo views, P off
    the block size and P = 0; the warm-up clamp's gradient mask.
"""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

from util import workload_settings  # noqa: F401  (path setup)
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.human_assets import (POSE_KEYS, constant_rotation_reference, decode_smplx_pose_reference,
                                                human_colors_reference, human_geometry_reference)

FAKE = 0x1000  # never dereferenced: validation fails before any launch
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
P_C4 = 167618


def _golden_module():
    spec = importlib.util.spec_from_file_location("make_human_assets_golden",
                                                  os.path.join(G, "make_human_assets_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _fin(t):
    return torch.where(torch.isfinite(t), t, torch.zeros_like(t))


def _geometry_inputs(inp):
    """The ops' inputs from a geometry_case: mask, the rig's already-masked pose offset, expr_offset (module.py:537)."""
    mask = ((inp["is_rhand"] + inp["is_lhand"] + inp["is_face_expr"]) > 0)
    pose_offset = inp["pose_offset"] * mask[:, None].to(inp["pose_offset"].dtype)
    return mask, pose_offset


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

def test_pose_restatement_reproduces_the_reference_golden():
    gm = _golden_module()
    gold = np.load(os.path.join(G, "human_assets.npz"))
    params, w = gm.pose_case()
    leaves = {k: v.clone().requires_grad_() for k, v in params.items()}
    out = decode_smplx_pose_reference(leaves)
    sum((out[k] * w[k]).sum() for k in POSE_KEYS).backward()
    for k in POSE_KEYS:
        for what, got in (("out", out[k].detach()), ("grad", leaves[k].grad)):
            ref = torch.from_numpy(gold[f"pose:{what}:{k}"])
            tol = 1e-12 * max(1.0, float(ref.abs().max()))
            torch.testing.assert_close(got, ref, rtol=0, atol=tol, msg=f"{what} {k}")
    assert torch.equal(out["full_pose"][1:22], out["body_pose"].detach())
    assert float(out["jaw_pose"].detach().abs().max()) == 0 and bool(torch.isfinite(leaves["jaw_pose"].grad).all())


@pytest.mark.parametrize("warmup", [0, 1])
def test_geometry_restatement_reproduces_the_reference_golden(warmup):
    gm = _golden_module()
    gold = np.load(os.path.join(G, "human_assets.npz"))
    inp, w = gm.geometry_case()
    mask, pose_offset = _geometry_inputs(inp)
    lv = {k: inp[k].clone().requires_grad_() for k in gm.GEO_LEAVES}
    expr_offset = (lv["expr"][None, None, :] * inp["expr_dirs"]).sum(2)
    res = human_geometry_reference(lv["mesh"], pose_offset, expr_offset, lv["geo"], lv["geo_offset"], mask,
                                   bool(warmup))
    res["rgb"], res["rgb_refined"] = human_colors_reference(lv["rgb"], lv["rgb_offset"])
    names = gm.GEO_OUTPUTS + (gm.WARMUP_OUTPUTS if warmup else ())
    assert set(names) == set(res)
    sum((_fin(res[k]) * w[k]).sum() for k in names).backward()
    for k in names:
        ref = torch.from_numpy(gold[f"w{warmup}:out:{k}"])
        torch.testing.assert_close(res[k].detach(), ref, rtol=0, atol=1e-12, equal_nan=True, msg=k)
    for k in gm.GEO_LEAVES:
        torch.testing.assert_close(lv[k].grad, torch.from_numpy(gold[f"w{warmup}:grad:{k}"]), rtol=0, atol=1e-12,
                                   msg=k)
    torch.testing.assert_close(constant_rotation_reference(gm.P), torch.from_numpy(gold[f"w{warmup}:out:rotation"]),
                               rtol=0, atol=0)
    assert bool((torch.from_numpy(gold[f"w{warmup}:out:opacity"]) == 1).all())
    if warmup:  # the fixture's scales straddle the clamp
        s = torch.from_numpy(gold["w1:out:scale_wo_clamp"])
        assert bool((s > 1e-3).any()) and bool((s < 1e-3).any())
    assert bool(torch.isnan(torch.from_numpy(gold[f"w{warmup}:out:mean_offset_offset"])[12]).any())


def test_cabi_symbols_struct_sizes_and_argument_checks():
    lib = L.load()
    raw = C.CDLL(L.LIB_PATH)
    for name in ("b2r_decode_pose_forward", "b2r_decode_pose_backward", "b2r_human_geometry_forward",
                 "b2r_human_geometry_backward", "b2r_human_colors_forward", "b2r_human_colors_backward"):
        assert hasattr(raw, name) and name in {s[0] for s in L.SYMBOLS}, name
    assert lib.b2r_sizeof(19) == C.sizeof(L.B2RSmplxPose) == 8 * 7 + 4 * 8
    assert lib.b2r_sizeof(20) == C.sizeof(L.B2RSmplxPoseGrads) == 8 * 7
    assert lib.b2r_sizeof(21) == C.sizeof(L.B2RHumanAssets) == 8 + 16 + 8 * 6
    assert lib.b2r_sizeof(22) == C.sizeof(L.B2RHumanAssetsGrads) == 8 * 11
    launches = lib.b2r_launch_count()

    def pose(**kw):
        p = L.B2RSmplxPose()
        for k, n in enumerate((1, 21, 1, 1, 1, 15, 15)):
            p.param[k], p.rows[k] = FAKE, n
        for k, v in kw.items():
            k, field = int(k[1:]), k[0]
            (p.param if field == "p" else p.rows)[k] = v
        return p

    pg = L.B2RSmplxPoseGrads()
    for k in range(7):
        pg.param[k] = FAKE
    fwd = lambda p, out=FAKE: lib.b2r_decode_pose_forward(C.byref(p), out, None)  # noqa: E731
    bwd = lambda p, g=pg, d=FAKE: lib.b2r_decode_pose_backward(C.byref(p), d, C.byref(g), None)  # noqa: E731
    for kw in ({"p1": None}, {"r0": -1}, {"r5": 65}, {"r6": 30}):  # the last: 40 + 30 joints > 64
        assert fwd(pose(**kw)) == -1 and bwd(pose(**kw)) == -1, kw
    empty = pose(**{f"r{k}": 0 for k in range(7)})
    assert fwd(empty) == -1 and bwd(empty) == -1
    assert lib.b2r_decode_pose_forward(None, FAKE, None) == -1
    assert fwd(pose(), None) == -1 and bwd(pose(), pg, None) == -1
    assert lib.b2r_decode_pose_backward(C.byref(pose()), FAKE, None, None) == -1
    g_hole = L.B2RSmplxPoseGrads()
    for k in range(6):
        g_hole.param[k] = FAKE
    assert bwd(pose(), g_hole) == -1

    def ha(**kw):
        h = L.B2RHumanAssets(P=1000, warmup=1, geo_stride=4, geo_offset_stride=8)
        for name, _ in L.B2RHumanAssets._fields_[4:]:
            setattr(h, name, FAKE)
        for k, v in kw.items():
            setattr(h, k, v)
        return h

    outs = [FAKE] * 7
    gfwd = lambda h, o=outs: lib.b2r_human_geometry_forward(C.byref(h), *o, None)  # noqa: E731
    hg = L.B2RHumanAssetsGrads(*([FAKE] * 11))
    gbwd = lambda h, g=hg: lib.b2r_human_geometry_backward(C.byref(h), C.byref(g), None)  # noqa: E731
    for kw in ({"P": -1}, {"warmup": 2}, {"geo_stride": 3}, {"geo_offset_stride": 0}, {"mesh": None},
               {"pose_offset": None}, {"expr_offset": None}, {"geo": None}, {"geo_offset": None}, {"mask": None}):
        assert gfwd(ha(**kw)) == -1 and gbwd(ha(**kw)) == -1, kw
    for i in range(7):  # every output; the two unclamped scales because warmup is on
        o = list(outs)
        o[i] = None
        assert gfwd(ha(), o) == -1, i
    for field in ("dL_dmesh", "dL_dexpr_offset", "dL_dgeo", "dL_dgeo_offset"):
        g = L.B2RHumanAssetsGrads(*([FAKE] * 11))
        setattr(g, field, None)
        assert gbwd(ha(), g) == -1, field
    assert lib.b2r_human_geometry_backward(C.byref(ha()), None, None) == -1
    assert lib.b2r_human_colors_forward(-1, FAKE, FAKE, FAKE, FAKE, None) == -1
    for i in range(4):
        a = [FAKE] * 4
        a[i] = None
        assert lib.b2r_human_colors_forward(10, *a, None) == -1, i
    for i in (0, 1, 4, 5):
        a = [FAKE] * 6
        a[i] = None
        assert lib.b2r_human_colors_backward(10, *a, None) == -1, i
    assert lib.b2r_launch_count() == launches


def test_cabi_accepts_an_empty_set_without_launching():
    lib = L.load()
    launches = lib.b2r_launch_count()
    h = L.B2RHumanAssets(P=0)
    assert lib.b2r_human_geometry_forward(C.byref(h), *([None] * 7), None) == 0
    assert lib.b2r_human_geometry_backward(C.byref(h), C.byref(L.B2RHumanAssetsGrads()), None) == 0
    assert lib.b2r_human_colors_forward(0, None, None, None, None, None) == 0
    assert lib.b2r_human_colors_backward(0, None, None, None, None, None, None, None) == 0
    assert lib.b2r_launch_count() == launches


def test_host_refuses_cpu_tensors():
    from exavatar_release_b200 import decode_smplx_pose
    params, _ = _golden_module().pose_case()
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        decode_smplx_pose({k: v.float() for k, v in params.items()})
    with pytest.raises(RuntimeError, match="CUDA"):
        from exavatar_release_b200 import HumanAssets
        HumanAssets(torch.zeros(4), torch.zeros(4), torch.zeros(4), device="cpu")


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

def _close(a, b, rel, name):
    scale = float(b.detach().abs().max())
    err = float((a.detach().double() - b.detach().double()).abs().max())
    assert err <= rel * max(scale, 1e-30), f"{name}: max error {err:.3e} vs {rel:.0e} x max {scale:.3e}"


def _rowwise(a, b, rel, floor, name):
    """|a - b| <= rel * max(max |b| over the row, floor), row by row."""
    a, b = a.double().reshape(a.shape[0] if a.dim() > 1 else 1, -1), b.double().reshape(a.shape[0] if a.dim() > 1
                                                                                     else 1, -1)
    lim = rel * b.abs().amax(1, keepdim=True).clamp_min(floor)
    bad = (a - b).abs() > lim
    assert not bool(bad.any()), f"{name}: rows {torch.nonzero(bad.any(1)).reshape(-1).tolist()} off by " \
                                f"{float((a - b).abs().max()):.3e}"


@pytest.mark.gpu
def test_decode_against_float64_at_every_fixture_row():
    from exavatar_release_b200 import decode_smplx_pose
    params, w = _golden_module().pose_case()
    p32 = {k: v.float().cuda().requires_grad_() for k, v in params.items()}
    p64 = {k: v.detach().cpu().double().requires_grad_() for k, v in p32.items()}
    out = decode_smplx_pose(p32)
    ref = decode_smplx_pose_reference(p64)
    for k in POSE_KEYS:
        assert out[k].shape == ref[k].shape, k
        _rowwise(out[k].detach().cpu().reshape(-1, 3), ref[k].detach().cpu().reshape(-1, 3), 4e-7, 1.0, k)
    sum((out[k] * w[k].float().cuda()).sum() for k in POSE_KEYS).backward()
    sum((ref[k] * w[k]).sum() for k in POSE_KEYS).backward()
    for k in POSE_KEYS:
        a, b = p32[k].grad.cpu(), p64[k].grad
        assert bool(torch.isfinite(a).all()), k
        _rowwise(a.reshape(-1, 6), b.reshape(-1, 6), 2e-6, 1e-3, f"d{k}")
    # exact identities (jaw, eyes) give exactly zero and a finite gradient; the views share full_pose's storage
    assert bool((out["jaw_pose"] == 0).all()) and out["jaw_pose"].shape == (3,)
    assert out["body_pose"].data_ptr() == out["full_pose"][1].data_ptr()
    assert out["expr"] is p32["expr"] and out["trans"] is p32["trans"]
    torch.testing.assert_close(out["full_pose"].detach().cpu().double(), ref["full_pose"].detach(), rtol=0, atol=2e-6)


@pytest.mark.gpu
def test_decode_rejects_rows_outside_the_55_joint_order():
    from exavatar_release_b200 import decode_smplx_pose
    params, _ = _golden_module().pose_case()
    p = {k: v.float().cuda() for k, v in params.items()}
    for k, bad in (("body_pose", p["body_pose"][:20]), ("root_pose", p["body_pose"][:2]),
                   ("lhand_pose", p["lhand_pose"].reshape(-1))):
        with pytest.raises(ValueError, match="55-joint"):
            decode_smplx_pose(dict(p, **{k: bad}))
    with pytest.raises(ValueError, match="float32"):
        decode_smplx_pose(dict(p, jaw_pose=p["jaw_pose"].double()))


def _c4_geometry(P=P_C4, seed=0):
    g = torch.Generator().manual_seed(200 + seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    m = torch.zeros(P, dtype=torch.bool)
    m[torch.randperm(P, generator=g)[:P // 3]] = True
    d = {"mesh": r(P, 3), "pose_offset": 0.01 * r(P, 3) * m[:, None], "expr_offset": 0.01 * r(P, 3),
         "geo": torch.cat([0.01 * r(P, 3), -6.9 + 0.5 * r(P, 1)], 1),
         "geo_offset": torch.cat([0.005 * r(P, 3), 0.3 * r(P, 1)], 1), "rgb": r(P, 3), "rgb_offset": 0.2 * r(P, 3)}
    d = {k: v.cuda() for k, v in d.items()}
    return d, m.cuda()


GEO_IN = ("mesh", "pose_offset", "expr_offset", "geo", "geo_offset")
GEO_GRAD = ("mesh", "expr_offset", "geo", "geo_offset", "rgb", "rgb_offset")


def _assets(mask):
    from exavatar_release_b200 import HumanAssets
    z = torch.zeros_like(mask)
    return HumanAssets(mask, z, z)


OUT_KEYS = ("mean_3d", "mean_3d_refined", "scale", "scale_refined", "mean_offset_offset", "scale_wo_clamp",
            "scale_refined_wo_clamp")


def _geo_loss(res, rgb, rgb_r, w):
    """A weighted sum of every geometry output present and the two colours: w holds 9 (P,3) factors."""
    loss = (rgb * w[7]).sum() + (rgb_r * w[8]).sum()
    return loss + sum((res[k] * w[i]).sum() for i, k in enumerate(OUT_KEYS) if k in res)


def _weights(P, n, seed=9):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(P, 3, generator=g).cuda() for _ in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("warmup", [False, True])
def test_geometry_and_colors_at_c4_against_float64_and_bit_identical_to_fp32_torch(warmup):
    d, mask = _c4_geometry()
    ha = _assets(mask)
    lv = {k: v.clone().requires_grad_() for k, v in d.items()}
    res = ha.geometry(*[lv[k] for k in GEO_IN], warmup=warmup)
    rgb, rgb_r = ha.colors(lv["rgb"], lv["rgb_offset"])
    # ExAvatar's fp32 torch expressions on the device: the same bits
    with torch.no_grad():
        t32 = human_geometry_reference(*[d[k] for k in GEO_IN], mask, warmup)
        c32 = human_colors_reference(d["rgb"], d["rgb_offset"])
    for k, v in t32.items():
        assert torch.equal(res[k], v), k
    assert torch.equal(rgb, c32[0]) and torch.equal(rgb_r, c32[1])
    assert res["mean_offset"].data_ptr() == lv["geo"].data_ptr()
    if warmup:
        assert bool((res["scale_wo_clamp"] > 1e-3).any()) and bool((res["scale_wo_clamp"] < 1e-3).any())
    # float64 restatement: outputs and gradients of a seeded loss
    l64 = {k: v.double().requires_grad_() for k, v in d.items()}
    r64 = human_geometry_reference(*[l64[k] for k in GEO_IN], mask, warmup)
    c64 = human_colors_reference(l64["rgb"], l64["rgb_offset"])
    for k, v in r64.items():
        _close(res[k], v, 1e-6, k)
    _close(rgb, c64[0], 1e-6, "rgb")
    _close(rgb_r, c64[1], 1e-6, "rgb_refined")
    w = _weights(P_C4, 9)
    _geo_loss(res, rgb, rgb_r, w).backward()
    _geo_loss(r64, *c64, [x.double() for x in w]).backward()
    assert lv["pose_offset"].grad is None
    for k in GEO_GRAD:
        _close(lv[k].grad, l64[k].grad, 1e-5, f"d{k}")


@pytest.mark.gpu
def test_runs_are_bit_identical():
    d, mask = _c4_geometry(seed=1)
    ha = _assets(mask)
    w = _weights(P_C4, 9)
    runs = []
    for _ in range(2):
        lv = {k: v.clone().requires_grad_() for k, v in d.items()}
        res = ha.geometry(*[lv[k] for k in GEO_IN], warmup=True)
        rgb, rgb_r = ha.colors(lv["rgb"], lv["rgb_offset"])
        _geo_loss(res, rgb, rgb_r, w).backward()
        runs.append([res[k].detach().clone() for k in OUT_KEYS] + [rgb.detach(), rgb_r.detach()] +
                    [lv[k].grad for k in GEO_GRAD])
    assert all(torch.equal(a, b) for a, b in zip(*runs))


@pytest.mark.gpu
@pytest.mark.parametrize("P", [0, 1, 255, 257, 1000 + 37])
def test_sizes_off_the_block_and_strided_geo_views(P):
    d, mask = _c4_geometry(P=P, seed=2)
    ha = _assets(mask)
    w = _weights(P, 9)
    wide = torch.cat([torch.zeros(P, 2, device="cuda"), d["geo"], torch.ones(P, 3, device="cuda"), d["geo_offset"]], 1)
    res_all = []
    for strided in (True, False):
        b = wide.clone().requires_grad_()
        geo, geo_off = (b[:, 2:6], b[:, 9:13]) if strided else (b[:, 2:6].detach().clone().requires_grad_(),
                                                               b[:, 9:13].detach().clone().requires_grad_())
        assert geo.is_contiguous() != strided or P <= 1
        lv = {k: d[k].clone().requires_grad_() for k in ("mesh", "expr_offset", "rgb", "rgb_offset")}
        res = ha.geometry(lv["mesh"], d["pose_offset"], lv["expr_offset"], geo, geo_off, warmup=True)
        rgb, rgb_r = ha.colors(lv["rgb"], lv["rgb_offset"])
        assert res["mean_3d"].shape == (P, 3) and rgb.shape == (P, 3)
        if P == 0:
            return
        _geo_loss(res, rgb, rgb_r, w).backward()
        gg = b.grad if strided else torch.cat([torch.zeros(P, 2, device="cuda"), geo.grad,
                                               torch.zeros(P, 3, device="cuda"), geo_off.grad], 1)
        res_all.append([res[k].detach() for k in OUT_KEYS] + [gg] + [lv[k].grad for k in lv])
        if strided:
            with torch.no_grad():
                t32 = human_geometry_reference(d["mesh"], d["pose_offset"], d["expr_offset"], d["geo"],
                                               d["geo_offset"], mask, True)
            for k, v in t32.items():
                assert torch.equal(res[k], v), k
    assert all(torch.equal(a, b) for a, b in zip(*res_all))


@pytest.mark.gpu
def test_warmup_clamp_gradient_mask():
    """torch.clamp(x, max=0.001) passes the gradient where x <= 0.001.  exp lands on fl(0.001) exactly for few or no
    fp32 inputs, so the test scans every fp32 log-scale within 400 ulps of log(0.001) on the device, takes ExAvatar's
    fp32 expression as the truth, and checks the mask element for element (at equality too, where one exists)."""
    hi = np.float32(0.001)
    x0 = np.float32(np.log(np.float64(hi)))
    xs = [x0]
    a = b = x0
    for _ in range(400):
        a, b = np.nextafter(a, np.float32(-10)), np.nextafter(b, np.float32(10))
        xs += [a, b]
    x = torch.tensor(np.array(sorted(xs), dtype=np.float32), device="cuda")
    P = x.numel()
    mask = torch.zeros(P, dtype=torch.bool, device="cuda")
    ha = _assets(mask)
    zeros3 = torch.zeros(P, 3, device="cuda")
    geo = torch.cat([zeros3, x[:, None]], 1).requires_grad_()
    geo_off = torch.zeros(P, 4, device="cuda").requires_grad_()
    res = ha.geometry(zeros3, zeros3, zeros3, geo, geo_off, warmup=True)
    res["scale"].sum().backward()
    gt = geo.detach().clone().requires_grad_()
    t = human_geometry_reference(zeros3, zeros3, zeros3, gt, geo_off.detach(), mask, True)
    t["scale"].sum().backward()
    assert torch.equal(res["scale"], t["scale"])
    s = res["scale_wo_clamp"][:, 0]
    passes = s <= float(hi)
    assert bool(passes.any()) and bool((~passes).any())
    assert bool((geo.grad[:, 3] != 0).eq(passes).all())  # gradient exactly where torch's mask passes
    assert bool((geo.grad[~passes, 3] == 0).all()) and bool((gt.grad[~passes, 3] == 0).all())
    torch.testing.assert_close(geo.grad, gt.grad, rtol=1e-6, atol=0)


@pytest.mark.gpu
def test_constant_rotation_and_opacity():
    ha = _assets(torch.zeros(300, dtype=torch.bool, device="cuda"))
    assert torch.equal(ha.rotation, constant_rotation_reference(300, torch.float32, "cuda"))
    assert torch.equal(ha.opacity, torch.ones(300, 1, device="cuda"))


def _chain_setup():
    from exavatar_release_b200 import SmplxRig
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.smplx_rig import upsample
    from exavatar_release_b200.synthetic import make_human_mesh, make_regs_labels, make_smplx_model
    dev = torch.device("cuda:0")
    mesh = make_human_mesh()
    model = make_smplx_model(mesh)
    rig = SmplxRig(**model, device=dev)
    m = rig.model
    skw = upsample(m["lbs_weights"], m["sub1"], m["sub2"]).float().to(dev).contiguous()
    labels = make_regs_labels(mesh)
    self_map = (labels["is_rhand"] | labels["is_lhand"] | labels["is_face"]).to(dev)
    from exavatar_release_b200 import HumanAssets
    ha = HumanAssets(model["is_rhand"], model["is_lhand"], model["is_face_expr"], device=dev)
    cam = look_at_cam_param(-6.0, (512, 512), device=dev)
    params, _ = _golden_module().pose_case()
    g = torch.Generator().manual_seed(21)
    P = rig.P
    leaves = {k: v.float().to(dev).requires_grad_() for k, v in params.items()}
    leaves["expr"] = torch.randn(rig.NE, generator=g).to(dev).requires_grad_()
    others = {"shape": torch.randn(rig.NB, generator=g).to(dev).requires_grad_(),
              "joint_offset": (0.01 * torch.randn(rig.J, 3, generator=g)).to(dev).requires_grad_(),
              "geo": torch.cat([0.01 * torch.randn(P, 3, generator=g), -6.9 + 0.5 * torch.randn(P, 1, generator=g)],
                               1).to(dev).requires_grad_(),
              "geo_offset": (0.01 * torch.randn(P, 4, generator=g)).to(dev).requires_grad_(),
              "rgb": torch.randn(P, 3, generator=g).to(dev).requires_grad_(),
              "rgb_offset": (0.1 * torch.randn(P, 3, generator=g)).to(dev).requires_grad_()}
    w = [torch.randn(P, 3, generator=g).to(dev) for _ in range(4)]
    return rig, ha, skw, self_map, cam, leaves, others, w


def _chain(rig, ha, skw, self_map, cam, leaves, others, w):
    from exavatar_release_b200 import nearest_rows, skin_gaussians
    from exavatar_release_b200 import decode_smplx_pose
    sp = decode_smplx_pose(leaves)
    out = rig(others["shape"], others["joint_offset"], sp["full_pose"], sp["expr"])
    a = ha.geometry(out.mesh_neutral_pose, out.pose_offset, out.expr_offset, others["geo"], others["geo_offset"],
                    warmup=True)
    rows = nearest_rows(a["mean_3d"].detach(), out.mesh_neutral_pose_wo_upsample.contiguous(), self_map)
    posed, posed_r = skin_gaussians(a["mean_3d"], a["mean_3d_refined"], skw, rows, out.joint_mats, sp["trans"],
                                    cam["R"], cam["t"])
    rgb, rgb_r = ha.colors(others["rgb"], others["rgb_offset"])
    loss = (posed * w[0]).sum() + (posed_r * w[1]).sum() + (rgb * w[2]).sum() + (rgb_r * w[3]).sum() + \
        (a["scale"] * w[2]).sum() + (a["scale_refined_wo_clamp"] * w[3]).sum()
    loss.backward()
    return loss


@pytest.mark.gpu
def test_chain_runs_without_host_sync_and_a_cuda_graph_replays_it():
    rig, ha, skw, self_map, cam, leaves, others, w = _chain_setup()
    allp = list(leaves.values()) + list(others.values())
    _chain(rig, ha, skw, self_map, cam, leaves, others, w)  # warm-up (module loads, allocator)
    torch.cuda.synchronize()
    for p in allp:
        p.grad = None
    torch.cuda.set_sync_debug_mode("error")
    try:
        _chain(rig, ha, skw, self_map, cam, leaves, others, w)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in allp)
    # graph: capture the chain once, update every parameter in place, replay, compare with an eager run
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            for p in allp:
                p.grad = None
            _chain(rig, ha, skw, self_map, cam, leaves, others, w)
    torch.cuda.current_stream().wait_stream(s)
    for p in allp:
        p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss_g = _chain(rig, ha, skw, self_map, cam, leaves, others, w)
    g = torch.Generator(device="cuda").manual_seed(5)
    with torch.no_grad():
        for p in allp:
            p.add_(0.01 * torch.randn(p.shape, generator=g, device="cuda"))
    graph.replay()
    got = [float(loss_g)] + [p.grad.clone() for p in allp]
    fresh_l = {k: v.detach().clone().requires_grad_() for k, v in leaves.items()}
    fresh_o = {k: v.detach().clone().requires_grad_() for k, v in others.items()}
    loss_e = _chain(rig, ha, skw, self_map, cam, fresh_l, fresh_o, w)
    want = [float(loss_e)] + [p.grad for p in list(fresh_l.values()) + list(fresh_o.values())]
    assert abs(got[0] - want[0]) <= 1e-6 * abs(want[0])
    for a, b in zip(got[1:], want[1:]):
        _close(a, b, 1e-5, "graph vs eager gradient")
    assert torch.equal(got[-2], want[-2]) and torch.equal(got[-1], want[-1])  # rgb, rgb_offset: the colour op alone
