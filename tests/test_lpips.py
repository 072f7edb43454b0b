"""ExAvatar's LPIPS-VGG terms (avatar/main/model.py:199, :206) as one op: `perceptual.LPIPS` / b2r_lpips_*.

These tests pin
  * without a device: the float64 restatement `lpips_reference` against tests/golden/lpips.npz (written by the
    reference's own `LPIPS` wrapper over an lpips shim), its VGG taps against torchvision's modules, `from_lpips`'s
    picking of the convs and lin weights, the closed-form head gradient the backward kernel evaluates, the C ABI
    (symbols, struct size, byte formulas, validation before any launch) and the Python argument checks;
  * on the GPU: the op against the float64 restatement at C4 size and on every fixture case, within 2x the error of the
    fp32 restatement on torch's default TF32 cuDNN convolutions; exact zeros outside the crop; NaN and a zero gradient
    under 16 px; N = 2 equal to two N = 1 calls; bit-identical runs; no host sync; CUDA-graph replay with a box of
    another size; and one C4 `TrainingFrameRenderer` frame with l1_ssim and the op against the fp32 restatement.
"""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import workload_settings  # noqa: F401  (path setup)
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.losses import crop_box, l1_ssim
from exavatar_release_b200.perceptual import EPS, LPIPS, lpips_reference, vgg_taps_reference

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FAKE = 0x1000  # never dereferenced: validation fails before any launch
NAMES = ("b2r_lpips_saved_bytes", "b2r_lpips_scratch_bytes", "b2r_lpips_forward", "b2r_lpips_backward")
LEVEL = (0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4)
COUT = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
TAPS = (64, 128, 256, 512, 512)


def _golden_module():
    spec = importlib.util.spec_from_file_location("make_lpips_golden", os.path.join(G, "make_lpips_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_GM = _golden_module()
_W = None


def _weights():
    global _W
    if _W is None:
        _W = _GM.lpips_weights()
    return _W


def _fixture():
    z = np.load(os.path.join(G, "lpips.npz"))
    img, target = _GM.lpips_images()
    cases = {}
    for name, box in _GM.LPIPS_CASES:
        cases[name] = dict(img=img, target=target, bbox=None if box is None else torch.tensor([box]),
                           loss=float(z[f"{name}_loss"]), idx=torch.from_numpy(z[f"{name}_grad_idx"]).long(),
                           grad=torch.from_numpy(z[f"{name}_grad_val"]).double(),
                           abs_sum=float(z[f"{name}_grad_abs_sum"]), nonzero=int(z[f"{name}_grad_nonzero"]))
    return cases


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", [c[0] for c in _GM.LPIPS_CASES])
def test_reference_matches_the_golden_fixture(name):
    c = _fixture()[name]
    feats, lins = _weights()
    x = c["img"].double().requires_grad_()
    loss = lpips_reference(x, c["target"], c["bbox"], feats, lins)
    assert loss.shape == (1, 1, 1, 1)
    loss.sum().backward()
    assert abs(float(loss.detach()) - c["loss"]) <= 1e-12 * max(abs(c["loss"]), 1e-30) + 1e-15
    g = x.grad.reshape(-1)
    assert torch.allclose(g[c["idx"]], c["grad"], rtol=1e-9, atol=1e-15)
    assert abs(float(g.abs().sum()) - c["abs_sum"]) <= 1e-9 * c["abs_sum"]
    assert int((g != 0).sum()) == c["nonzero"]


def test_reference_raises_under_16_px():
    feats, lins = _weights()
    img, target = _GM.lpips_images()
    with pytest.raises(RuntimeError):
        lpips_reference(img, target, torch.tensor([10.0, 10.0, 15.9, 40.0]), feats, lins)


def test_restated_taps_equal_torchvision_modules_in_float64():
    feats, _ = _weights()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 3, 37, 53, generator=g, dtype=torch.float64)
    mine = vgg_taps_reference(x, feats)
    net = _GM._Vgg16(feats).double()  # torchvision's own modules, run slice by slice
    theirs = net(x)
    for k, (a, b) in enumerate(zip(mine, theirs)):
        assert a.shape == b.shape, k
        assert torch.allclose(a, b, rtol=1e-12, atol=1e-14), k
    assert [t.shape[1:] for t in mine] == [(64, 37, 53), (128, 18, 26), (256, 9, 13), (512, 4, 6), (512, 2, 3)]


def test_from_lpips_picks_the_convs_and_lin_weights_in_order(monkeypatch):
    shim = _GM._LpipsShim()  # lpips's attribute layout: net.slice1..5 with torchvision's child indices, lin0..4
    seen = {}

    def fake_init(self, vgg_features, lin_weights, device):
        seen["convs"] = [m for m in vgg_features if isinstance(m, torch.nn.Conv2d)]
        seen["lins"] = list(lin_weights)
        seen["device"] = device

    monkeypatch.setattr(LPIPS, "__init__", fake_init)
    LPIPS.from_lpips(shim)
    feats = [shim.net.slice1, shim.net.slice2, shim.net.slice3, shim.net.slice4, shim.net.slice5]
    expect = [m for s in feats for m in s if isinstance(m, torch.nn.Conv2d)]
    assert len(seen["convs"]) == 13 and all(a is b for a, b in zip(seen["convs"], expect))
    assert [m.out_channels for m in seen["convs"]] == list(COUT)
    assert all(w is getattr(shim, f"lin{k}").model[-1].weight for k, w in enumerate(seen["lins"]))
    assert seen["device"] == torch.device("cpu")


def test_lpips_requires_cuda_and_checks_weights():
    feats, lins = _weights()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        LPIPS(feats, lins, "cpu")
    with pytest.raises(ValueError, match="13 convolutions"):
        LPIPS(list(feats)[:20], lins, "cpu")
    with pytest.raises(ValueError, match="5 lin weights"):
        LPIPS(feats, lins[:4], "cpu")


def test_lpips_argument_errors():
    meta = torch.device("meta")  # CUDA-agnostic stand-ins: every check fails before any launch

    class _Cuda(torch.Tensor):
        @property
        def is_cuda(self):
            return True

    def cu(*shape, dtype=torch.float32, grad=False):
        return torch.empty(*shape, device=meta, dtype=dtype).as_subclass(_Cuda).requires_grad_(grad)

    op = LPIPS.__new__(LPIPS)
    op.device = meta
    img = torch.rand(3, 32, 32)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        op(img, img.clone())
    cases = [
        ((cu(2, 4, 32, 32), cu(3, 32, 32)), {}, r"\(3,H,W\)"),
        ((cu(3, 32, 32), cu(2, 3, 32, 32)), {}, "batch"),
        ((cu(3, 32, 32), cu(3, 32, 33)), {}, "does not match"),
        ((cu(3, 15, 32), cu(3, 15, 32)), {}, "at least 16"),
        ((cu(3, 32, 32, dtype=torch.float64), cu(3, 32, 32)), {}, "float32"),
        ((cu(3, 32, 32), cu(3, 32, 32)), {"bbox": cu(5)}, "bbox"),
        ((cu(3, 32, 32), cu(3, 32, 32)), {"bbox": cu(4, dtype=torch.int64)}, "bbox"),
        ((cu(3, 32, 32), cu(3, 32, 32, grad=True)), {}, "img_target"),
    ]
    for args, kw, match in cases:
        with pytest.raises(ValueError, match=match):
            op(*args, **kw)


def _saved_formula(W, H, N):
    up = lambda v: (v + 255) // 256 * 256  # noqa: E731
    per = sum(up(4 * c * (H >> lv) * (W >> lv)) for c, lv in zip(COUT, LEVEL))
    return N * per + sum(up(4 * c * (H >> t) * (W >> t)) for t, c in enumerate(TAPS))


def test_lpips_symbols_struct_and_byte_formulas():
    lib = L.load()
    raw = C.CDLL(L.LIB_PATH)
    for name in NAMES:
        assert hasattr(raw, name), name
        assert name in {s[0] for s in L.SYMBOLS}, name
    assert C.sizeof(L.B2RLpips) == 16 + 8 * 3 + 8 * (13 * 3 + 5)
    for W, H, N in ((16, 16, 1), (96, 72, 1), (512, 512, 1), (512, 512, 2), (1000, 777, 3)):
        assert lib.b2r_lpips_saved_bytes(W, H, N) == _saved_formula(W, H, N), (W, H, N)
        up = lambda v: (v + 255) // 256 * 256  # noqa: E731
        scratch = 2 * up(4 * 64 * W * H) + sum(up(8 * (((H >> t) * (W >> t) + 31) // 32)) for t in range(5))
        assert lib.b2r_lpips_scratch_bytes(W, H) == scratch, (W, H)
    # 283 MB of ReLU outputs per image and 128 MB of target taps at 512^2
    assert round(_saved_formula(512, 512, 1) / 1e6) == 411 and round((_saved_formula(512, 512, 2) - _saved_formula(
        512, 512, 1)) / 1e6) == 283


def _struct(W=64, H=48, N=1, drop=None):
    p = L.B2RLpips(width=W, height=H, n_images=N, img=FAKE, target=FAKE, bbox=None)
    for k in range(13):
        p.w_fwd[k] = FAKE
        p.bias[k] = FAKE
        if k:
            p.w_bwd[k] = FAKE
    for k in range(5):
        p.lin[k] = FAKE
    if drop:
        field, k = drop
        if k is None:
            setattr(p, field, None)
        else:
            getattr(p, field)[k] = None
    return p


def test_lpips_validation_without_touching_cuda():
    lib = L.load()
    n0 = lib.b2r_launch_count()
    sv, sc = lib.b2r_lpips_saved_bytes(64, 48, 1), lib.b2r_lpips_scratch_bytes(64, 48)

    def fwd(p=None, out=FAKE, saved=FAKE, nsv=sv, scratch=FAKE, nsc=sc):
        return lib.b2r_lpips_forward(C.byref(p or _struct()), out, saved, nsv, scratch, nsc, None)

    def bwd(p=None, saved=FAKE, nsv=sv, dout=FAKE, dimg=FAKE, scratch=FAKE, nsc=sc):
        return lib.b2r_lpips_backward(C.byref(p or _struct()), saved, nsv, dout, dimg, scratch, nsc, None)

    bad = [_struct(W=15), _struct(H=15), _struct(N=0), _struct(W=1 << 15, H=1 << 14),
           _struct(drop=("img", None)), _struct(drop=("target", None)), _struct(drop=("w_fwd", 0)),
           _struct(drop=("w_fwd", 12)), _struct(drop=("w_bwd", 1)), _struct(drop=("bias", 5)),
           _struct(drop=("lin", 4))]
    for p in bad:
        assert fwd(p) == -1 and bwd(p) == -1
    assert lib.b2r_lpips_forward(None, FAKE, FAKE, sv, FAKE, sc, None) == -1
    assert fwd(out=None) == -1 and fwd(saved=None) == -1 and fwd(scratch=None) == -1
    assert fwd(nsv=sv - 1) == -2 and fwd(nsc=sc - 1) == -2
    assert bwd(dout=None) == -1 and bwd(dimg=None) == -1 and bwd(saved=None) == -1 and bwd(scratch=None) == -1
    assert bwd(nsv=sv - 1) == -2 and bwd(nsc=sc - 1) == -2
    assert fwd(_struct(N=2)) == -2  # the saved buffer of one image is too small for two
    assert lib.b2r_launch_count() == n0


def head_grad_closed_form(f, nt, w, G):
    """d/df of G * sum_c w_c (f_c / (|f| + eps) - nt_c)^2 per pixel, as lp_boundary_kernel evaluates it.  f, nt (C,P)."""
    r = torch.sqrt((f * f).sum(0, keepdim=True))
    s = r + EPS
    dn = G * 2 * w[:, None] * (f / s - nt)
    gr = (-(dn * f).sum(0, keepdim=True) / (s * s)) / r
    return dn / s + f * gr


def test_closed_form_head_gradient_matches_f64_autograd():
    g = torch.Generator().manual_seed(9)
    C_, P = 64, 50
    f = torch.relu(torch.randn(C_, P, generator=g, dtype=torch.float64))
    f[:, 7] = 0.0  # a pixel with every channel exactly 0
    nt = torch.rand(C_, P, generator=g, dtype=torch.float64)
    nt = nt / nt.norm(dim=0, keepdim=True)
    w = torch.rand(C_, generator=g, dtype=torch.float64)
    G = 0.37
    fa = f.clone().requires_grad_()
    n = fa / (torch.sqrt(torch.sum(fa ** 2, dim=0, keepdim=True)) + EPS)
    (G * (w[:, None] * (n - nt) ** 2).sum()).backward()
    mine = head_grad_closed_form(f, nt, w, G)
    ok = torch.ones(P, dtype=torch.bool)
    ok[7] = False
    assert torch.allclose(mine[:, ok], fa.grad[:, ok], rtol=1e-12, atol=1e-15)
    assert torch.isnan(fa.grad[:, 7]).all() and torch.isnan(mine[:, 7]).all()  # autograd's NaN, reproduced


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def op(dev):
    feats, lins = _weights()
    return LPIPS(feats, lins, dev)


def _c4_case():
    """C4 size: 512x512, a smooth render-like pair, a box of ~60 % of the image."""
    g = torch.Generator().manual_seed(21)
    base = F.interpolate(torch.rand(1, 3, 32, 32, generator=g), size=(512, 512), mode="bilinear")[0]
    img = (base + 0.05 * torch.randn(3, 512, 512, generator=g)).clamp(0, 1)
    return dict(img=img, target=base, bbox=torch.tensor([[85.3, 40.6, 330.2, 400.9]]))


def _all_cases():
    cases = _fixture()
    cases["c4"] = _c4_case()
    return cases


@pytest.mark.gpu
def test_op_error_is_within_twice_the_tf32_reference_error(dev, op):
    """Errors against the float64 restatement, of the op and of the fp32 restatement on torch's default (TF32) cuDNN
    convolutions, on every fixture case and at C4.  The gradient's error is |g - g64| / |g64| (L2 over the image): its
    max-norm counterpart is set by the few pixels where TF32 rounding flips a ReLU, one discrete event per arm, and is
    printed only.  It must be within 2x on every case.  The loss is one number per case, and cuDNN picks an FP32
    algorithm for some small crops, so per case it must be within 2x or within TF32's unit roundoff (2^-11) of the
    loss; summed over the cases it must be within 2x."""
    feats, lins = _weights()
    feats_d = feats.to(dev)
    tot = {"tf32": 0.0, "op": 0.0}
    for name, c in _all_cases().items():
        bbox = None if c["bbox"] is None else c["bbox"].to(dev)
        tgt = c["target"].to(dev)
        runs = {}
        for arm in ("f64", "tf32", "op"):
            x = c["img"].to(dev).requires_grad_()
            if arm == "op":
                loss = op(x, tgt, bbox)
            else:
                loss = lpips_reference(x, tgt, bbox, feats_d, lins,
                                       dtype=torch.float64 if arm == "f64" else torch.float32)
            loss.sum().backward()
            runs[arm] = (float(loss.detach()), x.grad.double())
        torch.cuda.synchronize()
        l64, g64 = runs["f64"]
        gmax = float(g64.abs().max())
        err = {a: (abs(runs[a][0] - l64), float((runs[a][1] - g64).norm() / g64.norm()),
                   float((runs[a][1] - g64).abs().max()) / gmax) for a in ("tf32", "op")}
        print(f"{name}: loss {l64:.8f}  |dloss|/loss op {err['op'][0] / l64:.2e} tf32 {err['tf32'][0] / l64:.2e}  "
              f"L2 dgrad op {err['op'][1]:.2e} tf32 {err['tf32'][1]:.2e}  "
              f"max|dgrad|/max|g| op {err['op'][2]:.2e} tf32 {err['tf32'][2]:.2e}")
        assert err["op"][1] <= 2 * err["tf32"][1], name
        assert err["op"][0] <= max(2 * err["tf32"][0], 2.0 ** -11 * abs(l64)), name
        for a in tot:
            tot[a] += err[a][0] / abs(l64)
    print(f"sum of |dloss|/loss: op {tot['op']:.2e} tf32 {tot['tf32']:.2e}")
    assert tot["op"] <= 2 * tot["tf32"]


@pytest.mark.gpu
def test_gradient_is_exactly_zero_outside_the_crop(dev, op):
    c = _c4_case()
    bbox = c["bbox"].to(dev)
    x = c["img"].to(dev).requires_grad_()
    op(x, c["target"].to(dev), bbox).sum().backward()
    torch.cuda.synchronize()
    x0, y0, x1, y1 = crop_box(bbox, 512, 512)
    inside = torch.zeros(512, 512, dtype=torch.bool, device=dev)
    inside[y0:y1, x0:x1] = True
    assert float(x.grad[:, ~inside].abs().max()) == 0.0
    assert int((x.grad[:, inside] != 0).sum()) > 0.9 * 3 * int(inside.sum())
    assert bool(torch.isfinite(x.grad).all())


@pytest.mark.gpu
@pytest.mark.parametrize("box", [(100.0, 100.0, 15.9, 200.0), (100.0, 100.0, 200.0, 15.0), (600.0, 10.0, 50.0, 50.0)])
def test_crop_under_16_px_gives_nan_and_zero_gradient(dev, op, box):
    c = _c4_case()
    x = c["img"].to(dev).requires_grad_()
    loss = op(x, c["target"].to(dev), torch.tensor(box, device=dev))
    loss.sum().backward()
    torch.cuda.synchronize()
    assert torch.isnan(loss).all()
    assert float(x.grad.abs().max()) == 0.0


def _fwd_bwd(op, img, target, bbox):
    x = img.clone().requires_grad_()
    lp = op(x, target, bbox)
    gx, = torch.autograd.grad((lp.reshape(-1) * torch.arange(1, lp.shape[0] + 1, device=lp.device)).sum(), (x,))
    return lp.detach(), gx


@pytest.mark.gpu
def test_pair_equals_two_single_calls(dev, op):
    c = _c4_case()
    a, b, tgt, bbox = c["img"].to(dev), c["target"].to(dev).flip(-1), c["target"].to(dev), c["bbox"].to(dev)
    lp2, g2 = _fwd_bwd(op, torch.stack((a, b)), tgt, bbox)
    lpa, ga = _fwd_bwd(op, a, tgt, bbox)
    lpb, gb = _fwd_bwd(op, b[None], tgt[None], bbox)
    torch.cuda.synchronize()
    assert torch.equal(lp2[0], lpa[0]) and torch.equal(lp2[1], lpb[0])
    assert torch.equal(g2[0], ga) and torch.equal(g2[1], 2 * gb[0])  # the pair weights image 1 by 2


@pytest.mark.gpu
def test_two_runs_are_bit_identical(dev, op):
    c = _c4_case()
    args = (torch.stack((c["img"], c["target"].flip(-2))).to(dev), c["target"].to(dev), c["bbox"].to(dev))
    a, b = _fwd_bwd(op, *args), _fwd_bwd(op, *args)
    torch.cuda.synchronize()
    for u, v in zip(a, b):
        assert torch.equal(u, v)


@pytest.mark.gpu
def test_forward_and_backward_do_not_sync(dev, op):
    c = _c4_case()
    args = (torch.stack((c["img"], c["target"].flip(-2))).to(dev), c["target"].to(dev), c["bbox"].to(dev))
    _fwd_bwd(op, *args)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _fwd_bwd(op, *args)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_cuda_graph_replay_with_a_box_of_another_size_equals_eager(dev, op):
    c = _c4_case()
    img = torch.stack((c["img"], c["target"].flip(-2))).to(dev)
    target, bbox = c["target"].to(dev), c["bbox"].to(dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        _fwd_bwd(op, img, target, bbox)
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = _fwd_bwd(op, img, target, bbox)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        img.copy_(torch.rand(2, 3, 512, 512, generator=g).to(dev))
        target.copy_(torch.rand(3, 512, 512, generator=g).to(dev))
        bbox.copy_(torch.tensor([[-30.5, 120.2, 250.7, 300.1]], device=dev))  # 250 x 300 instead of 330 x 400
    graph.replay()
    torch.cuda.synchronize()
    replayed = [t.clone() for t in static]
    eager = _fwd_bwd(op, img, target, bbox)
    torch.cuda.synchronize()
    for name, a, b in zip(("lpips", "grad"), replayed, eager):
        assert torch.equal(a, b), name
    feats, lins = _weights()
    ref = lpips_reference(img[:1], target, bbox, feats.to(dev), lins)
    assert abs(float(replayed[0][0]) - float(ref)) <= 1e-3 * abs(float(ref))  # the replay saw the new box


@pytest.mark.gpu
def test_c4_training_frame_with_l1_ssim_and_lpips(dev, op):
    from exavatar_release_b200 import TrainingFrameRenderer
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.losses import l1_ssim_reference
    from exavatar_release_b200.synthetic import WORKLOADS, make_population_assets
    wl = WORKLOADS["C4"]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets("C4", seed=0, device=dev)
    Ps, Ph = scene["mean_3d"].shape[0], human["mean_3d"].shape[0]
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    bg_r = torch.tensor([0.3, 0.7, 0.2], device=dev)
    g = torch.Generator().manual_seed(13)
    gt = F.interpolate(torch.rand(1, 3, 32, 32, generator=g), size=(H, W), mode="bilinear")[0].to(dev)
    bbox = torch.tensor([[85.3, 40.6, 330.2, 400.9]], device=dev)
    feats, lins = _weights()
    feats_d = feats.to(dev)
    fr = TrainingFrameRenderer(Ps, Ph, (H, W), dev, {"A": 8_000_000, "B": 8_000_000})
    res = {}
    for arm in ("op", "torch"):
        lv = [{k: v.detach().clone().requires_grad_() for k, v in d.items()} for d in (scene, human, refined)]
        out = fr(lv[0], lv[1], lv[2], cam, bg_r)
        pair = (out["scene_human"]["img"], out["scene_human_refined"]["img"])
        loss = 0.0
        for img in pair:
            l1, s = (l1_ssim if arm == "op" else l1_ssim_reference)(img, gt, bbox, **({} if arm == "op" else
                                                                                       {"dtype": torch.float32}))
            loss = loss + 0.8 * l1 + 0.2 * (1 - s)
        if arm == "op":
            lp = op(torch.stack(pair), gt, bbox)
        else:
            lp = torch.cat([lpips_reference(img, gt, bbox, feats_d, lins, dtype=torch.float32) for img in pair])
        loss = loss + 0.2 * lp.sum()
        loss.backward()
        torch.cuda.synchronize()
        assert not fr.overflowed()
        res[arm] = (float(loss), float(lp.sum()), lv)
    (l_op, lp_op, g_op), (l_ref, lp_ref, g_ref) = res["op"], res["torch"]
    print(f"loss op {l_op:.7f} torch {l_ref:.7f}  lpips op {lp_op:.7f} torch {lp_ref:.7f}")
    assert abs(l_op - l_ref) <= 1e-5 * abs(l_ref)
    for d_op, d_ref in zip(g_op, g_ref):
        for k in d_ref:
            if d_ref[k].grad is None:
                assert d_op[k].grad is None, k
                continue
            r = d_ref[k].grad
            lim = 2e-3 * float(r.abs().max())
            diff = float((d_op[k].grad - r).abs().max())
            print(f"  {k}: max|d| {diff:.2e} ({diff / max(float(r.abs().max()), 1e-30):.2e} of max)")
            assert diff <= lim, (k, diff, lim)
