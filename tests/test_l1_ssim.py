"""ExAvatar's photometric L1 + SSIM terms (avatar/main/model.py:196-215) as one op: `losses.l1_ssim` / b2r_l1ssim_*.

These tests pin
  * without a device: the C ABI (exported symbols, scratch size, validation before any launch), the float64 torch
    restatement `l1_ssim_reference` against tests/golden/loss.npz (written by the reference's own `RGBLoss` / `SSIM`),
    the closed-form gradient the backward kernel evaluates against autograd through that restatement, and the Python
    argument checks;
  * on the GPU: the op against the float64 restatement on every fixture case and at C4 size, exact zeros outside the
    crop and under mask = 0, bit-identical runs, no host synchronisation, CUDA-graph capture, and one C4
    `TrainingFrameRenderer` frame with ExAvatar's photometric block through the op vs. through the fp32 restatement.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import capture, golden_generator, no_host_sync
from util import dev  # noqa: F401
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.losses import C1, C2, crop_box, l1_ssim, l1_ssim_reference, ssim_window

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FAKE = 0x1000  # never dereferenced: validation fails before any launch
NAMES = ("b2r_l1ssim_scratch_bytes", "b2r_l1ssim_forward", "b2r_l1ssim_backward")


def _fixture():
    """The cases of loss.npz with their inputs, rebuilt bit for bit by the generator's integer-only `loss_images`."""
    gm = golden_generator("make_loss_golden")
    z = np.load(os.path.join(G, "loss.npz"))
    pairs = {k: gm.loss_images(*hw) for k, hw in gm.SIZES.items()}
    cases = {}
    for name, key, box, term in gm.LOSS_CASES:
        img, target, mask = (t.float() / 255 for t in pairs[key])
        cases[name] = dict(
            img=img, target=target, mask=mask, bg=torch.tensor(gm.BG), term=term,
            pixel_sums=[int(t.long().sum()) for t in pairs[key]], stored_pixel_sums=z[f"{key}_pixel_sums"].tolist(),
            bbox=None if box is None else torch.tensor([box], dtype=torch.float32), l1=float(z[f"{name}_l1"]),
            ssim=float(z[f"{name}_ssim"]), idx=torch.from_numpy(z[f"{name}_grad_idx"]).long(),
            grad=torch.from_numpy(z[f"{name}_grad_val"]).double(), abs_sum=float(z[f"{name}_grad_abs_sum"]),
            nonzero=int(z[f"{name}_grad_nonzero"]))
    return cases


def _run_case(fn, c, img, dev=None, **kw):
    """The ExAvatar term(s) of a fixture case through `fn` (l1_ssim or l1_ssim_reference): (l1, ssim, loss)."""
    to = (lambda t: t) if dev is None else (lambda t: None if t is None else t.to(dev))
    target, mask, bbox, bg = to(c["target"]), to(c["mask"]), to(c["bbox"]), to(c["bg"])
    if c["term"] == "scene":
        l1, s = fn(img, target, mask=1 - mask, **kw)
    elif c["term"] == "rand_bg":
        l1, s = fn(img, target * mask + (1 - mask) * bg[:, None, None], bbox, ssim=False, **kw)
    else:
        l1, s = fn(img, target, bbox, ssim=c["term"] == "l1_ssim", **kw)
    loss = 0.8 * l1 + 0.2 * (1 - s) if s is not None else l1
    return l1, s, loss


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

def test_l1ssim_symbols_and_scratch_size():
    lib = L.load()
    raw = C.CDLL(L.LIB_PATH)
    for name in NAMES:
        assert hasattr(raw, name), name
        assert name in {s[0] for s in L.SYMBOLS}, name
    last = 0
    for W, H in ((1, 1), (16, 16), (200, 136), (512, 512), (1920, 1080)):
        n = lib.b2r_l1ssim_scratch_bytes(W, H)
        assert n >= 9 * 4 * W * H and n > last, (W, H)
        last = n


def test_l1ssim_validation_without_touching_cuda():
    lib = L.load()
    n0 = lib.b2r_launch_count()
    need = lib.b2r_l1ssim_scratch_bytes(64, 48)

    def fwd(W=64, H=48, img=FAKE, tgt=FAKE, out=FAKE, scratch=FAKE, nbytes=need):
        return lib.b2r_l1ssim_forward(W, H, img, tgt, None, None, 1, out, scratch, nbytes, None)

    def bwd(W=64, H=48, img=FAKE, tgt=FAKE, dout=FAKE, dimg=FAKE, scratch=FAKE, nbytes=need, ssim=1):
        return lib.b2r_l1ssim_backward(W, H, img, tgt, None, None, ssim, dout, dimg, scratch, nbytes, None)

    for kw in ({"W": 0}, {"H": 0}, {"W": -5}, {"H": -1}, {"H": 65535 * 16 + 1}, {"W": 1 << 16, "H": 1 << 16},
               {"img": None}, {"tgt": None}):
        assert fwd(**kw) == -1, kw
        assert bwd(**kw) == -1, kw
    assert fwd(out=None) == -1
    assert fwd(scratch=None) == -1
    assert fwd(nbytes=need - 1) == -2
    assert bwd(dout=None) == -1
    assert bwd(dimg=None) == -1
    assert bwd(scratch=None) == -1                 # the SSIM backward reads the forward's partials
    assert bwd(nbytes=need - 1) == -2
    assert lib.b2r_launch_count() == n0            # nothing was launched by any of the above


def test_crop_rules():
    box = lambda *v: torch.tensor(v, dtype=torch.float32)  # noqa: E731
    assert crop_box(None, 200, 136) == (0, 0, 200, 136)
    assert crop_box(box(-20.7, -8.3, 300.9, 280.4), 512, 512) == (0, 0, 300, 280)  # trunc(-20.7) = -20 -> 0, moved
    assert crop_box(box(400.5, 380.2, 200.0, 250.0), 512, 512) == (400, 380, 512, 512)
    assert crop_box(box(13.6, 7.9, 150.3, 101.8), 200, 136) == (13, 7, 163, 108)
    assert crop_box(box(600.0, 10.0, 5.0, 5.0), 512, 512)[2:] == (600, 15)   # empty in x
    assert crop_box(box(10.0, 10.0, -4.0, 5.0), 512, 512)[::2] == (10, 10)    # negative width: empty


@pytest.mark.parametrize("name", ["neg_xy", "past_edge", "c4_box", "frac", "narrow", "one_px", "face_l1", "rand_bg",
                                  "scene"])
def test_reference_matches_the_golden_fixture(name):
    """l1_ssim_reference in float64 == the reference's RGBLoss / SSIM in fp32 (means and the gradient of the weighted
    loss at the stored sample), within fp32-versus-fp64 noise."""
    c = _fixture()[name]
    assert c["pixel_sums"] == c["stored_pixel_sums"]  # the rebuilt inputs are the ones the reference saw
    img = c["img"].double().requires_grad_()
    l1, s, loss = _run_case(l1_ssim_reference, c, img)
    loss.backward()
    assert abs(float(l1.detach()) - c["l1"]) <= 1e-7
    if s is not None:  # the fp32 sigma^2 = E[x^2] - mu^2 of the reference cancels: its mean is ~5e-6 off float64
        assert abs(float(s.detach()) - c["ssim"]) <= 1e-5
    else:
        assert np.isnan(c["ssim"])
    g = img.grad.reshape(-1)
    scale = float(c["grad"].abs().max())
    assert float((g[c["idx"]] - c["grad"]).abs().max()) <= 1e-4 * scale
    assert abs(float(g.abs().sum()) - c["abs_sum"]) <= 1e-4 * c["abs_sum"]
    assert int((g != 0).sum()) == c["nonzero"]


def _closed_form_grad(img, target, bbox, mask, g_l1, g_ss):
    """dL/dimg by the formulas the backward kernel evaluates, in float64: the partials dm/dmu_x, dm/dS_xx, dm/dS_xy of
    the SSIM map, windowed back onto the crop (the window is symmetric), plus the L1 sign term; 0 outside the crop."""
    H, W = img.shape[-2:]
    x0, y0, x1, y1 = crop_box(bbox, W, H)
    m = torch.ones(1, 1, H, W, dtype=torch.float64) if mask is None else mask.reshape(1, 1, H, W).double()
    x = (img.double()[None] * m)[:, :, y0:y1, x0:x1]
    y = (target.double()[None] * m)[:, :, y0:y1, x0:x1]
    n = x.numel()
    w = ssim_window().double()
    win = (w[:, None] * w[None, :]).expand(3, 1, 11, 11)
    conv = lambda t: F.conv2d(t, win, padding=5, groups=3)  # noqa: E731
    mx, my, sxx, syy, sxy = conv(x), conv(y), conv(x * x), conv(y * y), conv(x * y)
    A = 2 * mx * my + C1
    B = 2 * (sxy - mx * my) + C2
    Cc = mx * mx + my * my + C1
    D = sxx - mx * mx + syy - my * my + C2
    smap = A * B / (Cc * D)
    d_mu = (2 * my * (B - A) + 2 * mx * smap * (Cc - D)) / (Cc * D)
    d_sxx = -smap / D
    d_sxy = 2 * A / (Cc * D)
    gs = g_ss / n
    dx = gs * (conv(d_mu) + 2 * x * conv(d_sxx) + y * conv(d_sxy)) + torch.sign(x - y) * g_l1 / n
    full = torch.zeros(1, 3, H, W, dtype=torch.float64)
    full[:, :, y0:y1, x0:x1] = dx
    return (full * m)[0]


@pytest.mark.parametrize("masked", [False, True])
def test_closed_form_gradient_matches_f64_autograd(masked):
    """The backward's closed form (no division by A or B) == float64 autograd through l1_ssim_reference, on a 20x17 crop
    of a 40x36 image, with and without a mask that has zeros."""
    g = torch.Generator().manual_seed(3)
    H, W = 36, 40
    img = torch.rand(3, H, W, generator=g, dtype=torch.float64)
    target = (img + 0.1 * torch.randn(3, H, W, generator=g, dtype=torch.float64)).clamp(0, 1)
    target[:, 10, 10:14] = img[:, 10, 10:14]  # x' == y': sign(0) = 0
    mask = (torch.rand(H, W, generator=g, dtype=torch.float64) - 0.2).clamp_min(0) if masked else None
    bbox = torch.tensor([12.7, 4.2, 17.9, 20.5])
    x = img.clone().requires_grad_()
    l1, s = l1_ssim_reference(x, target, bbox, mask)
    (0.8 * l1 + 0.2 * (1 - s)).backward()
    ref = _closed_form_grad(img, target, bbox, mask, 0.8, -0.2)
    assert float((ref - x.grad).abs().max()) <= 1e-12 * float(x.grad.abs().max())
    assert float(x.grad.abs().max()) > 0


def test_reference_empty_crop_is_nan():
    img = torch.rand(3, 20, 30, dtype=torch.float64)
    l1, s = l1_ssim_reference(img, img * 0.5, torch.tensor([40.0, 2.0, 5.0, 5.0]))
    assert torch.isnan(l1) and torch.isnan(s)


def test_l1_ssim_argument_errors():
    img = torch.rand(3, 8, 8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        l1_ssim(img, img.clone())
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        l1_ssim(img, img.clone(), bbox=torch.zeros(4))
    meta = torch.device("meta")  # CUDA-agnostic stand-ins for the shape checks: they fail before any launch

    class _Cuda(torch.Tensor):
        @property
        def is_cuda(self):
            return True

    def cu(*shape, dtype=torch.float32, grad=False):
        return torch.empty(*shape, device=meta, dtype=dtype).as_subclass(_Cuda).requires_grad_(grad)

    cases = [
        ((cu(2, 3, 8, 8), cu(2, 3, 8, 8)), {}, "batch"),
        ((cu(4, 8, 8), cu(4, 8, 8)), {}, r"\(3,H,W\)"),
        ((cu(3, 8, 8), cu(3, 8, 9)), {}, "does not match"),
        ((cu(3, 8, 8, dtype=torch.float64), cu(3, 8, 8)), {}, "float32"),
        ((cu(3, 8, 8), cu(3, 8, 8)), {"mask": cu(8, 9)}, "mask"),
        ((cu(3, 8, 8), cu(3, 8, 8)), {"mask": cu(2, 8, 8)}, "mask"),
        ((cu(3, 8, 8), cu(3, 8, 8)), {"bbox": cu(5)}, "bbox"),
        ((cu(3, 8, 8), cu(3, 8, 8)), {"bbox": cu(4, dtype=torch.int64)}, "bbox"),
        ((cu(3, 8, 8), cu(3, 8, 8, grad=True)), {}, "target"),
        ((cu(3, 8, 8), cu(3, 8, 8)), {"mask": cu(8, 8, grad=True)}, "mask"),
    ]
    for args, kw, match in cases:
        with pytest.raises(ValueError, match=match):
            l1_ssim(*args, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

def _c4_case():
    """C4 size: 512x512, a smooth render-like pair, a box of ~60 % of the image."""
    g = torch.Generator().manual_seed(21)
    base = F.interpolate(torch.rand(1, 3, 32, 32, generator=g), size=(512, 512), mode="bilinear")[0]
    img = (base + 0.05 * torch.randn(3, 512, 512, generator=g)).clamp(0, 1)
    return dict(img=img, target=base, mask=torch.ones(1, 512, 512), bg=torch.zeros(3), term="l1_ssim",
                bbox=torch.tensor([[85.3, 40.6, 330.2, 400.9]]))


def _all_cases():
    cases = _fixture()
    cases["c4"] = _c4_case()
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["neg_xy", "past_edge", "c4_box", "frac", "narrow", "one_px", "face_l1", "rand_bg",
                                  "scene", "c4"])
def test_op_matches_f64_reference(dev, name):
    c = _all_cases()[name]
    x = c["img"].to(dev).requires_grad_()
    l1, s, loss = _run_case(l1_ssim, c, x, dev)
    loss.backward()
    xr = c["img"].double().requires_grad_()
    rl1, rs, rloss = _run_case(l1_ssim_reference, c, xr)
    rloss.backward()
    torch.cuda.synchronize()
    d_l1 = abs(float(l1) - float(rl1))
    d_s = 0.0 if s is None else abs(float(s) - float(rs))
    ref = xr.grad
    d_g = float((x.grad.cpu().double() - ref).abs().max())
    lim = 1e-4 * float(ref.abs().max())
    print(f"{name}: |dl1| {d_l1:.2e}  |dssim| {d_s:.2e}  max|dgrad| {d_g:.2e} = {d_g / float(ref.abs().max()):.2e} max")
    assert d_l1 <= 1e-5 and d_s <= 1e-5
    assert (s is None) == (rs is None)
    assert d_g <= lim


@pytest.mark.gpu
def test_gradient_is_exactly_zero_outside_the_crop_and_under_the_mask(dev):
    c = _c4_case()
    H, W = 512, 512
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    mask = ((xx // 7 + yy // 5) % 3 != 0).float().to(dev)  # a third of the pixels masked out
    bbox = c["bbox"].to(dev)
    x = c["img"].to(dev).requires_grad_()
    l1, s = l1_ssim(x, c["target"].to(dev), bbox, mask)
    (0.8 * l1 + 0.2 * (1 - s)).backward()
    torch.cuda.synchronize()
    x0, y0, x1, y1 = crop_box(bbox, W, H)
    inside = torch.zeros(H, W, dtype=torch.bool, device=dev)
    inside[y0:y1, x0:x1] = True
    gr = x.grad
    assert float(gr[:, ~inside].abs().max()) == 0.0
    assert float(gr[:, mask == 0].abs().max()) == 0.0
    assert int((gr[:, inside & (mask != 0)] != 0).sum()) > 0.9 * 3 * int((inside & (mask != 0)).sum())


@pytest.mark.gpu
def test_empty_crop_gives_nan_and_zero_gradient(dev):
    c = _c4_case()
    x = c["img"].to(dev).requires_grad_()
    l1, s = l1_ssim(x, c["target"].to(dev), torch.tensor([600.0, 10.0, 50.0, 50.0], device=dev))
    (l1 + s).backward()
    torch.cuda.synchronize()
    assert torch.isnan(l1) and torch.isnan(s)
    assert float(x.grad.abs().max()) == 0.0


def _fwd_bwd(dev, img, target, bbox, mask):
    x = img.clone().requires_grad_()
    l1, s = l1_ssim(x, target, bbox, mask)
    l1f, _ = l1_ssim(x, target, bbox, ssim=False)
    gx, = torch.autograd.grad(0.8 * l1 + 0.2 * (1 - s) + 0.5 * l1f, (x,))
    return l1.detach(), s.detach(), l1f.detach(), gx


@pytest.mark.gpu
def test_two_runs_are_bit_identical(dev):
    c = _c4_case()
    args = (c["img"].to(dev), c["target"].to(dev), c["bbox"].to(dev), (c["mask"] * 0.7).to(dev))
    a = _fwd_bwd(dev, *args)
    b = _fwd_bwd(dev, *args)
    torch.cuda.synchronize()
    for u, v in zip(a, b):
        assert torch.equal(u, v)


@pytest.mark.gpu
def test_forward_and_backward_do_not_sync(dev):
    c = _c4_case()
    args = (c["img"].to(dev), c["target"].to(dev), c["bbox"].to(dev), c["mask"].to(dev))
    _fwd_bwd(dev, *args)  # loads the library and warms the allocator
    with no_host_sync():
        _fwd_bwd(dev, *args)


@pytest.mark.gpu
def test_cuda_graph_replay_with_new_contents_equals_eager(dev):
    c = _c4_case()
    img, target = c["img"].to(dev), c["target"].to(dev)
    bbox, mask = c["bbox"].to(dev), c["mask"].to(dev)
    graph, static = capture(lambda: _fwd_bwd(dev, img, target, bbox, mask), 1)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        img.copy_(torch.rand(3, 512, 512, generator=g).to(dev))
        target.copy_(torch.rand(3, 512, 512, generator=g).to(dev))
        bbox.copy_(torch.tensor([[-30.5, 120.2, 250.7, 300.1]], device=dev))
    graph.replay()
    torch.cuda.synchronize()
    replayed = [t.clone() for t in static]
    eager = _fwd_bwd(dev, img, target, bbox, mask)
    torch.cuda.synchronize()
    for name, a, b in zip(("l1", "ssim", "l1_only", "grad"), replayed, eager):
        assert torch.equal(a, b), name
    rl1, _ = l1_ssim_reference(img.cpu(), target.cpu(), bbox.cpu(), mask.cpu(), ssim=False)
    assert abs(float(replayed[0]) - float(rl1)) <= 1e-5  # the replay saw the new contents, box included


def _photometric_block(fn, out, gt, bbox, mask, bg, faces):
    """ExAvatar's photometric terms (model.py:196-215 without LPIPS) through `fn`: rgb / ssim of both combined renders,
    the face composites, the random-background terms and the scene pair."""
    loss = 0.0
    for r, (face, is_face) in zip(("scene_human", "scene_human_refined"), faces):
        img = out[r]["img"]
        l1, s = fn(img, gt, bbox)
        loss = loss + 0.8 * l1 + 0.2 * (1 - s)
        l1f, _ = fn(img * (1 - is_face) + face * is_face, gt, bbox, ssim=False)
        loss = loss + 0.8 * l1f
    for r in ("human", "human_refined"):
        l1, _ = fn(out[r]["img"], gt * mask + (1 - mask) * bg[:, None, None], bbox, ssim=False)
        loss = loss + l1
    l1, s = fn(out["scene"]["img"], gt, mask=1 - mask)
    return loss + 0.8 * l1 + 0.2 * (1 - s)


@pytest.mark.gpu
def test_c4_training_frame_with_the_photometric_block(dev):
    from exavatar_release_b200 import TrainingFrameRenderer
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.synthetic import WORKLOADS, make_population_assets
    wl = WORKLOADS["C4"]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets("C4", seed=0, device=dev)
    Ps, Ph = scene["mean_3d"].shape[0], human["mean_3d"].shape[0]
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    bg_r = torch.tensor([0.3, 0.7, 0.2], device=dev)
    g = torch.Generator().manual_seed(13)
    gt = F.interpolate(torch.rand(1, 3, 32, 32, generator=g), size=(H, W), mode="bilinear")[0].to(dev)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1, 1, W), indexing="ij")
    mask = (1.5 - 2.0 * (xx ** 2 + (yy / 1.3) ** 2)).clamp(0, 1)[None].to(dev)
    bbox = torch.tensor([[85.3, 40.6, 330.2, 400.9]], device=dev)
    faces = []
    for _ in range(2):
        face = torch.rand(3, H, W, generator=g).to(dev)
        is_face = torch.zeros(1, H, W, device=dev)
        is_face[:, 100:180, 200:290] = 1.0
        faces.append((face, is_face))
    fr = TrainingFrameRenderer(Ps, Ph, (H, W), dev, {"A": 8_000_000, "B": 8_000_000})
    ref32 = lambda *a, **k: l1_ssim_reference(*a, dtype=torch.float32, **k)  # noqa: E731
    res = {}
    for arm, fn in (("op", l1_ssim), ("torch", ref32)):
        lv = [{k: v.detach().clone().requires_grad_() for k, v in d.items()} for d in (scene, human, refined)]
        out = fr(lv[0], lv[1], lv[2], cam, bg_r)
        loss = _photometric_block(fn, out, gt, bbox, mask, bg_r, faces)
        loss.backward()
        torch.cuda.synchronize()
        assert not fr.overflowed()
        res[arm] = (float(loss), lv)
    (l_op, g_op), (l_ref, g_ref) = res["op"], res["torch"]
    print(f"loss op {l_op:.7f} torch {l_ref:.7f}")
    assert abs(l_op - l_ref) <= 1e-5 * abs(l_ref)
    for d_op, d_ref in zip(g_op, g_ref):
        for k in d_ref:
            if d_ref[k].grad is None:
                assert d_op[k].grad is None, k
                continue
            r = d_ref[k].grad
            lim = 1e-4 * float(r.abs().max())
            diff = float((d_op[k].grad - r).abs().max())
            print(f"  {k}: max|d| {diff:.2e} ({diff / max(float(r.abs().max()), 1e-30):.2e} of max)")
            assert diff <= lim, (k, diff, lim)
