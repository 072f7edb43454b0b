"""`NeumanScores` (csrc/metrics.cu) on the GPU, through its C ABI and its Python call.

For every case of CASES (odd sizes, 31 x 31 up to 1080 x 1920, N = 1..3, no mask, 1- and 3-channel masks, binary and
fractional), with scratch prefilled with NaN and 4 KiB of guard bytes past `out` and `scratch`:
  * the quantised, composited images and the trunk's input in the scratch are bit-identical to torch's fp32 expressions;
  * PSNR and SSIM match the float64 restatement;
  * each AlexNet conv, fed from the op's own input (pooled in float64 from the op's previous tap), is within c S per
    element of relu(conv_f64(tf32(x), tf32(W)) + b), S = conv_f64(|tf32(x)|, |tf32(W)|) + |b|, and that TF32-exact
    reference explains the op's error RATIO times better than the unrounded conv (the rounding is cvt.rna's);
  * LPIPS matches the float64 head on the op's own taps, and the unrounded float64 reference within LPIPS_TOL;
  * a zero-prefilled run gives the same bits and no guard byte changes.
Then: identical frames give psnr inf and lpips 0 exactly, and ssim exactly 1 without flat windows; two calls are
bit-identical; nothing syncs; a captured CUDA graph replayed with new images equals eager; the device-built SSIM
window equals the kernel's constants.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from util import capture, no_host_sync
from util import dev  # noqa: F401
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.metrics import (ALEX_CONVS, SSIM_WINDOW, NeumanScores, composite, gaussian_window,
                                           neuman_scores_reference, png_round_trip)
from exavatar_release_b200.perceptual import EPS, SCALE, SHIFT
from test_lpips_layers import tf32
from test_neuman_reference import Layout, alex_weights

GUARD = 4096
# Bounds, each about 3x the worst value measured on the H100 (DESIGN.md section 8, row f-17)
C_F = 2.0 ** -18        # TF32 convs: fp32 accumulation of exact products over up to 3456 terms, in units of S
RATIO = 12.0            # least RMS ratio (unrounded reference error / TF32-exact reference error)
PSNR_TOL = 2e-6         # dB
SSIM_TOL = 1e-7
HEAD_TOL = 2e-7         # relative: LPIPS against the float64 head on the op's own taps
LPIPS_TOL = 1.5e-3      # relative: LPIPS against the unrounded float64 reference

# (id, H, W, N, mask: None or (channels, fractional))
CASES = [
    ("31x31_n1", 31, 31, 1, None),
    ("37x53_n2_m1", 37, 53, 2, (1, False)),
    ("53x37_n3_m3f", 53, 37, 3, (3, True)),
    ("255x511_n3_m1f", 255, 511, 3, (1, True)),
    ("512x512_n2_m3", 512, 512, 2, (3, False)),
    ("1080x1920_n1_m1f", 1080, 1920, 1, (1, True)),
]


def case_inputs(H, W, N, mask, seed):
    """(render, target, mask) on the CPU: smooth render-like images with noise, values a little outside [0,1], a few
    NaN / inf / code-tie pixels in the render; the target read from an 8-bit PNG (codes n / 255); a blob-shaped
    mask."""
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(N, 3, max(H // 8, 2), max(W // 8, 2), generator=g), size=(H, W), mode="bilinear")
    render = base * 1.2 - 0.1 + 0.03 * torch.randn(N, 3, H, W, generator=g)
    flat = render.view(-1)
    idx = torch.randint(0, flat.numel(), (64,), generator=g)
    flat[idx[:8]] = float("nan")
    flat[idx[8:12]] = float("inf")
    flat[idx[12:]] = ((torch.randint(0, 255, (52,), generator=g).double() + 0.5) / 255).float()
    target = ((base + 0.05 * torch.randn(N, 3, H, W, generator=g)).clamp(0, 1) * 255).round().double().div(255).float()
    m = None
    if mask is not None:
        ch, frac = mask
        blob = F.interpolate(torch.rand(N, ch, max(H // 16, 4), max(W // 16, 4), generator=g), size=(H, W),
                             mode="bilinear")
        m = blob if frac else (blob > 0.5).float()
    return render, target, m


class Buffers:
    """out and scratch, each followed by GUARD bytes of a pattern."""

    def __init__(self, lib, dev, W, H, N):
        self.size = dict(out=4 * 3 * N, scratch=lib.b2r_neuman_scratch_bytes(W, H, N))
        self.raw = {k: torch.empty(n + GUARD, dtype=torch.uint8, device=dev) for k, n in self.size.items()}
        self.pattern = ((torch.arange(GUARD) * 151 + 89) % 256).to(torch.uint8).to(dev)

    def body(self, k):
        return self.raw[k][:self.size[k]]

    def fill(self, value):
        for k, t in self.raw.items():
            self.body(k).view(torch.float32).fill_(value)
            t[self.size[k]:].copy_(self.pattern)

    def damaged_guards(self):
        return [k for k, t in self.raw.items() if not torch.equal(t[self.size[k]:], self.pattern)]


def _call(lib, op, bufs, render, target, mask):
    N, _, H, W = render.shape
    p = op._args(W, H, N, render, target, mask, 0 if mask is None else mask.shape[1])
    L.check(lib.b2r_neuman_scores(C.byref(p), bufs.raw["out"].data_ptr(), bufs.raw["scratch"].data_ptr(),
                                  bufs.size["scratch"], torch.cuda.current_stream().cuda_stream), "b2r_neuman_scores")
    torch.cuda.synchronize()


class CaseRun:
    """One case through the C ABI: copies of the outputs, the composited images, the trunk input and the taps of a
    NaN-prefilled run, and the buffer-hygiene findings of it and a zero-prefilled run."""

    def __init__(self, lib, op, dev, name, H, W, N, mask):
        self.name, self.H, self.W, self.N = name, H, W, N
        r, t, m = case_inputs(H, W, N, mask, seed=sum(map(ord, name)))
        self.render, self.target = r.to(dev), t.to(dev)
        self.mask = None if m is None else m.to(dev)
        lay = Layout(W, H, N)
        bufs = Buffers(lib, dev, W, H, N)
        bufs.fill(float("nan"))
        _call(lib, op, bufs, self.render, self.target, self.mask)
        self.damage = bufs.damaged_guards()
        sc = bufs.body("scratch")
        self.out = bufs.body("out").view(torch.float32).view(N, 3).clone()
        self.q = lay.images(sc).clone()
        self.in0 = lay.trunk_input(sc).clone()
        self.taps = [lay.tap(sc, k).clone() for k in range(5)]
        bufs.fill(0.0)
        _call(lib, op, bufs, self.render, self.target, self.mask)
        self.damage += bufs.damaged_guards()
        self.prefill_diff = [k for k, a, b in
                             [("out", self.out, bufs.body("out").view(torch.float32).view(N, 3)),
                              ("q", self.q, lay.images(sc)), ("in0", self.in0, lay.trunk_input(sc))] +
                             [(f"tap{k}", self.taps[k], lay.tap(sc, k)) for k in range(5)]
                             if not torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))]
        del bufs


@pytest.fixture(scope="module")
def weights():
    return alex_weights()


@pytest.fixture(scope="module")
def op(dev, weights):
    return NeumanScores(*weights, dev)


@pytest.fixture(scope="module", params=CASES, ids=[c[0] for c in CASES])
def run(request, dev, op):
    r = CaseRun(L.load(), op, dev, *request.param)
    yield r
    del r
    torch.cuda.empty_cache()


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.gpu
def test_composited_images_and_trunk_input_are_torchs_fp32_expressions(run):
    m = run.mask
    want = [composite(png_round_trip(t), m) for t in (run.render, run.target)]
    assert torch.equal(_bits(run.q[0]), _bits(want[0]))
    assert torch.equal(_bits(run.q[1]), _bits(want[1]))
    shift = torch.tensor(SHIFT, dtype=torch.float32, device=m.device if m is not None else run.render.device)
    scale = torch.tensor(SCALE, dtype=torch.float32, device=shift.device)
    x = torch.cat(want)
    assert torch.equal(_bits(run.in0), _bits(((x * 2 - 1) - shift[None, :, None, None]) / scale[None, :, None, None]))


@pytest.mark.gpu
def test_buffers_do_not_change_the_outputs(run):
    assert not run.damage, run.damage
    assert not run.prefill_diff, run.prefill_diff


@pytest.mark.gpu
def test_scores_match_the_float64_reference(run, weights):
    """PSNR and SSIM against the float64 restatement on the same composited images; LPIPS against the unrounded
    float64 trunk (the op's convolutions are TF32).  A frame whose composited images are equal scores inf / 1 / 0 on
    both sides."""
    ref = neuman_scores_reference(run.render, run.target, run.mask, *weights).cpu()
    out = run.out.double().cpu()
    same = torch.isinf(ref[:, 0])
    assert torch.equal(torch.isinf(out[:, 0]), same)
    assert torch.equal(out[same, 1:], ref[same, 1:]) and (ref[same, 1:] == torch.tensor([1.0, 0.0])).all()
    dp = float((out[~same, 0] - ref[~same, 0]).abs().max())
    ds = float((out[:, 1] - ref[:, 1]).abs().max())
    dl = float(((out[~same, 2] - ref[~same, 2]).abs() / ref[~same, 2]).max())
    print(f"\n{run.name} psnr {out[:, 0].tolist()} |d| {dp:.2e}  ssim |d| {ds:.2e}  lpips {out[:, 2].tolist()} "
          f"rel d vs unrounded {dl:.2e}")
    assert dp <= PSNR_TOL and ds <= SSIM_TOL
    assert dl <= LPIPS_TOL


def _conv_input(run, k):
    """Conv k's input from the op's own buffers, float64 (2N,C,h,w): the trunk input, or the previous tap, max-pooled
    before convs 1 and 2."""
    if k == 0:
        return run.in0.double()
    x = run.taps[k - 1].double()
    return F.max_pool2d(x, 3, 2) if k in (1, 2) else x


def _rms(t):
    return float(torch.sqrt((t * t).mean()))


@pytest.mark.gpu
def test_each_conv_matches_the_tf32_reference(run, weights):
    feats, _ = weights
    worst, least, bad = [], [], []
    for k, (i, _, _, _, s, p) in enumerate(ALEX_CONVS):
        conv = feats[i]
        w = conv.weight.detach().to(run.in0.device)
        b = conv.bias.detach().to(run.in0.device).double()
        x = _conv_input(run, k)
        y = F.relu(F.conv2d(tf32(x), tf32(w), b, stride=s, padding=p))
        S = F.conv2d(tf32(x).abs(), tf32(w).abs(), b.abs(), stride=s, padding=p)
        yu = F.relu(F.conv2d(x, w.double(), b, stride=s, padding=p))
        a = run.taps[k].double()
        d = (a - y).abs()
        pos = S > 0
        mx = float((d[pos] / S[pos]).max())
        ratio = _rms((a - yu)[pos] / S[pos]) / max(_rms((a - y)[pos] / S[pos]), 1e-300)
        worst.append(mx)
        least.append(ratio)
        if not bool((d <= C_F * S).all()):
            bad.append((k, "bound", mx))
        if ratio < RATIO:
            bad.append((k, "ratio", ratio))
        del x, y, S, yu, a, d, pos
    print(f"\n{run.name} conv max|d|/S " + " ".join(f"{v:.2e}" for v in worst) + "  RMS ratio "
          + " ".join(f"{v:.0f}" for v in least))
    assert not bad, bad


@pytest.mark.gpu
def test_lpips_is_the_head_of_the_ops_taps(run, weights):
    _, lins = weights
    N = run.N
    got = []
    for n in range(N):
        v = 0.0
        for k in range(5):
            fx, fy = run.taps[k][n].double(), run.taps[k][N + n].double()
            nx = fx / (torch.sqrt((fx * fx).sum(0, keepdim=True)) + EPS)
            ny = fy / (torch.sqrt((fy * fy).sum(0, keepdim=True)) + EPS)
            w = lins[k].detach().reshape(-1, 1, 1).to(fx.device).double()
            v += float((w * (nx - ny) ** 2).sum(0).mean())
        got.append(v)
    rel = max(abs(float(run.out[n, 2]) - got[n]) / max(got[n], 1e-30) for n in range(N))
    print(f"\n{run.name} lpips vs head on the op's taps: rel {rel:.2e}")
    assert rel <= HEAD_TOL


@pytest.mark.gpu
def test_identical_frames_score_exactly(dev, op, weights):
    """Identical frames: psnr +inf and lpips exactly 0.  SSIM is exactly 1 when no window is flat; a flat window of
    value v has E[x^2] - mu^2 = v^2 S (1 - S) < 0 with the window's sum S = 1 + 3.9e-8, which torchmetrics clamps to
    0 for the variances but not for the covariance, so frames with flat areas (clamped pixels, the white background)
    score just under 1 -- as the float64 restatement does."""
    g = torch.Generator().manual_seed(3)
    noise = (torch.randint(1, 255, (2, 3, 64, 96), generator=g).double() / 255).float().to(dev)
    out = op(noise, noise.clone()).cpu()
    assert torch.isinf(out[:, 0]).all() and (out[:, 0] > 0).all(), out
    assert torch.equal(out[:, 1:], torch.tensor([[1.0, 0.0], [1.0, 0.0]])), out
    for H, W, N, mask in ((31, 31, 1, None), (255, 511, 2, (3, True)), (1080, 1920, 1, (1, False))):
        r, _, m = case_inputs(H, W, N, mask, seed=H)
        r, m = r.to(dev), None if m is None else m.to(dev)
        out = op(r, r.clone(), m).cpu()
        ref = neuman_scores_reference(r, r, m, *weights).cpu()
        assert torch.isinf(out[:, 0]).all() and (out[:, 0] > 0).all(), out
        assert torch.equal(out[:, 2], torch.zeros(N)), out
        assert float((out[:, 1].double() - ref[:, 1]).abs().max()) <= SSIM_TOL, (out, ref)
        assert bool((out[:, 1] <= 1).all()), out


@pytest.mark.gpu
def test_repeatable_sync_free_and_graph_capturable(dev, op):
    H, W, N = 255, 511, 2
    r, t, m = (v.to(dev) for v in case_inputs(H, W, N, (1, True), seed=7))
    a = op(r, t, m)
    b = op(r, t, m)
    assert torch.equal(_bits(a), _bits(b))
    with no_host_sync():
        c = op(r, t, m)
    assert torch.equal(_bits(a), _bits(c))
    # a graph captured on one set of images, replayed on another
    sr, st, sm = r.clone(), t.clone(), m.clone()
    g, gout = capture(lambda: op(sr, st, sm), 1)
    r2, t2, m2 = (v.to(dev) for v in case_inputs(H, W, N, (1, True), seed=8))
    sr.copy_(r2)
    st.copy_(t2)
    sm.copy_(m2)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(gout), _bits(op(r2, t2, m2)))
    assert not torch.equal(_bits(gout), _bits(a))
    # unbatched frames are N = 1
    one = op(r[1], t[1], m[1])
    assert one.shape == (1, 3) and torch.equal(_bits(one[0]), _bits(a[1]))


@pytest.mark.gpu
def test_device_window_equals_the_kernel_constants(dev):
    """torchmetrics builds its window on the images' device: those are the kernel's bits."""
    assert torch.equal(_bits(gaussian_window(dev).cpu()), _bits(torch.tensor(SSIM_WINDOW, dtype=torch.float32)))


@pytest.mark.gpu
def test_argument_checks(dev, op):
    x = torch.rand(2, 3, 40, 40, device=dev)
    with pytest.raises(ValueError, match="at least 31"):
        op(x[..., :30], x[..., :30])
    with pytest.raises(ValueError, match="does not match"):
        op(x, x[:1])
    with pytest.raises(ValueError, match="mask"):
        op(x, x, torch.rand(2, 2, 40, 40, device=dev))
    with pytest.raises(ValueError, match="float32"):
        op(x, x.double())
    with pytest.raises(RuntimeError, match="CUDA"):
        op(x.cpu(), x.cpu())
