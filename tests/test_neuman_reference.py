"""The NeuMan test-set scores (`metrics.NeumanScores`, csrc/metrics.cu) without a device: the PNG round trip against a
real cv2 round trip, the float64 restatement `neuman_scores_reference` against independent forms, the AlexNet taps
against torchvision, `from_lpips` on a stand-in with lpips' attribute layout, the SSIM window constants of the kernel,
and the C ABI (struct size, scratch layout, validation before any launch)."""
import copy
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from util import workload_settings  # noqa: F401  (path setup)
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.metrics import (ALEX_SLICES, SSIM_WINDOW, NeumanScores, _alex_convs, alex_taps_reference,
                                           composite, gaussian_window, neuman_scores_reference, png_round_trip)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 0x1000  # never dereferenced: validation fails before any launch
COUT = (64, 192, 384, 256, 256)


def alex_weights(seed=0):
    """torchvision's alexnet().features with the default initialisation from `seed`, and five non-negative lin
    vectors (lpips' trained lin weights are non-negative; the pretrained ones need a download)."""
    import torchvision
    torch.manual_seed(seed)
    feats = torchvision.models.alexnet(weights=None).features.eval()
    g = torch.Generator().manual_seed(seed + 1)
    lins = [torch.rand(1, c, 1, 1, generator=g) * 0.2 for c in COUT]
    return feats, lins


def _up(v):
    return (v + 255) // 256 * 256


def act_dims(H, W):
    """(h, w) of relu1 ... relu5 (conv 11x11 stride 4 pad 2, then 3x3 stride-2 floor pools before conv 2 and 3)."""
    d = [((H - 7) // 4 + 1, (W - 7) // 4 + 1)]
    p1 = ((d[0][0] - 3) // 2 + 1, (d[0][1] - 3) // 2 + 1)
    p2 = ((p1[0] - 3) // 2 + 1, (p1[1] - 3) // 2 + 1)
    return d + [p1] + [p2] * 3


class Layout:
    """Byte offsets of csrc/metrics.cu's nm_layout (regions 256-byte aligned; image i < N is render i, N + i target
    i): q (2N,3,H,W), in0 (2N,H,W,4), act[l] (2N,h_l,w_l,C_l) NHWC, pool 1 and pool 2, the pixel kernels' partials
    and the heads'."""

    def __init__(self, W, H, N):
        self.W, self.H, self.N = W, H, N
        I, HW = 2 * N, W * H
        self.dims = act_dims(H, W)
        o = 0
        self.q = o
        o += _up(4 * I * 3 * HW)
        self.in0 = o
        o += _up(4 * I * 4 * HW)
        self.act = []
        for (h, w), c in zip(self.dims, COUT):
            self.act.append(o)
            o += _up(4 * I * h * w * c)
        for (h, w), c in zip(self.dims[1:3], COUT[:2]):
            o += _up(4 * I * h * w * c)
        ctas = -(-W // 32) * -(-H // 16)
        o += 2 * _up(8 * N * 3 * ctas)
        for h, w in self.dims:
            o += _up(8 * N * -(-(h * w) // 32))
        self.total = o

    def images(self, buf):
        """q as a (2,N,3,H,W) fp32 view: [0] the renders, [1] the targets."""
        return buf[self.q:self.q + 4 * 2 * self.N * 3 * self.H * self.W].view(torch.float32).view(
            2, self.N, 3, self.H, self.W)

    def trunk_input(self, buf):
        """in0 as a (2N,3,H,W) fp32 view (channel 3, always zero, dropped)."""
        t = buf[self.in0:self.in0 + 4 * 2 * self.N * 4 * self.H * self.W].view(torch.float32)
        return t.view(2 * self.N, self.H, self.W, 4).permute(0, 3, 1, 2)[:, :3]

    def tap(self, buf, l):
        """act[l] as a (2N,C,h,w) fp32 view."""
        (h, w), c = self.dims[l], COUT[l]
        t = buf[self.act[l]:self.act[l] + 4 * 2 * self.N * h * w * c].view(torch.float32)
        return t.view(2 * self.N, h, w, c).permute(0, 3, 1, 2)


# ---------------------------------------------------------------------------------------------------------------------
# The PNG round trip
# ---------------------------------------------------------------------------------------------------------------------

def _cv2_round_trip(x, path):
    """What test.py and eval_neuman.py do: cv2.imwrite(path, x * 255) of an (H,W,3) float32 image, then
    torch.FloatTensor(cv2.imread(path) / 255.)."""
    cv2 = pytest.importorskip("cv2")
    assert cv2.imwrite(path, x * 255)
    return torch.FloatTensor(cv2.imread(path) / 255.)


def _restated(x):
    return png_round_trip(torch.from_numpy(x))


def _pixel_for(v):
    """An fp32 x with fl(x * 255) == v (the value cv2 rounds) where the neighbours of v / 255 reach it (255.7 is
    reached only approximately), else v / 255."""
    v = np.float32(v)
    x0 = x = np.float32(np.float64(v) / 255)
    if not np.isfinite(v):
        return v
    for _ in range(8):
        p = np.float32(x * np.float32(255))
        if p == v:
            return x
        x = np.nextafter(x, np.float32(np.inf) if p < v else np.float32(-np.inf))
    return x0


def test_round_trip_matches_cv2_on_the_edge_values(tmp_path):
    vs = [0.5, 1.5, 2.5, 255.7, -3.0, np.nan, np.inf, 1e10, 3.5, 254.5, 256.0, -0.4, -0.5, -0.6, -np.inf, -1e10,
          2.0 ** 31, 2.0 ** 31 - 128, -(2.0 ** 31), 0.0, 127.5, 128.5]
    x = np.array([_pixel_for(v) for v in vs], dtype=np.float32)
    x = np.repeat(x[:, None], 3, axis=1).reshape(1, -1, 3)
    got = _cv2_round_trip(x, str(tmp_path / "e.png"))
    want = _restated(x)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (got[0, :, 0], want[0, :, 0])
    # the values the protocol's description names: 0.5 -> 0, 1.5 -> 2, 2.5 -> 2, 255.7 -> 255, -3 -> 0, NaN, +inf and
    # 1e10 -> 0
    assert (want[0, :8, 0].double() * 255).round().tolist() == [0, 2, 2, 255, 0, 0, 0, 0]
    assert _pixel_for(0.5) * np.float32(255) == 0.5 and _pixel_for(2.5) * np.float32(255) == 2.5


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_round_trip_matches_cv2_on_random_images(tmp_path, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-0.2, 1.2, size=(37, 53, 3)).astype(np.float32)
    x[rng.random(x.shape) < 0.1] = (rng.integers(0, 256, size=1) + 0.5) / 255  # ties around the codes
    got = _cv2_round_trip(x, str(tmp_path / f"r{seed}.png"))
    assert torch.equal(got.view(torch.int32), _restated(x).view(torch.int32))


def test_round_trip_is_the_identity_on_the_256_codes(tmp_path):
    codes = (torch.arange(256, dtype=torch.float64) / 255).to(torch.float32)
    assert torch.equal(png_round_trip(codes).view(torch.int32), codes.view(torch.int32))
    x = codes.numpy().reshape(1, 256, 1).repeat(3, axis=2)
    assert torch.equal(_cv2_round_trip(x, str(tmp_path / "c.png"))[0, :, 0].view(torch.int32), codes.view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------------
# The float64 restatement
# ---------------------------------------------------------------------------------------------------------------------

def _codes(shape, seed, lo=0, hi=256):
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(lo, hi, shape, generator=g).double() / 255).float()


def test_identical_images_score_inf_one_zero():
    feats, lins = alex_weights()
    x = _codes((2, 3, 40, 47), 0)
    m = torch.rand(2, 1, 40, 47, generator=torch.Generator().manual_seed(1))
    for mask in (None, m):
        s = neuman_scores_reference(x, x, mask, feats, lins)
        assert torch.isinf(s[:, 0]).all() and (s[:, 0] > 0).all()
        assert torch.equal(s[:, 1], torch.ones(2, dtype=torch.float64))
        assert torch.equal(s[:, 2], torch.zeros(2, dtype=torch.float64))


def test_constant_offset_psnr():
    feats, lins = alex_weights()
    for k in (1, 7, 40):
        x = _codes((1, 3, 33, 35), k, 0, 256 - k)
        y = ((x.double() * 255).round() + k).div(255).float()  # every element k codes above
        d = k / 255
        s = neuman_scores_reference(x, y, None, feats, lins)
        assert abs(float(s[0, 0]) - (-10 * math.log10(d * d))) <= 1e-5, (k, float(s[0, 0]))


def test_ssim_matches_a_scipy_restatement_over_the_valid_centres():
    from scipy.ndimage import correlate
    feats, lins = alex_weights()
    g = np.array(SSIM_WINDOW)
    win = np.outer(g, g)
    H, W = 41, 58
    x = _codes((2, 3, H, W), 3)
    y = (x + 0.08 * torch.randn(2, 3, H, W, generator=torch.Generator().manual_seed(4))).clamp(0, 1)
    m = (torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(5)) > 0.3).float()
    s = neuman_scores_reference(x, y, m, feats, lins)
    xq = composite(png_round_trip(x), m).double().numpy()
    yq = composite(png_round_trip(y), m).double().numpy()
    for n in range(2):
        vals = []
        for c in range(3):
            a, b = xq[n, c], yq[n, c]
            f = lambda t: correlate(t, win, mode="reflect")[5:-5, 5:-5]  # noqa: E731
            ma, mb = f(a), f(b)
            va, vb, cab = np.maximum(f(a * a) - ma * ma, 0), np.maximum(f(b * b) - mb * mb, 0), f(a * b) - ma * mb
            c1, c2 = 0.01 ** 2, 0.03 ** 2
            vals.append(((2 * ma * mb + c1) * (2 * cab + c2)) / ((ma * ma + mb * mb + c1) * (va + vb + c2)))
        want = float(np.mean(vals))
        assert abs(float(s[n, 1]) - want) <= 1e-12, (n, float(s[n, 1]), want)


def test_alex_taps_equal_torchvision_slices():
    feats, _ = alex_weights()
    x = torch.randn(2, 3, 67, 71, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    taps = alex_taps_reference(x, feats)
    h = x
    f64 = copy.deepcopy(feats).double()
    for t, (a, b) in zip(taps, ALEX_SLICES):
        h = f64[a:b](h)
        assert t.shape == h.shape
        assert torch.equal(t, h)


class _Lin(torch.nn.Module):
    def __init__(self, c):
        super().__init__()
        self.model = torch.nn.Sequential(torch.nn.Dropout(), torch.nn.Conv2d(c, 1, 1, bias=False))


class _StandIn(torch.nn.Module):
    """lpips.LPIPS(net='alex')'s attribute layout: net.slice1..5 holding alexnet().features[0:12] under torchvision's
    child indices, and lin0..4.model[-1].weight."""

    def __init__(self, feats):
        super().__init__()
        self.net = torch.nn.Module()
        for k, (a, b) in enumerate(ALEX_SLICES):
            s = torch.nn.Sequential()
            for i in range(a, b):
                s.add_module(str(i), feats[i])
            setattr(self.net, f"slice{k + 1}", s)
        for k, c in enumerate(COUT):
            setattr(self, f"lin{k}", _Lin(c))


def test_from_lpips_reads_the_convs_and_lin_weights():
    feats, _ = alex_weights()
    m = _StandIn(feats)

    class Probe(NeumanScores):
        def __init__(self, f, lins, device):
            self.args = (f, lins, device)

    f, lins, dev = Probe.from_lpips(m).args
    convs = _alex_convs(f)
    assert [c is feats[i] for c, i in zip(convs, (0, 3, 6, 8, 10))] == [True] * 5
    assert all(w is getattr(m, f"lin{k}").model[-1].weight for k, w in enumerate(lins))
    assert dev == torch.device("cpu")
    del m.net.slice5._modules["11"]
    with pytest.raises(ValueError, match="slice1..5"):
        Probe.from_lpips(m)
    with pytest.raises(ValueError, match="module 3"):
        _alex_convs(torch.nn.Sequential(*[feats[i] if i != 3 else torch.nn.Conv2d(64, 192, 3) for i in range(12)]))


def test_the_kernel_holds_torchmetrics_window():
    """The kernel's constants are SSIM_WINDOW (the CUDA build, checked bit for bit on the GPU), which is fp32, symmetric,
    and within 8 ulps of the CPU build of the same expression (the outer taps differ most)."""
    src = open(os.path.join(ROOT, "exavatar_release_b200", "csrc", "metrics.cu")).read()
    body = re.search(r"c_nm_gauss\[11\] = \{(.*?)\};", src, re.S).group(1)
    vals = torch.tensor([float.fromhex(v.strip().rstrip("f")) for v in body.split(",")], dtype=torch.float64)
    want = torch.tensor(SSIM_WINDOW, dtype=torch.float64)
    assert torch.equal(vals, want)
    assert torch.equal(want.float().double(), want) and torch.equal(want, want.flip(0))
    ulps = (want.float().view(torch.int32) - gaussian_window().view(torch.int32)).abs()
    assert int(ulps.max()) <= 8, ulps


# ---------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------

def test_struct_size_and_scratch_layout():
    lib = L.load()
    for W, H, N in ((31, 31, 1), (53, 37, 2), (511, 255, 3), (512, 512, 2), (1920, 1080, 1)):
        assert lib.b2r_neuman_scratch_bytes(W, H, N) == Layout(W, H, N).total, (W, H, N)
    assert Layout(31, 31, 1).dims[-1] == (1, 1)


def _valid():
    p = L.B2RNeumanScores(width=64, height=48, n_images=2, mask_channels=0, render=FAKE, target=FAKE)
    for k in range(5):
        p.w[k] = p.bias[k] = p.lin[k] = FAKE
    return p


def test_host_validation_returns_its_codes_before_any_launch():
    lib = L.load()
    launches = lib.b2r_launch_count()
    need = lib.b2r_neuman_scratch_bytes(64, 48, 2)
    run = lambda p, out=FAKE, scratch=FAKE, n=need: lib.b2r_neuman_scores(  # noqa: E731
        None if p is None else C.byref(p), out, scratch, n, None)
    assert run(None) == -1
    for field, bad in (("width", 30), ("height", 30), ("n_images", 0), ("render", None), ("target", None)):
        p = _valid()
        setattr(p, field, bad)
        assert run(p) == -1, field
    for arr in ("w", "bias", "lin"):
        for k in range(5):
            p = _valid()
            getattr(p, arr)[k] = None
            assert run(p) == -1, (arr, k)
    p = _valid()
    p.mask_channels = 1  # a channel count without a mask
    assert run(p) == -1
    p.mask = FAKE
    for mc in (0, 2, 4, -1):
        p.mask_channels = mc
        assert run(p) == -1, mc
    p = _valid()
    assert run(p, out=None) == -1 and run(p, scratch=None) == -1
    assert run(p, n=need - 1) == -2
    p.width, p.height = 1 << 15, 1 << 14
    assert run(p) == -1  # more than 2^28 pixels
    assert lib.b2r_launch_count() == launches
