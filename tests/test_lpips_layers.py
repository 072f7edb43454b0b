"""The LPIPS op (csrc/lpips.cu) layer by layer against a TF32-exact float64 reference, through its C ABI.

The convolutions' arithmetic is fully specified: both operands rounded to TF32 by `cvt.rna` (nearest, ties away from
zero), products exact in fp32, fp32 accumulation.  So each conv is checked on its own, from the op's own fp32 input
(the saved ReLU output below it, max-pooled at a level change), against
    y_ref = relu(conv_f64(tf32(x), tf32(W)) + b),   per element |y_op - y_ref| <= c S,
    S = conv_f64(|tf32(x)|, |tf32(W)|) + |b|,
which leaves only the fp32 accumulation to the bound, and the reference has to explain the op's error: the RMS of
(y_op - y_ref) / S must be far below that of (y_op - y_unrounded) / S.  A staging path that rounds toward zero or
leaves an operand for the tensor core to truncate stays inside TF32 noise but fails here.

The backward is checked as a chain from the op's saved activations: the head's closed-form gradient, max-pool routing
to the first maximum of the op's own window values, ReLU masks from the op's outputs (a select), and every conv input
gradient as conv_transpose_f64(tf32(g * [act > 0]), tf32(W)) -- no ReLU or argmax can flip between op and reference.
After the backward the scratch holds the last image's level-0 gradients, from which conv1_2's input-gradient conv and
lp_conv0_bwd_kernel are checked in isolation.

Every shape also runs with its buffers prefilled with zeros and with NaN (outputs bit-identical), with 4 KiB of guard
bytes past `out`, `saved`, `scratch` and `dimg` (untouched), and with a small box right after a large one in the same
buffers (bit-identical to fresh buffers).

Without a device: `tf32` against hand-built bit patterns, the layer chain with rounding off against `lpips_reference`
on every golden case, and the saved-buffer reader against b2r_lpips_saved_bytes.

Measured on an H100 80GB HBM3 (SXM, 700 W power limit), worst case over every shape, image and layer of SHAPES, and
the bounds set from it:
    forward, TF32 convs      max |d|/S 1.52e-6 (relu5_2/5_3 at full HD)        C_F = 2^-18 = 3.8e-6
                             RMS ratio >= 28 (relu5_1 at full HD; 200+ at relu1_2)   RATIO_F = 20
    forward, conv1_1         max |d|/S 3.75e-7                                 C_0 = 2^-20 = 9.5e-7
    conv1_2 input gradient   max |d|/S 1.32e-6, RMS ratio >= 199                C_F, RATIO_F
    conv1_1 input gradient   max |d|/S 3.73e-7                                 C_0
    target taps              max relative error 1.9e-7; losses 3.0e-8         1e-6 both
    chained backward         max |d| / max|dimg_ref| 7.2e-4 (all taps), 9.3e-4 (one tap alone)   C_B = 2e-3
                             RMS ratio, relu1_2's head alone >= 28.3            RATIO_B = 7
The RMS ratio of the whole chained backward is 1.1 to 1.25 on every shape (3.4 to 4.0 for relu2_2's head alone, 1.1 to
1.5 above), so it is printed, not asserted.  That is the arithmetic, not a kernel fault: the backward's gradients
cancel heavily (S >> |g|), so an fp32 accumulation error far below the per-conv bound is comparable to g's TF32
quantum, and on a sizeable share of elements the next conv's rounding picks the other TF32 neighbour than the float64
chain does; these differences compound through the convs below.  Adding Gaussian noise of 3e-7 S to every conv output
of the float64 chain reproduces both the ratio (1.13) and the maximum (5.7e-4).  With one level in the chain (relu1_2's
head alone) the reference explains the op's error again, and the convs of the backward are checked on their own at
level 0.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from util import dev  # noqa: F401
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.losses import crop_box
from exavatar_release_b200.perceptual import EPS, LPIPS, SCALE, SHIFT, lpips_reference
from test_lpips import COUT, LEVEL, TAPS, _fixture, _GM, _weights, head_grad_closed_form

TAP_LAYER = (1, 3, 6, 9, 12)
GUARD = 4096

# Per-element bounds in units of S (the convs checked on their own) or of max|dimg_ref| (the chained backward), and
# the least RMS ratios; each bound is 2.5 to 3x the worst value measured (module docstring).
C_F = 2.0 ** -18      # TF32 convs: fp32 accumulation of exact products over up to 9 x 512 terms
C_0 = 2.0 ** -20      # conv1_1 and its input gradient: fp32 FMA chains over 27 and 9 x 64 terms on the CUDA cores
C_B = 2e-3            # the chained backward, relative to max|dimg_ref|
RATIO_F, RATIO_B = 20.0, 7.0


# ---------------------------------------------------------------------------------------------------------------------
# The TF32-exact reference (device-agnostic)
# ---------------------------------------------------------------------------------------------------------------------

def tf32(x):
    """fp32 -> TF32 as cvt.rna.tf32.f32 does it: round to nearest, ties away from zero, low 13 bits cleared.  Adding
    0x1000 to the bit pattern carries into the kept bits at or above the half-way point, for either sign (finite
    values only).  Held in float64, which represents the result exactly."""
    b = x.to(torch.float32).contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32).to(torch.float64)


class Weights:
    """The 13 convs' weights and biases and the 5 lin vectors in float64 on `dev`, the weights also TF32-rounded."""

    def __init__(self, dev):
        feats, lins = _weights()
        convs = [m for m in feats if isinstance(m, torch.nn.Conv2d)]
        self.w = [m.weight.detach().to(dev, torch.float64) for m in convs]
        self.w_tf32 = [tf32(m.weight.detach().to(dev)) for m in convs]
        self.b = [m.bias.detach().to(dev, torch.float64) for m in convs]
        self.lin = [w.detach().reshape(-1).to(dev, torch.float64) for w in lins]
        self.scale = torch.tensor(SCALE, dtype=torch.float32).to(dev, torch.float64).reshape(1, 3, 1, 1)
        self.shift = torch.tensor(SHIFT, dtype=torch.float32).to(dev, torch.float64).reshape(1, 3, 1, 1)


def scaled_crop(img, crop, wt, rounding):
    """conv1_1's input (1,3,h,w) float64: x*2-1 and the ScalingLayer on the crop.  rounding: each operation rounded to
    fp32 as lp_conv0_fwd_kernel evaluates it (float64 then fp32 is a correctly rounded fp32 operation on fp32
    operands); otherwise in float64 as `lpips_reference`."""
    x0, y0, x1, y1 = crop
    p = img[None, :, y0:y1, x0:x1].to(torch.float64)
    if not rounding:
        return ((p * 2 - 1) - wt.shift) / wt.scale
    r = lambda t: t.to(torch.float32).to(torch.float64)  # noqa: E731
    return r(r(r(p * 2 - 1) - wt.shift) / wt.scale)


def conv_ref(x, w, b):
    """(relu(conv(x, w) + b), S = conv(|x|, |w|) + |b|) in float64 with zero padding 1 at x's border."""
    return F.relu(F.conv2d(x, w, b, padding=1)), F.conv2d(x.abs(), w.abs(), b.abs(), padding=1)


def layer_input(acts, l):
    """Layer l's input (l >= 1): act[l-1], through the 2x2 floor max pool at a level change."""
    x = acts[l - 1]
    return F.max_pool2d(x, 2, 2) if LEVEL[l] != LEVEL[l - 1] else x


def forward_chain(img, crop, wt, rounding):
    """The 13 ReLU outputs (1,C,h_l,w_l) float64 of one image, each layer fed by the previous one."""
    acts = [conv_ref(scaled_crop(img, crop, wt, rounding), wt.w[0], wt.b[0])[0]]
    for l in range(1, 13):
        x = layer_input(acts, l)
        acts.append(conv_ref(tf32(x), wt.w_tf32[l], wt.b[l])[0] if rounding else conv_ref(x, wt.w[l], wt.b[l])[0])
    return acts


def normalise(f):
    return f / (torch.sqrt((f * f).sum(1, keepdim=True)) + EPS)


def head_loss(taps, nt, wt):
    """sum_t mean_p sum_c w_tc (n_c(f_t) - nt_tc)^2 in float64; taps and nt (1,C,h_t,w_t)."""
    return sum(float((w.reshape(1, -1, 1, 1) * (normalise(f) - n) ** 2).sum(1).mean())
               for f, n, w in zip(taps, nt, wt.lin))


def backward_chain(acts, nt, wt, dout, rounding, lin=None):
    """dL/dcrop (1,3,h,w) float64 for L = dout * loss (lin: other lin vectors than wt's), routed through `acts` (the
    op's saved ReLU outputs on the GPU):
    at each level the head's closed-form gradient plus the level above's input gradient routed to the first maximum
    of each pool window, then the level's conv input gradients, each conv_transpose(g * [act > 0], W) with both
    operands TF32-rounded (rounding) as the op stages them, and conv1_1's input gradient with the ScalingLayer's
    2 / scale."""
    g_in = None  # the gradient at the input of the level above (its pool's output)
    for t in range(4, -1, -1):
        f = acts[TAP_LAYER[t]]
        c, h, w = f.shape[1:]
        g = head_grad_closed_form(f.reshape(c, -1), nt[t].reshape(c, -1), (lin or wt.lin)[t],
                                  dout / (h * w)).reshape(f.shape)
        if g_in is not None:
            _, idx = F.max_pool2d(f, 2, 2, return_indices=True)  # torch's first-maximum rule, on the op's values
            g = g + F.max_unpool2d(g_in, idx, 2, 2, output_size=(h, w))
        l = TAP_LAYER[t]
        while l > 0 and LEVEL[l] == t:
            m = torch.where(acts[l] > 0, g, 0.0)  # a select: zero-norm tap pixels carry NaN
            g = F.conv_transpose2d(tf32(m), wt.w_tf32[l], padding=1) if rounding else \
                F.conv_transpose2d(m, wt.w[l], padding=1)
            l -= 1
        g_in = g
    return F.conv_transpose2d(torch.where(acts[0] > 0, g, 0.0), wt.w[0], padding=1) * 2 / wt.scale


def _up(v):
    return (v + 255) // 256 * 256


class Layout:
    """Byte offsets of lp_saved_layout / lp_scratch_layout: planes 256-byte aligned, act[l] (H >> lv, W >> lv, C_l)
    NHWC per image, the target's 5 taps after all N images; scratch plane A, plane B (64 x H x W floats each), then
    the heads' fp64 per-CTA partials (32 pixels a CTA)."""

    def __init__(self, W, H, N):
        self.W, self.H, self.N = W, H, N
        o, self.act = 0, []
        for l in range(13):
            self.act.append(o)
            o += _up(4 * COUT[l] * (H >> LEVEL[l]) * (W >> LEVEL[l]))
        self.image = o
        o, self.tap = N * self.image, []
        for t in range(5):
            self.tap.append(o)
            o += _up(4 * TAPS[t] * (H >> t) * (W >> t))
        self.saved = o
        self.plane_a, self.plane_b = 0, _up(4 * 64 * H * W)
        self.scratch = 2 * self.plane_b + sum(_up(8 * (((H >> t) * (W >> t) + 31) // 32)) for t in range(5))

    def plane(self, buf, off, level, c, crop):
        """The valid extent of a (H >> level, W >> level, c) plane at byte `off` of `buf`, as a (1,c,h_l,w_l) fp32
        view."""
        Hl, Wl = self.H >> level, self.W >> level
        t = buf[off:off + 4 * c * Hl * Wl].view(torch.float32).view(Hl, Wl, c)
        return t[:(crop[3] - crop[1]) >> level, :(crop[2] - crop[0]) >> level].permute(2, 0, 1)[None]

    def act_of(self, buf, n, l, crop):
        return self.plane(buf, n * self.image + self.act[l], LEVEL[l], COUT[l], crop)

    def tap_of(self, buf, t, crop):
        return self.plane(buf, self.tap[t], t, TAPS[t], crop)


# ---------------------------------------------------------------------------------------------------------------------
# The shape table
# ---------------------------------------------------------------------------------------------------------------------

# (id, H, W, N, box (None: the whole image), a smaller box run after it in the same buffers)
SHAPES = [
    # smallest legal image: level-4 extent 1x1, partial conv tiles from level 1 up; the small box is 15 wide (NaN loss)
    ("16x16", 16, 16, 2, None, (1.5, 0.2, 15.0, 16.0)),
    # odd sizes: W >> l and H >> l truncate at every level, a one-column tail tile at level 0
    ("17x33", 17, 33, 2, None, (3.7, 0.0, 17.2, 16.9)),
    # width 8 * 16 + 1: a single-column tail tile; height exactly 3 row tiles
    ("24x129", 24, 129, 2, None, (5.0, 3.0, 100.0, 17.0)),
    # tall and wide grids, partial head CTAs
    ("200x40", 200, 40, 2, None, (7.0, 21.0, 24.0, 101.0)),
    ("40x200", 40, 200, 2, None, (21.0, 7.0, 101.0, 24.0)),
    # tail tiles in x (16) and y (8) at levels 0 and 2, odd crop origins: valid w x h at level 0 | level 2
    ("136x200_97x63", 136, 200, 2, (37.6, 21.3, 97.4, 63.8), (10.5, 9.5, 40.2, 33.3)),     # 16k+1 x 8k-1 | 24 x 8k-1
    ("136x200_127x65", 136, 200, 2, (13.2, 7.9, 127.5, 65.1), (150.2, 90.9, 33.0, 40.0)),  # 16k-1 x 8k+1 | 16k-1 x 16
    ("136x200_132x71", 136, 200, 2, (51.0, 45.0, 132.0, 71.0), (0.0, 0.0, 17.0, 16.0)),    # 132 x 8k-1 | 16k+1 x 8k+1
    ("136x200_128x55", 136, 200, 2, (3.0, 61.0, 128.9, 55.5), (60.7, 3.3, 31.0, 47.0)),    # 16k x 8k-1 | 16k x 13
    # C4: per-image offsets in `saved` beyond image 1
    ("512x512_n3", 512, 512, 3, (85.3, 40.6, 330.2, 400.9), (200.3, 150.8, 64.0, 48.0)),
    # full HD: most CTAs exit early, size_t offsets
    ("1080x1920_n2", 1080, 1920, 2, (700.4, 301.7, 900.2, 500.6), (1500.6, 900.2, 160.0, 120.0)),
]


def target_index(N):
    """The image that is the target itself: never the last one, whose gradients the scratch keeps."""
    return (N - 1) // 2


def shape_inputs(H, W, N, seed):
    """(img (N,3,H,W), target (3,H,W)): smooth render-like images with noise; image target_index(N) is the target."""
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(N + 1, 3, max(H // 8, 2), max(W // 8, 2), generator=g), size=(H, W),
                         mode="bilinear")
    x = (base + 0.05 * torch.randn(N + 1, 3, H, W, generator=g)).clamp(0, 1)
    img = x[:N].clone()
    img[target_index(N)] = x[N]
    return img, x[N].clone()


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

def _bits(t):
    return t.to(torch.float32).view(torch.int32)


def test_tf32_rounds_to_nearest_with_ties_away_from_zero():
    one = 0x3F800000
    cases = [
        (one + 0x1000, one + 0x2000),                            # 1 + 2^-11 -> 1 + 2^-10: a tie, kept bits even
        ((one + 0x1000) | 0x80000000, (one + 0x2000) | 0x80000000),  # its negative: away from zero
        (one + 0x3000, one + 0x4000),                            # a tie with odd kept bits
        (one + 0x0FFF, one), (one + 0x1001, one + 0x2000),       # just below and just above the half-way point
        ((one + 0x0FFF) | 0x80000000, one | 0x80000000),
        (0x3FFFF800, 0x40000000),                                # 2 - 2^-12 -> 2: carry into the exponent
        (0x3FFFF000, 0x40000000),                                # 2 - 2^-11: a tie that carries
        (0xBFFFF000, 0xC0000000),
        (0x477FE000, 0x477FE000),                                # 65504, representable
        (one, one), (one + 0x2000, one + 0x2000), (0x3F000000, 0x3F000000), (0x40400000, 0x40400000),
        (0x00800000, 0x00800000), (0xBE6AA000, 0xBE6AA000),     # the smallest normal; a negative representable
        (0x00000000, 0x00000000), (0x80000000, 0x80000000),     # +0, -0
    ]
    src = torch.tensor([a - (1 << 32) if a >= 1 << 31 else a for a, _ in cases], dtype=torch.int32)
    want = torch.tensor([b - (1 << 32) if b >= 1 << 31 else b for _, b in cases], dtype=torch.int32)
    got = _bits(tf32(src.view(torch.float32)))
    for (a, b), g in zip(cases, got.tolist()):
        assert g & 0xFFFFFFFF == b, f"tf32({a:#010x}) = {g & 0xFFFFFFFF:#010x}, expected {b:#010x}"
    assert float(tf32(torch.tensor(1 + 2.0 ** -11))) == 1 + 2.0 ** -10
    assert float(tf32(torch.tensor(-(1 + 2.0 ** -11)))) == -(1 + 2.0 ** -10)
    assert float(tf32(torch.tensor(2 - 2.0 ** -12))) == 2.0
    assert torch.equal(got, want)


@pytest.mark.parametrize("name", [c[0] for c in _GM.LPIPS_CASES])
def test_layer_chain_without_rounding_reproduces_lpips_reference(name):
    """The layer-by-layer forward, the head loss and the chained backward, in float64 without TF32 rounding, are
    `lpips_reference` and its autograd gradient on every golden case (and the golden loss)."""
    c = _fixture()[name]
    feats, lins = _weights()
    wt = Weights("cpu")
    img, target = c["img"], c["target"]
    H, W = img.shape[-2:]
    crop = crop_box(c["bbox"], W, H)
    acts = forward_chain(img, crop, wt, False)
    nt = [normalise(forward_chain(target, crop, wt, False)[L_]) for L_ in TAP_LAYER]
    loss = head_loss([acts[L_] for L_ in TAP_LAYER], nt, wt)
    x = img.double().requires_grad_()
    ref = lpips_reference(x, target, c["bbox"], feats, lins)
    ref.sum().backward()
    ref = float(ref.detach())
    assert abs(loss - ref) <= 1e-12 * abs(ref), (loss, ref)
    assert abs(loss - c["loss"]) <= 1e-12 * abs(c["loss"]), (loss, c["loss"])
    dout = 1.0
    g = torch.zeros(1, 3, H, W, dtype=torch.float64)
    x0, y0, x1, y1 = crop
    g[:, :, y0:y1, x0:x1] = backward_chain(acts, nt, wt, dout, False)
    gmax = float(x.grad.abs().max())
    err = float((g[0] - x.grad).abs().max())
    print(f"{name}: |loss - ref| / ref {abs(loss - ref) / ref:.1e}  max|g - ref| / max|ref| {err / gmax:.1e}")
    assert err <= 1e-9 * gmax
    assert torch.equal(g[0] != 0, x.grad != 0)


def test_saved_layout_reader_matches_the_byte_counts():
    lib = L.load()
    for _, H, W, N, _, _ in SHAPES:
        lay = Layout(W, H, N)
        assert lay.saved == lib.b2r_lpips_saved_bytes(W, H, N), (W, H, N)
        assert lay.scratch == lib.b2r_lpips_scratch_bytes(W, H), (W, H)
        assert all(o % 256 == 0 for o in lay.act + lay.tap + [lay.image, lay.plane_b])
    # the reader's views cover exactly their planes
    lay = Layout(33, 17, 2)
    buf = torch.zeros(lay.saved, dtype=torch.uint8)
    for n in range(2):
        for l in range(13):
            lay.act_of(buf, n, l, (0, 0, 33, 17)).view(torch.int32).fill_(0x01010101)
    for t in range(5):
        lay.tap_of(buf, t, (0, 0, 33, 17)).view(torch.int32).fill_(0x01010101)
    want = 2 * sum(4 * COUT[l] * (17 >> LEVEL[l]) * (33 >> LEVEL[l]) for l in range(13)) + \
        sum(4 * TAPS[t] * (17 >> t) * (33 >> t) for t in range(5))
    assert int((buf != 0).sum()) == want


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

class Buffers:
    """out, saved, scratch and dimg, each followed by GUARD bytes of a pattern."""

    def __init__(self, lib, dev, W, H, N):
        self.size = dict(out=4 * N, saved=lib.b2r_lpips_saved_bytes(W, H, N),
                         scratch=lib.b2r_lpips_scratch_bytes(W, H), dimg=4 * N * 3 * H * W)
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


def _call(lib, op, bufs, img, target, box, dout, damage, lins=None):
    """Forward then backward through the C ABI into `bufs`; guard damage after each call is appended to `damage`.
    lins: the backward alone, with these 5 lin vectors in place of the op's."""
    N, _, H, W = img.shape
    b = None if box is None else torch.tensor(box, dtype=torch.float32, device=img.device)
    p = op._args(W, H, N, img, target, b)
    st = torch.cuda.current_stream(img.device).cuda_stream
    ptr = lambda k: bufs.raw[k].data_ptr()  # noqa: E731
    if lins is None:
        L.check(lib.b2r_lpips_forward(C.byref(p), ptr("out"), ptr("saved"), bufs.size["saved"], ptr("scratch"),
                                      bufs.size["scratch"], st), "b2r_lpips_forward")
        torch.cuda.synchronize()
        damage += [f"forward {box}: {k}" for k in bufs.damaged_guards()]
    else:
        for k in range(5):
            p.lin[k] = lins[k].data_ptr()
    L.check(lib.b2r_lpips_backward(C.byref(p), ptr("saved"), bufs.size["saved"], dout.data_ptr(), ptr("dimg"),
                                   ptr("scratch"), bufs.size["scratch"], st), "b2r_lpips_backward")
    torch.cuda.synchronize()
    damage += [f"backward {box}: {k}" for k in bufs.damaged_guards()]


def _outputs(bufs, lay, crop, N, H, W):
    """Copies of the loss, dimg, and the valid extents of every saved plane."""
    sv = bufs.body("saved")
    return {"out": bufs.body("out").view(torch.float32).clone(),
            "dimg": bufs.body("dimg").view(torch.float32).view(N, 3, H, W).clone(),
            **{f"act[{n}][{l}]": lay.act_of(sv, n, l, crop).clone() for n in range(N) for l in range(13)},
            **{f"tap[{t}]": lay.tap_of(sv, t, crop).clone() for t in range(5)}}


def _bit_differences(a, b):
    return [k for k in a if not torch.equal(a[k].view(torch.int32), b[k].view(torch.int32))]


class ShapeRun:
    """One shape of SHAPES through the op: the outputs of a NaN-prefilled run, plus the buffer-hygiene findings."""

    def __init__(self, lib, op, dev, name, H, W, N, box, small):
        self.name, self.H, self.W, self.N = name, H, W, N
        img, target = shape_inputs(H, W, N, seed=sum(map(ord, name)))
        self.img, self.target = img.to(dev), target.to(dev)
        self.ti = target_index(N)
        self.dout = torch.tensor([0.75, 1.5, 1.25][:N], dtype=torch.float32, device=dev)
        self.crop = crop_box(None if box is None else torch.tensor(box), W, H)
        small_crop = crop_box(torch.tensor(small), W, H)
        lay = Layout(W, H, N)
        bufs = Buffers(lib, dev, W, H, N)
        self.damage = []
        bufs.fill(float("nan"))
        _call(lib, op, bufs, self.img, self.target, box, self.dout, self.damage)
        o = _outputs(bufs, lay, self.crop, N, H, W)
        self.out, self.dimg = o["out"], o["dimg"]
        self.acts = [[o[f"act[{n}][{l}]"] for l in range(13)] for n in range(N)]
        self.taps = [o[f"tap[{t}]"] for t in range(5)]
        sc = bufs.body("scratch")
        # after the backward the ping-pong planes hold the last image's level-0 gradients (launch_lpips_backward:
        # level 4 starts on plane A and each conv writes the other plane, so level 1 hands plane A to level 0):
        # plane B the boundary output at relu1_2, plane A conv1_2's input gradient at relu1_1, before
        # lp_conv0_bwd_kernel applies relu1_1's mask
        self.grad_relu1_2 = lay.plane(sc, lay.plane_b, 0, 64, self.crop).clone()
        self.grad_relu1_1 = lay.plane(sc, lay.plane_a, 0, 64, self.crop).clone()
        # the backward with every lin vector but tap t's zeroed: dimg of the head of tap t alone
        self.dimg_tap = []
        for t in range(5):
            lins = [w if k == t else torch.zeros_like(w) for k, w in enumerate(op.lin)]
            _call(lib, op, bufs, self.img, self.target, box, self.dout, self.damage, lins)
            self.dimg_tap.append(bufs.body("dimg").view(torch.float32).view(N, 3, H, W).clone())
        bufs.fill(0.0)
        _call(lib, op, bufs, self.img, self.target, box, self.dout, self.damage)
        self.prefill_diff = _bit_differences(o, _outputs(bufs, lay, self.crop, N, H, W))
        del o
        self.reuse_damage = []
        _call(lib, op, bufs, self.img, self.target, small, self.dout, self.reuse_damage)  # after the large box
        after = _outputs(bufs, lay, small_crop, N, H, W)
        bufs.fill(float("nan"))
        _call(lib, op, bufs, self.img, self.target, small, self.dout, self.reuse_damage)
        self.reuse_diff = _bit_differences(after, _outputs(bufs, lay, small_crop, N, H, W))
        del after, bufs


@pytest.fixture(scope="module")
def op(dev):
    feats, lins = _weights()
    return LPIPS(feats, lins, dev)


@pytest.fixture(scope="module")
def wt(dev):
    return Weights(dev)


@pytest.fixture(scope="module", params=SHAPES, ids=[s[0] for s in SHAPES])
def run(request, dev, op):
    r = ShapeRun(L.load(), op, dev, *request.param)
    yield r
    del r
    torch.cuda.empty_cache()


def _rms(t):
    return float(torch.sqrt((t * t).mean()))


def _in_units_of(d, S, c):
    """(max d / S over S > 0, whether d <= c S everywhere -- so d == 0 wherever S == 0)."""
    ok = S > 0
    return (float((d[ok] / S[ok]).max()) if bool(ok.any()) else 0.0), bool((d <= c * S).all())


@pytest.mark.gpu
def test_forward_layers_match_the_tf32_reference(run, wt):
    """Every image, every layer, every element of the valid extent: |act_op - y_ref| <= c S from the op's own input,
    and the TF32-exact reference explains the op's error RATIO_F times better than the unrounded conv."""
    worst, least, bad = [0.0] * 13, [float("inf")] * 13, []
    for n in range(run.N):
        acts = run.acts[n]
        y, S = conv_ref(scaled_crop(run.img[n], run.crop, wt, True), wt.w[0], wt.b[0])
        mx, ok = _in_units_of((acts[0] - y).abs(), S, C_0)
        worst[0] = max(worst[0], mx)
        if not ok:
            bad.append((n, 0, "bound", mx))
        for l in range(1, 13):
            x = layer_input(acts, l).double()
            y, S = conv_ref(tf32(x), wt.w_tf32[l], wt.b[l])
            yu = conv_ref(x, wt.w[l], wt.b[l])[0]
            a = acts[l].double()
            mx, ok = _in_units_of((a - y).abs(), S, C_F)
            pos = S > 0
            ratio = _rms((a - yu)[pos] / S[pos]) / max(_rms((a - y)[pos] / S[pos]), 1e-300)
            worst[l], least[l] = max(worst[l], mx), min(least[l], ratio)
            if not ok:
                bad.append((n, l, "bound", mx))
            if ratio < RATIO_F:
                bad.append((n, l, "ratio", ratio))
            del x, y, S, yu, a, pos
    print(f"\n{run.name} forward max|d|/S by layer: " + " ".join(f"{v:.2e}" for v in worst))
    print(f"{run.name} forward RMS ratio by layer 1..12: " + " ".join(f"{v:.0f}" for v in least[1:]))
    assert not bad, bad


@pytest.mark.gpu
def test_target_taps_and_heads(run, wt):
    """The target's saved taps are the normalised taps of the same image passed as an image; that image's loss and
    gradient are exactly zero; the other images' losses are the float64 head on the op's saved taps."""
    ti = run.ti
    worst, taps_ok = 0.0, []
    for t in range(5):
        ref = normalise(run.acts[ti][TAP_LAYER[t]].double())
        mx, ok = _in_units_of((run.taps[t].double() - ref).abs(), ref.abs(), 1e-6)
        worst = max(worst, mx)
        taps_ok.append(ok)
    nt = [tp.double() for tp in run.taps]
    rels = [abs(float(run.out[n]) - ref) / ref for n in range(run.N) if n != ti
            for ref in [head_loss([run.acts[n][L_].double() for L_ in TAP_LAYER], nt, wt)]]
    print(f"\n{run.name} target taps max rel {worst:.1e}  loss rel " + " ".join(f"{r:.1e}" for r in rels))
    assert all(taps_ok), taps_ok
    assert float(run.out[ti]) == 0.0
    assert int((run.dimg[ti] != 0).sum()) == 0
    assert max(rels) <= 1e-6, rels


def _backward_errors(run, wt, n, dimg, lin=None):
    """(max|dimg_op - dimg_ref| / max|dimg_ref| over the crop, RMS ratio against the unrounded chain, whether dimg is
    finite and exactly zero outside the crop) for image n."""
    x0, y0, x1, y1 = run.crop
    acts = [a.double() for a in run.acts[n]]
    nt = [tp.double() for tp in run.taps]
    d = float(run.dout[n])
    ref = backward_chain(acts, nt, wt, d, True, lin)[0]
    unr = backward_chain(acts, nt, wt, d, False, lin)[0]
    outside = dimg[n].clone()
    outside[:, y0:y1, x0:x1] = 0
    clean = int((outside != 0).sum()) == 0 and bool(torch.isfinite(dimg[n]).all())
    op_ = dimg[n, :, y0:y1, x0:x1].double()
    return (float((op_ - ref).abs().max()) / float(ref.abs().max()),
            _rms(op_ - unr) / max(_rms(op_ - ref), 1e-300), clean)


@pytest.mark.gpu
def test_backward_matches_the_chained_reference(run, wt):
    """dimg of every non-target image against the chain routed through the op's saved activations: per element
    within C_B max|dimg_ref|, finite, and exactly zero outside the crop.  The RMS ratio against the unrounded chain
    is printed only: across all five levels it is about 1 (see the module docstring)."""
    res = {n: _backward_errors(run, wt, n, run.dimg) for n in range(run.N) if n != run.ti}
    for n, (mx, ratio, _) in res.items():
        print(f"\n{run.name} image {n} backward max|d|/max|ref| {mx:.2e}  RMS ratio {ratio:.2f}", end="")
    assert all(clean for _, _, clean in res.values()), res
    assert all(mx <= C_B for mx, _, _ in res.values()), res


@pytest.mark.gpu
def test_single_tap_backward_matches_the_chained_reference(run, wt):
    """The backward of each tap's head alone (the other lin vectors zeroed), for the last image: per element within
    C_B max|dimg_ref|; for relu1_2 alone -- one level, one TF32 rounding of the gradient before conv1_1's input
    gradient -- the TF32-exact chain must also explain the op's error RATIO_B times better than the unrounded one."""
    n = run.N - 1
    res = []
    for t in range(5):
        lin = [w if k == t else torch.zeros_like(w) for k, w in enumerate(wt.lin)]
        res.append(_backward_errors(run, wt, n, run.dimg_tap[t], lin))
    print(f"\n{run.name} image {n} single-tap backward max|d|/max|ref| by tap: "
          + " ".join(f"{mx:.2e}" for mx, _, _ in res) + "  RMS ratio: " + " ".join(f"{r:.1f}" for _, r, _ in res))
    assert all(clean for _, _, clean in res), res
    assert all(mx <= C_B for mx, _, _ in res), res
    assert res[0][1] >= RATIO_B, res[0]


@pytest.mark.gpu
def test_level0_backward_kernels_in_isolation(run, wt):
    """From the scratch planes the backward leaves (the last image's gradients at relu1_2 and relu1_1): conv1_2's
    input-gradient conv and lp_conv0_bwd_kernel per element against S, and conv1_2's RMS ratio, as the forward is
    checked."""
    n = run.N - 1
    x0, y0, x1, y1 = run.crop
    a0, a1 = run.acts[n][0].double(), run.acts[n][1].double()
    g1 = run.grad_relu1_1.double()
    m = torch.where(a1 > 0, run.grad_relu1_2.double(), 0.0)
    ref = F.conv_transpose2d(tf32(m), wt.w_tf32[1], padding=1)
    unr = F.conv_transpose2d(m, wt.w[1], padding=1)
    S = F.conv_transpose2d(tf32(m).abs(), wt.w_tf32[1].abs(), padding=1)
    e1, ok1 = _in_units_of((g1 - ref).abs(), S, C_F)
    pos = S > 0
    ratio = _rms((g1 - unr)[pos] / S[pos]) / max(_rms((g1 - ref)[pos] / S[pos]), 1e-300)
    m = torch.where(a0 > 0, g1, 0.0)
    ref = F.conv_transpose2d(m, wt.w[0], padding=1) * 2 / wt.scale
    S = F.conv_transpose2d(m.abs(), wt.w[0].abs(), padding=1) * 2 / wt.scale
    e0, ok0 = _in_units_of((run.dimg[n, :, y0:y1, x0:x1].double()[None] - ref).abs(), S, C_0)
    print(f"\n{run.name} image {n} conv1_2 input gradient max|d|/S {e1:.2e} RMS ratio {ratio:.0f}  "
          f"conv1_1 input gradient max|d|/S {e0:.2e}")
    assert ok1, e1
    assert ratio >= RATIO_F, ratio
    assert ok0, e0


@pytest.mark.gpu
def test_outputs_do_not_depend_on_buffer_contents(run):
    """Zero- and NaN-prefilled buffers give bit-identical losses, gradients and saved planes, and nothing is written
    past any buffer."""
    assert not run.damage, run.damage
    assert not run.prefill_diff, run.prefill_diff


@pytest.mark.gpu
def test_small_box_after_large_box_equals_fresh_buffers(run):
    assert not run.reuse_damage, run.reuse_damage
    assert not run.reuse_diff, run.reuse_diff
