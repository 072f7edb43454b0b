"""`TriplaneFeatures` and `gn_mlp` (csrc/triplane.cu, csrc/gn_mlp.cu) at the shapes and edges the C4-sized tests in
test_human_nets.py never reach (those run P = 167 618 rows, K = 96 / 99, H = 3 / 4 and 3x32x128x128 planes).

The kernels change behaviour at these boundaries:
  gn_mlp    16-row tiles, 8 warps per CTA and at most 132 CTAs, so below 132 x 8 x 16 = 16 896 rows the grid is
            partial; the backward chain kernel always launches 132 CTAs and those without a tile still write a zero
            partial; the weight gradients are summed over 1024-row chunks in runs of max(8, ceil(n / 32)) partials,
            longer than 8 above 262 144 rows; first-layer widths K that are not a multiple of 8 (the KT / NT / KB
            tails) up to 128; 1 to 4 head outputs; constant blocks folded into the first bias before, between or
            after the per-row blocks.
  triplane  the backward strides a texel's C channels over the lanes of a warp (C > 32 takes a second trip, C < 32
            leaves lanes idle); non-square planes; texels no row samples and texels every row samples; samples on
            texel centres, texel edges, the +-1 border and beyond it.

These tests pin
  * without a device: gn_mlp_reference against the fp32 modules run in float64 for every new layout, and the exact
    sample grid of mirrored dyadic positions, which places the GPU cases' samples exactly;
  * on the GPU: gn_mlp against float64 over P, K and H; row results that do not depend on P or on the row's place
    in its tile; a no-grad forward that keeps nothing for the backward and gives the same bits; a backward without
    dX that gives the same parameter gradients; the bias gradients of mirrored rows; TriplaneFeatures over C, plane
    shape, P and face sets; and both ops through their C ABI with every output and scratch buffer filled with NaN and
    padded with a sentinel, so that a value left unwritten or written past the end shows.
"""
import copy
import ctypes as C

import pytest
import torch

from util import dev  # noqa: F401
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.human_nets import (TriplaneFeatures, bilinear_corners, gn_mlp, gn_mlp_reference,
                                              tri_feature_reference, triplane_grid)
from test_human_nets import _blend64, _params, _relu_edge_rows, _torch_module_forward, gn_stack

# Floor of the comparison with torch's fp32 error, relative to max|float64|: at a few rows torch's own error can be
# close to 0, so twice it is no yardstick there.  Measured on an H100 80GB HBM3 (700 W power limit) over every gn_mlp
# case below: where the op's error exceeds twice torch's, it is at most 6.8e-7 of max|float64| (P = 1, the output).
FLOOR = 1e-6
SENTINEL = 1234.5  # finite, written past the end of every output buffer of the C ABI tests
PAD = 64

HEADS = {1: (None, 1), 2: ([1, 1], None), 3: (None, 3), 4: ([3, 1], None)}  # H: (head widths, final Linear)
LAYOUTS = {  # name: (first-layer blocks (kind, width) in column order, head widths, final Linear)
    "const_first": ((("c", 4), ("row", 13)), [3, 1], None),
    "const_between": ((("row", 5), ("c", 7), ("row", 6)), None, 3),
    "k1": ((("row", 1),), [3, 1], None),
    "k128": ((("row", 128),), [3, 1], None),
    "h1": ((("row", 96),), None, 1),
    "h2": ((("row", 96),), [1, 1], None),
}
GEO_NET = ((("row", 96),), [3, 1], None)

PLANES = [(1, 1), (2, 3), (37, 64), (64, 37), (128, 128)]
TRI_CASES = [  # (C, (H, W), P, face rows, placement)
    (1, (37, 64), 4099, "mix", "spread"),
    (33, (37, 64), 85, "all", "spread"),
    (33, (64, 37), 4099, "mix", "spread"),
    (1, (64, 37), 85, "none", "spread"),
    (5, (1, 1), 2, "all", "spread"),
    (33, (2, 3), 2, "none", "spread"),
    (64, (2, 3), 85, "mix", "spread"),
    (32, (128, 128), 4099, "mix", "spread"),
    (64, (128, 128), 1, "none", "point"),
    (5, (2, 3), 4099, "none", "point"),
    (32, (1, 1), 85, "all", "point"),
]


def _tri_id(case):
    c, (h, w), p, face, placement = case
    return f"C{c}-{h}x{w}-P{p}-{face}-{placement}"


# ---------------------------------------------------------------------------------------------------------------------
# Inputs
# ---------------------------------------------------------------------------------------------------------------------

def _stack(blocks, head_widths, final, seed=0, device="cpu"):
    """gn_stack over the blocks' columns with a non-trivial GroupNorm affine."""
    torch.manual_seed(seed)
    trunk, heads = gn_stack(sum(k for _, k in blocks), head_widths, final)
    with torch.no_grad():
        for l in range(3):
            trunk[3 * l + 1].weight.uniform_(0.5, 1.5)
            trunk[3 * l + 1].bias.uniform_(-0.3, 0.3)
    return trunk.to(device), [h.to(device) for h in heads]


def _out_width(head_widths, final):
    return sum(head_widths) if head_widths else final


def _inputs(blocks, P, seed, device="cpu"):
    """A (P,k) block per "row" and a (k,) block per "c", drawn on the CPU so that every device sees the same rows."""
    g = torch.Generator().manual_seed(seed)
    ins = [torch.randn((P, k), generator=g) if kind == "row" else 0.5 * torch.randn((k,), generator=g)
           for kind, k in blocks]
    return [t.to(device) for t in ins]


def _const_cols(blocks):
    cols, col = [], 0
    for kind, k in blocks:
        if kind == "c":
            cols += range(col, col + k)
        col += k
    return cols


def _grads(fn, ins, trunk, heads, gout):
    """[output, every parameter's gradient, the gradient of every per-row block] of sum(fn(...) * gout), with the
    inputs in the modules' dtype and every per-row block requiring grad."""
    dtype = trunk[0].weight.dtype
    for p in _params(trunk, heads):
        p.grad = None
    leaves = [t.detach().to(dtype).clone().requires_grad_(t.dim() == 2) for t in ins]
    out = fn(leaves, trunk, heads)
    (out * gout.to(out.dtype)).sum().backward()
    return ([out.detach()] + [p.grad.detach().clone() for p in _params(trunk, heads)]
            + [t.grad.detach().clone() for t in leaves if t.dim() == 2])


def _names(trunk, heads, ins):
    return (["out"] + [n for n, _ in trunk.named_parameters()]
            + [f"head{i}.{n}" for i, h in enumerate(heads) for n, _ in h.named_parameters()]
            + [f"dx{i}" for i, t in enumerate(ins) if t.dim() == 2])


def _axis_values(n):
    """Coordinates on an axis of n texels, on the 2^-10 grid, by kind: texel centres, inner texel edges (the border
    for n = 1), the +-1 border, and points beyond it (every corner outside, except on the near side of a one-texel
    axis, where the inner corner keeps weight 0)."""
    snap = lambda v: round(v * 1024) / 1024  # noqa: E731
    centres = [snap((2 * i + 1) / n - 1) for i in range(n)]
    edges = [snap(2 * i / n - 1) for i in range(1, n)] or [-1.0, 1.0]
    beyond = min(2.0, snap(1 + 2.5 / n))
    return [torch.tensor(v, dtype=torch.float64) for v in (centres, edges, [-1.0, 1.0], [beyond, 2.0, -beyond, -2.0])]


def _placed_rows(P, plane, face, placement, seed):
    """(pos_enc_mesh (P,3) float32, is_face (P,) bool) on the CPU.  The rows come in +- pairs, the face rows among
    themselves, and for odd P one row sits at the origin (a face row only when every row is), so both means of
    triplane_grid are exactly 0 and with extents 2 the grid is the positions themselves.  Every coordinate is a
    multiple of 2^-10 in [-2, 2].
      "spread": each coordinate on a texel centre, an inner texel edge, the border or beyond it -- x on the W axis,
                z on the H axis, y on either (it is v on the xy plane and u on the yz plane);
      "point":  every row at the origin (the texels there hold every row)."""
    H, W = plane
    n = P // 2
    g = torch.Generator().manual_seed(seed)
    if placement == "point":
        half = torch.zeros((n, 3), dtype=torch.float64)
    else:
        def coord(cands):
            kind = torch.randint(0, len(cands), (n,), generator=g)
            v = torch.empty(n, dtype=torch.float64)
            for k, c in enumerate(cands):
                sel = kind == k
                v[sel] = c[torch.randint(0, len(c), (int(sel.sum()),), generator=g)]
            return v
        cw, ch = _axis_values(W), _axis_values(H)
        x, z = coord(cw), coord(ch)
        y = torch.where(torch.rand(n, generator=g, dtype=torch.float64) < 0.5, coord(ch), coord(cw))
        half = torch.stack((x, y, z), 1)
    if face == "mix":
        fh = torch.rand(n, generator=g) < 0.5
        fh[:2] = torch.tensor([True, False])[:n]
    else:
        fh = torch.full((n,), face == "all")
    pos = torch.cat((half, -half, torch.zeros((P % 2, 3), dtype=torch.float64))).float()
    is_face = torch.cat((fh, fh, torch.full((P % 2,), face == "all")))
    return pos, is_face


def _grid_of(pos):
    x, y, z = pos.unbind(1)
    return torch.stack((torch.stack((x, y), 1), torch.stack((x, z), 1), torch.stack((y, z), 1)), 1)


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(LAYOUTS))
def test_reference_is_the_float64_modules(name):
    """gn_mlp_reference, which the GPU tests compare against, is the modules run in float64 on the concatenated input
    (constant blocks repeated): the output, every parameter gradient and every per-row block's gradient."""
    blocks, hw, final = LAYOUTS[name]
    trunk, heads = _stack(blocks, hw, final, seed=1)
    trunk, heads = trunk.double(), [h.double() for h in heads]
    P = 37
    ins = _inputs(blocks, P, seed=2)
    gout = torch.randn((P, _out_width(hw, final)), generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    ref = _grads(lambda i, t, h: gn_mlp_reference(i, t, h), ins, trunk, heads, gout)
    mod = _grads(_torch_module_forward, ins, trunk, heads, gout)
    assert ref[0].shape == (P, _out_width(hw, final))
    for what, a, b in zip(_names(trunk, heads, ins), ref, mod):
        assert a.shape == b.shape, (name, what)
        scale = float(b.abs().max())
        assert scale > 0, (name, what)
        assert float((a - b).abs().max()) <= 1e-12 * scale, (name, what)


@pytest.mark.parametrize("P,face", [(1, "none"), (1, "all"), (2, "all"), (85, "mix"), (4099, "mix"), (4099, "none")])
def test_mirrored_dyadic_rows_give_an_exact_grid(P, face):
    """With +- paired dyadic rows and extents 2 the body and face means are exactly 0 and the divisor is 1, so the
    sample coordinates are the positions themselves: the GPU cases put their samples exactly on texel centres, edges,
    the border and beyond it."""
    for plane in PLANES:
        for placement in ("spread", "point"):
            pos, is_face = _placed_rows(P, plane, face, placement, seed=P)
            assert pos.shape == (P, 3) and is_face.shape == (P,)
            assert bool((pos.abs() <= 2).all()) and torch.equal(pos * 1024, torch.round(pos * 1024))
            assert not bool(torch.mean(pos, 0).any())
            if bool(is_face.any()):
                assert not bool(torch.mean(pos[is_face], 0).any())
            assert bool(is_face.all()) if face == "all" else (face == "mix") == bool(is_face.any())
            grid = triplane_grid(pos, is_face, 2.0, 2.0)
            assert grid.dtype == torch.float32 and torch.equal(grid, _grid_of(pos)), (plane, placement)
            if plane == (128, 128) and placement == "spread" and P == 4099:
                idx, w = bilinear_corners(grid, *plane)
                assert bool((w == 1).any())                 # on a texel centre in both axes
                assert bool((w == 0.5).any())               # on a texel edge in one axis
                assert bool((w == 0.25).any())              # on a texel corner
                assert bool((idx < 0).all(-1).any())        # every corner outside the plane


# ---------------------------------------------------------------------------------------------------------------------
# GPU: gn_mlp
# ---------------------------------------------------------------------------------------------------------------------

def _against_float64(blocks, hw, final, P, seed, device):
    """gn_mlp against gn_mlp_reference in float64 and against the fp32 modules, the ReLU-edge rows left out of the
    gradients (test_human_nets._relu_edge_rows).  Returns [(what, err / scale, err32 / scale)], then asserts
    err <= 1e-5 scale and err <= max(2 err32, FLOOR scale) for the output, every parameter gradient and dX."""
    trunk, heads = _stack(blocks, hw, final, seed, device)
    ins = _inputs(blocks, P, seed + 1, device)
    gout = torch.randn((P, _out_width(hw, final)), generator=torch.Generator().manual_seed(seed + 2)).to(device)
    t64, h64 = copy.deepcopy(trunk).double(), [copy.deepcopy(h).double() for h in heads]
    gout[_relu_edge_rows(ins, t64)] = 0
    op = _grads(lambda i, t, h: gn_mlp(i, t, h), ins, trunk, heads, gout)
    r64 = _grads(lambda i, t, h: gn_mlp_reference(i, t, h), ins, t64, h64, gout)
    t32 = _grads(_torch_module_forward, ins, trunk, heads, gout)
    rec, bad = [], []
    for what, a, b, r in zip(_names(trunk, heads, ins), op, t32, r64):
        assert a.shape == r.shape and a.dtype == torch.float32, what
        err = float((a.double() - r).abs().max())
        err32 = float((b.double() - r).abs().max())
        scale = float(r.abs().max())
        rec.append((what, err / scale if scale else err, err32 / scale if scale else err32))
        if not (err <= 1e-5 * scale and err <= max(2 * err32, FLOOR * scale)):
            bad.append((what, err, err32, scale))
    cols = _const_cols(blocks)
    if cols:  # the folded columns of W_0: (sum over the rows of dL/dz_0) x c
        w_op, w_ref = op[1][:, cols].double(), r64[1][:, cols]
        if not float((w_op - w_ref).abs().max()) <= 1e-5 * float(w_ref.abs().max()):
            bad.append(("folded W_0 columns", float((w_op - w_ref).abs().max()), None, float(w_ref.abs().max())))
    return rec, bad


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 15, 16, 17, 127, 128, 129, 1023, 1024, 1025, 8193, 16895, 16896, 16897, 300007])
def test_gn_mlp_row_counts_against_float64(P, dev):
    """geo_net's layout (K = 96, heads [3, 1]) at one row, around the 16-row tile, one CTA, the 1024-row chunk, a
    single pairwise run, one full wave of 132 CTAs and one tile more, and runs of more than 8 chunk partials."""
    _, bad = _against_float64(*GEO_NET, P, seed=P % 1000, device=dev)
    assert not bad, (P, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [1, 2, 3, 4])
@pytest.mark.parametrize("K", [1, 3, 8, 9, 127, 128])
def test_gn_mlp_widths_against_float64(K, H, dev):
    """First-layer widths from 1 to the supported 128 (tails of the forward's KT, the dX kernel's NT and the weight
    gradient's KB) with 1 to 4 head outputs, through heads or a final Linear."""
    _, bad = _against_float64((("row", K),), *HEADS[H], 1025, seed=10 * K + H, device=dev)
    assert not bad, (K, H, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["const_first", "const_between"])
def test_gn_mlp_folded_blocks_against_float64(name, dev):
    """A constant block first, and one between two per-row blocks that both require grad: dX split into two blocks
    and the folded columns' weight gradient."""
    _, bad = _against_float64(*LAYOUTS[name], 1025, seed=20, device=dev)
    assert not bad, (name, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("K,H", [(96, 4), (9, 1)])
def test_gn_mlp_rows_do_not_depend_on_their_place(K, H, dev):
    """Each row goes through the same mma, quad-shuffle and head arithmetic wherever it sits, so its output is the
    same bits for any P and any place in its tile; a no-grad call keeps no pre-GroupNorm activations and gives the
    same bits as a call that keeps them."""
    blocks = (("row", K),)
    trunk, heads = _stack(blocks, *HEADS[H], seed=30, device=dev)
    P = 1025
    x = _inputs(blocks, P, 31, dev)[0]
    x0 = _inputs(blocks, 15, 32, dev)[0]
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    with torch.no_grad():
        full = gn_mlp([x], trunk, heads)
    assert torch.cuda.max_memory_allocated(dev) - base < 3 * P * 128 * 4  # nothing kept for a backward
    assert full.shape == (P, H) and bool(torch.isfinite(full).all())
    with torch.no_grad():
        for n in (1, 15, 16, 17, 129, 1024):
            assert torch.equal(gn_mlp([x[:n]], trunk, heads), full[:n]), n
        for shift in (1, 8, 15):
            assert torch.equal(gn_mlp([torch.cat((x0[:shift], x))], trunk, heads)[shift:], full), shift
    xg = x.clone().requires_grad_()
    out = gn_mlp([xg], trunk, heads)
    assert out.grad_fn is not None and torch.equal(out.detach(), full)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["k128", "const_between"])
def test_gn_mlp_backward_without_dx(name, dev):
    """With no per-row block requiring grad the backward skips dX; the parameter gradients are the same bits as with
    it."""
    blocks, hw, final = LAYOUTS[name]
    trunk, heads = _stack(blocks, hw, final, seed=40, device=dev)
    P = 1025
    ins = _inputs(blocks, P, 41, dev)
    gout = torch.randn((P, _out_width(hw, final)), generator=torch.Generator().manual_seed(42)).to(dev)
    params = _params(trunk, heads)

    def run(row_grad):
        for p in params:
            p.grad = None
        leaves = [t.clone().requires_grad_(row_grad and t.dim() == 2) for t in ins]
        (gn_mlp(leaves, trunk, heads) * gout).sum().backward()
        return [p.grad.clone() for p in params], [t.grad for t in leaves if t.dim() == 2]
    g_dx, dx = run(True)
    g_no, no_dx = run(False)
    assert all(d is not None for d in dx) and all(d is None for d in no_dx)
    assert all(torch.equal(a, b) for a, b in zip(g_dx, g_no))


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1024, 16896])
def test_gn_mlp_bias_gradients_of_mirrored_rows(P, dev):
    """The rows twice, the copy with dL/dout negated and aligned to the 16-row tiles: every per-row contribution to
    db and dbh cancels.  Those two are summed from fp64 partials, so they stay within 1e-6 of the sum of the absolute
    contributions of the float64 result."""
    blocks = GEO_NET[0]
    trunk, heads = _stack(*GEO_NET, seed=50, device=dev)
    x = _inputs(blocks, P, 51, dev)[0]
    g = torch.randn((P, 4), generator=torch.Generator().manual_seed(52)).to(dev)
    x2, g2 = torch.cat((x, x)), torch.cat((g, -g))
    for p in _params(trunk, heads):
        p.grad = None
    (gn_mlp([x2], trunk, heads) * g2).sum().backward()
    got = [trunk[3 * l].bias.grad for l in range(3)] + [torch.cat([h[0].bias.grad for h in heads])]
    t64, h64 = copy.deepcopy(trunk).double(), [copy.deepcopy(h).double() for h in heads]
    for p in _params(t64, h64):
        p.grad = None
    zs = []

    def keep(module, inp, out):
        out.retain_grad()
        zs.append(out)
    hooks = [t64[3 * l].register_forward_hook(keep) for l in range(3)]
    try:
        (_torch_module_forward([x2.double()], t64, h64) * g2.double()).sum().backward()
    finally:
        for h in hooks:
            h.remove()
    ref = [t64[3 * l].bias.grad for l in range(3)] + [torch.cat([h[0].bias.grad for h in h64])]
    terms = [z.grad.abs().sum(0) for z in zs] + [g2.double().abs().sum(0)]
    for what, a, r, s in zip(("db0", "db1", "db2", "dbh"), got, ref, terms):
        assert bool((s > 0).all()), what
        err = (a.double() - r).abs()
        assert bool((err <= 1e-6 * s).all()), (what, float((err / s).max()))


def _poisoned(n, device):
    """n NaNs followed by PAD sentinels."""
    buf = torch.full((n + PAD,), float("nan"), dtype=torch.float32, device=device)
    buf[n:] = SENTINEL
    return buf


def _assert_written(what, buf, n, expect=None):
    """The first n values finite (and equal to `expect` bit for bit), the sentinels past them untouched."""
    got = buf[:n]
    assert bool(torch.isfinite(got).all()), (what, int((~torch.isfinite(got)).sum()), n)
    if expect is not None:
        assert torch.equal(got, expect.reshape(-1)), what
    assert bool((buf[n:] == SENTINEL).all()), what


@pytest.mark.gpu
@pytest.mark.parametrize("P", [17, 1025, 16897])
def test_gn_mlp_abi_writes_every_value_and_nothing_past_the_end(P, dev):
    """b2r_gn_mlp_forward / _backward with the scratch all NaN and out, saved, dX and the gradients NaN up to their
    ends and a sentinel after: everything written is finite and the Python route's bits, and nothing is written past
    an end.  At P = 17 one of the chain kernel's 132 CTAs has a tile; the other 131 must write zero partials."""
    K, H = 99, 4
    blocks = (("row", K),)
    trunk, heads = _stack(blocks, *HEADS[H], seed=60, device=dev)
    x = _inputs(blocks, P, 61, dev)[0]
    gout = torch.randn((P, H), generator=torch.Generator().manual_seed(62)).to(dev)
    lib = L.load()
    wh = torch.cat([h[0].weight.detach() for h in heads]).contiguous()
    bh = torch.cat([h[0].bias.detach() for h in heads]).contiguous()
    m = L.B2RGnMlp(P=P, K=K, H=H, x=x.data_ptr(), w_head=wh.data_ptr(), b_head=bh.data_ptr())
    for l in range(3):
        m.w[l], m.b[l] = trunk[3 * l].weight.data_ptr(), trunk[3 * l].bias.data_ptr()
        m.gamma[l], m.beta[l] = trunk[3 * l + 1].weight.data_ptr(), trunk[3 * l + 1].bias.data_ptr()
    n_grads = int(lib.b2r_gn_mlp_grads_count(K, H))
    out, saved, dx, grads = (_poisoned(n, dev) for n in (P * H, 3 * P * 128, P * K, n_grads))
    nbytes = int(lib.b2r_gn_mlp_scratch_bytes(P))
    scratch = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=dev)  # all-ones bytes: NaN as float and double
    st = torch.cuda.current_stream(dev).cuda_stream
    L.check(lib.b2r_gn_mlp_forward(C.byref(m), out.data_ptr(), saved.data_ptr(), st), "b2r_gn_mlp_forward")
    L.check(lib.b2r_gn_mlp_backward(C.byref(m), saved.data_ptr(), gout.data_ptr(), dx.data_ptr(), grads.data_ptr(),
                                    scratch.data_ptr(), nbytes, st), "b2r_gn_mlp_backward")
    torch.cuda.synchronize()
    py = _grads(lambda i, t, h: gn_mlp(i, t, h), [x], trunk, heads, gout)
    lin = [trunk[3 * l] for l in range(3)]
    gn = [trunk[3 * l + 1] for l in range(3)]
    hl = [h[0] for h in heads]
    flat = torch.cat([t.grad.reshape(-1) for t in (
        [m_.weight for m_ in lin] + [m_.weight for m_ in gn] + [m_.bias for m_ in gn] + [m_.bias for m_ in lin]
        + [m_.weight for m_ in hl] + [m_.bias for m_ in hl])])
    assert flat.numel() == n_grads
    _assert_written("out", out, P * H, py[0])
    _assert_written("saved", saved, 3 * P * 128)
    _assert_written("dx", dx, P * K, py[-1])
    _assert_written("grads", grads, n_grads, flat)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: TriplaneFeatures
# ---------------------------------------------------------------------------------------------------------------------

def _tri_case(case, device):
    Cc, plane, P, face, placement = case
    pos, is_face = _placed_rows(P, plane, face, placement, seed=P + Cc)
    tri = TriplaneFeatures(pos.to(device), is_face.to(device), 2.0, 2.0, plane)
    g = torch.Generator().manual_seed(Cc)
    tp = torch.randn((3, Cc) + plane, generator=g).to(device)
    tpf = torch.randn((3, Cc) + plane, generator=g).to(device)
    gout = torch.randn((P, 3 * Cc), generator=g).to(device)
    return tri, pos, tp, tpf, gout


def _empty_texels(tri, Cc):
    """(2, 3, C, H, W) bool: the texels of the body (0) and face (1) planes no row samples."""
    H, W = tri.plane_size
    n = (tri.offsets[1:] - tri.offsets[:-1]).reshape(2, 3, 1, H, W)
    return (n == 0).expand(2, 3, Cc, H, W)


@pytest.mark.gpu
@pytest.mark.parametrize("case", TRI_CASES, ids=_tri_id)
def test_triplane_shapes_against_float64(case, dev):
    """Features against the op's bilinear blend in float64 and against F.grid_sample in float64; both plane
    gradients against float64 autograd; texels no row samples exactly 0; no body gradient from face rows; and two
    backward runs bit-identical."""
    Cc = case[0]
    tri, pos, tp, tpf, gout = _tri_case(case, dev)
    assert torch.equal(tri.grid.cpu(), _grid_of(pos))  # the samples sit exactly where they were placed
    tp.requires_grad_()
    tpf.requires_grad_()
    feat = tri(tp, tpf)
    (feat * gout).sum().backward()
    d1, df1 = tp.grad.clone(), tpf.grad.clone()
    tp64 = tp.detach().double().requires_grad_()
    tpf64 = tpf.detach().double().requires_grad_()
    ref = _blend64(tri, tp64, tpf64)
    (ref * gout.double()).sum().backward()
    ref = ref.detach()
    assert feat.shape == ref.shape == (case[2], 3 * Cc)
    assert float((feat.double() - ref).abs().max()) <= 1e-6 * float(ref.abs().max())
    ref_gs = tri_feature_reference(tri.grid, tri.is_face, tp.detach().double(), tpf.detach().double())
    assert float((feat.double() - ref_gs).abs().max()) <= 1e-5 * float(ref_gs.abs().max())
    empty = _empty_texels(tri, Cc)
    for what, got, r, e in (("body", d1, tp64.grad, empty[0]), ("face", df1, tpf64.grad, empty[1])):
        assert float((got.double() - r).abs().max()) <= 1e-5 * float(r.abs().max()), what
        assert not bool(got[e].any()), what
    # face rows leave the body triplane's gradient untouched
    tp.grad = None
    tpf.grad = None
    (tri(tp, tpf) * gout * tri.is_face[:, None]).sum().backward()
    assert not bool(tp.grad.any())
    # bit-identical backward
    tp.grad = None
    tpf.grad = None
    (tri(tp, tpf) * gout).sum().backward()
    assert torch.equal(tp.grad, d1) and torch.equal(tpf.grad, df1)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [TRI_CASES[2], TRI_CASES[4], TRI_CASES[6]], ids=_tri_id)
def test_triplane_abi_writes_every_value_and_nothing_past_the_end(case, dev):
    """b2r_triplane_forward / _backward into buffers of NaN with a sentinel past their ends: every feature and every
    texel of both planes is written, finite and the Python route's bits, texels no row samples are exactly 0, and
    nothing is written past an end."""
    Cc, (H, W), P = case[:3]
    tri, _, tp, tpf, gout = _tri_case(case, dev)
    lib = L.load()
    st = torch.cuda.current_stream(dev).cuda_stream
    n_feat, n_tex = P * 3 * Cc, 3 * Cc * H * W
    feat = _poisoned(n_feat, dev)
    L.check(lib.b2r_triplane_forward(P, Cc, H, W, tp.data_ptr(), tpf.data_ptr(), tri.is_face.data_ptr(),
                                     tri.corners.data_ptr(), tri.weights.data_ptr(), feat.data_ptr(), st),
            "b2r_triplane_forward")
    d, df = _poisoned(n_tex, dev), _poisoned(n_tex, dev)
    L.check(lib.b2r_triplane_backward(P, Cc, H, W, gout.data_ptr(), tri.offsets.data_ptr(), tri.rows.data_ptr(),
                                      tri.entry_w.data_ptr(), d.data_ptr(), df.data_ptr(), st), "b2r_triplane_backward")
    torch.cuda.synchronize()
    tp_, tpf_ = tp.clone().requires_grad_(), tpf.clone().requires_grad_()
    f_py = tri(tp_, tpf_)
    (f_py * gout).sum().backward()
    _assert_written("feat", feat, n_feat, f_py.detach())
    empty = _empty_texels(tri, Cc)
    for what, buf, py, e in (("body", d, tp_.grad, empty[0]), ("face", df, tpf_.grad, empty[1])):
        _assert_written(what, buf, n_tex, py)
        assert not bool(buf[:n_tex].view(py.shape)[e].any()), what
