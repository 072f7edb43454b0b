"""The per-frame ops and the frame plans against poisoned, guarded and stale memory.

Every wrapper allocates its outputs and scratch with `torch.empty`.  In a test process that memory is usually fresh
(zeros) or the block the previous identical call just freed, so a kernel that skips a write, reads scratch before
writing it, or writes past an end can pass a comparison with a reference.  This file runs each op on the same inputs
  * plainly;
  * under `poisoned()`: torch's deterministic mode with `fill_uninitialized_memory`, so every `torch.empty` comes back
    NaN (floats), INT_MAX (integers) or 0xFF (bytes);
  * under `GuardedAllocations`: every buffer the package's Python code allocates -- each output and scratch array the
    wrapper hands the op's C ABI, in the struct its own helpers build -- sits between guard bands of a byte pattern,
    its body filled with NaN words, then again with zeros;
and requires every output and gradient to be the plain run's bits and every guard byte to be unchanged.  None of these
ops adds with float atomics, so any difference is an unwritten value, a read of unwritten scratch or a stray write.  At
the new shapes, ops with a float64 restatement are also held to it with the tolerance of their own test file.

State that lives on between calls by design is checked directly: the rasterizer's backward scratch must be all zero
after every backward (B2R_BWD_SCRATCH_ZEROED), across frames whose visible sets differ; the mesh renderers' per-pixel
key buffer must be all -1 after every call, at any sequence of output sizes; and reused op objects must give a fresh
object's bits.
"""
import contextlib
import sys

import numpy as np
import pytest
import torch

from util import workload_settings  # noqa: F401  (path setup)
from exavatar_release_b200.synthetic import make_human_mesh

PKG = "exavatar_release_b200"
NAN_WORD = 0x7FC00000  # the float32 quiet NaN, as one int32 word
GUARD = 512            # guard bytes before and after every guarded buffer (a multiple of 256 keeps the alignment)


# ---------------------------------------------------------------------------------------------------------------------
# Machinery
# ---------------------------------------------------------------------------------------------------------------------

@contextlib.contextmanager
def poisoned():
    """torch.empty / empty_like return NaN floats, INT_MAX integers and 0xFF bytes inside the block.  Deterministic
    mode swaps some torch ops (index_add_, scatter_add_, cumsum) for other kernels: build inputs and references
    outside, and call only the op inside."""
    det = torch.are_deterministic_algorithms_enabled()
    warn = torch.is_deterministic_algorithms_warn_only_enabled()
    fill = torch.utils.deterministic.fill_uninitialized_memory
    torch.use_deterministic_algorithms(True, warn_only=True)
    torch.utils.deterministic.fill_uninitialized_memory = True
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(det, warn_only=warn)
        torch.utils.deterministic.fill_uninitialized_memory = fill


def _pattern(n, device):
    return ((torch.arange(n) * 151 + 89) % 256).to(torch.uint8).to(device)


class GuardedAllocations:
    """While active, `torch.empty` and `torch.empty_like` called from the package's modules for a CUDA tensor return
    a view into a larger block: GUARD pattern bytes, the body (filled with the int32 word `fill`), then pattern bytes
    up to the next 256-byte boundary and GUARD more.  Other callers get torch's own functions.  `damaged()` lists the
    allocations whose guard bytes changed; the blocks stay alive with this object."""

    def __init__(self, fill):
        self.fill = fill
        self.blocks = []  # (raw block, body bytes, allocation site)
        self._saved = None

    def _guarded(self, shape, dtype, device, site):
        meta = self._saved[0](shape, dtype=dtype, device="meta")
        n = meta.numel() * meta.element_size()
        span = GUARD + (n + 255) // 256 * 256 + GUARD
        raw = self._saved[0](span, dtype=torch.uint8, device=device)
        raw.copy_(_pattern(span, device))
        raw[GUARD:GUARD + (n + 3) // 4 * 4].view(torch.int32).fill_(self.fill)
        raw[GUARD + n:GUARD + (n + 3) // 4 * 4].copy_(_pattern(span, device)[GUARD + n:GUARD + (n + 3) // 4 * 4])
        self.blocks.append((raw, n, site))
        return raw[GUARD:GUARD + n].view(meta.dtype).view(meta.shape)

    @staticmethod
    def _site():
        f = sys._getframe(2)
        return f.f_globals.get("__name__", ""), f.f_code.co_name, f.f_lineno

    def __enter__(self):
        empty, empty_like = torch.empty, torch.empty_like

        def g_empty(*size, dtype=None, device=None, **kw):
            site = self._site()
            shape = size[0] if len(size) == 1 and isinstance(size[0], (tuple, list)) else size
            dev = torch.device(device) if device is not None else None
            if not site[0].startswith(PKG) or kw or dev is None or dev.type != "cuda":
                return empty(*size, dtype=dtype, device=device, **kw)
            return self._guarded(tuple(shape), dtype or torch.get_default_dtype(), dev, site)

        def g_empty_like(t, dtype=None, device=None, **kw):
            site = self._site()
            dev = torch.device(device) if device is not None else t.device
            if not site[0].startswith(PKG) or kw or dev.type != "cuda":
                return empty_like(t, dtype=dtype, device=device, **kw)
            return self._guarded(tuple(t.shape), dtype or t.dtype, dev, site)

        self._saved = (empty, empty_like)
        torch.empty, torch.empty_like = g_empty, g_empty_like
        return self

    def __exit__(self, *exc):
        torch.empty, torch.empty_like = self._saved

    def damaged(self):
        bad = []
        for raw, n, site in self.blocks:
            want = _pattern(raw.numel(), raw.device)
            if not (torch.equal(raw[:GUARD], want[:GUARD]) and torch.equal(raw[GUARD + n:], want[GUARD + n:])):
                bad.append(site)
        return bad


def _flatten(x, name="out"):
    """[(name, clone)] of every tensor in nested tuples / lists / dicts."""
    if x is None:
        return []
    if isinstance(x, torch.Tensor):
        return [(name, x.detach().clone())]
    if isinstance(x, dict):
        return [p for k in sorted(x) for p in _flatten(x[k], f"{name}.{k}")]
    if isinstance(x, (tuple, list)):
        return [p for i, v in enumerate(x) for p in _flatten(v, f"{name}[{i}]")]
    return []


def _bits(t):
    if t.dtype.is_floating_point:
        return t.contiguous().view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])
    return t


def _same_bits(a, b, what):
    assert [n for n, _ in a] == [n for n, _ in b], what
    diff = [n for (n, x), (_, y) in zip(a, b) if x.shape != y.shape or x.dtype != y.dtype
            or not torch.equal(_bits(x), _bits(y))]
    assert not diff, (what, diff)


def check_memory(run, guard=True):
    """run() -> tensors (forward outputs and gradients).  The poisoned run, and with `guard` the guarded runs with NaN
    and zero bodies, must give the plain run's bits, and no guard byte may change.  Returns the plain results."""
    plain = _flatten(run())
    with poisoned():
        got = _flatten(run())
    _same_bits(plain, got, "poisoned")
    if guard:
        for fill in (NAN_WORD, 0):
            with GuardedAllocations(fill) as g:
                got = _flatten(run())
            torch.cuda.synchronize()
            assert g.blocks, "no allocation of the package was guarded"
            assert not g.damaged(), (hex(fill), g.damaged())
            _same_bits(plain, got, f"guarded, bodies {fill:#x}")
    return dict(plain)


def _err(a, b):
    return float((a.double() - b.double()).abs().max()) if a.numel() else 0.0


def _close(a, b, rel, what):
    scale = float(b.detach().double().abs().max()) if b.numel() else 0.0
    err = _err(a.detach(), b.detach())
    assert err <= rel * max(scale, 1e-30), f"{what}: max error {err:.3e} vs {rel:.0e} x max {scale:.3e}"


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the machinery itself
# ---------------------------------------------------------------------------------------------------------------------

def test_poisoned_fills_and_restores_even_on_failure():
    before = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
              torch.utils.deterministic.fill_uninitialized_memory)
    with poisoned():
        assert torch.are_deterministic_algorithms_enabled()
        assert torch.utils.deterministic.fill_uninitialized_memory
        assert bool(torch.isnan(torch.empty(37)).all())
        assert bool((torch.empty(5, dtype=torch.int32) == 2 ** 31 - 1).all())
        assert bool((torch.empty(5, dtype=torch.int64) == 2 ** 63 - 1).all())
        assert bool((torch.empty(9, dtype=torch.uint8) == 255).all())
        assert bool(torch.isnan(torch.empty(8, dtype=torch.uint8).view(torch.float32)).all())
    assert (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
            torch.utils.deterministic.fill_uninitialized_memory) == before
    with pytest.raises(RuntimeError, match="inside"):
        with poisoned():
            raise RuntimeError("a failure inside")
    assert (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
            torch.utils.deterministic.fill_uninitialized_memory) == before


class _CpuGuarded(GuardedAllocations):
    """The same blocks on the CPU, for the self-test (the product allocates on CUDA only)."""

    def __enter__(self):
        super().__enter__()
        g_empty = torch.empty
        torch.empty = lambda *s, dtype=None, device=None, **kw: (  # noqa: E731
            self._guarded(tuple(s[0] if len(s) == 1 and isinstance(s[0], (tuple, list)) else s),
                          dtype or torch.get_default_dtype(), torch.device("cpu"), ("test",) * 3)
            if device == "guarded" else g_empty(*s, dtype=dtype, device=device, **kw))
        return self


def test_guard_helper_sees_every_stray_byte():
    for shape, dtype in (((3, 5), torch.float32), ((7,), torch.int32), ((13,), torch.uint8), ((2, 3), torch.int64),
                         ((0, 3), torch.float32)):
        with _CpuGuarded(NAN_WORD) as g:
            t = torch.empty(shape, dtype=dtype, device="guarded")
        assert t.shape == shape and t.dtype == dtype and t.is_contiguous()
        raw, n, _ = g.blocks[0]
        assert t.numel() == 0 or t.data_ptr() - raw.data_ptr() == GUARD
        assert n == t.numel() * t.element_size()
        if dtype == torch.float32 and t.numel():
            assert bool(torch.isnan(t).all())
        assert g.damaged() == []
        t.fill_(0)  # every body byte written: no guard byte moves
        assert g.damaged() == []
        for where in (GUARD - 1, GUARD + n, raw.numel() - 1, GUARD + (n + 255) // 256 * 256):
            if where >= raw.numel():
                continue
            keep = raw[where].clone()
            raw[where] ^= 1
            assert len(g.damaged()) == 1, (shape, where)
            raw[where] = keep
        assert g.damaged() == []
    with _CpuGuarded(0) as g:
        t = torch.empty(10, dtype=torch.uint8, device="guarded")
    assert bool((t == 0).all())


def test_guarded_allocations_leave_other_callers_alone():
    with GuardedAllocations(NAN_WORD) as g:
        a = torch.empty(4)
        b = torch.empty_like(a)
    assert g.blocks == [] and a.shape == b.shape == (4,)
    assert torch.empty is not None and torch.empty(2).shape == (2,)


def test_bits_compare_nan_payloads_and_signed_zeros():
    a = torch.tensor([0.0, float("nan"), 1.0])
    _same_bits([("x", a)], [("x", a.clone())], "same")
    with pytest.raises(AssertionError):
        _same_bits([("x", a)], [("x", torch.tensor([-0.0, float("nan"), 1.0]))], "signed zero")


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


@pytest.mark.gpu
def test_poison_reaches_cuda_allocations(dev):
    """The file's premise: under poisoned(), a CUDA torch.empty is NaN / INT_MAX / 0xFF, for fresh and reused blocks."""
    for n in (1, 1000, 1 << 20):
        keep = torch.zeros(n, device=dev)
        del keep  # the next allocation of this size reuses the freed block of zeros
        with poisoned():
            f = torch.empty(n, device=dev)
            i = torch.empty(n, dtype=torch.int32, device=dev)
            q = torch.empty(n, dtype=torch.int64, device=dev)
            b = torch.empty(4 * n, dtype=torch.uint8, device=dev)
            fl = torch.empty_like(f)
        torch.cuda.synchronize()
        assert bool(torch.isnan(f).all()) and bool(torch.isnan(fl).all())
        assert bool((i == 2 ** 31 - 1).all()) and bool((q == 2 ** 63 - 1).all()) and bool((b == 255).all())
        assert bool(torch.isnan(b.view(torch.float32)).all())


# ---------------------------------------------------------------------------------------------------------------- skin

SKIN_P = [1, 31, 33, 255, 257, 4097]
SKIN_J = [1, 55, 64]
# (two sets, camera, rows given, dense weight rows): every value of each switch at every (P, J)
SKIN_VARIANTS = [(True, True, True, True), (False, False, False, True), (True, False, False, False),
                 (False, True, True, False)]


def _skin_case(P, J, two, cam, rows, dense, dev):
    from exavatar_release_b200.camera import look_at_cam_param
    g = torch.Generator().manual_seed(P * 100 + J)
    V = P + 5
    table = torch.rand(V, J, generator=g, dtype=torch.float64) + 0.05 if dense else torch.zeros(V, J, dtype=torch.float64)
    if dense:
        table /= table.sum(1, keepdim=True)
    A = torch.eye(4, dtype=torch.float64).repeat(J, 1, 1)
    A[:, :3, :] += 0.2 * torch.randn(J, 3, 4, generator=g, dtype=torch.float64)
    c = dict(xyz=torch.randn(P, 3, generator=g), xyz_r=torch.randn(P, 3, generator=g) if two else None,
             table=table.float(), A=A.float(), trans=0.1 * torch.randn(3, generator=g),
             rows=torch.randint(0, V, (P,), generator=g) if rows else None,
             gp=torch.randn(P, 3, generator=g), gq=torch.randn(P, 3, generator=g))
    c = {k: None if v is None else v.to(dev) for k, v in c.items()}
    c["R"] = c["t"] = None
    if cam:
        cp = look_at_cam_param(17.0, (64, 64), device=dev)
        c["R"], c["t"] = cp["R"], cp["t"]
    return c


def _skin_run(c):
    from exavatar_release_b200.skinning import skin_gaussians

    def run():
        x = c["xyz"].clone().requires_grad_()
        xr = None if c["xyz_r"] is None else c["xyz_r"].clone().requires_grad_()
        A, tr = c["A"].clone().requires_grad_(), c["trans"].clone().requires_grad_()
        posed, posed_r = skin_gaussians(x, xr, c["table"], c["rows"], A, tr, c["R"], c["t"])
        loss = (posed * c["gp"]).sum() + (0 if posed_r is None else (posed_r * c["gq"]).sum())
        loss.backward()
        return dict(posed=posed, posed_r=posed_r, dxyz=x.grad, dxyz_r=None if xr is None else xr.grad, dA=A.grad,
                    dtrans=tr.grad)
    return run


@pytest.mark.gpu
@pytest.mark.parametrize("J", SKIN_J)
@pytest.mark.parametrize("P", SKIN_P)
def test_skin_gaussians(P, J, dev):
    from exavatar_release_b200.renderer import lbs_reference
    from test_skin_pair import _skin_backward_f64
    for two, cam, rows, dense in SKIN_VARIANTS:
        c = _skin_case(P, J, two, cam, rows, dense, dev)
        got = check_memory(_skin_run(c))
        # float64, with test_skin_pair's bounds
        idx = c["rows"] if c["rows"] is not None else torch.arange(P, device=dev)
        w = c["table"].double()[idx].cpu()
        R = None if c["R"] is None else c["R"].double().cpu()
        t = None if c["t"] is None else c["t"].double().cpu()
        xs = [c["xyz"]] + ([c["xyz_r"]] if two else [])
        names = ["out.posed"] + (["out.posed_r"] if two else [])
        for x, n in zip(xs, names):
            ref = lbs_reference(x.double().cpu(), w, c["A"].double().cpu(), c["trans"].double().cpu(), R, t)
            _close(got[n].cpu(), ref, 1e-6, (P, J, two, cam, rows, dense, n))
        gs = [c["gp"].double().cpu()] + ([c["gq"].double().cpu()] if two else [])
        dxs, dA, dtrans = _skin_backward_f64([x.double().cpu() for x in xs], w, c["A"].double().cpu(),
                                             c["trans"].double().cpu(), None if R is None else torch.inverse(R), gs)
        for n, ref in zip(("out.dxyz", "out.dxyz_r"), dxs):
            _close(got[n].cpu(), ref, 1e-5, (P, J, n))
        _close(got["out.dA"][:, :3, :].cpu(), dA, 1e-5, (P, J, "dA"))
        assert not bool(got["out.dA"][:, 3, :].any())
        _close(got["out.dtrans"].cpu(), dtrans, 1e-5, (P, J, "dtrans"))


# ------------------------------------------------------------------------------------------------------------- l1_ssim

L1_SIZES = [(17, 33), (61, 45)]  # (W, H): neither a multiple of 16
L1_BOXES = {"whole": None, "top_left": [-3.0, -2.0, 9.0, 14.0], "bottom_right": [6.0, 9.0, 200.0, 200.0],
            "left_edge_only": [0.0, 4.0, 5.5, 11.0], "right_edge_only": [9.0, 3.0, 300.0, 7.0], "one_px": [4, 5, 1, 1]}


@pytest.mark.gpu
@pytest.mark.parametrize("ssim", [True, False])
@pytest.mark.parametrize("box", list(L1_BOXES))
@pytest.mark.parametrize("W,H", L1_SIZES)
def test_l1_ssim(W, H, box, ssim, dev):
    from exavatar_release_b200.losses import l1_ssim, l1_ssim_reference
    g = torch.Generator().manual_seed(W * H)
    img, target = torch.rand(3, H, W, generator=g), torch.rand(3, H, W, generator=g)
    mask = (torch.rand(H, W, generator=g) > 0.2).float() if box in ("whole", "bottom_right") else None
    bbox = None if L1_BOXES[box] is None else torch.tensor(L1_BOXES[box], dtype=torch.float32)
    gout = torch.tensor([0.7, -1.3])
    d = [None if v is None else v.to(dev) for v in (img, target, mask, bbox, gout)]

    def run():
        x = d[0].clone().requires_grad_()
        l1, s = l1_ssim(x, d[1], d[3], d[2], ssim=ssim)
        (l1 * d[4][0] + (0 if s is None else s * d[4][1])).backward()
        return l1, s, x.grad
    got = check_memory(run)
    xr = img.double().requires_grad_()
    rl1, rs = l1_ssim_reference(xr, target, bbox, mask, ssim=ssim)
    (rl1 * 0.7 + (0 if rs is None else rs * -1.3)).backward()
    assert abs(float(got["out[0]"]) - rl1.item()) <= 1e-5
    if ssim:
        assert abs(float(got["out[1]"]) - rs.item()) <= 1e-5
    assert _err(got["out[2]"].cpu(), xr.grad) <= 1e-4 * float(xr.grad.abs().max())


# ------------------------------------------------------------------------------------------- nearest_rows, normals

@pytest.mark.gpu
@pytest.mark.parametrize("V", [1, 31, 33, 257])
@pytest.mark.parametrize("P", [1, 31, 33, 255, 257, 4097])
def test_nearest_rows(P, V, dev):
    from exavatar_release_b200.geometry import nearest_rows, nearest_rows_reference
    g = torch.Generator().manual_seed(P + 7 * V)
    q, t = torch.randn(P, 3, generator=g), torch.randn(V, 3, generator=g)
    sm = torch.rand(P, generator=g) < 0.1
    q, t, sm = q.to(dev), t.to(dev), sm.to(dev)
    for self_map in (None, sm):
        got = check_memory(lambda: nearest_rows(q, t, self_map))["out"]
        assert torch.equal(got, nearest_rows_reference(q, t, self_map))


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [1, 30, 100])
def test_vertex_normals_with_vertices_in_no_face(extra, dev):
    from exavatar_release_b200.geometry import VertexNormals, vertex_normals_reference
    m = make_human_mesh(rings=7, segments=12)
    Vm = m["verts"].shape[0]
    V = Vm + extra  # the appended vertices lie in no face: normal 0 / max(0, eps) = 0
    g = torch.Generator().manual_seed(extra)
    x = torch.cat([m["verts"], torch.randn(extra, 3, generator=g)]).to(dev)
    flip = (torch.rand(V, generator=g) < 0.3).to(dev)
    vn = VertexNormals(m["faces"], V, flip=flip, device=dev)
    got = check_memory(lambda: vn(x))["out"]
    ref = vertex_normals_reference(x, m["faces"], flip)
    assert bool((got[Vm:] == 0).all())
    _close(got, ref, 1e-5, "normals")


# -------------------------------------------------------------------------------------------------------- mesh renders

MR_SMALL = 32  # csrc/mesh_raster.cu: a face whose pixel box has at most this many pixels is walked by one thread
# Corner triangles whose kernel box is exactly (w, h): mr_axis_range pads the pixel range by one pixel on each side and
# clamps it to the image, so a triangle from 0.1 to w - 1.7 pixels off two image edges gets columns / rows [0, w - 1]
# and covers pixel centres.  (corner, w, h): 4 x 8 = MR_SMALL pixels, 3 x 11 = MR_SMALL + 1.
CORNER_BOXES = [("top_left", 4, 8), ("top_right", 3, 11), ("bottom_left", 8, 4), ("bottom_right", 11, 3)]


def _corner_triangle(corner, w, h, H, W):
    pts = [(0.1, 0.1), (w - 1.7, 0.1), (0.1, h - 1.7)]
    right, bottom = corner.endswith("right"), corner.startswith("bottom")
    return [(W - u if right else u, H - v if bottom else v) for u, v in pts]


def _pix_triangles(n_corner, Fn, H, W, box_sizes, seed):
    """Fn triangles in camera coordinates: first the CORNER_BOXES triangles [n_corner[0], n_corner[1]) nearest the
    camera, then triangles whose pixel extent is about box_sizes (w, h) in turn, at distinct depths; and a camera at the
    origin looking down +z.  Returns (verts (3F,3), faces (F,3), cam)."""
    g = torch.Generator().manual_seed(seed)
    f = 300.0
    cam = {"R": torch.eye(3), "t": torch.zeros(3), "focal": torch.tensor([f, f]),
           "princpt": torch.tensor([W / 2.0, H / 2.0])}
    tris = [(1.5, _corner_triangle(*c, H, W)) for c in CORNER_BOXES[n_corner[0]:n_corner[1]]]
    for i in range(Fn - len(tris)):
        bw, bh = box_sizes[i % len(box_sizes)]
        u0 = float(torch.randint(0, max(W - bw, 1), (1,), generator=g)) + 0.25
        v0 = float(torch.randint(0, max(H - bh, 1), (1,), generator=g)) + 0.25
        corners = [(u0, v0), (u0 + bw - 0.5, v0), (u0, v0 + bh - 0.5)] if i % 2 == 0 else \
            [(u0, v0), (u0 + bw - 0.5, v0 + bh - 0.5), (u0 + bw - 0.5, v0)]
        tris.append((2.0 + 0.01 * i, corners))
    verts = [[(u - W / 2.0) * z / f, (v - H / 2.0) * z / f, z] for z, corners in tris for u, v in corners]
    return torch.tensor(verts), torch.arange(3 * Fn).reshape(Fn, 3), cam


def _kernel_box_areas(verts, cam, H, W):
    """Pixels in each face's box as mr_face_kernel computes it (mr_axis_range, in float32 as the --fmad=false kernel
    rounds it), for a camera with R = I and t = 0 and faces (3f, 3f+1, 3f+2)."""
    f32 = np.float32
    v = verts.cpu().numpy().astype(f32)
    fx, fy = (f32(x) for x in cam["focal"].tolist())
    cx, cy = (f32(x) for x in cam["princpt"].tolist())
    s = f32(0.5) * f32(min(W, H))
    x = (f32(0.5) * f32(W) - (fx * v[:, 0] / v[:, 2] + cx)) / s
    y = (f32(0.5) * f32(H) - (fy * v[:, 1] / v[:, 2] + cy)) / s

    def axis(a, b, n):
        ulo = f32(0.5) * f32(n) - b * s - f32(0.5)
        uhi = f32(0.5) * f32(n) - a * s - f32(0.5)
        lo = int(min(max(np.floor(ulo) - 1, 0), n))
        hi = int(max(min(np.ceil(uhi) + 1, n - 1), -1))
        return max(hi - lo + 1, 0)
    x, y = x.reshape(-1, 3), y.reshape(-1, 3)
    return [axis(x[i].min(), x[i].max(), W) * axis(y[i].min(), y[i].max(), H) for i in range(x.shape[0])]


MESH_CASES = [  # (corner triangles [a, b) of CORNER_BOXES, F, H, W, pixel extents (w, h) of the other faces)
    ((0, 1), 1, 45, 61, []),
    ((1, 2), 1, 45, 61, []),
    ((0, 4), 127, 45, 61, [(4, 8), (3, 11), (5, 7), (4, 7), (2, 17), (6, 6)]),
    ((0, 4), 129, 29, 37, [(3, 11), (4, 8), (1, 1), (20, 20)]),
    ((0, 4), 129, 100, 131, [(4, 8), (3, 11), (33, 1), (1, 32), (40, 25)]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", MESH_CASES, ids=lambda c: f"F{c[1]}-{c[2]}x{c[3]}-corners{c[0][0]}{c[0][1]}")
def test_face_and_shaded_mesh_renders(case, dev):
    from exavatar_release_b200.mesh_render import (FaceMeshRenderer, ShadedMeshRenderer, face_render_reference,
                                                   shaded_mesh_reference)
    from test_face_render import _smooth_pixels
    corners, Fn, H, W, boxes = case
    verts, faces, cam = _pix_triangles(corners, Fn, H, W, boxes, seed=Fn + H)
    V = verts.shape[0]
    # the corner faces' kernel boxes are exactly MR_SMALL and MR_SMALL + 1 pixels: both sides of the thread / warp split
    n_c = corners[1] - corners[0]
    areas = _kernel_box_areas(verts, cam, H, W)
    assert areas[:n_c] == [w * h for _, w, h in CORNER_BOXES[corners[0]:corners[1]]], areas[:n_c]
    assert set(areas[:n_c]) <= {MR_SMALL, MR_SMALL + 1}
    g = torch.Generator().manual_seed(5)
    uv = torch.rand(V, 2, generator=g)
    tex = torch.rand(1, 4, 16, 16, generator=g).to(dev)
    cam = {k: v.to(dev) for k, v in cam.items()}
    mesh = verts.to(dev)
    face_r = FaceMeshRenderer(uv, faces, faces, V, device=dev)
    # the gradient is compared on pixels whose float64 texel coordinates stay off texel-cell boundaries
    tables = {"verts": verts, "faces": faces, "face_uv": faces, "vertex_uv": uv, "texture": tex[0].cpu()}
    with torch.no_grad():
        p2f0 = face_r.render(tex, mesh[None], cam, (H, W))[1]
    G = torch.randn(1, 4, H, W, generator=g).to(dev) * _smooth_pixels(tables, cam, (H, W), p2f0)

    def run_face():
        m = mesh.clone().requires_grad_()
        img, p2f = face_r.render(tex, m[None], cam, (H, W))
        (img * G).sum().backward()
        return img, p2f, m.grad
    got = check_memory(run_face)
    assert bool((face_r._keys == -1).all())
    p2f = got["out[1]"]
    ref, ref_p2f = face_render_reference(tex, mesh[None], faces, uv, faces, cam, (H, W))
    assert torch.equal(p2f.long(), ref_p2f)
    fg = p2f >= 0
    assert int(fg.sum()) > 0
    visible = set(torch.unique(p2f[fg]).tolist())
    assert set(range(n_c)) <= visible, visible  # every corner face covers pixels
    assert float((got["out[0]"][0][:, fg] - ref[0][:, fg]).abs().max()) <= 2e-6
    assert bool((got["out[0]"][0][:, ~fg] == -1).all())
    # dL/dmesh against float64 on the op's faces, with test_face_render's bound
    m64 = mesh.double().requires_grad_()
    r64, _ = face_render_reference(tex, m64[None], faces, uv, faces, cam, (H, W), pix_to_face=p2f)
    (r64 * G.double()).sum().backward()
    scale = float(m64.grad.abs().max())
    assert scale > 0 and _err(got["out[2]"], m64.grad) <= 2e-3 * scale

    shade_r = ShadedMeshRenderer(faces, V, device=dev)
    bkg = (torch.rand(H, W, 3, generator=g) * 255).to(dev)
    got = check_memory(lambda: shade_r(mesh, cam, bkg))["out"]
    assert bool((shade_r._keys == -1).all())
    assert torch.equal(_bits(got[~fg]), _bits(bkg[~fg]))
    # covered pixels against the float32 and float64 restatements, with test_mesh_shade's bounds
    ref32, ref32_p2f = shaded_mesh_reference(mesh, faces, cam, bkg)
    assert torch.equal(ref32_p2f, p2f.long())
    ref64, _ = shaded_mesh_reference(mesh.double(), faces, cam, bkg, pix_to_face=p2f)
    d64 = (got[fg].double() - ref64[fg]).abs()
    r64 = (ref32[fg].double() - ref64[fg]).abs()
    assert float((got[fg] - ref32[fg]).abs().max()) <= 1e-3
    assert int((d64 > 1e-3).sum()) <= 1e-3 * d64.numel()
    assert float(d64.max()) <= max(1e-3, 2 * float(r64.max()))


# -------------------------------------------------------------------------------------------- triplane and GN-MLP

@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 17, 129, 1025, 16897])
def test_gn_mlp(P, dev):
    from exavatar_release_b200.human_nets import gn_mlp
    from test_human_nets_shapes import GEO_NET, LAYOUTS, _inputs, _out_width, _stack
    for blocks, hw, final in (GEO_NET, LAYOUTS["const_between"]):
        trunk, heads = _stack(blocks, hw, final, seed=P % 97, device=dev)
        ins = _inputs(blocks, P, seed=P, device=dev)
        gout = torch.randn((P, _out_width(hw, final)), generator=torch.Generator().manual_seed(P)).to(dev)
        params = [p for m in [trunk] + list(heads) for p in m.parameters()]

        def run():
            for p in params:
                p.grad = None
            leaves = [t.clone().requires_grad_(t.dim() == 2) for t in ins]
            out = gn_mlp(leaves, trunk, heads)
            (out * gout).sum().backward()
            return [out] + [p.grad for p in params] + [t.grad for t in leaves if t.dim() == 2]
        check_memory(run)
        with torch.no_grad():
            check_memory(lambda: gn_mlp(ins, trunk, heads))


@pytest.mark.gpu
@pytest.mark.parametrize("ci", [0, 1, 4, 7, 8, 9])
def test_triplane(ci, dev):
    from test_human_nets_shapes import TRI_CASES, _tri_case
    tri, _, tp, tpf, gout = _tri_case(TRI_CASES[ci], dev)

    def run():
        a, b = tp.clone().requires_grad_(), tpf.clone().requires_grad_()
        feat = tri(a, b)
        (feat * gout).sum().backward()
        return feat, a.grad, b.grad
    check_memory(run)


# ------------------------------------------------------------------------------------------------------- regularisers

REG_WINDOWS = {"normal": dict(arm_ny=(0.47, 0.53), arm_half_width=0.02),
               "k0": dict(arm_ny=(0.49, 0.51), arm_half_width=0.05),
               "no_lower": dict(arm_ny=(0.6, 0.7), arm_half_width=0.05),
               "wide": dict(arm_ny=(0.3, 0.7), arm_half_width=0.08),
               "narrow": dict(arm_ny=(0.49, 0.51), arm_half_width=0.004)}


def _regs_run(regs, mesh, ins, dev):
    from test_human_regularizers import _op
    return lambda: _op(regs, mesh, ins, dev)


def _regs_float64(regs, mesh, kw, ins, got, what):
    """The terms and gradients of one call against regs.reference in float64, with test_human_regularizers' bounds
    (the zero-offset hand row of mean_offset, where the gradient passes n / eps, is left to that file)."""
    from test_human_regularizers import INPUTS, _kink_row
    from exavatar_release_b200.regularizers import KEYS
    leaves = {k: v.double().requires_grad_() for k, v in ins.items()}
    ref = regs.reference(mesh, *[leaves[k] for k in INPUTS])
    vec = got["out[0]"]
    for i, k in enumerate(KEYS):
        r = ref[k].item()
        assert abs(float(vec[i]) - r) <= 1e-6 * abs(r), (what, k, float(vec[i]), r)
    sum(ref.values()).backward()
    row = _kink_row(kw)
    for k in INPUTS:
        want = leaves[k].grad.detach().clone()
        have = got[f"out[1].{k}"].double().cpu().reshape(want.shape).clone()
        if k == "mean_offset":
            have[0, row], want[0, row] = 0.0, 0.0
        scale = float(want.abs().max())
        assert scale > 0 and float((have - want).abs().max()) <= 1e-5 * scale, (what, k)


@pytest.mark.gpu
@pytest.mark.parametrize("window", list(REG_WINDOWS))
def test_human_regularizers(window, dev):
    """Every window's bits; against float64 where k > 0 ("normal" and "wide").  Without lower rows the reference
    raises in torch.min, and with k = 0 ("k0", "narrow") arm_rgb_reg is NaN, which test_human_regularizers covers."""
    from test_human_regularizers import _c4
    m, regs, kw, ins = _c4(dev, **REG_WINDOWS[window])
    print(f"{window}: {regs.n_arm} arm rows (RG_SPLIT_THREADS = 1024)")
    got = check_memory(_regs_run(regs, m["verts"], ins, dev))
    finite = bool(torch.isfinite(got["out[0]"]).all())
    assert finite == (window in ("normal", "wide")), (window, got["out[0]"])
    if finite:
        _regs_float64(regs, m["verts"], kw, ins, got, window)


@pytest.mark.gpu
def test_regularizer_arm_counts_straddle_the_split():
    """Float64-checked windows on both sides of RG_SPLIT_THREADS."""
    from test_human_regularizers import _c4
    dev = torch.device("cuda:0")
    n = {w: _c4(dev, **kw)[1].n_arm for w, kw in REG_WINDOWS.items()}
    assert n["normal"] < 1024 < n["wide"], n


def _turned(verts, deg):
    """The mesh turned by deg about the z axis: the arm normals' y, and so the upper / lower split and k, change."""
    a = torch.tensor(deg * torch.pi / 180, dtype=torch.float64)
    c, s_ = float(torch.cos(a)), float(torch.sin(a))
    R = torch.tensor([[c, -s_, 0.0], [s_, c, 0.0], [0.0, 0.0, 1.0]])
    return (verts @ R.t()).contiguous()


@pytest.mark.gpu
def test_regularizers_reused_across_windows_equal_fresh_objects(dev):
    """One object taken through meshes that give a k = 0 window, then a normal window, then no lower row, each with
    new inputs, against a fresh object's call on the same mesh and inputs."""
    from exavatar_release_b200 import HumanRegularizers
    from exavatar_release_b200.geometry import VertexNormals
    from exavatar_release_b200.regularizers import arm_selection_reference
    from test_human_regularizers import _c4
    m, regs, kw, ins = _c4(dev, **REG_WINDOWS["no_lower"])
    vn = VertexNormals(m["faces"], m["verts"].shape[0], device=dev)
    windows = []
    for step, deg in enumerate((45.0, 20.0, 0.0)):
        mesh = _turned(m["verts"], deg)
        lower, _, k, _ = arm_selection_reference(mesh, vn(mesh.to(dev)).cpu(), kw["is_arm"])
        windows.append((lower.numel() > 0, k))
        g = torch.Generator().manual_seed(step)
        new = {n: v * (1 + 0.1 * torch.rand(v.shape, generator=g)) for n, v in ins.items()}
        got = _flatten(_regs_run(regs, mesh, new, dev)())
        fresh = HumanRegularizers(m["faces"], m["verts"].shape[0], device=dev,
                                  **{n: (v.to(dev) if isinstance(v, torch.Tensor) else v) for n, v in kw.items()})
        _same_bits(got, _flatten(_regs_run(fresh, mesh, new, dev)()), (deg, windows[-1]))
    assert windows[0] == (True, 0) and windows[1][0] and windows[1][1] > 0 and not windows[2][0], windows


# -------------------------------------------------------------------------------------------------------- SMPL-X rig

def _rig_of(which, dev):
    from exavatar_release_b200.smplx_rig import SmplxRig
    from test_smplx_rig import _small
    if which == "small":
        _, model = _small()
    else:
        from exavatar_release_b200.synthetic import make_smplx_model
        model = make_smplx_model(make_human_mesh())
    return SmplxRig(**model, device=dev)


RIG_TRANS = (0.02, -0.05, 0.1)


def _body_weights(rig):
    return torch.randn((rig.V, 3), generator=torch.Generator().manual_seed(1)).cuda()


def _rig_run(rig, ins, w, dev):
    from test_smplx_rig import _loss, _leaves
    trans = torch.tensor(RIG_TRANS, device=dev)
    wb = _body_weights(rig)

    def run():
        a = _leaves(ins)
        out = rig(*a)
        _loss(out, w).backward()
        b = _leaves(ins)
        mesh = rig.body_mesh(*b, trans)
        (mesh * wb).sum().backward()
        return dict(rig=out._asdict(), d_rig=[x.grad for x in a], body=mesh, d_body=[x.grad for x in b])
    return run


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["small", "c4"])
def test_smplx_rig_and_body_mesh(which, dev):
    """Bits, then the rig's outputs and gradients and the body mesh and its gradients against float64 autograd, with
    the bounds of test_smplx_rig and test_smplx_body."""
    from exavatar_release_b200.smplx_rig import smplx_body_reference
    from test_smplx_rig import _inputs, _leaves, _loss, _loss_weights
    rig = _rig_of(which, dev)
    ins = _inputs(rig.J, rig.NB, rig.NE, seed=7, device="cuda")
    w = _loss_weights(rig)
    got = check_memory(_rig_run(rig, ins, w, dev))
    names = ("shape_param", "joint_offset", "full_pose", "expr")
    b = _leaves(ins, torch.float64)
    ref = rig.reference(*b, dtype=torch.float64, device="cuda", cache={})
    for name in ("mesh_neutral_pose", "mesh_neutral_pose_wo_upsample", "joint_mats"):
        _close(got[f"out.rig.{name}"], getattr(ref, name), 1e-6, (which, name))
    for name in ("pose_offset", "expr_offset"):
        _close(got[f"out.rig.{name}"], getattr(ref, name), 1e-5, (which, name))
    _loss(ref, [x.double() for x in w]).backward()
    for i, name in enumerate(names):
        _close(got[f"out.d_rig[{i}]"], b[i].grad, 1e-5, (which, "d" + name))
    c = _leaves(ins, torch.float64)
    trans = torch.tensor(RIG_TRANS, dtype=torch.float64, device="cuda")
    body = smplx_body_reference(rig.model, *c, trans)
    _close(got["out.body"], body, 1e-6, (which, "body_mesh"))
    (body * _body_weights(rig).double()).sum().backward()
    for i, name in enumerate(names):
        _close(got[f"out.d_body[{i}]"], c[i].grad, 2e-6, (which, "body d" + name))


@pytest.mark.gpu
def test_smplx_rig_reused_with_new_inputs_equals_a_fresh_rig(dev):
    from test_smplx_rig import _inputs, _loss_weights
    rig = _rig_of("small", dev)
    w = _loss_weights(rig)
    first = _inputs(rig.J, rig.NB, rig.NE, seed=1, device="cuda")
    second = _inputs(rig.J, rig.NB, rig.NE, seed=2, device="cuda")
    _rig_run(rig, first, w, dev)()
    got = _flatten(_rig_run(rig, second, w, dev)())
    _same_bits(got, _flatten(_rig_run(_rig_of("small", dev), second, w, dev)()), "reused rig")


@pytest.mark.gpu
def test_triplane_reused_with_new_planes_equals_a_fresh_object(dev):
    from exavatar_release_b200.human_nets import TriplaneFeatures
    from test_human_nets_shapes import TRI_CASES, _tri_case
    tri, pos, tp, tpf, gout = _tri_case(TRI_CASES[2], dev)
    fresh = TriplaneFeatures(pos.to(dev), tri.is_face, 2.0, 2.0, TRI_CASES[2][1])

    def run(op, a, b):
        a, b = a.clone().requires_grad_(), b.clone().requires_grad_()
        feat = op(a, b)
        (feat * gout).sum().backward()
        return _flatten((feat, a.grad, b.grad))
    run(tri, tp, tpf)
    _same_bits(run(tri, 2 * tpf, -tp), run(fresh, 2 * tpf, -tp), "reused triplane")


# --------------------------------------------------------------------------------------- pose decode and asset ops

@pytest.mark.gpu
def test_decode_smplx_pose(dev):
    from exavatar_release_b200 import decode_smplx_pose
    from test_human_assets import _golden_module
    params, w = _golden_module().pose_case()
    p32 = {k: v.float().to(dev) for k, v in params.items()}
    wd = {k: v.float().to(dev) for k, v in w.items()}

    def run():
        leaves = {k: v.clone().requires_grad_() for k, v in p32.items()}
        out = decode_smplx_pose(leaves)
        sum((out[k] * wd[k]).sum() for k in wd if k in out).backward()
        return {k: v for k, v in out.items() if k not in ("expr", "trans")}, \
            {k: v.grad for k, v in leaves.items() if v.grad is not None}
    check_memory(run)


@pytest.mark.gpu
@pytest.mark.parametrize("warmup", [False, True])
@pytest.mark.parametrize("P", [1, 255, 257])
def test_human_assets(P, warmup, dev):
    from exavatar_release_b200.human_assets import human_colors_reference, human_geometry_reference
    from test_human_assets import GEO_GRAD, GEO_IN, _assets, _c4_geometry, _geo_loss, _weights
    d, mask = _c4_geometry(P=P, seed=P)
    ha = _assets(mask)
    w = _weights(P, 9)

    def run():
        lv = {k: v.clone().requires_grad_() for k, v in d.items()}
        res = ha.geometry(*[lv[k] for k in GEO_IN], warmup=warmup)
        rgb, rgb_r = ha.colors(lv["rgb"], lv["rgb_offset"])
        _geo_loss(res, rgb, rgb_r, w).backward()
        return {k: v for k, v in res.items() if k != "mean_offset"}, rgb, rgb_r, {k: lv[k].grad for k in GEO_GRAD}
    got = check_memory(run)
    l64 = {k: v.double().requires_grad_() for k, v in d.items()}
    r64 = human_geometry_reference(*[l64[k] for k in GEO_IN], mask, warmup)
    c64 = human_colors_reference(l64["rgb"], l64["rgb_offset"])
    for k, v in r64.items():
        if f"out[0].{k}" in got:
            _close(got[f"out[0].{k}"], v, 1e-6, k)
    _close(got["out[1]"], c64[0], 1e-6, "rgb")
    _geo_loss(r64, *c64, [x.double() for x in w]).backward()
    for k in GEO_GRAD:
        _close(got[f"out[3].{k}"], l64[k].grad, 1e-5, f"d{k}")


@pytest.mark.gpu
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("P", [1, 255, 257])
def test_scene_assets(P, deg, dev):
    from test_scene_assets import _deg, _params, _run, _weights
    p = _params(P, seed=P)
    w = _weights(P)
    for rgb in (True, False):
        if not rgb and deg:
            continue
        check_memory(lambda: _run(p, w, rgb, _deg(deg)))


# ------------------------------------------------------------------------------------------------- Adam and camera

@pytest.mark.gpu
def test_adam_state_created_under_poison(dev):
    from exavatar_release_b200.optim import Adam
    g = torch.Generator().manual_seed(0)
    shapes = [(1,), (31, 3), (257, 1), (4097, 3), (33, 16, 3)]
    init = [torch.randn(s, generator=g).to(dev) for s in shapes]
    grads = [[torch.randn(s, generator=g).to(dev) for s in shapes] for _ in range(3)]

    def run():
        ps = [torch.nn.Parameter(t.clone()) for t in init]
        opt = Adam([{"params": ps[:2], "lr": 1e-3}, {"params": ps[2:], "lr": 5e-3}])
        for gs in grads:
            for p, gr in zip(ps, gs):
                p.grad = gr.clone()
            opt.step()
        return ps, [[opt.state[p][k] for k in sorted(opt.state[p]) if isinstance(opt.state[p][k], torch.Tensor)]
                    for p in ps]
    check_memory(run, guard=False)


@pytest.mark.gpu
def test_device_render_settings(dev):
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.renderer import device_render_settings
    for H, W in ((512, 512), (45, 61)):
        cam = look_at_cam_param(23.0, (H, W), device=dev)
        bg = torch.ones(3, device=dev)
        check_memory(lambda: [v for v in device_render_settings((H, W), cam, bg)._asdict().values()
                              if isinstance(v, torch.Tensor)], guard=False)


# -------------------------------------------------------------------------------------- rasterizer backward scratch

def _frame_inputs(dev, k):
    """Frame k of three: a different camera and shifted assets, so that Gaussians visible in one frame are culled in
    the next and the other way round."""
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.synthetic import WORKLOADS, make_population_assets
    wl = WORKLOADS["C4"]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets("C4", seed=k, device=dev)
    shift = torch.tensor([(-0.6, 0.0, 0.0), (0.5, 0.2, 0.0), (0.0, -0.4, 0.3)][k], device=dev)
    human = dict(human, mean_3d=human["mean_3d"] + shift)
    refined = dict(refined, mean_3d=refined["mean_3d"] + shift)
    cam = look_at_cam_param((-35.0, 10.0, 40.0)[k], (H, W), device=dev)
    return scene, human, refined, cam, H, W


def _scratch_clean(passes, what):
    for name, ps in passes.items():
        assert int(torch.count_nonzero(ps.bwd_scratch)) == 0, (what, name)


@pytest.mark.gpu
def test_frame_plan_scratch_is_left_zero_across_frames(dev):
    from exavatar_release_b200.plan import FramePlan, grad_bucket
    from exavatar_release_b200.renderer import render_settings
    from exavatar_release_b200.synthetic import make_grad_image
    from test_refined_pass import _close as close_grads
    frames = [_frame_inputs(dev, k) for k in range(3)]
    P = frames[0][0]["mean_3d"].shape[0]
    H, W = frames[0][4:]

    def one(plan, k, accumulate, bucket, densify=None):
        scene, _, _, cam, _, _ = frames[k]
        st = render_settings((H, W), cam, torch.ones(3, device=dev))
        sc = plan.scene(k, st, scene)
        plan.forward(sc)
        plan.backward(sc, make_grad_image("C4", k).to(dev), bucket, accumulate=accumulate, densify=densify)
        torch.cuda.synchronize()
        return plan.color.clone()

    plan = FramePlan(P, W, H, 8_000_000, dev)
    vis = []
    for k in range(3):
        _, bucket = grad_bucket(P, dev)
        for v in bucket.values():
            v.fill_(float("nan"))  # write mode: every row is written, zeros for culled Gaussians
        dens = {n: torch.zeros(P, device=dev) for n in ("grad_accum", "count", "radius_max")}
        img = one(plan, k, False, bucket, dens)
        assert int(torch.count_nonzero(plan.bwd_scratch)) == 0, k
        vis.append(plan.radii > 0)
        fresh = FramePlan(P, W, H, 8_000_000, dev)
        _, fb = grad_bucket(P, dev)
        fd = {n: torch.zeros(P, device=dev) for n in ("grad_accum", "count", "radius_max")}
        assert torch.equal(_bits(img), _bits(one(fresh, k, False, fb, fd))), k
        for n, v in fb.items():
            assert bool(torch.isfinite(bucket[n]).all()), (k, n)
            close_grads(bucket[n], v, (k, n))
        for n in dens:
            close_grads(dens[n], fd[n], (k, n))
        del fresh
    assert bool((vis[0] & ~vis[1]).any()) and bool((vis[1] & ~vis[0]).any())


@pytest.mark.gpu
@pytest.mark.parametrize("split", [True, False])
def test_merged_plan_scratch_is_left_zero_across_frames(split, dev):
    from exavatar_release_b200.plan import RENDERS
    from exavatar_release_b200.renderer import render_settings
    from exavatar_release_b200.synthetic import make_grad_image
    from test_refined_pass import _close as close_grads, _plan_classes
    cls = _plan_classes()[0 if split else 1]
    frames = [_frame_inputs(dev, k) for k in range(3)]
    Ps, Ph = frames[0][0]["mean_3d"].shape[0], frames[0][1]["mean_3d"].shape[0]
    H, W = frames[0][4:]
    bg_w, bg_r = torch.ones(3, device=dev), torch.tensor([0.3, 0.7, 0.2], device=dev)

    def frame(plan, k, accumulate, nan_buckets):
        scene, human, refined, cam, _, _ = frames[k]
        plan.set_scene(scene)
        if nan_buckets:
            for which in ("scene", "human", "human_refined"):
                for v in plan.grads(which).values():
                    v.fill_(float("nan"))
        gcol = {r: make_grad_image("C4", 10 * k + j).to(dev) for j, r in enumerate(RENDERS)}
        dens = {n: torch.zeros(Ps, device=dev) for n in ("grad_accum", "count", "radius_max")}
        plan.frame(k, render_settings((H, W), cam, bg_w), render_settings((H, W), cam, bg_r), scene, human, refined,
                   gcol, accumulate=accumulate, densify=dens)
        torch.cuda.synchronize()
        assert not plan.overflowed()
        return ({r: [t.clone() for t in plan.render_outputs(r)[:2]] for r in RENDERS},
                {w: {n: v.clone() for n, v in plan.grads(w).items()} for w in ("scene", "human", "human_refined")},
                dens, [plan.passes[p].radii.clone() for p in ("A", "B")])

    plan = cls(Ps, Ph, W, H, None, dev)
    prev = None
    for k in range(3):
        for accumulate in (False, True):
            got = frame(plan, k, accumulate, nan_buckets=not accumulate)
            _scratch_clean(plan.passes, (split, k, accumulate))
            if accumulate:  # the second backward of the frame added the same gradients once more
                for w, named in got[1].items():
                    for n, v in named.items():
                        close_grads(v, 2 * prev[1][w][n], (k, w, n, "accumulated"))
            else:
                fresh = cls(Ps, Ph, W, H, None, dev)
                ref = frame(fresh, k, False, nan_buckets=False)
                del fresh
                for r in RENDERS:
                    for x, y in zip(got[0][r], ref[0][r]):
                        assert torch.equal(x, y), (k, r)
                for w, named in ref[1].items():
                    for n, v in named.items():
                        assert bool(torch.isfinite(got[1][w][n]).all()), (k, w, n)
                        close_grads(got[1][w][n], v, (k, w, n))
                for n, v in ref[2].items():
                    close_grads(got[2][n], v, (k, n))
                if k:
                    assert bool(((got[3][0] > 0) & (prev[3][0] == 0)).any())
                    assert bool(((got[3][0] == 0) & (prev[3][0] > 0)).any())
                prev = got


@pytest.mark.gpu
@pytest.mark.parametrize("split", [True, False])
def test_training_frame_renderer_scratch_is_left_zero_across_frames(split, dev):
    from exavatar_release_b200.fused import TrainingFrameRenderer
    from exavatar_release_b200.plan import RENDERS
    from test_refined_pass import _close as close_grads
    frames = [_frame_inputs(dev, k) for k in range(3)]
    Ps, Ph = frames[0][0]["mean_3d"].shape[0], frames[0][1]["mean_3d"].shape[0]
    H, W = frames[0][4:]
    bg_r = torch.tensor([0.3, 0.7, 0.2], device=dev)

    def make():
        fr = TrainingFrameRenderer(Ps, Ph, (H, W), dev, {"A": 8_000_000, "B": 8_000_000})
        fr.plan.SPLIT = split
        return fr

    def frame(fr, k):
        scene, human, refined, cam, _, _ = frames[k]
        leaves = [{n: v.detach().clone().requires_grad_() for n, v in x.items()} for x in (scene, human, refined)]
        outs = fr(*leaves, cam, bg_r)
        sum((outs[r]["img"] * (0.5 + 0.1 * j)).sum() for j, r in enumerate(RENDERS)).backward()
        torch.cuda.synchronize()
        return ({r: outs[r]["img"].detach().clone() for r in RENDERS},
                [{n: v.grad.clone() for n, v in lv.items()} for lv in leaves])

    fr = make()
    for k in range(3):
        got = frame(fr, k)
        _scratch_clean(fr.plan.passes, (split, k))
        ref = frame(make(), k)
        for r in RENDERS:
            assert torch.equal(got[0][r], ref[0][r]), (k, r)
        for gs, gf in zip(got[1], ref[1]):
            for n, y in gf.items():
                close_grads(gs[n], y, (k, n))


# ---------------------------------------------------------------------------------------------- mesh key buffer

MESH_SIZES = [(512, 512), (1080, 1920), (45, 61), (512, 512)]  # (H, W): the buffer grows, then serves smaller sizes


@pytest.mark.gpu
def test_face_renderer_key_buffer_across_sizes(dev):
    from exavatar_release_b200.camera import look_at_cam_param
    from test_face_render import _renderer
    fx = _face_mesh()
    r = _renderer(fx, dev)
    tex = fx["texture"].to(dev)[None]
    mesh = fx["verts"].to(dev)
    for H, W in MESH_SIZES:
        cam = look_at_cam_param(8.0, (H, W), device=dev)
        G = torch.randn((1, 4, H, W), generator=torch.Generator().manual_seed(H)).to(dev)

        def run(op):
            m = mesh.clone().requires_grad_()
            img, p2f = op.render(tex, m[None], cam, (H, W))
            (img * G).sum().backward()
            return _flatten((img, p2f, m.grad))
        got = run(r)
        assert bool((r._keys == -1).all()), (H, W)
        _same_bits(got, run(_renderer(fx, dev)), (H, W))


def _face_mesh():
    from exavatar_release_b200.synthetic import make_face_mesh
    m = make_face_mesh()
    m["verts"] = make_human_mesh()["verts"][m["vertex_idx"]].contiguous()
    return m


@pytest.mark.gpu
def test_face_renders_in_exavatars_order_equal_each_render_alone(dev):
    """Forward A, forward B, backward B, backward A on one renderer -- ExAvatar renders the face twice per frame."""
    from exavatar_release_b200.camera import look_at_cam_param
    from test_face_render import _renderer
    fx = _face_mesh()
    r = _renderer(fx, dev)
    tex = fx["texture"].to(dev)[None]
    cams = [look_at_cam_param(y, (512, 512), device=dev) for y in (-10.0, 20.0)]
    Gs = [torch.randn((1, 4, 512, 512), generator=torch.Generator().manual_seed(s)).to(dev) for s in (1, 2)]
    meshes = [fx["verts"].to(dev).clone().requires_grad_() for _ in range(2)]
    outs = [r.render(tex, m[None], c, (512, 512)) for m, c in zip(meshes, cams)]
    (outs[1][0] * Gs[1]).sum().backward()
    (outs[0][0] * Gs[0]).sum().backward()
    assert bool((r._keys == -1).all())
    for k in range(2):
        m = fx["verts"].to(dev).clone().requires_grad_()
        img, p2f = _renderer(fx, dev).render(tex, m[None], cams[k], (512, 512))
        (img * Gs[k]).sum().backward()
        _same_bits(_flatten((outs[k][0], outs[k][1], meshes[k].grad)), _flatten((img, p2f, m.grad)), k)


@pytest.mark.gpu
def test_shaded_renderer_key_buffer_across_sizes(dev):
    from exavatar_release_b200.mesh_render import ShadedMeshRenderer
    from exavatar_release_b200.smplx_rig import SmplxRig
    from exavatar_release_b200.synthetic import make_smplx_model
    mesh = make_human_mesh()
    rig = SmplxRig(**make_smplx_model(mesh), device=dev)
    g = torch.Generator().manual_seed(11)
    ins = [t.to(dev) for t in (torch.randn(rig.NB, generator=g), 0.01 * torch.randn(rig.J, 3, generator=g),
                               0.1 * torch.randn(rig.J, 3, generator=g), torch.randn(rig.NE, generator=g))]
    with torch.no_grad():
        verts = rig.body_mesh(*ins, torch.tensor([0.02, -0.05, 0.0], device=dev))
    r = ShadedMeshRenderer(mesh["base_faces"], verts.shape[0], device=dev)
    for H, W in MESH_SIZES:
        s = min(H, W) / 512.0
        cam = {"focal": torch.tensor([1100.0 * s, 1080.0 * s], device=dev),
               "princpt": torch.tensor([W / 2.0, H / 2.0], device=dev)}
        bkg = (torch.rand(H, W, 3, generator=torch.Generator().manual_seed(W)) * 255).to(dev)
        got = r(verts, cam, bkg)
        assert bool((r._keys == -1).all()), (H, W)
        ref = ShadedMeshRenderer(mesh["base_faces"], verts.shape[0], device=dev)(verts, cam, bkg)
        assert torch.equal(_bits(got), _bits(ref)), (H, W)
        assert not torch.equal(got, bkg), (H, W)  # the mesh covers pixels at every size
