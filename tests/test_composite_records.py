"""The forward and backward composites (K4 `composite_fwd4.cu`, K5 `composite_bwd4.cu`) held per pixel and per
accumulator row against a float64 composite of exactly the records and tile lists they read (tests/composite_reference.py).

The C ABI is driven directly: b2r_forward_project -> b2r_forward_bin -> b2r_forward_composite (with or without a
B2RView) -> b2r_backward_composite, whose (P, 12) scratch is read back before any K6 runs.  Outputs start as NaN (and
n_contrib as 0xffffffff) with NaN guards around them.  Scenes are designed under the identity camera of the KATs: each
Gaussian is back-projected from a chosen pixel position, footprint and depth, so the lists hold what a case needs, and
every case asserts from the lists the kernels composited that it reaches its edge.

Kernel boundary                                             case that reaches it
-------------------------------------------------------------------------------------------------------------------------
list lengths 0, 1, 31..33, 127..129, 511..513, 1023..1025, 1537   lengths: one 16x16 tile per length, splats inside their
  (batch of 128 / cull chunk of 32 / SEG = 512 cuts, nrec)          tile, broad splats spanning tiles in the lower rows
stop (first splat not applied) at 0-based list position 510, 511,  stops: tiles 0 and 1, a 1 / 0.95 / 1 opacity stack at
  512 (first entry after a cut), 513, 1022..1025; n_contrib at     one pixel per target
  exactly 512 and 1024 (the cut), 513 and 1025 (one past)
a quarter whose 64 pixels all die before the first cut (the      stops: tile 2, quarter 1 (the forward's CTA break; the
  forward's CTA break, records 0 and 1 never written)               later records of that quarter are never written)
a dead warp beside a live partner                                stops: tile 2, quarter 3 (rows 8-11 dead before 512)
survivors per 32-entry chunk 0..32, every leftover modulo 4      groups: chunk c holds c splats in quarter 0's upper
  (forward group) and 2 (backward group), both circular queues     8x4 rect; > 500 survivors wrap both queues (36 / 48
  wrapped, a last phase-B drain of < 16 splats                      slots) many times
W % 4 == 0 (vector stores), fully-outside right quarters, a      edges (52, 35); the same outputs one float off
  bottom tile row where one warp has 3 live rows, the other none   (scalar stores) are bit-identical
scalar stores with a 5-column right quarter                      edges (61, 43)
a one-row image                                                  edges (17, 1)
views: an id range through a tile's lists, per-view background,  views: cat(scene from SH, human); the human-only view
  final_T, n_contrib and checkpoints, skip_below (with a tile      and the combined view (skip_below = first_row = #scene)
  whose largest id equals it), first_row on a hit Gaussian, two    into one scratch; an id range [#scene / 2, #scene + 7)
  views in one scratch, SH colours with clamped channels           bit-equal to a scene of only those rows
backward gradient inputs: none, depth, alpha, both (HAS_DA)      stops, lengths
checkpoints absent (lists are one segment)                       lengths, stops: forward bit-identical, backward vs ref

Tolerances (error model in composite_reference.py): |kernel - reference| <= c S per element, on the pixels and
Gaussians whose decisions do not sit on a threshold (flags: at most 0.5 % of a case's pixels).  Measured on an NVIDIA
H100 80GB HBM3 (700 W), largest over every case: forward |d| / S = 1.5e-7 (views/range), accumulator rows 6.3e-8
(edges 61 x 43) -- about one fp32 rounding per weighted term.  C_F and C_B leave 2.5x and 6x headroom for the run-to-run
order of the fp32 atomics.
"""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import composite_reference as R
from util import kat_settings, settings_on
from util import dev  # noqa: F401

F = 40.0              # focal length in pixels of the identity camera
SEG = R.SEG
BG = (0.25, 0.5, 0.75)
# |kernel - reference| <= C S per element; measured 1.5e-7 / 6.3e-8 on an H100 (see the docstring)
C_F = 4e-7
C_B = 4e-7
SENT = 0xFFFFFFFF


# ------------------------------------------------------------------ scenes ----------------------------------------------

def _splats(W, H, rows):
    """Assets from rows (x, y, sigma_u, sigma_v, theta, z, opacity, r, g, b): a Gaussian at pixel position (x, y) and
    view depth z whose screen footprint has standard deviations sigma_u, sigma_v (>= the 0.55 px of the low-pass
    dilation) along axes turned by theta."""
    r = np.asarray(rows, np.float64).reshape(-1, 10)
    x, y, su, sv, th, z, o = (r[:, k] for k in range(7))
    world = lambda s: np.sqrt(np.maximum(s * s - 0.3, 2e-3)) * z / F
    mean = np.stack([(x - W / 2 + 0.5) * z / F, (y - H / 2 + 0.5) * z / F, z], 1)
    scale = np.stack([world(su), world(sv), np.full_like(z, 1e-4)], 1)
    rot = np.stack([np.cos(th / 2), 0 * th, 0 * th, np.sin(th / 2)], 1)
    t = lambda a: torch.tensor(a, dtype=torch.float32)
    return dict(mean_3d=t(mean), scale=t(scale), rotation=t(rot), opacity=t(o[:, None]), rgb=t(r[:, 7:10]))


def _small(g, n, x0, x1, y0, y1, z, o):
    """n tiny splats (footprint 0.6 px) centred in [x0, x1] x [y0, y1] at depths z, opacities o."""
    z, o = np.broadcast_to(z, n), np.broadcast_to(o, n)
    return np.stack([g.uniform(x0, x1, n), g.uniform(y0, y1, n), np.full(n, 0.6), np.full(n, 0.6), np.zeros(n), z, o,
                     *g.uniform(0, 1, (3, n))], 1)


def _broad(g, n, x0, x1, y0, y1, s0, s1, z0=2.0, z1=6.0):
    return np.stack([g.uniform(x0, x1, n), g.uniform(y0, y1, n), g.uniform(s0, s1, n), g.uniform(s0, s1, n),
                     g.uniform(0, np.pi, n), g.uniform(z0, z1, n), g.uniform(0.1, 0.95, n), *g.uniform(0, 1, (3, n))], 1)


LENGTHS = (0, 1, 31, 32, 33, 127, 128, 129, 511, 512, 513, 1023, 1024, 1025, 1537)


def _lengths_rows():
    """128 x 64: tile (k % 8, k // 8) holds LENGTHS[k] splats inside it; tile rows 2-3 hold broad splats."""
    g = np.random.default_rng(11)
    rows = []
    for k, n in enumerate(LENGTHS):
        tx, ty = k % 8, k // 8
        o = (0.02, 0.3) if n < 200 else (0.01, 0.05)
        rows.append(_small(g, n, 16 * tx + 3.5, 16 * tx + 12.5, 16 * ty + 3.5, 16 * ty + 12.5, g.uniform(2, 6, n),
                           g.uniform(*o, n)))
    rows.append(_broad(g, 40, 2, 126, 47, 62, 1.5, 4.5))
    rows.append(_small(g, 60, 1, 127, 35, 63, g.uniform(2, 6, 60), g.uniform(0.1, 0.9, 60)))
    return np.concatenate(rows)


STOPS = {0: (511, 513, 1023, 1025), 1: (510, 512, 1022, 1024)}  # 0-based list position of the stopping splat
N_STOP_LIST = 1100


def _stops_rows():
    """48 x 16, lists of 1100 entries in designed order (depth rises with the list position).  Tiles 0 and 1: a faint
    veil, and for each target s an opacity-1 splat early, a 0.95 one at s - 1 and an opacity-1 one at s, all centred
    on one pixel.  Tile 2: forty 0.99 splats of footprint 3 px first (quarter 1 dies), forty flat ones on rows 8-11 of
    quarter 3 (its upper warp dies, the lower lives), then the veil."""
    g = np.random.default_rng(5)
    rows = []
    zpos = lambda k: 2.0 + 4.0 * k / N_STOP_LIST
    for t in range(3):
        x0 = 16 * t
        kinds = {}
        if t < 2:
            for i, s in enumerate(STOPS[t]):
                # a tenth of a pixel off the pixel centre: no exponent within 1e-6 of 0 (a flagged decision)
                px, py = x0 + 3.1 + 4 * (i % 3), 3.05 + 4 * (i // 3) + 4 * (i % 2)
                kinds[s - 200] = (px, py, 1.0)
                kinds[s - 1] = (px, py, 0.95)
                kinds[s] = (px, py, 1.0)
        else:
            for k in range(40):
                kinds[k] = ("q1", x0 + 11.5, 3.5)
                kinds[40 + k] = ("w", x0 + 11.5, 9.5)
        for k in range(N_STOP_LIST):
            z = zpos(k)
            v = kinds.get(k)
            if v is None:
                rows.append(_small(g, 1, x0 + 3, x0 + 12, 3, 12, z, g.uniform(0.01, 0.03))[0])
            elif v[0] == "q1":
                rows.append([v[1], v[2], 3.0, 3.0, 0.0, z, 0.99, *g.uniform(0, 1, 3)])
            elif v[0] == "w":
                rows.append([v[1], v[2], 3.0, 1.2, 0.0, z, 0.99, *g.uniform(0, 1, 3)])
            else:
                rows.append([v[0], v[1], 0.6, 0.6, 0.0, z, v[2], *g.uniform(0, 1, 3)])
    return np.array(rows)


def _groups_rows():
    """16 x 16, 33 chunks of 32 entries in designed order: chunk c holds c splats inside quarter 0's upper 8x4 rect and
    32 - c inside quarter 3, shuffled."""
    g = np.random.default_rng(9)
    rows = []
    for c in range(33):
        a = _small(g, c, 0.0, 7.0, 0.0, 3.0, 0.0, g.uniform(0.005, 0.012, c))
        b = _small(g, 32 - c, 9.5, 14.5, 9.5, 14.5, 0.0, g.uniform(0.01, 0.05, 32 - c))
        chunk = np.concatenate([a, b])[g.permutation(32)]
        chunk[:, 5] = 2.0 + 4.0 * (32 * c + np.arange(32)) / 1056
        rows.append(chunk)
    return np.concatenate(rows)


def _edges_rows(W, H, seed):
    g = np.random.default_rng(seed)
    n_s, n_b = 4 * W + 20, 25
    return np.concatenate([_small(g, n_s, -1.5, W + 0.5, -1.5, H + 0.5, g.uniform(2, 6, n_s), g.uniform(0.05, 0.9, n_s)),
                           _broad(g, n_b, -4, W + 4, -4, H + 4, 1.0, 6.0)])


def _views_rows():
    """64 x 32: scene rows (small and broad splats everywhere) and human rows.  The first human row is alone in tile
    (3, 1); the other human rows sit in tiles (1..2, 0..1), interleaved in depth with the scene."""
    g = np.random.default_rng(21)
    scene = np.concatenate([_small(g, 300, 0, 63, 0, 31, g.uniform(2, 6, 300), g.uniform(0.05, 0.8, 300)),
                            _broad(g, 30, 0, 63, 0, 31, 1.0, 5.0)])
    first = [[56.0, 24.0, 0.6, 0.6, 0.0, 2.5, 0.7, 0.9, 0.1, 0.4]]
    human = np.concatenate([_small(g, 120, 19, 37, 5, 27, g.uniform(2, 6, 120), g.uniform(0.1, 0.9, 120)),
                            _broad(g, 10, 22, 34, 10, 22, 1.0, 2.5)])
    return scene, np.concatenate([first, human])


# ------------------------------------------------------------------ harness ---------------------------------------------

def _L():
    from exavatar_release_b200 import _lib as L
    return L


class _Frame:
    """One scene projected and binned through the C ABI into a `_Workspace`, and the lists and records read back."""

    def __init__(self, dev, W, H, assets, bg=BG, shs=None, sh_degree=0):
        from exavatar_release_b200.plan import _Workspace
        from exavatar_release_b200.rasterizer import GaussianRasterizationSettings, _make_scene
        L = _L()
        self.dev, self.W, self.H, self.bg = dev, W, H, bg
        st = settings_on(kat_settings(W, H, F, bg), dev, GaussianRasterizationSettings)
        if shs is not None:
            st = st._replace(sh_degree=sh_degree)
        self.a = {k: v.to(dev).contiguous() for k, v in assets.items()}
        self.shs = None if shs is None else shs.to(dev).contiguous()
        self.P = P = self.a["mean_3d"].shape[0]
        self.sc, self.keep = _make_scene(st, self.a["mean_3d"], self.shs, None if shs is not None else self.a["rgb"],
                                         self.a["opacity"], self.a["scale"], self.a["rotation"], None, 0)
        self.ws = _Workspace(P, W, H, 40 * P + 4096, dev)
        s = self.stream = torch.cuda.current_stream(dev).cuda_stream
        lib = self.lib = L.load()
        L.check(lib.b2r_forward_project(C.byref(self.sc), C.byref(self.ws.ws), self.ws.radii.data_ptr(), s), "project")
        L.check(lib.b2r_forward_bin(C.byref(self.sc), C.byref(self.ws.ws), s), "bin")
        torch.cuda.synchronize()
        assert self.ws.status()["overflow"] == 0
        ctx = self.ws.read_ctx()
        self.geom, self.ranges, self.ids = ctx["geom"].copy(), ctx["ranges"].astype(np.int64), ctx["ids"].copy()
        assert np.array_equal(R.record_ids(self.geom)[self.ws.radii.cpu().numpy() > 0],
                              np.nonzero(self.ws.radii.cpu().numpy() > 0)[0])
        self.nockpt = type(self.ws.ws)(*[getattr(self.ws.ws, f) for f, _ in self.ws.ws._fields_[:8]], None, 0)

    def lists(self):
        return [self.ids[a:b].astype(np.int64) for a, b in self.ranges]

    def forward(self, view=None, ckpt=True, offset=0, own=True):
        """K4 into NaN-prefilled outputs (`offset` floats into their buffers, with 8 guard floats behind).  `view`: an
        R.View, composited through a B2RView (with its own final_T / n_contrib / checkpoints when `own`)."""
        L, W, H, N = _L(), self.W, self.H, self.W * self.H
        buf = lambda n: torch.full((offset + n + 8,), float("nan"), device=self.dev)
        out = {"color": buf(3 * N), "depth": buf(N), "alpha": buf(N)}
        ws = self.ws.ws if ckpt else self.nockpt
        v, keep = None, []
        if view is not None:
            bg = torch.tensor(view.bg if view.bg is not None else self.bg, dtype=torch.float32, device=self.dev)
            fT = buf(N) if own else None
            nc = torch.full((N,), -1, dtype=torch.int32, device=self.dev) if own else None
            ck = torch.empty(self.ws.ckpt_bytes, dtype=torch.uint8, device=self.dev) if own and ckpt else None
            keep = [bg, fT, nc, ck]
            v = L.B2RView(view.id_begin, view.id_end if view.id_end is not None else self.P, bg.data_ptr(),
                          L.ptr(fT[offset:offset + N] if fT is not None else None), L.ptr(nc),
                          L.ptr(ck), self.ws.ckpt_bytes if ck is not None else 0, view.skip_below, 0)
            if fT is not None:
                out["final_T"] = fT
        if "final_T" not in out:  # the ctx's own per-pixel state, prefilled as well
            fT_p = self.lib.b2r_ctx_final_T(C.byref(self.ws.ws), self.P, W, H)
            nc_p = self.lib.b2r_ctx_n_contrib(C.byref(self.ws.ws), self.P, W, H)
            base = self.ws.ctx_buf.data_ptr()
            self.ws.ctx_buf[fT_p - base:fT_p - base + 4 * N].view(torch.float32).fill_(float("nan"))
            self.ws.ctx_buf[nc_p - base:nc_p - base + 4 * N].view(torch.int32).fill_(-1)
        fo = L.B2RForwardOutputs(*(out[k][offset:].data_ptr() for k in ("color", "depth", "alpha")), None)
        L.check(self.lib.b2r_forward_composite(C.byref(self.sc), C.byref(ws), C.byref(v) if v is not None else None,
                                               C.byref(fo), self.stream), "forward_composite")
        torch.cuda.synchronize()
        res = {k: t.cpu().numpy() for k, t in out.items()}
        for k, a in res.items():  # the guards before and behind the outputs
            assert np.isnan(a[:offset]).all() and np.isnan(a[-8:]).all(), k
        res = {k: a[offset:-8] for k, a in res.items()}
        res["color"] = res["color"].reshape(3, H, W)
        for k in ("depth", "alpha", "final_T"):
            if k in res:
                res[k] = res[k].reshape(H, W)
        if view is not None and own:
            res["n_contrib"] = keep[2].cpu().numpy().view(np.uint32).reshape(H, W)
        else:
            ctx = self.ws.read_ctx()
            res["final_T"], res["n_contrib"] = ctx["final_T"].copy(), ctx["n_contrib"].copy()
        res["_view"], res["_keep"], res["_ws"] = v, keep, ws
        return res

    def backward(self, fwd, gcol, gd=None, ga=None, first_row=0, scratch=None):
        """K5 of the view `fwd` was composited with; flags = 0 (K5 clears the scratch) unless `scratch` is given, which
        it then accumulates into (B2R_BWD_SCRATCH_ZEROED: nothing is cleared).  Returns the scratch as (P, 12)."""
        L = _L()
        zeroed = scratch is not None
        if scratch is None:
            scratch = torch.full((self.ws.bwd_bytes // 4,), float("nan"), device=self.dev)
        t = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32,
                                                                  device=self.dev)
        imgs = [t(gcol), t(gd), t(ga)]
        args = L.B2RBackwardArgs(*(L.ptr(i) for i in imgs), *([None] * 8), L.B2R_BWD_SCRATCH_ZEROED if zeroed else 0,
                                 first_row, None, None, None, 0, 0)
        v = fwd["_view"]
        L.check(self.lib.b2r_backward_composite(C.byref(self.sc), C.byref(fwd["_ws"]), C.byref(v) if v is not None
                                                else None, C.byref(args), scratch.data_ptr(), self.ws.bwd_bytes,
                                                self.stream), "backward_composite")
        torch.cuda.synchronize()
        return scratch

    def rows(self, scratch):
        return scratch[:12 * self.P].cpu().numpy().astype(np.float64).reshape(self.P, 12)


def _check_forward(case, fr, got, view=None):
    """Per pixel against the reference; returns the reference's forward."""
    ref = R.forward(fr.geom, fr.ranges, fr.ids, fr.W, fr.H, fr.bg, view)
    wr, ok = ref["written"], ref["written"] & ~ref["flag"]
    nflag = int((ref["flag"] & wr).sum())
    assert nflag <= 0.005 * wr.sum() + 1, (case, nflag)
    for k in ("color", "depth", "alpha", "final_T"):
        assert np.isnan(got[k][..., ~wr]).all(), (case, k, "a skipped tile was written")
    assert (got["n_contrib"][~wr] == SENT).all(), case
    assert np.array_equal(got["n_contrib"][ok], ref["n_contrib"][ok]), case
    worst = 0.0
    for k, s in (("color", "S_color"), ("depth", "S_depth"), ("alpha", "S_alpha"), ("final_T", "S_T")):
        d = np.abs(got[k].astype(np.float64) - ref[k])[..., ok]
        S = ref[s][..., ok]
        assert np.isfinite(d).all(), (case, k)
        r = float((d / np.maximum(S, 1e-30)).max()) if d.size else 0.0
        worst = max(worst, r)
        assert (d <= C_F * S).all(), f"{case} {k}: max |d| / S = {r:.3e} > {C_F:.1e}"
    print(f"{case}: forward max |d|/S = {worst:.3e}, flagged pixels {nflag}", flush=True)
    return ref


def _check_rows(case, fr, got, want, S, gflag, zero=()):
    """Accumulator rows within C_B S, exactly zero where the reference has no term at all, and on `zero` rows."""
    ok = ~gflag
    assert gflag.sum() <= max(0.02 * fr.P, 3), (case, int(gflag.sum()))
    assert np.isfinite(got).all(), case
    d, Sk = np.abs(got - want)[ok], S[ok]
    r = float((d / np.maximum(Sk, 1e-30)).max())
    print(f"{case}: rows max |d|/S = {r:.3e}, flagged Gaussians {int(gflag.sum())}", flush=True)
    bad = d > C_B * Sk
    assert not bad.any(), f"{case}: {int(bad.sum())} elements, max |d| / S = {r:.3e} > {C_B:.1e}"
    none = ok & ~S.any(axis=1)
    assert not got[none].any(), (case, "rows without a term")
    assert not got[:, [7, 11]].any(), case
    for i in zero:
        assert not got[i].any(), (case, i)
    return int((ok & S.any(axis=1)).sum())


def _grad_images(H, W, seed):
    g = np.random.default_rng(seed)
    return g.standard_normal((3, H, W)), g.standard_normal((H, W)), g.standard_normal((H, W))


# ------------------------------------------------------------------ coverage --------------------------------------------

def _region_max_p2(rec, x0, y0, x1, y1):
    """common.cuh region_max_p2 in float64: the largest exponent over the rect [x0, x1] x [y0, y1]."""
    sx, sy, A2, B2, C2 = (rec[:, k].astype(np.float64) for k in range(5))
    lx, hx, ly, hy = sx - x1, sx - x0, sy - y1, sy - y0
    in_x, in_y = (lx <= 0) & (hx >= 0), (ly <= 0) & (hy >= 0)
    ex = np.where(lx > 0, lx, hx)
    dy = np.clip(-B2 * ex / (2 * C2), ly, hy)
    bx = np.where(~in_x, A2 * ex * ex + B2 * ex * dy + C2 * dy * dy, -np.inf)
    ey = np.where(ly > 0, ly, hy)
    dx = np.clip(-B2 * ey / (2 * A2), lx, hx)
    by = np.where(~in_y, A2 * dx * dx + B2 * dx * ey + C2 * ey * ey, -np.inf)
    return np.where(in_x & in_y, 0.0, np.maximum(bx, by))


def _survivors(fr, tile, quad, warp):
    """Per list entry of the tile: does it pass the 8x4 sub-tile cull of (quarter, warp)."""
    gx = (fr.W + 15) // 16
    tx, ty = tile % gx, tile // gx
    x0, y0 = 16 * tx + 8 * (quad & 1), 16 * ty + 8 * (quad >> 1) + 4 * warp
    x1, y1 = min(x0 + 7, fr.W - 1), min(y0 + 3, fr.H - 1)
    rec = fr.geom[fr.lists()[tile]]
    return ~(_region_max_p2(rec, x0, y0, x1, y1) < rec[:, 7].astype(np.float64))


# ------------------------------------------------------------------ frames ----------------------------------------------

@functools.lru_cache(maxsize=None)
def _frame(name, dev):
    if name == "lengths":
        return _Frame(dev, 128, 64, _splats(128, 64, _lengths_rows()))
    if name == "stops":
        return _Frame(dev, 48, 16, _splats(48, 16, _stops_rows()))
    if name == "groups":
        return _Frame(dev, 16, 16, _splats(16, 16, _groups_rows()))
    if name.startswith("edges"):
        W, H = (int(v) for v in name[5:].split("x"))
        return _Frame(dev, W, H, _splats(W, H, _edges_rows(W, H, W * 100 + H)))
    if name == "views":
        scene, human = _views_rows()
        a = _splats(64, 32, np.concatenate([scene, human]))
        g = torch.Generator().manual_seed(4)
        shs = 0.6 * torch.randn(a["mean_3d"].shape[0], 4, 3, generator=g)
        shs[:, 0] -= 0.6  # DC below -0.5 / C0 in places: clamped channels
        return _Frame(dev, 64, 32, a, shs=shs, sh_degree=1), len(scene)
    raise KeyError(name)


@pytest.mark.gpu
def test_list_lengths_at_every_batch_chunk_and_cut_boundary(dev):
    fr = _frame("lengths", dev)
    assert [int(b - a) for a, b in fr.ranges[:15]] == list(LENGTHS), "designed tiles"
    # broad splats span tiles: some Gaussians sit in the lists of three or more tiles
    assert (np.bincount(np.concatenate(fr.lists()), minlength=fr.P) >= 3).sum() >= 10
    f = fr.forward()
    ref = _check_forward("lengths", fr, f)
    g, gd, ga = _grad_images(fr.H, fr.W, 1)
    # pixels that walk past both cuts of the long tiles
    assert (ref["n_contrib"] > 2 * SEG).any()
    for name, (d, a) in {"none": (None, None), "depth": (gd, None), "alpha": (None, ga), "both": (gd, ga)}.items():
        rows = fr.rows(fr.backward(f, g, d, a))
        want, S, gflag = R.backward(fr.geom, fr.ranges, fr.ids, fr.W, fr.H, fr.bg, f["n_contrib"], g, d, a)
        assert _check_rows(f"lengths/{name}", fr, rows, want, S, gflag) > 0.5 * fr.P
    # without checkpoints: the forward bit for bit, the backward (one segment per list) against the reference
    f0 = fr.forward(ckpt=False)
    for k in ("color", "depth", "alpha", "final_T", "n_contrib"):
        assert np.array_equal(f0[k].view(np.uint32), f[k].view(np.uint32)), k
    rows = fr.rows(fr.backward(f0, g, gd, ga))
    want, S, gflag = R.backward(fr.geom, fr.ranges, fr.ids, fr.W, fr.H, fr.bg, f["n_contrib"], g, gd, ga, cuts=False)
    _check_rows("lengths/no-checkpoints", fr, rows, want, S, gflag)
    # view = NULL against a view of [0, P) with its own per-pixel state and checkpoints
    fv = fr.forward(view=R.View(0, fr.P, BG))
    for k in ("color", "depth", "alpha", "final_T", "n_contrib"):
        assert np.array_equal(fv[k].view(np.uint32), f[k].view(np.uint32)), k


@pytest.mark.gpu
def test_stops_at_cuts_early_death_and_gradient_inputs(dev):
    fr = _frame("stops", dev)
    lists = fr.lists()
    assert [l.size for l in lists] == [N_STOP_LIST] * 3
    f = fr.forward()
    ref = _check_forward("stops", fr, f)
    stop, nc = ref["stop"], ref["n_contrib"]
    for t, targets in STOPS.items():
        s = set(stop[:, 16 * t:16 * t + 16].ravel().tolist())
        assert s >= set(targets), (t, sorted(s & set(range(500, 1100))))
    assert {512, 513, 1024, 1025} <= set(nc.ravel().tolist())
    # tile 2: quarter 1 dies before the first cut, quarter 3's upper warp too while its lower warp walks past it
    q1 = stop[0:8, 40:48]
    assert (q1 >= 0).all() and (q1 < SEG).all()
    assert (stop[8:12, 40:48] >= 0).all() and (stop[8:12, 40:48] < SEG).all()
    assert (nc[12:16, 40:48] > SEG).any()
    g, gd, ga = _grad_images(fr.H, fr.W, 2)
    for name, (d, a) in {"none": (None, None), "depth": (gd, None), "alpha": (None, ga), "both": (gd, ga)}.items():
        rows = fr.rows(fr.backward(f, g, d, a))
        want, S, gflag = R.backward(fr.geom, fr.ranges, fr.ids, fr.W, fr.H, fr.bg, f["n_contrib"], g, d, a)
        _check_rows(f"stops/{name}", fr, rows, want, S, gflag)
    f0 = fr.forward(ckpt=False)
    for k in ("color", "depth", "alpha", "final_T", "n_contrib"):
        assert np.array_equal(f0[k].view(np.uint32), f[k].view(np.uint32)), k
    rows = fr.rows(fr.backward(f0, g, gd, ga))
    want, S, gflag = R.backward(fr.geom, fr.ranges, fr.ids, fr.W, fr.H, fr.bg, f["n_contrib"], g, gd, ga, cuts=False)
    _check_rows("stops/no-checkpoints", fr, rows, want, S, gflag)


@pytest.mark.gpu
def test_survivor_counts_leftovers_and_queue_wraps(dev):
    fr = _frame("groups", dev)
    n = fr.lists()[0].size
    assert n == 33 * 32
    f = fr.forward()
    ref = _check_forward("groups", fr, f)
    assert (ref["stop"][0:4, 0:8] < 0).all()  # the warp lives through the list: it culls every chunk
    hit = _survivors(fr, 0, 0, 0)
    per_chunk = hit.reshape(33, 32).sum(1)
    assert sorted(per_chunk.tolist()) == list(range(33))
    assert {int(c) % 4 for c in np.cumsum(per_chunk)} == {0, 1, 2, 3} and hit.sum() > 6 * 48
    # the backward's segments end in a phase-B drain of fewer than 16 splats and an odd leftover
    tails = []
    for q in range(4):
        for w in range(2):
            hs = _survivors(fr, 0, q, w)
            nmax = f["n_contrib"][8 * (q >> 1) + 4 * w:8 * (q >> 1) + 4 * w + 4, 8 * (q & 1):8 * (q & 1) + 8].max()
            for s0 in range(0, n, SEG):
                tails.append(int(hs[s0:min(s0 + SEG, nmax)].sum()) if nmax > s0 else 0)
    assert any(t % 16 and t % 2 for t in tails), tails
    g, gd, ga = _grad_images(fr.H, fr.W, 3)
    rows = fr.rows(fr.backward(f, g, gd, ga))
    want, S, gflag = R.backward(fr.geom, fr.ranges, fr.ids, fr.W, fr.H, fr.bg, f["n_contrib"], g, gd, ga)
    assert _check_rows("groups", fr, rows, want, S, gflag) > 0.9 * fr.P


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["52x35", "61x43", "17x1"])
def test_image_edges_and_store_paths(dev, size):
    fr = _frame("edges" + size, dev)
    W, H = fr.W, fr.H
    if size == "52x35":
        assert W % 4 == 0 and W % 16 <= 8 and H % 16 == 3  # right quarters outside; last row: 3 rows / 0 rows
    if size == "61x43":
        assert W % 16 == 13 and W % 4  # a 5-column right quarter, scalar stores
    f = fr.forward()
    _check_forward(f"edges/{size}", fr, f)
    f1 = fr.forward(offset=1)  # every output one float off its 16-byte alignment: the scalar store path
    for k in ("color", "depth", "alpha", "final_T", "n_contrib"):
        assert np.array_equal(f1[k].view(np.uint32), f[k].view(np.uint32)), k
    g, gd, ga = _grad_images(H, W, 4)
    rows = fr.rows(fr.backward(f, g, gd, ga))
    want, S, gflag = R.backward(fr.geom, fr.ranges, fr.ids, W, H, fr.bg, f["n_contrib"], g, gd, ga)
    assert _check_rows(f"edges/{size}", fr, rows, want, S, gflag) > 0


@pytest.mark.gpu
def test_views_into_one_scratch_skip_below_first_row_and_id_ranges(dev):
    fr, Ps = _frame("views", dev)
    P, W, H = fr.P, fr.W, fr.H
    lists = fr.lists()
    gx = (W + 15) // 16
    clamp = np.ascontiguousarray(fr.geom[:, 11]).view(np.uint32) >> 29
    assert (clamp != 0).sum() > 20  # SH colours clamped in some channel: the bits ride in the id word
    maxid = np.array([l.max() if l.size else 0 for l in lists])
    assert maxid[1 * gx + 3] == Ps                       # a tile whose largest id equals skip_below is composited
    assert (maxid < Ps).sum() >= 3                       # and tiles the combined view skips
    cut = [l for l in lists if ((l >= Ps // 2) & (l < Ps + 7)).any() and ((l < Ps // 2) | (l >= Ps + 7)).any()]
    assert len(cut) >= 4                                 # the id range cuts through lists
    g1, gd1, ga1 = _grad_images(H, W, 5)
    g2, _, _ = _grad_images(H, W, 6)
    vh = R.View(Ps, P, (0.9, 0.1, 0.3))
    vc = R.View(0, P, (0.2, 0.8, 0.4), skip_below=Ps)
    fh = fr.forward(view=vh)
    fc = fr.forward(view=vc)
    _check_forward("views/human", fr, fh, vh)
    rc = _check_forward("views/combined", fr, fc, vc)
    assert (~rc["written"]).any()
    scratch = fr.backward(fh, g1, gd1, ga1)
    fr.backward(fc, g2, first_row=Ps, scratch=scratch)
    rows = fr.rows(scratch)
    wh, Sh, fh_flag = R.backward(fr.geom, fr.ranges, fr.ids, W, H, fr.bg, fh["n_contrib"], g1, gd1, ga1, vh)
    wc, Sc, fc_flag = R.backward(fr.geom, fr.ranges, fr.ids, W, H, fr.bg, fc["n_contrib"], g2, None, None, vc,
                                 first_row=Ps)
    assert np.abs(wc[Ps]).max() > 0 and Sc[:Ps].max() == 0  # first_row falls on a Gaussian the combined view hits
    _check_rows("views/two-views", fr, rows, wh + wc, Sh + Sc, fh_flag | fc_flag, zero=range(Ps))
    # an id range through the lists, bit for bit a scene of only its rows
    a, b = Ps // 2, Ps + 7
    vr = R.View(a, b, (0.1, 0.2, 0.3))
    fv = fr.forward(view=vr)
    _check_forward("views/range", fr, fv, vr)
    rows = fr.rows(fr.backward(fv, g1, gd1, None))
    want, S, gflag = R.backward(fr.geom, fr.ranges, fr.ids, W, H, fr.bg, fv["n_contrib"], g1, gd1, None, vr)
    _check_rows("views/range", fr, rows, want, S, gflag, zero=[*range(a), *range(b, P)])
    sub = _Frame(dev, W, H, {k: v[a:b].cpu() for k, v in fr.a.items()}, bg=(0.1, 0.2, 0.3), shs=fr.shs[a:b].cpu(),
                 sh_degree=1)
    assert np.array_equal(sub.geom[:, :11].view(np.uint32), fr.geom[a:b, :11].view(np.uint32))
    fs = sub.forward()
    for k in ("color", "depth", "alpha", "final_T"):
        assert np.array_equal(fs[k].view(np.uint32), fv[k].view(np.uint32)), k

