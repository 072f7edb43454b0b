"""A float64 composite of the records and tile lists the composite kernels read (App. A.3 / A.4), for the tests.

Inputs are what `composite_fwd4.cu` (K4) and `composite_bwd4.cu` (K5) read from a workspace (`_Workspace.read_ctx()`):
  geom (P, 12) float32   px, py, A2, B2 | C2, opacity, depth, thr2 | r, g, b, id | clamp << 29 (uint bits)
  ranges (tiles, 2)      each 16x16 tile's [begin, end) in `ids`
  ids                    the depth-sorted Gaussian ids of every tile
and the image size, an optional `View` (id range, background, skip_below) and, for the backward, `first_row`.  Every
record value is taken as the exact number it is (float32 -> float64 is exact); everything else is float64.  So the
reference has no projection noise in it: it differs from the kernels only by their fp32 arithmetic and ex2.approx.

Forward, as the kernels state App. A.3 (x, y = the pixel centre; the splat's list position is its 0-based index in the
tile's list, views keep the positions of the whole list):
  p2 = A2 dx^2 + C2 dy^2 + B2 dx dy,  dx = px - x, dy = py - y;  a = o 2^p2;  alpha = min(0.99, a)
  a splat is skipped unless p2 <= 0 and a >= 1/255; entries outside the view's id range are absent;
  T_{k+1} = T_k (1 - alpha_k); the first accepted splat with T_{k+1} < 1e-4 stops the pixel WITHOUT being applied;
  colour = sum_k c_k alpha_k T_k + T_final bg,  depth = sum d_k alpha_k T_k,  alpha = sum alpha_k T_k,
  n_contrib = 1-based list position of the last applied splat (0: none).

Backward (App. A.4 with App. A.6's conventions): the applied splats are those the pixel accepts at list positions
< n_contrib, with n_contrib given per pixel (K5 reads the forward's), so the transmittance stop cannot be ambiguous; the
0.99 clamp is ignored (d alpha / d a = 1).  With v_k = c_k . g + d_k g_d + g_a and bg . g the pixel's gradient dotted:
  dL/dalpha_k = T_k v_k - (sum_{j>k} v_j alpha_j T_j + T_final bg . g) / (1 - alpha_k)
  q_k = a_k dL/dalpha_k  (= dL/dp2 / ln 2)
The K5 accumulator row of a Gaussian (the convention `project_bwd.cu` consumes: it multiplies the first two by
0.5 W ln 2 / 0.5 H ln 2 and the conic entries by -0.5 after their ln 2) sums over its applied pixels:
  [ sum q (2 A2 dx + B2 dy),  sum q (2 C2 dy + B2 dx),  sum q dx^2,  sum q dx dy |
    sum q dy^2,  sum q / o,  sum alpha T g_d,  0 |  sum alpha T g_r,  sum alpha T g_g,  sum alpha T g_b,  0 ]
i.e. dL/d(px, py, A2, B2, C2) / ln 2, dL/do, dL/ddepth, dL/d(r, g, b).  Rows of Gaussians below `first_row`, outside the
view, or met only in tiles the view skips (tile_maxid < skip_below) are zero.

Flags.  A pixel is flagged where one of its decisions sits on its threshold, with the oracle's margins
(`O.fragility`): 0 < |p2| < 1e-6, |a - 1/255| <= (eps_alpha + 4e-7 mag) / 255, and (forward only) for an accepted splat up to
the stop |T_{k+1} - 1e-4| <= eps_T 1e-4; eps_alpha = 2e-5, eps_T = 2e-3.  A Gaussian is flagged when it reaches
(p2 <= 1e-6, a >= 0.5 / 255) a flagged pixel among the positions that pixel walks.

Error model.  Next to every output element the reference returns a scale S: the same sum with every term replaced by
its absolute value, each term weighted by the conditioning of its fp32 evaluation, and the kernels are held to c S.
  * a term's transmittance is a product (forward) or a chain of divisions (backward) whose relative error grows by one
    rounding of 1 - alpha_j per splat, amplified by 1 / (1 - alpha_j) (alpha's own rounding enters 1 - alpha that
    much magnified): kappa = sum_j 1 / (1 - alpha_j) over the applied splats before the term (forward) or over all of
    the pixel's applied splats (backward, which re-enters from T_final or T(hi));
  * a term's exponent carries rounding in proportion to mag = |A2| dx^2 + |C2| dy^2 + |B2 dx dy|;
  so a term t is counted as |t| (1 + mag + kappa).  In the backward, dL/dalpha_k is scaled by
  T_k |v|_k + (sum_{j>k} |v|_j alpha_j T_j + T_final |bg| . |g|) / (1 - alpha_k), with |v| = |c| . |g| + |d g_d| + |g_a|.
  * A pixel that continues behind the 512-entry segment of k enters K5 at the cut hi from the forward's checkpoint
    record: B = (C_final - C_prefix(hi)) . g / T(hi).  The subtraction of the two fp32 sums loses their rounding, so B
    carries |g| . (|C_final| + |C_prefix|) / T(hi) (colour, depth and alpha sums), and that error reaches dL/dalpha_k
    multiplied by T_k / T_{k+1}: the term |g| . (|C_final| + |C_prefix(hi)|) / (1 - alpha_k) joins k's scale (DESIGN §3.3).
The constants c_f (forward) and c_b (gradient rows) that the kernels meet are measured in tests/test_composite_records.py.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np

TILE = 16
SEG = 512                  # list positions per segment (common.cuh SEG)
# the kernels' fp32 constants (common.cuh), as the float64 numbers they are
T_MIN = float(np.float32(1e-4))
ALPHA_MIN = float(np.float32(1.0) / np.float32(255.0))
ALPHA_MAX = float(np.float32(0.99))
LN2 = float(np.log(2.0))
EPS_ALPHA, EPS_T, EPS_POWER = 2e-5, 2e-3, 1e-6  # O.fragility's margins
ID_MASK = 0x1FFFFFFF


@dataclass
class View:
    """B2RView's selection: Gaussians [id_begin, id_end) take part (None: all), `bg` replaces the scene's background,
    tiles whose largest listed id is < skip_below are skipped (0: none)."""
    id_begin: int = 0
    id_end: Optional[int] = None
    bg: Optional[tuple] = None
    skip_below: int = 0


def record_ids(geom):
    """Gaussian id of every record (the clamp bits of the id word removed)."""
    return np.ascontiguousarray(geom[:, 11], dtype=np.float32).view(np.uint32) & ID_MASK


def tile_pixels(tile, W, H):
    """(x, y, flat index) of the tile's pixels inside the image, in row-major order."""
    gx = (W + TILE - 1) // TILE
    tx, ty = tile % gx, tile // gx
    ys, xs = np.mgrid[ty * TILE:min(ty * TILE + TILE, H), tx * TILE:min(tx * TILE + TILE, W)]
    xs, ys = xs.ravel(), ys.ravel()
    return xs, ys, ys * W + xs


def skipped_tiles(ranges, ids, skip_below):
    """Tiles a view with `skip_below` skips: the largest id of the list (0 for an empty one) is below it."""
    if not skip_below:
        return np.zeros(len(ranges), bool)
    mx = np.array([int(ids[a:b].max()) if b > a else 0 for a, b in ranges], np.int64)
    return mx < skip_below


class _Tile:
    """One tile's pixels x in-view list entries, everything App. A.3 evaluates per (pixel, splat), in float64."""

    def __init__(self, geom, ranges, ids, tile, W, H, view):
        a, b = (int(v) for v in ranges[tile])
        lst = np.asarray(ids[a:b], np.int64)
        lo, hi = view.id_begin, (view.id_end if view.id_end is not None else len(geom))
        keep = (lst >= lo) & (lst < hi)
        self.pos = np.nonzero(keep)[0]                 # list positions (0-based) of the in-view entries
        self.gid = lst[keep]
        self.x, self.y, self.pix = tile_pixels(tile, W, H)
        g = geom[self.gid].astype(np.float64)
        self.rec = g
        dx = g[None, :, 0] - self.x[:, None]
        dy = g[None, :, 1] - self.y[:, None]
        A2, B2, C2, o = g[:, 2], g[:, 3], g[:, 4], g[:, 5]
        self.dx, self.dy = dx, dy
        self.p2 = A2 * dx * dx + C2 * dy * dy + B2 * dx * dy
        self.mag = np.abs(A2) * dx * dx + np.abs(C2) * dy * dy + np.abs(B2 * dx * dy)
        self.G = np.exp2(self.p2)
        self.araw = o * self.G
        self.ok = (self.p2 <= 0) & (self.araw >= ALPHA_MIN)
        self.alpha = np.minimum(ALPHA_MAX, self.araw)
        # decisions on their threshold (the transmittance test is added by the forward)
        # (p2 == 0 exactly only at dx = dy = 0, which fp32 evaluates exactly as well)
        self.frag_a = ((self.p2 != 0) & (np.abs(self.p2) < EPS_POWER)) | (
            (self.p2 <= 0) & (np.abs(self.araw - ALPHA_MIN) <= (EPS_ALPHA + 4e-7 * self.mag) * ALPHA_MIN))
        self.reach = (self.p2 <= EPS_POWER) & (self.araw >= 0.5 * ALPHA_MIN)

    def transmittance(self, applied):
        """T before each entry, T_final and kappa (sum of 1 / (1 - alpha) over the applied splats before each entry)."""
        om = np.where(applied, 1.0 - self.alpha, 1.0)
        incl = np.cumprod(om, axis=1)
        Tb = np.concatenate([np.ones((om.shape[0], 1)), incl[:, :-1]], axis=1)
        inv = np.where(applied, 1.0 / om, 0.0)
        kap = np.cumsum(inv, axis=1) - inv
        Tf = incl[:, -1] if om.shape[1] else np.ones(om.shape[0])
        return Tb, Tf, kap, inv.sum(axis=1)


def _positions_walked(t, stop_idx):
    """(pixels, entries) mask: entries the pixel walks, i.e. in-view entries with list position <= the stop's."""
    return t.pos[None, :] <= stop_idx[:, None]


def forward(geom, ranges, ids, W, H, bg, view: Optional[View] = None):
    """Float64 forward composite.  Returns a dict of (3,H,W) colour, (H,W) depth, alpha, final_T, n_contrib (int64),
    their scales S_color, S_depth, S_alpha, S_T, the pixel flags `flag`, the Gaussian flags `gflag` (P), and
    `written` (H,W): pixels the kernel writes (False in tiles the view skips).  `stop` (H,W) is the 0-based list position
    of the splat that stopped the pixel (-1: none)."""
    view = view or View()
    bgv = np.asarray(view.bg if view.bg is not None else bg, np.float64)
    P, N = len(geom), W * H
    out = {k: np.zeros((3, N)) for k in ("color", "S_color")}
    out.update({k: np.zeros(N) for k in ("depth", "alpha", "final_T", "S_depth", "S_alpha", "S_T")})
    out["n_contrib"] = np.zeros(N, np.int64)
    out["stop"] = np.full(N, -1, np.int64)
    out["flag"] = np.zeros(N, bool)
    out["written"] = np.zeros(N, bool)
    out["gflag"] = np.zeros(P, bool)
    skip = skipped_tiles(ranges, ids, view.skip_below)
    for tile in range(len(ranges)):
        if skip[tile]:
            continue
        t = _Tile(geom, ranges, ids, tile, W, H, view)
        if t.pix.size == 0:
            continue
        m, n = t.p2.shape
        out["written"][t.pix] = True
        # the running product over every accepted splat, the stopping one included
        om = np.where(t.ok, 1.0 - t.alpha, 1.0)
        incl = np.cumprod(om, axis=1) if n else np.ones((m, 0))
        stopm = t.ok & (incl < T_MIN)
        has = stopm.any(axis=1)
        s = np.where(has, np.argmax(stopm, axis=1), n) if n else np.zeros(m, np.int64)
        applied = t.ok & (np.arange(n)[None, :] < s[:, None])
        Tb, Tf, kap, ktot = t.transmittance(applied)
        w = np.where(applied, t.alpha * Tb, 0.0)
        wt = w * (1.0 + t.mag + kap)
        c, d = t.rec[:, 8:11], t.rec[:, 6]
        out["color"][:, t.pix] = (w @ c).T + Tf[None, :] * bgv[:, None]
        out["S_color"][:, t.pix] = (wt @ np.abs(c)).T + (Tf * (1.0 + ktot))[None, :] * np.abs(bgv)[:, None]
        out["depth"][t.pix] = w @ d
        out["S_depth"][t.pix] = wt @ np.abs(d)
        out["alpha"][t.pix] = w.sum(axis=1)
        out["S_alpha"][t.pix] = wt.sum(axis=1)
        out["final_T"][t.pix] = Tf
        out["S_T"][t.pix] = Tf * (1.0 + ktot)
        last = np.where(applied, t.pos[None, :] + 1, 0)
        out["n_contrib"][t.pix] = last.max(axis=1) if n else 0
        out["stop"][t.pix] = np.where(has, t.pos[np.minimum(s, max(n - 1, 0))] if n else -1, -1)
        # flags: alpha / power decisions up to the stop, the transmittance test of every accepted splat up to it
        walked = np.arange(n)[None, :] <= s[:, None]
        frag = (t.frag_a & walked).any(axis=1)
        frag |= (t.ok & walked & (np.abs(incl - T_MIN) <= EPS_T * T_MIN)).any(axis=1)
        out["flag"][t.pix] |= frag
        if frag.any():
            out["gflag"][t.gid[(t.reach & walked)[frag].any(axis=0)]] = True
    shp = lambda a: a.reshape(a.shape[:-1] + (H, W))
    return {k: (shp(v) if k != "gflag" else v) for k, v in out.items()}


def backward(geom, ranges, ids, W, H, bg, n_contrib, dL_dcolor, dL_ddepth=None, dL_dalpha=None,
             view: Optional[View] = None, first_row: int = 0, cuts: bool = True):
    """Float64 K5: the (P, 12) accumulator rows, their scales S (P, 12), and the Gaussian flags (P).  `n_contrib` (H,W)
    is the forward's (the kernel's); `cuts`: lists of >= SEG entries are replayed from checkpoints (the workspace has a
    checkpoint store), which adds the cut term to the scale of the splats in front of a cut the pixel walks past."""
    view = view or View()
    bgv = np.asarray(view.bg if view.bg is not None else bg, np.float64)
    P, N = len(geom), W * H
    ncon = np.asarray(n_contrib, np.int64).reshape(N)
    gc = np.asarray(dL_dcolor, np.float64).reshape(3, N)
    gd = None if dL_ddepth is None else np.asarray(dL_ddepth, np.float64).reshape(N)
    ga = None if dL_dalpha is None else np.asarray(dL_dalpha, np.float64).reshape(N)
    rows, S = np.zeros((P, 12)), np.zeros((P, 12))
    gflag = np.zeros(P, bool)
    skip = skipped_tiles(ranges, ids, view.skip_below)
    for tile in range(len(ranges)):
        if skip[tile]:
            continue
        t = _Tile(geom, ranges, ids, tile, W, H, view)
        m, n = t.p2.shape
        if m == 0 or n == 0:
            continue
        nc = ncon[t.pix]
        applied = t.ok & (t.pos[None, :] < nc[:, None])
        Tb, Tf, _, ktot = t.transmittance(applied)
        g = gc[:, t.pix].T                                   # (m, 3)
        c, d = t.rec[:, 8:11], t.rec[:, 6]
        gdp = np.zeros(m) if gd is None else gd[t.pix]
        gap = np.zeros(m) if ga is None else ga[t.pix]
        v = g @ c.T + gdp[:, None] * d[None, :] + gap[:, None]
        va = np.abs(g) @ np.abs(c).T + np.abs(gdp)[:, None] * np.abs(d)[None, :] + np.abs(gap)[:, None]
        w = np.where(applied, t.alpha * Tb, 0.0)
        om = 1.0 - t.alpha
        term, terma = v * w, va * w
        suf = term.sum(axis=1, keepdims=True) - np.cumsum(term, axis=1)
        sufa = terma.sum(axis=1, keepdims=True) - np.cumsum(terma, axis=1)
        bgd = (g @ bgv) * Tf
        bga = (np.abs(g) @ np.abs(bgv)) * Tf
        dLda = np.where(applied, Tb * v - (suf + bgd[:, None]) / om, 0.0)
        sda = Tb * va + (sufa + bga[:, None]) / om
        rng = int(ranges[tile][1]) - int(ranges[tile][0])
        if cuts and rng >= SEG:
            # pixels that walk past the cut at the end of k's segment enter there from the checkpoint record
            hi = (t.pos // SEG + 1) * SEG                     # (n,) the cut behind each entry
            cont = nc[:, None] > hi[None, :]
            cum = np.cumsum(terma, axis=1)                    # |g| . |C_prefix| after each entry
            tot = cum[:, -1:]
            # |C_prefix(hi)|: the prefix up to the last in-view entry before the cut
            idx = np.searchsorted(t.pos, hi, side="left") - 1
            pre = np.where(idx[None, :] >= 0, cum[:, np.maximum(idx, 0)], 0.0)
            sda = sda + np.where(cont, (tot + pre) / om, 0.0)
        sda = np.where(applied, sda * (1.0 + t.mag + ktot[:, None]), 0.0)
        q = t.araw * dLda
        qa = t.araw * sda
        A2, B2, C2, o = t.rec[:, 2], t.rec[:, 3], t.rec[:, 4], t.rec[:, 5]
        dx, dy = t.dx, t.dy
        fx, fy = 2 * A2 * dx + B2 * dy, 2 * C2 * dy + B2 * dx
        fxa = np.abs(2 * A2 * dx) + np.abs(B2 * dy)
        fya = np.abs(2 * C2 * dy) + np.abs(B2 * dx)
        wgt = np.where(applied, 1.0 + t.mag + ktot[:, None], 0.0)
        acc = np.stack([(q * fx).sum(0), (q * fy).sum(0), (q * dx * dx).sum(0), (q * dx * dy).sum(0),
                        (q * dy * dy).sum(0), (dLda * t.G).sum(0), (w * gdp[:, None]).sum(0), np.zeros(n),
                        *[(w * g[:, ch:ch + 1]).sum(0) for ch in range(3)], np.zeros(n)], axis=1)
        acca = np.stack([(qa * fxa).sum(0), (qa * fya).sum(0), (qa * dx * dx).sum(0), (qa * np.abs(dx * dy)).sum(0),
                         (qa * dy * dy).sum(0), (sda * t.G).sum(0), (w * wgt * np.abs(gdp)[:, None]).sum(0), np.zeros(n),
                         *[(w * wgt * np.abs(g[:, ch:ch + 1])).sum(0) for ch in range(3)], np.zeros(n)], axis=1)
        np.add.at(rows, t.gid, acc)
        np.add.at(S, t.gid, acca)
        walked = t.pos[None, :] < nc[:, None]
        frag = (t.frag_a & walked).any(axis=1)
        if frag.any():
            gflag[t.gid[(t.reach & walked)[frag].any(axis=0)]] = True
    if first_row:
        rows[:first_row] = 0.0
        S[:first_row] = 0.0
    return rows, S, gflag


def backward_pixel_flags(geom, ranges, ids, W, H, n_contrib, view: Optional[View] = None):
    """(H,W) pixels whose alpha / power decisions among the entries before n_contrib sit on their threshold."""
    view = view or View()
    ncon = np.asarray(n_contrib, np.int64).reshape(W * H)
    flag = np.zeros(W * H, bool)
    skip = skipped_tiles(ranges, ids, view.skip_below)
    for tile in range(len(ranges)):
        if skip[tile]:
            continue
        t = _Tile(geom, ranges, ids, tile, W, H, view)
        if t.pix.size and t.pos.size:
            flag[t.pix] = (t.frag_a & (t.pos[None, :] < ncon[t.pix][:, None])).any(axis=1)
    return flag.reshape(H, W)
