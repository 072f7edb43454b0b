"""Work model of the composite kernels, computed on the CPU from the oracle's per-tile lists (analysis script, not a test).

  python tests/work_model.py [--workload C2] [--yaw 5]

SURVEY.md section 8d asks for the binding bound next to the HBM roofline: "pixel-splat evaluations E ... ALU bound =
E x instr/eval / (SMs x 128 x clk) ... state which bound binds".  This script counts, for one frame, exactly what the
CUDA composites are asked to do by their own culling rules (restated here in numpy from common.cuh `region_max_p2`):

  list entries        (tile, Gaussian) pairs of the 3-sigma rects                      -- reference list membership
  kept                ... that survive the exact 16x16 tile cull                        -- what K2/K3 bin and sort
  warp tests          kept entries x 8 warps per tile, up to where the warp's pixels are all finished
  warp hits           ... whose 8x4 pixel rect the splat can reach with alpha >= 1/255   -- trips of the hit loop
  lane evaluations    32 x warp hits
  useful evaluations  lanes that actually blend the splat (alive pixel, power <= 0, alpha >= 1/255)

and turns them into the issue-bound time of the composites on an H100 (132 SMs x 4 schedulers, 1.98 GHz) with the kernels'
instruction costs (31 / 61 warp-instructions per forward / backward hit, ~45 per 32-entry cull test + queue append).
"""
import argparse
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from util import workload_settings  # noqa: E402
from exavatar_release_b200.synthetic import WORKLOADS, make_assets  # noqa: E402
from oracle import oracle as O  # noqa: E402

LOG2E = 1.4426950408889634
SMS, GHZ = 132, 1.98  # H100 SXM: SMs and the top SM clock of a 700 W card
MARGIN = 0.02


def region_max_p2(sx, sy, A2, B2, C2, x0, y0, x1, y1):
    """numpy restatement of common.cuh region_max_p2 (upper bound of the log2 exponent over a pixel rect)."""
    lx, hx = sx - x1, sx - x0
    ly, hy = sy - y1, sy - y0
    in_x = (lx <= 0) & (hx >= 0)
    in_y = (ly <= 0) & (hy >= 0)
    best = np.full(sx.shape, -np.inf)
    ex = np.where(lx > 0, lx, hx)
    with np.errstate(divide="ignore", invalid="ignore"):
        dy = np.clip(-B2 * ex / (2 * C2), ly, hy)
        vx = A2 * ex * ex + B2 * ex * dy + C2 * dy * dy
        ey = np.where(ly > 0, ly, hy)
        dx = np.clip(-B2 * ey / (2 * A2), lx, hx)
        vy = A2 * dx * dx + B2 * dx * ey + C2 * ey * ey
    best = np.where(~in_x, np.maximum(best, vx), best)
    best = np.where(~in_y, np.maximum(best, vy), best)
    return np.where(in_x & in_y, 0.0, best)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C2")
    ap.add_argument("--yaw", type=float, default=5.0)
    ap.add_argument("--rect", default="8x4", help="pixel rect one cull test / hit covers (WxH), to compare decompositions: "
                                                    "8x4 is what the kernels use (one warp = one rect)")
    a = ap.parse_args()
    RW, RH = (int(v) for v in a.rect.split("x"))
    wl = WORKLOADS[a.workload]
    H, W = wl.height, wl.width
    assets = make_assets(a.workload, seed=0)
    st = workload_settings(a.workload, yaw=a.yaw)
    kw = dict(shs=assets["shs"]) if wl.sh_degree > 0 else dict(colors_precomp=assets["rgb"])
    if wl.sh_degree > 0:
        st = st._replace(sh_degree=wl.sh_degree)
    _, radii, _, _, ctx = O.forward(st, assets["mean_3d"], assets["opacity"], scales=assets["scale"],
                                    rotations=assets["rotation"], **kw)
    xy = ctx.xy().astype(np.float64)
    co = ctx.conic_opacity().astype(np.float64)
    A2, B2, C2, op = -0.5 * LOG2E * co[:, 0], -LOG2E * co[:, 1], -0.5 * LOG2E * co[:, 2], co[:, 3]
    with np.errstate(divide="ignore"):
        thr2 = np.where(op > 0, -np.log2(255.0 * np.maximum(op, 1e-300)) - MARGIN, np.inf)
    concave = (A2 < 0) & (C2 < 0) & (4 * A2 * C2 > B2 * B2)
    thr2 = np.where(concave | ~(op > 0), thr2, -np.inf)
    ids, ranges = ctx.sorted_ids(), ctx.ranges()
    ncon = ctx.n_contrib().astype(np.int64)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    tot = dict(entries=0, kept=0, warp_tests_f=0, warp_hits_f=0, useful_f=0, warp_tests_b=0, warp_hits_b=0, useful_b=0)
    longest = []
    for t in range(gx * gy):
        s, e = int(ranges[t][0]), int(ranges[t][1])
        n = e - s
        if n == 0:
            continue
        g = ids[s:e].astype(np.int64)
        pos = np.arange(n)  # 0-based position in the reference list; n_contrib counts positions 1-based
        tx, ty = t % gx, t // gx
        x0, y0 = tx * 16.0, ty * 16.0
        x1, y1 = min(x0 + 15, W - 1), min(y0 + 15, H - 1)
        keep = ~(region_max_p2(xy[g, 0], xy[g, 1], A2[g], B2[g], C2[g], x0, y0, x1, y1) < thr2[g])
        tot["entries"] += n
        tot["kept"] += int(keep.sum())
        g, pos = g[keep], pos[keep]
        tile_hits = 0
        for wy in range(16 // RH):   # 8x4: 8 warps per tile, 2 columns x 4 rows of pixel rects
            for wx in range(16 // RW):
                rx0, ry0 = x0 + RW * wx, y0 + RH * wy
                if rx0 >= W or ry0 >= H:
                    continue
                rx1, ry1 = min(rx0 + RW - 1, W - 1), min(ry0 + RH - 1, H - 1)
                px = np.arange(int(rx0), int(rx1) + 1)
                py = np.arange(int(ry0), int(ry1) + 1)
                nc = ncon[np.ix_(py, px)]                       # (rows, cols) contributors per pixel
                warp_n = int(nc.max())
                hit = ~(region_max_p2(xy[g, 0], xy[g, 1], A2[g], B2[g], C2[g], rx0, ry0, rx1, ry1) < thr2[g])
                # forward: the warp walks the list until every pixel is finished; a finished pixel has consumed
                # n_contrib entries and then met its stopper (or the list end): approximate the walk length by the
                # position of the last contributor of its slowest pixel plus the stopper
                live_f = pos <= warp_n                           # positions 0 .. warp_n (stopper included)
                unsat = (ctx.final_T()[np.ix_(py, px)] >= 1e-4)  # pixels that never saturate walk the whole list
                if unsat.any():
                    live_f = np.ones_like(live_f)
                live_b = pos < warp_n
                for tag, live in (("f", live_f), ("b", live_b)):
                    tot["warp_tests_" + tag] += int(live.sum())
                    h = hit & live
                    tot["warp_hits_" + tag] += int(h.sum())
                    if h.any():
                        gg, pp = g[h], pos[h]
                        dx = xy[gg, 0][:, None, None] - px[None, None, :]
                        dy = xy[gg, 1][:, None, None] - py[None, :, None]
                        p2 = A2[gg][:, None, None] * dx * dx + C2[gg][:, None, None] * dy * dy + B2[gg][:, None, None] * dx * dy
                        alpha = np.minimum(0.99, op[gg][:, None, None] * np.exp2(np.minimum(p2, 0)))
                        ok = (p2 <= 0) & (alpha >= 1.0 / 255.0) & (pp[:, None, None] < nc[None, :, :])
                        tot["useful_" + tag] += int(ok.sum())
                    if tag == "f":
                        tile_hits = max(tile_hits, int(h.sum()))
        longest.append((tile_hits, n, t))
    longest.sort(reverse=True)
    f = tot
    print(f"{a.workload} yaw {a.yaw}: P={len(radii)}, visible={(radii > 0).sum()}, {gx * gy} tiles, rect {RW}x{RH}")
    LANES = RW * RH
    print(f"  list entries (3-sigma rects)        {f['entries']:>10d}")
    print(f"  kept by the exact tile cull         {f['kept']:>10d}  ({100 * f['kept'] / f['entries']:.1f} %)")
    for tag, name, ipt in (("f", "forward", 31.0), ("b", "backward", 48.5 + 12.5)):
        wt, wh, us = f["warp_tests_" + tag], f["warp_hits_" + tag], f["useful_" + tag]
        inst = wh * ipt + wt / 32.0 * 45.0
        cyc = inst / (SMS * 4)
        print(f"  {name}: rect tests {wt:>9d}  rect hits {wh:>9d} ({100 * wh / max(wt, 1):.1f} %)  lane evaluations {LANES * wh:>10d}"
              f"  useful {us:>10d} ({100 * us / max(LANES * wh, 1):.1f} % of the lanes)")
        if LANES != 32:
            print(f"      (a {RW}x{RH} rect is {LANES} lanes: {LANES * wh / 32:.0f} warp-hit equivalents)")
            continue
        print(f"      modelled warp-instructions {inst / 1e6:6.1f} M  ->  {cyc / GHZ / 1e3:6.1f} us at one instruction per scheduler per cycle"
              f" ({SMS} SMs x 4, {GHZ} GHz); useful lane-evaluations at the same rate would need"
              f" {us / 32 * ipt / (SMS * 4) / GHZ / 1e3:5.1f} us")
    print("  heaviest quarter-tile warps (forward hits of the busiest warp, list length, tile):", longest[:5])


if __name__ == "__main__":
    main()
