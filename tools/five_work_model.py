"""Work model of the C4 training frame's five composite views, computed on the CPU from the oracle's lists (analysis
script, not a test).

  python tools/five_work_model.py [--yaw -6]

A merged training frame renders two passes, each from one set of tile lists: pass A = cat(scene, human) with the views
scene, human (random background) and scene + human; pass B = cat(scene, refined) with the views refined human and
scene + refined human.  Every view walks its pass's lists and culls the entries outside its own index range.  For
every view this counts, per 8x8 quarter tile and per 8x4 warp rect, by the kernels' own culling rules
(tests/work_model.py's `region_max_p2` restatement):

  entries walked      list entries a quarter tile walks (to the list end unless all its 64 pixels saturate)
  own entries         ... of them inside the view's index range
  cull chunks         32-entry cull tests per warp
  fwd hits            own entries whose warp rect the splat can reach with alpha >= 1/255 (trips of the forward hit loop)
  bwd hits            ... up to the warp's last contributor (the backward replays no entry behind it)

and turns them into modelled warp-instructions at the kernels' per-hit costs (DESIGN.md section 3.3): the forward's 31
per hit and the backward's itemised per-hit budget, before and after the phase-B record change, plus 45 per cull chunk.
Views that skip human-free tiles (everything but the scene view) skip them here too.
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from util import workload_settings  # noqa: E402
from work_model import LOG2E, MARGIN, SMS, GHZ, region_max_p2  # noqa: E402
from exavatar_release_b200.synthetic import WORKLOADS, make_population_assets  # noqa: E402
from oracle import oracle as O  # noqa: E402

FWD_PER_HIT = 31.0
CULL_PER_CHUNK = 45.0
# backward per warp hit, from the SASS of composite_bwd4_kernel<false> (DESIGN.md section 3.3): phase A replay per splat
# (one group / its size, with the group loop's tail), phase B per queued splat (one 16-splat drain / 16).  Before: 4-splat
# groups and a phase-B copy of each record; now: 2-splat groups, phase B reads the record from the survivor queue.  The
# smaller groups issue more per hit but run faster (DESIGN.md section 3.3): issue is not what bounds this loop.
BWD_PER_HIT = {"before": 165 / 4 + 5 / 4 + 217 / 16, "now": 78 / 2 + 5 / 2 + 221 / 16}


def _forward(a, st):
    return O.forward(st, a["mean_3d"], a["opacity"], colors_precomp=a["rgb"], scales=a["scale"],
                     rotations=a["rotation"])[4]


def count_pass(W, H, cat_ctx, views, skip_below):
    """views: name -> (oracle ctx of the view's own render, lo, hi, skips tiles without an index >= skip_below).
    Returns name -> totals."""
    xy = cat_ctx.xy().astype(np.float64)
    co = cat_ctx.conic_opacity().astype(np.float64)
    A2, B2, C2, op = -0.5 * LOG2E * co[:, 0], -LOG2E * co[:, 1], -0.5 * LOG2E * co[:, 2], co[:, 3]
    with np.errstate(divide="ignore"):
        thr2 = np.where(op > 0, -np.log2(255.0 * np.maximum(op, 1e-300)) - MARGIN, np.inf)
    concave = (A2 < 0) & (C2 < 0) & (4 * A2 * C2 > B2 * B2)
    thr2 = np.where(concave | ~(op > 0), thr2, -np.inf)
    ids, ranges = cat_ctx.sorted_ids(), cat_ctx.ranges()
    gx, gy = (W + 15) // 16, (H + 15) // 16
    # a view rendered on its own numbers its Gaussians from 0: offset them to the pass's index range
    per_view = {v: (c.final_T(), c.n_contrib().astype(np.int64), c.sorted_ids().astype(np.int64) + lo, c.ranges())
                for v, (c, lo, _, _) in views.items()}
    tot = {v: dict(quarters=0, walked=0, own=0, chunks=0, fwd_hits=0, bwd_hits=0) for v in views}
    for t in range(gx * gy):
        s, e = int(ranges[t][0]), int(ranges[t][1])
        if e == s:
            continue
        g = ids[s:e].astype(np.int64)
        x0, y0 = (t % gx) * 16, (t // gx) * 16
        keep = ~(region_max_p2(xy[g, 0], xy[g, 1], A2[g], B2[g], C2[g], x0, y0, min(x0 + 15, W - 1),
                               min(y0 + 15, H - 1)) < thr2[g])
        g = g[keep]
        n = len(g)
        has_h = bool((g >= skip_below).any())
        for v, (_, lo, hi, skip) in views.items():
            if skip and not has_h:
                continue
            fT, nc, vids, vranges = per_view[v]
            own = (g >= lo) & (g < hi)
            ownpos = np.nonzero(own)[0]  # positions in the pass's list of the view's own entries
            vbase = int(vranges[t][0])

            def last_pos(m):
                # n_contrib counts the view's own render list (1-based, before the tile cull): find its m-th entry,
                # a contributor and so a survivor of the cull, in the pass's list; 0-based index into ownpos
                return int(np.searchsorted(ownpos, int(np.nonzero(g == vids[vbase + m - 1])[0][0])))

            for q in range(4):
                qx, qy = x0 + (q & 1) * 8, y0 + (q >> 1) * 8
                if qx >= W or qy >= H:
                    continue
                py, px = np.arange(qy, min(qy + 8, H)), np.arange(qx, min(qx + 8, W))
                if (fT[np.ix_(py, px)] < 1e-4).all():  # every pixel saturates: the walk ends at the slowest stopper
                    m = int(nc[np.ix_(py, px)].max())
                    k = last_pos(m) + 1 if m > 0 else 0  # the stopper: the next own entry
                    walk = int(ownpos[k]) + 1 if k < len(ownpos) else n
                else:
                    walk = n
                T = tot[v]
                T["quarters"] += 1
                T["walked"] += walk
                T["own"] += int(own[:walk].sum())
                for wv in range(2):
                    ry0 = qy + 4 * wv
                    if ry0 >= H:
                        continue
                    rows = np.arange(ry0, min(ry0 + 4, H))
                    # the view's n_contrib counts its own entries (1-based): map the warp's last contributor to a
                    # position of the pass's list
                    m = int(nc[np.ix_(rows, px)].max())
                    last = int(ownpos[last_pos(m)]) + 1 if m > 0 else 0
                    T["chunks"] += -(-walk // 32)
                    sel = np.nonzero(own[:walk])[0]
                    gg = g[sel]
                    hit = ~(region_max_p2(xy[gg, 0], xy[gg, 1], A2[gg], B2[gg], C2[gg], qx, ry0, min(qx + 7, W - 1),
                                          min(ry0 + 3, H - 1)) < thr2[gg])
                    T["fwd_hits"] += int(hit.sum())
                    T["bwd_hits"] += int((hit & (sel < last)).sum())
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--yaw", type=float, default=-6.0)
    a = ap.parse_args()
    O.set_num_threads(os.cpu_count() or 1)
    wl = WORKLOADS["C4"]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets("C4", seed=0)
    Ps = scene["mean_3d"].shape[0]
    st_w = workload_settings("C4", yaw=a.yaw)
    st_r = workload_settings("C4", yaw=a.yaw, bg=(0.3, 0.7, 0.2))
    c_scene = _forward(scene, st_w)
    passes = []
    for tag, hum in (("A", human), ("B", refined)):
        Ph = hum["mean_3d"].shape[0]
        c_cat = _forward({k: torch.cat((scene[k], hum[k])) for k in scene}, st_w)
        c_hum = _forward(hum, st_r)
        views = {}
        if tag == "A":
            views["scene"] = (c_scene, 0, Ps, False)
        views["human (rand bg)"] = (c_hum, Ps, Ps + Ph, True)
        views["scene + human"] = (c_cat, 0, Ps + Ph, True)
        passes.append((tag, count_pass(W, H, c_cat, views, Ps)))

    rate = SMS * 4 * GHZ * 1e3  # warp-instructions per microsecond at one per scheduler per cycle
    print(f"C4 yaw {a.yaw}: {W}x{H}; backward warp-instructions per hit: "
          + ", ".join(f"{k} {v:.2f}" for k, v in BWD_PER_HIT.items()) + f"; forward {FWD_PER_HIT:.0f}; "
          f"{CULL_PER_CHUNK:.0f} per cull chunk; {SMS} SMs x 4 schedulers at {GHZ} GHz")
    hdr = (f"{'pass':4s} {'view':16s} {'quarters':>8s} {'walked':>9s} {'own':>9s} {'chunks':>8s} {'fwd hits':>9s} "
           f"{'bwd hits':>9s} {'fwd M':>7s} " + " ".join(f"{'bwd M ' + k:>15s}" for k in BWD_PER_HIT))
    print(hdr)
    frame = {"fwd": 0.0, **{k: 0.0 for k in BWD_PER_HIT}}
    for tag, tot in passes:
        for v, T in tot.items():
            cull = T["chunks"] * CULL_PER_CHUNK
            fwd = T["fwd_hits"] * FWD_PER_HIT + cull
            bwd = {k: T["bwd_hits"] * c + cull for k, c in BWD_PER_HIT.items()}
            frame["fwd"] += fwd
            for k in bwd:
                frame[k] += bwd[k]
            print(f"{tag:4s} {v:16s} {T['quarters']:8d} {T['walked'] / 1e6:8.2f}M {T['own'] / 1e6:8.2f}M "
                  f"{T['chunks'] / 1e6:7.3f}M {T['fwd_hits'] / 1e6:8.2f}M {T['bwd_hits'] / 1e6:8.2f}M {fwd / 1e6:7.1f} "
                  + " ".join(f"{bwd[k] / 1e6:15.1f}" for k in BWD_PER_HIT))
    print(f"frame: forward {frame['fwd'] / 1e6:.1f} M warp-instructions ({frame['fwd'] / rate:.0f} us); backward "
          + ", ".join(f"{k} {frame[k] / 1e6:.1f} M ({frame[k] / rate:.0f} us)" for k in BWD_PER_HIT)
          + f"; modelled saving {(frame['before'] - frame['now']) / 1e6:.1f} M warp-instructions "
          f"({(frame['before'] - frame['now']) / rate:.0f} us) per frame (not measured)")


if __name__ == "__main__":
    main()
