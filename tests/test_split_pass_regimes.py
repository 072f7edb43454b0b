"""The split refined pass of `MergedFivePlan` (pass B, cat(scene, human_refined)) against the CPU oracle, on frames whose
tile loads are chosen so that the per-tile sort reaches every regime a split pass can reach.

A split pass sorts only its own (refined) entries of a tile, but the tile scan classes the tile by the length of the
MERGED list (own entries + the scene entries of pass A's list of the tile): warp item < 512, CTA item 512..2047,
2048-entry chunks from 2048 on.  So it sorts lists a whole pass never meets in that class -- an own list of <= 32 entries
inside a CTA item, a chunked tile whose own list is one entry or ends before its later chunks -- and split_merge_kernel
merges sequences that are both longer than the 2048 entries it stages at once.  The frame stacks splats in designated
16x16 tiles under the identity camera of the KATs (view depth = z, so equal depth bits are made by copying z):

    tile  scene  human  refined  what it reaches
    a         0      0        0  empty in both passes
    b       600     50        0  no pass-B list: both human-only views show bare background there
    c         0      0       20  refined-only tile: filtered base list empty, register rank sort
    d       700      0       20  merged >= 512 (CTA item), own <= 32 -> warp_sort_tile inside it
    e       150    100      300  warp class, own > 256 (uncached peer rows of warp_sort_tile)
    f       400      0      900  CTA radix sort of the own list
    g      2500    100        1  chunk class by merged length, own list of one entry
    h      1500      0     1200  chunk class by merged length, own list < 2048 (empty later chunks)
    i      3000    200     4500  own list in 3 chunks + merge_chunks_kernel; both merge sides > 2048
    j       800      0      800  refined z copied from scene rows: equal depth bits across the populations and runs of
                                 ties inside the refined set

The human and refined sets have the same row count; the rows a set does not use (and a few scene rows) sit behind the
camera, radius 0.  Every regime is asserted from the oracle's lists of cat(scene, refined) (CPU test), so a change to the
projection cannot silently move a tile out of its row.  GPU: the lists of both passes driven through the C ABI against
the oracle's, entry for entry; the split pass with tile culling against the whole pass and the oracle; the five renders
and three gradient sets of the frame against five oracle renders (RGB and an SH degree-3 scene); the refined gradients
around the 256-row block that straddles the detached scene prefix; and an overflowed split pass."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from parity import compare
from test_refined_pass import _close, _plan_classes
from util import kat_settings, settings_on
from util import dev  # noqa: F401
from exavatar_release_b200.plan import RENDERS, merged_bucket_layout
from exavatar_release_b200.sh import sh_to_rgb
from oracle import oracle as O

SEG, CHUNK = 512, 2048  # the sort's CTA-class boundary and chunk length (common.cuh); split_merge stages 2048 entries
F = 60.0                # focal length in pixels of the identity camera
BG_W, BG_R = (1.0, 1.0, 1.0), (0.3, 0.7, 0.2)  # scene / combined views, human-only views
SIZES = ((96, 48), (88, 40))  # 6 x 3 tiles; at 88 x 40 the last tile column and row are 8 pixels (tile j)
KEYS = ("mean_3d", "scale", "rotation", "opacity", "rgb")
# name, (tile x, tile y), scene, human, refined
TABLES = {
    "full": (("a", (1, 1), 0, 0, 0), ("b", (0, 0), 600, 50, 0), ("c", (1, 0), 0, 0, 20), ("d", (2, 0), 700, 0, 20),
             ("e", (3, 0), 150, 100, 300), ("f", (4, 0), 400, 0, 900), ("g", (0, 1), 2500, 100, 1),
             ("h", (2, 1), 1500, 0, 1200), ("i", (4, 1), 3000, 200, 4500), ("j", (5, 2), 800, 0, 800)),
    # at most 255 scene rows (the prefix ends inside the first 256-row block)
    "small": (("b", (0, 0), 100, 30, 0), ("c", (1, 0), 0, 0, 20), ("e", (3, 0), 60, 40, 150),
              ("j", (5, 2), 80, 0, 80)),
}
P_SCENE = 9657  # the "full" scene (9650 rows) and 7 rows behind the camera; not a multiple of 256


def _behind(n):
    """n rows behind the camera: culled by the near plane, radius 0."""
    return dict(mean_3d=torch.tensor([[0.0, 0.0, -1.0]]).repeat(n, 1), scale=torch.full((n, 3), 0.005),
                rotation=torch.tensor([[1.0, 0.0, 0.0, 0.0]]).repeat(n, 1), opacity=torch.full((n, 1), 0.5),
                rgb=torch.full((n, 3), 0.5))


def _populations(table, W, H, P_scene, seed=0):
    """(scene, human, refined) assets on the CPU; each population's splats of a tile in the order of the table, then the
    rows behind the camera (scene up to P_scene rows, human and refined to the same count)."""
    g = torch.Generator().manual_seed(seed)
    U = lambda *s: torch.rand(*s, generator=g)
    parts = {"scene": [], "human": [], "refined": []}
    scene_z = {}
    for name, (tx, ty), *counts in table:
        (x0, x1), (y0, y1) = (16 * tx, min(16 * tx + 16, W)), (16 * ty, min(16 * ty + 16, H))
        # the footprint radius is 3 px (tiny scales: the 0.3 px^2 low-pass dominates), so pixel centres within 3.5 px of
        # the visible part's centre keep every splat inside its tile -- 0.5 px in an 8-pixel edge tile
        jx, jy = (max(0.0, min(4.0, (b - a) / 2 - 3.5)) for a, b in ((x0, x1), (y0, y1)))
        for which, n in zip(parts, counts):
            if n == 0:
                continue
            px = (x0 + x1) / 2 + jx * (2 * U(n) - 1)
            py = (y0 + y1) / 2 + jy * (2 * U(n) - 1)
            z = 2.0 + 4.0 * U(n)
            if which == "scene":
                scene_z[name] = z
            if which == "refined" and name == "j":  # every scene depth of the first n/2 twice: ties across and within
                z = scene_z[name][torch.arange(n) // 2].clone()
            faint = n > 32  # stacks: faint, so pixels walk deep into the lists; a few splats: clearly visible
            parts[which].append(dict(
                mean_3d=torch.stack([(px - W / 2 + 0.5) * z / F, (py - H / 2 + 0.5) * z / F, z], 1),
                scale=0.004 + 0.004 * U(n, 3),
                rotation=torch.nn.functional.normalize(torch.randn(n, 4, generator=g), dim=1),
                opacity=(0.004 + 0.008 * U(n, 1)) if faint else (0.15 + 0.3 * U(n, 1)),
                rgb=U(n, 3)))
    cat = lambda ds: {k: torch.cat([d[k] for d in ds]) for k in KEYS}
    n_used = {w: sum(d["mean_3d"].shape[0] for d in ds) for w, ds in parts.items()}
    assert n_used["scene"] <= P_scene
    Ph = max(n_used["human"], n_used["refined"]) + 3
    return tuple(cat(parts[w] + [_behind(rows - n_used[w])])
                 for w, rows in (("scene", P_scene), ("human", Ph), ("refined", Ph)))


@functools.lru_cache(maxsize=None)
def _frame(table, W, H, P_scene, sh):
    """Populations, settings, gradient images and the five oracle renders of one frame (forward, backward, fragility),
    plus the oracle's per-tile lists and view depths of the two merged populations."""
    scene, human, refined = _populations(TABLES[table], W, H, P_scene)
    Ph = human["mean_3d"].shape[0]
    if sh:
        g = torch.Generator().manual_seed(5)
        scene["shs"] = 0.3 * torch.randn(P_scene, 16, 3, generator=g)
    st_w, st_r = kat_settings(W, H, F, BG_W), kat_settings(W, H, F, BG_R)
    gcol = {r: torch.randn(3, H, W, generator=torch.Generator().manual_seed(11 + j)) for j, r in enumerate(RENDERS)}
    cat = lambda x, y: {k: torch.cat((x[k], y[k])) for k in KEYS}
    sc_rgb = scene
    if sh:  # the combined renders of the oracle take the scene's SH colours precomputed
        sc_rgb = dict(scene, rgb=sh_to_rgb(3, scene["shs"].double(), scene["mean_3d"].double(),
                                           st_w.campos.double()).float())
    sets = {"scene": (sc_rgb, st_w), "human": (human, st_r), "scene_human": (cat(sc_rgb, human), st_w),
            "human_refined": (refined, st_r), "scene_human_refined": (cat(sc_rgb, refined), st_w)}
    ora, lists, dups = {}, {}, 0
    for r, (a, st) in sets.items():
        kw = dict(colors_precomp=a["rgb"])
        if sh and r == "scene":
            st, kw = st._replace(sh_degree=3), dict(shs=scene["shs"])
        oc, orad, _, oa, octx = O.forward(st, a["mean_3d"], a["opacity"], scales=a["scale"], rotations=a["rotation"], **kw)
        ora[r] = dict(color=oc, radii=orad, alpha=oa, grads=O.backward(octx, gcol[r].numpy()), frag=O.fragility(octx))
        dups = max(dups, octx.num_dups)
        if r in ("scene_human", "scene_human_refined"):
            ids, rng = octx.sorted_ids(), octx.ranges()
            lists["A" if r == "scene_human" else "B"] = dict(
                tiles=[ids[a:b].astype(np.int64) for a, b in rng], radii=orad, depth=octx.depth())
    return dict(scene=scene, human=human, refined=refined, Ps=P_scene, Ph=Ph, P=P_scene + Ph, W=W, H=H, sh=sh,
                st_w=st_w, st_r=st_r, gcol=gcol, ora=ora, lists=lists, dups=dups, table=table)


def _tile_counts(fr):
    """Per designated tile: entries of the refined rows (own), length of the merged list, human entries of pass A."""
    Ps, gx = fr["Ps"], (fr["W"] + 15) // 16
    out = {}
    for name, (tx, ty), *_ in TABLES[fr["table"]]:
        t = ty * gx + tx
        a, b = fr["lists"]["A"]["tiles"][t], fr["lists"]["B"]["tiles"][t]
        out[name] = dict(tile=t, own=int((b >= Ps).sum()), merged=int(b.size), human=int((a >= Ps).sum()),
                         base=int(a.size))
    return out


REGIMES = {
    "a": lambda c: c["merged"] == 0 and c["base"] == 0,
    "b": lambda c: c["own"] == 0 and c["merged"] > 0 and c["human"] > 0,
    "c": lambda c: 0 < c["own"] <= 32 and c["merged"] == c["own"],
    "d": lambda c: SEG <= c["merged"] < CHUNK and 0 < c["own"] <= 32,
    "e": lambda c: c["merged"] < SEG and c["own"] > 256,
    "f": lambda c: SEG <= c["merged"] < CHUNK and c["own"] > 32,
    "g": lambda c: c["merged"] >= CHUNK and c["own"] == 1,
    "h": lambda c: c["merged"] >= CHUNK and 1 < c["own"] < CHUNK,
    # own entries in 3 chunks, fewer than the merged length's chunks, and more than 2048 scene entries to merge with
    "i": lambda c: c["own"] > 2 * CHUNK and -(-c["merged"] // CHUNK) > -(-c["own"] // CHUNK)
                   and c["merged"] - c["own"] > CHUNK,
    "j": lambda c: c["merged"] >= SEG and c["own"] > 32,
}


def _assert_regimes(fr):
    counts = _tile_counts(fr)
    print("REGIMES", fr["W"], fr["H"], {k: (c["own"], c["merged"]) for k, c in counts.items()}, flush=True)
    assert set(counts) == set(REGIMES)
    for name, c in counts.items():
        assert REGIMES[name](c), (name, c)
    # tile j: equal depth bits between a refined and a scene entry, and between two refined entries
    Ps, lst = fr["Ps"], fr["lists"]["B"]["tiles"][counts["j"]["tile"]]
    d = fr["lists"]["B"]["depth"][lst].view(np.uint32)
    ref = lst >= Ps
    assert np.isin(d[ref], d[~ref]).any() and np.unique(d[ref]).size < ref.sum()


def _subsequence(a, o):
    """a is an ordered subsequence of o (ids unique within a tile list)."""
    if a.size == 0:
        return True
    srt = np.argsort(o)
    k = np.searchsorted(o, a, sorter=srt)
    if np.any(k >= o.size):
        return False
    idx = srt[k]
    return bool(np.all(o[idx] == a) and np.all(np.diff(idx) > 0))


@pytest.mark.parametrize("size", SIZES)
def test_the_frame_reaches_every_sort_regime(size):
    _assert_regimes(_frame("full", *size, P_SCENE, False))


# ------------------------------------------------------------------ GPU ------------------------------------------------

def _pass_lists(ps):
    """(ranges (tiles, 2) int64, ids int64) of a pass's workspace."""
    ctx = ps.read_ctx()
    return ctx["ranges"].astype(np.int64), ctx["ids"].astype(np.int64)


def _abi_passes(dev, fr, cap_B=None):
    """Pass A (b2r_forward_project + b2r_forward_bin) and the split pass B (b2r_forward_project_split +
    b2r_forward_bin_split on pass A's workspace), in the order MergedFivePlan._start_pass enqueues them, without tile
    culling.  Radii and duplicate ids start as sentinels, so a row or slot nobody writes shows up."""
    from exavatar_release_b200 import _lib as L
    from exavatar_release_b200.plan import _Pass
    from exavatar_release_b200.rasterizer import GaussianRasterizationSettings, _make_scene
    lib = L.load()
    Ps, P, W, H = fr["Ps"], fr["P"], fr["W"], fr["H"]
    st = settings_on(fr["st_w"], dev, GaussianRasterizationSettings)
    cap = 2 * fr["dups"] + 4096
    passes = {"A": _Pass(P, W, H, cap, 1, dev), "B": _Pass(P, W, H, cap_B or cap, 1, dev, split=True)}
    s = torch.cuda.current_stream(dev).cuda_stream
    keep = []
    for pk, rows in (("A", fr["human"]), ("B", fr["refined"])):
        ps = passes[pk]
        ps.radii.fill_(-7)
        ps.ids.fill_(-1)
        a = {k: torch.cat((fr["scene"][k], rows[k])).to(dev).contiguous() for k in KEYS}
        sc, kp = _make_scene(st, a["mean_3d"], None, a["rgb"], a["opacity"], a["scale"], a["rotation"], None,
                             L.B2R_FLAG_NO_TILE_CULL)
        keep.append((a, kp, sc))
        if pk == "A":
            L.check(lib.b2r_forward_project(C.byref(sc), C.byref(ps.ws), ps.radii.data_ptr(), s), "project")
            L.check(lib.b2r_forward_bin(C.byref(sc), C.byref(ps.ws), s), "bin")
        else:
            L.check(lib.b2r_forward_project_split(C.byref(sc), C.byref(ps.ws), Ps, ps.radii.data_ptr(), s),
                    "project_split")
            L.check(lib.b2r_forward_bin_split(C.byref(sc), C.byref(ps.ws), C.byref(passes["A"].ws), Ps,
                                              ps.radii.data_ptr(), s), "bin_split")
    torch.cuda.synchronize()
    return passes


def _run_plan(dev, cls, fr, gcol, densify=False):
    """One MergedFivePlan frame (default flags: tile culling on); `densify`: the scene's densification statistics go to
    the tail of the flat gradient buffer."""
    from exavatar_release_b200 import rasterizer as rz
    to = lambda d: {k: d[k].to(dev) for k in KEYS}
    cap = 2 * fr["dups"] + 4096
    plan = cls(fr["Ps"], fr["Ph"], fr["W"], fr["H"], {"A": cap, "B": cap}, dev, sh_coeffs=16 if fr["sh"] else 0)
    sc = to(fr["scene"])
    if fr["sh"]:
        sc = dict({k: v for k, v in sc.items() if k != "rgb"}, shs=fr["scene"]["shs"].to(dev), sh_degree=3)
    plan.set_scene(sc)
    st_w, st_r = (settings_on(s, dev, rz.GaussianRasterizationSettings) for s in (fr["st_w"], fr["st_r"]))
    plan.frame(0, st_w, st_r, sc, to(fr["human"]), to(fr["refined"]), {r: g.to(dev) for r, g in gcol.items()},
               accumulate=False, densify=plan.stats() if densify else None)
    torch.cuda.synchronize()
    assert not plan.overflowed()
    return plan


def _compare_frame(case, plan, fr):
    """The five renders (colour, alpha, radii) and the three gradient sets against the oracle (`parity.compare`, its
    bounds); returns the expected gradients of each set."""
    ora, Ps, Ph = fr["ora"], fr["Ps"], fr["Ph"]
    for r in RENDERS:
        pm, _ = ora[r]["frag"]
        img, alpha, radii = plan.render_outputs(r)
        assert np.array_equal(radii.cpu().numpy(), ora[r]["radii"]), r
        compare(case + r, "color", img.cpu().numpy(), ora[r]["color"], pm[None], kind="image")
        compare(case + r, "alpha", alpha.cpu().numpy(), ora[r]["alpha"], pm[None], kind="image")
    common = ("means3D", "means2D", "opacities", "scales", "rotations")
    expected = {}
    for label, Pn, parts, names in (
            ("scene", Ps, [("scene", slice(0, Ps))], common + (("shs",) if fr["sh"] else ("colors",))),
            ("human", Ph, [("human", slice(0, Ph)), ("scene_human", slice(Ps, Ps + Ph))], common + ("colors",)),
            ("human_refined", Ph, [("human_refined", slice(0, Ph)), ("scene_human_refined", slice(Ps, Ps + Ph))],
             common + ("colors",))):
        y, flag = {}, None
        for r, rows in parts:
            g, (_, gm) = ora[r]["grads"], ora[r]["frag"]
            for k in names:
                v = g[k][rows].reshape(g[k][rows].shape[0], -1)
                y[k] = v if k not in y else y[k] + v
            flag = gm[rows] if flag is None else (flag | gm[rows])
        views = plan.grads(label)
        for k in names:
            compare(case + label, "d_" + k, views[k].cpu().numpy().reshape(Pn, -1), y[k], flag[:, None], kind="grad")
        expected[label] = (y, flag)
    return expected


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
def test_split_lists_equal_the_oracle_in_every_sort_regime(dev, size):
    """Both passes through the C ABI without tile culling: pass B's list of every tile its refined rows reach equals the
    oracle's list of cat(scene, refined) entry for entry, every other tile has no list (and the oracle's list there no
    refined entry); pass A's lists, both passes' radii and pass B's duplicate count equal the oracle's."""
    fr = _frame("full", *size, P_SCENE, False)
    _assert_regimes(fr)
    Ps, P, W, H = fr["Ps"], fr["P"], fr["W"], fr["H"]
    passes = _abi_passes(dev, fr)
    for pk in "AB":
        st = passes[pk].status()
        assert st["overflow"] == 0, pk
        assert np.array_equal(passes[pk].radii.cpu().numpy(), fr["lists"][pk]["radii"]), pk
    ranges, ids = _pass_lists(passes["A"])
    for t, o in enumerate(fr["lists"]["A"]["tiles"]):
        assert np.array_equal(ids[ranges[t, 0]:ranges[t, 1]], o), f"pass A, tile {t}"
    ranges, ids = _pass_lists(passes["B"])
    reached = 0
    for t, o in enumerate(fr["lists"]["B"]["tiles"]):
        got = ids[ranges[t, 0]:ranges[t, 1]]
        if got.size:
            assert np.array_equal(got, o), f"pass B, tile {t}"
            reached += o.size
        else:
            assert not np.any(o >= Ps), f"pass B, tile {t}: refined entries but no list"
    assert passes["B"].status()["num_dups"] == reached


@pytest.mark.gpu
@pytest.mark.parametrize("size,mode", [((96, 48), "rgb"), ((88, 40), "sh")])
def test_split_frame_equals_the_whole_pass_and_five_oracle_renders(dev, size, mode):
    """MergedFivePlan with tile culling, split and whole pass B: pass B's lists bit-equal between the two where the split
    pass builds one, both ordered subsequences of the oracle's lists; then the split frame's five renders and three
    gradient sets against five oracle renders."""
    fr = _frame("full", *size, P_SCENE, mode == "sh")
    Ps, P, W, H = fr["Ps"], fr["P"], fr["W"], fr["H"]
    Split, Full = _plan_classes()
    lists = {}
    for cls in (Full, Split):
        plan = _run_plan(dev, cls, fr, fr["gcol"])
        ranges, ids = _pass_lists(plan.passes["B"])
        lists[cls.SPLIT] = [ids[a:b] for a, b in ranges]
    n_lists = 0
    for t, o in enumerate(fr["lists"]["B"]["tiles"]):
        a, b = lists[True][t], lists[False][t]
        if a.size:
            assert np.array_equal(a, b), f"tile {t}"
            n_lists += 1
        else:
            assert not np.any(b >= Ps), f"tile {t}"
        assert _subsequence(a, o) and _subsequence(b, o), f"tile {t}: not an ordered subsequence of the oracle's list"
    assert n_lists >= 8
    _compare_frame(f"split/{W}x{H}/{mode}/", plan, fr)


@pytest.mark.gpu
@pytest.mark.parametrize("pad", ["256k", "256k+1", "255"])
def test_refined_gradients_around_the_detached_prefix_block(dev, pad):
    """The backward projection of pass B skips the 256-row blocks wholly inside the detached scene prefix.  With the
    prefix padded to 256 k, 256 k + 1 and 255 rows: the frame against the oracle, the refined rows of the block that
    straddles the prefix's end on their own, and every region of the flat gradient buffer outside pass B's rows
    bit-equal to a run with the whole pass B.  For that last comparison the image gradients of pass A's views are zero:
    the backward composites add with float atomics in no fixed order, so pass A's gradients of two runs may differ in
    the last bits, while zeros (and the visibility counts of the densification statistics) do not."""
    table, P_scene = {"256k": ("full", 256 * 38), "256k+1": ("full", 256 * 38 + 1), "255": ("small", 255)}[pad]
    fr = _frame(table, 96, 48, P_scene, False)
    Ps, Ph = fr["Ps"], fr["Ph"]
    Split, Full = _plan_classes()
    plan = _run_plan(dev, Split, fr, fr["gcol"])
    expected = _compare_frame(f"split/prefix{pad}/", plan, fr)
    if Ps % 256:  # refined rows [0, n) share a block with the last scene rows
        n = min(Ph, 256 - Ps % 256)
        y_all, flag = expected["human_refined"]
        got = plan.grads("human_refined")
        for k, y in y_all.items():
            x = got[k].cpu().numpy().reshape(Ph, -1)
            ninf = float(np.abs(y).max())
            err = float(np.abs(x[:n] - y[:n]).max())
            assert err <= 5e-3 * ninf, (k, err, ninf)  # parity.compare's bound for any element, no count allowance
        oy = y_all["opacities"][:n][~flag[:n]]
        assert oy.size and float(np.abs(oy).max()) > 0.02 * float(np.abs(y_all["opacities"]).max())
    zero_a = {r: (torch.zeros_like(g) if r in ("scene", "human", "scene_human") else g) for r, g in fr["gcol"].items()}
    flats = {cls.SPLIT: _run_plan(dev, cls, fr, zero_a, densify=True).flat_bucket().clone() for cls in (Full, Split)}
    lay = merged_bucket_layout(Ps, Ph, 0)
    for region in ("A", "A_shs", "stats"):
        o, n = lay[region]
        assert torch.equal(flats[True][o:o + n], flats[False][o:o + n]), region
    o, n = lay["stats"]
    assert float(flats[True][o:o + n].abs().sum()) > 0  # the visibility counts of the scene rows
    o, n = lay["B"]
    assert float(flats[True][o:o + n].abs().max()) > 0
    _close(flats[True][o:o + n], flats[False][o:o + n], "B")


@pytest.mark.gpu
def test_an_overflowed_split_pass_keeps_every_list_entry_a_valid_id(dev):
    """Pass B with a duplicate capacity between its own entry count and its merged count: the status block reports the
    overflow and the required count, and every entry inside pass B's ranges is an id in [0, P) (the fallback of
    split_merge_kernel).  Buffers are only read back; nothing is composited from the overflowed pass."""
    fr = _frame("full", 96, 48, P_SCENE, False)
    Ps, P, W, H = fr["Ps"], fr["P"], fr["W"], fr["H"]
    lists = fr["lists"]["B"]["tiles"]
    own = sum(int((o >= Ps).sum()) for o in lists)
    merged = sum(o.size for o in lists if np.any(o >= Ps))
    cap = (own + merged) // 2
    assert own < cap < merged
    passes = _abi_passes(dev, fr, cap_B=cap)
    st = passes["B"].status()
    assert st["overflow"] == 1 and st["num_dups"] == merged
    assert not passes["A"].status()["overflow"]
    ranges, ids = _pass_lists(passes["B"])
    assert ranges.min() >= 0 and ranges.max() <= cap and int((ranges[:, 1] - ranges[:, 0]).sum()) == cap
    for t, (a, b) in enumerate(ranges):
        got = ids[a:b]
        assert np.all((got >= 0) & (got < P)), f"tile {t}"
