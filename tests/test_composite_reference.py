"""The float64 composite of tests/composite_reference.py anchored without a device: its backward rows against torch
float64 autograd of a dense restatement of its forward, and its forward and rows against the fp64 oracle."""
import numpy as np
import pytest
import torch

import composite_reference as R
from util import workload_settings
from exavatar_release_b200.synthetic import make_assets, make_grad_image
from oracle import oracle as O

LOG2E = 1.0 / R.LN2


def _rec(x, y, a, b, c, o, z, rgb):
    """A record from a conic (a, b, c) in the oracle's units (power = -a dx^2 / 2 - b dx dy - c dy^2 / 2)."""
    return [x, y, -0.5 * LOG2E * a, -LOG2E * b, -0.5 * LOG2E * c, o, z, np.inf, *rgb, 0.0]


def _hand_lists():
    """One 16x16 tile and a hand-built list: a 0.99-clamped splat, a splat whose alpha is exactly 1/255 at its pixel,
    a stack of opaque splats that stops pixel (3, 3) without applying the last one, broad and anisotropic splats, and
    ids that interleave two id ranges (for a view)."""
    g = np.random.default_rng(3)
    recs = [
        _rec(3.0, 3.0, 0.5, 0.0, 0.5, 1.0, 1.0, (0.9, 0.2, 0.1)),       # 0: clamped to 0.99 at (3, 3)
        _rec(12.0, 4.0, 2.0, 0.0, 2.0, R.ALPHA_MIN, 1.1, (0.1, 0.8, 0.3)),  # 1: alpha exactly 1/255 at (12, 4)
        _rec(3.0, 3.0, 0.4, 0.1, 0.6, 0.6, 1.2, (0.3, 0.3, 0.9)),       # 2..4: with 0, stop (3, 3) at entry 4
        _rec(3.2, 2.9, 0.3, -0.05, 0.5, 0.97, 1.3, (0.5, 0.1, 0.4)),
        _rec(2.9, 3.1, 0.5, 0.0, 0.5, 0.99, 1.4, (0.2, 0.7, 0.6)),
    ]
    for k in range(11):                                                 # 5..15: random, broad and small
        a, c = g.uniform(0.02, 1.2, 2)
        b = g.uniform(-0.4, 0.4) * np.sqrt(a * c)
        recs.append(_rec(*g.uniform(-2, 18, 2), a, b, c, g.uniform(0.05, 0.9), 1.5 + 0.1 * k, g.uniform(-0.2, 1.0, 3)))
    geom = np.array(recs, np.float64)
    P = len(geom)
    ids = np.argsort(geom[:, 6], kind="stable").astype(np.uint32)  # depth order
    ranges = np.array([[0, P]], np.int64)
    return geom, ranges, ids


def _dense(geom, ranges, ids, W, H, bg, applied_pos, gcol, gd, ga, view):
    """Loss sum g . colour + g_d depth + g_a alpha restated densely in torch float64 over (pixels, in-view entries), the
    applied set a constant, the 0.99 clamp straight-through; returns autograd's d loss / d record (P, 12)."""
    G = torch.tensor(geom, dtype=torch.float64, requires_grad=True)
    lst = np.asarray(ids[ranges[0, 0]:ranges[0, 1]], np.int64)
    lo, hi = view.id_begin, view.id_end if view.id_end is not None else len(geom)
    keep = (lst >= lo) & (lst < hi)
    gid = torch.as_tensor(lst[keep])
    xs, ys, pix = R.tile_pixels(0, W, H)
    r = G[gid]
    dx = r[None, :, 0] - torch.as_tensor(xs, dtype=torch.float64)[:, None]
    dy = r[None, :, 1] - torch.as_tensor(ys, dtype=torch.float64)[:, None]
    p2 = r[:, 2] * dx * dx + r[:, 4] * dy * dy + r[:, 3] * dx * dy
    araw = r[:, 5] * torch.exp2(p2)
    alpha = araw + (torch.clamp(araw, max=R.ALPHA_MAX) - araw).detach()
    app = torch.as_tensor(applied_pos[:, keep])
    om = torch.where(app, 1 - alpha, torch.ones_like(alpha))
    T = torch.cat([torch.ones(len(pix), 1, dtype=torch.float64), torch.cumprod(om, 1)[:, :-1]], 1)
    w = torch.where(app, alpha * T, torch.zeros_like(alpha))
    Tf = torch.prod(om, 1)
    bgv = torch.tensor(view.bg if view.bg is not None else bg, dtype=torch.float64)
    col = w @ r[:, 8:11] + Tf[:, None] * bgv[None, :]
    gc = torch.as_tensor(gcol.reshape(3, -1)[:, pix].T)
    loss = (col * gc).sum()
    if gd is not None:
        loss = loss + ((w @ r[:, 6]) * torch.as_tensor(gd.reshape(-1)[pix])).sum()
    if ga is not None:
        loss = loss + (w.sum(1) * torch.as_tensor(ga.reshape(-1)[pix])).sum()
    loss.backward()
    return G.grad.numpy()


@pytest.mark.parametrize("grads", ["color", "depth", "alpha", "both"])
@pytest.mark.parametrize("view", ["all", "range"])
def test_backward_rows_equal_autograd_of_a_dense_restatement(grads, view):
    W = H = 16
    bg = (0.3, 0.6, 0.2)
    geom, ranges, ids = _hand_lists()
    v = R.View() if view == "all" else R.View(id_begin=2, id_end=11, bg=(0.7, 0.1, 0.5))
    f = R.forward(geom, ranges, ids, W, H, bg, v)
    # the list reaches what the test is about
    t = R._Tile(geom, ranges, ids, 0, W, H, v)
    pix33 = 3 * W + 3
    if view == "all":
        assert t.araw[pix33, list(t.gid).index(0)] > R.ALPHA_MAX                      # clamped
        assert t.araw[4 * W + 12, list(t.gid).index(1)] == R.ALPHA_MIN              # exactly at 1/255, accepted
        assert f["stop"].reshape(-1)[pix33] == 4 and f["n_contrib"].reshape(-1)[pix33] == 4  # stopped, not applied
    else:
        assert f["stop"].reshape(-1)[pix33] == -1 and set(t.gid) == set(range(2, 11))
    applied = t.ok & (t.pos[None, :] < f["n_contrib"].reshape(-1)[t.pix][:, None])
    full = np.zeros((len(t.pix), ranges[0, 1]), bool)
    full[:, t.pos] = applied
    g = np.random.default_rng(7)
    gcol = g.standard_normal((3, H, W))
    gd = g.standard_normal((H, W)) if grads in ("depth", "both") else None
    ga = g.standard_normal((H, W)) if grads in ("alpha", "both") else None
    rows, S, _ = R.backward(geom, ranges, ids, W, H, bg, f["n_contrib"], gcol, gd, ga, v)
    d = _dense(geom, ranges, ids, W, H, bg, full, gcol, gd, ga, v)
    want = np.concatenate([d[:, :5] / R.LN2, d[:, 5:7], np.zeros((len(d), 1)), d[:, 8:11], np.zeros((len(d), 1))], 1)
    assert np.all(S >= np.abs(rows) - 1e-15)
    np.testing.assert_allclose(rows, want, rtol=1e-11, atol=1e-13 * np.abs(want).max())
    if view == "range":
        assert not rows[[0, 1, 11, 12, 13, 14, 15]].any()
    if gd is None:
        assert not rows[:, 6].any()


@pytest.fixture(scope="module")
def t1_f64():
    """The fp64 oracle's T1 frame: its geometry as records, its lists, its forward and its backward."""
    assets = make_assets("T1", seed=0)
    st = workload_settings("T1", yaw=12.0, bg=(0.2, 0.5, 0.9))
    W, H = int(st.image_width), int(st.image_height)
    oc, _, od, oa, ctx = O.forward(st, assets["mean_3d"], assets["opacity"], colors_precomp=assets["rgb"],
                                   scales=assets["scale"], rotations=assets["rotation"], variant="f64")
    co = ctx.conic_opacity()
    geom = np.zeros((ctx.P, 12))
    geom[:, :2] = ctx.xy()
    geom[:, 2], geom[:, 3], geom[:, 4] = -0.5 * LOG2E * co[:, 0], -LOG2E * co[:, 1], -0.5 * LOG2E * co[:, 2]
    geom[:, 5], geom[:, 6], geom[:, 8:11] = co[:, 3], ctx.depth(), ctx.rgb()
    gi = make_grad_image("T1", 0).numpy().astype(np.float64)
    g = np.random.default_rng(1)
    gd, ga = g.standard_normal((H, W)), g.standard_normal((H, W))
    ob = O.backward(ctx, gi, gd, ga)
    bg = tuple(np.float32([0.2, 0.5, 0.9]).astype(np.float64))  # the settings hold it in float32
    return dict(W=W, H=H, bg=bg, geom=geom, ids=ctx.sorted_ids(), ranges=ctx.ranges(), color=oc,
                depth=od[0], alpha=oa[0], final_T=ctx.final_T(), n_contrib=ctx.n_contrib(), grads=ob, gi=gi, gd=gd,
                ga=ga)


def test_forward_equals_the_fp64_oracle(t1_f64):
    o = t1_f64
    f = R.forward(o["geom"], o["ranges"], o["ids"], o["W"], o["H"], o["bg"])
    assert f["written"].all() and (f["n_contrib"] > 0).mean() > 0.5 and (f["stop"] >= 0).any()
    assert np.array_equal(f["n_contrib"], o["n_contrib"])
    for k in ("color", "depth", "alpha", "final_T"):
        np.testing.assert_allclose(f[k], o[k], rtol=0, atol=1e-12 * np.abs(o[k]).max(), err_msg=k)
        assert np.all(f["S_" + ("T" if k == "final_T" else k)] >= np.abs(f[k]) * (1 - 1e-12)), k


def test_rows_equal_the_fp64_oracle_through_the_projection_scale_factors(t1_f64):
    o = t1_f64
    W, H = o["W"], o["H"]
    rows, S, _ = R.backward(o["geom"], o["ranges"], o["ids"], W, H, o["bg"], o["n_contrib"], o["gi"], o["gd"], o["ga"])
    got = {"means2D": np.stack([0.5 * W * R.LN2 * rows[:, 0], 0.5 * H * R.LN2 * rows[:, 1]], 1),
           "colors": rows[:, 8:11], "opacities": rows[:, 5:6]}
    for k, x in got.items():
        y = o["grads"][k][:, :x.shape[1]]
        assert np.abs(y).max() > 0
        np.testing.assert_allclose(x, y, rtol=0, atol=1e-9 * np.abs(y).max(), err_msg=k)
    assert np.all(S >= np.abs(rows) * (1 - 1e-12))
