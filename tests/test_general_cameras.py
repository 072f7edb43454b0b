"""The projection path under general cameras: pitch and roll, fx != fy, the frustum-clamp band and the near plane.

The other parity tests render through yaw-only cameras (`look_at_cam_param`) or the identity camera of the KATs, with
fx == fy.  A yaw-only view matrix has structural zeros (R01, R10, R12, R21 and t_y), so a kernel that read a transposed
view-matrix or R^-1 entry, or fx where it needs fy, would still pass them; and their scenes never reach the frustum-clamp
band (|x/z| > 1.3 tan(fov/2)), the near plane, or rects of more than 32 tiles at small image sizes.  The cameras here
have |R_ij| > 0.05 everywhere and |R_ij| != |R_ji|, t with three non-zero components, fx/fy = 1.35 or 0.75, an
off-centre principal point (ignored, camera.py), and odd image sizes; the populations are placed in camera space:

    clamp    spread to +-2 tan(fov/2): many visible Gaussians take the clamped Jacobian
    near     view depth in (0.2, 0.35], plus points whose fp32 view depth is exactly 0.2f or the next float above
    huge     footprints covering the whole tile grid, rects of more than 32 tiles
    awkward  un-normalised quaternions (norm 0.3 .. 3), one scale axis 1e-4 of the others
    plain    an ordinary mix

"near" and "huge" render on their own: their gradients are orders of magnitude larger than the others', and the
norm-relative bound of `parity.compare` would otherwise let them hide errors elsewhere.

CPU tier: the oracle's f64 build against `oracle/dense_autograd.py` (an independent fp64 autograd restatement) and its
f32 build against its f64 build on these inputs, so the reference the GPU tests lean on is pinned where they lean on it.
GPU tier: FramePlan (C ABI), the public `GaussianRasterizer` (both host routes), the stage buffers, `markVisible`, the
merged training frame (RGB and SH scene), skinning, and one 512x512 frame, each against the oracle.
"""
import math
import zlib

import numpy as np
import pytest
import torch

from parity import compare, contributor_report, last_contributor
from util import settings_on
from util import dev  # noqa: F401
from exavatar_release_b200.renderer import lbs_reference, render_settings
from exavatar_release_b200.sh import sh_to_rgb
from oracle import dense_autograd as DA
from oracle import oracle as O

BG = (0.2, 0.6, 0.9)
T_CAM = (0.13, -0.21, 0.37)
NEAR = np.float32(0.2)
# name: (W, H, pitch, yaw, roll, fx, fy)
CAMERAS = {
    "c13x40": (13, 40, 28.0, -24.0, -49.0, 27.0, 20.0),         # narrower than one tile; fx/fy = 1.35
    "c61x45": (61, 45, 25.0, -15.0, 35.0, 70.0, 52.0),          # fx/fy = 1.35
    "c29x37": (29, 37, -40.0, 30.0, 120.0, 30.0, 41.0),         # fx/fy = 0.73
    "c203x131": (203, 131, -22.0, 38.0, -63.0, 150.0, 200.0),   # fx/fy = 0.75
    "c512": (512, 512, 19.0, -31.0, 47.0, 760.0, 563.0),        # fx/fy = 1.35
}
SMALL = ("c13x40", "c61x45", "c29x37")
POPS = ("clamp", "near", "huge", "awkward", "plain")


def _rot(pitch, yaw, roll):
    p, y, r = (math.radians(a) for a in (pitch, yaw, roll))
    Rx = np.array([[1, 0, 0], [0, math.cos(p), -math.sin(p)], [0, math.sin(p), math.cos(p)]])
    Ry = np.array([[math.cos(y), 0, math.sin(y)], [0, 1, 0], [-math.sin(y), 0, math.cos(y)]])
    Rz = np.array([[math.cos(r), -math.sin(r), 0], [math.sin(r), math.cos(r), 0], [0, 0, 1]])
    return Rx @ Ry @ Rz


def camera(name, device="cpu"):
    """cam_param dict of a general camera; R = Rx(pitch) Ry(yaw) Rz(roll), principal point off-centre."""
    W, H, pitch, yaw, roll, fx, fy = CAMERAS[name]
    R = torch.tensor(_rot(pitch, yaw, roll), dtype=torch.float32)
    A = R.abs()
    off = ~torch.eye(3, dtype=torch.bool)
    # every entry non-zero and no entry equal in magnitude to its transpose: an index transposition changes the output
    assert float(A.min()) > 0.05 and float((A - A.t()).abs()[off].min()) > 0.04, name
    cam = {"R": R, "t": torch.tensor(T_CAM), "focal": torch.tensor([fx, fy], dtype=torch.float32),
           "princpt": torch.tensor([0.37 * W, 0.61 * H], dtype=torch.float32)}
    return {k: v.to(device) for k, v in cam.items()}


def settings(name, sh_degree=0, bg=BG):
    """Oracle settings built once on the CPU; `settings_on` hands the GPU the same bits."""
    W, H = CAMERAS[name][:2]
    st = render_settings((H, W), camera(name), torch.tensor(bg, dtype=torch.float32), O.OracleSettings)
    return st._replace(sh_degree=sh_degree)


def _view32(st):
    return st.viewmatrix.contiguous().reshape(-1).numpy().astype(np.float32)


def view_z32(p, st):
    """fp32 view depth in the kernels' order (gaussian_math.cuh dot4_rn: products and sums rounded left to right)."""
    v = _view32(st)
    p = np.asarray(p, np.float32)
    return ((v[2] * p[:, 0] + v[6] * p[:, 1]) + v[10] * p[:, 2]) + v[14]


_NUDGES = np.array(sorted(((a, b, c) for a in range(-4, 5) for b in range(-4, 5) for c in range(-4, 5)),
                          key=lambda d: sum(map(abs, d))), np.int32)


def near_plane_points(st, n_each, seed):
    """n_each world points whose fp32 view depth is exactly 0.2f (culled), then n_each at the next float above it
    (kept).  world -> view does not round-trip exactly, so each candidate is nudged by ulps until it lands."""
    R = np.asarray(camera_R(st), np.float64)
    t = np.asarray(T_CAM, np.float64)
    rng = np.random.default_rng(seed)
    out = []
    for target in (NEAR, np.nextafter(NEAR, np.float32(1))):
        found, tries = 0, 0
        while found < n_each:
            tries += 1
            assert tries < 500, "no landing point found"
            pc = np.array([(2 * rng.random() - 1) * 0.7 * st.tanfovx * target,
                           (2 * rng.random() - 1) * 0.7 * st.tanfovy * target, float(target)])
            pw = ((pc - t) @ R).astype(np.float32)
            cand = (pw.view(np.int32)[None, :] + _NUDGES).view(np.float32)
            hit = np.nonzero(view_z32(cand, st) == target)[0]
            if len(hit):
                out.append(cand[hit[0]])
                found += 1
    return np.stack(out)


def camera_R(st):
    """R of the settings' view matrix (stored transposed: element (r, c) at [4c + r])."""
    return st.viewmatrix.double().t()[:3, :3].numpy()


def population(kind, st, n, seed, sh=False, boundary=True):
    """Assets of one population placed in camera space and mapped to world with R^T (p - t); `_pcam` keeps the
    camera-space positions (float64)."""
    g = torch.Generator().manual_seed(seed)
    U = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    tx, ty = float(st.tanfovx), float(st.tanfovy)
    W, H = st.image_width, st.image_height
    f = 0.5 * (W / (2 * tx) + H / (2 * ty))  # focal length in pixels (mean of fx, fy)
    spread, z = 1.1, 1.5 + 6.0 * U(n)
    px = 0.5 + 4.0 * U(n)  # footprint scale in pixels at depth z
    opac = 0.1 + 0.8 * U(n)
    if kind == "clamp":  # footprints wide enough to reach back into the image from the band
        spread, z = 2.0, 1.0 + 5.0 * U(n)
        px = max(W, H) * (0.02 + 0.25 * U(n))
        opac = 0.05 + 0.5 * U(n)
    elif kind == "near":
        spread, z = 0.9, 0.35 - 0.15 * U(n)
        px = px / z  # world sizes of a depth-1 splat: the footprints grow as 1/z
        opac = 0.05 + 0.5 * U(n)
    elif kind == "huge":
        spread, z = 0.8, 1.5 + 3.0 * U(n)
        px = max(W, H) * (0.05 + 0.6 * U(n))
        opac = 0.02 + 0.2 * U(n)
    pc = torch.stack([(2 * U(n) - 1) * spread * tx * z, (2 * U(n) - 1) * spread * ty * z, z], 1)
    scale = (px * z / f)[:, None] * (0.3 + 0.7 * U(n, 3))
    q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    q = q / q.norm(dim=1, keepdim=True)
    if kind == "awkward":
        q = q * (0.3 + 2.7 * U(n, 1))
        flat = torch.randint(0, 3, (n,), generator=g)
        scale[torch.arange(n), flat] *= 1e-4
    R = torch.from_numpy(camera_R(st))
    world = (pc - torch.tensor(T_CAM, dtype=torch.float64)) @ R
    a = {"mean_3d": world.float(), "scale": scale.float(), "rotation": q.float(), "opacity": opac.float()[:, None],
         "rgb": U(n, 3).float()}
    if sh:
        a["shs"] = 0.5 * torch.randn(n, 16, 3, generator=g)
    if kind == "near" and boundary:
        k = 3
        pts = torch.from_numpy(near_plane_points(st, k, seed))
        extra = {"mean_3d": pts, "scale": torch.full((2 * k, 3), 2.0 / f), "rotation": torch.tensor([[1.0, 0, 0, 0]] * (2 * k)),
                 "opacity": torch.full((2 * k, 1), 0.5), "rgb": torch.full((2 * k, 3), 0.7)}
        if sh:
            extra["shs"] = 0.3 * torch.ones(2 * k, 16, 3)
        a = {key: torch.cat((a[key], extra[key])) for key in a}
        pc = torch.cat((pc, (pts.double() @ R.t()) + torch.tensor(T_CAM, dtype=torch.float64)))
    a["_pcam"] = pc
    return a


def _cat(*pops):
    return {k: torch.cat([p[k] for p in pops]) for k in pops[0]}


def _seed(*parts):
    return zlib.crc32("/".join(map(str, parts)).encode()) & 0x7fffffff


def clamped_rows(st, pc, radii):
    """(rows clamped in x, rows clamped in y) among the visible Gaussians."""
    pc = pc.numpy()
    vis = radii > 0
    cx = vis & (np.abs(pc[:, 0] / pc[:, 2]) > 1.3 * st.tanfovx)
    cy = vis & (np.abs(pc[:, 1] / pc[:, 2]) > 1.3 * st.tanfovy)
    return cx, cy


def grad_images(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(3, H, W, generator=g), torch.randn(1, H, W, generator=g), torch.randn(1, H, W, generator=g)


N_SMALL = {"clamp": 500, "near": 150, "huge": 60, "awkward": 400, "plain": 500}


def case_population(cam, pop, sh=False, boundary=True):
    st = settings(cam, 3 if sh else 0)
    mul = 1 if cam in SMALL else (2 if pop == "huge" else 4)
    return st, population(pop, st, N_SMALL[pop] * mul, _seed(cam, pop), sh=sh, boundary=boundary)


# ---------------------------------------------------------------------------------------------------------------------
# CPU tier: the reference at these edges
# ---------------------------------------------------------------------------------------------------------------------

def _oracle_kw(a, mode):
    """Colour and shape arguments of a render: mode "rgb", "sh" (degree 3) or "cov" (cov3D_precomp)."""
    if mode == "cov":
        return dict(colors_precomp=a["rgb"], cov3D_precomp=a["cov"])
    colour = dict(shs=a["shs"]) if mode == "sh" else dict(colors_precomp=a["rgb"])
    return dict(scales=a["scale"], rotations=a["rotation"], **colour)


def _with_cov(a, seed):
    g = torch.Generator().manual_seed(seed)
    P = a["mean_3d"].shape[0]
    s = a["scale"].double().mean(1)[:, None, None]
    A = torch.randn(P, 3, 3, generator=g, dtype=torch.float64) * s
    S = A @ A.transpose(1, 2) + 1e-4 * s * s * torch.eye(3, dtype=torch.float64)
    return dict(a, cov=torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).float())


CPU_CASES = [(c, p, "rgb") for c in SMALL for p in ("clamp", "near", "awkward", "plain")] + [
    ("c61x45", "clamp", "sh"), ("c29x37", "plain", "cov"), ("c13x40", "awkward", "sh")]


def _cpu_case(cam, pop, mode):
    st, a = case_population(cam, pop, sh=(mode == "sh"), boundary=False)
    a = {k: v[::3] for k, v in a.items()}  # dense_autograd loops over Gaussians in Python: ~150 per case
    if mode == "cov":
        a = _with_cov(a, _seed(cam, pop, "cov"))
    return st, a


@pytest.mark.parametrize("cam,pop,mode", CPU_CASES)
def test_f64_oracle_matches_dense_autograd(cam, pop, mode):
    st, a = _cpu_case(cam, pop, mode)
    H, W = st.image_height, st.image_width
    d = lambda t: t.double().clone().requires_grad_()
    L = {k: d(v) for k, v in a.items() if k != "_pcam"}
    P = L["mean_3d"].shape[0]
    m2 = torch.zeros(P, 3, dtype=torch.float64, requires_grad=True)
    kw = _oracle_kw(L, mode)
    c, r, dep, al = DA.render(st, L["mean_3d"], m2, L["opacity"], **kw)
    gi, gd, ga = (x.double() for x in grad_images(H, W, _seed(cam, pop, mode, "g")))
    ((c * gi).sum() + (dep * gd).sum() + (al * ga).sum()).backward()
    oc, orad, od, oa, ctx = O.forward(st, L["mean_3d"].detach(), L["opacity"].detach(), variant="f64",
                                      **{k: v.detach() for k, v in kw.items()})
    assert np.array_equal(orad, r.numpy())
    assert (orad > 0).sum() >= 0.3 * P
    if pop == "clamp":
        cx, cy = clamped_rows(st, a["_pcam"], orad)
        assert cx.sum() >= 10 and cy.sum() >= 10  # a third of the population of the GPU cases
    for x, y in ((oc, c), (od, dep), (oa, al)):
        y = y.detach().numpy()
        assert np.abs(x - y).max() <= 1e-9 * np.abs(y).max()
    og = O.backward(ctx, gi.numpy(), gd.numpy()[0], ga.numpy()[0])
    named = [("means3D", L["mean_3d"]), ("means2D", m2), ("opacities", L["opacity"])]
    if mode == "cov":
        named += [("colors", L["rgb"]), ("cov3D", L["cov"])]
    else:
        named += [("scales", L["scale"]), ("rotations", L["rotation"])]
        named += [("shs", L["shs"])] if mode == "sh" else [("colors", L["rgb"])]
    for k, t in named:
        ref = t.grad.numpy().reshape(og[k].shape)
        assert np.abs(ref).max() > 0, k
        assert np.abs(og[k] - ref).max() <= 1e-9 * np.abs(ref).max(), k


@pytest.mark.parametrize("cam,pop,mode", CPU_CASES)
def test_f32_oracle_agrees_with_f64_oracle(cam, pop, mode):
    """The fp32 noise floor at these edges, with the bounds of test_oracle_autograd.test_fp32_oracle_agrees_with_fp64_oracle."""
    st, a = _cpu_case(cam, pop, mode)
    H, W = st.image_height, st.image_width
    gi, gd, ga = grad_images(H, W, _seed(cam, pop, mode, "g"))
    out = {}
    for v in ("f32", "f64"):
        c, r, d, al, ctx = O.forward(st, a["mean_3d"], a["opacity"], variant=v, **_oracle_kw(a, mode))
        gr = O.backward(ctx, gi.numpy(), gd.numpy()[0], ga.numpy()[0])
        out[v] = (c, r, d, al, gr, O.fragility(ctx, 1e-4, 1e-3))
    c32, r32, d32, a32, g32, _ = out["f32"]
    c64, r64, d64, a64, g64, (pm, gm) = out["f64"]
    assert np.array_equal(r32, r64)
    ok = ~pm
    assert pm.mean() < 0.01
    rel = lambda x, y, floor: float(np.max(np.abs(x - y) / np.maximum(np.abs(y), floor))) if x.size else 0.0
    assert rel(c32[:, ok], c64[:, ok], 0.1) < 1e-4
    assert rel(d32[0][ok], d64[0][ok], 0.5) < 1e-4
    assert rel(a32[0][ok], a64[0][ok], 0.1) < 1e-4
    names = ("means3D", "means2D", "opacities", "colors", "cov3D") if mode == "cov" else (
        "means3D", "means2D", "opacities", "scales", "rotations", "shs" if mode == "sh" else "colors")
    for k in names:
        y, x = g64[k][~gm], g32[k][~gm]
        # the one place the floor sits higher: d_scales of the flat Gaussians (one axis 1e-4 of the others), where the
        # fp32 covariance chain cancels -- measured 5.7e-5 (c61x45), every other case and tensor <= 1.7e-5
        lim = 1e-4 if (pop == "awkward" and k == "scales") else 5e-5
        assert rel(x, y, np.abs(g64[k]).max()) < lim, k
        assert rel(x, y, 0.1 * np.abs(g64[k]).max()) < 5e-4, k


def test_populations_reach_their_edges():
    """Counts per edge, as test_oracle_autograd.test_frustum_clamp_case_is_exercised, on the GPU cases' inputs."""
    for cam in SMALL + ("c203x131",):
        st, a = case_population(cam, "clamp")
        _, orad, *_ = O.forward(st, a["mean_3d"], a["opacity"], colors_precomp=a["rgb"], scales=a["scale"],
                                rotations=a["rotation"])
        cx, cy = clamped_rows(st, a["_pcam"], orad)
        assert cx.sum() >= 30 and cy.sum() >= 30, cam
        st, a = case_population(cam, "near")
        _, orad, *_ = O.forward(st, a["mean_3d"], a["opacity"], colors_precomp=a["rgb"], scales=a["scale"],
                                rotations=a["rotation"])
        z = view_z32(a["mean_3d"].numpy(), st)
        assert ((z > NEAR) & (z <= np.float32(0.35)) & (orad > 0)).sum() >= 100, cam
        assert list(z[-6:]) == [NEAR] * 3 + [np.nextafter(NEAR, np.float32(1))] * 3, cam
        assert list(orad[-6:-3]) == [0, 0, 0] and (orad[-3:] > 0).all(), cam
        st, a = case_population(cam, "huge")
        *_, ctx = O.forward(st, a["mean_3d"], a["opacity"], colors_precomp=a["rgb"], scales=a["scale"],
                            rotations=a["rotation"])
        rect = ctx.rect()
        tiles = (rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1])
        gx, gy = (st.image_width + 15) // 16, (st.image_height + 15) // 16
        assert (tiles == gx * gy).sum() >= 3, cam
        if gx * gy > 32:
            assert (tiles > 32).sum() >= 20, cam
        st, a = case_population(cam, "awkward")
        n = a["rotation"].norm(dim=1)
        assert float(n.min()) < 0.5 and float(n.max()) > 2.0
        s = a["scale"].sort(1).values
        assert float((s[:, 0] / s[:, 1]).max()) < 4e-4  # 1e-4 of its own size; the other two differ by <= 1/0.3


# ---------------------------------------------------------------------------------------------------------------------
# GPU tier
# ---------------------------------------------------------------------------------------------------------------------

def _grad_names(mode):
    return ["means3D", "means2D", "opacities", "scales", "rotations", "shs" if mode == "sh" else "colors"]


def _plan_vs_oracle(dev, case, st_c, a, mode, clamp_rows=None, f64_refs=()):
    """One render through FramePlan (C ABI) against the oracle: radii, images, contributors, every gradient with depth
    and alpha losses in; `clamp_rows` (bool P) are compared again as a tensor of their own.  The gradients named in
    `f64_refs` are compared with the oracle's f64 build instead of its f32 build (see test_plan_matches_oracle)."""
    from exavatar_release_b200 import rasterizer as rz
    from exavatar_release_b200.plan import FramePlan, grad_bucket
    H, W = st_c.image_height, st_c.image_width
    M = 16 if mode == "sh" else 0
    oc, orad, od, oa, octx = O.forward(st_c, a["mean_3d"], a["opacity"], **_oracle_kw(a, mode))
    pm, gm = O.fragility(octx)
    P = a["mean_3d"].shape[0]
    plan = FramePlan(P, W, H, 2 * octx.num_dups + 4096, dev, sh_coeffs=M)
    sc = plan.scene(0, settings_on(st_c, dev, rz.GaussianRasterizationSettings),
                    {k: v.to(dev) for k, v in a.items() if k != "_pcam"})
    plan.forward(sc)
    torch.cuda.synchronize()
    assert plan.status()["overflow"] == 0
    assert np.array_equal(plan.radii.cpu().numpy(), orad), "radii must be identical"
    compare(case, "color", plan.color.cpu().numpy(), oc, pm[None], kind="image")
    compare(case, "depth", plan.depth.cpu().numpy(), od, pm[None], kind="image")
    compare(case, "alpha", plan.alpha.cpu().numpy(), oa, pm[None], kind="image")
    ctx = plan.read_ctx()
    contributor_report(case, last_contributor(ctx["ids"], ctx["ranges"], ctx["n_contrib"], W, H), ctx["final_T"],
                       last_contributor(octx.sorted_ids(), octx.ranges(), octx.n_contrib(), W, H), octx.final_T(), pm)
    gi, gd, ga = grad_images(H, W, _seed(case, "g"))
    flat, views = grad_bucket(P, dev, M)
    plan.backward(sc, gi.to(dev), views, g_depth=gd.to(dev), g_alpha=ga.to(dev))
    torch.cuda.synchronize()
    og = O.backward(octx, gi.numpy(), gd.numpy()[0], ga.numpy()[0])
    refs = {}
    if f64_refs:
        *_, c64 = O.forward(st_c, a["mean_3d"], a["opacity"], variant="f64", **_oracle_kw(a, mode))
        g64 = O.backward(c64, gi.numpy(), gd.numpy()[0], ga.numpy()[0])
        for k in f64_refs:
            # both fp32 results scatter around the f64 values; the CUDA one may not scatter more than 4x as widely as the
            # f32 oracle (unflagged p99.9 and max, units of max|y|)
            e = lambda t: (np.abs(np.asarray(t, np.float64) - g64[k]) / np.abs(g64[k]).max())[~gm]
            e_cuda, e_f32 = e(views[k].cpu().numpy().reshape(g64[k].shape)), e(og[k])
            q = lambda e_: f"p99 {np.quantile(e_, 0.99):.2e} p99.9 {np.quantile(e_, 0.999):.2e} max {e_.max():.2e}"
            print(f"F64FLOOR {case} d_{k}: cuda {q(e_cuda)}; f32 oracle {q(e_f32)}", flush=True)
            assert np.quantile(e_cuda, 0.999) <= 4 * np.quantile(e_f32, 0.999) + 1e-6, k
            assert e_cuda.max() <= 4 * e_f32.max() + 1e-6, k
            refs[k] = g64[k]
    for k in _grad_names(mode):
        y = refs.get(k, og[k])
        x = views[k].cpu().numpy().reshape(y.shape)
        row = gm.reshape((-1,) + (1,) * (y.ndim - 1))
        compare(case + ("/f64" if k in refs else ""), "d_" + k, x, y, row, kind="grad",
                **({"p999_unflagged": 1e-4} if k in refs else {}))
        if clamp_rows is not None:
            compare(case + "/clamped", "d_" + k, x[clamp_rows], y[clamp_rows], row[clamp_rows], kind="grad")
    assert float(views["means2D"][:, 2].abs().max()) == 0.0
    return orad


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["rgb", "sh"])
@pytest.mark.parametrize("pop", POPS)
@pytest.mark.parametrize("cam", SMALL + ("c203x131",))
def test_plan_matches_oracle(dev, cam, pop, mode):
    st, a = case_population(cam, pop, sh=(mode == "sh"))
    clamp = None
    if pop == "clamp":
        _, orad, *_ = O.forward(st, a["mean_3d"], a["opacity"], **_oracle_kw(a, mode))
        cx, cy = clamped_rows(st, a["_pcam"], orad)
        assert cx.sum() >= 30 and cy.sum() >= 30
        clamp = cx | cy
    # "awkward": un-normalised quaternions of norm up to 3 (R(q) = (1 - |q|^2) I + |q|^2 R(q/|q|): entries up to ~18 that
    # cancel) on flat scales make d_scales and d_rotations ill-conditioned in fp32.  On the c203x131 inputs the oracle's
    # own f32 build is off its f64 build by p99.9 3.6e-5 / max 1.4e-3 (d_scales) and 1.4e-5 / 4.9e-4 (d_rotations), so
    # the f32 build is no reference there: those two tensors are held against the f64 build, by compare's rules with
    # the unflagged p99.9 bound at 1e-4, and against the f32 build's own error.  The CUDA gradients are not bit-identical
    # from run to run (fp32 atomic sums), and the conditioning turns that into a spread: over repeated runs on an H100
    # the CUDA p99.9 against f64 went from 1.4e-5 to 3.2e-5, up to 2.2x the f32 build's.
    f64_refs = ("scales", "rotations") if pop == "awkward" else ()
    _plan_vs_oracle(dev, f"gencam/{cam}/{pop}/{mode}", st, a, mode, clamp, f64_refs)


def _mixed(cam, seed_tag, n_plain, n_clamp):
    st = settings(cam)
    return st, _cat(population("plain", st, n_plain, _seed(cam, seed_tag, "plain")),
                    population("clamp", st, n_clamp, _seed(cam, seed_tag, "clamp")))


@pytest.mark.gpu
@pytest.mark.parametrize("capacity", ["adaptive", "fixed"])
@pytest.mark.parametrize("mode", ["rgb", "cov"])
def test_public_rasterizer_matches_oracle(dev, capacity, mode):
    """GaussianRasterizer with scale / rotation or cov3D_precomp at a general camera, against the oracle; with the
    adaptive duplicate capacity and with a fixed one (`set_fixed_capacity`, the graph-capturable call)."""
    from exavatar_release_b200 import rasterizer as rz
    cam = "c203x131"
    st, a = _mixed(cam, "public", 1500, 300)
    if mode == "cov":
        a = _with_cov(a, _seed(cam, "cov"))
    H, W = st.image_height, st.image_width
    case = f"gencam/public/{capacity}/{mode}"
    oc, orad, od, oa, octx = O.forward(st, a["mean_3d"], a["opacity"], **_oracle_kw(a, mode))
    pm, gm = O.fragility(octx)
    P = a["mean_3d"].shape[0]
    L = {k: v.to(dev).requires_grad_() for k, v in a.items() if k != "_pcam"}
    m2 = torch.zeros(P, 3, device=dev, requires_grad=True)
    rz.set_fixed_capacity(octx.num_dups + 4096 if capacity == "fixed" else None)
    try:
        color, radii, depth, alpha = rz.GaussianRasterizer(settings_on(st, dev, rz.GaussianRasterizationSettings))(
            means3D=L["mean_3d"], means2D=m2, opacities=L["opacity"], **_oracle_kw(L, mode))
        gi, gd, ga = grad_images(H, W, _seed(case))
        ((color * gi.to(dev)).sum() + (depth * gd.to(dev)).sum() + (alpha * ga.to(dev)).sum()).backward()
        assert not rz.overflowed()
    finally:
        rz.set_fixed_capacity(None)
    assert np.array_equal(radii.cpu().numpy(), orad)
    compare(case, "color", color.detach().cpu().numpy(), oc, pm[None], kind="image")
    compare(case, "depth", depth.detach().cpu().numpy(), od, pm[None], kind="image")
    compare(case, "alpha", alpha.detach().cpu().numpy(), oa, pm[None], kind="image")
    og = O.backward(octx, gi.numpy(), gd.numpy()[0], ga.numpy()[0])
    pairs = [("means3D", L["mean_3d"].grad), ("means2D", m2.grad), ("opacities", L["opacity"].grad),
             ("colors", L["rgb"].grad)]
    pairs += [("cov3D", L["cov"].grad)] if mode == "cov" else [("scales", L["scale"].grad), ("rotations", L["rotation"].grad)]
    for k, t in pairs:
        y = og[k]
        compare(case, "d_" + k, t.cpu().numpy().reshape(y.shape), y, gm.reshape((-1,) + (1,) * (y.ndim - 1)), kind="grad")
    assert float(m2.grad[:, 2].abs().max()) == 0.0


@pytest.mark.gpu
def test_stage_buffers_with_huge_splats(dev):
    """Population "huge" at a general camera (203x131: 13x9 tiles): the geometry record (pixel centre, pre-scaled conic,
    depth, rect) against the oracle; per-tile lists identical without tile culling (the scatter's cooperative replay of
    rects > 32 tiles) and ordered subsets with it (the row-interval culling of big rects)."""
    from exavatar_release_b200 import _lib as L
    from exavatar_release_b200 import rasterizer as rz
    from exavatar_release_b200.plan import FramePlan
    st, a = case_population("c203x131", "huge")
    W, H = st.image_width, st.image_height
    P = a["mean_3d"].shape[0]
    _, orad, _, _, ctx = O.forward(st, a["mean_3d"], a["opacity"], colors_precomp=a["rgb"], scales=a["scale"],
                                   rotations=a["rotation"])
    vis = orad > 0
    rect = ctx.rect()
    tiles = (rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1])
    assert (tiles > 32).sum() >= 20 and (tiles == ((W + 15) // 16) * ((H + 15) // 16)).sum() >= 3
    o_ids, o_ranges = ctx.sorted_ids(), ctx.ranges()
    st_g = settings_on(st, dev, rz.GaussianRasterizationSettings)
    ga = {k: v.to(dev) for k, v in a.items() if k != "_pcam"}
    for flags in (L.B2R_FLAG_NO_TILE_CULL, 0):
        plan = FramePlan(P, W, H, 2 * ctx.num_dups + 4096, dev)
        plan.forward(plan.scene(0, st_g, ga, flags=flags))
        torch.cuda.synchronize()
        status = plan.status()
        assert status["overflow"] == 0
        lists = plan.read_ctx()
        ranges, ids, geom, aux = lists["ranges"], lists["ids"], lists["geom"], lists["aux"]
        if flags:
            assert np.array_equal(aux[:, 2], orad)
            assert status["num_visible"] == int(vis.sum())
            assert np.allclose(geom[vis, 0:2], ctx.xy()[vis], rtol=0, atol=2e-4)
            assert np.allclose(geom[vis, 6], ctx.depth()[vis], rtol=1e-6)
            L2E = 1.4426950408889634
            co = ctx.conic_opacity()[vis]
            assert np.allclose(geom[vis, 2] / (-0.5 * L2E), co[:, 0], rtol=2e-5, atol=1e-7)
            assert np.allclose(geom[vis, 3] / (-L2E), co[:, 1], rtol=2e-5, atol=1e-6)
            assert np.allclose(geom[vis, 4] / (-0.5 * L2E), co[:, 2], rtol=2e-5, atol=1e-7)
            rv = rect[vis]
            assert np.array_equal(aux[vis, 0] & 0xffff, rv[:, 0]) and np.array_equal(aux[vis, 0] >> 16, rv[:, 1])
            assert np.array_equal(aux[vis, 1] & 0xffff, rv[:, 2]) and np.array_equal(aux[vis, 1] >> 16, rv[:, 3])
            assert status["num_dups"] == ctx.num_dups
            for t in range(ranges.shape[0]):
                assert np.array_equal(ids[ranges[t, 0]:ranges[t, 1]], o_ids[o_ranges[t, 0]:o_ranges[t, 1]]), f"tile {t}"
        else:
            assert status["num_dups"] <= ctx.num_dups
            for t in range(ranges.shape[0]):
                it = iter(o_ids[o_ranges[t, 0]:o_ranges[t, 1]].tolist())
                assert all(m in it for m in ids[ranges[t, 0]:ranges[t, 1]].tolist()), f"tile {t}: not an ordered subsequence"


@pytest.mark.gpu
@pytest.mark.parametrize("cam", SMALL + ("c203x131",))
def test_mark_visible_on_the_near_plane(dev, cam):
    """markVisible against the oracle's pv.z > 0.2 decision, bit for bit on the boundary floats."""
    from exavatar_release_b200 import rasterizer as rz
    st, a = case_population(cam, "near")
    p = a["mean_3d"]
    expect = view_z32(p.numpy(), st) > NEAR
    assert list(expect[-6:]) == [False] * 3 + [True] * 3
    gpu = rz.GaussianRasterizer(settings_on(st, dev, rz.GaussianRasterizationSettings)).markVisible(p.to(dev)).cpu().numpy()
    assert np.array_equal(O.mark_visible(p, st.viewmatrix).numpy(), expect)
    assert np.array_equal(gpu, expect)


def _frame_populations(cam, sh):
    """Scene (plain + clamp band), human (a compact cluster) and refined (the human with small offsets)."""
    st = settings(cam)
    scene = _cat(population("plain", st, 1500, _seed(cam, "scene"), sh=sh),
                 population("clamp", st, 300, _seed(cam, "scene-clamp"), sh=sh))
    hum = population("plain", st, 1200, _seed(cam, "human"))
    g = torch.Generator().manual_seed(_seed(cam, "refined"))
    ref = dict(hum, mean_3d=hum["mean_3d"] + 0.01 * torch.randn(hum["mean_3d"].shape, generator=g),
               scale=hum["scale"] * (1.0 + 0.1 * torch.rand(hum["scale"].shape, generator=g)),
               rgb=(hum["rgb"] + 0.1 * torch.randn(hum["rgb"].shape, generator=g)).clamp(0, 1))
    strip = lambda d, keep: {k: d[k] for k in keep}
    hk = ("mean_3d", "scale", "rotation", "opacity", "rgb")
    return strip(scene, hk + (("shs",) if sh else ())), strip(hum, hk), strip(ref, hk)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["rgb", "sh"])
def test_merged_frame_vs_five_oracle_renders(dev, mode):
    """MergedFivePlan at 203x131 under a general camera, every view against its own oracle render (the comparison of
    test_gpu_fullsize.test_c4_five_render_frame_vs_five_oracle_renders); mode "sh": a degree-3 SH scene coloured inside
    the passes (test_frame_sh.test_c4_sh_frame_vs_oracle_renders)."""
    from exavatar_release_b200 import rasterizer as rz
    from exavatar_release_b200.plan import RENDERS, MergedFivePlan
    cam = "c203x131"
    W, H = CAMERAS[cam][:2]
    sh = mode == "sh"
    scene, human, refined = _frame_populations(cam, sh)
    Ps, Ph = scene["mean_3d"].shape[0], human["mean_3d"].shape[0]
    bg_w, bg_r = torch.ones(3), torch.tensor([0.3, 0.7, 0.2])
    st_w, st_r = settings(cam, bg=(1.0, 1.0, 1.0)), settings(cam, bg=(0.3, 0.7, 0.2))
    gcol = {r: grad_images(H, W, _seed(mode, r))[0] for r in RENDERS}
    cat = lambda x, y: {k: torch.cat((x[k], y[k])) for k in ("mean_3d", "scale", "rotation", "opacity", "rgb")}
    sc_rgb = scene
    if sh:
        sc_rgb = dict(scene, rgb=sh_to_rgb(3, scene["shs"].double(), scene["mean_3d"].double(), st_w.campos.double()).float())
    sets = {"scene": (sc_rgb, st_w), "human": (human, st_r), "scene_human": (cat(sc_rgb, human), st_w),
            "human_refined": (refined, st_r), "scene_human_refined": (cat(sc_rgb, refined), st_w)}
    ora, dups = {}, 0
    for r, (a, st) in sets.items():
        kw = dict(colors_precomp=a["rgb"])
        if sh and r == "scene":
            st, kw = st._replace(sh_degree=3), dict(shs=scene["shs"])
        oc, orad, _, oa, octx = O.forward(st, a["mean_3d"], a["opacity"], scales=a["scale"], rotations=a["rotation"], **kw)
        ora[r] = dict(color=oc, radii=orad, alpha=oa, grads=O.backward(octx, gcol[r].numpy()), frag=O.fragility(octx))
        dups = max(dups, octx.num_dups)
    to = lambda d: {k: v.to(dev) for k, v in d.items()}
    plan = MergedFivePlan(Ps, Ph, W, H, {"A": 2 * dups + 4096, "B": 2 * dups + 4096}, dev, sh_coeffs=16 if sh else 0)
    sc_dev = to(scene)
    if sh:
        sc_dev = dict({k: v for k, v in sc_dev.items() if k != "rgb"}, sh_degree=3)
    plan.set_scene(sc_dev)
    st_wg, st_rg = (settings_on(s, dev, rz.GaussianRasterizationSettings) for s in (st_w, st_r))
    plan.frame(0, st_wg, st_rg, sc_dev, to(human), to(refined), {r: g.to(dev) for r, g in gcol.items()}, accumulate=False)
    torch.cuda.synchronize()
    assert not plan.overflowed()
    case = f"gencam/merged/{mode}/"
    for r in RENDERS:
        pm, _ = ora[r]["frag"]
        img, alpha, radii = plan.render_outputs(r)
        assert np.array_equal(radii.cpu().numpy(), ora[r]["radii"]), r
        compare(case + r, "color", img.cpu().numpy(), ora[r]["color"], pm[None], kind="image")
        compare(case + r, "alpha", alpha.cpu().numpy(), ora[r]["alpha"], pm[None], kind="image")
    plan.reduce()
    common = ("means3D", "means2D", "opacities", "scales", "rotations")

    def expect(parts, names):
        out, flag = {}, None
        for r, rows in parts:
            g, (_, gm) = ora[r]["grads"], ora[r]["frag"]
            for k in names:
                y = g[k][rows].reshape(g[k][rows].shape[0], -1)
                out[k] = y if k not in out else out[k] + y
            flag = gm[rows] if flag is None else (flag | gm[rows])
        return out, flag

    for label, Pn, parts, names in (
            ("scene", Ps, [("scene", slice(0, Ps))], common + (("shs",) if sh else ("colors",))),
            ("human", Ph, [("human", slice(0, Ph)), ("scene_human", slice(Ps, Ps + Ph))], common + ("colors",)),
            ("human_refined", Ph, [("human_refined", slice(0, Ph)), ("scene_human_refined", slice(Ps, Ps + Ph))],
             common + ("colors",))):
        views = plan.grads(label)
        y, flag = expect(parts, names)
        for k in names:
            compare(case + label, "d_" + k, views[k].cpu().numpy().reshape(Pn, -1), y[k], flag[:, None], kind="grad")


def _skin_rig(cam, dev, P=4000, J=55):
    """A 4-sparse (P, J) weight table read through random rows, small joint rotations and translations, and canonical
    positions that the rig and the camera (world = R^-1 (posed - t)) bring back to a plain population in view."""
    st = settings(cam)
    g = torch.Generator().manual_seed(_seed(cam, "rig"))
    w = torch.zeros(P, J)
    idx = torch.rand(P, J, generator=g).topk(4, dim=1).indices
    val = torch.rand(P, 4, generator=g) + 0.05
    w.scatter_(1, idx, val / val.sum(1, keepdim=True))
    ax = torch.randn(J, 3, generator=g)
    ax = ax / ax.norm(dim=1, keepdim=True) * (0.15 * torch.rand(J, 1, generator=g))
    K = torch.zeros(J, 3, 3)
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -ax[:, 2], ax[:, 1], -ax[:, 0]
    K = K - K.transpose(1, 2)
    A = torch.eye(4).repeat(J, 1, 1)
    A[:, :3, :3] = torch.linalg.matrix_exp(K)
    A[:, :3, 3] = 0.02 * torch.randn(J, 3, generator=g)
    trans = torch.tensor([0.01, -0.02, 0.03])
    rows = torch.randint(0, P, (P,), generator=g)
    rows[:500] = torch.arange(500)
    cp = camera(cam)
    hum = population("plain", st, P, _seed(cam, "skin"))
    xyz = hum["mean_3d"] @ cp["R"].t() + cp["t"].view(1, 3)
    xyz_r = xyz + 0.01 * torch.randn(P, 3, generator=g)
    to = lambda t: t.to(dev)
    return dict(st=st, xyz=to(xyz), xyz_r=to(xyz_r), table=to(w), rows=to(rows), A=to(A), trans=to(trans),
                R=to(cp["R"]), t=to(cp["t"]), human={k: to(v) for k, v in hum.items() if k != "_pcam"})


@pytest.mark.gpu
def test_skinning_under_a_general_camera(dev):
    """skin_gaussians' posed positions and gradients against float64 autograd through lbs_reference, with cam_R / cam_t
    of a general camera (test_skin_pair's comparisons): every entry of R^-1 is non-zero and none equals its transpose."""
    from exavatar_release_b200.skinning import skin_gaussians
    rig = _skin_rig("c61x45", dev)
    P = rig["xyz"].shape[0]
    g = torch.Generator().manual_seed(4)
    gp, gq = torch.randn(P, 3, generator=g).to(dev), torch.randn(P, 3, generator=g).to(dev)
    x, xr = rig["xyz"].clone().requires_grad_(), rig["xyz_r"].clone().requires_grad_()
    A, tr = rig["A"].clone().requires_grad_(), rig["trans"].clone().requires_grad_()
    posed, posed_r = skin_gaussians(x, xr, rig["table"], rig["rows"], A, tr, rig["R"], rig["t"])
    ((posed * gp).sum() + (posed_r * gq).sum()).backward()
    torch.cuda.synchronize()
    w = rig["table"].double()[rig["rows"]]
    lx = [rig["xyz"].double().requires_grad_(), rig["xyz_r"].double().requires_grad_()]
    lA, lt = rig["A"].double().requires_grad_(), rig["trans"].double().requires_grad_()
    R, t = rig["R"].double(), rig["t"].double()
    ref = [lbs_reference(v, w, lA, lt, R, t) for v in lx]
    for got, r in zip((posed, posed_r), ref):
        r = r.detach()
        assert float((got.double() - r).abs().max()) <= 1e-6 * float(r.abs().max())
    ((ref[0] * gp.double()).sum() + (ref[1] * gq.double()).sum()).backward()
    for name, got, r in (("xyz", x.grad, lx[0].grad), ("xyz_refined", xr.grad, lx[1].grad), ("A", A.grad, lA.grad),
                         ("trans", tr.grad, lt.grad)):
        d = float((got.double() - r).abs().max())
        assert d <= 1e-5 * float(r.abs().max()), (name, d, float(r.abs().max()))


@pytest.mark.gpu
def test_skinned_rasterizer_under_a_general_camera(dev):
    """SkinnedGaussianRasterizer's `posed` equals skin_gaussians bit for bit, and its gradients (image and posed
    terms of the loss) equal those of skin_gaussians + GaussianRasterizer."""
    from exavatar_release_b200 import rasterizer as rz
    from exavatar_release_b200.skinning import skin_gaussians
    rig = _skin_rig("c203x131", dev)
    st = settings_on(rig["st"], dev, rz.GaussianRasterizationSettings)
    h = rig["human"]
    P = rig["xyz"].shape[0]
    H, W = st.image_height, st.image_width
    gi = grad_images(H, W, 11)[0].to(dev)
    gp = torch.randn(P, 3, generator=torch.Generator().manual_seed(12)).to(dev)
    w_gathered = rig["table"][rig["rows"]].contiguous()

    def leaves():
        return {k: v.clone().requires_grad_() for k, v in (("xyz", rig["xyz"]), ("A", rig["A"]), ("trans", rig["trans"]),
                                                             ("opacity", h["opacity"]), ("rgb", h["rgb"]),
                                                             ("scale", h["scale"]), ("rotation", h["rotation"]))}

    a = leaves()
    m2a = torch.zeros(P, 3, device=dev, requires_grad=True)
    posed_a = skin_gaussians(a["xyz"], None, rig["table"], rig["rows"], a["A"], a["trans"], rig["R"], rig["t"])[0]
    img_a, rad_a, _, _ = rz.GaussianRasterizer(st)(means3D=posed_a, means2D=m2a, opacities=a["opacity"],
                                                  colors_precomp=a["rgb"], scales=a["scale"], rotations=a["rotation"])
    ((img_a * gi).sum() + (posed_a * gp).sum()).backward()
    b = leaves()
    m2b = torch.zeros(P, 3, device=dev, requires_grad=True)
    img_b, rad_b, _, _, posed_b = rz.SkinnedGaussianRasterizer(st)(b["xyz"], w_gathered, b["A"], b["trans"], rig["R"],
                                                                   rig["t"], m2b, b["opacity"], b["rgb"], b["scale"],
                                                                   b["rotation"])
    ((img_b * gi).sum() + (posed_b * gp).sum()).backward()
    torch.cuda.synchronize()
    assert torch.equal(posed_b, posed_a.detach())
    assert torch.equal(rad_b, rad_a) and int((rad_a > 0).sum()) > P // 2
    assert torch.allclose(img_b, img_a, atol=1e-6)
    for k in a:
        y = a[k].grad
        assert float(y.abs().max()) > 0, k
        assert float((b[k].grad - y).abs().max()) <= 1e-4 * float(y.abs().max()), k
    assert float((m2b.grad - m2a.grad).abs().max()) <= 1e-4 * float(m2a.grad.abs().max())


@pytest.mark.gpu
def test_full_size_general_camera(dev):
    """512x512 with pitch, roll and fx != fy: 60 000 plain Gaussians plus 1 % in the clamp band, through FramePlan
    against the oracle (test_gpu_fullsize._plan_vs_oracle's assertions, depth and alpha losses in)."""
    st, a = _mixed("c512", "full", 60000, 600)
    _plan_vs_oracle(dev, "gencam/c512", st, a, "rgb")
