"""SH-coloured scene Gaussians inside the merged training frame (SURVEY.md section 8f-4 + 8f-3).

ExAvatar renders cat(scene, human) twice per training frame (avatar/main/model.py:117-162).  With the scene coloured from
SH coefficients and the human sets from RGB, those combined renders need a pass whose first rows take their colour from
`shs` and the rest from `colors_precomp`: B2RScene.sh_rows.  These tests pin
  * the C ABI of that mixed pass (struct layout, host-side validation) and the gradient bucket of `MergedFivePlan`
    with an SH scene, without a device;
  * the f64 oracle reference the GPU tests build on (caller-side sh_to_rgb + autograd == the oracle's own SH render);
  * on the GPU: mixed pass == the single-source renders, `TrainingFrameRenderer` with an SH scene == the same renderer
    fed caller-side RGB (eager and CUDA graph, SH degree raised between frames), and every view of a full C4 frame
    against its own oracle render.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from util import settings_on, workload_settings  # noqa: F401  (also sets up the import path)
from util import dev  # noqa: F401
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.camera import look_at_cam_param
from exavatar_release_b200.plan import FiveRenderPlan, merged_bucket_layout
from exavatar_release_b200.renderer import render_settings, scene_gaussian_assets
from exavatar_release_b200.sh import sh_to_rgb
from exavatar_release_b200.synthetic import (WORKLOADS, make_grad_image, make_population_assets,
                                             make_scene_sh_params)
from oracle import oracle as O

FAKE = 0x1000  # never dereferenced: validation fails before any launch


# ---------------------------------------------------------------------------------------------------------------------
# CPU: ABI, validation, bucket layout, oracle reference
# ---------------------------------------------------------------------------------------------------------------------

def test_sh_rows_takes_the_place_of_the_reserved_field():
    names = [f[0] for f in L.B2RScene._fields_]
    assert "skin_reserved" not in names and names[-1] == "sh_rows"
    # the int32 sits right after the last per-Gaussian pointer, at the end of the struct (then 4 bytes of tail padding
    # to the pointers' 8-byte alignment)
    assert L.B2RScene.sh_rows.offset == L.B2RScene.cov3D_precomp.offset + 8
    assert L.B2RScene.sh_rows.offset + 8 == C.sizeof(L.B2RScene)
    assert L.B2RScene.sh_rows.size == 4


def _valid_scene(P=64):
    sc = L.B2RScene()
    sc.P, sc.width, sc.height, sc.tanfovx, sc.tanfovy = P, 32, 32, 0.5, 0.5
    sc.bg = sc.viewmatrix = sc.projmatrix = sc.campos = FAKE
    sc.means3D = sc.opacities = sc.scales = sc.rotations = FAKE
    sc.shs = sc.colors_precomp = FAKE
    sc.sh_degree, sc.sh_coeffs, sc.sh_rows = 3, 16, 40
    return sc


def test_mixed_colour_source_validation_without_touching_cuda():
    lib = L.load()
    n0 = lib.b2r_launch_count()
    sc = _valid_scene()
    ws = L.B2RWorkspace()
    ws.ctx, ws.ctx_bytes = FAKE, 16  # too small on purpose: a scene that validates reaches the workspace check (-2)
    out = L.B2RForwardOutputs()
    fwd = lambda: lib.b2r_forward(C.byref(sc), C.byref(ws), C.byref(out), None)
    proj = lambda: lib.b2r_forward_project(C.byref(sc), C.byref(ws), FAKE, None)
    assert fwd() == -2 and proj() == -2        # both sources + 0 < sh_rows <= P: valid
    sc.sh_rows = 64
    assert fwd() == -2                         # sh_rows == P: every row from SH, still valid
    sc.sh_rows = 65
    assert fwd() == -1 and proj() == -1        # sh_rows > P
    sc.sh_rows = -1
    assert fwd() == -1                         # negative
    sc.sh_rows = 40
    sc.colors_precomp = None
    assert fwd() == -1 and proj() == -1        # mixed needs the colour rows' source
    sc.colors_precomp, sc.shs = FAKE, None
    assert fwd() == -1 and proj() == -1        # ... and the SH rows' source
    sc.shs = FAKE
    sc.sh_coeffs = 9
    assert fwd() == -1                         # the sh_degree / sh_coeffs rules still apply
    sc.sh_degree, sc.sh_coeffs = 1, 17
    assert fwd() == -1
    sc.sh_degree, sc.sh_coeffs = 3, 16
    # sh_rows == 0 keeps the one-source rule
    sc.sh_rows = 0
    assert fwd() == -1
    sc.shs = None
    assert fwd() == -2
    sc.shs, sc.sh_rows = FAKE, 40

    # backward: dL_dshs is required while SH rows at or above first_row exist
    ws.ctx_bytes = lib.b2r_ctx_bytes(64, 32, 32)
    args = L.B2RBackwardArgs()
    args.dL_dcolor = FAKE
    bwd = lambda: lib.b2r_backward(C.byref(sc), C.byref(ws), C.byref(args), FAKE, 1 << 20, None)
    bproj = lambda: lib.b2r_backward_project(C.byref(sc), C.byref(ws), C.byref(args), FAKE, 1 << 20, None)
    for first_row in (0, 39):
        args.first_row = first_row
        assert bwd() == -1 and bproj() == -1, first_row
    # a scene of sh_rows == 0 with shs keeps requiring dL_dshs for every row
    sc.colors_precomp, sc.sh_rows = None, 0
    args.first_row = 50
    assert bwd() == -1 and bproj() == -1
    assert lib.b2r_launch_count() == n0        # nothing was launched by any of the above


def test_merged_bucket_layout_with_an_sh_scene():
    PER = FiveRenderPlan.PER
    Ps, Ph = 130, 167
    # sh_coeffs = 0: the layout of the plan without SH -- pass A | pass B | densification tail
    lay0 = merged_bucket_layout(Ps, Ph, 0)
    assert lay0["A"] == (0, PER * (Ps + Ph))
    assert lay0["A_shs"][1] == 0
    assert lay0["B"] == (PER * (Ps + Ph), PER * Ph)
    assert lay0["stats"] == (PER * (Ps + 2 * Ph), 2 * Ps)
    assert lay0["total"] == (0, PER * (Ps + 2 * Ph) + 2 * Ps)
    for M in (4, 9, 16):
        lay = merged_bucket_layout(Ps, Ph, M)
        assert lay["A"] == lay0["A"]
        assert lay["A_shs"] == (PER * (Ps + Ph), 3 * M * Ps)          # right after pass A
        assert lay["B"] == (PER * (Ps + Ph) + 3 * M * Ps, PER * Ph)
        o, n = lay["stats"]
        assert n == 2 * Ps and o + n == lay["total"][1]               # the tail stays the tail
        assert lay["total"][1] == lay0["total"][1] + 3 * M * Ps
        # regions tile the buffer without gaps or overlap
        regions = sorted(lay[k] for k in ("A", "A_shs", "B", "stats"))
        end = 0
        for off, num in regions:
            assert off == end
            end = off + num
        assert end == lay["total"][1]


def _oracle_sh_scene_reference(st, scene_p, deg, gi):
    """f64 oracle: scene colour = sh.sh_to_rgb in f64 with autograd through it, rendered from `colors_precomp`.
    Returns (image, {param: grad}, mean_2d grad)."""
    class F64(O.OracleRasterizer):
        def __init__(self, raster_settings):
            super().__init__(raster_settings, variant="f64")

    leaves = {k: v.detach().double().clone().requires_grad_() for k, v in scene_p.items()}
    shs = torch.cat((leaves["feature_dc"], leaves["feature_rest"]), 1)
    rgb = sh_to_rgb(deg, shs, leaves["mean"], st.campos.double())
    m2 = torch.zeros(leaves["mean"].shape[0], 3, dtype=torch.float64, requires_grad=True)
    img, radii, _, _ = F64(st)(means3D=leaves["mean"], means2D=m2, colors_precomp=rgb,
                               opacities=torch.sigmoid(leaves["opacity_logit"]), scales=torch.exp(leaves["log_scale"]),
                               rotations=leaves["rotation"])
    (img * gi.double()).sum().backward()
    return img.detach(), {k: v.grad for k, v in leaves.items()}, m2.grad, radii


@pytest.mark.parametrize("deg", [1, 3])
def test_oracle_reference_equals_the_oracle_sh_render(deg):
    """The reference of the GPU tests (caller-side SH in f64 + autograd + oracle) is the oracle's own SH render."""
    wl = WORKLOADS["T1"]
    H, W = wl.height, wl.width
    scene, _, _ = make_population_assets("T1", seed=2)
    p = make_scene_sh_params(scene, 3, seed=2)
    st = render_settings((H, W), look_at_cam_param(7.0, (H, W)), torch.tensor([0.2, 0.4, 0.6]), O.OracleSettings)
    gi = make_grad_image("T1", 5)
    img_a, g_a, m2_a, rad_a = _oracle_sh_scene_reference(st, p, deg, gi)
    # the oracle's SH path: coefficients in, dL/dSH and the view-direction term of dL/dmean out
    shs = torch.cat((p["feature_dc"], p["feature_rest"]), 1).double()
    opac = torch.sigmoid(p["opacity_logit"].double())
    scl = torch.exp(p["log_scale"].double())
    oc, orad, _, _, octx = O.forward(st._replace(sh_degree=deg), p["mean"].double(), opac, shs=shs, scales=scl,
                                     rotations=p["rotation"].double(), variant="f64")
    og = O.backward(octx, gi.double().numpy())
    assert np.array_equal(rad_a.numpy(), orad)
    assert float(img_a.abs().max()) > 0.1
    # the oracle's SH polynomial and the PyTorch restatement agree to ~1e-8 in f64 (fp32-rounded SH constants), far
    # below the 1e-4 of the GPU comparisons this reference serves
    tol = 1e-6
    assert np.abs(img_a.numpy() - oc).max() < tol
    rel = lambda x, y: np.abs(np.asarray(x) - y).max() / max(np.abs(y).max(), 1e-300)
    g_sh = torch.cat((g_a["feature_dc"], g_a["feature_rest"]), 1).numpy()
    assert rel(g_sh, og["shs"]) < tol
    assert not np.any(og["shs"][:, (deg + 1) ** 2:, :])  # coefficients above the active degree: exactly zero
    assert rel(g_a["mean"].numpy(), og["means3D"]) < tol
    assert rel(m2_a.numpy(), og["means2D"]) < tol
    # the pre-activation parameters see the chain rule of the activations on top of the oracle's gradients
    assert rel(g_a["opacity_logit"].numpy(), og["opacities"] * (opac * (1 - opac)).numpy()) < tol
    assert rel(g_a["log_scale"].numpy(), og["scales"] * scl.numpy()) < tol
    assert rel(g_a["rotation"].numpy(), og["rotations"]) < tol


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

def _close(x, y, rel=1e-4):
    x, y = x.detach(), y.detach()
    return float((x - y).abs().max()) <= rel * float(y.abs().max()) + 1e-12


@pytest.mark.gpu
def test_mixed_pass_equals_the_single_source_renders(dev):
    """C ABI: sh_rows = P with a colour pointer set == the shs-only render, bit for bit; sh_rows = P_sh < P with colour
    rows holding the RGB their SH would produce == the all-RGB render (1e-4 max); the backward writes dL/dSH for the SH
    rows, zeros to dL/dcolors there, and a detached SH prefix (first_row >= sh_rows) needs no dL_dshs."""
    from exavatar_release_b200.plan import FramePlan
    from exavatar_release_b200.rasterizer import GaussianRasterizationSettings as GS
    from exavatar_release_b200.rasterizer import _make_scene
    from exavatar_release_b200.synthetic import make_assets
    wl = WORKLOADS["T2"]
    H, W = wl.height, wl.width
    a = {k: v.to(dev) for k, v in make_assets("T2", seed=4).items()}
    P, M, deg = a["mean_3d"].shape[0], 16, 3
    st = workload_settings("T2", yaw=-4.0, device=dev, settings_cls=GS)._replace(sh_degree=deg)
    rgb_of_sh = sh_to_rgb(deg, a["shs"], a["mean_3d"], st.campos).contiguous()  # fp32, what K1 evaluates
    gi = make_grad_image("T2", 3).to(dev)
    plan = FramePlan(P, W, H, 2_000_000, dev, sh_coeffs=M)

    def run(shs, colors, sh_rows, first_row=0, with_dshs=True):
        sc, keep = _make_scene(st, a["mean_3d"], shs, colors, a["opacity"], a["scale"], a["rotation"], None, 0)
        sc.sh_rows = sh_rows
        plan.forward(sc)
        rows = P - first_row
        g = {k: torch.full((rows, w), float("nan"), device=dev) for k, w in
             (("means3D", 3), ("means2D", 3), ("opacities", 1), ("scales", 3), ("rotations", 4), ("colors", 3))}
        n_sh = max(0, (sh_rows if sh_rows else (P if shs is not None else 0)) - first_row)
        if with_dshs and n_sh:
            g["shs"] = torch.full((n_sh, M, 3), float("nan"), device=dev)
        plan.backward(sc, gi, g, first_row=first_row)
        torch.cuda.synchronize()
        del keep
        return plan.color.clone(), plan.radii.clone(), g

    img_sh, rad_sh, g_sh = run(a["shs"], None, 0)
    img_rgb, rad_rgb, g_rgb = run(None, rgb_of_sh, 0)
    junk = torch.rand(P, 3, device=dev)  # never read: every row is an SH row
    img_m, rad_m, g_m = run(a["shs"], junk, P)
    assert torch.equal(rad_m, rad_sh) and torch.equal(img_m, img_sh)
    for k in ("means3D", "means2D", "opacities", "scales", "rotations", "shs"):
        assert _close(g_m[k], g_sh[k]), k  # K6's mixed instantiation may contract its arithmetic differently
    assert float(g_m["colors"].abs().max()) == 0.0  # every element written: zeros on SH rows

    for n_sh in (1234, 37):  # not a multiple of 32: one warp straddles the boundary
        colors = torch.where(torch.arange(P, device=dev)[:, None] < n_sh, junk, rgb_of_sh).contiguous()
        shs = a["shs"][:n_sh].contiguous()
        img, rad, g = run(shs, colors, n_sh)
        assert torch.equal(rad, rad_rgb)
        assert _close(img, img_rgb)
        for k in ("means2D", "opacities", "scales", "rotations"):
            assert _close(g[k], g_rgb[k]), (n_sh, k)
        # colour rows: the RGB render's gradients; SH rows: the SH render's (dL/dmean includes the view-direction term)
        assert _close(g["colors"][n_sh:], g_rgb["colors"][n_sh:]) and float(g["colors"][:n_sh].abs().max()) == 0.0
        assert _close(g["means3D"][n_sh:], g_rgb["means3D"][n_sh:])
        assert _close(g["means3D"][:n_sh], g_sh["means3D"][:n_sh])
        assert _close(g["shs"], g_sh["shs"][:n_sh])
        # detached prefix past the SH rows (pass B of the merged frame): no dL_dshs needed, rows land at i - first_row
        fr = n_sh + 5
        _, _, gb = run(shs, colors, n_sh, first_row=fr, with_dshs=False)
        assert _close(gb["means3D"], g_rgb["means3D"][fr:]) and _close(gb["colors"], g_rgb["colors"][fr:])
        # a detached prefix INSIDE the SH rows: dL_dshs has sh_rows - first_row rows
        fr = n_sh // 2
        _, _, gc = run(shs, colors, n_sh, first_row=fr)
        assert gc["shs"].shape[0] == n_sh - fr and _close(gc["shs"], g_sh["shs"][fr:n_sh])
        assert not torch.isnan(gc["means3D"]).any()


def _frame_inputs(wl_name, dev, seed=0):
    scene, human, refined = make_population_assets(wl_name, seed=seed, device=dev)
    p = make_scene_sh_params(scene, 3, seed=seed)
    return p, human, refined


def _leaves(p, human, refined):
    sp = {k: v.detach().clone().requires_grad_() for k, v in p.items()}
    hs = {k: v.detach().clone().requires_grad_() for k, v in human.items()}
    rs = {k: v.detach().clone().requires_grad_() for k, v in refined.items()}
    return sp, hs, rs


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("wl_name", ["T1", "C4"])
def test_training_frame_renderer_sh_scene_equals_caller_side_rgb(dev, wl_name, use_graph):
    """`TrainingFrameRenderer(sh_coeffs=16)` fed `scene_gaussian_assets(in_kernel_sh=True)` == the same renderer fed
    caller-side RGB (`in_kernel_sh=False`): radii / is_vis identical, images, masks and every gradient -- SH features,
    scene mean_3d (view-direction term included), opacity, scale, rotation, the human and refined sets, the scene
    mean_2d and the densification statistics -- within 1e-4 max.  Three frames with new cameras and SH degree 1 -> 3 -> 3;
    with use_graph the third frame is a pure replay."""
    from exavatar_release_b200 import TrainingFrameRenderer
    from exavatar_release_b200.plan import RENDERS
    lib = L.load()
    wl = WORKLOADS[wl_name]
    H, W = wl.height, wl.width
    p, human, refined = _frame_inputs(wl_name, dev)
    Ps, Ph = p["mean"].shape[0], human["mean_3d"].shape[0]
    bg_r = torch.tensor([0.3, 0.7, 0.2], device=dev)
    gcol = {r: make_grad_image(wl_name, 70 + j, device=dev) for j, r in enumerate(RENDERS)}
    gmask = make_grad_image(wl_name, 80, device=dev)[:1]
    caps = {"A": 2_000_000, "B": 2_000_000} if wl_name == "T1" else {"A": 8_000_000, "B": 8_000_000}
    fr = {sh: TrainingFrameRenderer(Ps, Ph, (H, W), dev, caps, use_graph=use_graph, graph_depth_alpha=use_graph,
                                    sh_coeffs=16 if sh else 0) for sh in (False, True)}
    dens = {sh: {k: torch.zeros(Ps, 1, device=dev) for k in ("grad_accum", "count", "radius_max")} for sh in (False, True)}
    for sh in fr:
        fr[sh].densify = dens[sh]
    for f, (yaw, deg) in enumerate(((-9.0, 1), (6.0, 3), (14.0, 3))):
        cam = look_at_cam_param(yaw, (H, W), device=dev)
        res = {}
        for sh in (False, True):
            sp, hs, rs = _leaves(p, human, refined)
            scene = scene_gaussian_assets(sp["mean"], sp["opacity_logit"], sp["log_scale"], sp["rotation"],
                                          sp["feature_dc"], sp["feature_rest"], deg, cam, in_kernel_sh=sh)
            torch.cuda.synchronize()
            n0 = lib.b2r_launch_count()
            out = fr[sh](scene, hs, rs, cam, bg_r)
            loss = sum((out[r]["img"] * gcol[r]).sum() for r in RENDERS) + (out["human"]["mask"] * gmask).sum()
            loss.backward()
            torch.cuda.synchronize()
            launches = lib.b2r_launch_count() - n0
            assert not fr[sh].overflowed()
            res[sh] = (out, sp, hs, rs, launches)
        (oa, spa, hsa, rsa, _), (ob, spb, hsb, rsb, launches) = res[False], res[True]
        if use_graph and f == 2:
            assert launches == 0, "third frame (same intrinsics, same SH degree) must replay the captured graphs"
        for r in RENDERS:
            assert torch.equal(ob[r]["radius"], oa[r]["radius"]) and torch.equal(ob[r]["is_vis"], oa[r]["is_vis"]), r
            assert _close(ob[r]["img"], oa[r]["img"]) and _close(ob[r]["mask"], oa[r]["mask"]), r
            assert _close(ob[r]["depthmap"], oa[r]["depthmap"]), r
        for k in spa:
            assert spb[k].grad is not None and _close(spb[k].grad, spa[k].grad), (f, "scene", k)
        assert float(spa["feature_rest"].grad.abs().max()) > 0
        for name, la, lb in (("human", hsa, hsb), ("refined", rsa, rsb)):
            for k in la:
                assert _close(lb[k].grad, la[k].grad), (f, name, k)
        assert _close(ob["scene"]["mean_2d"].grad, oa["scene"]["mean_2d"].grad)
        for k in dens[True]:
            assert _close(dens[True][k], dens[False][k]), k


@pytest.mark.gpu
def test_c4_sh_frame_vs_oracle_renders(dev):
    """BASELINE configs[3] with a degree-3 SH scene on MergedFivePlan(sh_coeffs=16), every view against its own oracle
    render (tests/parity.py bounds): the scene view against an oracle SH render, the human views against RGB renders,
    the combined views against renders of cat(sh_to_rgb(scene).detach(), human_rgb).  Gradients: the scene bucket
    (dL/dSH, dL/dmean with the view-direction term) is the scene render's; the human buckets add the human rows of
    the combined renders."""
    from parity import compare
    from exavatar_release_b200 import rasterizer as rz
    from exavatar_release_b200.plan import RENDERS, MergedFivePlan
    wl = WORKLOADS["C4"]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets("C4", seed=0)
    p = make_scene_sh_params(scene, 3, seed=0)
    shs = torch.cat((p["feature_dc"], p["feature_rest"]), 1).contiguous()
    Ps, Ph = scene["mean_3d"].shape[0], human["mean_3d"].shape[0]
    bg_w, bg_r = torch.ones(3), torch.tensor([0.3, 0.7, 0.2])
    cam = look_at_cam_param(-6.0, (H, W))
    st_w, st_r = (render_settings((H, W), cam, b, O.OracleSettings) for b in (bg_w, bg_r))
    gcol = {r: make_grad_image("C4", 40 + j) for j, r in enumerate(RENDERS)}
    scene_rgb = sh_to_rgb(3, shs.double(), scene["mean_3d"].double(), st_w.campos.double()).float()
    cat = lambda a, b: {k: torch.cat((a[k], b[k])) for k in a}
    sc_rgb = dict(scene, rgb=scene_rgb)
    sets = {"human": (human, st_r), "scene_human": (cat(sc_rgb, human), st_w), "human_refined": (refined, st_r),
            "scene_human_refined": (cat(sc_rgb, refined), st_w)}
    ora = {}
    oc, orad, _, oa, octx = O.forward(st_w._replace(sh_degree=3), scene["mean_3d"], scene["opacity"], shs=shs,
                                      scales=scene["scale"], rotations=scene["rotation"])
    ora["scene"] = dict(color=oc, radii=orad, alpha=oa, grads=O.backward(octx, gcol["scene"].numpy()), frag=O.fragility(octx))
    for r, (a, st) in sets.items():
        oc, orad, _, oa, octx = O.forward(st, a["mean_3d"], a["opacity"], colors_precomp=a["rgb"], scales=a["scale"],
                                          rotations=a["rotation"])
        ora[r] = dict(color=oc, radii=orad, alpha=oa, grads=O.backward(octx, gcol[r].numpy()), frag=O.fragility(octx))

    to = lambda d: {k: v.to(dev) for k, v in d.items()}
    plan = MergedFivePlan(Ps, Ph, W, H, None, dev, sh_coeffs=16)
    sc_dev = dict(to({k: v for k, v in scene.items() if k != "rgb"}), shs=shs.to(dev), sh_degree=3)
    plan.set_scene(sc_dev)
    st_wg = settings_on(st_w, dev, rz.GaussianRasterizationSettings)
    st_rg = settings_on(st_r, dev, rz.GaussianRasterizationSettings)
    plan.frame(0, st_wg, st_rg, sc_dev, to(human), to(refined), {r: g.to(dev) for r, g in gcol.items()}, accumulate=False)
    torch.cuda.synchronize()
    assert not plan.overflowed()
    for r in RENDERS:
        pm, _ = ora[r]["frag"]
        img, alpha, radii = plan.render_outputs(r)
        assert np.array_equal(radii.cpu().numpy(), ora[r]["radii"]), r
        compare("C4-sh/" + r, "color", img.cpu().numpy(), ora[r]["color"], pm[None], kind="image")
        compare("C4-sh/" + r, "alpha", alpha.cpu().numpy(), ora[r]["alpha"], pm[None], kind="image")
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

    views = plan.grads("scene")
    assert "colors" not in views and tuple(views["shs"].shape) == (Ps, 16, 3)
    y, flag = expect([("scene", slice(0, Ps))], common + ("shs",))
    for k in common + ("shs",):
        compare("C4-sh/scene", "d_" + k, views[k].cpu().numpy().reshape(Ps, -1), y[k], flag[:, None], kind="grad")
    for label, parts in (("human", [("human", slice(0, Ph)), ("scene_human", slice(Ps, Ps + Ph))]),
                         ("human_refined", [("human_refined", slice(0, Ph)), ("scene_human_refined", slice(Ps, Ps + Ph))])):
        views = plan.grads(label)
        y, flag = expect(parts, common + ("colors",))
        for k in common + ("colors",):
            compare("C4-sh/" + label, "d_" + k, views[k].cpu().numpy().reshape(Ph, -1), y[k], flag[:, None], kind="grad")
