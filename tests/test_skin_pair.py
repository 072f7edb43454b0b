"""Standalone skinning of both human Gaussian sets (SURVEY.md section 8f-2): `skinning.skin_gaussians` / B2RSkin.

ExAvatar poses `mean_3d` and `mean_3d_refined` with one rig (avatar/common/nets/module.py:549-557) before anything is
rendered.  These tests pin
  * the C ABI (struct layout, exported symbols, host-side validation) and a float64 restatement of the backward
    formulas against autograd through `renderer.lbs_reference`, without a device;
  * on the GPU at C4 human size: posed positions against lbs_reference, bit-identity with the fifth output of
    `SkinnedGaussianRasterizer`, gradients against float64 autograd, bit-reproducible backward, CUDA-graph capture,
    and one C4 training frame through `TrainingFrameRenderer` posed by the op vs. by the unfused ops.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from util import workload_settings  # noqa: F401  (path setup)
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.camera import look_at_cam_param
from exavatar_release_b200.renderer import lbs_reference, render_settings
from exavatar_release_b200.synthetic import WORKLOADS, make_grad_image, make_population_assets
from test_fused_skinning import _close, _rig

FAKE = 0x1000  # never dereferenced: validation fails before any launch
J = 55


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

def test_skin_struct_layout_and_symbols():
    lib = L.load()
    assert lib.b2r_abi_version() == 4
    raw = C.CDLL(L.LIB_PATH)
    for name in ("b2r_skin_forward", "b2r_skin_backward", "b2r_skin_scratch_bytes"):
        assert hasattr(raw, name), name
        assert name in {s[0] for s in L.SYMBOLS}, name
    # one (J*12 + 3)-float partial per 256 Gaussians, at least
    assert lib.b2r_skin_scratch_bytes(167000, 55) >= ((167000 + 255) // 256) * (55 * 12 + 3) * 4
    assert lib.b2r_skin_scratch_bytes(0, 55) > 0


def _valid_skin(P=64):
    s = L.B2RSkin()
    s.P, s.J, s.V = P, J, 100
    s.weights = s.rows = s.joint_mats = s.trans = s.cam_Rinv = s.cam_t = FAKE
    s.xyz[0] = s.xyz[1] = s.posed[0] = s.posed[1] = FAKE
    return s


def test_skin_validation_without_touching_cuda():
    lib = L.load()
    n0 = lib.b2r_launch_count()
    fwd = lambda s: lib.b2r_skin_forward(C.byref(s), None)
    g = (C.c_void_p * 2)(FAKE, FAKE)
    d = (C.c_void_p * 2)(FAKE, FAKE)
    bwd = lambda s, g=g, scratch=FAKE, nbytes=1: lib.b2r_skin_backward(C.byref(s), g, d, FAKE, FAKE, scratch, nbytes,
                                                                        None)
    cases = {
        "null struct": None,
        "weights": ("weights", None), "joint_mats": ("joint_mats", None), "trans": ("trans", None),
        "J = 0": ("J", 0), "J < 0": ("J", -3), "J = 65": ("J", 65), "V = 0": ("V", 0), "V < 0": ("V", -1),
        "P < 0": ("P", -1), "cam_Rinv without cam_t": ("cam_t", None),
    }
    for what, change in cases.items():
        if change is None:
            assert lib.b2r_skin_forward(None, None) == -1
            assert lib.b2r_skin_backward(None, g, d, FAKE, FAKE, FAKE, 1 << 30, None) == -1
            continue
        s = _valid_skin()
        setattr(s, *change)
        assert fwd(s) == -1, what
        assert bwd(s) == -1, what
    s = _valid_skin()
    s.xyz[0] = None
    assert fwd(s) == -1 and bwd(s) == -1
    s = _valid_skin()
    s.posed[0] = None
    assert fwd(s) == -1                                    # the forward's output
    s = _valid_skin()
    s.xyz[1] = None
    assert fwd(s) == -1 and bwd(s) == -1                   # posed[1] without xyz[1]
    s.posed[1] = None
    assert bwd(s) == -1                                    # dL_dpos[1] without xyz[1]
    s = _valid_skin()
    s.rows, s.V = None, 63
    assert fwd(s) == -1                                    # row i of the table without `rows`: V >= P
    s = _valid_skin()
    assert bwd(s, scratch=None, nbytes=1 << 30) == -1      # joint / translation gradient needs the scratch
    assert bwd(s, nbytes=8) == -2                          # ... of b2r_skin_scratch_bytes
    assert lib.b2r_launch_count() == n0                    # nothing was launched by any of the above


def _skin_backward_f64(xyz_sets, w, A, trans, Rinv, g_sets):
    """The formulas of b2r_skin_backward in float64: g_cam = Rinv^T g, dL/dx = M3^T g_cam,
    dL/dA_j[:3,:] = sum_i w_ij sum_s g_cam [x, 1]^T, dL/dtrans = sum_i sum_s g_cam."""
    M = (w @ A.reshape(-1, 16)).reshape(-1, 4, 4)[:, :3, :]  # (P,3,4)
    dA = torch.zeros(A.shape[0], 3, 4, dtype=torch.float64)
    dtrans = torch.zeros(3, dtype=torch.float64)
    dxs = []
    for x, g in zip(xyz_sets, g_sets):
        gc = g @ Rinv if Rinv is not None else g  # row i: (Rinv^T g_i)^T = g_i^T Rinv
        dxs.append(torch.einsum("prc,pr->pc", M[:, :, :3], gc))
        x1 = torch.cat((x, torch.ones_like(x[:, :1])), 1)
        dA += torch.einsum("pj,pr,pc->jrc", w, gc, x1)
        dtrans += gc.sum(0)
    return dxs, dA, dtrans


@pytest.mark.parametrize("world", [True, False])
def test_f64_restatement_of_the_backward_matches_autograd(world):
    """The reference the GPU backward is held to: the kernel's formulas in float64 == autograd through lbs_reference on
    two sets sharing a rig, with weight rows looked up through a row index."""
    P, V = 300, 250
    table, A, trans = _rig(V, J, torch.float64, "cpu")
    g = torch.Generator().manual_seed(2)
    rows = torch.randint(0, V, (P,), generator=g)
    rows[:40] = torch.arange(40)  # rows mapped to themselves (hands / face in ExAvatar)
    w = table[rows]
    xs = [torch.randn(P, 3, generator=g, dtype=torch.float64) for _ in range(2)]
    gs = [torch.randn(P, 3, generator=g, dtype=torch.float64) for _ in range(2)]
    cam = look_at_cam_param(10.0, (96, 128))
    R, t = (cam["R"].double(), cam["t"].double()) if world else (None, None)
    lx = [x.clone().requires_grad_() for x in xs]
    lA, lt = A.clone().requires_grad_(), trans.clone().requires_grad_()
    loss = sum((lbs_reference(x, w, lA, lt, R, t) * gg).sum() for x, gg in zip(lx, gs))
    loss.backward()
    dxs, dA, dtrans = _skin_backward_f64(xs, w, A, trans, torch.inverse(R) if world else None, gs)
    for a, b in zip(dxs, lx):
        assert torch.allclose(a, b.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(dA, lA.grad[:, :3, :], rtol=1e-12, atol=1e-12)
    assert float(lA.grad[:, 3, :].abs().max()) == 0.0
    assert torch.allclose(dtrans, lt.grad, rtol=1e-12, atol=1e-12)


def test_skin_gaussians_rejects_cpu_tensors():
    from exavatar_release_b200.skinning import skin_gaussians
    w, A, trans = _rig(8, J, torch.float32, "cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        skin_gaussians(torch.zeros(8, 3), None, w, None, A, trans)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _c4_rig(dev, world=True):
    """C4 human size: P = 167 000 Gaussians, a (V = P, 55) 4-sparse weight table read through `rows` (a random row
    for most Gaussians, its own row for the first 20 000 -- ExAvatar maps hand and face Gaussians to themselves)."""
    wl = WORKLOADS["C4"]
    H, W = wl.height, wl.width
    _, human, refined = make_population_assets("C4", seed=0, device=dev)
    P = human["mean_3d"].shape[0]
    table, A, trans = _rig(P, J, torch.float32, dev)
    g = torch.Generator().manual_seed(9)
    rows = torch.randint(0, P, (P,), generator=g)
    rows[:20000] = torch.arange(20000)
    rows = rows.to(dev)
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    if world:  # canonical positions in the frame the skinning works in; R^-1 (. - t) brings them back to the scene
        xyz = human["mean_3d"] @ cam["R"].t() + cam["t"].view(1, 3)
        xyz_r = refined["mean_3d"] @ cam["R"].t() + cam["t"].view(1, 3)
        R, t = cam["R"], cam["t"]
    else:
        xyz, xyz_r, R, t = human["mean_3d"].clone(), refined["mean_3d"].clone(), None, None
    return dict(xyz=xyz.contiguous(), xyz_r=xyz_r.contiguous(), table=table, rows=rows, A=A, trans=trans, R=R, t=t,
                cam=cam, human=human, refined=refined, H=H, W=W)


def _f64_ref(rig, xs):
    w = rig["table"].double()[rig["rows"]]
    R = None if rig["R"] is None else rig["R"].double()
    t = None if rig["t"] is None else rig["t"].double()
    return [lbs_reference(x.double(), w, rig["A"].double(), rig["trans"].double(), R, t) for x in xs]


@pytest.mark.gpu
@pytest.mark.parametrize("world", [True, False])
def test_posed_positions_match_lbs_reference(dev, world):
    from exavatar_release_b200.skinning import skin_gaussians
    rig = _c4_rig(dev, world)
    with torch.no_grad():
        posed, posed_r = skin_gaussians(rig["xyz"], rig["xyz_r"], rig["table"], rig["rows"], rig["A"], rig["trans"],
                                        rig["R"], rig["t"])
        one, none = skin_gaussians(rig["xyz"], None, rig["table"], rig["rows"], rig["A"], rig["trans"], rig["R"], rig["t"])
    torch.cuda.synchronize()
    assert none is None and torch.equal(one, posed)  # one set or two: the same blend
    for got, ref in zip((posed, posed_r), _f64_ref(rig, (rig["xyz"], rig["xyz_r"]))):
        lim = 1e-6 * float(ref.abs().max())
        assert float((got.double() - ref).abs().max()) <= lim


@pytest.mark.gpu
def test_posed_positions_equal_the_fused_rasteriser_bit_for_bit(dev):
    """The op and SkinnedGaussianRasterizer's fifth output write the same bits, for both sets."""
    from exavatar_release_b200 import rasterizer as RZ
    from exavatar_release_b200.skinning import skin_gaussians
    rig = _c4_rig(dev)
    st = render_settings((rig["H"], rig["W"]), rig["cam"], torch.tensor([0.2, 0.4, 0.9], device=dev))
    h = rig["human"]
    P = h["mean_3d"].shape[0]
    w_gathered = rig["table"][rig["rows"]].contiguous()
    with torch.no_grad():
        posed, posed_r = skin_gaussians(rig["xyz"], rig["xyz_r"], rig["table"], rig["rows"], rig["A"], rig["trans"],
                                        rig["R"], rig["t"])
        for x, mine in ((rig["xyz"], posed), (rig["xyz_r"], posed_r)):
            fused = RZ.SkinnedGaussianRasterizer(st)(x, w_gathered, rig["A"], rig["trans"], rig["R"], rig["t"],
                                                     torch.zeros(P, 3, device=dev), h["opacity"], h["rgb"], h["scale"],
                                                     h["rotation"])[4]
            torch.cuda.synchronize()
            assert torch.equal(fused, mine)


def _grads_of(rig, dev, two, gp, gq):
    from exavatar_release_b200.skinning import skin_gaussians
    x = rig["xyz"].clone().requires_grad_()
    xr = rig["xyz_r"].clone().requires_grad_() if two else None
    A = rig["A"].clone().requires_grad_()
    tr = rig["trans"].clone().requires_grad_()
    posed, posed_r = skin_gaussians(x, xr, rig["table"], rig["rows"], A, tr, rig["R"], rig["t"])
    loss = (posed * gp).sum() + ((posed_r * gq).sum() if two else 0.0)
    loss.backward()
    out = {"xyz": x.grad, "A": A.grad, "trans": tr.grad}
    if two:
        out["xyz_r"] = xr.grad
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("two", [False, True])
@pytest.mark.parametrize("world", [True, False])
def test_gradients_match_f64_autograd(dev, two, world):
    rig = _c4_rig(dev, world)
    P = rig["xyz"].shape[0]
    g = torch.Generator().manual_seed(4)
    gp, gq = torch.randn(P, 3, generator=g).to(dev), torch.randn(P, 3, generator=g).to(dev)
    got = _grads_of(rig, dev, two, gp, gq)
    torch.cuda.synchronize()
    # float64 autograd through the unfused ops
    lx = [rig["xyz"].double().requires_grad_()] + ([rig["xyz_r"].double().requires_grad_()] if two else [])
    lA, lt = rig["A"].double().requires_grad_(), rig["trans"].double().requires_grad_()
    w = rig["table"].double()[rig["rows"]]
    R = None if rig["R"] is None else rig["R"].double()
    t = None if rig["t"] is None else rig["t"].double()
    loss = sum((lbs_reference(x, w, lA, lt, R, t) * gg.double()).sum() for x, gg in zip(lx, (gp, gq)))
    loss.backward()
    ref = {"xyz": lx[0].grad, "A": lA.grad, "trans": lt.grad}
    if two:
        ref["xyz_r"] = lx[1].grad
    for k, r in ref.items():
        d = float((got[k].double() - r).abs().max())
        assert d <= 1e-5 * float(r.abs().max()), (k, d, float(r.abs().max()))
    assert float(got["A"][:, 3, :].abs().max()) == 0.0


@pytest.mark.gpu
def test_backward_is_bit_reproducible(dev):
    rig = _c4_rig(dev)
    P = rig["xyz"].shape[0]
    g = torch.Generator().manual_seed(6)
    gp, gq = torch.randn(P, 3, generator=g).to(dev), torch.randn(P, 3, generator=g).to(dev)
    a = _grads_of(rig, dev, True, gp, gq)
    b = _grads_of(rig, dev, True, gp, gq)
    torch.cuda.synchronize()
    for k in a:
        assert torch.equal(a[k], b[k]), k


@pytest.mark.gpu
def test_forward_and_backward_capture_in_a_cuda_graph(dev):
    """Forward + backward captured once; a replay with new joint transforms / translation copied into the captured
    leaves equals an eager run on those values, bit for bit (no torch.inverse, no host synchronisation inside)."""
    from exavatar_release_b200.skinning import skin_gaussians
    rig = _c4_rig(dev)
    P = rig["xyz"].shape[0]
    g = torch.Generator().manual_seed(8)
    gp, gq = torch.randn(P, 3, generator=g).to(dev), torch.randn(P, 3, generator=g).to(dev)
    x = rig["xyz"].clone().requires_grad_()
    xr = rig["xyz_r"].clone().requires_grad_()
    A = rig["A"].clone().requires_grad_()
    tr = rig["trans"].clone().requires_grad_()

    def step():
        posed, posed_r = skin_gaussians(x, xr, rig["table"], rig["rows"], A, tr, rig["R"], rig["t"])
        loss = (posed * gp).sum() + (posed_r * gq).sum()
        return (posed.detach(), posed_r.detach()) + torch.autograd.grad(loss, (x, xr, A, tr))

    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        step()  # warm-up outside the capture
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_out = step()
    _, A2, tr2 = _rig(P, J, torch.float32, dev, seed=17)
    tr2 = tr2 + 0.05
    with torch.no_grad():
        A.copy_(A2)
        tr.copy_(tr2)
    graph.replay()
    torch.cuda.synchronize()
    replayed = [t.clone() for t in static_out]
    eager = step()
    torch.cuda.synchronize()
    names = ("posed", "posed_refined", "d_xyz", "d_xyz_refined", "d_joint", "d_trans")
    for name, a, b in zip(names, replayed, eager):
        assert torch.equal(a, b), name
    # and the replay did see the new rig
    ref = _f64_ref(dict(rig, A=A2, trans=tr2), (rig["xyz"],))[0]
    assert float((replayed[0].double() - ref).abs().max()) <= 1e-6 * float(ref.abs().max())


@pytest.mark.gpu
def test_c4_training_frame_posed_by_the_op(dev):
    """One C4 frame through TrainingFrameRenderer with both human sets posed by skin_gaussians, against the same frame
    posed by ExAvatar's unfused ops (lbs_reference).
      * "ops_st": the op's posed values with the gradient routed through lbs_reference (straight-through): identical
        renders and dL/dposed, so the images are bit-identical and the gradients at xyz, xyz_refined, joint_mats and
        trans meet the full tolerance of test_fused_skinning._close -- the op's backward behind the real frame.
      * "ops": posed by lbs_reference alone.  The two paths round the positions differently (a dense GEMM vs. the
        sparse blend, ~1e-7 relative), which can swap the depth order of two near-coincident splats: a few pixels and
        the gradient of a single Gaussian then move by a lot (seen: 9 % of max|dL/dxyz| on one element of 167 k).  So
        here only the outlier fraction of _close is held (<= 0.2 % of the elements beyond 1e-4 * max), for the images
        and the per-Gaussian gradients.
      * every image of the op-posed frame is held to the parity bounds of tests/parity.py against the CPU oracle
        rendering the same posed positions."""
    from parity import compare
    from exavatar_release_b200 import TrainingFrameRenderer
    from exavatar_release_b200.plan import RENDERS
    from exavatar_release_b200.skinning import skin_gaussians
    from oracle import oracle as O
    rig = _c4_rig(dev)
    H, W = rig["H"], rig["W"]
    scene, _, _ = make_population_assets("C4", seed=0, device=dev)
    human, refined = rig["human"], rig["refined"]
    Ps, Ph = scene["mean_3d"].shape[0], human["mean_3d"].shape[0]
    bg_r = torch.tensor([0.3, 0.7, 0.2], device=dev)
    gcol = {r: make_grad_image("C4", 90 + j, device=dev) for j, r in enumerate(RENDERS)}
    fr = TrainingFrameRenderer(Ps, Ph, (H, W), dev, {"A": 8_000_000, "B": 8_000_000})
    w_gathered = rig["table"][rig["rows"]]
    res = {}
    fused_values = None
    for arm in ("fused", "ops_st", "ops"):
        x = rig["xyz"].clone().requires_grad_()
        xr = rig["xyz_r"].clone().requires_grad_()
        A = rig["A"].clone().requires_grad_()
        tr = rig["trans"].clone().requires_grad_()
        if arm == "fused":
            posed, posed_r = skin_gaussians(x, xr, rig["table"], rig["rows"], A, tr, rig["R"], rig["t"])
            fused_values = (posed.detach().clone(), posed_r.detach().clone())
        else:
            posed = lbs_reference(x, w_gathered, A, tr, rig["R"], rig["t"])
            posed_r = lbs_reference(xr, w_gathered, A, tr, rig["R"], rig["t"])
            if arm == "ops_st":  # value: the op's positions exactly (x - x == 0); gradient: through lbs_reference
                posed = fused_values[0] + (posed - posed.detach())
                posed_r = fused_values[1] + (posed_r - posed_r.detach())
        out = fr(scene, dict(human, mean_3d=posed), dict(refined, mean_3d=posed_r), rig["cam"], bg_r)
        sum((out[r]["img"] * gcol[r]).sum() for r in RENDERS).backward()
        torch.cuda.synchronize()
        assert not fr.overflowed()
        res[arm] = ({r: out[r]["img"].detach().clone() for r in RENDERS},
                    {"xyz": x.grad, "xyz_refined": xr.grad, "joint_mats": A.grad, "trans": tr.grad})
    img_b, g_b = res["fused"]
    img_st, g_st = res["ops_st"]
    img_a, g_a = res["ops"]
    assert float(g_b["joint_mats"][:, 3, :].abs().max()) == 0.0
    for r in RENDERS:
        assert float(img_b[r].abs().max()) > 0.1, r
        assert torch.equal(img_st[r], img_b[r]), r
    for k in g_st:
        assert float(g_st[k].abs().max()) > 0, k
        _close(k, g_b[k], g_st[k])

    def outliers_only(name, x, y):  # the outlier criterion of _close without its max bound
        frac = float(((x - y).abs() > 1e-4 * float(y.abs().max())).float().mean())
        assert frac <= 2e-3, (name, frac)

    for r in RENDERS:
        outliers_only("image " + r, img_b[r], img_a[r])
    for k in ("xyz", "xyz_refined"):
        outliers_only(k, g_b[k], g_a[k])
    hp, rp = (v.cpu() for v in fused_values)

    # the op-posed frame against the oracle's renders of the same posed positions
    cpu = lambda d: {k: v.detach().cpu() for k, v in d.items()}
    cam_c = look_at_cam_param(-6.0, (H, W))
    st_w = render_settings((H, W), cam_c, torch.ones(3), O.OracleSettings)
    st_r = render_settings((H, W), cam_c, bg_r.cpu(), O.OracleSettings)
    sc, hs, rs = cpu(scene), dict(cpu(human), mean_3d=hp), dict(cpu(refined), mean_3d=rp)
    cat = lambda a, b: {k: torch.cat((a[k], b[k])) for k in a}
    sets = {"scene": (sc, st_w), "human": (hs, st_r), "scene_human": (cat(sc, hs), st_w), "human_refined": (rs, st_r),
            "scene_human_refined": (cat(sc, rs), st_w)}
    for r, (a, st) in sets.items():
        oc, _, _, _, octx = O.forward(st, a["mean_3d"], a["opacity"], colors_precomp=a["rgb"], scales=a["scale"],
                                      rotations=a["rotation"])
        pm, _ = O.fragility(octx)
        compare("C4-skin-pair/" + r, "color", img_b[r].cpu().numpy(), oc, pm[None], kind="image")
