"""ExAvatar's regulariser block (avatar/main/model.py:217-257) as the sync-free CUDA op `HumanRegularizers`
(csrc/regularizers.cu, b2r_regs_*).

These tests pin
  * without a device: `human_regularizers_reference` against tests/golden/regs.npz (made by the reference's own loss
    classes, get_arm and model.py lines), the Laplacian table against LaplacianReg's on the synthetic C4 mesh (108-
    neighbour poles truncated to 10), the weight columns against model.py's, and the C ABI and argument checks;
  * on the GPU at C4 size (P = 167 618): every term against float64, every gradient against float64 autograd, the arm
    selection against the reference's, small windows (k < 50, k = 0, no lower row), bit-identical runs, no host sync,
    forward + backward replayed from one CUDA graph with a new mesh, and the f-7 human chain followed by the op.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from util import capture, golden_generator, no_host_sync
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.geometry import vertex_normals_reference
from exavatar_release_b200.regularizers import (KEYS, arm_selection_reference, human_regularizers_reference,
                                                laplacian_table, make_tables, weight_columns)
from exavatar_release_b200.synthetic import make_human_mesh, make_regs_labels

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FAKE = 0x1000  # never dereferenced: validation fails before any launch
P_C4 = 167618
INPUTS = ("mean_offset", "mean_offset_offset", "scale_offset", "scale", "scale_refined", "rgb", "rgb_refined",
          "joint_offset")


# SMPL-X's joint names as the golden generator read them from the reference (avatar/common/utils/smpl_x.py)
JOINTS = tuple(str(n) for n in np.load(os.path.join(G, "regs.npz"))["joints_name"])


def _case(names=JOINTS):
    return golden_generator("make_regs_golden").regs_inputs(list(names))


def _kink_row(labels):
    """The hand row `pin_kinks` gives a zero mean_offset: its gradient is n / 1e-12 and is compared on its own."""
    return int(torch.nonzero(labels["is_rhand"])[0])


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

def test_restatement_reproduces_the_reference_golden():
    mesh, labels, ins, target, hand_joints, pairs = _case()
    gold = np.load(os.path.join(G, "regs.npz"))
    leaves = {k: v.clone().requires_grad_() for k, v in ins.items()}
    args = [leaves[k] for k in INPUTS]
    kw = dict(labels, joint_offset_target=target, hand_joints=hand_joints, sym_pairs=pairs)
    out = human_regularizers_reference(mesh["faces"], mesh["verts"], *args, **kw)
    for k in KEYS:
        ref = float(gold[f"term:{k}"])
        assert abs(float(out[k].detach()) - ref) <= 1e-12 * abs(ref), (k, float(out[k].detach()), ref)
    sum(out.values()).backward()
    row = _kink_row(labels)
    for k in INPUTS:
        flat = leaves[k].grad.reshape(-1).numpy().copy()
        if k == "mean_offset":  # HandMeanReg's dot is exactly 0 there: clamp passes n / eps
            kink = flat[3 * row:3 * row + 3]
            np.testing.assert_allclose(kink, gold["kink_grad:mean_offset"], rtol=1e-12)
            assert np.abs(kink).max() > 1e8
            flat[3 * row:3 * row + 3] = 0.0
        scale = max(1.0, float(gold[f"grad_abs:{k}"]))
        np.testing.assert_allclose(flat[gold[f"grad_idx:{k}"]], gold[f"grad_val:{k}"], rtol=0, atol=1e-12 * scale,
                                   err_msg=k)
        np.testing.assert_allclose(np.abs(flat).sum(), gold[f"grad_abs:{k}"], rtol=1e-12, err_msg=k)
    # the warm-up's scale_wo_clamp replaces `scale` in gaussian_scale_reg
    sw = ins["scale_wo_clamp"].clone().requires_grad_()
    warm = human_regularizers_reference(mesh["faces"], mesh["verts"], *[ins[k] for k in INPUTS], scale_reg=sw, **kw)
    ref = float(gold["warmup_gaussian_scale_reg"])
    assert abs(float(warm["gaussian_scale_reg"]) - ref) <= 1e-12 * ref
    warm["gaussian_scale_reg"].backward()
    np.testing.assert_allclose(sw.grad.reshape(-1).numpy()[gold["grad_idx:scale_wo_clamp"]],
                               gold["grad_val:scale_wo_clamp"], rtol=0, atol=1e-15)
    normals = vertex_normals_reference(mesh["verts"], mesh["faces"], dtype=torch.float32)
    _, _, k, _ = arm_selection_reference(mesh["verts"], normals, labels["is_arm"])
    assert 0 < k < 50 and int(gold["n_lower"]) > 0  # the golden case exercises a window below the cap


def test_laplacian_table_is_the_reference_table_on_the_c4_mesh():
    gm = golden_generator("make_regs_golden")
    gold = np.load(os.path.join(G, "regs.npz"))
    m = make_human_mesh()
    idx, w = laplacian_table(m["faces"].numpy(), P_C4)
    assert gm.table_digest(idx, w) == str(gold["c4_table_sha256"])
    poles = gold["c4_pole_rows"]
    np.testing.assert_array_equal(idx[poles], gold["c4_pole_idx"])
    np.testing.assert_array_equal(w[poles], gold["c4_pole_w"])
    assert (w[poles] == np.float32(-0.1)).all()  # 108 neighbours, the reference keeps 10


def test_weight_columns_are_model_py_s():
    mesh, labels, *_ = _case()
    gold = np.load(os.path.join(G, "regs.npz"))
    P = mesh["verts"].shape[0]
    w = weight_columns(P, labels["is_rhand"], labels["is_lhand"], labels["is_face"], labels["is_face_expr"],
                       labels["is_cavity"])
    np.testing.assert_array_equal(w.numpy(), gold["weights"])
    assert bool((labels["is_rhand"] & labels["is_face"]).any())  # a later assignment overwrites an earlier one


def test_tables_reject_unequal_hands_and_bad_joints():
    mesh, labels, ins, target, hand_joints, pairs = _case()
    P = mesh["verts"].shape[0]
    kw = dict(labels, joint_offset_target=target, hand_joints=hand_joints, sym_pairs=pairs, nbr=(None, None))
    lh = labels["is_lhand"].clone()
    lh[torch.nonzero(~lh)[0]] = True
    with pytest.raises(ValueError, match="equal counts"):
        make_tables(None, P, **dict(kw, is_lhand=lh))
    with pytest.raises(ValueError, match="joint ids"):
        make_tables(None, P, **dict(kw, hand_joints=[99]))
    with pytest.raises(ValueError, match="sym_pairs"):
        make_tables(None, P, **dict(kw, sym_pairs=([1], [])))


def test_abi_symbols_structs_and_validation_without_touching_cuda():
    lib = L.load()
    raw = C.CDLL(L.LIB_PATH)
    for name in ("b2r_regs_scratch_bytes", "b2r_regs_forward", "b2r_regs_backward"):
        assert hasattr(raw, name) and name in {s[0] for s in L.SYMBOLS}, name
    assert C.sizeof(L.B2RRegs) == 32 + 8 * 25
    assert C.sizeof(L.B2RRegsGrads) == 8 * 9
    # the scratch holds the normals and six Laplacians per vertex, and grows with the arm capacity
    assert lib.b2r_regs_scratch_bytes(P_C4, 0) >= 21 * 4 * P_C4
    assert lib.b2r_regs_scratch_bytes(P_C4, 8000) > lib.b2r_regs_scratch_bytes(P_C4, 0)
    n0 = lib.b2r_launch_count()
    ptrs = [f[0] for f in L.B2RRegs._fields_ if f[1] is L._fp and f[0] != "scale_reg"]

    def regs(**kw):
        r = L.B2RRegs(P=64, J=55, n_arm=8, n_pairs=26, n_hand=10, n_rhand=5, **{p: FAKE for p in ptrs})
        for k, v in kw.items():
            setattr(r, k, v)
        return r

    need = lib.b2r_regs_scratch_bytes(64, 8)
    grads = L.B2RRegsGrads(*[FAKE] * 9)
    for kw in ({"P": 0}, {"J": 0}, {"J": 257}, {"n_arm": 65}, {"n_arm": -1}, {"n_pairs": 0}, {"n_hand": 65},
               {"mesh": None}, {"rgb_refined": None}, {"lapT_w": None}, {"arm_idx": None}, {"sym_pairs": None}):
        r = regs(**kw)
        assert lib.b2r_regs_forward(C.byref(r), FAKE, FAKE, need, None) == -1, kw
        assert lib.b2r_regs_backward(C.byref(r), FAKE, C.byref(grads), FAKE, need, None) == -1, kw
    r = regs()
    assert lib.b2r_regs_forward(None, FAKE, FAKE, need, None) == -1
    assert lib.b2r_regs_forward(C.byref(r), None, FAKE, need, None) == -1
    assert lib.b2r_regs_forward(C.byref(r), FAKE, FAKE, need - 1, None) == -2
    assert lib.b2r_regs_backward(C.byref(r), FAKE, C.byref(grads), FAKE, need - 1, None) == -2
    assert lib.b2r_regs_backward(C.byref(r), None, C.byref(grads), FAKE, need, None) == -1
    g2 = L.B2RRegsGrads(*[FAKE] * 9)
    g2.rgb = None
    assert lib.b2r_regs_backward(C.byref(r), FAKE, C.byref(g2), FAKE, need, None) == -1
    g2.rgb, g2.scale_reg = FAKE, None
    r.scale_reg = FAKE  # a scale_reg input needs its gradient
    assert lib.b2r_regs_backward(C.byref(r), FAKE, C.byref(g2), FAKE, need, None) == -1
    assert lib.b2r_launch_count() == n0


def test_op_rejects_bad_inputs_before_any_launch():
    from exavatar_release_b200.regularizers import _rows
    with pytest.raises(ValueError, match=r"\(64,3\)"):
        _rows("rgb", torch.zeros(2, 64, 3), 64, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        _rows("rgb", torch.zeros(64, 3), 64, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        _rows("scale_offset", torch.zeros(1, 64), 64, 1)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

_CACHE = {}


def _c4(dev, **label_kw):
    """The synthetic C4 mesh, its labels, a HumanRegularizers over them and seeded fp32 inputs."""
    from exavatar_release_b200 import HumanRegularizers
    key = tuple(sorted(label_kw.items()))
    if "mesh" not in _CACHE:
        _CACHE["mesh"] = make_human_mesh()
    m = _CACHE["mesh"]
    if key not in _CACHE:
        labels = make_regs_labels(m, **label_kw)
        _, _, _, target, hand_joints, pairs = _case()
        kw = dict(labels, joint_offset_target=target.float(), hand_joints=hand_joints, sym_pairs=pairs)
        regs = HumanRegularizers(m["faces"], P_C4, device=dev,
                                 **{k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
        _CACHE[key] = (regs, kw)
    regs, kw = _CACHE[key]
    g = torch.Generator().manual_seed(23)
    ins = {"mean_offset": 1e-3 * torch.randn(1, P_C4, 3, generator=g),
           "mean_offset_offset": 5e-4 * torch.randn(1, P_C4, 3, generator=g),
           "scale_offset": 1e-2 * torch.randn(1, P_C4, 1, generator=g),
           "scale": torch.exp(-5.5 + 0.3 * torch.randn(1, P_C4, 3, generator=g)),
           "scale_refined": torch.exp(-5.5 + 0.3 * torch.randn(1, P_C4, 3, generator=g)),
           "rgb": torch.rand(1, P_C4, 3, generator=g), "rgb_refined": torch.rand(1, P_C4, 3, generator=g),
           "joint_offset": 1e-2 * torch.randn(55, 3, generator=g)}
    golden_generator("make_regs_golden").pin_kinks(ins, kw, list(JOINTS))
    return m, regs, kw, ins


def _op(regs, mesh, ins, dev, dout=None, scale_reg=None):
    leaves = {k: v.to(dev).clone().requires_grad_() for k, v in ins.items()}
    sreg = None if scale_reg is None else scale_reg.to(dev).clone().requires_grad_()
    out = regs(mesh.to(dev), *[leaves[k] for k in INPUTS], scale_reg=sreg)
    vec = torch.stack([out[k] for k in KEYS])
    vec.backward(torch.ones(10, device=dev) if dout is None else dout.to(dev))
    grads = {k: leaves[k].grad for k in INPUTS}
    if sreg is not None:
        grads["scale_reg"] = sreg.grad
    return vec.detach(), grads


@pytest.mark.gpu
@pytest.mark.parametrize("warmup", [False, True])
def test_c4_terms_and_gradients_against_float64(warmup):
    dev = torch.device("cuda:0")
    m, regs, kw, ins = _c4(dev)
    sreg = torch.exp(-5.5 + 0.3 * torch.randn(1, P_C4, 3, generator=torch.Generator().manual_seed(8))) if warmup else None
    vec, grads = _op(regs, m["verts"], ins, dev, scale_reg=sreg)
    leaves = {k: v.double().requires_grad_() for k, v in ins.items()}
    s64 = None if sreg is None else sreg.double().requires_grad_()
    ref = regs.reference(m["verts"], *[leaves[k] for k in INPUTS], scale_reg=s64)
    for i, k in enumerate(KEYS):
        r = float(ref[k])
        assert abs(float(vec[i]) - r) <= 1e-6 * abs(r), (k, float(vec[i]), r)
    # lap_mean: the op takes the Laplacian of the offsets; ExAvatar's own fp32 evaluation, lap(mnp + o) - lap(mnp),
    # is no closer to float64 than the op
    tab = regs.tables
    nidx, nw = torch.from_numpy(tab["nbr_idx"]).to(dev), torch.from_numpy(tab["nbr_w"]).to(dev)
    lap = lambda x: x + (x[nidx] * nw[:, :, None]).sum(1)  # noqa: E731
    base = m["verts"].to(dev)
    mo, moo = ins["mean_offset"][0].to(dev), ins["mean_offset_offset"][0].to(dev)
    lit = (((lap(base + mo) - lap(base)) ** 2 + (lap(base + mo + moo) - lap(base)) ** 2) * 100000
           * tab["weights"][2].to(dev)[:, None]).mean()
    r = float(ref["lap_mean"])
    err_op, err_fp32 = abs(float(vec[KEYS.index("lap_mean")]) - r), abs(float(lit) - r)
    print(f"lap_mean relative error: op {err_op / r:.2e}, ExAvatar's fp32 form {err_fp32 / r:.2e}")
    assert err_op <= err_fp32
    sum(ref.values()).backward()
    pairs = [(k, grads[k], leaves[k].grad) for k in INPUTS] + ([("scale_reg", grads["scale_reg"], s64.grad)]
                                                               if warmup else [])
    row = _kink_row(kw)
    for k, got, want in pairs:
        got = got.double().cpu().reshape(want.shape).clone()
        want = want.detach().clone()
        if k == "mean_offset":  # the zero-offset hand row: clamp passes at exactly 0, n / eps through F.normalize
            kg, kw_ = got[0, row], want[0, row]
            assert float((kg - kw_).abs().max()) <= 1e-5 * float(kw_.abs().max()) and float(kw_.abs().max()) > 1e6, \
                (kg, kw_)
            got[0, row], want[0, row] = 0.0, 0.0
        scale = float(want.abs().max())
        err = float((got - want).abs().max())
        assert scale > 0 and err <= 1e-5 * scale, (k, err, scale)
    # abs's gradient at exactly 0: the pinned elbow pair's x and y terms vanish
    jr, jl = JOINTS.index("R_Elbow"), JOINTS.index("L_Elbow")
    jo = ins["joint_offset"]
    assert float(jo[jr, 0] + jo[jl, 0]) == 0.0 and float(jo[jr, 1] - jo[jl, 1]) == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("label_kw", [{}, {"arm_ny": (0.47, 0.53), "arm_half_width": 0.02}],
                         ids=["k50", "k_below_50"])
def test_arm_selection_matches_the_reference(label_kw):
    """Only arm_rgb_reg's upstream gradient: the rgb gradient of a lower row is c (rgb - target), which gives the op's
    targets.  They equal the means over the reference's selection except at rows whose k-th and (k+1)-th distances
    tie; equal targets on every other row also mean equal k."""
    dev = torch.device("cuda:0")
    m, regs, kw, ins = _c4(dev, **label_kw)
    dout = torch.zeros(10)
    dout[KEYS.index("arm_rgb_reg")] = 1.0
    vec, grads = _op(regs, m["verts"], ins, dev, dout=dout)
    from exavatar_release_b200.geometry import VertexNormals
    normals = VertexNormals(m["faces"], P_C4, device=dev)(m["verts"].to(dev)).cpu()
    lower, sel, k, tie = arm_selection_reference(m["verts"], normals, kw["is_arm"])
    assert lower.numel() > 0 and k > 0 and (k == 50) == (not label_kw)
    rgb = ins["rgb"][0].double()
    want = rgb[sel.reshape(-1)].reshape(lower.numel(), k, 3).mean(1)
    c = 2 * 0.1 / (3 * lower.numel())
    g = grads["rgb"][0].double().cpu()
    got = rgb[lower] - g[lower] / c
    assert bool((g.abs().sum(1) > 0)[lower].all()) and int((g.abs().sum(1) > 0).sum()) <= lower.numel()
    bad = (got - want).abs().max(1).values > 1e-4
    print(f"arm rows {lower.numel()}, k {k}, tie rows {int(tie.sum())}, differing rows {int(bad.sum())}")
    assert not bool((bad & ~tie).any())
    assert int(tie.sum()) <= max(2, lower.numel() // 100)


@pytest.mark.gpu
def test_small_windows_nan_and_no_lower_rows():
    dev = torch.device("cuda:0")
    i = KEYS.index("arm_rgb_reg")
    # k = 0: some lower row has no upper row within 1 cm in x -> NaN for the term and its lower rows' gradient
    m, regs, kw, ins = _c4(dev, arm_ny=(0.49, 0.51), arm_half_width=0.05)
    vec, grads = _op(regs, m["verts"], ins, dev)
    assert torch.isnan(vec[i]) and bool(torch.isfinite(torch.cat([vec[:i], vec[i + 1:]])).all())
    from exavatar_release_b200.geometry import VertexNormals
    normals = VertexNormals(m["faces"], P_C4, device=dev)(m["verts"].to(dev)).cpu()
    lower, _, k, _ = arm_selection_reference(m["verts"], normals, kw["is_arm"])
    assert k == 0 and lower.numel() > 0
    g = grads["rgb"][0].cpu()
    assert bool(torch.isnan(g[lower]).all())
    others = torch.ones(P_C4, dtype=torch.bool)
    others[lower] = False
    assert bool(torch.isfinite(g[others]).all()) and bool(torch.isfinite(grads["mean_offset"]).all())
    # no lower row (the reference raises in torch.min): NaN for the term, finite gradients everywhere
    m, regs, kw, ins = _c4(dev, arm_ny=(0.6, 0.7), arm_half_width=0.05)
    lower, _, _, _ = arm_selection_reference(m["verts"], normals, kw["is_arm"])
    assert lower.numel() == 0 and int(kw["is_arm"].sum()) > 0
    vec, grads = _op(regs, m["verts"], ins, dev)
    assert torch.isnan(vec[i]) and all(bool(torch.isfinite(v).all()) for v in grads.values())


@pytest.mark.gpu
def test_bit_identical_no_sync_and_graph_replay():
    dev = torch.device("cuda:0")
    m, regs, kw, ins = _c4(dev, arm_ny=(0.47, 0.53), arm_half_width=0.02)
    a, b = _op(regs, m["verts"], ins, dev), _op(regs, m["verts"], ins, dev)
    assert torch.equal(a[0], b[0]) and all(torch.equal(a[1][k], b[1][k]) for k in INPUTS)
    mesh = m["verts"].to(dev)
    leaves = {k: v.to(dev).clone().requires_grad_() for k, v in ins.items()}
    with no_host_sync():
        out = regs(mesh, *[leaves[k] for k in INPUTS])
        sum(out.values()).backward()

    # forward + backward in one graph, replayed with a sheared mesh (new upper / lower split and k) and new inputs
    static_mesh = mesh.clone()
    static = {k: v.detach().clone().requires_grad_() for k, v in leaves.items()}

    def step():
        out = regs(static_mesh, *[static[k] for k in INPUTS])
        vec = torch.stack([out[k] for k in KEYS])
        vec.sum().backward()
        return vec

    def no_grads():
        for v in static.values():
            v.grad = None

    graph, vec_g = capture(step, 2, reset=no_grads)
    sheared = m["verts"].clone()
    sheared[:, 1] += 0.4 * sheared[:, 0]
    g = torch.Generator().manual_seed(99)
    new = {k: (v * (1 + 0.5 * torch.rand(v.shape, generator=g))) for k, v in ins.items()}
    with torch.no_grad():
        static_mesh.copy_(sheared.to(dev))
        for k in INPUTS:
            static[k].copy_(new[k].to(dev))
    graph.replay()
    torch.cuda.synchronize()
    vec_e, grads_e = _op(regs, sheared, new, dev)
    assert torch.equal(vec_g.detach(), vec_e)
    assert all(torch.equal(static[k].grad, grads_e[k]) for k in INPUTS)
    from exavatar_release_b200.geometry import VertexNormals
    vn = VertexNormals(m["faces"], P_C4, device=dev)
    k0 = arm_selection_reference(m["verts"], vn(mesh).cpu(), kw["is_arm"])[2]
    k1 = arm_selection_reference(sheared, vn(sheared.to(dev)).cpu(), kw["is_arm"])[2]
    assert k0 != k1  # the replay really moved the split and the window


@pytest.mark.gpu
def test_human_chain_then_regularizers_against_the_fp32_restatement():
    """The f-7 human chain of a C4 frame (test_human_nets._chain_setup, networks as the ops) followed by the op, against
    the same chain followed by human_regularizers_reference in fp32: the loss within 1e-6, every network, triplane and
    input gradient within 1e-4 of its max."""
    from test_human_nets import _chain_setup
    from exavatar_release_b200.human_nets import gn_mlp
    dev = torch.device("cuda:0")
    s = _chain_setup(dev)
    m, regs, kw, _ = _c4(dev)
    mesh = m["verts"].to(dev)
    jo = (1e-2 * torch.randn((55, 3), generator=torch.Generator().manual_seed(4))).to(dev).requires_grad_()
    params = [s["tp"], s["tpf"], jo] + [p for t, hs in s["nets"].values() for mm in [t, *hs] for p in mm.parameters()]
    res = {}
    for use_op in (True, False):
        for p in params:
            p.grad = None
        tri = s["tri"](s["tp"], s["tpf"])
        run = lambda k, ins: gn_mlp(ins, *s["nets"][k])  # noqa: E731
        geo, geo_off, rgb = run("geo", [tri]), run("geo_offset", [tri, s["pose"]]), run("rgb", [tri])
        normal = s["normals"](mesh)
        rgb_off = run("rgb_offset", [tri, s["pose"], normal])
        args = (0.01 * geo[:, :3], 0.005 * geo_off[:, :3], 0.1 * geo_off[:, 3:],
                s["human"]["scale"] * torch.exp(0.1 * geo[:, 3:]),
                s["human"]["scale"] * torch.exp(0.1 * (geo[:, 3:] + geo_off[:, 3:])),
                (torch.tanh(rgb) + 1) / 2, (torch.tanh(rgb + rgb_off) + 1) / 2, jo)
        out = regs(mesh, *args) if use_op else regs.reference(mesh, *args, dtype=torch.float32)
        loss = sum(out.values())
        loss.backward()
        torch.cuda.synchronize()
        res[use_op] = (float(loss), [p.grad.detach().clone().to(dev) for p in params])
    (lo, go), (lt, gt) = res[True], res[False]
    assert abs(lo - lt) <= 1e-6 * abs(lt), (lo, lt)
    for i, (a, b) in enumerate(zip(go, gt)):
        scale = float(b.abs().max())
        err = float((a - b).abs().max())
        assert scale > 0 and err <= 1e-4 * scale, (i, tuple(a.shape), err, scale)
