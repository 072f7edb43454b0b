"""HumanGaussian's networks (avatar/common/nets/module.py:424-457 extract_tri_feature, layer.py make_linear_layers with
GroupNorm) as sync-free CUDA ops: `human_nets.TriplaneFeatures` (b2r_triplane_*) and `human_nets.gn_mlp`
(b2r_gn_mlp_*, 3xTF32 on the tensor cores).

These tests pin
  * without a device: the C ABI (symbols, struct size, validation before any launch), the plain-torch restatement
    against tests/golden/human_nets.npz (made by the reference's own make_linear_layers / extract_tri_feature), the
    bilinear corner table against F.grid_sample, and the shape checks of gn_mlp;
  * on the GPU at C4 size (P = 167 618): the triplane features and both plane gradients against float64, the four
    stacks' outputs and every parameter gradient against float64 with the fp32 torch modules' own error as the
    yardstick, a constant GroupNorm group and exact-zero pre-activations, the folded pose block's weight gradient,
    bit-identical runs, no host sync, and forward + backward replayed from one CUDA graph after an optimizer step.
"""
import copy
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from util import capture, golden_generator, no_host_sync
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.human_nets import (TriplaneFeatures, bilinear_corners, gn_mlp, gn_mlp_reference,
                                              human_nets_reference, tri_feature_reference, triplane_grid)

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FAKE = 0x1000  # never dereferenced: validation fails before any launch
P_C4 = 167618


def gn_stack(k_in, head_dims=None, final=None):
    """make_linear_layers([k_in, 128, 128, 128], use_gn=True) (+ a final Linear(128, final)) and head Linears."""
    mods = []
    for k in (k_in, 128, 128):
        mods += [nn.Linear(k, 128), nn.GroupNorm(4, 128), nn.ReLU(inplace=True)]
    if final:
        mods.append(nn.Linear(128, final))
    heads = [nn.Sequential(nn.Linear(128, h)) for h in (head_dims or [])]
    return nn.Sequential(*mods), heads


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

def test_abi_symbols_and_struct():
    lib = L.load()
    raw = C.CDLL(L.LIB_PATH)
    for name in ("b2r_triplane_forward", "b2r_triplane_backward", "b2r_gn_mlp_scratch_bytes", "b2r_gn_mlp_grads_count",
                 "b2r_gn_mlp_forward", "b2r_gn_mlp_backward"):
        assert hasattr(raw, name), name
        assert name in {s[0] for s in L.SYMBOLS}, name
    assert C.sizeof(L.B2RGnMlp) == 16 + 8 * 15
    assert lib.b2r_gn_mlp_grads_count(222, 4) == 128 * 222 + 2 * 128 * 128 + 9 * 128 + 4 * 128 + 4
    # the backward keeps dz_0..2 and a_0, a_1 (5 x P x 128 fp32) plus its partials
    assert lib.b2r_gn_mlp_scratch_bytes(P_C4) >= 5 * P_C4 * 128 * 4


def test_validation_without_touching_cuda():
    lib = L.load()
    n0 = lib.b2r_launch_count()

    def mlp(**kw):
        m = L.B2RGnMlp(P=64, K=96, H=4, x=FAKE, w_head=FAKE, b_head=FAKE)
        for i in range(3):
            m.w[i] = m.b[i] = m.gamma[i] = m.beta[i] = FAKE
        for k, v in kw.items():
            if k in ("w", "b", "gamma", "beta"):
                getattr(m, k)[1] = v
            else:
                setattr(m, k, v)
        return m

    for kw in ({"P": 0}, {"K": 0}, {"K": 129}, {"H": 0}, {"H": 5}, {"x": None}, {"w_head": None}, {"w": None},
               {"gamma": None}):
        m = mlp(**kw)
        assert lib.b2r_gn_mlp_forward(C.byref(m), FAKE, None, None) == -1, kw
        assert lib.b2r_gn_mlp_backward(C.byref(m), FAKE, FAKE, None, FAKE, FAKE, 1 << 40, None) == -1, kw
    m = mlp()
    assert lib.b2r_gn_mlp_forward(C.byref(m), None, None, None) == -1
    need = lib.b2r_gn_mlp_scratch_bytes(64)
    assert lib.b2r_gn_mlp_backward(C.byref(m), FAKE, FAKE, None, FAKE, FAKE, need - 1, None) == -2
    assert lib.b2r_gn_mlp_backward(C.byref(m), None, FAKE, None, FAKE, FAKE, need, None) == -1
    for args in ((64, 0, 8, 8), (64, 32, 0, 8), (-1, 32, 8, 8)):
        assert lib.b2r_triplane_forward(*args, FAKE, FAKE, None, FAKE, FAKE, FAKE, None) == -1, args
    assert lib.b2r_triplane_forward(64, 32, 8, 8, None, FAKE, None, FAKE, FAKE, FAKE, None) == -1
    assert lib.b2r_triplane_backward(64, 32, 8, 8, FAKE, None, FAKE, FAKE, FAKE, FAKE, None) == -1
    assert lib.b2r_triplane_forward(0, 32, 8, 8, None, None, None, None, None, None, None) == 0  # nothing to do
    assert lib.b2r_launch_count() == n0


def test_restatement_reproduces_the_reference_golden():
    """tri_feature_reference + gn_mlp_reference (human_nets_reference) against the reference's own code in float64:
    pins the column order, the face overwrite, the pose in the middle of the concat and GroupNorm's group layout."""
    gm = golden_generator("make_human_nets_golden")
    gold = np.load(os.path.join(G, "human_nets.npz"))
    nets = {}
    for k, (dims, relu_final) in gm.layer_dims().items():
        if len(dims) == 2:
            nets[k] = nn.Sequential(nn.Linear(*dims))
        else:
            trunk, _ = gn_stack(dims[0], final=dims[-1] if len(dims) == 5 else None)
            nets[k] = trunk
        nets[k] = nets[k].double()
    gm.set_parameters(nets)
    pos, is_face, tp, tpf, pose, normal = gm.case_inputs()
    tp.requires_grad_()
    tpf.requires_grad_()
    grid = triplane_grid(pos, is_face, gm.SHAPE_3D, gm.FACE_SHAPE_3D)
    outs = human_nets_reference(grid, is_face, tp, tpf, nets, pose, normal)
    for k, v in outs.items():
        ref = gold[f"out_{k}"]
        assert v.shape == ref.shape, k
        np.testing.assert_allclose(v.detach().numpy(), ref, rtol=0, atol=1e-12 * max(1.0, np.abs(ref).max()), err_msg=k)
    loss = sum((gm.output_weights(k, tuple(v.shape)) * v).sum() for k, v in outs.items())
    loss.backward()
    grads = {"triplane": tp.grad, "triplane_face": tpf.grad}
    for name in gm.NETS:
        for pname, p in nets[name].named_parameters():
            grads[f"{name}.{pname}"] = p.grad
    for k, v in grads.items():
        flat = v.reshape(-1).numpy()
        scale = max(1.0, float(gold[f"grad_abs:{k}"]))
        np.testing.assert_allclose(flat[gold[f"grad_idx:{k}"]], gold[f"grad_val:{k}"], rtol=0, atol=1e-12 * scale,
                                   err_msg=k)
        np.testing.assert_allclose(np.abs(flat).sum(), gold[f"grad_abs:{k}"], rtol=1e-12, err_msg=k)
    assert bool(is_face.any()) and bool((grid.abs() > 1).any())  # face rows and samples outside [-1, 1] are covered


def test_corner_table_is_grid_sample():
    """The op's constant corners and weights, blended in float64, are F.grid_sample's bilinear sample."""
    g = torch.Generator().manual_seed(3)
    grid = (torch.rand((500, 3, 2), generator=g) * 2.6 - 1.3).float()
    planes = torch.randn((3, 5, 9, 14), generator=g, dtype=torch.float64)
    idx, w = bilinear_corners(grid, 9, 14)
    flat = planes.reshape(3, 5, -1)
    got = torch.zeros((500, 3, 5), dtype=torch.float64)
    for p in range(3):
        for k in range(4):
            i = idx[:, p, k].long()
            ok = i >= 0
            got[ok, p] += w[ok, p, k, None].double() * flat[p][:, i[ok]].t()
    ref = torch.stack([F.grid_sample(planes[p, None], grid[None, :, None, p, :].double(), align_corners=False)[0, :, :, 0]
                       .t() for p in range(3)], 1)
    assert float((got - ref).abs().max()) <= 1e-7 * float(ref.abs().max())
    assert bool((idx < 0).any())  # zero padding is exercised


def test_gn_mlp_rejects_unsupported_shapes():
    trunk, heads = gn_stack(96, [3, 1])
    x = torch.zeros(8, 96)
    with pytest.raises(ValueError, match="GroupNorm"):
        t2 = copy.deepcopy(trunk)
        t2[1] = nn.GroupNorm(8, 128)
        gn_mlp([x], t2, heads)
    with pytest.raises(ValueError, match="Linear"):
        t2 = copy.deepcopy(trunk)
        t2[3] = nn.Linear(128, 64)
        gn_mlp([x], t2, heads)
    with pytest.raises(ValueError, match="at most 4"):
        gn_mlp([x], trunk, heads + [nn.Sequential(nn.Linear(128, 2))])
    with pytest.raises(ValueError, match="unsupported stack"):
        gn_mlp([x], nn.Sequential(*list(trunk)[:6]), heads)
    with pytest.raises(ValueError, match="columns"):
        gn_mlp([torch.zeros(8, 95)], trunk, heads)
    big, bh = gn_stack(200, [3])
    with pytest.raises(ValueError, match="at most 128"):
        gn_mlp([torch.zeros(8, 200)], big, bh)
    with pytest.raises(ValueError, match="requires grad"):
        t3, h3 = gn_stack(96 + 126, [3])
        gn_mlp([x, torch.zeros(126, requires_grad=True)], t3, h3)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

def _c4_rows(dev, seed=0):
    """(pos_enc_mesh, is_face) of a C4-sized upsampled human: a body box with some rows beyond it and a head."""
    g = torch.Generator(device=dev).manual_seed(seed)
    pos = (torch.rand((P_C4, 3), generator=g, device=dev) - 0.5) * torch.tensor([0.9, 1.9, 0.4], device=dev)
    pos[:2000] *= 1.8  # beyond the [-1, 1] square of the body planes
    is_face = pos[:, 1] > 0.72
    pos[is_face] = pos[is_face] * torch.tensor([0.3, 0.2, 0.5], device=dev) + torch.tensor([0, 0.75, 0.05], device=dev)
    return pos, is_face


@pytest.mark.gpu
def test_triplane_c4_against_float64_and_bit_identical():
    dev = torch.device("cuda:0")
    pos, is_face = _c4_rows(dev)
    tri = TriplaneFeatures(pos, is_face)
    g = torch.Generator(device=dev).manual_seed(1)
    tp = torch.randn((3, 32, 128, 128), generator=g, device=dev).requires_grad_()
    tpf = torch.randn((3, 32, 128, 128), generator=g, device=dev).requires_grad_()
    feat = tri(tp, tpf)
    gout = torch.randn(feat.shape, generator=g, device=dev)
    (feat * gout).sum().backward()
    d1, df1 = tp.grad.clone(), tpf.grad.clone()
    # float64 with the op's constant sample weights: the bilinear blend and the adjoint in float64
    tp64 = tp.detach().double().requires_grad_()
    tpf64 = tpf.detach().double().requires_grad_()
    ref = _blend64(tri, tp64, tpf64)
    (ref * gout.double()).sum().backward()
    assert float((feat.double() - ref.detach()).abs().max()) <= 1e-6 * float(ref.detach().abs().max())
    for got, r in ((d1, tp64.grad), (df1, tpf64.grad)):
        assert float((got.double() - r).abs().max()) <= 1e-5 * float(r.abs().max())
    # face rows leave the body triplane's gradient untouched
    tp.grad = None
    tpf.grad = None
    (tri(tp, tpf) * gout * is_face[:, None]).sum().backward()
    assert float(tp.grad.abs().max()) == 0.0 and float(tpf.grad.abs().max()) > 0
    # the reference's own grid_sample at the fp32 coordinates agrees closely too
    ref_gs = tri_feature_reference(tri.grid, is_face, tp.detach().double(), tpf.detach().double())
    assert float((feat.double() - ref_gs).abs().max()) <= 1e-4 * float(ref_gs.abs().max())
    # bit-identical backward
    tp.grad = None
    tpf.grad = None
    (tri(tp, tpf) * gout).sum().backward()
    assert torch.equal(tp.grad, d1) and torch.equal(tpf.grad, df1)


def _blend64(tri, tp, tpf):
    C_ = tp.shape[1]
    feats = []
    for p in range(3):
        idx = tri.corners[:, p].long()
        w = tri.weights[:, p].double()
        out = 0
        for k in range(4):
            i = idx[:, k].clamp_min(0)
            body = tp[p].reshape(C_, -1)[:, i].t()
            face = tpf[p].reshape(C_, -1)[:, i].t()
            v = torch.where(tri.is_face.bool()[:, None], face, body)
            out = out + torch.where((idx[:, k] >= 0)[:, None], v * w[:, k, None], torch.zeros_like(v))
        feats.append(out)
    return torch.cat(feats, 1)


STACKS = {  # name: (per-row width, constant width, heads, final)
    "geo_net": (96, 0, [3, 1], None),
    "geo_offset_net": (96, 126, [3, 1], None),
    "rgb_net": (96, 0, None, 3),
    "rgb_offset_net": (96 + 3, 126, None, 3),
}


def _make_stack(name, dev, seed=0):
    k_row, k_const, heads, final = STACKS[name]
    torch.manual_seed(seed)
    trunk, hs = gn_stack(k_row + k_const, heads, final)
    with torch.no_grad():  # non-trivial GroupNorm affine
        for l in range(3):
            trunk[3 * l + 1].weight.uniform_(0.5, 1.5)
            trunk[3 * l + 1].bias.uniform_(-0.3, 0.3)
    return trunk.to(dev), [h.to(dev) for h in hs]


def _inputs(name, dev, seed=0):
    k_row, k_const, _, _ = STACKS[name]
    g = torch.Generator(device=dev).manual_seed(seed + 10)
    tri = torch.randn((P_C4, 96), generator=g, device=dev)
    ins = [tri]
    if k_const:
        ins.append(torch.randn((126,), generator=g, device=dev) * 0.5)
    if k_row > 96:
        n = torch.randn((P_C4, 3), generator=g, device=dev)
        ins.append(n / n.norm(dim=1, keepdim=True))
    return ins


def _params(trunk, heads):
    return list(trunk.parameters()) + [p for h in heads for p in h.parameters()]


def _run(fn, ins, trunk, heads, gout):
    for p in _params(trunk, heads):
        p.grad = None
    ins = [t.detach().clone().requires_grad_(t.dim() == 2 and i == 0) for i, t in enumerate(ins)]
    out = fn(ins, trunk, heads)
    (out * gout.to(out.dtype)).sum().backward()
    return out.detach(), [p.grad.detach().clone() for p in _params(trunk, heads)], ins[0].grad.detach().clone()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STACKS))
def test_stack_c4_against_float64(name):
    dev = torch.device("cuda:0")
    trunk, heads = _make_stack(name, dev)
    with torch.no_grad():
        # layer 0 group 0 constant for every row (variance 0: eps decides); group 1 pre-activations exactly 0 with
        # beta 0 in its first 8 channels (ReLU at exactly 0)
        trunk[0].weight[:32] = 0
        trunk[0].bias[:32] = 0.25
        trunk[0].weight[32:64] = 0
        trunk[0].bias[32:64] = 0
        trunk[1].bias[32:40] = 0
    ins = _inputs(name, dev)
    H = 4 if heads else 3
    gout = torch.randn((P_C4, H), generator=torch.Generator(device=dev).manual_seed(7), device=dev)
    t64, h64 = copy.deepcopy(trunk).double(), [copy.deepcopy(h).double() for h in heads]
    edge = _relu_edge_rows(ins, t64)
    assert int(edge.sum()) < 0.05 * P_C4
    gout[edge] = 0
    fwd = lambda i, t, h: gn_mlp(i, t, h)  # noqa: E731
    out, grads, dx = _run(fwd, ins, trunk, heads, gout)
    o64, g64, dx64 = _run(lambda i, t, h: gn_mlp_reference(i, t, h), ins, t64, h64, gout)
    tfwd = lambda i, t, h: _torch_module_forward(i, t, h)  # noqa: E731
    o32, g32, dx32 = _run(tfwd, ins, trunk, heads, gout)
    names = ["out"] + [n for n, _ in trunk.named_parameters()] + [f"head{i}.{n}" for i, h in enumerate(heads)
                                                                  for n, _ in h.named_parameters()] + ["dx"]
    for what, a, b, r in zip(names, [out] + grads + [dx], [o32] + g32 + [dx32], [o64] + g64 + [dx64]):
        err = float((a.double() - r).abs().max())
        err32 = float((b.double() - r).abs().max())
        scale = float(r.abs().max())
        assert err <= 1e-5 * scale, (name, what, err, scale)
        assert err <= 2 * err32, (name, what, err, err32, scale)
    # the folded constant block's weight gradient: the reference's gradient for those columns
    if STACKS[name][1]:
        cols = slice(96, 96 + 126)
        w_op, w_ref = grads[0][:, cols].double(), g64[0][:, cols]
        assert float((w_op - w_ref).abs().max()) <= 1e-5 * float(w_ref.abs().max())


@torch.no_grad()
def _relu_edge_rows(ins, t64, rel=2e-5):
    """Rows with a hidden pre-activation y within rel * max|y| of 0 but not exactly 0 (float64).  An fp32 evaluation
    -- the op's or torch's -- may put such a y on the other side of the ReLU, which moves every weight gradient by that
    row's whole contribution (about 1e-3 of the max at this size); the gradient comparisons leave these rows out.
    Exact zeros stay in: both sides agree there (relu'(0) = 0)."""
    P = next(t.shape[0] for t in ins if t.dim() == 2)
    x = torch.cat([(t if t.dim() == 2 else t.reshape(1, -1).expand(P, -1)).double() for t in ins], 1)
    edge = torch.zeros(P, dtype=torch.bool, device=x.device)
    for l in range(3):
        lin, gn = t64[3 * l], t64[3 * l + 1]
        z = (x @ lin.weight.t() + lin.bias).reshape(P, 4, 32)
        m = z.mean(-1, keepdim=True)
        v = ((z - m) ** 2).mean(-1, keepdim=True)
        y = ((z - m) / torch.sqrt(v + 1e-5)).reshape(P, 128) * gn.weight + gn.bias
        a = y.abs()
        edge |= ((a > 0) & (a < rel * a.max())).any(1)
        x = torch.relu(y)
    return edge


def _torch_module_forward(ins, trunk, heads):
    """ExAvatar's own evaluation in fp32: the modules on the concatenated input (constant blocks repeated)."""
    P = next(t.shape[0] for t in ins if t.dim() == 2)
    x = torch.cat([t if t.dim() == 2 else t.reshape(1, -1).repeat(P, 1).detach() for t in ins], 1)
    feat = trunk(x)
    return torch.cat([h(feat) for h in heads], 1) if heads else feat


@pytest.mark.gpu
def test_stack_bit_identical_no_sync_and_graph():
    dev = torch.device("cuda:0")
    trunk, heads = _make_stack("rgb_offset_net", dev)
    ins = _inputs("rgb_offset_net", dev)
    gout = torch.randn((P_C4, 3), generator=torch.Generator(device=dev).manual_seed(9), device=dev)
    run = lambda: _run(lambda i, t, h: gn_mlp(i, t, h), ins, trunk, heads, gout)  # noqa: E731
    a, b = run(), run()
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    assert all(torch.equal(x, y) for x, y in zip(a[1], b[1]))
    with no_host_sync():
        run()

    # forward + backward in one graph; replayed after an optimizer step changed the weights, equal to eager
    params = _params(trunk, heads)
    opt = torch.optim.Adam(params, lr=1e-3)
    x = ins[0].detach().clone().requires_grad_()
    static = [x] + [t.detach().clone() for t in ins[1:]]

    def step():
        out = gn_mlp(static, trunk, heads)
        (out * gout).sum().backward()
        return out

    def no_grads():
        for p in (*params, x):
            p.grad = None

    graph, out_g = capture(step, 2, reset=no_grads)
    graph.replay()
    opt.step()  # new weights, same parameter storage
    graph.replay()
    torch.cuda.synchronize()
    g_graph = [p.grad.clone() for p in params]
    o_graph, dx_graph = out_g.detach().clone(), x.grad.clone()
    o_e, g_e, dx_e = _run(lambda i, t, h: gn_mlp(i, t, h), static, trunk, heads, gout)
    assert torch.equal(o_graph, o_e) and torch.equal(dx_graph, dx_e)
    assert all(torch.equal(a_, b_) for a_, b_ in zip(g_graph, g_e))


# ---------------------------------------------------------------------------------------------------------------------
# The human chain of a C4 training frame
# ---------------------------------------------------------------------------------------------------------------------

def _chain_setup(dev):
    """A C4 training frame around the synthetic human mesh: the networks, the triplanes, the rig, the scene, the
    renderer and a target image."""
    from test_fused_skinning import _rig
    from exavatar_release_b200 import TrainingFrameRenderer
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.geometry import VertexNormals
    from exavatar_release_b200.synthetic import WORKLOADS, Workload, make_human_mesh, make_population_assets
    mesh = make_human_mesh()
    P = mesh["verts"].shape[0]
    c4 = WORKLOADS["C4"]
    H, W = c4.height, c4.width
    wl = Workload("C4 with the synthetic mesh's Gaussians", H, W, P, c4.n_scene, 0, True)
    scene, human, _ = make_population_assets(wl, seed=0, device=dev)
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    R, tc = cam["R"], cam["t"]
    to_cam = lambda x: (x.to(dev) @ R.t() + tc.view(1, 3)).contiguous()  # noqa: E731  (the skinning's frame)
    torch.manual_seed(3)
    nets = {"geo": gn_stack(96, [3, 1]), "geo_offset": gn_stack(96 + 126, [3, 1]), "rgb": gn_stack(96, None, 3),
            "rgb_offset": gn_stack(96 + 126 + 3, None, 3)}
    nets = {k: (t.to(dev), [h.to(dev) for h in hs]) for k, (t, hs) in nets.items()}
    # GroupNorm beta = 4: y = z_hat gamma + 4 is rarely near 0.  Two fp32 evaluations of the same stack (the op's and
    # torch's) put a y within rounding of 0 on different sides of the ReLU, and one such row moves the gradients it
    # reaches by ~1e-3 of their max (with beta = 0 here: 1.2e-2 on geo_net's first weight, 3e-3 on the triplane; with
    # beta = 4: below 4e-5 everywhere).  The stack tests cover beta around 0 with those rows left out.
    with torch.no_grad():
        for t, _ in nets.values():
            for l in range(3):
                t[3 * l + 1].bias.fill_(4.0)
    g = torch.Generator(device=dev).manual_seed(4)
    verts = mesh["verts"].to(dev)
    is_face = verts[:, 1] > 0.6  # the head cap
    table, A, tr = _rig(P, 55, torch.float32, dev)
    return {
        "P": P, "cam": cam, "R": R, "tc": tc, "scene": scene, "human": human,
        "canon": to_cam(mesh["queries"]), "targets": to_cam(mesh["targets"]), "self_map": mesh["self_map"].to(dev),
        "normals": VertexNormals(mesh["faces"], P, flip=mesh["flip"].to(dev)),
        "tri": TriplaneFeatures(verts, is_face), "is_face": is_face, "nets": nets,
        "tp": (0.3 * torch.randn((3, 32, 128, 128), generator=g, device=dev)).requires_grad_(),
        "tpf": (0.3 * torch.randn((3, 32, 128, 128), generator=g, device=dev)).requires_grad_(),
        "pose": 0.5 * torch.randn(126, generator=g, device=dev),
        "table": table, "A": A, "tr": tr,
        "fr": TrainingFrameRenderer(scene["mean_3d"].shape[0], P, (H, W), dev, {"A": 8_000_000, "B": 8_000_000}),
        "target": torch.rand((3, H, W), generator=g, device=dev),
        "bg": torch.tensor([0.3, 0.7, 0.2], device=dev),
    }


def _human_chain(s, ops: bool):
    """TriplaneFeatures -> geo / geo_offset / rgb stacks -> offsets -> nearest_rows -> skin_gaussians -> VertexNormals
    -> rgb_offset stack -> TrainingFrameRenderer -> l1_ssim, with the networks as the ops (ops=True) or as the fp32
    torch modules with F.grid_sample (ExAvatar's evaluation).  Returns (loss, rows)."""
    from exavatar_release_b200.geometry import nearest_rows
    from exavatar_release_b200.losses import l1_ssim
    from exavatar_release_b200.plan import RENDERS
    from exavatar_release_b200.skinning import skin_gaussians
    nets = s["nets"]
    if ops:
        tri = s["tri"](s["tp"], s["tpf"])
        run = lambda k, ins: gn_mlp(ins, *nets[k])  # noqa: E731
    else:
        tri = tri_feature_reference(s["tri"].grid, s["is_face"], s["tp"], s["tpf"])
        run = lambda k, ins: _torch_module_forward(ins, *nets[k])  # noqa: E731
    geo = run("geo", [tri])
    geo_off = run("geo_offset", [tri, s["pose"]])
    rgb = run("rgb", [tri])
    mean_3d = s["canon"] + 0.01 * geo[:, :3]
    mean_3d_refined = mean_3d + 0.005 * geo_off[:, :3]
    scale = s["human"]["scale"] * torch.exp(0.1 * geo[:, 3:])
    scale_refined = s["human"]["scale"] * torch.exp(0.1 * (geo[:, 3:] + geo_off[:, 3:]))
    rows = nearest_rows(mean_3d.detach(), s["targets"], s["self_map"])
    posed, posed_r = skin_gaussians(mean_3d, mean_3d_refined, s["table"], rows, s["A"], s["tr"], s["R"], s["tc"])
    normal = s["normals"](posed_r)
    rgb_off = run("rgb_offset", [tri, s["pose"], normal])
    human = dict(s["human"], mean_3d=posed, scale=scale, rgb=(torch.tanh(rgb) + 1) / 2)
    refined = dict(s["human"], mean_3d=posed_r, scale=scale_refined, rgb=(torch.tanh(rgb + rgb_off) + 1) / 2)
    out = s["fr"](s["scene"], human, refined, s["cam"], s["bg"])
    loss = 0
    for r in RENDERS:
        l1, ss = l1_ssim(out[r]["img"], s["target"])
        loss = loss + 0.8 * l1 + 0.2 * (1 - ss)
    return loss, rows


@pytest.mark.gpu
def test_human_chain_c4_frame_ops_match_torch_networks():
    """The whole human chain of a C4 training frame with the networks as the ops against the same chain with them as
    fp32 torch modules: the loss and every network and triplane gradient within 1e-4 of the max."""
    dev = torch.device("cuda:0")
    s = _chain_setup(dev)
    params = [s["tp"], s["tpf"]] + [p for t, hs in s["nets"].values() for m in [t, *hs] for p in m.parameters()]
    res = {}
    for ops in (True, False):
        for p in params:
            p.grad = None
        loss, rows = _human_chain(s, ops)
        loss.backward()
        torch.cuda.synchronize()
        assert not s["fr"].overflowed()
        res[ops] = (loss.detach(), rows, [p.grad.detach().clone() for p in params])
    (lo, ro, go), (lt, rt, gt) = res[True], res[False]
    assert torch.equal(ro, rt)  # both arms pose every Gaussian with the same rig rows
    assert abs(float(lo) - float(lt)) <= 1e-4 * abs(float(lt)), (float(lo), float(lt))
    for i, (a, b) in enumerate(zip(go, gt)):
        scale = float(b.abs().max())
        assert scale > 0, i
        err = float((a - b).abs().max())
        assert err <= 1e-4 * scale, (i, tuple(a.shape), err, scale)


@pytest.mark.gpu
@pytest.mark.parametrize("tri_grad", [True, False])
def test_second_row_block_gradient(tri_grad):
    """dX split into every per-row block that requires grad -- here rgb_offset_net's normal block behind the folded
    pose -- also when the first block does not require grad."""
    dev = torch.device("cuda:0")
    trunk, heads = _make_stack("rgb_offset_net", dev)
    g = torch.Generator(device=dev).manual_seed(21)
    P = 8192
    tri = torch.randn((P, 96), generator=g, device=dev)
    pose = 0.5 * torch.randn((126,), generator=g, device=dev)
    n = F.normalize(torch.randn((P, 3), generator=g, device=dev), dim=1)
    t64 = copy.deepcopy(trunk).double()
    gout = torch.randn((P, 3), generator=g, device=dev)
    gout[_relu_edge_rows([tri, pose, n], t64)] = 0
    grads = {}
    for name, fn, tt in (("op", lambda i: gn_mlp(i, trunk, heads), trunk),
                         ("f64", lambda i: gn_mlp_reference(i, t64, None), t64)):
        a = tri.detach().clone().requires_grad_(tri_grad)
        b = n.detach().clone().requires_grad_()
        (fn([a, pose, b]) * gout).sum().backward()
        grads[name] = (a.grad, b.grad)
    assert (grads["op"][0] is None) == (not tri_grad)
    for k in ((0, 1) if tri_grad else (1,)):
        got, ref = grads["op"][k].double(), grads["f64"][k]
        assert float((got - ref).abs().max()) <= 1e-5 * float(ref.abs().max()), k
