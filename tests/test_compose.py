"""The image composites on the device (`compose.face_composite`, `compose.test_outputs`, csrc/compose.cu): bit-identical
to the torch / numpy references at odd and full sizes and N = 1..3, torch autograd's gradients, repeatable, every
output element written, no host sync, CUDA-graph replays with new inputs, and the test pass end to end from
TrainingFrameRenderer and FaceMeshRenderer to NeumanScores."""
import numpy as np
import pytest
import torch

from test_compose_reference import inputs, same_bits
from test_poisoned_buffers import poisoned
from exavatar_release_b200 import compose as CP
from exavatar_release_b200.compose import COMPOSITE_KEYS, RENDER_KEYS, face_composite, face_composite_reference
from exavatar_release_b200.plan import RENDERS

SIZES = [(1, 31, 37), (3, 31, 37), (2, 512, 512), (1, 1080, 1920), (3, 1080, 1920)]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def on(dev, renders, *ts):
    r = {k: {n: t.to(dev) for n, t in v.items()} for k, v in renders.items()}
    return (r, *(None if t is None else t.to(dev) for t in ts))


def check_outputs(out, ref, png=True):
    for k in RENDER_KEYS + COMPOSITE_KEYS:
        assert same_bits(out[k], ref[k]), k
    if png:
        np.testing.assert_array_equal(out["png"].cpu().numpy(), ref["png"])


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W", SIZES)
def test_test_outputs_equal_the_reference(dev, N, H, W):
    renders, face, face_r, gt = on(dev, *inputs(N, H, W, seed=N + H))
    with torch.no_grad():
        out = CP.test_outputs(renders, face, face_r, gt)
        check_outputs(out, CP.test_outputs_reference(renders, face, face_r, gt))
        assert out["png"].shape == (10, N, H, W, 3)
        no_gt = CP.test_outputs(renders, face, face_r)
        assert torch.equal(no_gt["png"], out["png"][:9])
        assert "png" not in CP.test_outputs(renders, face, face_r, gt, png=False)


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W", SIZES)
def test_face_composite_and_gradient_equal_torch(dev, N, H, W):
    renders, face, _, _ = on(dev, *inputs(N, H, W, seed=7 * N + W))
    img = renders["scene_human"]["img"]
    g = torch.randn(N, 3, H, W, device=dev)
    g[:, :, 0] = -0.0
    x, f = img.clone().requires_grad_(), face.clone().requires_grad_()
    out = face_composite(x, f)
    out.backward(g)
    x2, f2 = img.clone().requires_grad_(), face.clone().requires_grad_()
    ref = face_composite_reference(x2, f2)
    ref.backward(g)
    assert same_bits(out, ref)
    assert same_bits(x.grad, x2.grad)
    assert same_bits(f.grad, f2.grad)
    assert f.grad[:, 3].abs().max() == 0
    # only one input asks for a gradient
    x3 = img.clone().requires_grad_()
    face_composite(x3, face).backward(g)
    assert same_bits(x3.grad, x2.grad)
    f3 = face.clone().requires_grad_()
    face_composite(img, f3).backward(g)
    assert same_bits(f3.grad, f2.grad)


@pytest.mark.gpu
def test_unbatched_and_strided_inputs(dev):
    renders, face, face_r, gt = on(dev, *inputs(1, 45, 61, seed=2))
    un = {r: {k: t[0] for k, t in v.items()} for r, v in renders.items()}
    with torch.no_grad():
        check_outputs(CP.test_outputs(un, face[0], face_r[0], gt[0]), CP.test_outputs_reference(renders, face, face_r, gt))
    wide = torch.zeros(1, 3, 45, 64, device=dev)
    wide[..., :61] = renders["scene_human"]["img"]
    img = wide[..., :61]
    assert not img.is_contiguous()
    assert same_bits(face_composite(img, face), face_composite_reference(img, face))


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W", [(2, 31, 37), (1, 1080, 1920)])
def test_repeatable_and_every_element_written(dev, N, H, W):
    renders, face, face_r, gt = on(dev, *inputs(N, H, W, seed=11))
    with torch.no_grad():
        a = CP.test_outputs(renders, face, face_r, gt)
        b = CP.test_outputs(renders, face, face_r, gt)
        with poisoned():
            c = CP.test_outputs(renders, face, face_r, gt)
            assert torch.empty(4, device=dev).isnan().all()  # the fill is on
    for k in COMPOSITE_KEYS:
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k
        assert torch.equal(a[k].view(torch.int32), c[k].view(torch.int32)), k
    assert torch.equal(a["png"], b["png"]) and torch.equal(a["png"], c["png"])
    x, f = renders["scene_human"]["img"].clone().requires_grad_(), face.clone().requires_grad_()
    g = torch.randn(N, 3, H, W, device=dev)
    res = []
    for poison in (False, False, True):
        x.grad = f.grad = None
        if poison:
            with poisoned():
                y = face_composite(x, f)
                y.backward(g)
        else:
            y = face_composite(x, f)
            y.backward(g)
        res.append((y.detach(), x.grad, f.grad))
    for r in res[1:]:
        for u, v in zip(res[0], r):
            assert torch.equal(u.view(torch.int32), v.view(torch.int32))


@pytest.mark.gpu
def test_no_host_sync(dev):
    renders, face, face_r, gt = on(dev, *inputs(1, 512, 512, seed=4))
    x, f = renders["scene_human"]["img"].clone().requires_grad_(), face.clone().requires_grad_()
    g = torch.randn(1, 3, 512, 512, device=dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.no_grad():
            CP.test_outputs(renders, face, face_r, gt)
        face_composite(x, f).backward(g)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_cuda_graph_replays_new_inputs(dev):
    N, H, W = 1, 512, 512
    static = on(dev, *inputs(N, H, W, seed=20))
    renders, face, face_r, gt = static
    x = renders["scene_human"]["img"].clone().requires_grad_()
    f = face.clone().requires_grad_()
    g = torch.randn(N, 3, H, W, device=dev)

    def step():
        with torch.no_grad():
            o = CP.test_outputs(renders, face, face_r, gt)
        x.grad = f.grad = None
        y = face_composite(x, f)
        y.backward(g)
        return o, y, x.grad, f.grad

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o, y, gx, gf = step()
    for seed in (21, 22):
        new = on(dev, *inputs(N, H, W, seed=seed))
        for r in RENDERS:
            for k, t in new[0][r].items():
                renders[r][k].copy_(t)
        face.copy_(new[1])
        face_r.copy_(new[2])
        gt.copy_(new[3])
        with torch.no_grad():
            x.copy_(renders["scene_human"]["img"])
            f.copy_(face)
        g.copy_(torch.randn(N, 3, H, W, device=dev))
        graph.replay()
        torch.cuda.synchronize()
        check_outputs(o, CP.test_outputs_reference(renders, face, face_r, gt))
        x2, f2 = x.detach().clone().requires_grad_(), f.detach().clone().requires_grad_()
        ref = face_composite_reference(x2, f2)
        ref.backward(g)
        assert same_bits(y, ref) and same_bits(gx, x2.grad) and same_bits(gf, f2.grad)


@pytest.mark.gpu
def test_test_pass_end_to_end_c4(dev):
    """TrainingFrameRenderer under no_grad with bg_human = ones, two FaceMeshRenderer calls, then test_outputs: the
    model.py expressions on the same renders, and NeumanScores of the refined composed image equal to NeumanScores of
    its PNG bytes decoded by cv2, as eval_neuman reads them."""
    cv2 = pytest.importorskip("cv2")
    from test_neuman_reference import alex_weights
    from exavatar_release_b200 import FaceMeshRenderer, NeumanScores, TrainingFrameRenderer
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.synthetic import WORKLOADS, make_face_mesh, make_human_mesh, make_population_assets
    from test_compose_reference import model_py_test
    wl = WORKLOADS["C4"]
    H, W = wl.height, wl.width
    scene, human, refined = make_population_assets("C4", seed=0, device=dev)
    frame = TrainingFrameRenderer(scene["mean_3d"].shape[0], human["mean_3d"].shape[0], (H, W), dev,
                                  {"A": 1_000_000, "B": 1_000_000})
    cam = look_at_cam_param(0.0, (H, W), device=dev)
    fm = make_face_mesh()
    verts = make_human_mesh()["verts"][fm["vertex_idx"]].contiguous().to(dev)
    fr = FaceMeshRenderer(fm["vertex_uv"], fm["face_uv"], fm["faces"], verts.shape[0], device=dev)
    tex = fm["texture"].to(dev)[None]
    gt = torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(3)).to(dev)
    with torch.no_grad():
        renders = frame(scene, human, refined, cam, torch.ones(3, device=dev))
        face = fr(tex, verts[None], cam, (H, W))
        face_r = fr(tex, (verts + 0.002)[None], cam, (H, W))
        out = CP.test_outputs(renders, face, face_r, gt)
    assert float((face[:, 3] == 1).float().sum()) > 300  # the face covers pixels
    stacked = {r: {k: renders[r][k].reshape(1, -1, H, W) for k in ("img", "mask")} for r in RENDERS}
    want = model_py_test(stacked, face, face_r)
    for k in want:
        assert same_bits(out[k], want[k]), k
    np.testing.assert_array_equal(out["png"].cpu().numpy(), CP.test_outputs_reference(stacked, face, face_r, gt)["png"])
    assert float((renders["human_refined"]["mask"] > 0.9).float().mean()) > 0.01  # both composite branches are taken

    feats, lins = alex_weights()
    neuman = NeumanScores(feats, lins, dev)
    a = neuman(out["scene_human_img_refined_composed"], gt)
    ok, buf = cv2.imencode(".png", out["png"][8, 0].cpu().numpy())
    assert ok
    read = cv2.imdecode(buf, cv2.IMREAD_COLOR)[:, :, ::-1].transpose(2, 0, 1) / 255  # eval_neuman's imread / 255
    b = neuman(torch.from_numpy(read.astype(np.float32)).to(dev)[None], gt)
    assert torch.equal(a, b), (a, b)
