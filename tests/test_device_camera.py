"""Render settings from a CUDA camera on the device: `b2r_camera_setup`, `B2RScene.tanfov` and
`renderer.device_render_settings`.

CPU: a float64 / float32 restatement of the camera block's arithmetic against camera.py (the host mirror) on 10 000
random cameras, and the C ABI of the new field and entry point.
GPU: the block against the reference's own CUDA expressions; the pointer path against the by-value path, bit for bit
in every forward output and tile list, gradients up to the backward's float-atomic reordering (single render with an
SH scene, the five-render training frame eager and captured, general cameras); one capture
serving six focal lengths; a C4 frame from the camera to the loss's backward without a host synchronisation; invalid
cameras cull everything without a fault.
"""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

from util import ROOT  # noqa: F401  (path setup)
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.camera import get_fov, get_proj_matrix, get_view_matrix

FAKE = 0x1000  # never dereferenced: validation fails before any launch
f32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------
# the block's arithmetic, restated (csrc/camera.cu)
# ---------------------------------------------------------------------------------------------------------------------

def fov_restated(focal, W, H):
    """fp32 fov as torch's device kernels evaluate 2 * atan(W / (2 f)): reciprocal(2 f) * W, atan (here fp64 rounded
    once, where the device runs atanf), x 2."""
    out = []
    for f, n in ((focal[0], W), (focal[1], H)):
        x = (f32(1) / (f32(2) * f32(f))) * f32(n)
        out.append(f32(2) * f32(math.atan(float(x))))
    return out


def proj_restated(fov):
    """transforms.py:43-64 in fp64 from the fp32 fov, rounded once; stored transposed ([4c + r])."""
    top = math.tan(float(fov[1]) / 2) * 0.01
    right = math.tan(float(fov[0]) / 2) * 0.01
    m = np.zeros((4, 4), np.float64)
    m[0, 0] = 2.0 * 0.01 / (right - (-right))
    m[1, 1] = 2.0 * 0.01 / (top - (-top))
    m[0, 2] = (right + -right) / (right - -right)
    m[1, 2] = (top + -top) / (top - -top)
    m[3, 2] = 1.0
    m[2, 2] = 1.0 * 100 / (100 - 0.01)
    m[2, 3] = -(100 * 0.01) / (100 - 0.01)
    return m.astype(f32).T.copy()


def mm_left_to_right(a, b):
    """(4,4) x (4,4) in fp32, every entry's four rounded products summed left to right."""
    out = np.zeros((4, 4), f32)
    for i in range(4):
        for j in range(4):
            s = f32(a[i, 0] * b[0, j])
            for k in range(1, 4):
                s = f32(s + f32(a[i, k] * b[k, j]))
            out[i, j] = s
    return out


def block_restated(R, t, focal, W, H, fov=None):
    """(view, full, campos, tanfov) of one camera; `fov` overrides the restated fov bits."""
    R, t = np.asarray(R, f32), np.asarray(t, f32)
    fov = fov_restated(focal, W, H) if fov is None else fov
    view = np.zeros((4, 4), f32)
    view[:3, :3] = R.T
    view[3, :3] = t
    view[3, 3] = 1
    full = mm_left_to_right(view, proj_restated(fov))
    Rd, td = R.astype(np.float64), t.astype(np.float64)
    campos = np.array([-((Rd[0, c] * td[0] + Rd[1, c] * td[1]) + Rd[2, c] * td[2]) for c in range(3)]).astype(f32)
    tanfov = [f32(math.tan(float(f32(x * f32(0.5))))) for x in fov]
    return view, full, campos, tanfov


def random_cameras(n, seed):
    """n cameras: random rotation, |t| up to 3, focal 50..10 000 px with fx != fy, sizes 96x128 .. 1080x1920."""
    rng = np.random.default_rng(seed)
    cams = []
    for _ in range(n):
        q, r = np.linalg.qr(rng.standard_normal((3, 3)))
        q = q * np.sign(np.diag(r))
        if np.linalg.det(q) < 0:
            q[:, 0] = -q[:, 0]
        H, W = int(rng.integers(96, 1081)), int(rng.integers(128, 1921))
        fx = f32(np.exp(rng.uniform(np.log(50), np.log(10000))))
        fy = f32(fx * f32(rng.uniform(0.7, 1.4)))
        if fy == fx:
            fy = np.nextafter(fx, f32(np.inf))
        cams.append((q.astype(f32), rng.uniform(-3, 3, 3).astype(f32), np.array([fx, fy], f32), W, H))
    return cams


def ulps(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

def test_restated_block_against_the_host_mirror_on_10000_cameras():
    """view bit-equal; projection and full projection bit-equal given the host mirror's fov bits; tan(fov) within two
    ulps (one in most cases); campos (rigid inverse) within 16 eps max|campos| of the host mirror's LU inverse."""
    worst_campos, tan_off, tan_two = 0.0, 0, 0
    for R, t, focal, W, H in random_cameras(10_000, seed=1):
        Rt, tt, ft = torch.from_numpy(R), torch.from_numpy(t), torch.from_numpy(focal)
        fov_h = get_fov(ft, None, (H, W))
        view_h = get_view_matrix(Rt, tt).permute(1, 0)
        proj_h = get_proj_matrix(ft, None, (H, W), 0.01, 100, 1.0).permute(1, 0)
        full_h = torch.mm(view_h, proj_h)
        campos_h = view_h.inverse()[3, :3].numpy()
        tan_h = [f32(float(torch.tan(fov_h[k] / 2))) for k in range(2)]

        view, full, campos, tanfov = block_restated(R, t, focal, W, H, fov=[f32(float(x)) for x in fov_h])
        assert np.array_equal(view, view_h.numpy())
        assert np.array_equal(proj_restated([f32(float(x)) for x in fov_h]), proj_h.numpy())
        assert np.array_equal(full, full_h.numpy()), (focal, W, H)

        _, _, _, tanfov = block_restated(R, t, focal, W, H)  # the block's own fov bits
        d = ulps(tanfov, tan_h)
        # one ulp from tan itself, one more where the fov's atan already differed by one ulp
        assert d.max() <= 2, (focal, W, H, tanfov, tan_h)
        tan_off += int((d > 0).any())
        tan_two += int((d > 1).any())
        scale = float(np.abs(campos_h).max())
        err = float(np.abs(campos.astype(np.float64) - campos_h).max()) / (float(np.finfo(f32).eps) * scale)
        worst_campos = max(worst_campos, err)
    assert worst_campos <= 16, worst_campos
    # the host mirror's CPU atan / tan differ from fp64-rounded values on a minority of cameras
    assert tan_off < 2_000 and tan_two < 100, (tan_off, tan_two)
    print(f"tan(fov) off by 1 / 2 ulps on {tan_off} / {tan_two} cameras; campos within {worst_campos:.1f} eps")


def test_scene_struct_carries_the_device_tanfov_pointer():
    assert L.B2RScene.tanfov.offset == L.B2RScene.tanfovy.offset + 8  # 4 bytes of padding to the pointer
    assert L.B2RScene.bg.offset == L.B2RScene.tanfov.offset + 8
    assert L.B2RScene().tanfov is None  # a zeroed struct: the by-value floats


def test_device_tanfov_skips_the_host_check_and_a_zeroed_struct_validates_as_before():
    lib = L.load()
    n0 = lib.b2r_launch_count()
    sc = L.B2RScene()
    sc.P, sc.width, sc.height = 10, 32, 32
    sc.bg = sc.viewmatrix = sc.projmatrix = sc.campos = FAKE
    sc.means3D = sc.opacities = sc.colors_precomp = sc.scales = sc.rotations = FAKE
    ws = L.B2RWorkspace()
    ws.ctx, ws.ctx_bytes = FAKE, 16  # too small on purpose: a scene that validates reaches the workspace check (-2)
    out = L.B2RForwardOutputs()
    fwd = lambda: lib.b2r_forward(C.byref(sc), C.byref(ws), C.byref(out), None)
    assert fwd() == -1                  # zeroed tanfovx / tanfovy, no pointer: rejected as before
    sc.tanfovx, sc.tanfovy = 0.5, -1.0
    assert fwd() == -1
    sc.tanfovy = 0.5
    assert fwd() == -2
    sc.tanfovx = sc.tanfovy = 0.0
    sc.tanfov = FAKE                    # device values are not read on the host: the floats are ignored
    assert fwd() == -2
    sc.tanfovx = sc.tanfovy = float("nan")
    assert fwd() == -2
    assert lib.b2r_launch_count() == n0


def test_camera_setup_validates_on_the_host():
    lib = L.load()
    n0 = lib.b2r_launch_count()
    assert lib.b2r_camera_setup(None, FAKE, FAKE, 32, 32, FAKE, None) == -1
    assert lib.b2r_camera_setup(FAKE, None, FAKE, 32, 32, FAKE, None) == -1
    assert lib.b2r_camera_setup(FAKE, FAKE, None, 32, 32, FAKE, None) == -1
    assert lib.b2r_camera_setup(FAKE, FAKE, FAKE, 32, 32, None, None) == -1
    assert lib.b2r_camera_setup(FAKE, FAKE, FAKE, 0, 32, FAKE, None) == -1
    assert lib.b2r_camera_setup(FAKE, FAKE, FAKE, 32, -1, FAKE, None) == -1
    assert lib.b2r_launch_count() == n0


def test_device_render_settings_rejects_a_cpu_camera():
    from exavatar_release_b200.camera import look_at_cam_param
    from exavatar_release_b200.renderer import device_render_settings
    with pytest.raises(RuntimeError, match="CUDA"):
        device_render_settings((64, 48), look_at_cam_param(10.0, (64, 48)), torch.ones(3))


def test_rasterizer_takes_tensor_tanfov_only_as_a_cuda_pair():
    from exavatar_release_b200.rasterizer import GaussianRasterizationSettings, device_tanfov
    st = GaussianRasterizationSettings(8, 8, 0.5, 0.5, torch.ones(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3),
                                       False, False)
    assert device_tanfov(st) is None
    with pytest.raises(TypeError):
        device_tanfov(st._replace(tanfovx=torch.tensor(0.5)))
    with pytest.raises(RuntimeError, match="CUDA"):
        device_tanfov(st._replace(tanfovx=torch.tensor(0.5), tanfovy=torch.tensor(0.5)))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _device_cam(R, t, focal, dev):
    return {"R": torch.from_numpy(np.asarray(R, f32)).to(dev), "t": torch.from_numpy(np.asarray(t, f32)).to(dev),
            "focal": torch.from_numpy(np.asarray(focal, f32)).to(dev), "princpt": torch.zeros(2, device=dev)}


@pytest.mark.gpu
def test_block_matches_the_reference_cuda_expressions(dev):
    """tan(fov) bit-equal to torch.tan(get_fov(.) / 2) on CUDA tensors; view bit-equal; full projection bit-equal to the
    left-to-right product of the view with get_proj_matrix of the CUDA fov (math.tan in fp64); campos = -R^T t in fp64
    rounded once."""
    from exavatar_release_b200.renderer import device_render_settings
    for R, t, focal, W, H in random_cameras(300, seed=2):
        cam = _device_cam(R, t, focal, dev)
        st = device_render_settings((H, W), cam, torch.ones(3, device=dev))
        block = torch.cat((st.viewmatrix.reshape(16), st.projmatrix.reshape(16), st.campos,
                           st.tanfovx.reshape(1), st.tanfovy.reshape(1))).cpu().numpy()
        fov = get_fov(cam["focal"], None, (H, W))
        tan_ref = torch.tan(fov / 2).cpu().numpy()
        assert np.array_equal(block[35:37], tan_ref), (focal, W, H, block[35:37], tan_ref)
        view_ref = get_view_matrix(cam["R"], cam["t"]).permute(1, 0).cpu().numpy()
        assert np.array_equal(block[0:16].reshape(4, 4), view_ref)
        proj_ref = get_proj_matrix(cam["focal"], None, (H, W), 0.01, 100, 1.0).permute(1, 0).cpu().numpy()
        assert np.array_equal(block[16:32].reshape(4, 4), mm_left_to_right(view_ref, proj_ref)), (focal, W, H)
        _, _, campos, _ = block_restated(R, t, focal, W, H)
        assert np.array_equal(block[32:35], campos)


def _same_grads(x, y, what):
    """The backward composite adds screen-space gradients with float atomics, so two runs of the SAME settings differ
    in the last bits of a few sums; gradients are compared within that reordering (1e-5 of the largest magnitude)."""
    for i, (u, v) in enumerate(zip(x, y)):
        assert float((u - v).abs().max()) <= 1e-5 * float(v.abs().max()) + 1e-12, (what, i)


def _float_twin(st):
    """The same settings with tan(fov) read back into Python floats: the by-value path."""
    return st._replace(tanfovx=float(st.tanfovx), tanfovy=float(st.tanfovy))


def _render(st, a, dev, sh):
    from exavatar_release_b200 import rasterizer as rz
    leaves = {k: a[k].to(dev).clone().requires_grad_() for k in ("mean_3d", "scale", "rotation", "opacity",
                                                                  "shs" if sh else "rgb")}
    m2d = torch.zeros_like(leaves["mean_3d"], requires_grad=True)
    color, radii, depth, alpha = rz.GaussianRasterizer(st._replace(sh_degree=3 if sh else 0))(
        means3D=leaves["mean_3d"], means2D=m2d, opacities=leaves["opacity"], scales=leaves["scale"],
        rotations=leaves["rotation"], **({"shs": leaves["shs"]} if sh else {"colors_precomp": leaves["rgb"]}))
    g = torch.Generator(device=dev).manual_seed(5)
    gc, gd, ga = (torch.randn(x.shape, generator=g, device=dev) for x in (color, depth, alpha))
    ((color * gc).sum() + (depth * gd).sum() + (alpha * ga).sum()).backward()
    return [color, radii, depth, alpha], [m2d.grad] + [leaves[k].grad for k in sorted(leaves)]


def _plan_lists(st, a, dev):
    """Per-tile sorted id lists of one FramePlan forward: (num_dups, ids[:num_dups])."""
    from exavatar_release_b200.plan import FramePlan
    H, W = st.image_height, st.image_width
    plan = FramePlan(a["mean_3d"].shape[0], W, H, 400_000, dev)
    assets = {k: a[k].to(dev) for k in ("mean_3d", "scale", "rotation", "opacity", "rgb")}
    plan.forward(plan.scene(0, st, assets))
    n = plan.status()["num_dups"]
    return n, plan.ids[:n].clone(), plan.color.clone(), plan.radii.clone()


@pytest.mark.gpu
@pytest.mark.parametrize("cam_name", ["c61x45", "c203x131", "c512"])
def test_pointer_path_equals_by_value_path_single_render(dev, cam_name):
    """The C2-style single render through GaussianRasterizer, an SH scene and an RGB scene, and the tile lists of a
    FramePlan: device settings and their float twin give bit-identical images, depth, alpha, radii and lists, and the
    same gradients (up to the float-atomic reordering of any two runs), under general cameras (pitch, roll, fx != fy,
    the frustum-clamp band)."""
    from test_general_cameras import _cat, camera, case_population
    from exavatar_release_b200.renderer import device_render_settings
    st_cpu, a = case_population(cam_name, "clamp", sh=True, boundary=False)
    _, b = case_population(cam_name, "plain", sh=True, boundary=False)
    a = _cat({k: v for k, v in a.items() if k != "_pcam"}, {k: v for k, v in b.items() if k != "_pcam"})
    H, W = st_cpu.image_height, st_cpu.image_width
    st = device_render_settings((H, W), camera(cam_name, dev), torch.tensor([0.2, 0.6, 0.9], device=dev))
    for sh in (False, True):
        (x, gx), (y, gy) = _render(st, a, dev, sh), _render(_float_twin(st), a, dev, sh)
        for i, (u, v) in enumerate(zip(x, y)):
            assert torch.equal(u, v), (cam_name, sh, i)
        _same_grads(gx, gy, (cam_name, sh))
        assert int((x[1] > 0).sum()) > 100
    n_d, ids_d, col_d, rad_d = _plan_lists(st, a, dev)
    n_f, ids_f, col_f, rad_f = _plan_lists(_float_twin(st), a, dev)
    assert n_d == n_f > 0 and torch.equal(ids_d, ids_f) and torch.equal(col_d, col_f) and torch.equal(rad_d, rad_f)


def _frame_case(cam_name, dev):
    from test_general_cameras import case_population
    strip = lambda p: {k: v.to(dev) for k, v in p.items() if k != "_pcam"}  # noqa: E731
    st, s = case_population(cam_name, "clamp", boundary=False)
    _, h = case_population(cam_name, "plain", boundary=False)
    g = torch.Generator().manual_seed(11)
    # the refined set has the human's rows (one skinning, two offsets in ExAvatar): moved and re-shaped a little
    r = dict(h, mean_3d=h["mean_3d"] + 0.02 * torch.randn(h["mean_3d"].shape, generator=g),
             scale=h["scale"] * (0.8 + 0.4 * torch.rand(h["scale"].shape, generator=g)))
    return (st.image_height, st.image_width), strip(s), strip(h), strip(r)


def _run_frame(fr, st, scene, human, refined, bg_h, seed):
    from exavatar_release_b200.plan import RENDERS
    leaves = [{k: v.clone().requires_grad_() for k, v in p.items()} for p in (scene, human, refined)]
    out = fr(*leaves, None, bg_h, raster_settings=st)
    g = torch.Generator(device=bg_h.device).manual_seed(seed)
    loss = sum((out[r]["img"] * torch.randn(out[r]["img"].shape, generator=g, device=bg_h.device)).sum() for r in RENDERS)
    loss.backward()
    res = [out[r][k] for r in RENDERS for k in ("img", "depthmap", "mask", "radius")]
    return res, [out["scene"]["mean_2d"].grad] + [p[k].grad for p in leaves for k in sorted(p)]


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("cam_name", ["c61x45", "c203x131", "c512"])
def test_pointer_path_equals_by_value_path_training_frame(dev, cam_name, use_graph):
    """TrainingFrameRenderer's five renders fed device settings == fed their float twin: images, depth, masks and radii
    bit-identical, every gradient equal up to float-atomic reordering, eager and captured, under general cameras."""
    from test_general_cameras import camera
    from exavatar_release_b200 import TrainingFrameRenderer
    from exavatar_release_b200.renderer import device_render_settings
    (H, W), scene, human, refined = _frame_case(cam_name, dev)
    bg_h = torch.tensor([0.3, 0.7, 0.2], device=dev)
    caps = {"A": 1_000_000, "B": 1_000_000}
    fr = {k: TrainingFrameRenderer(scene["mean_3d"].shape[0], human["mean_3d"].shape[0], (H, W), dev, caps,
                                   use_graph=use_graph) for k in ("device", "float")}
    st = device_render_settings((H, W), camera(cam_name, dev), torch.ones(3, device=dev))
    for frame in range(2):
        x, gx = _run_frame(fr["device"], st, scene, human, refined, bg_h, frame)
        y, gy = _run_frame(fr["float"], _float_twin(st), scene, human, refined, bg_h, frame)
        for i, (u, v) in enumerate(zip(x, y)):
            assert torch.equal(u, v), (cam_name, use_graph, frame, i)
        _same_grads(gx, gy, (cam_name, use_graph, frame))
    assert not fr["device"].overflowed()


@pytest.mark.gpu
def test_one_capture_serves_every_focal_length(dev):
    """use_graph=True over six frames whose focal lengths (and rotations) all differ: one capture, and every frame equal
    to the eager renderer fed the same device settings."""
    from test_general_cameras import camera
    from exavatar_release_b200 import TrainingFrameRenderer
    from exavatar_release_b200.renderer import device_render_settings
    (H, W), scene, human, refined = _frame_case("c203x131", dev)
    bg_h = torch.tensor([0.3, 0.7, 0.2], device=dev)
    caps = {"A": 1_000_000, "B": 1_000_000}
    graph, eager = (TrainingFrameRenderer(scene["mean_3d"].shape[0], human["mean_3d"].shape[0], (H, W), dev, caps,
                                          use_graph=g) for g in (True, False))
    base = camera("c203x131", dev)
    focals = set()
    for f in range(6):
        a = math.radians(4.0 * f)
        rot = torch.tensor([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]], device=dev)
        cam = dict(base, R=(base["R"] @ rot).contiguous(), focal=base["focal"] * (0.8 + 0.08 * f))
        focals.add(tuple(cam["focal"].tolist()))
        st = device_render_settings((H, W), cam, torch.ones(3, device=dev))
        x, gx = _run_frame(graph, st, scene, human, refined, bg_h, f)
        y, gy = _run_frame(eager, st, scene, human, refined, bg_h, f)
        for i, (u, v) in enumerate(zip(x, y)):
            assert torch.equal(u, v), (f, i)
        _same_grads(gx, gy, f)
        assert int((x[3] > 0).sum()) > 50  # scene radii: the view is not empty
    assert len(focals) == 6 and len(graph._graphs) == 1


@pytest.mark.gpu
def test_c4_frame_from_camera_to_backward_without_a_host_sync(dev):
    """tools/c4_frame.py's C4 frame -- decode_smplx_pose -> SmplxRig -> nets -> nearest_rows -> skin_gaussians ->
    VertexNormals -> device_render_settings + TrainingFrameRenderer(use_graph=True) -> l1_ssim + regularisers ->
    backward -- with a new camera every frame raises nothing under sync debug mode "error" (after the warm-up frame
    that captures the graphs)."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from bench_human_assets import pose_params
    from c4_frame import FrameArm, make_frame
    from exavatar_release_b200 import decode_smplx_pose
    from exavatar_release_b200.renderer import device_render_settings
    frame, fr = make_frame(dev, use_graph=True)
    fp = {k: v.requires_grad_() for k, v in pose_params(dev).items()}
    step = [0]

    def camera(shape, cam, bg):
        step[0] += 1
        fresh = {k: v.clone() for k, v in cam.items()}
        fresh["focal"] = fresh["focal"] * (1.0 + 0.01 * step[0])
        return device_render_settings(shape, fresh, bg)

    def rig(r, d, x):
        for v in fp.values():
            v.grad = None
        return r(x[0], x[1], decode_smplx_pose(fp)["full_pose"], x[3])

    arm = FrameArm(rig=rig, camera=camera)
    frame(arm)  # warm-up: captures the renderer's graphs, first-use set-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        frame(arm)
        frame(arm)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert len(fr._graphs) == 1 and not fr.overflowed()


@pytest.mark.gpu
@pytest.mark.parametrize("focal", [(0.0, 500.0), (float("nan"), float("nan")), (500.0, 0.0)])
def test_invalid_device_camera_culls_everything(dev, focal):
    """A focal length of 0 or NaN gives a tan(fov) that is not finite and > 0: radii 0, the background image, zero
    gradients, no fault and no CUDA error afterwards."""
    from test_general_cameras import camera, case_population
    from exavatar_release_b200.renderer import device_render_settings
    st_cpu, a = case_population("c61x45", "plain", boundary=False)
    H, W = st_cpu.image_height, st_cpu.image_width
    cam = dict(camera("c61x45", dev), focal=torch.tensor(focal, device=dev))
    bg = torch.tensor([0.2, 0.6, 0.9], device=dev)
    st = device_render_settings((H, W), cam, bg)
    (color, radii, depth, alpha), grads = _render(st, {k: v for k, v in a.items() if k != "_pcam"}, dev, False)
    torch.cuda.synchronize()
    assert int(radii.abs().sum()) == 0
    assert torch.equal(color, bg.view(3, 1, 1).expand_as(color))
    assert int(torch.count_nonzero(depth)) == 0 and int(torch.count_nonzero(alpha)) == 0
    for g in grads:
        assert int(torch.count_nonzero(g)) == 0
    torch.ones(4, device=dev).sum().item()  # the context is healthy
