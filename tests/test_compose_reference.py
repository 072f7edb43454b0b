"""The image composites (`compose.face_composite`, `compose.test_outputs`, csrc/compose.cu) without a device: the
references' bytes against a real cv2 PNG round trip, the references against model.py's expressions as written, and the
C ABI (struct sizes, validation before any launch)."""
import ctypes as C

import numpy as np
import pytest
import torch

from util import workload_settings  # noqa: F401  (path setup)
from exavatar_release_b200 import _lib as L
from exavatar_release_b200 import compose as CP  # the module: pytest would collect its test_* names
from exavatar_release_b200.compose import COMPOSITE_KEYS, PNG_ORDER, RENDER_KEYS, face_composite_reference, png_bytes
from exavatar_release_b200.plan import RENDERS

cv2 = pytest.importorskip("cv2")
FAKE = 0x1000  # never dereferenced: validation fails before any launch


def special_values():
    """float32 values whose bytes exercise cv2's conversion: every code k / 255, the exact ties fl(x 255) = k + 0.5 that
    exist, values just around the ties, below 0 and above 1, +-inf, NaN, -0 and values past 2^31 / 255."""
    k = np.arange(256, dtype=np.float64)
    codes = (k / 255).astype(np.float32)
    ties = []
    for t in k[:-1] + 0.5:
        x = np.float32(t / 255)
        for _ in range(4):  # walk a few ulps to the value whose product rounds to the tie exactly
            v = np.float32(x * np.float32(255))
            if v == t:
                ties += [x, np.nextafter(x, np.float32(0)), np.nextafter(x, np.float32(2))]
                break
            x = np.nextafter(x, np.float32(2) if v < t else np.float32(0))
    big = np.float32(2.0 ** 31 / 255)
    extra = np.array([-0.0, -1e-3, -0.5 / 255, -0.6 / 255, -1.0, 1.0 + 1e-3, 1.5, 300.0, np.inf, -np.inf, np.nan,
                      big, np.nextafter(big, np.float32(0)), -big, 1e30, -1e30], np.float32)
    return np.concatenate([codes, np.array(ties, np.float32), extra]), len(ties) // 3


def cv2_bytes(chw: np.ndarray) -> np.ndarray:
    """What test.py's cv2.imwrite stores for a float32 (3,H,W) image, read back with cv2.imdecode (BGR uint8)."""
    ok, buf = cv2.imencode(".png", chw.transpose(1, 2, 0)[:, :, ::-1] * 255)
    assert ok
    return cv2.imdecode(buf, cv2.IMREAD_UNCHANGED)


def inputs(N, H, W, seed=0):
    """Renders, masks, face renders and gt with the cases the expressions distinguish: uncovered face pixels (-1 in
    every channel), face[3] at 1, just below 1, fractional, -1 and 0, face colours that are -1 on a covered pixel,
    masks around 0.9, and -0 renders."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g)  # noqa: E731
    img = {r: rnd(N, 3, H, W) * 1.2 - 0.1 for r in RENDERS}
    for r in RENDERS:
        img[r][rnd(N, 3, H, W) < 0.1] = -0.0
        img[r][rnd(N, 3, H, W) < 0.05] = 0.0
    masks = {}
    for r in ("human", "human_refined"):
        m = rnd(N, 1, H, W)
        pick = rnd(N, 1, H, W)
        m[pick < 0.2] = 0.9
        m[(pick >= 0.2) & (pick < 0.3)] = float(np.nextafter(np.float32(0.9), np.float32(1)))
        m[(pick >= 0.3) & (pick < 0.4)] = 1.0
        m[(pick >= 0.4) & (pick < 0.5)] = 0.0
        masks[r] = m
    faces = []
    for _ in range(2):
        f = rnd(N, 4, H, W)
        a = rnd(N, 1, H, W)
        f[:, 3:][a < 0.3] = 1.0
        f[:, 3:][(a >= 0.3) & (a < 0.4)] = float(np.nextafter(np.float32(1), np.float32(0)))
        f[:, 3:][(a >= 0.4) & (a < 0.5)] = 0.0
        cover = (rnd(N, 1, H, W) < 0.35).expand(N, 4, H, W)
        f[cover] = -1.0  # no face: every channel -1
        f[:, :3][rnd(N, 3, H, W) < 0.05] = -1.0  # a colour channel of -1 on its own
        faces.append(f)
    renders = {r: {"img": img[r]} for r in RENDERS}
    for r in ("human", "human_refined"):
        renders[r]["mask"] = masks[r]
    return renders, faces[0], faces[1], rnd(N, 3, H, W)


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Bitwise equality, every NaN counted equal to every NaN."""
    if a.shape != b.shape:
        return False
    a, b = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    nan = lambda t: (t & 0x7fffffff) > 0x7f800000  # noqa: E731
    return bool(((a == b) | (nan(a) & nan(b))).all())


def test_png_bytes_equal_a_real_cv2_png_round_trip():
    vals, n_ties = special_values()
    assert n_ties > 200  # most ties k + 0.5 are reachable as fl(x 255)
    W = 64
    vals = np.concatenate([vals, np.zeros(-len(vals) % (3 * W), np.float32)])
    img = vals.reshape(3, -1, W)
    np.testing.assert_array_equal(png_bytes(img), cv2_bytes(img))
    np.testing.assert_array_equal(png_bytes(img[::-1].copy()), cv2_bytes(img[::-1].copy()))


@pytest.mark.parametrize("N,H,W", [(1, 31, 37), (2, 16, 24)])
def test_reference_bytes_equal_cv2_for_all_ten_images(N, H, W):
    renders, face, face_r, gt = inputs(N, H, W, seed=3)
    vals, _ = special_values()
    flat = renders["scene"]["img"].view(-1)  # the special values go through the first image and gt
    flat[:len(vals)] = torch.from_numpy(vals)
    gt.view(-1)[-len(vals):] = torch.from_numpy(vals[::-1].copy())
    ref = CP.test_outputs_reference(renders, face, face_r, gt)
    assert ref["png"].shape == (10, N, H, W, 3) and ref["png"].dtype == np.uint8
    for k, name in enumerate(PNG_ORDER):
        t = gt if name == "gt" else ref[name]
        for n in range(N):
            np.testing.assert_array_equal(ref["png"][k, n], cv2_bytes(t[n].numpy()), err_msg=name)
    assert CP.test_outputs_reference(renders, face, face_r)["png"].shape == (9, N, H, W, 3)
    assert "png" not in CP.test_outputs_reference(renders, face, face_r, gt, png=False)


def model_py_test(renders, face_renders, face_renders_refined):
    """avatar/main/model.py:262-276 as written, on the stacked renders."""
    scene_renders, human_renders, scene_human_renders, human_renders_refined, scene_human_renders_refined = (
        renders[r] for r in RENDERS)
    out = {}
    out['scene_img'] = scene_renders['img']
    out['human_img'] = human_renders['img']
    out['scene_human_img'] = scene_human_renders['img']
    out['human_img_refined'] = human_renders_refined['img']
    out['scene_human_img_refined'] = scene_human_renders_refined['img']
    is_face = (face_renders[:, :3] != -1).float() * face_renders[:, 3:]
    out['human_face_img'] = human_renders['img'] * (1 - is_face) + face_renders[:, :3] * is_face
    is_face = (face_renders_refined[:, :3] != -1).float() * face_renders_refined[:, 3:]
    out['human_face_img_refined'] = human_renders_refined['img'] * (1 - is_face) + face_renders_refined[:, :3] * is_face
    is_fg = human_renders['mask'] > 0.9
    out['scene_human_img_composed'] = is_fg * human_renders['img'] + (1 - is_fg.float()) * scene_human_renders['img']
    is_fg = human_renders_refined['mask'] > 0.9
    out['scene_human_img_refined_composed'] = is_fg * human_renders_refined['img'] + (1 - is_fg.float()) * \
        scene_human_renders_refined['img']
    return out


@pytest.mark.parametrize("seed", [0, 1])
def test_test_reference_is_model_py(seed):
    renders, face, face_r, gt = inputs(2, 19, 23, seed)
    ref = CP.test_outputs_reference(renders, face, face_r, gt, png=False)
    want = model_py_test(renders, face, face_r)
    assert set(ref) == set(RENDER_KEYS + COMPOSITE_KEYS)
    for k in want:
        assert same_bits(ref[k], want[k]), k
    # the soft mask's -0 (face colour -1, face[3] = -1) meets a -0 render: torch's expression gives +0
    f = face.clone()
    f[0, :, 0, 0] = -1.0
    renders["human"]["img"][0, :, 0, 0] = -0.0
    out = CP.test_outputs_reference(renders, f, face_r, png=False)["human_face_img"][0, :, 0, 0]
    assert same_bits(out, torch.zeros(3)) and same_bits(out, model_py_test(renders, f, face_r)["human_face_img"][0, :, 0, 0])


def test_face_reference_is_model_py_and_its_gradient():
    renders, face, _, _ = inputs(2, 17, 29, seed=5)
    img = renders["scene_human"]["img"]
    x, f = img.clone().requires_grad_(), face.clone().requires_grad_()
    out = face_composite_reference(x, f)
    is_face = ((face[:, :3] != -1) * (face[:, 3:] == 1)).float()  # model.py:200-201
    assert same_bits(out, img * (1 - is_face) + face[:, :3] * is_face)
    assert 0 < float(is_face.mean()) < 1
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(1))
    g[0, 0, :2] = -0.0
    out.backward(g)
    assert same_bits(x.grad, g * (1 - is_face))
    assert same_bits(f.grad[:, :3], g * is_face)
    assert same_bits(f.grad[:, 3], torch.zeros_like(f.grad[:, 3]))


# ---------------------------------------------------------------------------------------------------------------------
# The C ABI without a device
# ---------------------------------------------------------------------------------------------------------------------

def test_struct_sizes():
    assert C.sizeof(L.B2RFaceComposite) == 32
    assert C.sizeof(L.B2RTestOutputs) == 96


def test_face_composite_validation():
    lib = L.load()
    good = dict(width=8, height=4, n_images=1, img=FAKE, face=FAKE)
    fwd = lambda p, out=FAKE: lib.b2r_face_composite_forward(C.byref(p), out, None)  # noqa: E731
    bwd = lambda p, d=FAKE, di=FAKE, df=FAKE: lib.b2r_face_composite_backward(C.byref(p), d, di, df, None)  # noqa: E731
    assert lib.b2r_face_composite_forward(None, FAKE, None) == -1
    assert lib.b2r_face_composite_backward(None, FAKE, FAKE, FAKE, None) == -1
    for bad in ({"width": 0}, {"height": -3}, {"n_images": 0}, {"n_images": -1}, {"face": None},
                {"width": 1 << 16, "height": 1 << 16, "n_images": 16}):
        p = L.B2RFaceComposite(**{**good, **bad})
        assert fwd(p) == -1, bad
        assert bwd(p) == -1, bad
    p = L.B2RFaceComposite(**{**good, "img": None})
    assert fwd(p) == -1
    p = L.B2RFaceComposite(**good)
    assert fwd(p, out=None) == -1
    assert bwd(p, d=None) == -1
    assert bwd(p, di=None, df=None) == -1
    assert lib.b2r_launch_count() == 0


def test_test_outputs_validation():
    lib = L.load()
    comp = (L._fp * 4)(FAKE, FAKE, FAKE, FAKE)

    def make(**kw):
        p = L.B2RTestOutputs(width=kw.get("width", 8), height=kw.get("height", 4), n_images=kw.get("n", 2), gt=None)
        for i in range(5):
            p.render[i] = FAKE
        for k in range(2):
            p.mask[k] = p.face[k] = FAKE
        return p

    call = lambda p, c=comp: lib.b2r_test_outputs(C.byref(p) if p is not None else None, c, None, None)  # noqa: E731
    assert call(None) == -1
    for kw in ({"width": 0}, {"height": -1}, {"n": 0}, {"n": -2}):
        assert call(make(**kw)) == -1, kw
    for field, idx in (("render", i) for i in range(5)):
        p = make()
        getattr(p, field)[idx] = None
        assert call(p) == -1
    for field in ("mask", "face"):
        for k in range(2):
            p = make()
            getattr(p, field)[k] = None
            assert call(p) == -1, (field, k)
    assert call(make(), c=None) == -1
    for k in range(4):
        c = (L._fp * 4)(FAKE, FAKE, FAKE, FAKE)
        c[k] = None
        assert call(make(), c=c) == -1, k
    assert lib.b2r_launch_count() == 0


def test_python_checks_without_a_device():
    renders, face, face_r, gt = inputs(1, 8, 8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        CP.face_composite(renders["scene_human"]["img"], face)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        with torch.no_grad():
            CP.test_outputs(renders, face, face_r, gt)
    with pytest.raises(ValueError, match="human_refined"):
        bad = {r: dict(v) for r, v in renders.items()}
        del bad["human_refined"]["mask"]
        CP.test_outputs(bad, face, face_r, gt)
    with pytest.raises(RuntimeError, match="no_grad"):
        CP.test_outputs(renders, face.clone().requires_grad_(), face_r, gt)
