"""MotionTable and AvatarAnimator (exavatar_release_b200/animator.py): the motion folder read as animate.py reads it,
with its refusals before any upload (no device); on the H100, the animator against the full HumanGaussian chain
through the existing ops (all four stacks, both sets, the refined set discarded) bit for bit, graph replay against
eager with no host sync, the pinned ring, the orbit mode against animate_view_rot.py's lines, and the overflow report."""
import json
import os

import cv2
import numpy as np
import pytest
import torch

from util import ROOT  # noqa: F401  (path setup)
from util import no_host_sync
from util import dev  # noqa: F401
from c4_frame import SyntheticAvatar, write_motion_frame
from exavatar_release_b200.animator import SMPLX_KEYS, MotionTable, read_motion
from exavatar_release_b200.human_assets import POSE_KEYS

EPS = 2.0 ** -23
LENGTHS = {"root_pose": 3, "body_pose": 63, "jaw_pose": 3, "leye_pose": 3, "reye_pose": 3, "lhand_pose": 45,
           "rhand_pose": 45, "expr": 10, "trans": 3}


def _host_frame(seed, H=6, W=8, n_expr=10):
    """Parameters as float64 lists (their fp32 rounding is what the reader must reproduce), nested like ExAvatar's
    files (R as 3 rows), and a random BGR image."""
    g = np.random.default_rng(seed)
    smplx = {k: (0.3 * g.standard_normal(n if k != "expr" else n_expr)).tolist() for k, n in LENGTHS.items()}
    smplx["body_pose"] = np.asarray(smplx["body_pose"]).reshape(21, 3).tolist()
    cam = {"R": (np.eye(3) + 0.01 * g.standard_normal((3, 3))).tolist(), "t": g.standard_normal(3).tolist(),
           "focal": [1000.0 + g.random(), 1001.5], "princpt": [W / 2 + g.random(), H / 2]}
    return smplx, cam, g.integers(0, 256, (H, W, 3), dtype=np.uint8)


def _bits(t):
    return t.contiguous().view(torch.int32)


def test_host_half_reads_the_scripts_values(tmp_path):
    root = str(tmp_path)
    data = {idx: _host_frame(idx) for idx in (100, 2, 10)}
    for idx, d in data.items():
        write_motion_frame(root, idx, *d)
    m = read_motion(root)
    assert m["frame_idx"].tolist() == [2, 10, 100]  # numeric order, not "10" < "100" < "2"
    for i, idx in enumerate((2, 10, 100)):
        with open(os.path.join(root, "smplx_optimized", "smplx_params_smoothed", f"{idx}.json")) as f:
            sp = {k: torch.FloatTensor(v).view(-1) for k, v in json.load(f).items()}
        with open(os.path.join(root, "cam_params", f"{idx}.json")) as f:
            cp = {k: torch.FloatTensor(v) for k, v in json.load(f).items()}
        assert torch.equal(_bits(m["pose"][i]), _bits(torch.cat([sp[k] for k in POSE_KEYS]).view(55, 3)))
        assert torch.equal(_bits(m["expr"][i]), _bits(sp["expr"]))
        assert torch.equal(_bits(m["trans"][i]), _bits(sp["trans"]))
        for k in ("R", "t", "focal", "princpt"):
            assert torch.equal(_bits(m[k][i]), _bits(cp[k])), k
        img = cv2.imread(os.path.join(root, "frames", f"{idx}.png"))
        assert m["frames"][i].dtype == np.uint8 and np.array_equal(m["frames"][i], img)
        assert np.array_equal(img, data[idx][2])


def _break(root, case):
    """Writes a valid three-frame motion, then spoils it as `case` says."""
    for idx in (3, 7, 12):
        smplx, cam, img = _host_frame(idx)
        if idx == 7:
            if case == "missing_key":
                del smplx["jaw_pose"]
            elif case == "short_value":
                smplx["lhand_pose"] = smplx["lhand_pose"][:-1]
            elif case == "expr_length":
                smplx["expr"] = smplx["expr"] + [0.0]
            elif case == "scalar_value":
                smplx["trans"] = 0.5
            elif case == "missing_cam_key":
                del cam["princpt"]
            elif case == "cam_length":
                cam["focal"] = [1000.0]
            elif case == "frame_size":
                img = np.zeros((6, 9, 3), dtype=np.uint8)
        write_motion_frame(root, idx, smplx, cam, img)
    if case == "missing_cam":
        os.remove(os.path.join(root, "cam_params", "7.json"))
    elif case == "missing_png":
        os.remove(os.path.join(root, "frames", "12.png"))
    elif case == "bad_name":
        os.rename(os.path.join(root, "smplx_optimized", "smplx_params_smoothed", "7.json"),
                  os.path.join(root, "smplx_optimized", "smplx_params_smoothed", "seven.json"))
    elif case == "empty":
        for f in os.listdir(os.path.join(root, "smplx_optimized", "smplx_params_smoothed")):
            os.remove(os.path.join(root, "smplx_optimized", "smplx_params_smoothed", f))


@pytest.mark.parametrize("case", ["missing_key", "short_value", "expr_length", "scalar_value", "missing_cam_key",
                                  "cam_length", "frame_size", "missing_cam", "missing_png", "bad_name", "empty"])
def test_host_half_refusals_before_upload(tmp_path, case, monkeypatch):
    _break(str(tmp_path), case)
    uploads = []
    monkeypatch.setattr(torch.Tensor, "to", lambda *a, **k: uploads.append(a) or pytest.fail("uploaded"))
    with pytest.raises(ValueError, match="MotionTable"):
        MotionTable.from_folder(str(tmp_path), "cuda")
    assert not uploads


def test_table_refuses_a_cpu_device(tmp_path):
    _break(str(tmp_path), "none")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        MotionTable.from_folder(str(tmp_path), "cpu")


def test_smplx_keys_are_the_scripts_nine():
    assert SMPLX_KEYS == ("root_pose", "body_pose", "jaw_pose", "leye_pose", "reye_pose", "lhand_pose", "rhand_pose",
                          "expr", "trans")


# ---------------------------------------------------------------------------------------------------------------------
# On the H100: the synthetic C4 avatar (tools/c4_frame.setup's SMPL-X rig, P = 167 618)

N_FRAMES = 6
FRAME_IDX = (2, 10, 100, 101, 250, 1000)
CAPACITY = 1 << 23
SIZES = ((512, 512), (1920, 1080))  # (H, W)


@pytest.fixture(scope="module")
def avatar(dev):
    return SyntheticAvatar(dev)


@pytest.fixture(scope="module")
def motions(avatar, dev, tmp_path_factory):
    out = {}
    for H, W in SIZES:
        root = str(tmp_path_factory.mktemp(f"motion_{H}x{W}"))
        avatar.write_motion(root, FRAME_IDX, H, W)
        out[(H, W)] = MotionTable.from_folder(root, dev)
    return out


def _eq(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES, ids=["512x512", "1920x1080"])
@pytest.mark.parametrize("orbit", [False, True], ids=["animate", "view_rot"])
def test_animator_equals_the_full_chain_eager_and_graphed(avatar, motions, dev, size, orbit):
    from exavatar_release_b200.animation import OrbitCamera
    from exavatar_release_b200.rasterizer import set_fixed_capacity
    motion = motions[size]
    assert motion.frame_idx == list(FRAME_IDX) and motion.image_shape == size
    assert motion.nbytes >= N_FRAMES * size[0] * size[1] * 3
    eager = avatar.animator(motion, orbit=orbit, capacity=CAPACITY, use_graph=False)
    ref_orbit = OrbitCamera(16, N_FRAMES, dev) if orbit else None
    panels = []
    set_fixed_capacity(CAPACITY)
    try:
        for i in range(N_FRAMES):
            a, r = eager.frame(i), avatar.full_chain(motion(i), i, motion.image_shape, ref_orbit)
            if i == 0:
                assert _eq(eager.scale, r["scale"]) and _eq(eager.rgb, r["rgb"])
            for k in ("mean_3d", "render", "mesh_panel", "panel"):
                assert _eq(a[k], r[k]), (i, k)
            panels.append(a["panel"].cpu().numpy())
            assert (panels[-1][:, 2 * size[1]:] < 255).any() and (panels[-1][:, size[1]:2 * size[1]] < 255).any()
    finally:
        set_fixed_capacity(None)
    assert not all(np.array_equal(panels[0], p) for p in panels[1:])
    # the same sequence through frames(): eager, then graphed (first pass captures, second pass only replays)
    for i, (f, p) in enumerate(eager.frames()):
        assert f == FRAME_IDX[i] and np.array_equal(p, panels[i]), i
    graphed = avatar.animator(motion, orbit=orbit, capacity=CAPACITY, use_graph=True)
    first = [(f, p.copy()) for f, p in graphed.frames()]
    assert [f for f, _ in first] == list(FRAME_IDX)
    with no_host_sync():
        second = [(f, p.copy()) for f, p in graphed.frames()]
    for i in range(N_FRAMES):
        assert np.array_equal(first[i][1], panels[i]), i
        assert np.array_equal(second[i][1], panels[i]), i


@pytest.mark.gpu
@pytest.mark.parametrize("in_flight", [1, 2, 3])
def test_ring_buffers_hold_their_own_frame_until_taken(avatar, motions, in_flight):
    motion = motions[SIZES[0]]
    eager = avatar.animator(motion, capacity=CAPACITY, use_graph=False)
    want = [eager.frame(i)["panel"].cpu().numpy() for i in range(N_FRAMES)]
    anim = avatar.animator(motion, capacity=CAPACITY, use_graph=True, in_flight=in_flight)
    for _ in range(2):
        seen = set()
        for i, (f, p) in enumerate(anim.frames()):
            assert f == FRAME_IDX[i]
            assert np.array_equal(p, want[i]), i
            torch.cuda.synchronize()  # the frames queued behind this one have landed in the other buffers
            assert np.array_equal(p, want[i]), i
            p[:4] = 0  # the caller may draw on its buffer (cv2.putText)
            seen.add(p.__array_interface__["data"][0])
        assert len(seen) == min(in_flight, N_FRAMES)


@pytest.mark.gpu
def test_orbit_mode_matches_the_scripts_lines(avatar, motions, dev):
    from exavatar_release_b200.animation import orbit_reference
    motion = motions[SIZES[0]]
    plain = avatar.animator(motion, capacity=CAPACITY, use_graph=False)
    orbit = avatar.animator(motion, orbit=True, capacity=CAPACITY, use_graph=False)
    anchors = {}
    for i in range(N_FRAMES):
        fr = motion(i)
        world = plain.frame(i)["mean_3d"]
        o = orbit.frame(i)
        with torch.no_grad():
            mesh_layer, joints = avatar.rig.body_mesh(avatar.beta, avatar.jo, fr["pose"], fr["expr"], fr["trans"],
                                                      joints=True)
        ref = orbit_reference(fr["cam"], mesh_layer.clone(), joints[0], i, N_FRAMES, anchors, mean_3d=world)
        if i == 0:
            for name, a, b in (("at", orbit.orbit.at, anchors["at_point"]), ("elev", orbit.orbit.elev,
                                                                             anchors["elev"]),
                               ("dist", orbit.orbit.dist, anchors["dist"])):
                d = float((a - b).abs().max()) / (EPS * max(1.0, float(b.abs().max())))
                print(f"anchor {name}: {d:.1f} ulps from the script's lines")
                assert d <= 8, name
        R, t = ref["cam_param_rot"]["R"], ref["cam_param_rot"]["t"]
        assert torch.allclose(o["camera"]["R"], R, atol=2e-6), i
        assert torch.allclose(o["camera"]["t"], t, atol=2e-6 * float(t.norm())), i
        assert torch.allclose(o["mean_3d"], ref["mean_3d"], atol=4e-6), i
        assert torch.allclose(o["mesh"], ref["mesh"], atol=1e-5), i


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
def test_small_capacity_is_reported_with_the_frame(avatar, dev, tmp_path, use_graph):
    from exavatar_release_b200.rasterizer import last_duplicate_count
    H, W = SIZES[0]
    near = 3
    avatar.write_motion(str(tmp_path), FRAME_IDX, H, W, near=near)
    motion = MotionTable.from_folder(str(tmp_path), dev)
    counts = []
    for i in range(N_FRAMES):
        avatar.full_chain(motion(i), i, motion.image_shape)
        counts.append(last_duplicate_count(dev, avatar.rig.P, W, H))
    others = max(c for i, c in enumerate(counts) if i != near)
    print(f"duplicate counts {counts}")
    assert counts[near] > others
    anim = avatar.animator(motion, capacity=others, use_graph=use_graph, in_flight=2)
    got = []
    with pytest.raises(RuntimeError, match=rf"frame {FRAME_IDX[near]} \(position {near}\) needed"):
        for f, _ in anim.frames():
            got.append(f)
    assert got == list(FRAME_IDX[:near])


@pytest.mark.gpu
def test_default_capacity_comes_from_the_first_frame(avatar, motions, dev):
    """Without `capacity`, frame 0 renders with the adaptive policy and the capacity becomes twice its duplicate count
    + 4096; the status blocks are the renders' own, so no other render's state (here: none) is read."""
    from exavatar_release_b200.rasterizer import _compiled_binding, last_duplicate_count
    motion = motions[SIZES[0]]
    H, W = SIZES[0]
    want = [p.copy() for _, p in avatar.animator(motion, capacity=CAPACITY, use_graph=False).frames()]
    for use_graph in (False, True):
        _compiled_binding().clear_recent()
        anim = avatar.animator(motion, use_graph=use_graph)
        assert anim.capacity is None
        got = [(f, p.copy()) for f, p in anim.frames()]
        assert [f for f, _ in got] == list(FRAME_IDX)
        assert all(np.array_equal(p, w) for (_, p), w in zip(got, want)), use_graph
        assert anim.capacity == 2 * last_duplicate_count(dev, avatar.rig.P, W, H) + 4096
