"""SegmentationTable (exavatar_release_b200/frames.py, csrc/frames.cu b2r_segmentation_unpack) and AvatarTester
(exavatar_release_b200/tester.py): ExAvatar's test.py + eval_neuman.py pass on the device.  CPU: the host half reads
cv2's BGR bytes in row order and refuses bad files before any upload, the C ABI's refusals, the struct's layout, and
the tester's refusals.  GPU, with the C4 human and scene over 6 frames: the mask unpack against eval's expression bit
for bit, the tester against `SyntheticAvatar.test_chain` + NeumanScores bit for bit (eager and graphed, with and
without masks, unscored and without bytes), the end-to-end eval loop over written PNGs, the ring, the overflow
report, and in-place reads with `invalidate()`."""
import ctypes as C
import os
from types import SimpleNamespace

import cv2
import numpy as np
import pytest
import torch

from util import ROOT  # noqa: F401  (path setup)
from util import header_structs, no_host_sync
from util import dev  # noqa: F401
from c4_frame import SyntheticAvatar, write_segmentation
from exavatar_release_b200 import _lib as L
from exavatar_release_b200 import frames as FR
from exavatar_release_b200.compose import PNG_ORDER
from exavatar_release_b200.frames import SegmentationTable, read_segmentations
from exavatar_release_b200.metrics import MIN_SIZE
from exavatar_release_b200.tester import AvatarTester


# ---------------------------------------------------------------------------------------------------------- CPU tests

def _stand_in_frames(frame_idx, H, W):
    """What from_folder reads of a FrameTable: its rows' frame indices and its image size."""
    return SimpleNamespace(frame_idx=torch.tensor(frame_idx), height=H, width=W)


def test_host_half_reads_cv2_bgr_bytes_in_row_order(tmp_path):
    root = str(tmp_path)
    ids = [250, 3, 1000]
    want = {f: write_segmentation(root, f, 9, 13, seed=f) for f in ids}
    assert all((want[f][..., 0] != want[f][..., 1]).any() for f in ids)  # the channels differ
    got = read_segmentations(root, ids, (9, 13))
    for f, img in zip(ids, got):
        assert img.dtype == np.uint8 and img.shape == (9, 13, 3)
        assert np.array_equal(img, cv2.imread(os.path.join(root, "segmentations", "%05d.png" % f)))
        assert np.array_equal(img, want[f])


@pytest.mark.parametrize("case", ["missing", "unreadable", "size"])
def test_host_half_refusals_before_upload(tmp_path, monkeypatch, case):
    root = str(tmp_path)
    ids = [4, 17, 9]
    for f in ids:
        write_segmentation(root, f, 9, 13, seed=f)
    path = os.path.join(root, "segmentations", "%05d.png" % 17)
    if case == "missing":
        os.remove(path)
        msg = "frame 17: missing or unreadable"
    elif case == "unreadable":
        with open(path, "wb") as f:
            f.write(b"not a png")
        msg = "frame 17: missing or unreadable"
    else:
        write_segmentation(root, 17, 9, 12, seed=0)
        msg = "frame 17: .* is 9x12, the frames 9x13"
    monkeypatch.setattr(FR, "_upload_segmentations", lambda *a: pytest.fail("uploaded"))
    with pytest.raises(ValueError, match=msg):
        SegmentationTable.from_folder(root, _stand_in_frames(ids, 9, 13), "cuda")


def test_table_refuses_a_cpu_device(tmp_path):
    write_segmentation(str(tmp_path), 4, 9, 13, seed=0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        SegmentationTable.from_folder(str(tmp_path), _stand_in_frames([4], 9, 13), "cpu")


def test_struct_layout_and_abi_refusals_without_touching_cuda():
    lib = L.load()
    assert L.B2RSegmentation.ID == 34 and lib.b2r_sizeof(34) == C.sizeof(L.B2RSegmentation) == 24 + 3 * 8
    assert [f for f, _ in L.B2RSegmentation._fields_] == header_structs()["B2RSegmentation"]
    fake = 0x1000  # never dereferenced: every call below fails on the host
    launches = lib.b2r_launch_count()
    s = L.B2RSegmentation(n_rows=3, n_slots=5, height=4, width=8, host_slot=0, pixels=fake, slot_row=fake)
    assert lib.b2r_segmentation_unpack(None, fake, None) == -1
    assert lib.b2r_segmentation_unpack(C.byref(s), None, None) == -1
    for field, bad in (("pixels", None), ("slot_row", None), ("n_rows", 0), ("n_slots", 0), ("height", 0),
                       ("width", -1), ("host_slot", -1), ("host_slot", 5)):
        good = getattr(s, field)
        setattr(s, field, bad)
        assert lib.b2r_segmentation_unpack(C.byref(s), fake, None) == -1, field
        setattr(s, field, good)
    s.slot = fake  # a device slot: the host slot is not looked at, but sizes and pointers still are
    s.host_slot = 99
    s.height = 0
    assert lib.b2r_segmentation_unpack(C.byref(s), fake, None) == -1
    assert lib.b2r_launch_count() == launches


def _tester_args(H=64, W=48, slots=("1", "2"), param_slots=("1", "2"), shape=None, **kw):
    frames = SimpleNamespace(frames=list(slots), height=H, width=W)
    params = SimpleNamespace(frames=list(param_slots))
    renderer = SimpleNamespace(img_shape=shape or (H, W), use_graph=False)
    nets = dict(triplane=None, triplane_face=None, geo_net=None, geo_offset_net=None, rgb_net=None,
                rgb_offset_net=None, shape_param=None, joint_offset=None, skinning_weight=None, self_map=None,
                scene={}, active_sh_degree=None, face_uvmap=None, face_vertex_idx=None)
    nets.update(kw)
    return (frames, params, None, None, None, None, None, renderer), nets


@pytest.mark.parametrize("case", ["slots", "order", "shape", "graph_renderer", "min_size", "in_flight_0",
                                  "in_flight_bool", "in_flight_float", "masks_without_scorer", "other_masks",
                                  "scene_keys"])
def test_tester_refusals(case):
    msg = {"slots": "slots", "order": "slots", "shape": "renders", "graph_renderer": "use_graph=False",
           "min_size": f"at least {MIN_SIZE}x{MIN_SIZE}", "in_flight_0": "in_flight", "in_flight_bool": "in_flight",
           "in_flight_float": "in_flight", "masks_without_scorer": "need a `scorer`",
           "other_masks": "this frame table", "scene_keys": "lacks"}[case]
    if case == "slots":
        args, kw = _tester_args(param_slots=("1", "3"))
    elif case == "order":
        args, kw = _tester_args(param_slots=("2", "1"))
    elif case == "shape":
        args, kw = _tester_args(shape=(48, 64))
    elif case == "graph_renderer":
        args, kw = _tester_args()
        args[7].use_graph = True
    elif case == "min_size":
        args, kw = _tester_args(H=30, W=48, scorer=object())
    elif case.startswith("in_flight"):
        args, kw = _tester_args(in_flight={"in_flight_0": 0, "in_flight_bool": True, "in_flight_float": 2.0}[case])
    elif case == "masks_without_scorer":
        args, kw = _tester_args(masks=SimpleNamespace(frames=None))
    elif case == "other_masks":
        args, kw = _tester_args(scorer=object(), masks=SimpleNamespace(frames=SimpleNamespace()))
    else:
        args, kw = _tester_args(scene={"mean": None})
    with pytest.raises(ValueError, match=msg):
        AvatarTester(*args, **kw)


def test_png_order_is_test_pys_ten_writes():
    assert PNG_ORDER == ("scene_img", "human_img", "scene_human_img", "human_img_refined", "scene_human_img_refined",
                         "human_face_img", "human_face_img_refined", "scene_human_img_composed",
                         "scene_human_img_refined_composed", "gt")


# ---------------------------------------------------------------------------------------------------------------------
# On the H100: the synthetic C4 avatar (P = 167 618) and a 130 000-Gaussian scene

N_FRAMES = 6
FRAME_IDX = (12, 3, 250, 41, 1000, 7)  # test_split.txt order; the SMPL-X table holds them reversed plus one more
CAPACITY = 1 << 23
H0, W0 = 512, 512


@pytest.fixture(scope="module")
def avatar(dev):
    return SyntheticAvatar(dev)


@pytest.fixture(scope="module")
def split(avatar, tmp_path_factory):
    root = str(tmp_path_factory.mktemp("split"))
    return root, avatar.test_setup(root, FRAME_IDX, H0, W0, CAPACITY)


@pytest.fixture(scope="module")
def scorer(dev):
    from test_neuman_reference import alex_weights
    from exavatar_release_b200 import NeumanScores
    return NeumanScores(*alex_weights(), dev)


def _bits(t):
    return t.contiguous().view(torch.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(37, 53), (512, 512), (1080, 1920)], ids=["37x53", "512x512", "1080x1920"])
def test_mask_unpack_is_evals_mask(avatar, dev, tmp_path, size):
    from c4_frame import TestSplit
    from exavatar_release_b200 import FrameTable
    H, W = size
    ids = [5, 90, 31]
    imgs = [np.zeros((H, W, 3), np.uint8)] * 3
    cam = {"R": np.eye(3, dtype=np.float32), "t": np.zeros(3, np.float32), "focal": np.ones(2, np.float32),
           "princpt": np.ones(2, np.float32)}
    segs = [write_segmentation(str(tmp_path), f, H, W, seed=f) for f in ids]
    frames = FrameTable.from_dataset(TestSplit(ids, imgs, [cam] * 3), dev, slots=["0", "31", "5", "90"], workers=0)
    masks = SegmentationTable.from_folder(str(tmp_path), frames, dev)
    assert masks.nbytes == 3 * H * W * 4
    slot_t = torch.zeros(1, dtype=torch.int32, device=dev)
    for f, seg in zip(ids, segs):
        want = torch.FloatTensor(1 - cv2.imread(os.path.join(str(tmp_path), "segmentations", "%05d.png" % f)) / 255.)
        want = want.permute(2, 0, 1)[None]
        assert not torch.equal(want[:, 0], want[:, 2])  # B and R planes differ: a reversed order would fail
        slot = frames.slot_of(f)
        slot_t.fill_(slot)
        for got in (masks(slot), masks(slot_t)):
            assert got.shape == (1, 3, H, W) and got.dtype == torch.float32
            assert torch.equal(_bits(got.cpu()), _bits(want)), f
    for bad in (0, -1, 4, 1 << 30):  # a slot without a frame, and slots outside [0, 4)
        slot_t.fill_(bad)
        assert torch.isnan(masks(slot_t)).all(), bad
    with pytest.raises(IndexError, match="no frame"):
        masks(0)
    with pytest.raises(IndexError, match="outside"):
        masks(4)


def _reference(avatar, s, scorer, masks, png=True):
    """test_chain + NeumanScores of every frame in row order: [(png host bytes or None, scores or None)]."""
    out = []
    for r in range(N_FRAMES):
        slot = s.frames.slot_of(FRAME_IDX[r])
        res = avatar.test_chain(s, slot, png=png)
        sc = None
        if scorer is not None:
            mask = s.masks(slot) if masks else None
            sc = scorer(res["scene_human_img_refined_composed"], res["gt"], mask)[0].cpu()
        out.append((res["png"][:, 0].cpu().numpy() if png else None, sc))
    return out


def _check(got, want, what):
    assert [f for f, _, _ in got] == list(FRAME_IDX), what
    for r, ((_, p, sc), (wp, wsc)) in enumerate(zip(got, want)):
        if wp is None:
            assert p is None, (what, r)
        else:
            assert np.array_equal(p, wp), (what, r)
        if wsc is None:
            assert sc is None, (what, r)
        else:
            assert torch.equal(_bits(torch.from_numpy(sc)), _bits(wsc)), (what, r, sc, wsc)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["masks", "include_bkg", "custom"])
def test_tester_equals_test_chain_eager_and_graphed(avatar, split, scorer, mode):
    """Every frame's ten byte arrays and three scores equal test_chain + NeumanScores bit for bit, eagerly and
    graphed; the second graphed pass only replays and makes no host sync.  'custom' is scorer=None with png=False."""
    _, s = split
    use_scorer = scorer if mode != "custom" else None
    masks = s.masks if mode == "masks" else None
    png = mode != "custom"
    want = _reference(avatar, s, use_scorer, masks is not None, png)
    if png:
        assert not all(np.array_equal(want[0][0], w[0]) for w in want[1:])
        assert (want[0][0][1] < 255).any()  # the human is in view
    for use_graph in (False, True):
        t = avatar.tester(s, scorer=use_scorer, masks=masks, png=png, use_graph=use_graph)
        got = [(f, None if p is None else p.copy(), None if sc is None else sc.copy()) for f, p, sc in t.frames()]
        _check(got, want, ("first pass", use_graph))
        if use_graph:
            with no_host_sync():
                got = [(f, None if p is None else p.copy(), None if sc is None else sc.copy())
                       for f, p, sc in t.frames()]
            _check(got, want, ("replays", use_graph))
        if use_scorer is not None:
            table = t.scores().cpu()
            assert torch.equal(_bits(table), _bits(torch.stack([w[1] for w in want])))


@pytest.mark.gpu
def test_end_to_end_against_evals_loop(avatar, split, scorer, tmp_path):
    """The ring's bytes written with cv2.imwrite and scored as eval_neuman's loop reads them (the output PNG, the gt
    from the table's bytes, the mask from the segmentation PNG) equal the tester's scores; summary() is the fp64
    in-order mean rounded once, and within 2 ulp of eval's fp32 mean."""
    root, s = split
    t = avatar.tester(s, scorer=scorer, masks=s.masks)
    out = str(tmp_path)
    got = []
    for f, png, sc in t.frames():
        for k, name in enumerate(PNG_ORDER):
            assert cv2.imwrite(os.path.join(out, f"{f}_{name}.png"), png[k])
        got.append(sc.copy())
    results = []
    dev = scorer.device
    for r, f in enumerate(FRAME_IDX):
        o = cv2.imread(os.path.join(out, f"{f}_scene_human_img_refined_composed.png"))[:, :, ::-1] / 255.
        o = torch.FloatTensor(o.copy()).permute(2, 0, 1)[None].to(dev)
        gt = cv2.imread(os.path.join(out, f"{f}_gt.png"))[:, :, ::-1] / 255.
        gt = torch.FloatTensor(gt.copy()).permute(2, 0, 1)[None].to(dev)
        assert torch.equal(gt, s.frames(s.frames.slot_of(f))["img"])  # the table's bytes are eval's ground truth
        mask = 1 - cv2.imread(os.path.join(root, "segmentations", "%05d.png" % f)) / 255.
        mask = torch.FloatTensor(mask).permute(2, 0, 1)[None].to(dev)
        sc = scorer(o, gt, mask)[0].cpu()
        assert torch.equal(_bits(sc), _bits(torch.from_numpy(got[r]))), (f, sc, got[r])
        results.append(sc)
    summary = t.summary().cpu()
    v = torch.stack(results).double()
    acc = v[0].clone()
    for r in range(1, N_FRAMES):
        acc += v[r]
    assert torch.equal(_bits(summary), _bits((acc / N_FRAMES).float()))
    evals = torch.stack([torch.FloatTensor([float(x[k]) for x in results]).mean() for k in range(3)])
    ulp = (summary - evals).abs() / torch.tensor([np.spacing(np.float32(abs(float(x)))) for x in evals])
    print(f"summary {summary.tolist()} vs eval's fp32 mean {evals.tolist()}: {ulp.tolist()} ulp")
    assert bool((ulp <= 2).all())


@pytest.mark.gpu
@pytest.mark.parametrize("in_flight", [1, 2, 3])
def test_ring_buffers_hold_their_own_frame_until_taken(avatar, split, scorer, in_flight):
    _, s = split
    want = _reference(avatar, s, scorer, True)
    t = avatar.tester(s, scorer=scorer, masks=s.masks, in_flight=in_flight)
    for _ in range(2):
        seen = set()
        for r, (f, p, sc) in enumerate(t.frames()):
            assert f == FRAME_IDX[r]
            torch.cuda.synchronize()  # the frames queued behind this one have landed in the other buffers
            assert np.array_equal(p, want[r][0]) and torch.equal(torch.from_numpy(sc), want[r][1]), r
            p[:, :4] = 0  # the caller may use its buffer
            seen.add(p.__array_interface__["data"][0])
        assert len(seen) == min(in_flight, N_FRAMES)


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
def test_small_capacity_is_reported_with_the_frame(avatar, split, dev, use_graph):
    """A renderer whose pass-A lists hold the entries of the frames before position `near` but not those of frame
    `near` raises at that frame, after handing back the frames before it."""
    from exavatar_release_b200 import TrainingFrameRenderer
    _, s = split
    dups = []
    for r in range(N_FRAMES):
        avatar.test_chain(s, s.frames.slot_of(FRAME_IDX[r]), png=False)
        dups.append(L.read_status(s.renderer.plan.passes["A"].ctx_buf)["num_dups"])
    # the first position past the captured one whose frame needs more entries than every frame before it
    near = next(r for r in range(2, N_FRAMES) if dups[r] > max(dups[:r]))
    cap = max(dups[:near])
    print(f"pass A duplicates {dups}; capacity {cap}, first overflow at position {near}")
    small = TrainingFrameRenderer(s.scene["mean"].shape[0], avatar.rig.P, (H0, W0), dev, {"A": cap, "B": CAPACITY})
    t = avatar.tester(s._replace(renderer=small), png=False, use_graph=use_graph)
    got = []
    with pytest.raises(RuntimeError, match=rf"frame {FRAME_IDX[near]} \(position {near}\) needed \d+ render list "
                                           rf"entries in pass A, the capacity is {cap}"):
        for f, _, _ in t.frames():
            got.append(f)
    assert got == list(FRAME_IDX[:near])


@pytest.mark.gpu
def test_replays_read_parameters_in_place_and_invalidate_recaptures(avatar, split, scorer, dev):
    """After in-place updates of a triplane, a stack weight and a scene parameter, a replay equals a fresh tester's
    eager pass; after a scene tensor is replaced, invalidate() recaptures and matches again."""
    _, s = split
    scene = dict(s.scene)
    s = s._replace(scene=scene)
    t = avatar.tester(s, scorer=scorer, masks=s.masks)
    list(t.frames())  # eager position 0, capture at position 1
    saved = (avatar.tp.clone(), next(avatar.nets["rgb"][0].parameters()).detach().clone(), scene["feature_dc"].clone())
    try:
        with torch.no_grad():
            avatar.tp.mul_(1.1)
            next(avatar.nets["rgb"][0].parameters()).add_(0.01)
            scene["feature_dc"].add_(0.2)
        fresh = [(f, p.copy(), sc.copy()) for f, p, sc in
                 avatar.tester(s, scorer=scorer, masks=s.masks, use_graph=False).frames()]
        with no_host_sync():
            got = [(f, p.copy(), sc.copy()) for f, p, sc in t.frames()]
        _check(got, [(p, torch.from_numpy(sc)) for _, p, sc in fresh], "in place")
        scene["opacity_logit"] = scene["opacity_logit"] - 1.0  # a new tensor: the graph still reads the old one
        fresh = [(f, p.copy(), sc.copy()) for f, p, sc in
                 avatar.tester(s, scorer=scorer, masks=s.masks, use_graph=False).frames()]
        stale = [(f, p.copy(), sc.copy()) for f, p, sc in t.frames()]
        assert not all(np.array_equal(a[1], b[1]) for a, b in zip(stale[1:], fresh[1:]))
        t.invalidate()
        got = [(f, p.copy(), sc.copy()) for f, p, sc in t.frames()]
        _check(got, [(p, torch.from_numpy(sc)) for _, p, sc in fresh], "recaptured")
    finally:
        with torch.no_grad():
            avatar.tp.copy_(saved[0])
            next(avatar.nets["rgb"][0].parameters()).copy_(saved[1])
            s.scene["feature_dc"].copy_(saved[2])

