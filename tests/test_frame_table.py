"""`FrameTable` (exavatar_release_b200/frames.py, csrc/frames.cu b2r_frame_unpack): every frame of a split on the
device, the frame of a slot expanded into the DataLoader's collated batch.  CPU: the C ABI's refusals and the builder's checks, which raise before anything is uploaded for the frame they name.  GPU:
the unpack bit-identical to torch's default collate of NeuMan's __getitem__ at 37x53, 512x512 and 1080x1920 through
host and device slots; slots shared with a SmplxParamTable; out-of-range slots inside guarded allocations; one graph
replayed for every slot without a host sync; eval_neuman's ground-truth read; and a training iteration under
IterationGraph with the table read inside the graph, bit-identical to staging the collated inputs."""
import contextlib
import ctypes as C
import multiprocessing
import re

import numpy as np
import pytest
import torch
from torch.utils.data import default_collate

from exavatar_release_b200 import _lib as L
from exavatar_release_b200 import frames as FR
from exavatar_release_b200.frames import FrameTable
from util import no_host_sync
from util import dev  # noqa: F401


# ---------------------------------------------------------------------------------------------------------- CPU tests

def test_abi_refusals_without_touching_cuda():
    lib = L.load()
    fake = 0x1000  # never dereferenced: every call below fails on the host
    launches = lib.b2r_launch_count()
    arrays = ("pixels", "bbox", "R", "t", "focal", "princpt", "frame_idx", "slot_row")
    t = L.B2RFrameTable(n_rows=3, n_slots=5, height=4, width=8, host_slot=0, **{n: fake for n in arrays})
    outs = [fake] * 8
    call = lambda *o: lib.b2r_frame_unpack(C.byref(t), *o, None)  # noqa: E731
    assert lib.b2r_frame_unpack(None, *outs, None) == -1
    for field, bad in [(n, None) for n in arrays] + [("n_rows", 0), ("n_slots", 0), ("height", 0), ("width", -1),
                                                     ("host_slot", -1), ("host_slot", 5)]:
        good = getattr(t, field)
        setattr(t, field, bad)
        assert call(*outs) == -1, field
        setattr(t, field, good)
    for i in range(8):  # every output
        assert call(*outs[:i], None, *outs[i + 1:]) == -1, i
    t.slot = fake  # a device slot: the host slot is not looked at, but sizes and pointers still are
    t.host_slot = 99
    t.height = 0
    assert call(*outs) == -1
    assert lib.b2r_launch_count() == launches


class ListDataset:
    """An ExAvatar-shaped dataset over prepared dicts: frame_idx_list repeats their frames, dataset[i] is a dict."""

    def __init__(self, items, repeat=2):
        self.items = items
        self.frame_idx_list = [d["frame_idx"] for d in items] * repeat

    def __len__(self):
        return len(self.frame_idx_list)

    def __getitem__(self, i):
        return self.items[i % len(self.items)]


def frame_dict(f, H=6, W=10, seed=0):
    g = torch.Generator().manual_seed(seed + f)
    k = torch.randint(0, 256, (3, H, W), generator=g).to(torch.float32)
    return {"img": k / 255., "mask": (torch.rand((1, H, W), generator=g) > 0.5).to(torch.float32),
            "bbox": np.array([1, 2, 3, 4], np.float32),
            "cam_param": {"R": np.eye(3, dtype=np.float32), "t": np.zeros(3, np.float32),
                          "focal": np.full(2, 5, np.float32), "princpt": np.full(2, 3, np.float32)},
            "frame_idx": f}


@pytest.fixture
def uploads(monkeypatch):
    """Stands in for the device upload: records the frames that reached it, then stops the build."""
    seen = []

    def fake(rows, n, device):
        for row in rows:
            seen.append(row["frame_idx"])
        raise _Uploaded

    monkeypatch.setattr(FR, "_upload", fake)
    return seen


class _Uploaded(Exception):
    pass


@pytest.mark.parametrize("workers", [0, 2])
def test_builder_refuses_bad_frames_before_uploading_them(uploads, workers):
    good = [frame_dict(f) for f in (7, 3, 11, 5)]
    ds = ListDataset(good)
    with pytest.raises(_Uploaded):
        FrameTable.from_dataset(ds, "cuda", workers=workers)
    assert uploads == [7, 3, 11, 5]  # each distinct frame once, in first-appearance order
    cases = []
    bad = dict(good[2], img=good[2]["img"].clone())
    bad["img"][1, 2, 3] = 0.5  # between two byte values
    cases.append((bad, "frame 11: `img`"))
    bad = dict(good[2], img=good[2]["img"].clone())
    bad["img"][0, 0, 0] = 256 / 255.  # k / 255 but not a byte
    cases.append((bad, "frame 11: `img`"))
    bad = dict(good[2], mask=good[2]["mask"].clone())
    bad["mask"][0, 1, 1] = 0.5
    cases.append((bad, "frame 11: `mask`"))
    bad = dict(good[2], mask=good[2]["mask"].clone())
    bad["mask"][0, 1, 1] = -0.0  # would unpack as +0
    cases.append((bad, "frame 11: `mask`"))
    cases.append((frame_dict(11, H=7), "frame 11 is 7x10, the first frame 6x10"))
    cases.append((dict(good[2], bbox=good[2]["bbox"].astype(np.float64)), "frame 11: `bbox`"))
    for item, msg in cases:
        uploads.clear()
        with pytest.raises(ValueError, match=re.escape(msg)):
            FrameTable.from_dataset(ListDataset(good[:2] + [item] + good[3:]), "cuda", workers=workers)
        assert uploads == [7, 3], msg
        assert not multiprocessing.active_children()
    uploads.clear()
    bad = dict(good[0], img=good[0]["img"].clone())
    bad["img"][0, 0, 0] = float("nan")
    with pytest.raises(ValueError, match="frame 7"):
        FrameTable.from_dataset(ListDataset([bad] + good[1:]), "cuda", workers=workers)
    assert uploads == []  # the first frame: nothing allocated at all
    assert not multiprocessing.active_children()


def test_builder_refuses_bad_slots_before_reading(uploads):
    ds = ListDataset([frame_dict(f) for f in (7, 3)])
    for slots, msg in (([7, 3, 7], "more than once"), (["3", "7", "3"], "more than once"), ([3, "3"], "more than once"),
                       ([3, 12], "frame 7 of the dataset has no slot"), ([], "empty"), ("73", "list"),
                       (torch.tensor([7, 3]), "list"), ([7, 3.0], "str or an int"), ([7, True], "str or an int"),
                       ([7, None], "str or an int")):
        with pytest.raises(ValueError, match=msg):
            FrameTable.from_dataset(ds, "cuda", slots=slots, workers=0)
    assert uploads == []
    with pytest.raises(RuntimeError, match="CUDA"):
        FrameTable.from_dataset(ds, "cpu", workers=0)
    with pytest.raises(ValueError, match="workers"):
        FrameTable.from_dataset(ds, "cuda", workers=-1)
    ds.frame_idx_list = [7, 3.0]
    with pytest.raises(ValueError, match="not an int"):
        FrameTable.from_dataset(ds, "cuda", workers=0)
    ds.frame_idx_list = []
    with pytest.raises(ValueError, match="no frames"):
        FrameTable.from_dataset(ds, "cuda", workers=0)
    assert uploads == []


def test_image_quotient_is_ieee_division():
    """The unpack's fl(k / 255) is both NeuMan's training read and eval_neuman's float64 read rounded to fp32; the
    reciprocal product is not."""
    k = np.arange(256)
    q = k.astype(np.float32) / np.float32(255)
    assert np.array_equal((k / 255.).astype(np.float32).view(np.int32), q.view(np.int32))
    assert torch.equal((torch.arange(256, dtype=torch.float32) / 255.).view(torch.int32), torch.from_numpy(q.view(np.int32)))
    assert (k.astype(np.float32) * np.float32(1 / 255) != q).sum() == 126


# ---------------------------------------------------------------------------------------------------------- GPU tests

def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def assert_batch(got, want, what):
    """Same keys, shapes, dtypes and bits (want on the host)."""
    assert set(got) == set(want), what
    for k in want:
        if isinstance(want[k], dict):
            assert_batch(got[k], want[k], f"{what} {k}")
            continue
        g, w = got[k], want[k]
        assert g.is_cuda and g.shape == w.shape and g.dtype == w.dtype, (what, k, g.shape, w.shape, g.dtype, w.dtype)
        assert torch.equal(bits(g).cpu(), bits(w)), (what, k)


def collated(ds, i):
    return default_collate([ds[i]])


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(37, 53), (512, 512), (1080, 1920)])
def test_unpack_matches_collated_dataset(H, W, dev, tmp_path):
    from bench_frame_table import NeumanFrames
    ds = NeumanFrames(str(tmp_path), [4, 17, 9], H, W, repeat=3, seed=H)
    table = FrameTable.from_dataset(ds, dev, workers=2)
    assert not multiprocessing.active_children()
    assert table.n_rows == table.n_slots == 3 and (table.height, table.width) == (H, W)
    assert table.pixels.shape == (3, H, W, 4) and table.nbytes >= 3 * H * W * 4
    slot_t = torch.zeros(1, dtype=torch.int32, device=dev)
    positions = range(len(ds)) if H * W < 10_000 else range(3)
    for i in positions:
        want = collated(ds, i)
        slot = table.slot_of(ds.frame_idx_list[i])
        assert slot == [4, 17, 9].index(ds.frame_idx_list[i])
        assert_batch(table(slot), want, f"{H}x{W} position {i} host slot")
        slot_t.fill_(slot)
        assert_batch(table(slot_t), want, f"{H}x{W} position {i} device slot")


@pytest.mark.gpu
def test_slots_of_a_param_table(dev, tmp_path):
    from bench_frame_table import NeumanFrames
    from exavatar_release_b200 import SmplxParamTable
    keys = ["100", "4", "3", "17", "200"]  # SMPLXParamDict holds frames outside the split
    F = len(keys)
    pt = SmplxParamTable(torch.zeros((F, 55, 6), device=dev), torch.zeros((F, 10), device=dev),
                         torch.zeros((F, 3), device=dev), frames=keys)
    ds = NeumanFrames(str(tmp_path), [17, 4], 21, 16, repeat=2)
    table = FrameTable.from_dataset(ds, dev, slots=pt.frames, workers=0)
    assert table.frames == keys and table.n_slots == F and table.n_rows == 2
    assert table.slot_row.cpu().tolist() == [-1, 1, -1, 0, -1]
    slot_t = torch.zeros(1, dtype=torch.int32, device=dev)
    for f in (17, 4):
        s = pt.slot_of(f)
        assert table.slot_of(f) == s
        assert_batch(table(s), collated(ds, ds.frame_idx_list.index(f)), f"frame {f}")
        slot_t.fill_(s)
        assert_batch(table(slot_t), collated(ds, ds.frame_idx_list.index(f)), f"frame {f} device")
    for s in (0, 2, 4):  # slots without a frame of the split
        slot_t.fill_(s)
        out = table(slot_t)
        for x in (out["img"], out["mask"], out["bbox"], *out["cam_param"].values()):
            assert torch.isnan(x).all(), s
        assert out["frame_idx"].item() == -1
        with pytest.raises(IndexError, match="no frame"):
            table(s)
    with pytest.raises(IndexError):
        table(F)
    with pytest.raises(ValueError, match="int32"):
        table(torch.zeros(1, dtype=torch.int64, device=dev))
    with pytest.raises(KeyError):
        table.slot_of(5)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(37, 53), (64, 96)])
def test_out_of_range_slots_inside_guarded_allocations(H, W, dev, tmp_path):
    from bench_frame_table import NeumanFrames
    from test_poisoned_buffers import NAN_WORD, GuardedAllocations, check_memory, poisoned
    ds = NeumanFrames(str(tmp_path), [2, 5, 8], H, W)
    table = FrameTable.from_dataset(ds, dev, workers=0)
    slot_t = torch.zeros(1, dtype=torch.int32, device=dev)
    before = [x.clone() for x in (table.pixels, table.bbox, table.R, table.t, table.frame_idx, table.slot_row)]
    for s in range(3):  # a valid slot writes every element of its poisoned / guarded outputs
        slot_t.fill_(s)
        plain = check_memory(lambda: table(slot_t))
        assert_batch(table(s), collated(ds, s), f"slot {s}")
        assert not any(torch.isnan(v).any() for k, v in plain.items() if v.is_floating_point()), s
    for bad in (-1, 3, 2 ** 31 - 1):
        slot_t.fill_(bad)
        for fill in (NAN_WORD, 0):
            with GuardedAllocations(fill) as g:
                out = table(slot_t)
            torch.cuda.synchronize()
            assert g.blocks and not g.damaged(), (bad, hex(fill), g.damaged())
            for x in (out["img"], out["mask"], out["bbox"], *out["cam_param"].values()):
                assert torch.isnan(x).all(), (bad, fill)
            assert out["frame_idx"].item() == -1
        with poisoned():
            out = table(slot_t)
        assert torch.isnan(out["img"]).all() and out["frame_idx"].item() == -1
    for x, b in zip((table.pixels, table.bbox, table.R, table.t, table.frame_idx, table.slot_row), before):
        assert torch.equal(x, b)  # the table is read only


@pytest.mark.gpu
def test_one_graph_replayed_for_every_slot(dev, tmp_path):
    from bench_frame_table import NeumanFrames
    ds = NeumanFrames(str(tmp_path), [1, 6, 3, 9], 48, 64, repeat=2)
    table = FrameTable.from_dataset(ds, dev, workers=2)
    slot_t = torch.zeros(1, dtype=torch.int32, device=dev)
    table(slot_t)  # loads the module outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = table(slot_t)
    lib = L.load()
    for rep in range(2):
        for s in (3, 0, 2, 1, 9, -1):
            n0 = lib.b2r_launch_count()
            with no_host_sync():
                slot_t.fill_(s)
                g.replay()
            assert lib.b2r_launch_count() == n0
            if 0 <= s < 4:
                assert_batch(out, collated(ds, s), f"replay {rep} slot {s}")
            else:
                assert torch.isnan(out["img"]).all() and out["frame_idx"].item() == -1


@pytest.mark.gpu
def test_unpacked_image_is_evals_ground_truth(dev, tmp_path):
    """eval_neuman reads the ground truth as FloatTensor(cv2.imread(p)[:,:,::-1] / 255.): float64, then fp32."""
    import cv2
    from bench_frame_table import NeumanFrames
    ds = NeumanFrames(str(tmp_path), [0, 1], 37, 53)
    table = FrameTable.from_dataset(ds, dev, workers=0)
    for f in (0, 1):
        gt = torch.FloatTensor(cv2.imread(ds.img_paths[f])[:, :, ::-1] / 255.).permute(2, 0, 1)[None]
        assert torch.equal(bits(table(table.slot_of(f))["img"]).cpu(), bits(gt))
        assert table(f)["img"].shape == gt.shape


def reduced_chain(scene, sp, data, bg, warm):
    """A renderer-free iteration that reads the frame's image, mask, box and camera: the loss terms."""
    from exavatar_release_b200.losses import l1_ssim
    cam = data["cam_param"]
    img = scene["img"] * bg.view(1, 3, 1, 1) + 0.01 * sp["trans"].sum()
    if warm:
        img = torch.clamp(img, max=0.9)
    l1, ss = l1_ssim(img, data["img"], data["bbox"], mask=data["mask"])
    uv = (scene["pts"] @ cam["R"][0].t() + cam["t"][0])[:, :2] * cam["focal"] + cam["princpt"]
    return {"l1": 0.8 * l1, "ssim": 0.2 * (1 - ss), "pose": (sp["full_pose"] ** 2).mean(),
            "uv": 1e-6 * (uv ** 2).mean()}


@pytest.mark.gpu
def test_iteration_graph_with_the_table_matches_staged_inputs(dev, tmp_path):
    from bench_frame_table import NeumanFrames
    from exavatar_release_b200 import Adam, IterationGraph, SmplxParamTable
    H, W = 40, 56
    frame_ids = [0, 1, 2, 3, 4]
    F = len(frame_ids)
    ds = NeumanFrames(str(tmp_path), frame_ids, H, W, repeat=3, seed=4)
    seq = np.random.default_rng(3).permutation(len(ds))[:14].tolist()
    warm = [i < 6 for i in range(len(seq))]  # the key changes at iteration 6

    def model():
        g = torch.Generator(device=dev).manual_seed(11)
        scene = {"img": torch.rand((1, 3, H, W), generator=g, device=dev).requires_grad_(),
                 "pts": torch.randn((257, 3), generator=g, device=dev).requires_grad_()}
        pt = SmplxParamTable(0.1 * torch.randn((F, 55, 6), generator=g, device=dev),
                             0.1 * torch.randn((F, 10), generator=g, device=dev),
                             0.1 * torch.randn((F, 3), generator=g, device=dev), frames=[str(f) for f in frame_ids])
        for p in pt.parameters():
            p.requires_grad_()
        groups = [{"params": [scene["img"]], "name": "img_scene", "lr": 1e-2},
                  {"params": [scene["pts"]], "name": "pts_scene", "lr": 1e-3},
                  {"params": pt.parameters(), "name": "smplx", "lr": 1e-3, "frame_rows": True}]
        return scene, pt, Adam(groups, lr=0.0, eps=1e-15)

    scene_a, pt_a, opt_a = model()
    scene_b, pt_b, opt_b = model()
    table = FrameTable.from_dataset(ds, dev, slots=pt_b.frames, workers=2)
    cur = {"warm": True}

    def step_a(inputs, slot):  # the DataLoader route: the collated batch staged into static buffers
        data = {"img": inputs["img"], "mask": inputs["mask"], "bbox": inputs["bbox"],
                "cam_param": {k: inputs[k] for k in ("R", "t", "focal", "princpt")}}
        losses = reduced_chain(scene_a, pt_a(slot), data, inputs["bg"], cur["warm"])
        sum(losses.values()).backward()
        return losses

    def step_b(inputs, slot):  # the table read inside the graph
        losses = reduced_chain(scene_b, pt_b(slot), table(slot), inputs["bg"], cur["warm"])
        sum(losses.values()).backward()
        return losses

    def staged(batch, bg):
        d = {k: batch[k] for k in ("img", "mask", "bbox")}
        d.update(batch["cam_param"], bg=bg)
        return d

    bgs = torch.rand((len(seq), 3), generator=torch.Generator().manual_seed(5))
    it_a = IterationGraph(step_a, opt_a, staged(collated(ds, 0), bgs[0]))
    it_b = IterationGraph(step_b, opt_b, {"bg": bgs[0]})
    lib = L.load()
    for itr, pos in enumerate(seq):
        batch = collated(ds, pos)
        slot = pt_a.slot_of(int(batch["frame_idx"][0]))
        cur["warm"] = warm[itr]
        la = it_a.run(staged(batch, bgs[itr]), slot, key=warm[itr])
        replay = warm[itr] in it_b._graphs
        n0 = lib.b2r_launch_count()
        with no_host_sync() if replay else contextlib.nullcontext():
            lb = it_b.run({"bg": bgs[itr]}, table.slot_of(ds.frame_idx_list[pos]), key=warm[itr])
        if replay:
            assert lib.b2r_launch_count() == n0
        assert la.keys() == lb.keys()
        for k in la:
            assert torch.equal(bits(la[k]), bits(lb[k])), (itr, k)
        for ga, gb in zip(opt_a.param_groups, opt_b.param_groups):
            for pa, pb in zip(ga["params"], gb["params"]):
                assert torch.equal(bits(pa), bits(pb)), (itr, ga["name"])
                for m in ("step", "exp_avg", "exp_avg_sq"):
                    assert torch.equal(bits(opt_a.state[pa][m]), bits(opt_b.state[pb][m])), (itr, ga["name"], m)
    assert set(it_b._graphs) == {True, False}
