"""FrameTable: the frame's image, mask, box and camera read on the device, against ExAvatar's DataLoader route.

  unpack   b2r_frame_unpack alone at 512 x 512 and 1080 x 1920, eager and replayed in a CUDA graph of 20 unpacks:
           microseconds per unpack, the bytes it moves (4 read and 16 written per pixel, plus the row's box and camera) and that rate
           against the H100 SXM data sheet's 3.35 TB/s.
  e2e      the C4 training iteration of tools/bench_iteration_graph.py's Chain under IterationGraph, F = 100 frames,
           at 512 x 512 and 1080 x 1920, in two arms alternated window by window:
             loader  ExAvatar's route: the frames are PNGs written with cv2 into a temporary directory,
                     `NeumanFrames` restates NeuMan's __getitem__, and DataLoader(batch_size=1, num_workers=8,
                     pin_memory=True) feeds IterationGraph.run's staged inputs;
             table   FrameTable.from_dataset over the same dataset, read inside the graph; only the background is
                     staged.
           Both arms visit the same slot sequence (a fixed index sampler) and stage the same backgrounds.  The
           inputs their first iteration reads (image, box, camera) must be bit-identical, or the script exits; the
           record says whether the first iteration's loss terms, eager from the same seeded state in two Chain
           instances, are too, and by how much each term that is not differs.  Later iterations differ in the last
           bits through the renderer's float-atomic backward composite, in either arm.
Reported: iterations/s (median, min, max over the windows), host ms per iteration (the time until the Python call
returns: the loader's next batch plus IterationGraph.run), the table's build time and bytes, the card and the host's
CPU count.  Temporary files are removed and every DataLoader worker is joined before the script exits.

`NeumanFrames` is also the dataset of tests/test_frame_table.py.
"""
import os
import sys
import tempfile
import time

import cv2
import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset, default_collate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from benchkit import HBM_BYTES_PER_S, alternate, arg_parser, card, cuda_device, emit, graph_replay, stats  # noqa: E402
from exavatar_release_b200 import FrameTable, IterationGraph  # noqa: E402
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402


def get_bbox(joint_img, joint_valid, extend_ratio=1.2):
    """ExAvatar's get_bbox (common/utils/preprocessing.py): the valid keypoints' box, widened by extend_ratio, as
    float32 [xmin, ymin, width, height]."""
    x_img, y_img = joint_img[:, 0][joint_valid == 1], joint_img[:, 1][joint_valid == 1]
    xmin, ymin, xmax, ymax = min(x_img), min(y_img), max(x_img), max(y_img)
    x_center, width = (xmin + xmax) / 2., xmax - xmin
    xmin, xmax = x_center - 0.5 * width * extend_ratio, x_center + 0.5 * width * extend_ratio
    y_center, height = (ymin + ymax) / 2., ymax - ymin
    ymin, ymax = y_center - 0.5 * height * extend_ratio, y_center + 0.5 * height * extend_ratio
    return np.array([xmin, ymin, xmax - xmin, ymax - ymin]).astype(np.float32)


class NeumanFrames(Dataset):
    """A NeuMan-layout subject in `root`: images/<f>.png and masks/<f>.png written with cv2, whole-body keypoints and
    one camera per frame; `frame_idx_list` is the frames repeated `repeat` times.  `__getitem__` restates NeuMan's
    (avatar/data/NeuMan/NeuMan.py:130-147) with torchvision's ToTensor of a float32 array written out."""

    def __init__(self, root, frame_ids, H, W, repeat=1, seed=0):
        rng = np.random.default_rng(seed)
        os.makedirs(os.path.join(root, "images"), exist_ok=True)
        os.makedirs(os.path.join(root, "masks"), exist_ok=True)
        cam = look_at_cam_param(-6.0, (H, W))
        self.img_paths, self.mask_paths, self.kpts, self.cam_params = {}, {}, {}, {}
        yy, xx = np.mgrid[0:H, 0:W]
        for i, f in enumerate(frame_ids):
            base = (xx * 3 + yy * 5 + 40 * i)[..., None] + np.array([0, 85, 170])
            img = ((base + rng.integers(0, 24, (H, W, 3))) % 256).astype(np.uint8)  # BGR, as cv2 writes it
            mask = np.zeros((H, W), np.uint8)
            mask[H // 4:3 * H // 4, W // 3:2 * W // 3] = 255
            mask[rng.random((H, W)) < 0.05] = rng.choice([0, 100, 128, 200], 1)[0]  # edges of a real matte
            self.img_paths[f] = os.path.join(root, "images", f"{f}.png")
            self.mask_paths[f] = os.path.join(root, "masks", f"{f}.png")
            cv2.imwrite(self.img_paths[f], img)
            cv2.imwrite(self.mask_paths[f], np.repeat(mask[..., None], 3, axis=2))
            kp = np.concatenate([rng.uniform([0.2 * W, 0.1 * H], [0.8 * W, 0.9 * H], (133, 2)),
                                 rng.uniform(0, 1, (133, 1))], axis=1).astype(np.float32)
            kp[0, 2] = 1.0
            self.kpts[f] = kp
            self.cam_params[f] = {"R": cam["R"].numpy().astype(np.float32),
                                  "t": (cam["t"].numpy() + np.float32(0.002 * i)).astype(np.float32),
                                  "focal": cam["focal"].numpy().astype(np.float32),
                                  "princpt": cam["princpt"].numpy().astype(np.float32)}
        self.frame_idx_list = list(frame_ids) * repeat

    def __len__(self):
        return len(self.frame_idx_list)

    def __getitem__(self, idx):
        frame_idx = self.frame_idx_list[idx]
        img = cv2.imread(self.img_paths[frame_idx], cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)
        img = img[:, :, ::-1].copy().astype(np.float32)                       # load_img
        img = torch.from_numpy(img.transpose((2, 0, 1))).contiguous() / 255.  # ToTensor(img) / 255.
        mask = cv2.imread(self.mask_paths[frame_idx])[:, :, 0, None] / 255.
        mask = torch.from_numpy((mask > 0.5).astype(np.float32).transpose((2, 0, 1))).contiguous()
        joint_img = self.kpts[frame_idx][:, :2]
        joint_valid = (self.kpts[frame_idx][:, 2:] > 0.5).astype(np.float32)
        bbox = get_bbox(joint_img, joint_valid[:, 0])
        return {"img": img, "mask": mask, "bbox": bbox, "cam_param": self.cam_params[frame_idx],
                "frame_idx": frame_idx}


def chain_inputs(data, bg):
    """Chain.terms' inputs from a collated batch of one frame (on the device) and the background."""
    cam = data["cam_param"]
    return {"img": data["img"][0], "bbox": data["bbox"][0], "R": cam["R"][0], "t": cam["t"][0],
            "focal": cam["focal"][0], "princpt": cam["princpt"][0], "bg": bg}


def shutdown(it):
    """Joins a DataLoader iterator's worker processes."""
    stop = getattr(it, "_shutdown_workers", None)
    if stop is not None:
        stop()


PER_GRAPH = 20  # unpacks in one captured graph: the graph arm's time per unpack is the kernel's, not a launch's


def unpack_bytes(H, W):
    return H * W * (4 + 16) + 20 * 4 * 2 + 8 * 2 + 4 * 2  # pixels in, planes out; box and camera; index; slot and row


def measure_unpack(a, dev, H, W, tmp):
    n = 8
    ds = NeumanFrames(os.path.join(tmp, f"unpack_{H}x{W}"), list(range(n)), H, W)
    frames = FrameTable.from_dataset(ds, dev, workers=min(8, n))
    slot = torch.zeros(1, dtype=torch.int32, device=dev)

    def eager():
        frames(slot)

    replay = graph_replay(lambda: [frames(slot) for _ in range(PER_GRAPH)], warmup=1)
    times = alternate({"eager": eager, "graph": replay}, a.iters * 50, a.rounds, warmup=5)
    times["graph"] = [v / PER_GRAPH for v in times["graph"]]
    nbytes = unpack_bytes(H, W)
    out = {"bytes": nbytes, "unpacks_per_graph": PER_GRAPH}
    for k, v in times.items():
        us = stats(v, 1e6, 2)
        out[k] = {"us": us, "GB_per_s": round(nbytes / (us["median"] * 1e-6) / 1e9, 1),
                  "of_3.35_TB_per_s": round(nbytes / (us["median"] * 1e-6) / HBM_BYTES_PER_S, 3)}
    return out


def measure_e2e(a, dev, H, W, F, tmp):
    from bench_iteration_graph import Chain
    ds = NeumanFrames(os.path.join(tmp, f"e2e_{H}x{W}"), list(range(F)), H, W, repeat=2)
    n_iter = a.warmup + a.rounds * a.iters
    positions = np.random.default_rng(0).integers(0, len(ds), n_iter).tolist()
    bgs = torch.rand((n_iter, 3), generator=torch.Generator().manual_seed(1)).pin_memory()
    capacity = int(8_000_000 * max(1.0, H * W / 512 ** 2))
    chains = {k: Chain(dev, "table", F, H, W, 130_000, use_graph=False, capacity=capacity) for k in ("loader", "table")}
    t0 = time.perf_counter()
    frames = FrameTable.from_dataset(ds, dev, slots=chains["table"].table.frames, workers=8)
    build_s = time.perf_counter() - t0
    cl = chains["loader"]
    it_l = IterationGraph(lambda ins, slot_t: cl.terms(cl.table(slot_t), ins, False), cl.opt,
                          chain_inputs(frames(0), torch.zeros(3, device=dev)))
    ct = chains["table"]
    it_t = IterationGraph(lambda ins, slot_t: ct.terms(ct.table(slot_t), chain_inputs(frames(slot_t), ins["bg"]), False),
                          ct.opt, {"bg": torch.zeros(3, device=dev)})
    pos = {"loader": 0, "table": 0}
    first = {}
    batches = None

    def one(name):
        i = pos[name]
        pos[name] += 1
        if name == "loader":
            b = next(batches) if batches is not None else default_collate([ds[positions[i]]])
            slot = frames.slot_of(int(b["frame_idx"][0]))
            terms = it_l.run(chain_inputs(b, bgs[i]), slot, key=False)
        else:
            slot = frames.slot_of(ds.frame_idx_list[positions[i]])
            terms = it_t.run({"bg": bgs[i]}, slot, key=False)
        if i == 0:
            first[name] = {k: v.clone() for k, v in terms.items()}
            first[name + "_inputs"] = ({k: v.clone() for k, v in it_l.inputs.items() if k != "bg"} if name == "loader"
                                      else {k: v.clone() for k, v in chain_inputs(frames(slot), None).items()
                                            if k != "bg"})

    try:
        # the warm-up holds each arm's captures; a capture must not overlap the loader's pin-memory thread (its host
        # allocations invalidate a capture in progress), so the loader starts after them, at the first timed iteration
        for name in ("loader", "table"):
            for _ in range(a.warmup):
                one(name)
        torch.cuda.synchronize()
        batches = iter(DataLoader(ds, batch_size=1, sampler=positions[a.warmup:], num_workers=8, pin_memory=True))
        bitwise = lambda x, y: {k: torch.equal(x[k].view(torch.int32), y[k].view(torch.int32)) for k in x}  # noqa: E731
        same_inputs = bitwise(first["loader_inputs"], first["table_inputs"])
        if not all(same_inputs.values()):
            raise SystemExit(f"bench_frame_table: the two arms' first inputs differ: {same_inputs}")
        same = bitwise(first["loader"], first["table"])
        diff = {k: float((first["loader"][k] - first["table"][k]).abs()) for k, v in same.items() if not v}
        res = {k: {"s": [], "host": []} for k in ("loader", "table")}
        for _ in range(a.rounds):
            for name in ("loader", "table"):
                torch.cuda.synchronize()
                t0, host = time.perf_counter(), 0.0
                for _ in range(a.iters):
                    h0 = time.perf_counter()
                    one(name)
                    host += time.perf_counter() - h0
                torch.cuda.synchronize()
                res[name]["s"].append((time.perf_counter() - t0) / a.iters)
                res[name]["host"].append(host / a.iters)
    finally:
        shutdown(batches)
        batches = None
    for c in chains.values():
        if c.fr.overflowed():
            raise SystemExit("bench_frame_table: a render overflowed its list capacity")
    out = {k: {"iters_per_s": stats([1 / s for s in v["s"]], nd=2), "host_ms": stats(v["host"], 1e3, 3)}
           for k, v in res.items()}
    out.update(first_inputs_bit_identical=True, first_loss_terms_bit_identical=all(same.values()),
               first_loss_terms_differing=diff, table_build_s=round(build_s, 2), table_bytes=frames.nbytes,
               frames=F, list_capacity=capacity)
    return out


def main():
    ap = arg_parser(__doc__, iters=20, rounds=3)
    ap.add_argument("--sizes", default="512x512,1080x1920", help="H x W of the frames")
    ap.add_argument("--frames", type=int, default=100, help="distinct frames F of the end-to-end arms")
    ap.add_argument("--warmup", type=int, default=4, help="untimed iterations per end-to-end arm")
    a = ap.parse_args()
    dev = cuda_device("bench_frame_table")
    out = {"card": card(), "host_cpus": os.cpu_count(), "host_cpus_usable": len(os.sched_getaffinity(0)),
           "iters_per_window": a.iters, "rounds": a.rounds,
           "workload": "C4 iteration (130 000 scene + 167 618 human Gaussians, SMPL-X rig, l1_ssim x5, regulariser "
                       "op) under IterationGraph"}
    with tempfile.TemporaryDirectory(prefix="bench_frame_table_") as tmp:
        for size in a.sizes.split(","):
            H, W = (int(x) for x in size.split("x"))
            out[f"unpack {H}x{W}"] = measure_unpack(a, dev, H, W, tmp)
            print(f"unpack {H}x{W}:", out[f"unpack {H}x{W}"], flush=True)
            out[f"e2e {H}x{W}"] = measure_e2e(a, dev, H, W, a.frames, tmp)
            print(f"e2e {H}x{W}:", out[f"e2e {H}x{W}"], flush=True)
            torch.cuda.empty_cache()
    out["card_after"] = card()
    emit(out, a.json)


if __name__ == "__main__":
    main()
