"""`FrameTable`: every training frame of an ExAvatar split on one CUDA device, the frame of a slot read on the device
(csrc/frames.cu b2r_frame_unpack), so that a captured training iteration reads its image, mask, box and camera itself
instead of having them copied in from a DataLoader on every iteration.

    frames = FrameTable.from_dataset(trainset, "cuda", slots=param_table.frames)   # NeuMan / Custom, decoded once
    data = frames(slot_t)          # inside IterationGraph's step_fn: the collated batch of the frame, for Model.forward

Storage, per distinct frame (row) of the split, on one device:

    pixels    (N, H, W, 4) uint8   R, G, B as ExAvatar's bytes, and the training mask as 0 / 1
    bbox      (N, 4)       fp32
    R         (N, 3, 3)    fp32
    t         (N, 3)       fp32
    focal     (N, 2)       fp32
    princpt   (N, 2)       fp32
    frame_idx (N,)         int64
    slot_row  (F,)         int32   slot -> row, -1 for a slot without a frame

at 4 bytes per pixel (1 000 frames at 1080 x 1920 are 8.3 GB).  `table(slot)` expands the row into fresh tensors shaped
and typed like torch's default collate of `dataset[i]` with batch size 1, bit for bit: the image is fl(k / 255) per
byte k, which is what NeuMan / Custom `__getitem__` compute (`ToTensor(img) / 255.` of cv2's bytes), and also what
eval_neuman's float64 read of the same PNG rounds to in fp32.
"""
from __future__ import annotations

import ctypes as C
import numbers

import torch
from torch.utils.data import DataLoader, Dataset

from . import _lib as L

# the fp32 per-frame values besides the pixels, in the order of one table row's metadata
META = (("bbox", (4,)), ("R", (3, 3)), ("t", (3,)), ("focal", (2,)), ("princpt", (2,)))
_ONE_BITS = 0x3F800000  # 1.0f


def pack_frame(data, frame_idx: int) -> dict:
    """One `dataset[i]` dict as a table row: {"pixels": (H, W, 4) uint8, "meta": {name: fp32 tensor}, "frame_idx"}.
    Raises ValueError naming the frame unless `img` is (3, H, W) fp32 of values k / 255 (fp32 division) for bytes k,
    `mask` is (1, H, W) fp32 of 0 and 1, the box and camera are fp32 of ExAvatar's shapes and `frame_idx` is the one
    the dataset's frame list gives."""
    where = f"FrameTable: frame {frame_idx}"
    got = data["frame_idx"]
    if isinstance(got, bool) or not isinstance(got, numbers.Integral) or int(got) != frame_idx:
        raise ValueError(f"{where}: `frame_idx` is {got!r}")
    img, mask = torch.as_tensor(data["img"]), torch.as_tensor(data["mask"])
    if img.dtype != torch.float32 or img.dim() != 3 or img.shape[0] != 3:
        raise ValueError(f"{where}: `img` must be (3, H, W) float32, got {img.dtype} {tuple(img.shape)}")
    H, W = img.shape[1:]
    if mask.dtype != torch.float32 or tuple(mask.shape) != (1, H, W):
        raise ValueError(f"{where}: `mask` must be (1, {H}, {W}) float32, got {mask.dtype} {tuple(mask.shape)}")
    img, mask = img.contiguous(), mask.contiguous()
    u = torch.round(img * 255)
    if not bool(((u >= 0) & (u <= 255)).all()) or not torch.equal((u / 255.).view(torch.int32), img.view(torch.int32)):
        raise ValueError(f"{where}: `img` holds a value that is not k / 255 for a byte k")
    mb = mask.view(torch.int32)
    if not bool(((mb == 0) | (mb == _ONE_BITS)).all()):
        raise ValueError(f"{where}: `mask` holds a value other than 0 and 1")
    cam = data["cam_param"]
    meta = {}
    for name, shape in META:
        v = torch.as_tensor(data["bbox"] if name == "bbox" else cam[name])
        if v.dtype != torch.float32 or tuple(v.shape) != shape:
            raise ValueError(f"{where}: `{name}` must be {shape} float32, got {v.dtype} {tuple(v.shape)}")
        meta[name] = v
    pixels = torch.stack((u[0], u[1], u[2], mask[0]), dim=-1).to(torch.uint8)
    return {"pixels": pixels, "meta": meta, "frame_idx": frame_idx}


class _Rows(Dataset):
    """The distinct frames of a dataset, row r read at its first position in `frame_idx_list` and packed."""

    def __init__(self, dataset, positions, frame_ids):
        self.dataset, self.positions, self.frame_ids = dataset, positions, frame_ids

    def __len__(self):
        return len(self.positions)

    def __getitem__(self, r):
        return pack_frame(self.dataset[self.positions[r]], self.frame_ids[r])


def _same_size(rows, frame_ids):
    """The packed rows in order, each checked to have the first one's (H, W) before it is passed on."""
    size = None
    for r, row in enumerate(rows):
        hw = tuple(row["pixels"].shape[:2])
        if size is None:
            size = hw
        elif hw != size:
            raise ValueError(f"FrameTable: frame {frame_ids[r]} is {hw[0]}x{hw[1]}, the first frame "
                             f"{size[0]}x{size[1]}; all frames must have one size")
        yield row


def _upload(rows, n, device) -> dict:
    """The table's device arrays from the checked rows: the pixel array is allocated when the first row arrives, and
    every row goes up through one pinned staging buffer, so the host holds a few frames at a time."""
    pixels = staging = done = None
    meta = {name: [] for name, _ in META}
    ids = []
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
        for r, row in enumerate(rows):
            px = row["pixels"]
            if pixels is None:
                pixels = torch.empty((n, *px.shape), dtype=torch.uint8, device=device)
                staging = torch.empty(px.shape, dtype=torch.uint8, pin_memory=True)
                done = torch.cuda.Event()
            else:
                done.synchronize()  # the previous row's copy has read the staging buffer
            staging.copy_(px)
            pixels[r].copy_(staging, non_blocking=True)
            done.record()
            for name, _ in META:
                meta[name].append(row["meta"][name])
            ids.append(row["frame_idx"])
        out = {name: torch.stack(v).to(device) for name, v in meta.items()}
        out["frame_idx"] = torch.tensor(ids, dtype=torch.int64).to(device)
        torch.cuda.current_stream(device).synchronize()
    out["pixels"] = pixels
    return out


def _slot_keys(slots, frame_ids):
    """The slot keys (str) and the slot of each frame of the split; raises ValueError on bad or duplicate keys and on
    a frame that has no slot."""
    fn = "FrameTable.from_dataset"
    if slots is None:
        keys = [str(f) for f in frame_ids]
    else:
        if isinstance(slots, (str, bytes, torch.Tensor)) or not isinstance(slots, (list, tuple)):
            raise ValueError(f"{fn}: `slots` must be a list of frame keys (str or int), got {type(slots).__name__}")
        keys = []
        for s in slots:
            if isinstance(s, str):
                keys.append(s)
            elif isinstance(s, numbers.Integral) and not isinstance(s, bool):
                keys.append(str(int(s)))
            else:
                raise ValueError(f"{fn}: a slot key must be a str or an int, got {type(s).__name__}")
        if not keys:
            raise ValueError(f"{fn}: `slots` is empty")
        seen = set()
        for k in keys:
            if k in seen:
                raise ValueError(f"{fn}: slot key {k!r} appears more than once")
            seen.add(k)
    if len(keys) >= 2 ** 31:
        raise ValueError(f"{fn}: at most 2^31 - 1 slots")
    slot_of = {k: i for i, k in enumerate(keys)}
    missing = [f for f in frame_ids if str(f) not in slot_of]
    if missing:
        raise ValueError(f"{fn}: frame {missing[0]} of the dataset has no slot in `slots`")
    return keys, [slot_of[str(f)] for f in frame_ids]


class FrameTable:
    """Every distinct frame of a split on one CUDA device; `table(slot)` is the frame's collated batch, one launch."""

    def __init__(self, pixels, bbox, R, t, focal, princpt, frame_idx, slot_row, slots):
        """The device arrays of the module docstring, used as they are; `slots` the F slot keys (str) in order."""
        fn = "FrameTable"
        dev = pixels.device if isinstance(pixels, torch.Tensor) else None
        arrays = (("pixels", pixels, torch.uint8), ("bbox", bbox, torch.float32), ("R", R, torch.float32),
                  ("t", t, torch.float32), ("focal", focal, torch.float32), ("princpt", princpt, torch.float32),
                  ("frame_idx", frame_idx, torch.int64), ("slot_row", slot_row, torch.int32))
        for name, x, dtype in arrays:
            L.cuda(fn, name, x, dev)
            if x.dtype != dtype or not x.is_contiguous():
                raise ValueError(f"{fn}: `{name}` must be contiguous {dtype}, got {x.dtype}")
        N = pixels.shape[0] if pixels.dim() == 4 else 0
        if N < 1 or pixels.shape[3] != 4 or pixels.shape[1] < 1 or pixels.shape[2] < 1:
            raise ValueError(f"{fn}: `pixels` must be (N, H, W, 4) with N >= 1, got {tuple(pixels.shape)}")
        for (name, shape), x in zip(META, (bbox, R, t, focal, princpt)):
            if tuple(x.shape) != (N, *shape):
                raise ValueError(f"{fn}: `{name}` must be ({N}, *{shape}), got {tuple(x.shape)}")
        if tuple(frame_idx.shape) != (N,):
            raise ValueError(f"{fn}: `frame_idx` must be ({N},), got {tuple(frame_idx.shape)}")
        F = len(slots)
        if tuple(slot_row.shape) != (F,) or F < 1:
            raise ValueError(f"{fn}: `slot_row` must be ({F},) for the {F} slots, got {tuple(slot_row.shape)}")
        rows = slot_row.cpu()
        if bool(((rows < -1) | (rows >= N)).any()):
            raise ValueError(f"{fn}: `slot_row` values must lie in [-1, {N})")
        self.pixels, self.bbox, self.R, self.t, self.focal, self.princpt = pixels, bbox, R, t, focal, princpt
        self.frame_idx, self.slot_row = frame_idx, slot_row
        self.device = dev
        self.n_rows, self.height, self.width = N, int(pixels.shape[1]), int(pixels.shape[2])
        self.frames = list(slots)
        self._slot = {k: i for i, k in enumerate(self.frames)}
        self._row = rows.tolist()

    @property
    def n_slots(self) -> int:
        return len(self.frames)

    @property
    def nbytes(self) -> int:
        """Device bytes of the table."""
        return sum(x.numel() * x.element_size() for x in (self.pixels, self.bbox, self.R, self.t, self.focal,
                                                         self.princpt, self.frame_idx, self.slot_row))

    @classmethod
    def from_dataset(cls, dataset, device, slots=None, workers: int = 8) -> "FrameTable":
        """The table of an ExAvatar dataset (NeuMan, Custom: `frame_idx_list` and `dataset[i]`'s dict of img, mask,
        bbox, cam_param and frame_idx), each distinct frame read once, at its first position in `frame_idx_list`,
        through a DataLoader with `workers` processes; every worker has exited when this returns or raises.

        `slots`: the slot keys, e.g. `SmplxParamTable.frames`, so that one device slot drives both tables (a slot
        without a frame of the split maps to no row); default the split's frames in first-appearance order.  Raises
        ValueError for bad or duplicate keys, a frame of the dataset without a slot, frames of different sizes, an
        image value that is not k / 255 or a mask value other than 0 and 1, naming the frame, before anything is
        allocated or uploaded for it."""
        fn = "FrameTable.from_dataset"
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError(f"{fn}: the table lives on a CUDA device, got {device}; there is no CPU fallback")
        if isinstance(workers, bool) or not isinstance(workers, numbers.Integral) or workers < 0:
            raise ValueError(f"{fn}: `workers` must be an int >= 0, got {workers!r}")
        first = {}
        for pos, f in enumerate(dataset.frame_idx_list):
            if isinstance(f, bool) or not isinstance(f, numbers.Integral):
                raise ValueError(f"{fn}: frame_idx_list[{pos}] is {f!r}, not an int")
            first.setdefault(int(f), pos)
        if not first:
            raise ValueError(f"{fn}: the dataset has no frames")
        frame_ids = list(first)
        keys, frame_slots = _slot_keys(slots, frame_ids)
        loader = DataLoader(_Rows(dataset, [first[f] for f in frame_ids], frame_ids), batch_size=None,
                            shuffle=False, num_workers=int(workers))
        it = iter(loader)
        try:
            arrays = _upload(_same_size(it, frame_ids), len(frame_ids), device)
        finally:
            shutdown = getattr(it, "_shutdown_workers", None)  # joins the worker processes, also on an error
            if shutdown is not None:
                shutdown()
            del it
        slot_row = torch.full((len(keys),), -1, dtype=torch.int32)
        slot_row[torch.tensor(frame_slots, dtype=torch.int64)] = torch.arange(len(frame_ids), dtype=torch.int32)
        return cls(arrays["pixels"], *(arrays[name] for name, _ in META), arrays["frame_idx"],
                   slot_row.to(arrays["pixels"].device), keys)

    def slot_of(self, frame_idx) -> int:
        """The slot of a frame: its key, or ExAvatar's int frame index (looked up as str(int(frame_idx)))."""
        key = frame_idx if isinstance(frame_idx, str) else str(int(frame_idx))
        if key not in self._slot:
            raise KeyError(f"FrameTable: no frame {key!r}")
        return self._slot[key]

    def __call__(self, slot) -> dict:
        """The collated batch of the frame in `slot`: {"img": (1,3,H,W), "mask": (1,1,H,W), "bbox": (1,4),
        "cam_param": {"R": (1,3,3), "t": (1,3), "focal": (1,2), "princpt": (1,2)}, "frame_idx": (1,) int64}, fresh
        tensors.  `slot` is a host int (checked on the host: IndexError outside [0, F) or for a slot without a frame)
        or a one-element int32 CUDA tensor read on the device; for a device slot outside [0, F) or without a frame,
        no row is read: the float outputs are NaN and frame_idx -1.  Nothing is read back to the host."""
        fn = "FrameTable"
        if isinstance(slot, torch.Tensor):
            L.cuda(fn, "slot", slot, self.device)
            if slot.dtype != torch.int32 or slot.numel() != 1 or not slot.is_contiguous():
                raise ValueError(f"{fn}: a tensor `slot` must be one contiguous int32 value, got {slot.dtype} "
                                 f"{tuple(slot.shape)}")
            slot_t, host_slot = slot, 0
        elif isinstance(slot, numbers.Integral) and not isinstance(slot, bool):
            if not 0 <= int(slot) < self.n_slots:
                raise IndexError(f"{fn}: slot {int(slot)} outside [0, {self.n_slots})")
            if self._row[int(slot)] < 0:
                raise IndexError(f"{fn}: slot {int(slot)} ({self.frames[int(slot)]!r}) has no frame in the table")
            slot_t, host_slot = None, int(slot)
        else:
            raise ValueError(f"{fn}: `slot` must be an int or a (1,) int32 CUDA tensor, got {type(slot).__name__}")
        dev, H, W = self.device, self.height, self.width
        img = torch.empty((1, 3, H, W), dtype=torch.float32, device=dev)
        mask = torch.empty((1, 1, H, W), dtype=torch.float32, device=dev)
        meta = {name: torch.empty((1, *shape), dtype=torch.float32, device=dev) for name, shape in META}
        frame_idx = torch.empty((1,), dtype=torch.int64, device=dev)
        st = L.B2RFrameTable(n_rows=self.n_rows, n_slots=self.n_slots, height=H, width=W, host_slot=host_slot,
                             pixels=L.ptr(self.pixels), **{name: L.ptr(getattr(self, name)) for name, _ in META},
                             frame_idx=L.ptr(self.frame_idx), slot_row=L.ptr(self.slot_row), slot=L.ptr(slot_t))
        L.run("b2r_frame_unpack", dev, C.byref(st), L.ptr(img), L.ptr(mask),
              *(L.ptr(meta[name]) for name, _ in META), L.ptr(frame_idx))
        return {"img": img, "mask": mask, "bbox": meta["bbox"],
                "cam_param": {k: meta[k] for k in ("R", "t", "focal", "princpt")}, "frame_idx": frame_idx}
