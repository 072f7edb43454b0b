"""Frame sharding over ranks with one gradient all-reduce per step (SURVEY.md section 8e).

The reference trains one frame at a time on one GPU (`cfg.num_gpus = 1`, `cfg.batch_size = 1`,
/root/reference/avatar/main/config.py:44-45) and has no collective anywhere.  Frames are independent units
(avatar/main/model.py:81 loops per frame), so this build shards them: rank r renders frames r, r+world, ... of the
step's batch against a full replica of the Gaussian parameters, every frame's gradients are summed into ONE flat
fp32 bucket per rank, and the ranks sum their buckets with a single all-reduce (NCCL on GPUs, gloo in CPU tests).
The loss of each frame is pre-divided by the global batch size so the reduced gradient equals the gradient of
`loss.mean()` over the whole batch (avatar/main/train.py:43) and `mean_2d.grad` keeps the magnitude the densification
threshold expects (avatar/main/config.py:21).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Sequence

import torch
import torch.distributed as dist


def shard_frames(num_frames: int, rank: int, world: int) -> List[int]:
    """Indices of the batch's frames this rank renders (round-robin, as SURVEY section 8e)."""
    if not (0 <= rank < world):
        raise ValueError(f"rank {rank} outside world of {world}")
    return list(range(rank, num_frames, world))


class GradBucket:
    """Named views into one flat fp32 buffer, so a step needs exactly one collective."""

    def __init__(self, shapes: Dict[str, Sequence[int]], device="cpu"):
        self.shapes = {k: tuple(v) for k, v in shapes.items()}
        total = sum(int(torch.Size(s).numel()) for s in self.shapes.values())
        self.flat = torch.zeros(total, dtype=torch.float32, device=device)
        self.views, o = {}, 0
        for k, s in self.shapes.items():
            n = int(torch.Size(s).numel())
            self.views[k] = self.flat[o:o + n].view(*s)
            o += n

    def zero_(self):
        self.flat.zero_()

    def add_(self, grads: Dict[str, torch.Tensor]):
        for k, g in grads.items():
            if g is not None and k in self.views:
                self.views[k].add_(g.reshape(self.views[k].shape))

    def all_reduce(self):
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM)
        return self.flat


def sharded_step(frames: Sequence, frame_grads: Callable[[object, float], Dict[str, torch.Tensor]], bucket: GradBucket,
                 rank: int = 0, world: int = 1) -> torch.Tensor:
    """Runs this rank's share of `frames`; `frame_grads(frame, loss_scale)` returns that frame's per-tensor gradients.

    Returns the all-reduced flat bucket (identical on every rank).
    """
    bucket.zero_()
    scale = 1.0 / max(len(frames), 1)
    for i in shard_frames(len(frames), rank, world):
        bucket.add_(frame_grads(frames[i], scale))
    return bucket.all_reduce()


def reduce_densify_stats(stats: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The second, small collective of a sharded step (SURVEY.md section 8e): ExAvatar's densification bookkeeping of the
    scene Gaussians -- `xyz_grad_accum` and `track_cnt` are SUMS over the frames of the batch, `radius_max` a MAX
    (avatar/common/nets/module.py:111-113, 155-157; avatar/main/model.py:283-285) -- so every replica prunes and
    densifies from the statistics of the whole batch.  Keys: 'grad_accum', 'count', 'radius_max' (in place)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(stats["grad_accum"], op=dist.ReduceOp.SUM)
        dist.all_reduce(stats["count"], op=dist.ReduceOp.SUM)
        dist.all_reduce(stats["radius_max"], op=dist.ReduceOp.MAX)
    return stats


def split_noise_generator(step: int, device="cpu", base_seed: int = 0) -> torch.Generator:
    """Generator for `split_points`' `torch.normal` (avatar/common/nets/module.py:198).  Replicas must clone and split
    the SAME Gaussians at the SAME offsets or their parameter sets diverge; seeding from the step counter (identical on
    every rank) instead of the process-global RNG makes the draw independent of what each rank rendered before."""
    g = torch.Generator(device=device)
    g.manual_seed((int(base_seed) * 1_000_003 + int(step)) & 0x7FFFFFFF)
    return g
