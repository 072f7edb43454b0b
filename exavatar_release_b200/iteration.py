"""`IterationGraph`: ExAvatar's whole training iteration -- forward, backward and the Adam step -- as one CUDA graph per
key, replayed for every frame.

What makes that possible: `SmplxParamTable` reads the frame's SMPL-X parameters through a slot on the device, so one
graph serves every frame; `Adam.stage(rows=slot)` does a step's host work (step counts, lr, scalars) and writes the
segment table into a resident device table, so the captured `Adam.launch()` replays with this iteration's scalars; and
frame-row param groups step only the frame's row of the table, as torch.optim.Adam over ExAvatar's per-frame groups
does.

    it = IterationGraph(step_fn, optimizer, {"img": img, "mask": mask, "bbox": box, "R": R, "t": t, "focal": f,
                                             "princpt": c, "bg": bg})   # templates of the static inputs
    for itr, data in enumerate(loader):
        set_lr(optimizer, itr)                                           # the host stages the new lr
        if surgery_happened:                                             # densification replaced the scene tensors
            it.invalidate()
        slot = table.slot_of(data["frame_idx"])
        losses = it.run(inputs, slot, key=(cfg.is_warmup, sh_degree))

`step_fn(inputs, slot)` is the caller's forward and backward of one iteration: it reads the static input buffers
(`inputs`, a dict) and the (1,) int32 CUDA `slot`, calls `loss.backward()` and returns its loss terms (a dict of
tensors).  It uses the ops with `TrainingFrameRenderer(use_graph=False)` -- a graph cannot be launched inside a capture
-- and must not read the device on the host.

Protocol, per key (the caller's hashable: e.g. HumanAssets.geometry's warm-up flag and the host SH degree):
  - the first iteration of a key runs eagerly: `step_fn`, then `optimizer.step(rows=slot)`;
  - the next one is captured -- gradients zeroed, `step_fn`, `optimizer.launch()` -- on one memory pool shared by every
    key's graph, and replayed once; the capture itself runs nothing;
  - later ones stage the inputs and `optimizer.stage(rows=slot)` on the host and replay.
So every iteration runs exactly once, and neither Adam nor the densification statistics see a warm-up pass.

Gradients: every iteration starts from zero gradients, zeroed in place (inside the graph once captured), so each
parameter's `.grad` keeps one address that every key's graph writes and the staged Adam pointers stay valid.  The
caller must not `zero_grad(set_to_none=True)` or replace a `.grad`.

Layout: the optimizer pins one layout -- the params with gradients and their tensors -- for all of its captured
graphs, so every key's iteration must give gradients to the same params (ExAvatar's warm-up and later iterations do).
A key whose eager iteration leaves a different set raises `StaleLayoutError` from its Adam step, after its backward.

Invalidation: `invalidate()` drops the graphs; call it after anything that replaces the optimizer's tensors (ExAvatar's
densification surgery, every 100 iterations between 500 and 15 000).  The next iteration of each key runs the
eager-then-capture protocol again.  Without it, the replay's `optimizer.stage()` sees the new layout and raises
`StaleLayoutError` instead of replaying a graph that holds the old tensors.

Autograd history: autograd runs a leaf's AccumulateGrad on the stream its node was created on, and the node lives as
long as any graph that reaches the leaf.  A view of a parameter taken with grad enabled outside `run` (e.g.
`table.pose[slot]` for logging) and kept alive binds that node to the caller's stream, and the next capture's backward
would have to make that stream wait on the capture, which CUDA refuses.  Take such views under `torch.no_grad()` or
from `.detach()`.

Losses: the returned tensors (detached) are static outputs of the graph, valid until the next `run`; reading them on
the host synchronises, which is the caller's choice (ExAvatar's train.py:67 logs every iteration).

Host-side state of the ops inside `step_fn` is frozen at capture: `TrainingFrameRenderer._frame_no` counts Python calls
and stops counting under replay; it feeds no computation.  Per-iteration values must come in through `inputs` or the
slot: ExAvatar's `torch.rand(3)` background is drawn by the caller and staged as `bg`.
"""
from __future__ import annotations

from typing import Callable, Dict, Hashable

import torch

from .optim import Adam, StaleLayoutError


def _detached(losses):
    # the loss terms must not keep an iteration's autograd graph alive: its AccumulateGrad nodes stay bound to the
    # stream they were created on, and a later capture on another stream would wait on that stream and fail
    return {k: v.detach() for k, v in losses.items()}


class IterationGraph:
    def __init__(self, step_fn: Callable, optimizer: Adam, inputs: Dict[str, torch.Tensor], device=None):
        """`inputs` maps each static input's name to a template tensor (shape and dtype); the buffers live on
        `device` (default: the optimizer's)."""
        if not isinstance(optimizer, Adam):
            raise TypeError("IterationGraph: the optimizer must be exavatar_release_b200.Adam (stage() / launch())")
        device = torch.device(device) if device is not None else optimizer._device()
        if device is None or device.type != "cuda":
            raise RuntimeError(f"IterationGraph: a CUDA device is needed, got {device}")
        self.step_fn, self.optimizer, self.device = step_fn, optimizer, device
        self.inputs = {k: torch.zeros(v.shape, dtype=v.dtype, device=device) for k, v in inputs.items()}
        self.slot = torch.zeros(1, dtype=torch.int32, device=device)
        self._warm = set()   # keys whose eager iteration ran
        self._graphs = {}    # key -> (graph, loss terms)
        self._pool = None

    def _grads(self):
        return [p.grad for gr in self.optimizer.param_groups for p in gr["params"] if p.grad is not None]

    def _stage_inputs(self, inputs, slot: int) -> None:
        if set(inputs) != set(self.inputs):
            raise ValueError(f"IterationGraph: inputs must be {sorted(self.inputs)}, got {sorted(inputs)}")
        for k, v in inputs.items():
            self.inputs[k].copy_(v, non_blocking=True)
        self.slot.fill_(slot)

    def run(self, inputs: Dict[str, torch.Tensor], slot: int, key: Hashable = None) -> Dict[str, torch.Tensor]:
        """One training iteration on frame slot `slot` (a host int), in the graph of `key`; returns the loss terms."""
        slot = int(slot)
        self._stage_inputs(inputs, slot)
        if key in self._graphs:
            g, losses = self._graphs[key]
            try:
                self.optimizer.stage(rows=slot)
            except StaleLayoutError as e:
                raise StaleLayoutError(f"IterationGraph: {e}; call invalidate() after optimizer surgery") from None
            g.replay()
            return losses
        for gr in self._grads():
            gr.zero_()
        if key not in self._warm:  # the key's first iteration: eager
            losses = _detached(self.step_fn(self.inputs, self.slot))
            self.optimizer.step(rows=slot)
            self._warm.add(key)
            return losses
        # the capture bakes in the staged table's size, so stage first; a capture that fails takes the counts back
        state = self.optimizer.state
        had = set(state)
        counts = [(st["step"], st["step"].clone()) for st in state.values() if "step" in st]
        self.optimizer.stage(rows=slot)
        g = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(g, pool=self._pool):
                for gr in self._grads():
                    gr.zero_()
                losses = _detached(self.step_fn(self.inputs, self.slot))
                self.optimizer.launch()
        except BaseException:
            for step, before in counts:
                step.copy_(before)
            for p in set(state) - had:
                del state[p]
            if not self._graphs:
                self.optimizer.release_graph()
            raise
        if self._pool is None:
            self._pool = g.pool()
        self._graphs[key] = (g, losses)
        g.replay()
        return losses

    def invalidate(self) -> None:
        """Drops every graph (after optimizer surgery); the next iteration of each key runs eagerly again."""
        self._graphs.clear()
        self._warm.clear()
        self._pool = None
        self.optimizer.release_graph()
