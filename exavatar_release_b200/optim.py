"""`Adam`: ExAvatar's optimizer step (avatar/common/base.py:83-85, `torch.optim.Adam(params, lr=0.0, eps=1e-15)`) as
one CUDA launch per `step()`, bit-identical to torch's default foreach path.

The class is a `torch.optim.Optimizer` with torch.optim.Adam's state layout: `state[p]` holds `step` (0-dim CPU
float32), `exp_avg` and `exp_avg_sq` (shaped, typed and placed as p), and the param groups keep their keys (`name`,
`lr`, `betas`, `eps`).  ExAvatar's `set_lr`, its optimizer surgery (module.py:17-72) and state dicts of either class
work unchanged.  `step()` is `stage()` then `launch()`, two calls of the compiled binding (csrc_torch/b2r_torch.cpp):
`stage()` walks the groups, creates the lazy state, advances the step counts, computes every tensor's scalars with
torch's own double expressions (rounded to fp32 once), stages the segment table in pinned memory and copies it into a
resident device table with one async H2D copy; `launch()` is one launch of csrc/adam.cu on the current stream, which
a CUDA graph can capture and replay after each `stage()`.  Nothing copies back and nothing synchronises.
"""
from __future__ import annotations

import torch

from . import _lib as L

_CHUNK = None


def _chunk() -> int:
    global _CHUNK
    if _CHUNK is None:
        _CHUNK = int(L.load().b2r_adam_chunk_elems())
    return _CHUNK


def _binding():
    from .rasterizer import _compiled_binding
    return _compiled_binding()


class StaleLayoutError(RuntimeError):
    """Adam.stage() after a captured launch(): the staged layout is not the one the graph holds."""


class Adam(torch.optim.Optimizer):
    """Drop-in for `torch.optim.Adam(params, lr, betas, eps)` on fp32 CUDA tensors of one device.

    What ExAvatar does not use raises `ValueError` instead of taking a slower path: weight_decay != 0, amsgrad,
    maximize, sparse grads, and parameters that are not fp32 CUDA tensors of one device or whose layout is neither
    contiguous nor rows of contiguous floats at one stride (the views feature[:, 0:1] and feature[:, 1:] of ExAvatar's
    scene features are such rows).  Gradients and state must be contiguous, as autograd and zeros_like make them.

    Frame rows: a param group with `frame_rows=True`, e.g. {'params': [table.pose, table.expr, table.trans],
    'frame_rows': True, 'name': 'smplx', 'lr': ...}, holds params whose dim 0 is the frame (SmplxParamTable's).
    `step(rows=slot)` steps only row `slot` of each of them, with that row's own step count: state[p]["step"] is a
    (frames,) CPU float32 tensor, torch's 0-dim per-param step once per row.  Over any frame sequence this is
    bit-identical to torch.optim.Adam over ExAvatar's per-frame groups (module.py:666-671) with zero_grad(set_to_none)
    each iteration; the other rows, and their moments and counts, stay untouched.  Stepping such a group without
    `rows` raises ValueError.  state_dict() / load_state_dict() round-trip, but the per-row step counts make that
    state unloadable by torch.optim.Adam (ExAvatar never reloads optimizer state).
    """

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0,
                 amsgrad: bool = False, *, maximize: bool = False):
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError(f"Invalid beta parameters: {betas}")
        self._table = None     # the resident device segment table stage() writes and launch() reads
        self._staged = None    # (n_segments, n_chunks, layout, device index) of the last stage()
        self._captured = None  # the layout a captured launch() pinned
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                                      maximize=maximize))

    def _check_group(self, group):
        if group.get("weight_decay", 0) != 0:
            raise ValueError("Adam: weight_decay != 0 is not supported")
        if group.get("amsgrad", False):
            raise ValueError("Adam: amsgrad is not supported")
        if group.get("maximize", False):
            raise ValueError("Adam: maximize is not supported")
        for k in ("capturable", "differentiable", "fused"):  # keys of a loaded torch.optim.Adam state dict
            if group.get(k):
                raise ValueError(f"Adam: {k}=True is not supported")
        for p in group["params"]:
            self._check_param(p)
            if group.get("frame_rows", False) and (p.dim() < 1 or not p.is_contiguous()):
                raise ValueError("Adam: a frame-row parameter must be contiguous with dim 0 = frame")

    def _device(self):
        """The CUDA device of the first parameter: every parameter has to live there."""
        for group in self.param_groups:
            for p in group["params"]:
                return p.device
        return None

    def _check_param(self, p):
        if p.dtype != torch.float32 or p.device.type != "cuda":
            raise ValueError(f"Adam: parameters must be float32 CUDA tensors, got {p.dtype} on {p.device}")
        dev = self._device()
        if dev is not None and p.device != dev:
            raise ValueError(f"Adam: parameters on more than one device ({dev} and {p.device})")
        if not _binding().adam_row_layout(p)[0]:
            raise ValueError("Adam: a parameter must be contiguous or rows of contiguous floats at one stride")

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        self._check_group(self.param_groups[-1])

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        for group in self.param_groups:
            self._check_group(group)

    def stage(self, rows=None) -> None:
        """The host half of `step()`: walks the groups, creates the lazy state, advances the step counts, computes
        every tensor's scalars from the groups' current lr in torch's doubles (rounded once) and writes the segment
        table into the optimizer's resident device table with one async H2D copy on the current stream.  Nothing
        synchronises.  `rows` is the frame slot that frame-row groups step (see the class).

        After a `launch()` was captured in a CUDA graph, that graph reads this table at a fixed address with a fixed
        segment and chunk count.  A stage whose layout differs from the captured one -- another set of params with
        gradients, new tensors after optimizer surgery, another chunk count -- raises `StaleLayoutError` before it
        creates, counts or writes anything; `release_graph()` forgets the captured layout.  One layout is pinned at a
        time: every graph holding a `launch()` of this optimizer must stage the same params with gradients."""
        dev = self._device()
        if dev is None:
            self._staged = None
            return
        table, n_seg, n_chunks, layout = _binding().adam_stage(self.param_groups, self.state, dev.index, _chunk(),
                                                                rows, self._table, self._captured)
        if self._captured is not None and layout != self._captured:
            raise StaleLayoutError("Adam.stage: the parameters, their gradients or their sizes changed since "
                                   "launch() was captured in a CUDA graph; drop that graph and call release_graph() "
                                   "instead of replaying it")
        self._table = table
        self._staged = (n_seg, n_chunks, layout, dev.index)

    def launch(self) -> None:
        """The device half of `step()`: one launch of the Adam kernel over the table `stage()` wrote, on the current
        stream.  It reads everything from device memory, so a CUDA graph can capture it and replay it after each
        `stage()`; a captured launch pins the staged layout (see `stage`)."""
        if self._staged is None:
            return
        n_seg, n_chunks, layout, index = self._staged
        if torch.cuda.is_current_stream_capturing():
            self._captured = layout
        if n_chunks == 0:  # no parameter with a gradient (or only empty ones): nothing to launch, as before the split
            return
        _binding().adam_launch(self._table, n_seg, n_chunks, index)

    def release_graph(self) -> None:
        """Forgets the layout a captured `launch()` pinned: call it when the graphs holding that launch are dropped."""
        self._captured = None

    @torch.no_grad()
    def step(self, closure=None, rows=None):
        """`stage(rows)` then `launch()`: one Adam step over every param with a gradient."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.stage(rows)
        self.launch()
        return loss

    def __setstate__(self, state):  # a copy or unpickled optimizer starts with no staging and no captured graph
        super().__setstate__(state)
        for k in ("_table", "_staged", "_captured"):
            self.__dict__.setdefault(k, None)
