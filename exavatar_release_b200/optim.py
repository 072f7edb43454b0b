"""`Adam`: ExAvatar's optimizer step (avatar/common/base.py:83-85, `torch.optim.Adam(params, lr=0.0, eps=1e-15)`) as
one CUDA launch per `step()`, bit-identical to torch's default foreach path.

The class is a `torch.optim.Optimizer` with torch.optim.Adam's state layout: `state[p]` holds `step` (0-dim CPU
float32), `exp_avg` and `exp_avg_sq` (shaped, typed and placed as p), and the param groups keep their keys (`name`,
`lr`, `betas`, `eps`).  ExAvatar's `set_lr`, its optimizer surgery (module.py:17-72) and state dicts of either class
work unchanged.  `step()` is one call of the compiled binding (csrc_torch/b2r_torch.cpp `adam_step`): it walks the
groups, creates the lazy state, advances the step counts, computes every tensor's scalars with torch's own double
expressions (rounded to fp32 once), stages the segment table in pinned memory, copies it with one async H2D copy and
makes one launch of csrc/adam.cu on the current stream; nothing copies back and nothing synchronises.
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


class Adam(torch.optim.Optimizer):
    """Drop-in for `torch.optim.Adam(params, lr, betas, eps)` on fp32 CUDA tensors of one device.

    What ExAvatar does not use raises `ValueError` instead of taking a slower path: weight_decay != 0, amsgrad,
    maximize, sparse grads, and parameters that are not fp32 CUDA tensors of one device or whose layout is neither
    contiguous nor rows of contiguous floats at one stride (the views feature[:, 0:1] and feature[:, 1:] of ExAvatar's
    scene features are such rows).  Gradients and state must be contiguous, as autograd and zeros_like make them.
    """

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0,
                 amsgrad: bool = False, *, maximize: bool = False):
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError(f"Invalid beta parameters: {betas}")
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

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        dev = self._device()
        if dev is not None:
            _binding().adam_step(self.param_groups, self.state, dev.index, _chunk())
        return loss
