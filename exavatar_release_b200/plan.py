"""`FramePlan`: allocation-free, sync-free, CUDA-graph-capturable use of the C ABI.

The autograd front-end (`rasterizer.py`) must size buffers per call because it cannot know the caller's next scene.
A training loop that renders the same Gaussian set frame after frame (ExAvatar: avatar/main/train.py:24-57) can do
better: fix the duplicate capacity once, keep every buffer resident, and enqueue forward + backward with no host
round-trip at all -- which also makes the whole step capturable in a CUDA graph (`torch.cuda.graph`), so a step of F
frames costs one graph launch instead of ~9 F kernel launches.  Overflow of the fixed capacity is detected from the
device status block (`status()`), checked by the caller outside the hot loop.

Gradients are written (or, with `accumulate=True`, summed) into caller-provided tensors, e.g. views of the flat
bucket that is all-reduced once per step (SURVEY.md section 8e).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib as L
from .rasterizer import _f32c, _make_scene

# the per-Gaussian asset tensors of a render: asset key -> (name of its gradient, floats per Gaussian)
ASSETS = {"mean_3d": ("means3D", 3), "opacity": ("opacities", 1), "scale": ("scales", 3), "rotation": ("rotations", 4),
          "rgb": ("colors", 3)}


def _backward_args(images, grads, accumulate: bool = False, first_row: int = 0, densify=None, densify_rows: int = 0):
    """B2RBackwardArgs of (dL/dcolor, dL/ddepth, dL/dalpha) `images` and the named gradient outputs `grads` (keys
    means3D, means2D, shs, colors, opacities, scales, rotations, cov3D; missing -> not written).  `densify`:
    {'grad_accum', 'count', 'radius_max'} updated for rows [0, densify_rows) (0: all)."""
    outs = [grads.get(k) for k in ("means3D", "means2D", "shs", "colors", "opacities", "scales", "rotations", "cov3D")]
    dens = [(densify or {}).get(k) for k in ("grad_accum", "count", "radius_max")]
    flags = (L.B2R_BWD_ACCUMULATE if accumulate else 0) | L.B2R_BWD_SCRATCH_ZEROED
    return L.B2RBackwardArgs(*map(L.ptr, images), *map(L.ptr, outs), flags, int(first_row), *map(L.ptr, dens),
                             int(densify_rows) if densify is not None else 0)


class _Workspace:
    """The resident buffers of one projection + binning of P Gaussians with a fixed duplicate capacity, and the
    B2RWorkspace pointing at them: ctx (status block first), duplicate ids, forward scratch, backward scratch and the
    forward composite's segment table + blend-state checkpoints."""

    def __init__(self, P: int, width: int, height: int, dup_capacity: int, device, split: bool = False):
        self.lib = L.load()
        self.P, self.W, self.H = int(P), int(width), int(height)
        self.device = dev = torch.device(device)
        self.capacity = int(dup_capacity)
        self.radii = torch.empty(P, dtype=torch.int32, device=dev)
        self.ctx_bytes = self.lib.b2r_ctx_bytes(P, width, height)
        self.ctx_buf = torch.empty(self.ctx_bytes, dtype=torch.uint8, device=dev)
        self.ids = torch.empty(max(self.capacity, 1), dtype=torch.int32, device=dev)
        # a split pass (b2r_forward_bin_split) keeps the sorted ids of its own rows behind the keys
        nbytes = self.lib.b2r_split_scratch_bytes if split else self.lib.b2r_scratch_bytes
        self.scratch_bytes = nbytes(P, width, height, self.capacity)
        self.scratch = torch.empty(self.scratch_bytes, dtype=torch.uint8, device=dev)
        self.bwd_bytes = self.lib.b2r_backward_scratch_bytes(P)
        # zero once: every backward leaves it zero again (B2R_BWD_SCRATCH_ZEROED), so no memset node per render
        self.bwd_scratch = torch.zeros(self.bwd_bytes, dtype=torch.uint8, device=dev)
        # segment table + blend-state checkpoints of the forward composite: the backward replays 512-entry list
        # segments as independent work items
        self.ckpt_bytes = self.lib.b2r_checkpoint_bytes(width, height, self.capacity)
        self.ckpt = torch.empty(max(self.ckpt_bytes, 1), dtype=torch.uint8, device=dev)
        self.ws = L.B2RWorkspace(self.ctx_buf.data_ptr(), self.ctx_bytes, self.ids.data_ptr(), self.capacity,
                                 self.scratch.data_ptr(), self.scratch_bytes, None, 0, self.ckpt.data_ptr(),
                                 self.ckpt_bytes)

    def status(self) -> dict:
        return L.read_status(self.ctx_buf)


class FramePlan(_Workspace):
    def __init__(self, P: int, width: int, height: int, dup_capacity: int, device, sh_coeffs: int = 0):
        super().__init__(P, width, height, dup_capacity, device)
        self.M = int(sh_coeffs)
        f = lambda *s: torch.empty(s, dtype=torch.float32, device=self.device)
        self.color, self.depth, self.alpha = f(3, height, width), f(1, height, width), f(1, height, width)
        self.out = L.B2RForwardOutputs(self.color.data_ptr(), self.depth.data_ptr(), self.alpha.data_ptr(),
                                       self.radii.data_ptr())
        self._scenes = {}
        self._primed = False

    def scene(self, key, settings, assets: Dict[str, torch.Tensor], flags: int = 0):
        """Builds (and caches under `key`) the B2RScene for one frame; tensors must stay alive and in place."""
        if key in self._scenes:
            return self._scenes[key][0]
        g = lambda k: None if assets.get(k) is None else _f32c(assets[k], k)
        shs = g("shs") if self.M > 0 else None
        sc, keep = _make_scene(settings, g("mean_3d"), shs, None if shs is not None else g("rgb"), g("opacity"),
                               g("scale"), g("rotation"), None, flags)
        self._scenes[key] = (sc, keep)
        return sc

    def forward(self, sc) -> None:
        # from the second forward on the ctx counters are known to be zero (every forward leaves them so): no reset launch
        base = sc.flags & ~L.B2R_FLAG_CTX_CLEAN
        sc.flags = base | (L.B2R_FLAG_CTX_CLEAN if self._primed else 0)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream(self.device).cuda_stream
            L.check(self.lib.b2r_forward(C.byref(sc), C.byref(self.ws), C.byref(self.out), st), "b2r_forward")
        sc.flags = base
        self._primed = True

    def backward(self, sc, g_color: torch.Tensor, grads: Dict[str, Optional[torch.Tensor]], accumulate: bool = False,
                 g_depth: Optional[torch.Tensor] = None, g_alpha: Optional[torch.Tensor] = None,
                 densify: Optional[Dict[str, torch.Tensor]] = None, first_row: int = 0) -> None:
        """grads keys: means3D, means2D, shs, colors, opacities, scales, rotations, cov3D (missing -> not written).
        densify (optional): {'grad_accum', 'count', 'radius_max'} fp32 (P) tensors updated in place by the backward
        projection kernel -- ExAvatar's `track_stats` + `radius_max` update (module.py:155-157, model.py:283-285).
        first_row: Gaussians [0, first_row) are a detached prefix (cat(scene.detach(), human), model.py:117-125): the
        `grads` tensors then have P - first_row rows and receive the gradient of the remaining Gaussians only."""
        a = _backward_args((g_color, g_depth, g_alpha), grads, accumulate, first_row, densify)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream(self.device).cuda_stream
            L.check(self.lib.b2r_backward(C.byref(sc), C.byref(self.ws), C.byref(a), self.bwd_scratch.data_ptr(),
                                          self.bwd_bytes, st), "b2r_backward")


def grad_bucket(P: int, device, sh_coeffs: int = 0):
    """One flat fp32 buffer holding every per-Gaussian gradient, plus named views into it."""
    per = 3 + 3 + 1 + 3 + 4 + (3 * sh_coeffs if sh_coeffs > 0 else 3)
    return _views_of(torch.zeros(per * P, dtype=torch.float32, device=device), P, sh_coeffs)


class FrameLanes:
    """S concurrent `FramePlan`s ("lanes"), each on its own CUDA stream with its own workspace and gradient bucket.

    Frames of a training batch are independent (SURVEY.md section 8e; avatar/main/model.py:81 loops over them), and at
    ExAvatar's sizes a single frame cannot fill an H100: the scan / sort kernels are latency-bound single-wave launches
    and the composites end in a tail of long tile lists.  Running frame f on lane f mod S lets the hardware fill those
    holes with another frame's kernels.  The lanes fork from and join back into the caller's current stream, so the
    whole step is still one CUDA-graph capture.  Gradients of the frames of one lane are summed inside the backward
    projection kernel (`accumulate`); the S lane buckets are then added in a fixed order (deterministic result) into
    `bucket`, the tensor that is all-reduced once per step.
    """

    def __init__(self, lanes: int, P: int, width: int, height: int, dup_capacity: int, device, sh_coeffs: int = 0):
        self.S = max(1, int(lanes))
        self.device = torch.device(device)
        self.plans = [FramePlan(P, width, height, dup_capacity, device, sh_coeffs) for _ in range(self.S)]
        self.streams = [torch.cuda.Stream(self.device) for _ in range(self.S)]
        flat0, _ = grad_bucket(P, device, sh_coeffs)
        self.lane_flat = torch.zeros(self.S, flat0.numel(), dtype=torch.float32, device=device)
        self.lane_views = []
        for s in range(self.S):
            _, v = _views_of(self.lane_flat[s], P, sh_coeffs)
            self.lane_views.append(v)
        self.bucket = self.lane_flat[0] if self.S == 1 else flat0
        _, self.views = _views_of(self.bucket, P, sh_coeffs)

    def scene(self, key, settings, assets, flags: int = 0):
        return self.plans[0].scene(key, settings, assets, flags)

    def step(self, scenes, g_colors, backward: bool = True) -> None:
        """Forward (+ backward) of every frame in `scenes`; on return (stream order) `bucket` holds the summed gradients."""
        cur = torch.cuda.current_stream(self.device)
        F = len(scenes)
        for s in range(self.S):
            st = self.streams[s]
            st.wait_stream(cur)
            with torch.cuda.stream(st):
                plan = self.plans[s]
                for j, f in enumerate(range(s, F, self.S)):
                    plan.forward(scenes[f])
                    if backward:
                        plan.backward(scenes[f], g_colors[f], self.lane_views[s], accumulate=(j > 0))
        for st in self.streams:
            cur.wait_stream(st)
        if backward and self.S > 1:
            torch.sum(self.lane_flat[: min(self.S, F)], dim=0, out=self.bucket)

    def status(self) -> dict:
        sts = [p.status() for p in self.plans]
        out = dict(sts[0])
        out["overflow"] = int(any(s["overflow"] for s in sts))
        return out


def _views_of(flat: torch.Tensor, P: int, sh_coeffs: int = 0):
    widths = [("means3D", 3), ("means2D", 3), ("opacities", 1), ("scales", 3), ("rotations", 4)]
    widths.append(("shs", 3 * sh_coeffs) if sh_coeffs > 0 else ("colors", 3))
    views, o = {}, 0
    for name, w in widths:
        views[name] = flat[o:o + w * P].view(P, w) if name != "shs" else flat[o:o + w * P].view(P, sh_coeffs, 3)
        o += w * P
    return flat, views


RENDERS = ("scene", "human", "scene_human", "human_refined", "scene_human_refined")


class _FiveRenders:
    """What the two five-render plans share: the row width of their gradient buckets, the densification sums at the
    tail of the flat bucket (`_stats`) and the status of their workspaces (`_ws`: name -> _Workspace)."""
    PER = 3 + 3 + 1 + 3 + 4 + 3  # floats per Gaussian in a bucket

    def stats(self) -> Dict[str, torch.Tensor]:
        """Per-step sums of ExAvatar's densification statistics (module.py:155-157), stored at the tail of the flat
        bucket so the step's ONE sum all-reduce covers them; zero them at the start of a step (`zero_stats`)."""
        return {"grad_accum": self._stats[: self.Ps], "count": self._stats[self.Ps:]}

    def zero_stats(self) -> None:
        self._stats.zero_()

    def dups(self) -> Dict[str, int]:
        return {k: w.status()["num_dups"] for k, w in self._ws.items()}

    def overflowed(self) -> bool:
        return any(w.status()["overflow"] for w in self._ws.values())


class FiveRenderPlan(_FiveRenders):
    """One ExAvatar training frame = five rasteriser calls with one camera (avatar/main/model.py:81-162):

        scene                      -> gradients to the scene Gaussians
        human            (bg rand) -> gradients to the human Gaussians
        cat(scene.detach(), human) -> gradients to the human Gaussians only        (model.py:117-125)
        human_refined    (bg rand) -> gradients to the refined human Gaussians
        cat(scene.detach(), human_refined) -> gradients to the refined human Gaussians only

    The reference runs them one after the other, each with its own device->host sync.  Here the five renders are
    independent until their gradients meet, so each runs on its own CUDA stream (fork / join inside the caller's
    stream: capturable in one CUDA graph with the rest of the step); the "detached prefix" of the combined renders is a
    field of the backward call (`first_row`), so the human part of their gradient is written straight into a
    human-sized bucket and nothing is computed-then-discarded on the host side.  Frames of a step accumulate into the
    same five buckets; `reduce()` folds them into the three parameter sets (scene, human, human_refined).

    All gradients live in ONE flat fp32 buffer (`flat_bucket()`: scene | human | human_refined after `reduce()`), the
    tensor a multi-GPU step all-reduces once (SURVEY.md section 8e).  `MergedFivePlan` below produces the same results
    from two projection / binning passes instead of five (SURVEY.md section 8f-3).
    """

    def __init__(self, P_scene: int, P_human: int, width: int, height: int, caps: Optional[Dict[str, int]], device):
        self.Ps, self.Ph = int(P_scene), int(P_human)
        self.device = torch.device(device)
        caps = caps or {r: 8_000_000 for r in RENDERS}
        sizes = {"scene": self.Ps, "human": self.Ph, "scene_human": self.Ps + self.Ph, "human_refined": self.Ph,
                 "scene_human_refined": self.Ps + self.Ph}
        self._ws = self.plans = {r: FramePlan(sizes[r], width, height, caps[r], device) for r in RENDERS}
        self.streams = {r: torch.cuda.Stream(self.device) for r in RENDERS}
        self.first_row = {"scene": 0, "human": 0, "scene_human": self.Ps, "human_refined": 0, "scene_human_refined": self.Ps}
        out_rows = {"scene": self.Ps, "human": self.Ph, "scene_human": self.Ph, "human_refined": self.Ph,
                    "scene_human_refined": self.Ph}
        # one allocation: [scene | human | human_refined | scene_human | scene_human_refined]; the first three segments
        # are what reduce() leaves the step's gradients in
        order = ("scene", "human", "human_refined", "scene_human", "scene_human_refined")
        tail = 2 * self.Ps  # per-step densification sums of the scene Gaussians ride in the all-reduced buffer (stats())
        self.all_flat = torch.zeros(self.PER * sum(out_rows[r] for r in order) + tail, dtype=torch.float32, device=device)
        self.flat, self.views, o = {}, {}, 0
        for r in order:
            n = self.PER * out_rows[r]
            self.flat[r], self.views[r] = _views_of(self.all_flat[o:o + n], out_rows[r])
            o += n
            if r == "human_refined":
                self._stats = self.all_flat[o:o + tail]
                o += tail
        self._reduced = self.PER * (self.Ps + 2 * self.Ph) + tail
        f = lambda w: torch.empty(self.Ps + self.Ph, w, dtype=torch.float32, device=device)
        self.cat = {r: {k: f(w) for k, (_, w) in ASSETS.items()} for r in ("scene_human", "scene_human_refined")}

    def describe(self) -> str:
        return "five independent renders (project+bin+sort+composite each) on five CUDA streams per frame"

    def set_scene(self, scene_assets: Dict[str, torch.Tensor]) -> None:
        """Copies the (detached) scene Gaussians into the prefix of the two combined asset sets; once per step."""
        for r in self.cat:
            for k, buf in self.cat[r].items():
                buf[: self.Ps].copy_(scene_assets[k].reshape(self.Ps, -1))

    def assets_of(self, render: str, scene, human, refined):
        if render == "scene":
            return scene
        if render in ("human", "human_refined"):
            return human if render == "human" else refined
        src = human if render == "scene_human" else refined
        for k, buf in self.cat[render].items():
            buf[self.Ps:].copy_(src[k].reshape(self.Ph, -1))
        return self.cat[render]

    def frame(self, key, settings, settings_human_bg, scene, human, refined, g_colors: Dict[str, torch.Tensor],
              accumulate: bool, densify: Optional[Dict[str, torch.Tensor]] = None, serial: bool = False) -> None:
        """Forward + backward of the five renders of one frame.  `settings_human_bg` carries the random background of
        the human-only renders (model.py:72).  `key` caches the per-(frame, render) scene descriptors.  `densify`:
        ExAvatar's densification statistics of the SCENE Gaussians, fed by the scene render (model.py:193, 279-285).
        `serial`: all five on the caller's stream, one after the other (per-kernel profiling)."""
        cur = torch.cuda.current_stream(self.device)
        for r in RENDERS:
            st = cur if serial else self.streams[r]
            if not serial:
                st.wait_stream(cur)
            with torch.cuda.stream(st):
                plan = self.plans[r]
                assets = self.assets_of(r, scene, human, refined)
                sc = plan.scene((key, r), settings_human_bg if r in ("human", "human_refined") else settings, assets)
                plan.forward(sc)
                plan.backward(sc, g_colors[r], self.views[r], accumulate=accumulate, first_row=self.first_row[r],
                              densify=densify if r == "scene" else None)
        if not serial:
            for r in RENDERS:
                cur.wait_stream(self.streams[r])

    def render_outputs(self, render: str):
        """(color (3,H,W), alpha (1,H,W), radii) of one of the five renders of the last frame (valid until the next)."""
        p = self.plans[render]
        return p.color, p.alpha, p.radii

    def reduce(self):
        """(scene, human, human_refined) flat gradient buckets of the step (the first three segments of the flat bucket;
        the combined renders' human rows are folded in, in a fixed order)."""
        self.flat["human"].add_(self.flat["scene_human"])
        self.flat["human_refined"].add_(self.flat["scene_human_refined"])
        return self.flat["scene"], self.flat["human"], self.flat["human_refined"]

    def grads(self, which: str) -> Dict[str, torch.Tensor]:
        """Named gradient tensors of one parameter set ("scene" | "human" | "human_refined"), valid after reduce()."""
        return dict(self.views[which])

    def flat_bucket(self) -> torch.Tensor:
        return self.all_flat[: self._reduced]

    def consumed(self) -> Dict[str, list]:
        st = [self.plans[r].status() for r in RENDERS]
        return {"fwd": [s["consumed_fwd"] / s["consumed_fwd_div"] for s in st],
                "bwd": [s["consumed_bwd"] / s["consumed_bwd_div"] for s in st]}


class _Pass(_Workspace):
    """One projection + binning of cat(scene, X) and the views composited from it (MergedFivePlan)."""

    def __init__(self, P, W, H, cap, n_views, device, split=False):
        super().__init__(P, W, H, cap, device, split=split)
        dev = self.device
        # every view keeps its own checkpoints for its backward; the workspace points at the first view's
        self.ck = [self.ckpt] + [torch.empty_like(self.ckpt) for _ in range(n_views - 1)]
        f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        self.img = [(f(3, H, W), f(1, H, W), f(1, H, W)) for _ in range(n_views)]
        self.state = [(f(H * W), torch.empty(H * W, dtype=torch.int32, device=dev)) for _ in range(n_views)]
        self.cat = {k: f(P, w) for k, (_, w) in ASSETS.items()}
        self.streams = [torch.cuda.Stream(dev) for _ in range(n_views)]
        self.primed = False


def merged_bucket_layout(P_scene: int, P_human: int, sh_coeffs: int = 0) -> Dict[str, tuple]:
    """(offset, numel) of every region of `MergedFivePlan`'s flat gradient buffer, in floats:

        A      pass A, `_views_of` layout with P_scene + P_human rows (means3D | means2D | opacities | scales | rotations
               | colors); with an SH scene the colour rows of the scene are written as zeros
        A_shs  (P_scene, M, 3) dL/dSH of the scene Gaussians (sh_coeffs = M > 0 only; numel 0 otherwise)
        B      pass B, `_views_of` layout with P_human rows (the refined human set)
        stats  per-step densification sums of the scene Gaussians (grad_accum | count), the tail of the buffer
        total  the whole buffer

    sh_coeffs = 0 is the layout of a plan without SH: A | B | stats."""
    PER = _FiveRenders.PER
    Ps, Ph, M = int(P_scene), int(P_human), int(sh_coeffs)
    nA, nS, nB = PER * (Ps + Ph), 3 * M * Ps, PER * Ph
    return {"A": (0, nA), "A_shs": (nA, nS), "B": (nA + nS, nB), "stats": (nA + nS + nB, 2 * Ps),
            "total": (0, nA + nS + nB + 2 * Ps)}


class MergedFivePlan(_FiveRenders):
    """ExAvatar's five renders per training frame (avatar/main/model.py:81-162) from TWO projection + binning passes
    instead of five (SURVEY.md section 8f-3, kernel half):

        pass A  Gaussians cat(scene, human)          views  scene-only | human-only (random bg) | both
        pass B  Gaussians cat(scene, human_refined)  views               human-only (random bg) | both

    The five renders share one camera, so the scene Gaussians project, bin and depth-sort identically in renders 1, 3, 5
    and the human Gaussians in 2, 3 (refined: 4, 5).  A view (B2RView) composites the merged per-tile lists keeping only
    one index range -- entries of the other population are dropped when a batch is staged -- with its own background and
    per-pixel state.  Backward: the views of a pass accumulate their screen-space gradients into ONE scratch (the
    combined view skips the detached scene prefix, `first_row`), and the backward projection runs once per pass: scene
    rows carry the scene render's gradient, human rows the sum of the human-only and the combined render's -- what
    `loss.backward()` leaves in the leaves of model.py:117-125.  Same results as five separate renders (tests/), 2/5 of
    the projection / scatter / sort work.  Interface of FiveRenderPlan.

    sh_coeffs = M > 0: the scene Gaussians are coloured from (P_scene, M, 3) SH coefficients inside the projection
    kernels (SURVEY.md section 8f-4) and the human sets from RGB -- both passes are mixed-source scenes
    (B2RScene.sh_rows = P_scene) reading ONE coefficient buffer (`use_scene_shs`).  The scene assets then carry `shs` +
    `sh_degree` instead of `rgb`, and `grads("scene")` holds `shs` instead of `colors`."""
    VIEWS = {"A": ("scene", "human", "scene_human"), "B": ("human_refined", "scene_human_refined")}
    # Pass B projects, bins and sorts only the refined rows and takes the scene entries of its lists from pass A (the
    # split pass of the C ABI).  SPLIT = False: the whole cat(scene, refined) again, the reference the tests compare the
    # split pass against.  Read per frame; pass B's scratch is sized by its value at construction (the split pass needs
    # more, so a split-built plan may be switched to the whole pass).
    SPLIT = True

    def __init__(self, P_scene: int, P_human: int, width: int, height: int, caps: Optional[Dict[str, int]], device,
                 sh_coeffs: int = 0):
        self.lib = L.load()
        self.Ps, self.Ph, self.P = int(P_scene), int(P_human), int(P_scene) + int(P_human)
        self.W, self.H = int(width), int(height)
        self.M = int(sh_coeffs)
        self.device = torch.device(device)
        caps = caps or {"A": 8_000_000, "B": 8_000_000}
        self._ws = self.passes = {k: _Pass(self.P, self.W, self.H, caps[k], len(v), self.device,
                                           split=(k == "B" and self.SPLIT)) for k, v in self.VIEWS.items()}
        self.pass_streams = {k: torch.cuda.Stream(self.device) for k in self.passes}
        # one flat gradient buffer: [pass A: scene rows | human rows][scene dL/dSH][pass B: refined rows][stats]
        lay = merged_bucket_layout(self.Ps, self.Ph, self.M)
        self.all_flat = torch.zeros(lay["total"][1], dtype=torch.float32, device=device)
        o, n = lay["stats"]
        self._stats = self.all_flat[o:o + n]  # per-step densification sums ride in the all-reduced buffer (stats())
        o, n = lay["B"]
        _, (self.views_A, self.views_B) = self.grad_buffers((self.all_flat[:o], self.all_flat[o:o + n]))
        # the scene's SH coefficients: the caller's tensor (eager) or this resident copy (`use_scene_shs`)
        self.shs = torch.zeros(self.Ps, self.M, 3, dtype=torch.float32, device=device) if self.M > 0 else None
        self._shs_src, self.sh_degree = self.shs, 0
        Ps, P = self.Ps, self.P
        self.ranges = {"scene": (0, Ps), "human": (Ps, P), "scene_human": (0, P), "human_refined": (Ps, P),
                       "scene_human_refined": (0, P)}
        self.first_row = {"scene": 0, "human": Ps, "scene_human": Ps, "human_refined": Ps, "scene_human_refined": Ps}
        self._scenes = {}
        self._current = {}  # pass -> (descriptor, views) of the frame in flight
        self._keep = []

    def describe(self) -> str:
        return ("two merged passes per frame (cat(scene,human): 3 views; cat(scene,refined): 2 views), each one "
                "projection + binning + sort; composites of a pass on parallel CUDA streams")

    def set_scene(self, scene_assets: Dict[str, torch.Tensor]) -> None:
        for ps in self.passes.values():
            self._copy_rows(ps, scene_assets, scene=True)
        if self.M > 0:
            self.use_scene_shs(scene_assets["shs"], scene_assets["sh_degree"])

    def load_rows(self, human: Dict[str, torch.Tensor], refined: Dict[str, torch.Tensor]) -> None:
        """Copies the human and refined rows behind the scene prefix of pass A and pass B, on the current stream: what
        `forward_frame(copy_inputs=False)` leaves out, so that a captured graph reads fixed addresses and the copies
        from the caller's tensors stay outside it."""
        for ps, rows in zip(self.passes.values(), (human, refined)):
            self._copy_rows(ps, rows)

    def _copy_rows(self, ps, assets, scene: bool = False) -> None:
        """Copies the scene's rows (`scene`) into the prefix of pass `ps`, or the human or refined set's behind it."""
        lo, n = (0, self.Ps) if scene else (self.Ps, self.Ph)
        for k, buf in ps.cat.items():
            if not (scene and k == "rgb" and self.M > 0):  # SH scene: the colour rows of the scene are never read
                buf[lo:lo + n].copy_(assets[k].reshape(n, -1))

    def use_scene_shs(self, shs: torch.Tensor, sh_degree: int, copy: bool = False) -> None:
        """The scene's (P_scene, M, 3) SH coefficients and active degree for the next frames.  Both passes read ONE
        buffer: the caller's tensor itself when it is contiguous fp32 on the plan's device (it must then stay unchanged
        until the backward), otherwise -- or with copy=True, for a captured graph that reads fixed addresses -- the plan's
        resident copy `self.shs`."""
        if self.M == 0:
            raise ValueError("MergedFivePlan: built without SH (sh_coeffs=0); pass the scene colours as `rgb`")
        t = shs.detach()
        if tuple(t.shape) != (self.Ps, self.M, 3):
            raise ValueError(f"MergedFivePlan: scene `shs` must be ({self.Ps}, {self.M}, 3), got {tuple(t.shape)}")
        if copy or t.dtype != torch.float32 or not t.is_contiguous() or t.device != self.device:
            self.shs.copy_(t)
            t = self.shs
        self._shs_src, self.sh_degree = t, int(sh_degree)

    def _scene_desc(self, key, ps, settings):
        """B2RScene of a pass for one camera; cached under `key` (the settings' tensors are then kept alive), or built
        afresh when key[0] is None (a caller with a new camera every frame)."""
        def make():
            shs = self._shs_src if self.M > 0 else None
            sc, keep = _make_scene(settings, ps.cat["mean_3d"], shs, ps.cat["rgb"], ps.cat["opacity"], ps.cat["scale"],
                                   ps.cat["rotation"], None, 0)
            if shs is not None:  # scene rows from SH, human rows from RGB
                sc.sh_rows, sc.sh_degree = self.Ps, self.sh_degree
            return sc, keep

        if key[0] is None:
            sc, keep = make()
            ps.last_scene = (sc, keep)  # alive until the pass is used again
            return sc
        if self.M > 0:  # the descriptor holds the coefficient pointer and the degree
            key = (key, self._shs_src.data_ptr(), self.sh_degree)
        if key not in self._scenes:
            self._scenes[key] = make()
        return self._scenes[key][0]

    def _human_bg(self, settings_human_bg) -> torch.Tensor:
        """The background of the human-only views on the device, kept alive while views that read it may be queued."""
        bg_h = _f32c(settings_human_bg.bg.to(self.device), "bg")
        self._keep.append(bg_h)
        del self._keep[:-64]
        return bg_h

    def _view(self, ps, v, name, bg):
        lo, hi = self.ranges[name]
        fT, nc = ps.state[v]
        # Tiles no human Gaussian reaches: a combined view equals the scene-only view there and carries no gradient; a
        # human-only view shows the bare background there.  Both are pre-filled (`_forward_view`) and skipped by the
        # kernels.
        skip = self.Ps if name != "scene" else 0
        return L.B2RView(lo, hi, L.ptr(bg), fT.data_ptr(), nc.data_ptr(), ps.ck[v].data_ptr(), ps.ckpt_bytes, skip, 0)

    # ---- the steps of a frame; each enqueues on the stream `s` it is given, which is also the current stream ----
    def _start_pass(self, s, pk, key, settings, src, bg_h, a_binned) -> None:
        """Copies the rows of `src` (the human or refined set) behind the scene prefix of the pass -- src None: the
        caller already wrote them -- then projects and bins it.  Pass A records `a_binned` once its lists exist; a split
        pass B projects its refined rows, waits for it and merges the scene entries of pass A's lists into its own.  Its
        descriptor and views stay in `_current[pk]` until the next frame."""
        ps = self.passes[pk]
        if src is not None:
            self._copy_rows(ps, src)
        sc = self._scene_desc((key, pk), ps, settings)
        sc.flags = L.B2R_FLAG_CTX_CLEAN if ps.primed else 0  # every pass leaves its ctx counters zero
        ps.primed = True
        if pk == "B" and self.SPLIT:
            L.check(self.lib.b2r_forward_project_split(C.byref(sc), C.byref(ps.ws), self.Ps, ps.radii.data_ptr(),
                                                       s.cuda_stream), "b2r_forward_project_split")
            s.wait_event(a_binned)
            L.check(self.lib.b2r_forward_bin_split(C.byref(sc), C.byref(ps.ws), C.byref(self.passes["A"].ws), self.Ps,
                                                   ps.radii.data_ptr(), s.cuda_stream), "b2r_forward_bin_split")
        else:
            L.check(self.lib.b2r_forward_project(C.byref(sc), C.byref(ps.ws), ps.radii.data_ptr(), s.cuda_stream),
                    "b2r_forward_project")
            L.check(self.lib.b2r_forward_bin(C.byref(sc), C.byref(ps.ws), s.cuda_stream), "b2r_forward_bin")
            if pk == "A":
                a_binned.record(s)
        views = [self._view(ps, v, n, bg_h if n in ("human", "human_refined") else None)
                 for v, n in enumerate(self.VIEWS[pk])]
        self._current[pk] = (sc, views)

    def _forward_view(self, s, pk, v, bg_h, scene_done) -> None:
        """Forward composite of view v of pass pk, after the pre-fill of the tiles it skips.  The scene-only view records
        `scene_done`; the combined views of both passes copy its image."""
        ps, name = self.passes[pk], self.VIEWS[pk][v]
        sc, views = self._current[pk]
        color, depth, alpha = ps.img[v]
        if views[v].skip_below and name in ("human", "human_refined"):  # bare background, no depth / alpha
            color.copy_(bg_h.view(3, 1, 1).expand_as(color))
            depth.zero_()
            alpha.zero_()
        elif views[v].skip_below:  # pre-fill with the scene-only render; the composite overwrites human tiles
            s.wait_event(scene_done)
            for dst, src in zip(ps.img[v], self.passes["A"].img[0]):
                dst.copy_(src)
        out = L.B2RForwardOutputs(color.data_ptr(), depth.data_ptr(), alpha.data_ptr(), ps.radii.data_ptr())
        L.check(self.lib.b2r_forward_composite(C.byref(sc), C.byref(ps.ws), C.byref(views[v]), C.byref(out),
                                               s.cuda_stream), "b2r_forward_composite")
        if name == "scene":
            scene_done.record(s)

    def _backward_view(self, s, pk, v, g_color, g_depth, g_alpha) -> None:
        """Backward composite of view v of pass pk: its screen-space gradients are added into the pass's scratch.  No
        dL/dcolor: zeros.  The gradient images are kept alive while the launch may be queued."""
        ps = self.passes[pk]
        sc, views = self._current[pk]
        if g_color is None:
            g_color = torch.zeros(3, self.H, self.W, dtype=torch.float32, device=self.device)
        self._keep.append((g_color, g_depth, g_alpha))
        a = _backward_args((g_color, g_depth, g_alpha), {}, first_row=self.first_row[self.VIEWS[pk][v]])
        L.check(self.lib.b2r_backward_composite(C.byref(sc), C.byref(ps.ws), C.byref(views[v]), C.byref(a),
                                                ps.bwd_scratch.data_ptr(), ps.bwd_bytes, s.cuda_stream),
                "b2r_backward_composite")

    def _backward_project(self, s, pk, g, accumulate, densify) -> None:
        """The one backward projection of pass pk, from the scratch its views filled into the gradient views `g`."""
        ps = self.passes[pk]
        sc, _ = self._current[pk]
        # pass B: the scene prefix (SH rows included) is detached; the densification statistics are the scene rows'
        a = _backward_args((None, None, None), g, accumulate, first_row=0 if pk == "A" else self.Ps,
                           densify=densify if pk == "A" else None, densify_rows=self.Ps)
        L.check(self.lib.b2r_backward_project(C.byref(sc), C.byref(ps.ws), C.byref(a), ps.bwd_scratch.data_ptr(),
                                              ps.bwd_bytes, s.cuda_stream), "b2r_backward_project")

    def _walk(self, key=None, settings=None, settings_human_bg=None, rows=None, g_images=None, grads=None,
              accumulate: bool = False, densify=None, serial: bool = False, probe=None) -> None:
        """Enqueues a frame pass by pass.  With `settings`: its forward -- each pass starts (`rows[pass]`: the rows to
        copy behind its scene prefix, or None) and composites its views.  With `grads` (pass -> gradient views): its
        backward -- each view composites the gradients g_images = (g_colors, g_depths, g_alphas) of its render (dicts,
        None or a missing entry: no such gradient; a view with none at all is skipped), then each pass runs its backward
        projection into grads[pass].  Each pass runs on its own stream and forks one stream per view, on which the
        view's backward composite follows its forward composite; the pass joins its views before its backward
        projection.  `serial`: everything on the caller's stream, and `probe(label)` is called after every stage."""
        probe = probe if (probe is not None and serial) else (lambda label: None)
        cur = torch.cuda.current_stream(self.device)
        bg_h = self._human_bg(settings_human_bg) if settings is not None else None
        scene_done, a_binned = torch.cuda.Event(), torch.cuda.Event()
        for pk, names in self.VIEWS.items():
            ps = self.passes[pk]
            st = cur if serial else self.pass_streams[pk]
            if not serial:
                st.wait_stream(cur)
            with torch.cuda.stream(st):
                if settings is not None:
                    self._start_pass(st, pk, key, settings, rows[pk], bg_h, a_binned)
                    probe(f"{pk}:bin")
                for v, n in enumerate(names):
                    g = [(d or {}).get(n) for d in g_images] if grads is not None else [None] * 3
                    backward = any(x is not None for x in g)
                    if settings is None and not backward:
                        continue  # this render was not used downstream
                    vs = st if serial else ps.streams[v]
                    if not serial:
                        vs.wait_stream(st)
                    with torch.cuda.stream(vs):
                        if settings is not None:
                            self._forward_view(vs, pk, v, bg_h, scene_done)
                            probe(f"{pk}:{n}:fwd")
                        if backward:
                            self._backward_view(vs, pk, v, *g)
                            probe(f"{pk}:{n}:bwd")
                if not serial:
                    for v in range(len(names)):
                        st.wait_stream(ps.streams[v])
                if grads is not None:
                    self._backward_project(st, pk, grads[pk], accumulate, densify)
                    probe(f"{pk}:project_bwd")
        if not serial:
            for pk in self.passes:
                cur.wait_stream(self.pass_streams[pk])

    def frame(self, key, settings, settings_human_bg, scene, human, refined, g_colors: Dict[str, torch.Tensor],
              accumulate: bool, densify: Optional[Dict[str, torch.Tensor]] = None, serial: bool = False, probe=None) -> None:
        """Forward + backward of the five renders.  `serial`: everything on the caller's stream.  `probe(label)` (serial
        mode): called after every stage -- bench.py reads the in-library profiler there to get per-view kernel times."""
        self._walk(key, settings, settings_human_bg, {"A": human, "B": refined}, (g_colors, None, None),
                   {"A": self.views_A, "B": self.views_B}, accumulate, densify, serial, probe)

    # ---- the same frame in two halves (forward now, backward when the caller's gradients exist): fused.py ----
    def forward_frame(self, key, settings, settings_human_bg, scene, human, refined, copy_inputs: bool = True) -> None:
        """Forward of the five renders; images in `image()` / `render_outputs()`, per-pixel state and checkpoints stay
        in the plan until `backward_frame` (so the plan must not start another frame in between).  copy_inputs=False:
        the caller already wrote the human / refined rows (`load_rows`)."""
        rows = {"A": human, "B": refined} if copy_inputs else {"A": None, "B": None}
        self._walk(key, settings, settings_human_bg, rows)

    def backward_frame(self, g_colors: Dict[str, Optional[torch.Tensor]], grads_A: Dict[str, torch.Tensor],
                       grads_B: Dict[str, torch.Tensor], g_depths: Optional[Dict[str, torch.Tensor]] = None,
                       g_alphas: Optional[Dict[str, torch.Tensor]] = None, accumulate: bool = False,
                       densify: Optional[Dict[str, torch.Tensor]] = None) -> None:
        """Backward of the frame `forward_frame` rendered.  g_colors[name] = dL/dimage of a render, or None when the render
        was not used downstream.  grads_A / grads_B: pass A's and pass B's gradient views (`grad_buffers`)."""
        self._walk(g_images=(g_colors, g_depths, g_alphas), grads={"A": grads_A, "B": grads_B}, accumulate=accumulate,
                   densify=densify)

    def grad_buffers(self, flats=None):
        """((flat_a, flat_b), (views_a, views_b)): pass A's and pass B's gradient buffers -- `flats`, or a fresh
        uninitialised pair -- and their named views, what `backward_frame` takes as grads_A / grads_B.  flat_a is laid
        out as the A | A_shs regions of `merged_bucket_layout` (scene rows then human rows, plus the scene's dL/dSH
        (P_scene, M, 3) as "shs" when M > 0), flat_b as its B region (refined rows)."""
        lay = merged_bucket_layout(self.Ps, self.Ph, self.M)
        (_, na), (_, ns), (_, nb) = lay["A"], lay["A_shs"], lay["B"]
        if flats is None:
            flats = tuple(torch.empty(n, dtype=torch.float32, device=self.device) for n in (na + ns, nb))
        _, views_a = _views_of(flats[0][:na], self.P)
        if self.M > 0:
            views_a["shs"] = flats[0][na:].view(self.Ps, self.M, 3)
        _, views_b = _views_of(flats[1], self.Ph)
        return flats, (views_a, views_b)

    def image(self, render: str):
        """(color (3,H,W), depth (1,H,W), alpha (1,H,W)) of one of the five renders of the last frame (valid until the
        next)."""
        pk = "A" if render in self.VIEWS["A"] else "B"
        return self.passes[pk].img[self.VIEWS[pk].index(render)]

    def render_outputs(self, render: str):
        color, _, alpha = self.image(render)
        lo, hi = self.ranges[render]
        return color, alpha, self.passes["A" if render in self.VIEWS["A"] else "B"].radii[lo:hi]

    def reduce(self):
        """(scene, human, human_refined) flat gradient buckets of the step.  Nothing to fold: the backward projection of
        a pass already summed the renders that share a parameter set.  NOTE the buckets are row-interleaved views of the
        pass buffers (means3D of all rows, then means2D ...); `grads(which)` gives named per-set tensors."""
        return self.grads("scene"), self.grads("human"), self.grads("human_refined")

    def grads(self, which: str) -> Dict[str, torch.Tensor]:
        """Named gradient tensors of one parameter set; an SH scene has `shs` (P_scene, M, 3) instead of `colors`."""
        if which == "scene":
            out = {k: v[: self.Ps] for k, v in self.views_A.items() if k != "shs"}
            if self.M > 0:
                del out["colors"]
                out["shs"] = self.views_A["shs"]
            return out
        if which == "human":
            return {k: v[self.Ps:] for k, v in self.views_A.items() if k != "shs"}
        return dict(self.views_B)

    def flat_bucket(self) -> torch.Tensor:
        return self.all_flat

    def consumed(self) -> Dict[str, list]:
        fwd, bwd = [], []
        for pk, names in self.VIEWS.items():  # the views of a pass add into the same counters: per-launch averages
            s = self.passes[pk].status()
            fwd += [s["consumed_fwd"] / L.CONSUMED_FWD_DIV / len(names)] * len(names)
            bwd += [s["consumed_bwd"] / L.CONSUMED_BWD_DIV / len(names)] * len(names)
        return {"fwd": fwd, "bwd": bwd}
