"""`TrainingFrameRenderer`: ExAvatar's five renders of a training frame as ONE autograd call (SURVEY.md section 8f-3).

`Model.forward` renders every frame five times with the same camera (avatar/main/model.py:117-162):

    scene_render                = gaussian_renderer(scene_asset, ...)
    human_render                = gaussian_renderer(human_asset, ..., bg)
    scene_human_render          = gaussian_renderer(cat(scene_asset.detach(), human_asset), ...)
    human_render_refined        = gaussian_renderer(human_asset_refined, ..., bg)
    scene_human_render_refined  = gaussian_renderer(cat(scene_asset.detach(), human_asset_refined), ...)

Through the drop-in `GaussianRasterizer` those are five full projection / binning / sort / composite pipelines.  This
module renders the same five images from TWO projection + binning passes (`plan.MergedFivePlan`: views of
cat(scene, human) and cat(scene, human_refined), human-free tiles of the human-only and combined views skipped) and
back-propagates into the three asset dicts exactly what `loss.backward()` leaves there: the scene render's gradient in the
scene assets, human-only + combined render in the human assets (the scene part of the combined renders is detached, as in
the reference), likewise for the refined set.  INTEGRATION.md shows the replacement of model.py:117-162.

    frame = TrainingFrameRenderer(P_scene, P_human, (H, W), device, dup_capacity)
    out = frame(scene_asset, human_asset, human_asset_refined, cam_param, bg_human)
    out["scene"]["img"], out["human"]["mask"], out["scene_human"]["img"], ...      # same keys as GaussianRenderer
    out["scene"]["mean_2d"].grad                                                   # after backward (train.py:51)

The duplicate capacity is fixed per instance (every buffer is resident; nothing is polled or synchronised, so the call
is capturable in a CUDA graph); `overflowed()` reports if a frame needed more (its lists were truncated, never corrupt).
One frame may be in flight per instance: run backward (or drop the outputs) before the next call.

`use_graph=True`: the first frame captures the forward and the backward of the plan into two CUDA graphs; later frames
copy their inputs into the plan's resident buffers (assets, camera, dL/dimage) and replay.  The Python cost of a frame
drops from ~2.9 ms (hundreds of stream switches, ctypes calls and small copies) to a few copies and two graph launches,
so an otherwise EAGER training loop runs the raster part at graph speed.  Kernel arguments passed by value are frozen in
the graphs: with float settings (`render_settings`) a change of the intrinsics (tan fov) re-captures.  Settings from
`renderer.device_render_settings` carry tan(fov) on the device; it is copied into the resident block with the matrices
and the graphs read it from there, so one capture per SH degree serves every camera.  Every render's backward runs (a
render left out of the loss contributes zeros).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
from torch import nn

from .plan import ASSETS, RENDERS, MergedFivePlan
from .rasterizer import GaussianRasterizationSettings, _f32c, device_tanfov
from .renderer import render_settings

_KEYS = tuple(ASSETS)
_SH_KEYS = tuple(k for k in ASSETS if k != "rgb") + ("shs",)  # a scene coloured from SH inside the kernels
_GRAD_OF = {k: g for k, (g, _) in ASSETS.items()}


class _FrameFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mod, settings, settings_h, sh_degree, scene_m2d, *tensors):
        plan: MergedFivePlan = mod.plan
        scene, human, refined = (dict(zip(keys, (_f32c(t.detach(), k) for k, t in zip(keys, tensors[i * 5:i * 5 + 5]))))
                                 for i, keys in enumerate((mod._scene_keys, _KEYS, _KEYS)))
        if plan.M > 0:
            scene["sh_degree"] = sh_degree
        mod._frame_no += 1
        plan.set_scene(scene)  # an SH scene: both passes read the caller's coefficient tensor itself (eager)
        if mod.use_graph:
            mod._graph_forward(settings, settings_h, scene, human, refined)
        else:
            plan.forward_frame(None, settings, settings_h, scene, human, refined)  # no descriptor cache: cameras change
        # fresh tensors: the plan's buffers are overwritten by the next frame
        outs = [t.clone() for r in RENDERS for t in plan.image(r)]
        # the radii of a combined render are those of every row of its pass
        radii_a, radii_b = (plan.render_outputs(r)[2].clone() for r in ("scene_human", "scene_human_refined"))
        ctx.mod = mod
        ctx.shapes = [t.shape for t in tensors]
        ctx.m2d_shape = scene_m2d.shape
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(radii_a, radii_b)
        return (*outs, radii_a, radii_b)

    @staticmethod
    def backward(ctx, *grads):
        mod = ctx.mod
        plan: MergedFivePlan = mod.plan
        g = grads[:15]
        gc = {r: (None if g[3 * i] is None else _f32c(g[3 * i], "grad_color")) for i, r in enumerate(RENDERS)}
        gd = {r: (None if g[3 * i + 1] is None else _f32c(g[3 * i + 1], "grad_depth")) for i, r in enumerate(RENDERS)}
        ga = {r: (None if g[3 * i + 2] is None else _f32c(g[3 * i + 2], "grad_alpha")) for i, r in enumerate(RENDERS)}
        if mod.use_graph:  # views of fresh copies of the resident gradient buffers
            _, (va, vb) = plan.grad_buffers(mod._graph_backward(gc, gd, ga))
        else:
            _, (va, vb) = plan.grad_buffers()
            plan.backward_frame(gc, va, vb, g_depths=gd, g_alphas=ga, densify=mod.densify)
        Ps = plan.Ps
        out = [None, None, None, None, va["means2D"][:Ps].reshape(ctx.m2d_shape)]
        for k in mod._scene_keys:
            out.append(va["shs"] if k == "shs" else va[_GRAD_OF[k]][:Ps])
        for k in _KEYS:
            out.append(va[_GRAD_OF[k]][Ps:])
        for k in _KEYS:
            out.append(vb[_GRAD_OF[k]])
        for i, shp in enumerate(ctx.shapes):
            out[5 + i] = out[5 + i].reshape(shp)
        return tuple(out)


class TrainingFrameRenderer(nn.Module):
    """sh_coeffs = M > 0: the scene asset dict carries `shs` (P_scene, M, 3) + `sh_degree` instead of `rgb` -- what
    `renderer.scene_gaussian_assets(..., in_kernel_sh=True)` returns -- and the scene is coloured inside the projection
    kernels of both merged passes (SURVEY.md section 8f-4); its gradient reaches `shs` and, through the view direction,
    `mean_3d`.  The human sets keep `rgb`."""

    def __init__(self, P_scene: int, P_human: int, img_shape, device, dup_capacity: Optional[Dict[str, int]] = None,
                 use_graph: bool = False, graph_depth_alpha: bool = False, sh_coeffs: int = 0):
        super().__init__()
        self.img_shape = (int(img_shape[0]), int(img_shape[1]))
        self.plan = MergedFivePlan(P_scene, P_human, self.img_shape[1], self.img_shape[0], dup_capacity, device,
                                   sh_coeffs=sh_coeffs)
        self._scene_keys = _SH_KEYS if self.plan.M > 0 else _KEYS
        self.densify = None  # optional {'grad_accum','count','radius_max'} (P_scene) tensors updated by the backward
        self._frame_no = 0
        self.use_graph = bool(use_graph)
        if self.use_graph:
            dev, (H, W) = self.plan.device, self.img_shape
            # resident camera / background block the captured kernels read: view (16) | full projection (16) | campos (3) |
            # bg (3) | bg of the human-only renders (3) | tan(fov_x/2), tan(fov_y/2) of device settings (2)
            self._cam = torch.zeros(43, dtype=torch.float32, device=dev)
            self._gin = {r: torch.zeros(3, H, W, dtype=torch.float32, device=dev) for r in RENDERS}
            # dL/ddepth and dL/dalpha inputs only when asked for: their backward variant is the slower one
            self._gin_d = {r: torch.zeros(1, H, W, dtype=torch.float32, device=dev) for r in RENDERS} if graph_depth_alpha else None
            self._gin_a = {r: torch.zeros(1, H, W, dtype=torch.float32, device=dev) for r in RENDERS} if graph_depth_alpha else None
            # resident gradient buffers the captured backward writes, and their views
            self._flats, self._grad_views = self.plan.grad_buffers()
            # (tanfovx, tanfovy or "device", scale_modifier, densify buffers, sh_degree) -> (settings, settings_h,
            # forward graph, backward graph)
            self._graphs = {}
            self._cur = None

    # ---- use_graph=True ----
    def _resident_settings(self, settings, settings_h):
        c = self._cam
        # device settings: the captured kernels read tan(fov) from the resident block, floats stay kernel arguments
        tx, ty = (settings.tanfovx, settings.tanfovy) if device_tanfov(settings) is None else (c[41], c[42])
        mk = lambda bg: GaussianRasterizationSettings(
            image_height=settings.image_height, image_width=settings.image_width, tanfovx=tx, tanfovy=ty, bg=bg,
            scale_modifier=settings.scale_modifier, viewmatrix=c[0:16].view(4, 4), projmatrix=c[16:32].view(4, 4),
            sh_degree=0, campos=c[32:35], prefiltered=False, debug=False)
        return mk(c[35:38]), mk(c[38:41])

    def _load_inputs(self, settings, settings_h, scene, human, refined):
        plan, c = self.plan, self._cam
        c[0:16].copy_(settings.viewmatrix.reshape(16))
        c[16:32].copy_(settings.projmatrix.reshape(16))
        c[32:35].copy_(settings.campos.reshape(3))
        c[35:38].copy_(settings.bg.reshape(3))
        c[38:41].copy_(settings_h.bg.reshape(3))
        tanfov = device_tanfov(settings)
        if tanfov is not None:
            c[41:43].copy_(tanfov)
        plan.load_rows(human, refined)  # set_scene already copied the scene rows into both passes
        if plan.M > 0:  # the captured kernels read the coefficients at a fixed address
            plan.use_scene_shs(scene["shs"], scene["sh_degree"], copy=True)

    def _graph_forward(self, settings, settings_h, scene, human, refined):
        plan = self.plan
        self._load_inputs(settings, settings_h, scene, human, refined)
        dn = self.densify or {}
        # the SH degree is a kernel argument frozen in the graphs: ExAvatar raises it on a schedule (module.py:152-153),
        # so each degree is captured once and replayed afterwards
        fov = ("device",) if device_tanfov(settings) is not None else (float(settings.tanfovx), float(settings.tanfovy))
        key = (*fov, float(settings.scale_modifier),
               tuple(0 if dn.get(k) is None else dn[k].data_ptr() for k in ("grad_accum", "count", "radius_max")),
               plan.sh_degree if plan.M > 0 else None)
        if key not in self._graphs:
            st, st_h = self._resident_settings(settings, settings_h)
            va, vb = self._grad_views

            def fwd():
                plan.forward_frame(("graph", key), st, st_h, None, None, None, copy_inputs=False)

            def bwd(densify):
                plan.backward_frame(self._gin, va, vb, g_depths=self._gin_d, g_alphas=self._gin_a, densify=densify)

            cur = torch.cuda.current_stream(plan.device)
            side = torch.cuda.Stream(plan.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):  # warm-up (also primes the ctx counters), then capture
                fwd()
                # no densification bookkeeping in the warm-up: it would count a frame that is not one (with the
                # previous frame's dL/dimage still in the resident inputs) every time a new key is captured
                bwd(None)
            cur.wait_stream(side)
            torch.cuda.synchronize(plan.device)
            gf, gb = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(gf):
                fwd()
            with torch.cuda.graph(gb, pool=gf.pool()):
                bwd(self.densify)
            self._graphs[key] = (st, st_h, gf, gb)
        self._cur = self._graphs[key]
        self._cur[2].replay()

    def _graph_backward(self, gc, gd, ga):
        for dst, src in ((self._gin, gc), (self._gin_d, gd), (self._gin_a, ga)):
            if dst is None:
                if any(v is not None for v in src.values()):
                    raise RuntimeError("TrainingFrameRenderer(use_graph=True): gradients of depthmap / mask need "
                                       "graph_depth_alpha=True")
                continue
            for r in RENDERS:
                if src[r] is None:
                    dst[r].zero_()
                else:
                    dst[r].copy_(src[r].reshape(dst[r].shape))
        self._cur[3].replay()
        return tuple(f.clone() for f in self._flats)

    def overflowed(self) -> bool:
        return self.plan.overflowed()

    def forward(self, scene_asset, human_asset, human_asset_refined, cam_param, bg_human, bg=None, raster_settings=None,
                raster_settings_human=None):
        """Asset dicts as `GaussianRenderer.forward` takes them (mean_3d, opacity, scale, rotation, rgb; the scene asset
        carries shs + sh_degree instead of rgb when the renderer was built with sh_coeffs > 0); `bg_human` is the
        background of the two human-only renders (model.py:72), `bg` of the others (white by default, module.py:592).
        `raster_settings` (default `render_settings(cam_param)`) may come from `renderer.device_render_settings`: the
        frame then runs from camera to loss without a device->host read.
        Returns {render name: {img, depthmap, mask, radius, is_vis[, mean_2d]}} for the five renders of plan.RENDERS."""
        sh_scene = "shs" in scene_asset and "rgb" not in scene_asset
        if sh_scene != (self.plan.M > 0):
            raise ValueError("TrainingFrameRenderer: " + (
                "the scene asset carries `shs`: build the renderer with sh_coeffs=M" if sh_scene else
                f"built with sh_coeffs={self.plan.M}: the scene asset must carry `shs` + `sh_degree` instead of `rgb`"))
        dev = scene_asset["mean_3d"].device
        if bg is None:
            bg = torch.ones(3, dtype=torch.float32, device=dev)
        st = raster_settings or render_settings(self.img_shape, cam_param, bg, GaussianRasterizationSettings)
        st_h = raster_settings_human or st._replace(bg=bg_human)
        Ps = scene_asset["mean_3d"].shape[0]
        mean_2d = torch.zeros((Ps, 3), dtype=torch.float32, device=dev, requires_grad=True)  # module.py:626-629
        flat = [scene_asset[k] for k in self._scene_keys] + [a[k] for a in (human_asset, human_asset_refined) for k in _KEYS]
        sh_degree = int(scene_asset["sh_degree"]) if sh_scene else 0
        res = _FrameFn.apply(self, st, st_h, sh_degree, mean_2d, *flat)
        radii_a, radii_b = res[15], res[16]
        radius = {"scene": radii_a[:Ps], "human": radii_a[Ps:], "scene_human": radii_a, "human_refined": radii_b[Ps:],
                  "scene_human_refined": radii_b}
        out = {}
        for i, r in enumerate(RENDERS):
            out[r] = {"img": res[3 * i], "depthmap": res[3 * i + 1], "mask": res[3 * i + 2], "radius": radius[r],
                      "is_vis": radius[r] > 0}
        out["scene"]["mean_2d"] = mean_2d
        return out
