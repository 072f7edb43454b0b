"""A trained avatar tested on the device: ExAvatar's test.py and tools/eval_neuman.py over every held-out frame, one
CUDA graph replay per frame.

test.py decodes each frame through a DataLoader, runs `Model.forward(mode='test')` eagerly, copies ten images to the
host one `.cpu()` at a time and writes them with `cv2.imwrite`; eval_neuman.py reads the PNGs back with the frame's
`images/%05d.png` and `segmentations/%05d.png` and reads each score back on the host.  `AvatarTester` runs the same
forward from the resident tables, every input read through one (1,) int32 device slot:

    frames = FrameTable.from_dataset(testset, "cuda", slots=table.frames)
    masks = SegmentationTable.from_folder(subject_root, frames, "cuda")          # eval's mask; None = --include_bkg
    tester = AvatarTester(frames, table, rig, tri, assets, normals, face_renderer, renderer, ..., scorer=neuman,
                          masks=masks)
    for frame_idx, png, scores in tester.frames():   # png (10,H,W,3) uint8 BGR in compose.PNG_ORDER; scores (3,)
        ... cv2.imwrite(f"{frame_idx}_{name}.png", png[k]) for the caller's names
    psnr, ssim, lpips = tester.summary()              # eval's printed means

Per frame the device runs the existing ops: `FrameTable` and `SmplxParamTable` reads, `SmplxRig`, `TriplaneFeatures`,
the four `gn_mlp` stacks, `HumanAssets.geometry(warmup=False)`, `nearest_rows`, `skin_gaussians` on both sets,
`VertexNormals` and the colours, `scene_assets` in rgb mode with the frame's camera, `device_render_settings`, the five
renders of `TrainingFrameRenderer` with bg_human = ones, the two `FaceMeshRenderer` calls, `test_outputs` and
`NeumanScores`.  Position 0 runs eagerly (the face renderer and the scorer allocate at this size there), position 1 is
captured, and every later frame is one replay with the slot filled in.

The parameters are read in place, not copied: the graph bakes in the tensors' addresses, so in-place updates (an
optimizer step) are seen by the next replay, and held-out frames can be scored between training iterations.  After
anything that replaces a tensor (densification, a new entry in the `scene` dict), call `invalidate()`: the next frame
captures again, the contract of `IterationGraph.invalidate()`.
"""
from __future__ import annotations

import ctypes as C
from collections import deque
from typing import Iterator, Optional, Tuple

import numpy as np
import torch

from . import _lib as L
from .compose import PNG_ORDER, test_outputs
from .geometry import nearest_rows
from .human_nets import gn_mlp
from .metrics import MIN_SIZE
from .renderer import device_render_settings
from .scene_assets import scene_assets
from .skinning import skin_gaussians

# the scene's raw parameters in scene_assets' argument order
SCENE_KEYS = ("mean", "opacity_logit", "log_scale", "rotation6d", "feature_dc", "feature_rest")
_STATUS_BYTES = C.sizeof(L.B2RStatus)
_PASSES = ("A", "B")  # the renderer's two projection + binning passes


class AvatarTester:
    """ExAvatar's test pass over every frame of a `FrameTable`, in its row order (test.py's `shuffle=False` order and
    eval's test_split.txt order).

    frames, params    the split's `FrameTable` and the `SmplxParamTable` whose slots it shares (`slots=params.frames`)
    rig, tri, assets, normals   `SmplxRig`, `TriplaneFeatures`, `HumanAssets`, `VertexNormals` of the avatar
    face_renderer     `FaceMeshRenderer(flame.vertex_uv, flame.face_uv, flame.face, flame.vertex_num)`
    renderer          a caller-built `TrainingFrameRenderer(P_scene, P_human, (H, W), ..., use_graph=False)`; its list
                      capacity is the pass's
    triplane, triplane_face          HumanGaussian.triplane / triplane_face
    geo_net, geo_offset_net, rgb_net, rgb_offset_net   the four stacks as (trunk, heads) for `gn_mlp`
    shape_param, joint_offset, skinning_weight, self_map   as `AvatarAnimator` takes them
    scene             {SCENE_KEYS: the scene's raw parameters}, as `scene_assets` takes them; the dict itself is kept,
                      and read at each eager frame and capture
    active_sh_degree  ExAvatar's (1,) float CUDA buffer
    face_uvmap        (1,4,Ht,Wt) cat(flame.texture, flame.texture_mask[0:1]); face_vertex_idx (Vf,) int64 CUDA
    scorer            `NeumanScores`, or None (Custom: no eval script, no scores)
    masks             `SegmentationTable` of `frames`, or None (eval's --include_bkg); needs a scorer
    png               also hand back test.py's ten images' bytes
    use_graph         position 0 eagerly, position 1 captured, every later position one replay
    in_flight         pinned host buffers in the ring `frames()` yields from (>= 1)

    Nothing is copied: the graph reads the tensors given here at their addresses (the module docstring)."""

    def __init__(self, frames, params, rig, tri, assets, normals, face_renderer, renderer, *, triplane, triplane_face,
                 geo_net, geo_offset_net, rgb_net, rgb_offset_net, shape_param, joint_offset, skinning_weight, self_map,
                 scene: dict, active_sh_degree, face_uvmap, face_vertex_idx, scorer=None, masks=None, png: bool = True,
                 use_graph: bool = True, in_flight: int = 2):
        fn = "AvatarTester"
        if isinstance(in_flight, bool) or not isinstance(in_flight, int) or in_flight < 1:
            raise ValueError(f"{fn}: in_flight must be an int >= 1, got {in_flight!r}")
        if list(params.frames) != list(frames.frames):
            raise ValueError(f"{fn}: the SMPL-X table's slots and the frame table's differ; build the frame table with "
                             "slots=params.frames")
        H, W = frames.height, frames.width
        if tuple(renderer.img_shape) != (H, W):
            raise ValueError(f"{fn}: the renderer renders {tuple(renderer.img_shape)}, the frames are {(H, W)}")
        if getattr(renderer, "use_graph", False):
            raise ValueError(f"{fn}: the renderer must be built with use_graph=False (the tester captures the frame)")
        if scorer is not None and (H < MIN_SIZE or W < MIN_SIZE):
            raise ValueError(f"{fn}: scored images must be at least {MIN_SIZE}x{MIN_SIZE}, the frames are {H}x{W}")
        if masks is not None:
            if scorer is None:
                raise ValueError(f"{fn}: `masks` paint the scored images' background; they need a `scorer`")
            if masks.frames is not frames:
                raise ValueError(f"{fn}: `masks` must be a SegmentationTable of this frame table")
        missing = [k for k in SCENE_KEYS if k not in scene]
        if missing:
            raise ValueError(f"{fn}: `scene` lacks {missing}")
        self.frames_table, self.params = frames, params
        self.rig, self.tri, self.assets, self.normals = rig, tri, assets, normals
        self.face_renderer, self.renderer = face_renderer, renderer
        self.triplane, self.triplane_face = triplane, triplane_face
        self.nets = {"geo": geo_net, "geo_offset": geo_offset_net, "rgb": rgb_net, "rgb_offset": rgb_offset_net}
        self.shape_param, self.joint_offset = shape_param, joint_offset
        self.skinning_weight, self.self_map = skinning_weight, self_map
        self.scene, self.active_sh_degree = scene, active_sh_degree
        self.face_uvmap, self.face_vertex_idx = face_uvmap, face_vertex_idx
        self.scorer, self.masks = scorer, masks
        self.png, self.use_graph, self.in_flight = bool(png), bool(use_graph), in_flight
        dev = self.device = frames.device
        # rows in table order, each read through its slot
        n = self.n_frames = frames.n_rows
        slot_of_row = [None] * n
        for s, r in enumerate(frames._row):
            if r >= 0 and slot_of_row[r] is None:
                slot_of_row[r] = s
        self.slots = slot_of_row
        self.frame_idx = [int(f) for f in frames.frame_idx.tolist()]
        self.image_shape = (H, W)
        self._ones = torch.ones(3, dtype=torch.float32, device=dev)
        self._slot = torch.zeros(1, dtype=torch.int32, device=dev)
        self._pos = torch.zeros(1, dtype=torch.int64, device=dev)
        self._scores = torch.full((n, 3), float("nan"), dtype=torch.float32, device=dev) \
            if scorer is not None else None
        self._ring = torch.empty((in_flight, len(PNG_ORDER), H, W, 3), dtype=torch.uint8, pin_memory=True) \
            if self.png else None
        self._ring_scores = torch.empty((in_flight, 3), dtype=torch.float32, pin_memory=True) \
            if scorer is not None else None
        self._ring_status = torch.empty((in_flight, len(_PASSES), _STATUS_BYTES), dtype=torch.uint8, pin_memory=True)
        self._events = [torch.cuda.Event() for _ in range(in_flight)]
        self._graph = None
        self._static = None
        self._ran = False

    @torch.no_grad()
    def _device_frame(self, slot: torch.Tensor) -> dict:
        """Model.forward(mode='test') of one frame on the device, every input read through `slot`; the frame's score
        row lands at `self._pos` of the score table."""
        data = self.frames_table(slot)
        gt = data["img"]
        cam = {k: v[0] for k, v in data["cam_param"].items()}
        sp = self.params(slot)
        trans = sp["trans"]
        out = self.rig(self.shape_param, self.joint_offset, sp["full_pose"], sp["expr"])
        f = self.tri(self.triplane, self.triplane_face)
        net = lambda k, ins: gn_mlp(ins, *self.nets[k])  # noqa: E731
        geo, geo_off, rgb = net("geo", [f]), net("geo_offset", [f, out.pose_6d]), net("rgb", [f])
        ga = self.assets.geometry(out.mesh_neutral_pose, out.pose_offset, out.expr_offset, geo, geo_off, warmup=False)
        rows = nearest_rows(ga["mean_3d"], out.mesh_neutral_pose_wo_upsample.contiguous(), self.self_map)
        posed, posed_r = skin_gaussians(ga["mean_3d"], ga["mean_3d_refined"], self.skinning_weight, rows,
                                        out.joint_mats, trans, cam["R"], cam["t"])
        rgb_c, rgb_r = self.assets.colors(rgb, net("rgb_offset", [f, out.pose_6d, self.normals(posed_r)]))
        ha = self.assets
        human = {"mean_3d": posed, "opacity": ha.opacity, "scale": ga["scale"], "rotation": ha.rotation, "rgb": rgb_c}
        refined = {"mean_3d": posed_r, "opacity": ha.opacity, "scale": ga["scale_refined"], "rotation": ha.rotation,
                   "rgb": rgb_r}
        scene = scene_assets(*(self.scene[k] for k in SCENE_KEYS), self.active_sh_degree, cam)
        settings = device_render_settings(self.image_shape, cam, self._ones)
        renders = self.renderer(scene, human, refined, cam, self._ones, raster_settings=settings)
        face = self.face_renderer(self.face_uvmap, posed[self.face_vertex_idx][None], cam, self.image_shape)
        face_r = self.face_renderer(self.face_uvmap, posed_r[self.face_vertex_idx][None], cam, self.image_shape)
        res = test_outputs(renders, face, face_r, gt=gt, png=self.png)
        res["gt"] = gt
        if self.scorer is not None:
            mask = self.masks(slot) if self.masks is not None else None
            res["scores"] = self.scorer(res["scene_human_img_refined_composed"], gt, mask)
            self._scores.index_copy_(0, self._pos, res["scores"])
        return res

    def _fill(self, i: int) -> None:
        self._slot.fill_(self.slots[i])
        self._pos.fill_(i)

    def _eager(self, i: int) -> dict:
        self._fill(i)
        out = self._device_frame(self._slot)
        self._ran = True
        return out

    def frame(self, i: int) -> dict:
        """Position i of the pass, eagerly: Model.forward(mode='test')'s nine images (compose.RENDER_KEYS and
        COMPOSITE_KEYS, (1,3,H,W) fp32), "gt", "png" (10,1,H,W,3) uint8 with `png`, and "scores" (1,3) with a scorer,
        on the device; the score also lands in row i of `scores()`."""
        if not 0 <= int(i) < self.n_frames:
            raise IndexError(f"AvatarTester: position {i} outside [0, {self.n_frames})")
        return self._eager(int(i))

    def invalidate(self) -> None:
        """Drops the captured frame: call it after anything replaces a tensor the tester reads (densification, a new
        entry in `scene`); the next frame captures again.  In-place updates need no call."""
        self._graph = None
        self._static = None

    def _submit(self, i: int, k: int) -> None:
        if not self.use_graph or not self._ran:
            out = self._eager(i)
        else:
            if self._graph is None:
                self._fill(i)
                self._graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self._graph):
                    self._static = self._device_frame(self._slot)
            self._fill(i)
            self._graph.replay()
            out = self._static
        if self.png:
            self._ring[k].copy_(out["png"][:, 0], non_blocking=True)
        if self.scorer is not None:
            self._ring_scores[k].copy_(out["scores"][0], non_blocking=True)
        for j, pk in enumerate(_PASSES):
            self._ring_status[k, j].copy_(self.renderer.plan.passes[pk].ctx_buf[:_STATUS_BYTES], non_blocking=True)
        self._events[k].record()

    def _collect(self, i: int, k: int):
        self._events[k].synchronize()
        for j, pk in enumerate(_PASSES):
            st = L.B2RStatus.from_buffer_copy(self._ring_status[k, j].numpy().tobytes())
            if st.overflow:
                raise RuntimeError(f"AvatarTester: frame {self.frame_idx[i]} (position {i}) needed {st.num_dups} "
                                   f"render list entries in pass {pk}, the capacity is {st.dup_capacity}; its renders "
                                   "are truncated (build the TrainingFrameRenderer with a larger dup_capacity)")
        png = self._ring[k].numpy() if self.png else None
        scores = self._ring_scores[k].numpy() if self.scorer is not None else None
        return self.frame_idx[i], png, scores

    def frames(self) -> Iterator[Tuple[int, Optional[np.ndarray], Optional[np.ndarray]]]:
        """(frame_idx, png, scores) for every frame in table row order.  png is the (10,H,W,3) uint8 BGR bytes of
        test.py's ten writes in compose.PNG_ORDER, scores the frame's (3,) psnr / ssim / lpips; each is a view of one
        of `in_flight` pinned buffers (None without `png` / a scorer).  The buffers stay the caller's until the next
        iteration; up to `in_flight` frames are queued on the device meanwhile.  A frame whose render lists overflowed
        the renderer's capacity raises RuntimeError naming it when it is collected."""
        n = self.in_flight
        pending = deque()
        for i in range(self.n_frames):
            if len(pending) == n:
                yield self._collect(*pending.popleft())
            k = i % n
            self._submit(i, k)
            pending.append((i, k))
        while pending:
            yield self._collect(*pending.popleft())

    def scores(self) -> torch.Tensor:
        """The (n,3) fp32 device table of psnr / ssim / lpips, row i the frame at position i of the last pass (NaN
        before a frame is scored)."""
        if self._scores is None:
            raise RuntimeError("AvatarTester: built without a scorer")
        return self._scores

    def summary(self) -> torch.Tensor:
        """eval_neuman's printed means as a (3,) fp32 device tensor: the rows of `scores()` summed in fp64 in pass
        order, divided by n and rounded to fp32 once.  A frame with psnr = +inf gives a mean of +inf, as eval's."""
        s = self.scores().double()
        acc = s[0].clone()
        for i in range(1, self.n_frames):
            acc += s[i]
        return (acc / self.n_frames).float()
