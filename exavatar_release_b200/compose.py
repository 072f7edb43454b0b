"""ExAvatar's image composites as sync-free CUDA ops (csrc/compose.cu): the face composite in front of the rgb_face
terms, and the test-time outputs with the bytes test.py writes.

Training (avatar/main/model.py:200-201, 207-208) composites the face render over each combined render before the L1:

    is_face = ((face[:,:3] != -1) * (face[:,3:] == 1)).float()
    scene_human * (1 - is_face) + face[:,:3] * is_face

`face_composite(img, face)` is that expression as one autograd op, one launch forward and one backward.

Testing (model.py:268-276, main/test.py:40-64) composites four images and test.py copies ten images to the host one by
one, each `.cpu()` a host sync, to write them with `cv2.imwrite(x.transpose(1,2,0)[:,:,::-1]*255)`.
`test_outputs(renders, face, face_refined, gt)` computes the four composites and, with `png=True`, the ten images'
bytes as one uint8 (10,N,H,W,3) BGR tensor, in one launch:

    with torch.no_grad():
        renders = frame(scene_asset, human_asset, human_asset_refined, cam_param, bg_human=torch.ones(3))
        out = test_outputs(renders, face_render, face_render_refined, gt)
    host = torch.empty(out["png"].shape, dtype=torch.uint8, pin_memory=True)
    host.copy_(out["png"], non_blocking=True)                      # the frame's one device-to-host copy
    scores = neuman(out["scene_human_img_refined_composed"], gt)   # NeumanScores, on the device

`face_composite_reference` and `test_outputs_reference` restate the semantics in torch fp32 and numpy; the tests
compare the ops with them and the ops never call them.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib as L
from .plan import RENDERS

# Model.forward(mode='test')'s image keys, then test.py's write order of the ten images (the renders of plan.RENDERS,
# the four composites, gt)
RENDER_KEYS = ("scene_img", "human_img", "scene_human_img", "human_img_refined", "scene_human_img_refined")
COMPOSITE_KEYS = ("human_face_img", "human_face_img_refined", "scene_human_img_composed",
                  "scene_human_img_refined_composed")
PNG_ORDER = RENDER_KEYS + COMPOSITE_KEYS + ("gt",)


def _frames(fn: str, name: str, t: torch.Tensor, C_: int, shape=None) -> torch.Tensor:
    """`t` ((C,H,W) or (N,C,H,W), fp32 CUDA) as a contiguous (N,C,H,W) tensor, checked against `shape` (N,H,W)."""
    L.cuda(fn, name, t)
    L.float32(fn, name, t)
    if t.dim() not in (3, 4) or t.shape[-3] != C_:
        raise ValueError(f"{fn}: `{name}` must be ({C_},H,W) or (N,{C_},H,W), got {tuple(t.shape)}")
    t = t.reshape(-1, C_, t.shape[-2], t.shape[-1])
    if shape is not None and (t.shape[0], t.shape[2], t.shape[3]) != shape:
        raise ValueError(f"{fn}: `{name}` {tuple(t.shape)} does not match the frames' (N,H,W) = {shape}")
    if t.shape[0] == 0 or t.shape[2] == 0 or t.shape[3] == 0:
        raise ValueError(f"{fn}: `{name}` is empty: {tuple(t.shape)}")
    return t.detach().contiguous()


class _FaceComposite(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, face):
        img, face = img.detach().contiguous(), face.detach().contiguous()
        N, _, H, W = img.shape
        p = L.B2RFaceComposite(width=W, height=H, n_images=N, img=L.ptr(img), face=L.ptr(face))
        out = torch.empty((N, 3, H, W), dtype=torch.float32, device=img.device)
        L.run("b2r_face_composite_forward", img.device, C.byref(p), L.ptr(out))
        ctx.save_for_backward(face)
        return out

    @staticmethod
    def backward(ctx, dout):
        face, = ctx.saved_tensors
        want_img, want_face = ctx.needs_input_grad[:2]
        if not (want_img or want_face):
            return None, None
        N, _, H, W = face.shape
        g = dout.to(torch.float32).contiguous()
        dimg = torch.empty((N, 3, H, W), dtype=torch.float32, device=face.device) if want_img else None
        dface = torch.empty((N, 4, H, W), dtype=torch.float32, device=face.device) if want_face else None
        p = L.B2RFaceComposite(width=W, height=H, n_images=N, face=L.ptr(face))
        L.run("b2r_face_composite_backward", face.device, C.byref(p), L.ptr(g), L.ptr(dimg), L.ptr(dface))
        return dimg, dface


def face_composite(img: torch.Tensor, face: torch.Tensor) -> torch.Tensor:
    """ExAvatar's rgb_face composite: `img * (1 - is_face) + face[:,:3] * is_face` with
    `is_face = ((face[:,:3] != -1) * (face[:,3:] == 1)).float()`, per channel, as one differentiable CUDA op.

    img   (3,H,W) or (N,3,H,W) fp32 CUDA tensor: the combined render (scene_human or scene_human_refined)
    face  (4,H,W) or (N,4,H,W) fp32 CUDA tensor: FaceMeshRenderer's output, -1 where no face

    Returns (N,3,H,W) fp32, bit-identical to torch's fp32 expression.  Its gradients are torch autograd's:
    dL/dimg = g (1 - is_face), dL/dface = g is_face in channels 0-2 and zero in channel 3.  Forward and backward are
    one launch each, read nothing back on the host and can be captured in a CUDA graph; there is no CPU fallback.
    """
    x = _frames("face_composite", "img", img, 3)
    f = _frames("face_composite", "face", face, 4, (x.shape[0], x.shape[2], x.shape[3]))
    L.same_device("face_composite", (x, f))
    return _FaceComposite.apply(img.reshape(x.shape), face.reshape(f.shape))


def test_outputs(renders: Dict[str, Dict[str, torch.Tensor]], face: torch.Tensor, face_refined: torch.Tensor,
                 gt: Optional[torch.Tensor] = None, png: bool = True) -> Dict[str, torch.Tensor]:
    """The image outputs of ExAvatar's `Model.forward(mode='test')` and, with `png`, the bytes of test.py's writes.

    renders       TrainingFrameRenderer's output (or any {name: {"img", "mask"}} of plan.RENDERS), rendered under
                  torch.no_grad() with bg_human = ones as the test pass renders: "img" (3,H,W) or (N,3,H,W), and
                  "mask" (1,H,W) or (N,1,H,W) of "human" and "human_refined", fp32 CUDA
    face          FaceMeshRenderer's (N,4,H,W) output for the human, -1 where no face; `face_refined` the refined one
    gt            (N,3,H,W) fp32 ground truth, or None
    png           also return "png": uint8 (K,N,H,W,3), K = 10 with gt and 9 without, in test.py's write order
                  (PNG_ORDER): each image's bytes as `cv2.imwrite(x.transpose(1,2,0)[:,:,::-1] * 255)` stores them,
                  BGR, with cv2's float-to-uint8 conversion (rint with ties to even, NaN and |v| >= 2^31 to 0)

    Returns the renders as (N,3,H,W) views under RENDER_KEYS, the four composites (fresh (N,3,H,W) fp32 tensors,
    bit-identical to model.py's expressions) under COMPOSITE_KEYS, and "png".  One launch; nothing is read back on the
    host, so the caller moves "png" with one non-blocking copy into pinned memory.  Forward only: raises if grad mode
    is on and an input requires grad.
    """
    fn = "test_outputs"
    for r in RENDERS:
        if r not in renders or "img" not in renders[r]:
            raise ValueError(f"{fn}: renders[{r!r}]['img'] is missing")
    for r in ("human", "human_refined"):
        if "mask" not in renders[r]:
            raise ValueError(f"{fn}: renders[{r!r}]['mask'] is missing")
    inputs = [renders[r]["img"] for r in RENDERS] + [renders["human"]["mask"], renders["human_refined"]["mask"], face,
                                                      face_refined, gt]
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in inputs):
        raise RuntimeError(f"{fn}: forward only; call it under torch.no_grad() (an input requires grad)")
    imgs = [_frames(fn, f"renders[{r!r}]['img']", renders[r]["img"], 3) for r in RENDERS]
    N, _, H, W = imgs[0].shape
    shape = (N, H, W)
    imgs = [_frames(fn, f"renders[{r!r}]['img']", t, 3, shape) for r, t in zip(RENDERS, imgs)]
    masks = [_frames(fn, f"renders[{r!r}]['mask']", renders[r]["mask"], 1, shape) for r in ("human", "human_refined")]
    faces = [_frames(fn, n, t, 4, shape) for n, t in (("face", face), ("face_refined", face_refined))]
    g = None if gt is None else _frames(fn, "gt", gt, 3, shape)
    dev = imgs[0].device
    L.same_device(fn, (*imgs, *masks, *faces, g))
    p = L.B2RTestOutputs(width=W, height=H, n_images=N, gt=L.ptr(g))
    for i, t in enumerate(imgs):
        p.render[i] = L.ptr(t)
    for k in range(2):
        p.mask[k], p.face[k] = L.ptr(masks[k]), L.ptr(faces[k])
    comp = [torch.empty((N, 3, H, W), dtype=torch.float32, device=dev) for _ in COMPOSITE_KEYS]
    out_png = torch.empty((10 if g is not None else 9, N, H, W, 3), dtype=torch.uint8, device=dev) if png else None
    ptrs = (L._fp * 4)(*(L.ptr(t) for t in comp))
    L.run("b2r_test_outputs", dev, C.byref(p), ptrs, L.ptr(out_png))
    out = dict(zip(RENDER_KEYS, imgs))
    out.update(zip(COMPOSITE_KEYS, comp))
    if png:
        out["png"] = out_png
    return out


# ---------------------------------------------------------------------------------------------------------------------
# References (tests and measurements; the ops never call them)
# ---------------------------------------------------------------------------------------------------------------------

def face_composite_reference(img: torch.Tensor, face: torch.Tensor) -> torch.Tensor:
    """model.py:200-201's expression in torch fp32, differentiable, on any device; (N,3,H,W)."""
    H, W = img.shape[-2:]
    img = img.reshape(-1, 3, H, W)
    face = face.reshape(-1, 4, H, W)
    is_face = ((face[:, :3] != -1) * (face[:, 3:] == 1)).float()
    return img * (1 - is_face) + face[:, :3] * is_face


def png_bytes(x: np.ndarray) -> np.ndarray:
    """The bytes `cv2.imwrite(path, x.transpose(1,2,0)[:,:,::-1] * 255)` stores for a float32 (3,H,W) or (N,3,H,W)
    array, as uint8 (H,W,3) / (N,H,W,3) BGR: v = float32(x * 255), then cv2's saturate_cast -- 0 where v is NaN or
    |v| >= 2^31, else rint(v) (ties to even) clamped to [0, 255]."""
    x = np.asarray(x, dtype=np.float32)
    v = np.moveaxis(x, -3, -1)[..., ::-1] * np.float32(255)
    with np.errstate(invalid="ignore"):
        bad = np.isnan(v) | (np.abs(v) >= np.float32(2.0 ** 31))
        r = np.clip(np.rint(np.where(bad, np.float32(0), v)), 0, 255)
    return r.astype(np.uint8)


@torch.no_grad()
def test_outputs_reference(renders: Dict[str, Dict[str, torch.Tensor]], face: torch.Tensor,
                           face_refined: torch.Tensor, gt: Optional[torch.Tensor] = None, png: bool = True) -> dict:
    """`test_outputs` restated: model.py:268-276's expressions in torch fp32 on the inputs' device, and test.py's bytes
    by `png_bytes` in numpy (a host copy; "png" is a numpy (K,N,H,W,3) uint8 array)."""
    H, W = renders["scene"]["img"].shape[-2:]
    img = {r: renders[r]["img"].reshape(-1, 3, H, W) for r in RENDERS}
    face = face.reshape(-1, 4, H, W)
    face_refined = face_refined.reshape(-1, 4, H, W)
    out = dict(zip(RENDER_KEYS, (img[r] for r in RENDERS)))
    is_face = (face[:, :3] != -1).float() * face[:, 3:]
    out["human_face_img"] = img["human"] * (1 - is_face) + face[:, :3] * is_face
    is_face = (face_refined[:, :3] != -1).float() * face_refined[:, 3:]
    out["human_face_img_refined"] = img["human_refined"] * (1 - is_face) + face_refined[:, :3] * is_face
    is_fg = renders["human"]["mask"].reshape(-1, 1, H, W) > 0.9
    out["scene_human_img_composed"] = is_fg * img["human"] + (1 - is_fg.float()) * img["scene_human"]
    is_fg = renders["human_refined"]["mask"].reshape(-1, 1, H, W) > 0.9
    out["scene_human_img_refined_composed"] = (is_fg * img["human_refined"] +
                                               (1 - is_fg.float()) * img["scene_human_refined"])
    if png:
        imgs = [out[k] for k in RENDER_KEYS + COMPOSITE_KEYS] + ([] if gt is None else [gt.reshape(-1, 3, H, W)])
        out["png"] = np.stack([png_bytes(t.cpu().numpy()) for t in imgs])
    return out
