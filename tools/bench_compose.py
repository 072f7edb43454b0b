"""ExAvatar's image composites the way model.py and test.py compute them vs. `compose.test_outputs` and
`compose.face_composite`.

  python tools/bench_compose.py [--iters 10] [--rounds 5] [--encode-iters 2] [--json out.json]

Test arm, one frame (N = 1) at 512 x 512 and at 1080 x 1920, from the five renders, two masks, two face renders and gt
in device memory to the ten uint8 BGR images on the host:
  1. exavatar:  model.py:268-276's four composites in torch, then test.py's ten `.cpu().numpy()` (a host sync each),
                `transpose(1,2,0)[:,:,::-1] * 255` and cv2's float-to-uint8 conversion (saturate_cast, what
                cv2.imwrite's convertTo does; cv2.add with dtype=CV_8U runs the same conversion without encoding);
  2. op:        `test_outputs` and one non-blocking copy of its (10,1,H,W,3) bytes into pinned memory, then a sync.
  Both again with `cv2.imencode('.png', ...)` of the ten images (exavatar_png, op_png), so the PNG compression neither
  touches is visible next to the part that changes.
Train arm, the rgb_face pair at C4 size (512 x 512): forward and backward of the two face composites of model.py:200-201
and 207-208 (torch's expression vs. `face_composite`), eager and captured in a CUDA graph.
Arms alternate window by window in one process (host clock around the calls + device sync): median (min-max) ms.
The op's device time comes from CUDA events around 50 back-to-back calls, and its share of the HBM3 data-sheet
bandwidth (3.35 TB/s) from the bytes it must read and write.
Prints the card name and power limit with the numbers.
"""
import os
import sys

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, graph_replay, host_syncs, stats  # noqa: E402
from exavatar_release_b200 import _lib as L  # noqa: E402
from exavatar_release_b200.compose import (COMPOSITE_KEYS, RENDER_KEYS, face_composite,  # noqa: E402
                                           face_composite_reference, test_outputs)
from exavatar_release_b200.plan import RENDERS  # noqa: E402

SIZES = ((512, 512), (1080, 1920))


def frame_inputs(dev, H, W, seed):
    """Renders in [0,1], soft masks, face renders with -1 off the face (a face box over a sixth of the image), gt."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, device=dev, generator=g)  # noqa: E731
    renders = {r: {"img": rnd(1, 3, H, W)} for r in RENDERS}
    for r in ("human", "human_refined"):
        renders[r]["mask"] = rnd(1, 1, H, W)
    faces = []
    for _ in range(2):
        f = torch.full((1, 4, H, W), -1.0, device=dev)
        f[:, :, H // 4:H // 2, W // 3:2 * W // 3] = rnd(1, 4, H // 2 - H // 4, 2 * W // 3 - W // 3)
        f[:, 3:][f[:, 3:] > 0.2] = 1.0
        faces.append(f)
    return renders, faces[0], faces[1], rnd(1, 3, H, W)


def exavatar_test(renders, face, face_r, gt, encode):
    """model.py:268-276 in torch, then test.py's host copies and conversions (or PNG encodes) of the ten images."""
    h, hr = renders["human"], renders["human_refined"]
    out = {k: renders[r]["img"] for k, r in zip(RENDER_KEYS, RENDERS)}
    is_face = (face[:, :3] != -1).float() * face[:, 3:]
    out["human_face_img"] = h["img"] * (1 - is_face) + face[:, :3] * is_face
    is_face = (face_r[:, :3] != -1).float() * face_r[:, 3:]
    out["human_face_img_refined"] = hr["img"] * (1 - is_face) + face_r[:, :3] * is_face
    is_fg = h["mask"] > 0.9
    out["scene_human_img_composed"] = is_fg * h["img"] + (1 - is_fg.float()) * renders["scene_human"]["img"]
    is_fg = hr["mask"] > 0.9
    out["scene_human_img_refined_composed"] = is_fg * hr["img"] + (1 - is_fg.float()) * \
        renders["scene_human_refined"]["img"]
    host = [out[k].cpu().numpy() for k in RENDER_KEYS + COMPOSITE_KEYS] + [gt.cpu().numpy()]
    res = []
    for x in host:
        v = x[0].transpose(1, 2, 0)[:, :, ::-1] * 255
        res.append(cv2.imencode(".png", v)[1] if encode else cv2.add(v, (0.0, 0.0, 0.0, 0.0), dtype=cv2.CV_8U))
    return res


def op_test(renders, face, face_r, gt, pinned, encode):
    out = test_outputs(renders, face, face_r, gt)
    pinned.copy_(out["png"], non_blocking=True)
    torch.cuda.current_stream().synchronize()
    host = pinned.numpy()
    return [cv2.imencode(".png", host[k, 0])[1] for k in range(host.shape[0])] if encode else host


def device_ms(fn, n):
    """Device milliseconds per call of `fn`: CUDA events around `n` back-to-back calls, and the library's launches per
    call."""
    lib = L.load()
    fn()
    torch.cuda.synchronize()
    c0 = lib.b2r_launch_count()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n, (lib.b2r_launch_count() - c0) / n


def main():
    ap = arg_parser(__doc__, iters=10)
    ap.add_argument("--encode-iters", type=int, default=2, help="frames per timed window of the PNG-encoding arms")
    args = ap.parse_args()
    dev = cuda_device("bench_compose")
    result = {"card": card(), "test": {}, "train": {}}
    for H, W in SIZES:
        renders, face, face_r, gt = frame_inputs(dev, H, W, H)
        pinned = torch.empty((10, 1, H, W, 3), dtype=torch.uint8, pin_memory=True)
        with torch.no_grad():
            ref = exavatar_test(renders, face, face_r, gt, False)
            got = op_test(renders, face, face_r, gt, pinned, False)
            same = all(np.array_equal(ref[k], got[k, 0]) for k in range(10))
            arms = {"exavatar": lambda: exavatar_test(renders, face, face_r, gt, False),
                    "op": lambda: op_test(renders, face, face_r, gt, pinned, False)}
            times = alternate(arms, args.iters, args.rounds, warmup=3)
            enc = {"exavatar_png": lambda: exavatar_test(renders, face, face_r, gt, True),
                   "op_png": lambda: op_test(renders, face, face_r, gt, pinned, True)}
            times.update(alternate(enc, args.encode_iters, args.rounds, warmup=1))
            op_ms, op_launches = device_ms(lambda: test_outputs(renders, face, face_r, gt), 50)
            result["test"][f"{H}x{W}"] = {
                "ms_per_frame": {k: stats(v, 1e3, 3) for k, v in times.items()},
                "bytes_equal": same,
                "host_syncs": {"exavatar": host_syncs(lambda: exavatar_test(renders, face, face_r, gt, False)),
                               "op": host_syncs(lambda: op_test(renders, face, face_r, gt, pinned, False))},
                "op_device_us": round(op_ms * 1e3, 1), "op_launches": op_launches,
                # bytes the op must move: 5 renders, 2 masks, 2 face renders and gt in, 4 composites and 10 images out
                "op_share_of_hbm_peak": round((H * W * 4 * (15 + 2 + 8 + 3 + 12) + H * W * 30) / 3.35e12
                                              / (op_ms * 1e-3), 3),
            }

    H, W = 512, 512
    renders, face, face_r, _ = frame_inputs(dev, H, W, 1)
    x = [renders[r]["img"].clone().requires_grad_() for r in ("scene_human", "scene_human_refined")]
    f = [t.clone().requires_grad_() for t in (face, face_r)]
    g = [torch.rand(1, 3, H, W, device=dev) for _ in range(2)]

    def step(fn):
        for t in x + f:
            t.grad = None
        ys = [fn(x[i], f[i]) for i in range(2)]
        torch.autograd.backward(ys, g)

    torch_step, op_step = (lambda: step(face_composite_reference)), (lambda: step(face_composite))
    times = alternate({"torch": torch_step, "op": op_step, "torch_graph": graph_replay(torch_step, 3),
                       "op_graph": graph_replay(op_step, 3)}, args.iters * 10, args.rounds, warmup=3)
    result["train"][f"{H}x{W}"] = {"ms_per_pair_fwd_bwd": {k: stats(v, 1e3, 4) for k, v in times.items()},
                                   "op_launches": device_ms(op_step, 10)[1]}
    emit(result, args.json)


if __name__ == "__main__":
    main()
