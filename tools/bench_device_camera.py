"""C4 training frames with the camera set up on the host vs. on the device (`renderer.device_render_settings`).

  python tools/bench_device_camera.py [--rounds 5] [--frames 10] [--json out.json]

tools/c4_frame.py's frame (rig op, networks, skinning, the five renders through TrainingFrameRenderer, l1_ssim, the
regularisers, one backward) with a fresh camera tensor every frame, as ExAvatar's data loader hands one over.  Arms:
  host:    render_settings -> renderer._device_camera: the camera is read back to the host (one synchronisation in
           the middle of the frame), evaluated on the CPU and uploaded;
  device:  device_render_settings: one b2r_camera_setup launch, no host read.
Each arm runs with an eager TrainingFrameRenderer and with use_graph=True (with float settings a new focal length would
re-capture; here the intrinsics stay fixed, so both graph arms replay).  Arms alternate window by window in one
process.  Reported: training frames/s (host clock around a window of frames that ends in a device sync) and host time
per frame (the mean time the frame's Python call takes before returning, i.e. how long the host is busy or blocked).
Prints the card name and power limit with the numbers.
"""
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from benchkit import arg_parser, card, cuda_device, emit, stats  # noqa: E402
from c4_frame import FrameArm, make_frame  # noqa: E402
from exavatar_release_b200.renderer import device_render_settings, render_settings  # noqa: E402


def fresh(cam):
    """A new tensor per key, as the data loader hands over every frame (the host mirror's cache cannot hit)."""
    return {k: v.clone() for k, v in cam.items()}


ARMS = {"host": FrameArm(camera=lambda shape, cam, bg: render_settings(shape, fresh(cam), bg)),
        "device": FrameArm(camera=lambda shape, cam, bg: device_render_settings(shape, fresh(cam), bg))}


def timed(frame, arms, n, rounds, warmup=3):
    """{arm: ([seconds per frame], [host seconds per frame])}, one value per round, arms alternated."""
    for arm in arms.values():
        for _ in range(warmup):
            frame(arm)
    out = {k: ([], []) for k in arms}
    for _ in range(rounds):
        for k, arm in arms.items():
            torch.cuda.synchronize()
            host = 0.0
            t0 = time.perf_counter()
            for _ in range(n):
                h0 = time.perf_counter()
                frame(arm)
                host += time.perf_counter() - h0
            torch.cuda.synchronize()
            out[k][0].append((time.perf_counter() - t0) / n)
            out[k][1].append(host / n)
    return out


def main():
    a = arg_parser(__doc__, iters=None, frames=10).parse_args()
    dev = cuda_device("bench_device_camera")
    res = {"card": card(), "frames_per_window": a.frames, "rounds": a.rounds}
    for mode, use_graph in (("eager", False), ("graph", True)):
        frame, fr = make_frame(dev, use_graph)
        t = timed(frame, ARMS, a.frames, a.rounds)
        if fr.overflowed():
            raise SystemExit("bench_device_camera: a render overflowed its list capacity")
        for k, (wall, host) in t.items():
            res[f"{mode}_{k}"] = {"frames_per_s": stats([1 / s for s in wall], nd=2),
                                  "host_ms_per_frame": stats(host, 1e3, nd=2)}
        if use_graph:
            res["graph_captures"] = len(fr._graphs)
        del frame, fr
        torch.cuda.empty_cache()
    emit(res, a.json)


if __name__ == "__main__":
    main()
