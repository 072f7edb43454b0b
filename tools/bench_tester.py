"""ExAvatar's test pass (test.py + eval_neuman.py) on a trained avatar: the scripts' structure with the repo's ops vs.
AvatarTester, eager and graphed.

  python tools/bench_tester.py [--frames 16] [--rounds 3] [--json out.json]

The C4 human (tools/c4_frame.py's SyntheticAvatar: the synthetic SMPL-X rig, P = 167 618 Gaussians, all four GroupNorm
stacks and the triplanes seeded) and a 130 000-Gaussian SH-degree-3 scene, over a test split of --frames frames at
512 x 512 and 1080 x 1920 (portrait: H = 1920, W = 1080), with eval's masks.  Every arm goes from the resident tables
to each frame's ten images' bytes and three scores on the host:
  1. script:  test.py's and eval_neuman's structure with the repo's ops -- per frame, the frame's and the SMPL-X
              table's rows read by host slot, the test forward eagerly (SyntheticAvatar.test_chain), the ten images
              copied to the host one `.cpu()` at a time and turned into bytes there (compose.png_bytes, what
              cv2.imwrite stores), then NeumanScores with the mask and each score read back with `float()`;
  2. eager:   AvatarTester(use_graph=False).frames();
  3. graph:   AvatarTester(use_graph=True, in_flight=2).frames().
Each arm runs once without and once with host PNG encoding (cv2.imencode of the ten images, what cv2.imwrite spends
before the file write).  Arms alternate pass by pass over the whole split in one process, every arm warmed at every
size (host clock around each pass, device synchronised at both ends): median (min-max) frames/s.  Prints the card name
and power limit read in the same run.
"""
import os
import sys
import tempfile

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, stats  # noqa: E402
from c4_frame import SyntheticAvatar  # noqa: E402
from exavatar_release_b200 import NeumanScores  # noqa: E402
from exavatar_release_b200.compose import PNG_ORDER, png_bytes  # noqa: E402

SIZES = ((512, 512), (1920, 1080))  # (H, W)
CAPACITY = 1 << 24


def alex_scorer(dev, seed=0):
    """NeumanScores with torchvision's AlexNet at its seeded default initialisation and non-negative lin weights (the
    trained weights need a download; the op's cost does not depend on the values)."""
    import torchvision
    torch.manual_seed(seed)
    feats = torchvision.models.alexnet(weights=None).features.eval()
    g = torch.Generator().manual_seed(seed + 1)
    return NeumanScores(feats, [torch.rand(1, c, 1, 1, generator=g) * 0.2 for c in (64, 192, 384, 256, 256)], dev)


def encode(images):
    return [cv2.imencode(".png", x)[1] for x in images]


def script_pass(av, s, scorer, frame_idx, png):
    """One pass of test.py then eval_neuman's loop, in their structure."""
    out = []
    with torch.no_grad():
        for f in frame_idx:
            slot = s.frames.slot_of(f)
            res = av.test_chain(s, slot, png=False)
            host = [res[k].cpu().numpy() for k in PNG_ORDER]  # ten .cpu() copies, each a host sync
            images = [png_bytes(x[0]) for x in host]
            if png:
                encode(images)
            sc = scorer(res["scene_human_img_refined_composed"], res["gt"], s.masks(slot))[0]
            out.append((images, [float(sc[0]), float(sc[1]), float(sc[2])]))  # eval reads each score back
    return out


def tester_pass(t, png):
    out = []
    for _, images, sc in t.frames():
        if png:
            encode(images)
        out.append((images.copy(), sc.tolist()))
    return out


def main():
    ap = arg_parser(__doc__, iters=None, rounds=3, frames=16)
    args = ap.parse_args()
    dev = cuda_device("bench_tester")
    result = {"card": card(), "frames_per_split": args.frames, "sizes": {}}
    av = SyntheticAvatar(dev)
    scorer = alex_scorer(dev)
    frame_idx = list(range(3, 3 + 5 * args.frames, 5))
    for H, W in SIZES:
        with tempfile.TemporaryDirectory() as root:
            s = av.test_setup(root, frame_idx, H, W, CAPACITY)
            eager = av.tester(s, scorer=scorer, masks=s.masks, use_graph=False)
            graph = av.tester(s, scorer=scorer, masks=s.masks, in_flight=2)
            runs = {}
            for enc in (False, True):
                tag = "encode" if enc else "bytes"
                runs[f"script_{tag}"] = lambda enc=enc: script_pass(av, s, scorer, frame_idx, enc)
                runs[f"eager_{tag}"] = lambda enc=enc: tester_pass(eager, enc)
                runs[f"graph_{tag}"] = lambda enc=enc: tester_pass(graph, enc)
            outs = {k: runs[k]() for k in ("script_bytes", "eager_bytes", "graph_bytes")}
            ref = outs["script_bytes"]
            same = {k: all(all(np.array_equal(a, b) for a, b in zip(x[0], y[0])) and x[1] == y[1]
                           for x, y in zip(o, ref)) for k, o in outs.items()}
            times = alternate(runs, 1, args.rounds, 1)
            result["sizes"][f"{H}x{W}"] = {
                "frames_per_s": {k: stats([args.frames / v for v in vs], 1.0, 2) for k, vs in times.items()},
                "bytes_and_scores_equal_to_script": same,
                "tables_mb": round((s.frames.nbytes + s.masks.nbytes) / 1e6, 1),
            }
            del eager, graph, s
    emit(result, args.json)


if __name__ == "__main__":
    main()
