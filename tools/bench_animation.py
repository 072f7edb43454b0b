"""One animate_view_rot video frame the way the script computes it vs. the animation ops.

  python tools/bench_animation.py [--iters 10] [--rounds 5] [--json out.json]

Each arm goes from the frame's SMPL-X parameters, its camera and the source frame's bytes (a host uint8 array, as
cv2.imread returns it) to the uint8 (H, 3W, 3) panel on the host with the script's three labels and frame number
(cv2.putText), at 512 x 512 and at 1080 x 1920 (portrait: H = 1920, W = 1080), on the synthetic C4 rig with P = rig.P
posed Gaussians around its body.  Frames cycle through 8 poses and cameras; the orbit runs over 8 frames (k = 16).
  1. script:     animate_view_rot.py:78-117's host math as written -- torch.inverse of the camera three times on
                 frame 0 and twice after, pytorch3d's look-at restated on the CPU (look_at_view_transform_reference),
                 torch.inverse of its R, the uploads, indexed recentring, torch.matmul into the orbit camera, the
                 render's .cpu().numpy() conversion, the mesh panel's .cpu() and astype, np.concatenate.  Existing ops
                 stand in for what the script takes from elsewhere: SmplxRig.body_mesh for smplx_layer, render_settings
                 + GaussianRasterizer for gaussian_renderer, ShadedMeshRenderer for pytorch3d's render_mesh;
  2. ops:        body_mesh(joints=True), OrbitCamera, orbit_points x 2, device_render_settings, GaussianRasterizer,
                 ShadedMeshRenderer, animation_panel; the source frame goes up and the panel comes back through pinned
                 buffers, then cv2.putText on the panel's column views;
  3. ops_graph:  the device part of 2, copies included, captured as one CUDA graph and replayed per frame.
Every arm renders in the rasteriser's fixed-capacity mode (no duplicate-count polling), which a graph needs.
The HumanGaussian forward and video encoding are in neither arm.  Arms alternate window by window in one process (host
clock around the frames + device sync): median (min-max) ms per frame.  The panel kernel's device time comes from CUDA
events around one graph of 50 back-to-back launches, and its share of the HBM3 data-sheet bandwidth (3.35 TB/s) from the 36 H W bytes
it must move.  Prints the card name and power limit with the numbers.
"""
import math
import os
import sys

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import (HBM_BYTES_PER_S, alternate, arg_parser, card, cuda_device, emit, graph_replay,  # noqa: E402
                      host_syncs, stats)
from c4_frame import setup  # noqa: E402
from exavatar_release_b200 import GaussianRasterizer  # noqa: E402
from exavatar_release_b200.animation import (OrbitCamera, animation_panel, look_at_view_transform_reference,  # noqa: E402
                                             orbit_points)
from exavatar_release_b200.mesh_render import ShadedMeshRenderer  # noqa: E402
from exavatar_release_b200.rasterizer import set_fixed_capacity  # noqa: E402
from exavatar_release_b200.renderer import device_render_settings, render_settings  # noqa: E402
from exavatar_release_b200.synthetic import make_human_mesh, make_smplx_model  # noqa: E402

SIZES = ((512, 512), (1920, 1080))  # (H, W)
N_FRAMES = 8


def put_labels(img, mesh_render, render):
    """animate_view_rot.py:109-113."""
    font_size = 1.5
    thick = 3
    cv2.putText(img, 'image', (int(1 / 3 * img.shape[1]), int(0.05 * img.shape[0])), cv2.FONT_HERSHEY_SIMPLEX,
                font_size, [51, 51, 255], thick, 2)
    cv2.putText(mesh_render, 'rendered SMPL-X mesh', (int(1 / 5 * mesh_render.shape[1]), int(0.05 * mesh_render.shape[0])),
                cv2.FONT_HERSHEY_SIMPLEX, font_size, [51, 51, 255], thick, 2)
    cv2.putText(render, 'render', (int(1 / 3 * render.shape[1]), int(0.05 * render.shape[0])), cv2.FONT_HERSHEY_SIMPLEX,
                font_size, [51, 51, 255], thick, 2)


def put_number(out, frame_idx):
    return cv2.putText(out, str(frame_idx), (int(out.shape[1] * 0.05), int(out.shape[0] * 0.05)),
                       cv2.FONT_HERSHEY_SIMPLEX, 1.0, (0, 0, 255), 2, 2)


class Workload:
    def __init__(self, dev, H, W):
        hm = make_human_mesh()
        self.rig, _, x, _ = setup(dev, make_smplx_model(hm))
        self.mesh_r = ShadedMeshRenderer(hm["base_faces"], self.rig.V, device=dev)
        self.H, self.W = H, W
        beta, jo, pose, expr = (t.detach() for t in x)
        self.frames = []
        for i in range(N_FRAMES):
            g = torch.Generator().manual_seed(i)
            a = 0.1 * torch.randn(1, generator=g).item()
            R = torch.tensor([[math.cos(a), 0.0, math.sin(a)], [0.0, 1.0, 0.0], [-math.sin(a), 0.0, math.cos(a)]])
            cam = {"R": R.to(dev), "t": (0.05 * torch.randn(3, generator=g)).to(dev),
                   "focal": torch.tensor([1.2 * H, 1.2 * H], device=dev),
                   "princpt": torch.tensor([W / 2, H / 2], device=dev)}
            ins = [beta, jo, pose + 0.05 * torch.randn(pose.shape, generator=g).to(dev), expr,
                   (0.02 * torch.randn(3, generator=g)).to(dev)]
            img = np.random.default_rng(i).integers(0, 256, (H, W, 3), dtype=np.uint8)
            self.frames.append((ins, cam, img))
        with torch.no_grad():
            world = self.rig.body_mesh(*self.frames[0][0], self.frames[0][1]["R"], self.frames[0][1]["t"])
        P = self.rig.P
        g = torch.Generator(device=dev).manual_seed(0)
        rot = torch.zeros(P, 4, device=dev)
        rot[:, 0] = 1
        self.assets = {"mean_3d": world[torch.arange(P, device=dev) % world.shape[0]] +
                       0.01 * torch.randn(P, 3, device=dev, generator=g),
                       "scale": 0.003 + 0.004 * torch.rand(P, 3, device=dev, generator=g), "rotation": rot,
                       "opacity": 0.2 + 0.7 * torch.rand(P, 1, device=dev, generator=g),
                       "rgb": torch.rand(P, 3, device=dev, generator=g)}
        self.bkg = torch.full((H, W, 3), 255.0, device=dev)
        self.bg = torch.ones(3, device=dev)

    def render(self, mean_3d, settings):
        a = self.assets
        return GaussianRasterizer(settings)(means3D=mean_3d, means2D=torch.zeros_like(mean_3d),
                                            opacities=a["opacity"], colors_precomp=a["rgb"], scales=a["scale"],
                                            rotations=a["rotation"])[0]


class ScriptArm:
    def __init__(self, w):
        self.w, self.i, self.st = w, 0, {}

    @torch.no_grad()
    def __call__(self):
        w, i = self.w, self.i % N_FRAMES
        ins, cam_param, img = w.frames[i]
        mesh, joints = w.rig.body_mesh(*ins, joints=True)
        root_joint_cam = joints[0]
        mesh = torch.matmul(torch.inverse(cam_param['R']), (mesh - cam_param['t'].view(-1, 3)).permute(1, 0)).permute(1, 0)
        root_joint_world = torch.matmul(torch.inverse(cam_param['R']), root_joint_cam - cam_param['t'])
        azim = math.pi + math.pi * 16 * i / N_FRAMES
        st = self.st
        if i == 0:
            st["at_point_orig"] = root_joint_world.clone()
            st["at_point"] = root_joint_world
            cam_pos = torch.matmul(torch.inverse(cam_param['R']), -cam_param['t'].view(3, 1)).view(3)
            st["elev"] = torch.arctan(torch.abs(root_joint_cam[1]) / torch.abs(root_joint_cam[2]))
            st["dist"] = torch.sqrt(torch.sum((cam_pos - st["at_point"]) ** 2))
        mesh[:, [0, 2]] = mesh[:, [0, 2]] - root_joint_world[None, [0, 2]] + st["at_point_orig"][None, [0, 2]]
        R, t = look_at_view_transform_reference(dist=st["dist"], elev=st["elev"], azim=azim, degrees=False,
                                                at=st["at_point"][None, :], up=((0, 1, 0),))
        R = torch.inverse(R)
        cam_param_rot = {'R': R[0].cuda(), 't': t[0].cuda(), 'focal': cam_param['focal'],
                         'princpt': cam_param['princpt']}
        mesh = torch.matmul(cam_param_rot['R'], mesh.permute(1, 0)).permute(1, 0) + cam_param_rot['t'].view(1, 3)
        mesh_render = w.mesh_r(mesh, cam_param, w.bkg).cpu().numpy().astype(np.uint8)
        mean_3d = w.assets["mean_3d"].clone()
        mean_3d[:, [0, 2]] = mean_3d[:, [0, 2]] - root_joint_world[None, [0, 2]] + st["at_point_orig"][None, [0, 2]]
        human_render = {"img": w.render(mean_3d, render_settings((w.H, w.W), cam_param_rot, w.bg))}
        img = img.copy()  # cv2.imread's fresh array
        render = (human_render['img'].cpu().numpy().transpose(1, 2, 0)[:, :, ::-1] * 255).copy().astype(np.uint8)
        put_labels(img, mesh_render, render)
        out = np.concatenate((img, mesh_render, render), 1).astype(np.uint8)
        self.i += 1
        return put_number(out, i)


class OpsArm:
    def __init__(self, w, dev, graph):
        self.w, self.i = w, 0
        self.orbit = OrbitCamera(16, N_FRAMES, dev)
        self.index = torch.zeros(1, dtype=torch.int32, device=dev)
        self.src = torch.empty((w.H, w.W, 3), dtype=torch.uint8, pin_memory=True)
        self.dst = torch.empty((w.H, 3 * w.W, 3), dtype=torch.uint8, pin_memory=True)
        self.frame = torch.empty((w.H, w.W, 3), dtype=torch.uint8, device=dev)
        # the per-frame inputs live in fixed buffers so one graph replays every frame
        ins0, cam0, _ = w.frames[0]
        self.ins = [t.clone() for t in ins0]
        self.cam = {k: v.clone() for k, v in cam0.items()}
        self.replay = None
        if graph:
            self._load(0)
            self.device_frame()  # frame 0 eagerly: the first calls at this size allocate
            side = torch.cuda.Stream(dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                self.device_frame()
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self.device_frame()
            self.replay = g.replay

    def _load(self, i):
        ins, cam, img = self.w.frames[i]
        with torch.no_grad():
            for a, b in zip(self.ins, ins):
                a.copy_(b, non_blocking=True)
            for k in ("R", "t"):
                self.cam[k].copy_(cam[k], non_blocking=True)
            self.index.fill_(i)
        np.copyto(self.src.numpy(), img)

    @torch.no_grad()
    def device_frame(self):
        w = self.w
        self.frame.copy_(self.src, non_blocking=True)
        mesh, joints = w.rig.body_mesh(*self.ins, self.cam["R"], self.cam["t"], joints=True)
        cam_rot = self.orbit(self.cam, joints[0], self.index)
        mesh_cam = orbit_points(mesh, self.orbit, view=True)
        mean_3d = orbit_points(w.assets["mean_3d"], self.orbit)
        render = w.render(mean_3d, device_render_settings((w.H, w.W), cam_rot, w.bg))
        self.dst.copy_(animation_panel(self.frame, w.mesh_r(mesh_cam, self.cam, w.bkg), render), non_blocking=True)

    def __call__(self):
        i = self.i % N_FRAMES
        torch.cuda.current_stream().synchronize()  # the pinned buffers are free again
        self._load(i)
        if self.replay is not None:
            self.replay()
        else:
            self.device_frame()
        torch.cuda.current_stream().synchronize()
        out = self.dst.numpy().copy()
        W = self.w.W
        put_labels(out[:, :W], out[:, W:2 * W], out[:, 2 * W:])
        self.i += 1
        return put_number(out, i)


def panel_device_ms(w, dev, n=50):
    """Device milliseconds per panel launch: CUDA events around the replay of one graph of `n` launches, so the host's
    per-call checks stay out of the kernel's time."""
    H, W = w.H, w.W
    g = torch.Generator(device=dev).manual_seed(1)
    frame = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, device=dev, generator=g)
    mesh = torch.rand(H, W, 3, device=dev, generator=g) * 255
    render = torch.rand(3, H, W, device=dev, generator=g)
    replay = graph_replay(lambda: [animation_panel(frame, mesh, render) for _ in range(n)], 2)
    replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = arg_parser(__doc__, iters=10)
    args = ap.parse_args()
    dev = cuda_device("bench_animation")
    result = {"card": card(), "frames": {}}
    set_fixed_capacity(1 << 23)
    try:
        for H, W in SIZES:
            w = Workload(dev, H, W)
            script, ops, ops_graph = ScriptArm(w), OpsArm(w, dev, False), OpsArm(w, dev, True)
            # one pass over the orbit: the ops' panels against the script's
            same = []
            for _ in range(N_FRAMES):
                a, b, c = script(), ops(), ops_graph()
                same.append((bool(np.array_equal(b, c)), float(np.mean(a != b))))
            times = alternate({"script": script, "ops": ops, "ops_graph": ops_graph}, args.iters, args.rounds,
                              warmup=N_FRAMES)
            ms = panel_device_ms(w, dev)
            result["frames"][f"{H}x{W}"] = {
                "P": w.rig.P,
                "ms_per_frame": {k: stats(v, 1e3, 3) for k, v in times.items()},
                "host_syncs": {"script": host_syncs(script), "ops": host_syncs(ops)},
                "ops_graph_equals_ops_eager": all(s[0] for s in same),
                # the script renders through its own camera (torch.inverse, the CPU look-at), so a few edge pixels
                # may differ from the ops' panel; tests/test_animation.py checks the bytes with one camera
                "share_of_panel_bytes_differing_from_script": round(max(s[1] for s in same), 6),
                "panel_kernel_us": round(ms * 1e3, 1),
                "panel_kernel_share_of_hbm_peak": round(36 * H * W / HBM_BYTES_PER_S / (ms * 1e-3), 3),
            }
    finally:
        set_fixed_capacity(None)
    emit(result, args.json)


if __name__ == "__main__":
    main()
