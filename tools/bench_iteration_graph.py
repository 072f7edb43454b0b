"""Training iterations/s of ExAvatar's whole iteration -- SMPL-X decode, rig, networks, assets, skinning, the five
renders, L1 + SSIM, the regulariser op and the Adam step -- in three forms, alternated window by window in one call:

  frames  ExAvatar's structure: per-frame ParameterDicts, decode_smplx_pose, Adam.step() over nine param groups per
          frame, TrainingFrameRenderer(use_graph=True);
  table   SmplxParamTable and one frame-row Adam group, eager, TrainingFrameRenderer(use_graph=True);
  graph   the table form under IterationGraph (TrainingFrameRenderer(use_graph=False) inside the capture).

Every iteration visits a different frame slot, in a shuffled order, at F = 100 and F = 1 000 frames.  Each form runs
without and with a per-iteration host read of its loss terms (ExAvatar's train.py:67 logs them every iteration).
Reported: iterations/s (median, min, max over the windows) and the host time per iteration (the time the Python call
takes to return, which without a read is the enqueue cost).  The frame is tools/c4_frame.py's C4 frame (512 x 512,
130 000 scene and the synthetic mesh's 167 618 human Gaussians, the SMPL-X rig in front).

`Chain` builds the frame at any size; tests/test_iteration_graph.py runs it small to check that the three forms give
bit-identical parameters, Adam state, loss terms and densification statistics.
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from benchkit import arg_parser, card, cuda_device, emit, stats  # noqa: E402
from bench_human_nets import stack  # noqa: E402
from bench_human_regs import INPUTS as REG_INPUTS  # noqa: E402
from bench_human_regs import setup as regs_setup  # noqa: E402
from exavatar_release_b200 import (Adam, HumanAssets, IterationGraph, SmplxParamTable, SmplxRig,  # noqa: E402
                                   TrainingFrameRenderer, decode_smplx_pose, skin_gaussians)
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.geometry import VertexNormals, nearest_rows  # noqa: E402
from exavatar_release_b200.human_assets import POSE_KEYS, POSE_ROWS  # noqa: E402
from exavatar_release_b200.human_nets import TriplaneFeatures, gn_mlp  # noqa: E402
from exavatar_release_b200.losses import l1_ssim  # noqa: E402
from exavatar_release_b200.plan import RENDERS  # noqa: E402
from exavatar_release_b200.renderer import device_render_settings  # noqa: E402
from exavatar_release_b200.smplx_rig import axis_angle_to_matrix, matrix_to_rotation_6d, upsample  # noqa: E402
from exavatar_release_b200.synthetic import Workload, make_population_assets, make_smplx_model  # noqa: E402

POSITION_LR = (1.6e-4, 1.6e-6)
N_INPUTS = 8  # distinct frames' inputs (image, box, camera, background), cycled over the slots


def set_lr(opt, itr, tot_itr, lr=1e-3):
    """ExAvatar's set_lr (base.py:94-108): the scene mean's exponential schedule, human and SMPL-X groups / 10 past
    75 % and / 100 past 95 % of the run."""
    t = min(max(itr / tot_itr, 0.0), 1.0)
    for gr in opt.param_groups:
        if gr["name"] == "mean_scene":
            gr["lr"] = float(np.exp(np.log(POSITION_LR[0] * 2.5) * (1 - t) + np.log(POSITION_LR[1] * 2.5) * t))
        elif "human" in gr["name"] or "smplx" in gr["name"]:
            gr["lr"] = lr / 10 if 0.75 * tot_itr < itr <= 0.95 * tot_itr else lr / 100 if itr > 0.95 * tot_itr else lr


class Chain:
    """One model and its optimizer in one form ("frames" or "table"), seeded so that every form starts from the same
    values.  `terms(slot, inputs, warm)` runs forward and backward and returns the loss terms."""

    def __init__(self, dev, form, F, H, W, n_scene, use_graph, seed=0, capacity=8_000_000):
        self.form, self.H, self.W = form, H, W
        dr, self.regs, _ = regs_setup(dev)
        m, P = dr["m"], dr["P"]
        scene, _, _ = make_population_assets(Workload("iteration", H, W, P, n_scene, 0, True), seed=seed, device=dev)
        cam = look_at_cam_param(-6.0, (H, W), device=dev)
        R, tc = cam["R"], cam["t"]
        to_cam = lambda x: (x.double() @ R.cpu().double().t() + tc.cpu().double().view(1, 3)).float()  # noqa: E731
        model = make_smplx_model(dict(m, targets=to_cam(m["targets"])))
        self.rig = SmplxRig(**model, device=dev)
        rm = self.rig.model
        self.skw = upsample(rm["lbs_weights"].to(dev, torch.float32), rm["sub1"], rm["sub2"]).contiguous()
        self.ha = HumanAssets(model["is_rhand"], model["is_lhand"], model["is_face_expr"], device=dev)
        self.self_map = m["self_map"].to(dev)
        verts = dr["mesh"]
        self.tri = TriplaneFeatures(verts, verts[:, 1] > 0.6)
        self.vn = VertexNormals(m["faces"], P, flip=m["flip"].to(dev))
        torch.manual_seed(seed + 3)
        self.nets = {"geo": stack(96, [3, 1]), "geo_offset": stack(96 + 126, [3, 1]), "rgb": stack(96, None, 3),
                     "rgb_offset": stack(96 + 126 + 3, None, 3)}
        g = torch.Generator().manual_seed(seed + 5)
        leaf = lambda t: t.to(dev).requires_grad_()  # noqa: E731
        self.tp, self.tpf = (leaf(0.3 * torch.randn((3, 32, 128, 128), generator=g)) for _ in range(2))
        self.shape = leaf(torch.randn(self.rig.NB, generator=g))
        self.joint_offset = leaf(0.01 * torch.randn(self.rig.J, 3, generator=g))
        self.scene = {k: v.detach().clone().requires_grad_() for k, v in scene.items()}
        frames = {}
        for f in range(F):
            rot6 = matrix_to_rotation_6d(axis_angle_to_matrix(0.3 * torch.randn(55, 3, generator=g))).float()
            d, r0 = {}, 0
            for k, n in zip(POSE_KEYS, POSE_ROWS):
                d[k] = (rot6[r0] if n == 1 else rot6[r0:r0 + n]).to(dev)
                r0 += n
            d["expr"] = (0.1 * torch.randn(self.rig.NE, generator=g)).to(dev)
            d["trans"] = (0.01 * torch.randn(3, generator=g)).to(dev)
            frames[str(f)] = d
        groups = [{"params": [v], "name": "mean_scene" if k == "mean_3d" else f"{k}_scene", "lr": 1e-3}
                  for k, v in self.scene.items()]
        human = [self.tp, self.tpf, self.shape, self.joint_offset] + [p for t, hs in self.nets.values()
                                                                      for mm in [t, *hs] for p in mm.parameters()]
        groups += [{"params": [p], "name": f"p{i}_human", "lr": 1e-3} for i, p in enumerate(human)]
        if form == "frames":
            self.pd = {f: {k: torch.nn.Parameter(v.clone()) for k, v in d.items()} for f, d in frames.items()}
            groups += [{"params": [p], "name": f"smplx_{k}_{f}", "lr": 1e-3} for f, d in self.pd.items()
                       for k, p in d.items()]
        else:
            self.table = SmplxParamTable.from_param_dict(frames)
            groups.append({"params": self.table.parameters(), "name": "smplx", "lr": 1e-3, "frame_rows": True})
        self.opt = Adam(groups, lr=0.0, eps=1e-15)
        self.P_human, self.capacity = P, {"A": capacity, "B": capacity}
        self.fr = TrainingFrameRenderer(n_scene, P, (H, W), dev, self.capacity, use_graph=use_graph)
        self.fr.densify = {k: torch.zeros(n_scene, device=dev) for k in ("grad_accum", "count", "radius_max")}
        self.white = torch.ones(3, device=dev)

    def append_scene(self, rows):
        """Densification's optimizer surgery (module.py:17-36): the rows {key: (n, ...)} appended to every scene
        parameter with zero moments and the step kept; the renderer and the densification buffers grow with them."""
        for gr in self.opt.param_groups:
            k = next((k for k, v in self.scene.items() if gr["params"][0] is v), None)
            if k is None:
                continue
            old = gr["params"][0]
            st = self.opt.state.pop(old)
            new = torch.cat((old.detach(), rows[k])).requires_grad_()
            for m in ("exp_avg", "exp_avg_sq"):
                st[m] = torch.cat((st[m], torch.zeros_like(rows[k])))
            self.opt.state[new] = st
            gr["params"][0] = self.scene[k] = new
        P_scene, n = self.scene["mean_3d"].shape[0], rows["mean_3d"].shape[0]
        old_fr = self.fr
        self.fr = TrainingFrameRenderer(P_scene, self.P_human,
                                        (self.H, self.W), old_fr.plan.device, self.capacity, use_graph=old_fr.use_graph)
        self.fr.densify = {k: torch.cat((v, torch.zeros(n, device=v.device))) for k, v in old_fr.densify.items()}

    def decode(self, slot):
        return decode_smplx_pose(self.pd[str(int(slot))]) if self.form == "frames" else self.table(slot)

    def terms(self, sp, inputs, warm):
        """Forward and backward of one iteration from the frame's decoded SMPL-X parameters `sp`; the loss terms."""
        out = self.rig(self.shape, self.joint_offset, sp["full_pose"], sp["expr"])
        f = self.tri(self.tp, self.tpf)
        net = lambda k, ins: gn_mlp(ins, *self.nets[k])  # noqa: E731
        geo, geo_off, rgb = net("geo", [f]), net("geo_offset", [f, out.pose_6d]), net("rgb", [f])
        a = self.ha.geometry(out.mesh_neutral_pose, out.pose_offset, out.expr_offset, geo, geo_off, warmup=warm)
        rows = nearest_rows(a["mean_3d"].detach(), out.mesh_neutral_pose_wo_upsample.contiguous(), self.self_map)
        posed, posed_r = skin_gaussians(a["mean_3d"], a["mean_3d_refined"], self.skw, rows, out.joint_mats,
                                        sp["trans"], inputs["R"], inputs["t"])
        rgb_off = net("rgb_offset", [f, out.pose_6d, self.vn(posed_r)])
        rgb_h, rgb_r = self.ha.colors(rgb, rgb_off)
        hv = dict(mean_3d=posed, opacity=self.ha.opacity, scale=a["scale"], rotation=self.ha.rotation, rgb=rgb_h)
        rv = dict(mean_3d=posed_r, opacity=self.ha.opacity, scale=a["scale_refined"], rotation=self.ha.rotation,
                  rgb=rgb_r)
        cam = {k: inputs[k] for k in ("R", "t", "focal", "princpt")}
        st = device_render_settings((self.H, self.W), cam, self.white)
        o = self.fr(self.scene, hv, rv, cam, inputs["bg"], raster_settings=st)
        terms = {}
        for r in RENDERS:
            l1, ss = l1_ssim(o[r]["img"], inputs["img"], inputs["bbox"])
            terms[f"l1_{r}"], terms[f"ssim_{r}"] = 0.8 * l1, 0.2 * (1 - ss)
        y = dict(a, rgb=rgb_h, rgb_refined=rgb_r, joint_offset=self.joint_offset)
        terms.update(self.regs(out.mesh_neutral_pose.detach(), *[y[k] for k in REG_INPUTS]))
        sum(terms.values()).backward()
        return terms

    def eager(self, slot, inputs, warm):
        """One eager iteration as ExAvatar runs it: zero_grad(set_to_none), forward, backward, Adam step."""
        self.opt.zero_grad(set_to_none=True)
        terms = self.terms(self.decode(slot), inputs, warm)
        self.opt.step(rows=None if self.form == "frames" else int(slot))
        return terms

    def graph(self, template):
        """The table form under IterationGraph; `run(slot, inputs, warm)` is one iteration."""
        it = IterationGraph(lambda inputs, slot_t: self.terms(self.table(slot_t), inputs, self._warm), self.opt,
                            template)

        def run(slot, inputs, warm):
            self._warm = warm
            return it.run(inputs, slot, key=warm)
        return it, run


def make_inputs(dev, H, W, n=N_INPUTS, seed=100):
    """n frames' static inputs: target image, box, camera (a small shift per frame) and background."""
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    out = []
    for i in range(n):
        g = torch.Generator(device=dev).manual_seed(seed + i)
        out.append({"img": torch.rand((3, H, W), generator=g, device=dev),
                    "bbox": torch.tensor([0.05 * W + i, 0.1 * H, 0.8 * W - i, 0.75 * H], device=dev),
                    "R": cam["R"].to(dev, torch.float32).contiguous(),
                    "t": (cam["t"].to(dev, torch.float32) + 0.002 * i).contiguous(),
                    "focal": cam["focal"].to(dev, torch.float32).reshape(2).contiguous(),
                    "princpt": cam["princpt"].to(dev, torch.float32).reshape(2).contiguous(),
                    "bg": torch.rand(3, generator=g, device=dev)})
    return out


def measure(a, dev, F):
    H = W = 512
    inputs = make_inputs(dev, H, W)
    order = np.random.default_rng(0).permutation(np.resize(np.arange(F), a.warmup + a.rounds * a.iters * 6))
    arms = {}
    for name, form, use_graph in (("frames", "frames", True), ("table", "table", True), ("graph", "table", False)):
        c = Chain(dev, form, F, H, W, 130_000, use_graph)
        if name == "graph":
            _, run = c.graph(inputs[0])
        else:
            run = c.eager
        arms[name] = (c, run)
    pos = {"i": 0}

    def one(run, read):
        s = int(order[pos["i"] % len(order)])
        pos["i"] += 1
        t0 = time.perf_counter()
        terms = run(s, inputs[s % N_INPUTS], False)
        host = time.perf_counter() - t0
        if read:
            torch.stack([v.detach().reshape(()) for v in terms.values()]).tolist()
        return host

    for c, run in arms.values():  # warm-up: every arm's eager, capture and first replays
        for _ in range(a.warmup):
            one(run, False)
    res = {}
    for _ in range(a.rounds):
        for read in (False, True):
            for name, (c, run) in arms.items():
                torch.cuda.synchronize()
                t0, host = time.perf_counter(), 0.0
                for _ in range(a.iters):
                    host += one(run, read)
                torch.cuda.synchronize()
                r = res.setdefault(f"{name}{'_read' if read else ''}", {"s": [], "host": []})
                r["s"].append((time.perf_counter() - t0) / a.iters)
                r["host"].append(host / a.iters)
    for c, _ in arms.values():
        if c.fr.overflowed():
            raise SystemExit("bench_iteration_graph: a render overflowed its list capacity")
    return {k: {"iters_per_s": stats([1 / s for s in v["s"]], nd=2), "host_ms": stats(v["host"], 1e3, 3)}
            for k, v in res.items()}


def main():
    ap = arg_parser(__doc__, iters=20, rounds=3)
    ap.add_argument("--frames-list", default="100,1000", help="frame counts F")
    ap.add_argument("--warmup", type=int, default=4, help="untimed iterations per arm (eager, capture, replays)")
    a = ap.parse_args()
    dev = cuda_device("bench_iteration_graph")
    out = {"card": card(), "workload": "C4 512x512, 130 000 scene + 167 618 human Gaussians, SMPL-X rig, l1_ssim x5, "
           "regulariser op", "iters_per_window": a.iters, "rounds": a.rounds}
    for F in (int(x) for x in a.frames_list.split(",")):
        out[f"F={F}"] = measure(a, dev, F)
        torch.cuda.empty_cache()
    out["card_after"] = card()
    emit(out, a.json)


if __name__ == "__main__":
    main()
