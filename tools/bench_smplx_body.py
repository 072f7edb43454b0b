"""ExAvatar's get_smplx_outputs (avatar/main/model.py:37-58) in PyTorch ops vs. `SmplxRig.body_mesh`.

  python tools/bench_smplx_body.py [--iters 50] [--rounds 5] [--frames 10] [--json out.json]

The frame's SMPL-X body mesh at C4 size (make_smplx_model on make_human_mesh: V = 10 478, 55 joints, 100 shape and 50
expression coefficients) in world coordinates, forward only (as test.py and animate.py run it) and forward + backward
of a seeded weighted sum of the mesh.  Arms:
  1. exavatar:  `smplx_body_reference` in fp32 torch ops on the device, ExAvatar's form: shapedirs and expr_dirs
                concatenated per call, one einsum, J_regressor, batch_rodrigues of full_pose + pose_mean, the posedirs
                product, the Python FK loop of 55 4x4 matmuls, LBS, + transl, then torch.inverse(R) (mesh - t).  The
                SMPL-X layer's landmarks (find_dynamic_lmk_idx_and_bcoords, vertices2landmarks) and extra joints are
                omitted, because the reference cannot be read here: this arm UNDERSTATES ExAvatar's cost;
  2. op:        `SmplxRig.body_mesh`, eager;
  3. op_graph:  arm 2 captured once in a CUDA graph and replayed.
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Host
syncs per call are counted with torch's sync debug mode ("warn"); device time and launches per call come from a
separate torch.profiler run, which also lists the op's kernels one by one.  The op's algorithmic bytes (the model
tables it must read and the mesh I/O, from shapes) are reported over its kernels' device time as a share of the H100's
3.35 TB/s data-sheet bandwidth.  Finally C4 training frames/s of tools/c4_frame.py's frame with the body mesh computed
every frame in ExAvatar's form (mesh_exavatar), by the op (mesh_op) and not at all (mesh_none).  Prints the card name
and power limit with the numbers.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import (HBM_BYTES_PER_S, alternate, arg_parser, card, cuda_device, emit, graph_replay,  # noqa: E402
                      host_syncs, kernel_events, stats)
from c4_frame import FrameArm, frames_per_second  # noqa: E402
from exavatar_release_b200.smplx_rig import SmplxRig, batch_rodrigues, smplx_body_reference  # noqa: E402
from exavatar_release_b200.synthetic import make_human_mesh, make_smplx_model  # noqa: E402


def device_model(rig):
    """rig.model with its float tables on the rig's device in fp32 (ExAvatar keeps the layer's buffers there); the
    integer tables stay on the host, where the Python FK loop reads `parents`."""
    return {k: v.to(rig.device, torch.float32) if isinstance(v, torch.Tensor) and v.is_floating_point() else v
            for k, v in rig.model.items()}


def algorithmic_bytes(rig):
    """Bytes the op must move at least, from shapes: forward reads template, shapedirs, expr_dirs, posedirs,
    lbs_weights and the J_regressor CSR and writes the mesh; the backward reads posedirs, lbs_weights, shapedirs,
    expr_dirs and the transposed CSR again and the mesh's gradient."""
    V, J, NB, NE = rig.V, rig.J, rig.NB, rig.NE
    K = 9 * (J - 1)
    tables = 4 * V * 3 * (1 + NB + NE + K) + 4 * V * J
    jreg = 8 * int(rig.jreg_cols.numel()) + 4 * (J + 1)
    fwd = tables + jreg + 4 * 3 * V
    bwd = 4 * V * 3 * (NB + NE + K) + 4 * V * J + 8 * int(rig.jregT_rows.numel()) + 4 * (V + 1) + 4 * 3 * V
    return {"forward": fwd, "forward_backward": fwd + bwd, "posedirs": 4 * V * 3 * K}


def main():
    a = arg_parser(__doc__, iters=50, frames=10).parse_args()
    dev = cuda_device("bench_smplx_body")
    rig = SmplxRig(**make_smplx_model(make_human_mesh()), device=dev)
    dm = device_model(rig)
    g = torch.Generator().manual_seed(0)
    J = rig.J
    x = [torch.randn(rig.NB, generator=g), 0.01 * torch.randn(J, 3, generator=g), 0.3 * torch.randn(J, 3, generator=g),
         torch.randn(rig.NE, generator=g), torch.tensor([0.1, -0.2, 3.0])]
    x = [t.to(dev).requires_grad_() for t in x]
    R = batch_rodrigues(torch.tensor([[0.3, -0.5, 0.2]], dtype=torch.float64))[0].float().to(dev)
    t = torch.tensor([0.2, 0.1, -0.4], device=dev)
    w = torch.randn((rig.V, 3), generator=g).to(dev)

    def exavatar(xs=x):
        return smplx_body_reference(dm, *xs, R, t, dtype=torch.float32, device=dev)

    def op(xs=x):
        return rig.body_mesh(*xs, R, t)

    def fwd(fn):
        def run():
            with torch.no_grad():
                fn()
        return run

    def fwd_bwd(fn):
        def run():
            (fn() * w).sum().backward()
            for v in x:
                v.grad = None
        return run

    with torch.no_grad():
        ref64 = smplx_body_reference(rig.model, *[v.double() for v in x], R.double(), t.double(), device=dev)
        agree = {k: float((fn().double() - ref64).abs().max()) for k, fn in (("exavatar", exavatar), ("op", op))}
        agree["max_abs"] = float(ref64.abs().max())

    modes = (("fwd", fwd), ("fwd_bwd", fwd_bwd))
    graphs = {mode: graph_replay(wrap(op), 2) for mode, wrap in modes}
    arms = {}
    for mode, wrap in modes:
        arms[f"exavatar_{mode}"] = wrap(exavatar)
        arms[f"op_{mode}"] = wrap(op)
        arms[f"op_graph_{mode}"] = graphs[mode]
    times = alternate(arms, a.iters, a.rounds, 3)
    syncs = {k: host_syncs(fn) for k, fn in arms.items() if "graph" not in k}

    prof = {}
    for k, fn in arms.items():
        ev, prof[k] = kernel_events(fn)
        own = {}
        for e in ev:
            if e.name.startswith("b2r::"):
                name = e.name.split("(")[0][len("b2r::"):]
                own[name] = own.get(name, 0.0) + e.device_time / 1e3
        prof[k]["op_kernels_ms"] = own

    nbytes = algorithmic_bytes(rig)
    bw = {}
    for mode, key in (("fwd", "forward"), ("fwd_bwd", "forward_backward")):
        ms = sum(prof[f"op_{mode}"]["op_kernels_ms"].values())  # the op's kernels, not the loss's torch ops
        bw[mode] = {"bytes": nbytes[key], "device_ms": ms, "TB_per_s": nbytes[key] / (ms * 1e-3) / 1e12,
                    "share_of_3.35TBps": nbytes[key] / (ms * 1e-3) / HBM_BYTES_PER_S}

    models = {}

    def mesh_exavatar(r, beta, jo, pose, expr, trans, cam_R, cam_t):
        if id(r) not in models:
            models[id(r)] = device_model(r)
        return smplx_body_reference(models[id(r)], beta, jo, pose, expr, trans, cam_R, cam_t, dtype=torch.float32,
                                    device=dev)

    meshes = {"mesh_exavatar": FrameArm(mesh=mesh_exavatar),
              "mesh_op": FrameArm(mesh=lambda r, *ins: r.body_mesh(*ins)),
              "mesh_none": FrameArm(mesh=lambda *ins: None)}
    res = {"card": card(), "V": rig.V, "J": rig.J,
           "ms": {k: stats(v, 1e3) for k, v in times.items()},
           "host_syncs_per_call": syncs, "profile": prof, "algorithmic_bytes": nbytes, "op_bandwidth": bw,
           "max_abs_error_vs_float64": agree,
           "frames_per_s": frames_per_second(a, dev, meshes)}
    emit(res, a.json)


if __name__ == "__main__":
    main()
