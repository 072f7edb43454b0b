"""ExAvatar's per-frame nearest-vertex rows and posed-mesh normals (avatar/common/nets/module.py:541-546, 501-504):
PyTorch restatement vs. `geometry.nearest_rows` + `geometry.VertexNormals`.

  python tools/bench_human_geometry.py [--iters 20] [--frames 10] [--rounds 5] [--json out.json]

Workload: the synthetic human mesh of `synthetic.make_human_mesh` at C4 human size (V = 10 478 targets, P = 167 618
queries with a 30 % self-map, 335 232 faces).  Arms:
  1. torch:     the lines restated in PyTorch -- a chunked brute-force fp32 argmin standing in for pytorch3d's
                knn_points (pytorch3d is not installable offline; its own kernels are not measured), the boolean-mask
                override with the per-frame `torch.arange(P).cuda()` upload, and the per-frame upload of the int64 face
                list + float index_add of the face normals + F.normalize + the cavity flip;
  2. op:        nearest_rows + VertexNormals, eager;
  3. op_graph:  arm 2 captured once in a CUDA graph and replayed;
  4. frame_*:   C4 training frames/s: rows -> skin_gaussians -> normals, then `TrainingFrameRenderer(use_graph=True)`
                forward + backward, with the rows and normals of arm 1 or of arm 2.
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Kernel
times come from a separate torch.profiler run.  Prints the card name and power limit with the numbers.
"""
import os
import sys
from functools import partial

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, graph_replay, stats  # noqa: E402
from exavatar_release_b200 import TrainingFrameRenderer  # noqa: E402
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.geometry import VertexNormals, nearest_rows, nearest_rows_reference  # noqa: E402
from exavatar_release_b200.plan import RENDERS  # noqa: E402
from exavatar_release_b200.skinning import skin_gaussians  # noqa: E402
from exavatar_release_b200.synthetic import WORKLOADS, Workload, make_human_mesh, make_population_assets  # noqa: E402


def torch_rows(q, t, mask):
    rows = nearest_rows_reference(q, t, query_chunk=16384, target_chunk=t.shape[0]).long()
    rows[mask] = torch.arange(q.shape[0]).cuda()[mask]  # a nonzero (device->host sync) and a host->device upload
    return rows


def torch_normals(xyz, faces_np, is_cavity):
    faces = torch.LongTensor(faces_np).cuda()  # pageable host -> device, every frame
    v0, v1, v2 = xyz[faces[:, 0]], xyz[faces[:, 1]], xyz[faces[:, 2]]
    fn = torch.cross(v1 - v0, v2 - v0, dim=1)
    n = torch.zeros_like(xyz)
    for c in range(3):
        n.index_add_(0, faces[:, c], fn)
    n = F.normalize(n, eps=1e-6, dim=1)
    cav = is_cavity[:, None].float()
    return n * (1 - cav) + (-n) * cav


def main():
    ap = arg_parser(__doc__, iters=20, frames=10)
    ap.add_argument("--profile-iters", type=int, default=5)
    a = ap.parse_args()
    dev = cuda_device("bench_human_geometry")
    m = make_human_mesh()
    P, V = m["verts"].shape[0], m["targets"].shape[0]
    q, t, x = m["queries"].to(dev), m["targets"].to(dev), m["verts"].to(dev)
    sm, cav = m["self_map"].to(dev), m["flip"].to(dev)
    faces_np = m["faces"].numpy()
    vn = VertexNormals(faces_np, P, flip=cav)
    result = {"workload": f"C4 human mesh: P={P} queries, V={V} targets, F={len(faces_np)} faces",
              "card": card(), "ms": {}, "frame_fps": {}, "kernels": {}}

    # the two arms agree: rows exactly, normals to fp32 summation order
    r_t, r_o = torch_rows(q, t, sm), nearest_rows(q, t, sm)
    n_t, n_o = torch_normals(x, faces_np, cav), vn(x)
    torch.cuda.synchronize()
    assert torch.equal(r_t.int(), r_o)
    result["normals_max_abs_diff"] = float((n_t - n_o).abs().max())

    def arm_torch():
        torch_rows(q, t, sm)
        torch_normals(x, faces_np, cav)

    def arm_op():
        nearest_rows(q, t, sm)
        vn(x)

    arms = {"torch": arm_torch, "op": arm_op, "op_graph": graph_replay(arm_op, 3)}
    times = alternate(arms, a.iters, a.rounds, 3)
    result["ms"] = {k: stats(v, 1e3, 3) for k, v in times.items()}

    from torch.profiler import ProfilerActivity, profile
    for k in ("torch", "op"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_iters):
                arms[k]()
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" and e.device_time_total > 0:
                per[e.key] = (e.device_time_total / a.profile_iters, e.count / a.profile_iters)
        top = sorted(per.items(), key=lambda kv: -kv[1][0])
        result["kernels"][k] = {"device_us_per_call": round(sum(v[0] for v in per.values()), 1),
                                "launches_per_call": round(sum(v[1] for v in per.values()), 1),
                                "top": {n[:90]: [round(v[0], 1), v[1]] for n, v in top[:8]}}

    # C4 training frames/s: rows -> pose both sets -> normals, then the merged five-render frame, forward + backward
    c4 = WORKLOADS["C4"]
    H, W = c4.height, c4.width
    wl = Workload("C4 with the synthetic mesh's Gaussians", H, W, P, c4.n_scene, 0, True)
    scene, human, refined = make_population_assets(wl, seed=0, device=dev)
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    R, tc = cam["R"], cam["t"]
    to_cam = lambda v: (v @ R.t() + tc.view(1, 3)).contiguous()  # noqa: E731
    qc, tcam, qrc = to_cam(q), to_cam(t), to_cam(q + 0.002)
    g = torch.Generator().manual_seed(5)
    table = torch.zeros(P, 55)
    idx = torch.rand(P, 55, generator=g).topk(4, dim=1).indices
    table.scatter_(1, idx, torch.full((P, 4), 0.25))
    table = table.to(dev)
    A = torch.eye(4).repeat(55, 1, 1).to(dev)
    A[:, :3, 3] = 0.01 * torch.randn(55, 3, generator=g).to(dev)
    A.requires_grad_()
    tr = torch.zeros(3, device=dev, requires_grad=True)
    xyz = qc.clone().requires_grad_()
    xyz_r = qrc.clone().requires_grad_()
    lv = {k: v.detach().clone().requires_grad_() for k, v in scene.items()}
    hv = {k: v for k, v in human.items() if k != "mean_3d"}
    rv = {k: v for k, v in refined.items() if k != "mean_3d"}
    bg = torch.tensor([0.3, 0.7, 0.2], device=dev)
    fr = TrainingFrameRenderer(scene["mean_3d"].shape[0], P, (H, W), dev, {"A": 8_000_000, "B": 8_000_000},
                               use_graph=True)
    leaves = [xyz, xyz_r, A, tr, *lv.values()]

    def frame(which):
        if which == "torch":
            rows = torch_rows(xyz.detach(), tcam, sm)
        else:
            rows = nearest_rows(xyz.detach(), tcam, sm)
        posed, posed_r = skin_gaussians(xyz, xyz_r, table, rows, A, tr, R, tc)
        with torch.no_grad():
            normal = torch_normals(posed_r, faces_np, cav) if which == "torch" else vn(posed_r.detach())
        out = fr(lv, dict(hv, mean_3d=posed), dict(rv, mean_3d=posed_r), cam, bg)
        loss = sum((out[r]["img"] * 1e-3).sum() for r in RENDERS) + 0.0 * normal.sum()
        loss.backward()
        for v in leaves:
            v.grad = None

    times = alternate({k: partial(frame, k) for k in ("torch", "op")}, a.frames, a.rounds, 3)
    assert not fr.overflowed()
    result["frame_fps"] = {"frame_" + k: stats([1 / s for s in v], 1.0, 1) for k, v in times.items()}
    emit(result, a.json)


if __name__ == "__main__":
    main()
