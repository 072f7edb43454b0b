"""ExAvatar's two face renders of a training frame (avatar/main/model.py:170-175), forward + backward:
`mesh_render.FaceMeshRenderer` eager, as a CUDA graph, and the torch restatement `face_render_reference`.

  python tools/bench_face_render.py [--iters 20] [--rounds 5] [--json out.json]

Workload: C4 size -- a 512x512 frame from the yawed synthetic camera, the synthetic FLAME-sized face mesh of
`synthetic.make_face_mesh` (5 023 vertices, ~9.6 k faces) on the C4 avatar's head, a 4-channel 512x512 texture; the
second render uses the mesh moved by N(0, 2 mm) (the refined set).  The loss is a fixed random weighting of both images.
pytorch3d's MeshRasterizer itself cannot be installed offline and is not measured.  Arms alternate window by window
in one process (host clock around N frames + device sync): median (min-max).  Kernel times come from a separate
torch.profiler run.  Prints the card name and power limit with the numbers.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, graph_replay, stats  # noqa: E402
from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.mesh_render import FaceMeshRenderer, face_render_reference  # noqa: E402
from exavatar_release_b200.synthetic import make_face_mesh, make_human_mesh  # noqa: E402


def main():
    ap = arg_parser(__doc__, iters=20)
    ap.add_argument("--profile-iters", type=int, default=5)
    a = ap.parse_args()
    dev = cuda_device("bench_face_render")
    H, W = 512, 512
    face = make_face_mesh()
    verts = make_human_mesh()["verts"][face["vertex_idx"]].to(dev)
    g = torch.Generator().manual_seed(2)
    verts_r = verts + 0.002 * torch.randn(verts.shape, generator=g).to(dev)
    tex = face["texture"].to(dev)[None]
    cam = look_at_cam_param(-6.0, (H, W), device=dev)
    G = torch.randn(2, 1, 4, H, W, generator=g).to(dev)
    r = FaceMeshRenderer(face["vertex_uv"], face["face_uv"], face["faces"], verts.shape[0], device=dev)
    m0 = verts.clone().requires_grad_()
    m1 = verts_r.clone().requires_grad_()
    result = {"workload": f"C4 face renders: {H}x{W}, V={verts.shape[0]}, F={face['faces'].shape[0]}, "
                          f"texture {tuple(tex.shape[1:])}, 2 renders fwd+bwd per frame",
              "card": card(), "ms": {}, "kernels": {}}

    def frame_op():
        loss = (r(tex, m0[None], cam, (H, W)) * G[0]).sum() + (r(tex, m1[None], cam, (H, W)) * G[1]).sum()
        loss.backward()

    def frame_ref():
        ref = lambda m: face_render_reference(tex, m, face["faces"], face["vertex_uv"], face["face_uv"], cam,  # noqa
                                              (H, W))[0]
        loss = (ref(m0) * G[0]).sum() + (ref(m1) * G[1]).sum()
        loss.backward()

    def clear():
        m0.grad = m1.grad = None

    # parity of the two arms at this size: the per-pixel face and the gradient
    img, p2f = r.render(tex, verts[None], cam, (H, W))
    ref, ref_p2f = face_render_reference(tex, verts, face["faces"], face["vertex_uv"], face["face_uv"], cam, (H, W))
    torch.cuda.synchronize()
    result["pix_to_face_equal"] = bool(torch.equal(p2f.long(), ref_p2f))
    result["covered_pixels"] = int((p2f >= 0).sum())
    result["image_max_abs_diff"] = float((img - ref).abs().max())

    # the graph owns the .grad it accumulates into; replays overwrite it
    arms = {"reference": lambda: (frame_ref(), clear()), "op": lambda: (frame_op(), clear()),
            "op_graph": graph_replay(frame_op, 3, reset=clear)}
    times = alternate(arms, a.iters, a.rounds, 3)
    result["ms"] = {k: stats(v, 1e3, 3) for k, v in times.items()}

    from torch.profiler import ProfilerActivity, profile
    for k in ("op", "reference"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_iters):
                arms[k]()
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" and e.device_time_total > 0:
                per[e.key] = (e.device_time_total / a.profile_iters, e.count / a.profile_iters)
        top = sorted(per.items(), key=lambda kv: -kv[1][0])
        result["kernels"][k] = {"device_us_per_frame": round(sum(v[0] for v in per.values()), 1),
                                "launches_per_frame": round(sum(v[1] for v in per.values()), 1),
                                "top": {n[:90]: [round(v[0], 1), v[1]] for n, v in top[:8]}}
    emit(result, a.json)


if __name__ == "__main__":
    main()
