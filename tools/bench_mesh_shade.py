"""The mesh panel of ExAvatar's animation scripts (animate.py:81-83, animate_view_rot.py:98 -> utils/vis.py render_mesh):
`mesh_render.ShadedMeshRenderer` eager, as a CUDA graph, and the float32 torch restatement `shaded_mesh_reference`.

  python tools/bench_mesh_shade.py [--iters 20] [--rounds 5] [--json out.json]

Workload: the synthetic SMPL-X-sized base mesh (make_human_mesh: 10 478 vertices, 20 952 faces) posed by
`SmplxRig.body_mesh` in camera coordinates, rendered over a white 0-255 background at 512x512 and in a 1080x1920
portrait video frame.  Arms per size:
  render_op / render_op_graph / render_reference   the render alone, from the posed mesh to the (H,W,3) panel;
  panel_op         one animation frame's panel: body_mesh -> the op -> .to(torch.uint8) -> .cpu();
  panel_reference  smplx_body_reference(float32) -> the restatement's colour and zbuf -> two .cpu() copies -> vis.py's
                   composite and .astype(np.uint8) in numpy, as render_mesh ends.
pytorch3d cannot be installed offline and is not measured: the restatement stands in for its rasteriser and shader and
does not include building its Meshes / cameras / shader objects per call.  The two panel arms pose the mesh by
different arithmetic (the op's fp64 chain, fp32 torch), so a few silhouette pixels of their uint8 panels differ.
Arms alternate window by window in one process (host clock around N calls + device sync): median (min-max).  Prints
the card name and power limit.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from benchkit import alternate, arg_parser, card, cuda_device, emit, graph_replay, host_syncs, stats  # noqa: E402
from exavatar_release_b200.mesh_render import (ShadedMeshRenderer, _shade_reference,  # noqa: E402
                                               shaded_mesh_reference)
from exavatar_release_b200.smplx_rig import SmplxRig, smplx_body_reference  # noqa: E402
from exavatar_release_b200.synthetic import make_human_mesh, make_smplx_model  # noqa: E402

SIZES = {"512x512": ((512, 512), (1100.0, 1080.0), (250.0, 262.0)),
         "1080x1920": ((1920, 1080), (3600.0, 3650.0), (545.0, 950.0))}  # (H, W): a portrait video frame


def main():
    a = arg_parser(__doc__, iters=20).parse_args()
    dev = cuda_device("bench_mesh_shade")
    mesh = make_human_mesh()
    rig = SmplxRig(**make_smplx_model(mesh), device=dev)
    model32 = {k: v.to(dev, torch.float32) if isinstance(v, torch.Tensor) and v.is_floating_point() else v
               for k, v in rig.model.items()}
    faces = mesh["base_faces"]
    face_np = faces.numpy()
    g = torch.Generator().manual_seed(11)
    ins = [torch.randn(rig.NB, generator=g), 0.01 * torch.randn(rig.J, 3, generator=g),
           0.1 * torch.randn(rig.J, 3, generator=g), torch.randn(rig.NE, generator=g), torch.tensor([0.02, -0.05, 0.0])]
    ins = [t.to(dev) for t in ins]
    r = ShadedMeshRenderer(faces, rig.V, device=dev)
    result = {"workload": f"SMPL-X-sized body mesh V={rig.V}, F={faces.shape[0]}, posed by body_mesh in camera "
                          "coordinates, white background, blend_ratio 1", "card": card(), "sizes": {}}
    for name, (shape, focal, princpt) in SIZES.items():
        H, W = shape
        cam = {"focal": torch.tensor(focal, device=dev), "princpt": torch.tensor(princpt, device=dev)}
        bkg = torch.full((H, W, 3), 255.0, device=dev)
        bkg_np = np.ones((H, W, 3), dtype=np.float32) * 255
        with torch.no_grad():
            posed = rig.body_mesh(*ins)

        def render_op():
            return r(posed, cam, bkg)

        def render_ref():
            return shaded_mesh_reference(posed, faces, cam, bkg)[0]

        def panel_op():
            with torch.no_grad():
                return r(rig.body_mesh(*ins), cam, bkg).to(torch.uint8).cpu()

        def panel_ref():
            with torch.no_grad():
                m = smplx_body_reference(model32, *ins, dtype=torch.float32, device=dev)
                c, zbuf, _ = _shade_reference(m, face_np, cam, H, W)
            is_bkg = (zbuf <= 0).float().cpu().numpy()[:, :, None]
            render = c.cpu().numpy()
            fg = render * 1.0 + bkg_np / 255 * (1 - 1.0)
            return (fg * (1 - is_bkg) * 255 + bkg_np * is_bkg).astype(np.uint8)

        # agreement at this size
        out, ref = render_op(), render_ref()
        a_op, a_ref = panel_op().numpy(), panel_ref()
        torch.cuda.synchronize()
        rec = {"covered_pixels": int((out != bkg).any(-1).sum()),
               "render_max_abs_diff_vs_float32_reference": float((out - ref).abs().max()),
               "panel_uint8_pixels_differing": int((a_op != a_ref).any(-1).sum()),
               "panel_uint8_max_abs_diff": int(np.abs(a_op.astype(np.int16) - a_ref.astype(np.int16)).max())}
        arms = {"render_op": render_op, "render_op_graph": graph_replay(render_op, 3),
                "render_reference": render_ref, "panel_op": panel_op, "panel_reference": panel_ref}
        times = alternate(arms, a.iters, a.rounds, 3)
        rec["ms"] = {k: stats(v, 1e3, 3) for k, v in times.items()}
        rec["host_syncs_per_call"] = {k: host_syncs(arms[k]) for k in ("render_op", "panel_op")}
        result["sizes"][name] = rec
    emit(result, a.json)


if __name__ == "__main__":
    main()
