"""Generates tests/golden/scene.npz from the original ExAvatar_RELEASE's own scene-asset code.

    python tests/golden/make_scene_golden.py /path/to/ExAvatar_RELEASE

`SceneGaussian.forward` (avatar/common/nets/module.py) and `eval_sh` with its C0..C4 tables
(avatar/common/utils/transforms.py) are executed from their source, in float64, against a stub `self` holding the
seeded parameters as leaves and the float `active_sh_degree` buffer, once per degree 0..3.  pytorch3d's
`rotation_6d_to_matrix` and `matrix_to_quaternion` are shims over `exavatar_release_b200.smplx_rig`'s restatement, so
the fixture pins the reference's module.py and eval_sh lines verbatim, not pytorch3d.

The inputs are not stored: `scene_case` rebuilds them from seeds.  Stored (float64), per degree d: the outputs
`d{d}:out:<opacity|scale|rotation|rgb>` and the gradients `d{d}:grad:<mean|opacity|scale|rotation|feature_dc|
feature_rest>` of a seeded weighted sum of the four outputs (zeros where autograd gives None: the mean at degree 0).
"""
import ast
import os
import sys
import textwrap
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from exavatar_release_b200 import smplx_rig as R  # noqa: E402

OUTPUTS = ("opacity", "scale", "rotation", "rgb")
PARAMS = ("mean", "opacity", "scale", "rotation", "feature_dc", "feature_rest")  # SceneGaussian's attribute names
P, M = 96, 16


def scene_case():
    """(params, cam_param, weights), float64, from seeds only.  params maps SceneGaussian's attribute names to (P,3)
    mean, (P,1) opacity logit, (P,3) log scale, (P,6) 6D rotation, (P,1,3) feature_dc and (P,15,3) feature_rest.  Rows
    0..3 of the rotation are the identity and 180-degree turns about x, y and z; the camera is a seeded rotation and
    translation looking at the points.  weights hold the loss's (P,1), (P,3), (P,4), (P,3) factors."""
    g = torch.Generator().manual_seed(41)
    d = torch.float64
    rot = torch.randn(P, 6, generator=g, dtype=d)
    rot[0] = torch.tensor([1.0, 0, 0, 0, 1, 0])
    rot[1] = torch.tensor([1.0, 0, 0, 0, -1, 0])   # 180 degrees about x
    rot[2] = torch.tensor([-1.0, 0, 0, 0, 1, 0])   # about y
    rot[3] = torch.tensor([-1.0, 0, 0, 0, -1, 0])  # about z
    params = {"mean": torch.randn(P, 3, generator=g, dtype=d),
              "opacity": 2 * torch.randn(P, 1, generator=g, dtype=d),
              "scale": -4 + torch.randn(P, 3, generator=g, dtype=d),
              "rotation": rot,
              "feature_dc": torch.randn(P, 1, 3, generator=g, dtype=d),
              "feature_rest": 0.3 * torch.randn(P, M - 1, 3, generator=g, dtype=d)}
    cam = {"R": R.axis_angle_to_matrix(0.5 * torch.randn(3, generator=g, dtype=d)),
           "t": torch.tensor([0.1, -0.2, 4.0], dtype=d) + 0.1 * torch.randn(3, generator=g, dtype=d)}
    w = [torch.randn(s, generator=g, dtype=d) for s in ((P, 1), (P, 3), (P, 4), (P, 3))]
    return params, cam, w


def _method(path, cls_name, fn_name):
    src = open(path).read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == cls_name)
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == fn_name)
    return textwrap.dedent(ast.get_source_segment(src, fn))


def _module_level(path, names):
    """Source of the top-level assignments and functions of `path` named in `names`, in file order."""
    src = open(path).read()
    out = []
    for n in ast.parse(src).body:
        if isinstance(n, ast.Assign) and any(isinstance(t, ast.Name) and t.id in names for t in n.targets):
            out.append(ast.get_source_segment(src, n))
        elif isinstance(n, ast.FunctionDef) and n.name in names:
            out.append(ast.get_source_segment(src, n))
    return "\n\n".join(out)


def main(ref_root):
    torch.set_default_dtype(torch.float64)
    tpath = os.path.join(ref_root, "avatar", "common", "utils", "transforms.py")
    mpath = os.path.join(ref_root, "avatar", "common", "nets", "module.py")
    ns = {"torch": torch, "F": torch.nn.functional, "rotation_6d_to_matrix": R.rotation_6d_to_matrix,
          "matrix_to_quaternion": R.matrix_to_quaternion}
    exec(compile(_module_level(tpath, {"C0", "C1", "C2", "C3", "C4", "eval_sh"}), tpath, "exec"), ns)
    exec(compile(_method(mpath, "SceneGaussian", "forward"), mpath, "exec"), ns)
    params, cam, w = scene_case()
    out = {}
    for deg in range(4):
        leaves = {k: v.clone().requires_grad_() for k, v in params.items()}
        self = types.SimpleNamespace(**leaves, active_sh_degree=torch.tensor([float(deg)]))
        res = ns["forward"](self, cam)
        loss = sum((res[k] * wk).sum() for k, wk in zip(OUTPUTS, w))
        loss.backward()
        for k in OUTPUTS:
            out[f"d{deg}:out:{k}"] = res[k].detach().numpy()
        for k in PARAMS:
            g = leaves[k].grad  # None for the mean at degree 0: eval_sh does not read the direction there
            out[f"d{deg}:grad:{k}"] = (torch.zeros_like(leaves[k]) if g is None else g).detach().numpy()
    dst = os.path.join(HERE, "scene.npz")
    np.savez_compressed(dst, **out)
    print(f"wrote {dst}: " + ", ".join(f"{k} {v.shape}" for k, v in out.items() if k.startswith("d0")))


if __name__ == "__main__":
    main(sys.argv[1])
