"""Generates tests/golden/human_assets.npz from the original ExAvatar_RELEASE's own code.

    python tests/golden/make_human_assets_golden.py /path/to/ExAvatar_RELEASE

Executed from their source, in float64, against stub `self`s holding seeded leaves:
  * `SMPLXParamDict.forward` (avatar/common/nets/module.py) for one frame of 6D pose parameters;
  * the statements of `HumanGaussian.forward` from `geo_feat = ...` up to the nearest-vertex search (module.py:524-539)
    and from `rgb, rgb_refined = ...` through the asset dicts (:561-585), with the networks stubbed to return the
    seeded head outputs and `get_mean_offset_offset` running its own combining statements (:489-493) on a seeded
    pose offset;
  * `Model.forward`'s warm-up clamp (avatar/main/model.py:92-96), with cfg.is_warmup off and on.
pytorch3d's `rotation_6d_to_matrix`, `matrix_to_axis_angle` and `matrix_to_quaternion` are shims over
`exavatar_release_b200.smplx_rig`'s restatement, and `.cuda()` returns the tensor, so the fixture pins the reference's
module.py and model.py lines verbatim, not pytorch3d.

The inputs are not stored: `pose_case` and `geometry_case` rebuild them from seeds.  Stored (float64): `pose:out:<key>`
and `pose:grad:<key>` for the seven pose keys (a seeded weighted sum of the axis-angle outputs), and per warm-up flag w
`w{w}:out:<name>` for the assets and offsets and `w{w}:grad:<leaf>` for a seeded weighted sum of them.
"""
import ast
import math
import os
import sys
import textwrap
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from exavatar_release_b200 import smplx_rig as R  # noqa: E402

POSE_KEYS = ("root_pose", "body_pose", "jaw_pose", "leye_pose", "reye_pose", "lhand_pose", "rhand_pose")
POSE_ROWS = (1, 21, 1, 1, 1, 15, 15)
GEO_OUTPUTS = ("mean_3d", "mean_3d_refined", "scale", "scale_refined", "mean_offset_offset", "rgb", "rgb_refined")
WARMUP_OUTPUTS = ("scale_wo_clamp", "scale_refined_wo_clamp")
GEO_LEAVES = ("mesh", "geo", "geo_offset", "expr", "rgb", "rgb_offset")
P, NE = 200, 4


def _aa_6d(aa):
    return R.matrix_to_rotation_6d(R.axis_angle_to_matrix(aa))


def special_rows():
    """The 6D rows that exercise the conversion's branches, float64: the identity, 180-degree turns about x, y, z and
    about the diagonals (two equal q_abs), angles 1e-7, 1e-6 and 1e-3 (around the |angle| < 1e-6 branch), angles
    pi - 1e-3 and pi - 1e-6, and degenerate rows: a zero vector, a zero first column, parallel columns."""
    g = torch.Generator().manual_seed(7)
    d = torch.float64
    axis = lambda: (lambda v: v / v.norm())(torch.randn(3, generator=g, dtype=d))  # noqa: E731
    rows = [torch.tensor([1.0, 0, 0, 0, 1, 0], dtype=d), torch.tensor([1.0, 0, 0, 0, -1, 0], dtype=d),
            torch.tensor([-1.0, 0, 0, 0, 1, 0], dtype=d), torch.tensor([-1.0, 0, 0, 0, -1, 0], dtype=d),
            torch.tensor([0.0, 1, 0, 1, 0, 0], dtype=d), torch.tensor([0.0, 0, 1, 0, -1, 0], dtype=d)]
    for angle in (1e-7, 1e-6, 1e-3, math.pi - 1e-3, math.pi - 1e-6):
        rows.append(_aa_6d(angle * axis()))
    rows += [torch.zeros(6, dtype=d), torch.tensor([0.0, 0, 0, 0.3, -1.0, 2.0], dtype=d),
             torch.tensor([1.0, 0, 0, 2.0, 0, 0], dtype=d), torch.tensor([0.0, 3.0, 0, 0, -1.5, 0], dtype=d)]
    return torch.stack(rows)


def pose_case():
    """(params, weights), float64, from seeds only.  params: the seven 6D pose parameters of one frame as ExAvatar
    stores them -- (6,) for root / jaw / eyes, (n,6) otherwise -- plus expr (NE) and trans (3).  The root is a
    180-degree turn, jaw and eyes are exact identities, the body's rows start with special_rows() and the hands mix
    rotations of seeded axis-angles with raw (non-orthonormal) 6D rows.  weights: one (n,3) / (3,) factor per key."""
    g = torch.Generator().manual_seed(43)
    d = torch.float64
    sp = special_rows()
    body = torch.cat([sp, _aa_6d(0.5 * torch.randn(21 - len(sp), 3, generator=g, dtype=d))])
    hand = lambda: torch.cat([_aa_6d(0.4 * torch.randn(8, 3, generator=g, dtype=d)),  # noqa: E731
                              torch.randn(7, 6, generator=g, dtype=d)])
    eye = torch.tensor([1.0, 0, 0, 0, 1, 0], dtype=d)
    params = {"root_pose": sp[1].clone(), "body_pose": body, "jaw_pose": eye.clone(), "leye_pose": eye.clone(),
              "reye_pose": eye.clone(), "lhand_pose": hand(), "rhand_pose": hand(),
              "expr": torch.randn(NE, generator=g, dtype=d), "trans": torch.randn(3, generator=g, dtype=d)}
    w = {k: torch.randn(params[k].shape[:-1] + (3,), generator=g, dtype=d) for k in POSE_KEYS}
    return params, w


def geometry_case():
    """(inputs, weights), float64, from seeds only.  inputs: mesh (P,3), the unmasked pose offset (P,3), expr (NE) and
    expr_dirs (P,3,NE) (expr_offset = (expr * expr_dirs).sum(2), module.py:537), geo (P,4) with log-scales around
    log(0.001) so the warm-up clamp cuts some rows and not others, geo_offset (P,4), rgb and rgb_offset (P,3), the
    three (P,) 0/1 masks; NaN and inf in mean_offset_offset on two masked rows.  weights: one factor per output."""
    g = torch.Generator().manual_seed(47)
    d = torch.float64
    r = lambda *s: torch.randn(*s, generator=g, dtype=d)  # noqa: E731
    geo = torch.cat([0.01 * r(P, 3), -6.9 + 0.5 * r(P, 1)], 1)
    geo_offset = torch.cat([0.005 * r(P, 3), 0.3 * r(P, 1)], 1)
    is_rhand = torch.zeros(P, dtype=d)
    is_lhand = torch.zeros(P, dtype=d)
    is_face_expr = torch.zeros(P, dtype=d)
    is_rhand[10:30], is_lhand[25:50], is_face_expr[150:180] = 1, 1, 1
    geo_offset[12, 0], geo_offset[160, 2] = float("nan"), float("inf")
    inputs = {"mesh": r(P, 3), "pose_offset": 0.01 * r(P, 3), "expr": r(NE), "expr_dirs": 0.01 * r(P, 3, NE),
              "geo": geo, "geo_offset": geo_offset, "rgb": r(P, 3), "rgb_offset": 0.2 * r(P, 3),
              "is_rhand": is_rhand, "is_lhand": is_lhand, "is_face_expr": is_face_expr}
    names = GEO_OUTPUTS + WARMUP_OUTPUTS
    return inputs, {k: r(P, 3) for k in names}


def _method(path, cls_name, fn_name):
    src = open(path).read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == cls_name)
    return src, next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == fn_name)


def _statements(src, fn, first, stop):
    """Source of fn's top-level statements from the one whose text starts with `first` up to (not including) the one
    starting with `stop` (None: to the end)."""
    segs = [textwrap.dedent(ast.get_source_segment(src, n)) for n in fn.body]
    i = next(k for k, s in enumerate(segs) if s.startswith(first))
    j = next((k for k, s in enumerate(segs) if stop is not None and s.startswith(stop)), len(segs))
    return "\n".join(segs[i:j])


def _pose_golden(mpath, out):
    src, fn = _method(mpath, "SMPLXParamDict", "forward")
    ns = {"torch": torch, "rotation_6d_to_matrix": R.rotation_6d_to_matrix,
          "matrix_to_axis_angle": R.matrix_to_axis_angle}
    exec(compile(textwrap.dedent(ast.get_source_segment(src, fn)), mpath, "exec"), ns)
    params, w = pose_case()
    leaves = {k: v.clone().requires_grad_() for k, v in params.items()}
    self = types.SimpleNamespace(smplx_params={"0": leaves})
    res = ns["forward"](self, [0])[0]
    sum((res[k] * w[k]).sum() for k in POSE_KEYS).backward()
    for k in POSE_KEYS:
        out[f"pose:out:{k}"] = res[k].detach().numpy()
        out[f"pose:grad:{k}"] = leaves[k].grad.numpy()


def _geometry_golden(mpath, model_path, out):
    src, fwd = _method(mpath, "HumanGaussian", "forward")
    part1 = _statements(src, fwd, "geo_feat =", "nn_vertex_idxs =")
    part2 = _statements(src, fwd, "rgb, rgb_refined =", "return")
    msrc, mmo_fn = _method(mpath, "HumanGaussian", "get_mean_offset_offset")
    combine = "def combine(self, smplx_pose_offset, mean_offset_offset):\n" + textwrap.indent(
        _statements(msrc, mmo_fn, "mask =", None), "    ")
    model_src, model_fwd = _method(model_path, "Model", "forward")
    loop = next(n for n in ast.walk(model_fwd) if isinstance(n, ast.For))
    warm = "\n".join(textwrap.dedent(ast.get_source_segment(model_src, n)) for n in loop.body
                     if isinstance(n, ast.If) and "is_warmup" in ast.get_source_segment(model_src, n))
    ns = {"torch": torch, "matrix_to_quaternion": R.matrix_to_quaternion}
    exec(compile(combine, mpath, "exec"), ns)
    inputs, w = geometry_case()
    for warmup in (0, 1):
        lv = {k: inputs[k].clone().requires_grad_() for k in GEO_LEAVES}
        hg = types.SimpleNamespace(
            geo_net=lambda t: None, mean_offset_net=lambda f: lv["geo"][:, :3], scale_net=lambda f: lv["geo"][:, 3:],
            rgb_net=lambda t: lv["rgb"], forward_geo_network=lambda t, sp: (lv["geo_offset"][:, :3],
                                                                             lv["geo_offset"][:, 3:]),
            is_rhand=inputs["is_rhand"], is_lhand=inputs["is_lhand"], is_face_expr=inputs["is_face_expr"],
            expr_dirs=inputs["expr_dirs"])
        hg.get_mean_offset_offset = lambda sp, mmo: ns["combine"](hg, inputs["pose_offset"], mmo)
        loc = {"self": hg, "tri_feat": None, "mesh_neutral_pose": lv["mesh"], "smplx_param": {"expr": lv["expr"]},
               "rgb_offset": lv["rgb_offset"], "torch": torch, "smpl_x": types.SimpleNamespace(vertex_num_upsampled=P)}
        loc.update(ns)
        exec(compile(part1 + "\n" + part2, mpath, "exec"), loc)
        wl = {"human_asset": loc["assets"], "human_asset_refined": loc["assets_refined"], "mode": "train",
              "cfg": types.SimpleNamespace(is_warmup=bool(warmup)), "key_list": [], "torch": torch}
        exec(compile(warm, model_path, "exec"), wl)
        ha, har, offs = wl["human_asset"], wl["human_asset_refined"], loc["offsets"]
        res = {"mean_3d": ha["mean_3d"], "mean_3d_refined": har["mean_3d"], "scale": ha["scale"],
               "scale_refined": har["scale"], "mean_offset_offset": offs["mean_offset_offset"], "rgb": ha["rgb"],
               "rgb_refined": har["rgb"]}
        if warmup:
            res.update(scale_wo_clamp=ha["scale_wo_clamp"], scale_refined_wo_clamp=har["scale_wo_clamp"])
        fin = lambda t: torch.where(torch.isfinite(t), t, torch.zeros_like(t))  # noqa: E731
        sum((fin(res[k]) * w[k]).sum() for k in res).backward()
        for k, v in res.items():
            out[f"w{warmup}:out:{k}"] = v.detach().numpy()
        for k in GEO_LEAVES:
            out[f"w{warmup}:grad:{k}"] = lv[k].grad.numpy()
        out[f"w{warmup}:out:rotation"] = ha["rotation"].detach().double().numpy()
        out[f"w{warmup}:out:opacity"] = ha["opacity"].detach().double().numpy()


def main(ref_root):
    torch.set_default_dtype(torch.float64)
    torch.Tensor.cuda = lambda self, *a, **k: self  # the reference's constants are built with .cuda()
    mpath = os.path.join(ref_root, "avatar", "common", "nets", "module.py")
    model_path = os.path.join(ref_root, "avatar", "main", "model.py")
    out = {}
    _pose_golden(mpath, out)
    _geometry_golden(mpath, model_path, out)
    dst = os.path.join(HERE, "human_assets.npz")
    np.savez_compressed(dst, **out)
    print(f"wrote {dst}: " + ", ".join(f"{k} {v.shape}" for k, v in out.items()))


if __name__ == "__main__":
    main(sys.argv[1])
