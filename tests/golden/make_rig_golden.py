"""Generates tests/golden/rig.npz from the original ExAvatar_RELEASE's own SMPL-X rig code.

    python tests/golden/make_rig_golden.py /path/to/ExAvatar_RELEASE

A small synthetic SMPL-X model file is written from seeds (`make_smplx_model` on `make_human_mesh(rings=7,
segments=12)`: 86 base vertices, 1 346 after two subdivisions, SMPL-X's 55-joint tree) with the 15 keys the reference's
`SMPLX` reads (v_template, f, shapedirs with the expression columns at 300:350, posedirs, J_regressor, kintree_table,
weights, the hands' components and means -- the means become pose_mean -- and the static and dynamic landmark tables).
The vendored `smplx` package's `SMPLX` is instantiated from that file with ExAvatar's `layer_arg` (avatar/common/utils/
smpl_x.py), in float64; its extra-joint vertex ids (real SMPL-X vertex numbers) are remapped onto the small mesh, which
changes only joints ExAvatar discards.  `HumanGaussian.get_neutral_pose_human`, `get_zero_pose_human`,
`get_transform_mat_joint`, `get_mean_offset_offset`, the pose lines of `forward_geo_network` and the expression line of
`forward` (avatar/common/nets/module.py) are executed from their source against a stub `self` and a stub `smpl_x`
whose `get_joint_offset` is the reference's own method; `pose_dirs` / `expr_dirs` are built by init's lines 297-298 and
305-306.  `.cuda()` is the identity and `.float()` gives float64, so every tensor is float64.  pytorch3d's
`axis_angle_to_matrix`, `matrix_to_axis_angle`, `matrix_to_rotation_6d` and the subdivision of `smpl_x.upsample_mesh`
are shims over `exavatar_release_b200.smplx_rig`'s restatement: the fixture pins the reference's SMPL-X layer, `lbs`
and module.py lines verbatim, not pytorch3d.

The inputs are not stored: `rig_case` rebuilds them from seeds.  Stored (float64): the six outputs and the gradients
of a seeded weighted sum of mesh_neutral_pose, joint_mats and expr_offset with respect to shape_param, joint_offset,
the (55,3) pose in `cat_full_pose` order, and expr.
"""
import ast
import os
import sys
import tempfile
import textwrap
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from exavatar_release_b200 import smplx_rig as R  # noqa: E402
from exavatar_release_b200.synthetic import make_human_mesh, make_smplx_model  # noqa: E402

MESH = {"rings": 7, "segments": 12}
POSE_KEYS = (("root_pose", 1), ("body_pose", 21), ("jaw_pose", 1), ("leye_pose", 1), ("reye_pose", 1),
             ("lhand_pose", 15), ("rhand_pose", 15))
OUTPUTS = ("mesh_neutral_pose", "mesh_neutral_pose_wo_upsample", "joint_mats", "pose_offset", "expr_offset", "pose_6d")
GRADS = ("shape_param", "joint_offset", "full_pose", "expr")


def rig_case():
    """(mesh, model, inputs, weights): the golden case, from seeds only.  inputs hold float64 shape_param (100),
    joint_offset (55,3), the seven pose entries of smplx_param and expr (50); weights the loss's (P,3), (55,4,4),
    (P,3)."""
    mesh = make_human_mesh(**MESH)
    model = make_smplx_model(mesh)
    P = mesh["verts"].shape[0]
    g = torch.Generator().manual_seed(23)
    d = torch.float64
    ins = {"shape_param": torch.randn(100, generator=g, dtype=d),
           "joint_offset": 0.01 * torch.randn(55, 3, generator=g, dtype=d)}
    for k, n in POSE_KEYS:
        ins[k] = 0.4 * torch.randn(n, 3, generator=g, dtype=d)
    ins["expr"] = torch.randn(50, generator=g, dtype=d)
    w = [torch.randn(s, generator=g, dtype=d) for s in ((P, 3), (55, 4, 4), (P, 3))]
    return mesh, model, ins, w


def full_pose(ins):
    return torch.cat([ins[k].reshape(-1, 3) for k, _ in POSE_KEYS])


def write_model_file(model, path):
    V = model["v_template"].shape[0]
    J = len(model["parents"])
    g = np.random.default_rng(31)
    f = model["faces"].numpy()
    sd = np.zeros((V, 3, 400))
    sd[:, :, :100] = model["shapedirs"].numpy()
    sd[:, :, 300:350] = model["expr_dirs"].numpy()
    bary = lambda *s: (lambda b: b / b.sum(-1, keepdims=True))(g.uniform(0.1, 1.0, s + (3,)))  # noqa: E731
    pm = model["pose_mean"].numpy()
    np.savez(path, v_template=model["v_template"].numpy(), f=f.astype(np.uint32), shapedirs=sd,
             posedirs=model["posedirs"].numpy().T.reshape(V, 3, -1),
             J_regressor=model["J_regressor"].numpy(), weights=model["lbs_weights"].numpy(),
             kintree_table=np.stack([model["parents"].numpy(), np.arange(J)]).astype(np.int64),
             hands_componentsl=np.eye(45), hands_componentsr=np.eye(45),
             hands_meanl=pm[75:120], hands_meanr=pm[120:165],
             lmk_faces_idx=g.integers(0, len(f), 51), lmk_bary_coords=bary(51),
             dynamic_lmk_faces_idx=g.integers(0, len(f), (79, 17)), dynamic_lmk_bary_coords=bary(79, 17))


def _method(path, cls_name, fn_name):
    src = open(path).read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == cls_name)
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == fn_name)
    return textwrap.dedent(ast.get_source_segment(src, fn))


def main(ref_root):
    torch.set_default_dtype(torch.float64)
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.Tensor.float = lambda self, *a, **k: self.double()
    sys.path.insert(0, os.path.join(ref_root, "avatar", "common", "utils", "smplx"))
    import smplx  # the reference's vendored copy
    from smplx.lbs import batch_rigid_transform

    mesh, model, ins, w = rig_case()
    m = R.validate_model(**model)
    V, P, J = m["V"], m["P"], m["J"]
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "smplx"))
        path = os.path.join(tmp, "smplx", "SMPLX_NEUTRAL.npz")
        write_model_file(model, path)
        layer_arg = {"create_global_orient": False, "create_body_pose": False, "create_left_hand_pose": False,
                     "create_right_hand_pose": False, "create_jaw_pose": False, "create_leye_pose": False,
                     "create_reye_pose": False, "create_betas": False, "create_expression": False,
                     "create_transl": False}
        layer = smplx.create(tmp, "smplx", gender="neutral", num_betas=100, num_expression_coeffs=50, use_pca=False,
                             use_face_contour=True, dtype=torch.float64, **layer_arg)
    ej = layer.vertex_joint_selector.extra_joints_idxs
    layer.vertex_joint_selector.extra_joints_idxs = ej % V

    def upsample_mesh(self, vert, feat_list=None):  # pytorch3d SubdivideMeshes twice, as a shim
        if feat_list is None:
            return R.upsample(vert, m["sub1"], m["sub2"])
        return (R.upsample(vert, m["sub1"], m["sub2"]), *[R.upsample(x, m["sub1"], m["sub2"]) for x in feat_list])

    spath = os.path.join(ref_root, "avatar", "common", "utils", "smpl_x.py")
    mpath = os.path.join(ref_root, "avatar", "common", "nets", "module.py")
    ns = {"torch": torch, "np": np, "axis_angle_to_matrix": R.axis_angle_to_matrix,
          "matrix_to_axis_angle": R.matrix_to_axis_angle, "matrix_to_rotation_6d": R.matrix_to_rotation_6d,
          "batch_rigid_transform": batch_rigid_transform}
    exec(compile(_method(spath, "SMPLX", "get_joint_offset"), spath, "exec"), ns)
    smpl_x = types.SimpleNamespace(
        joint_num=J, root_joint_idx=0, vertex_num=V, vertex_num_upsampled=P, shape_param_dim=100, expr_param_dim=50,
        joint_part={"body": range(0, 22), "face": range(22, 25), "lhand": range(25, 40), "rhand": range(40, 55)},
        neutral_body_pose=model["neutral_body_pose"].double(), neutral_jaw_pose=torch.tensor([1 / 3, 0.0, 0.0]),
        face_offset=model["face_offset"].double())
    smpl_x.get_joint_offset = types.MethodType(ns["get_joint_offset"], smpl_x)
    smpl_x.upsample_mesh = types.MethodType(upsample_mesh, smpl_x)
    ns["smpl_x"] = smpl_x
    for fn in ("get_neutral_pose_human", "get_zero_pose_human", "get_transform_mat_joint", "get_mean_offset_offset"):
        exec(compile(_method(mpath, "HumanGaussian", fn), mpath, "exec"), ns)

    lines = open(mpath).read().split("\n")
    run = lambda a, b, env: exec(compile(textwrap.dedent("\n".join(lines[a - 1:b])), mpath, "exec"), env)  # noqa: E731
    hg = types.SimpleNamespace(smplx_layer=layer, shape_param=ins["shape_param"].clone().requires_grad_(),
                               joint_offset=ins["joint_offset"].clone().requires_grad_(),
                               is_rhand=model["is_rhand"], is_lhand=model["is_lhand"],
                               is_face_expr=model["is_face_expr"])
    env = dict(ns, self=hg)
    run(297, 298, env)  # init: the base pose_dirs / expr_dirs views
    _, pd, ed = smpl_x.upsample_mesh(torch.ones((V, 3)), [env["pose_dirs"], env["expr_dirs"]])
    env.update(pose_dirs=pd, expr_dirs=ed)
    run(305, 306, env)  # init: the upsampled tables' layout
    hg.pose_dirs, hg.expr_dirs = env["pose_dirs"], env["expr_dirs"]
    for fn in ("get_neutral_pose_human", "get_zero_pose_human", "get_transform_mat_joint", "get_mean_offset_offset"):
        setattr(hg, fn, types.MethodType(ns[fn], hg))

    smplx_param = {k: ins[k].clone().requires_grad_() for k, _ in POSE_KEYS}
    smplx_param["expr"] = ins["expr"].clone().requires_grad_()
    smplx_param["trans"] = torch.zeros(3)
    mesh_neutral_pose, mesh_wo, _, transform_mat_neutral_pose = hg.get_neutral_pose_human(jaw_zero_pose=True,
                                                                                         use_id_info=True)
    joint_zero_pose = hg.get_zero_pose_human()
    joint_mats = hg.get_transform_mat_joint(transform_mat_neutral_pose, joint_zero_pose, smplx_param)
    pose_offset, _ = hg.get_mean_offset_offset(smplx_param, torch.zeros((P, 3)))
    env = dict(ns, self=hg, smplx_param=smplx_param)
    run(537, 537, env)  # smplx_expr_offset
    run(461, 461, env)  # forward_geo_network: body_pose
    run(464, 464, env)  # forward_geo_network: the 6D pose, repeated per row
    outs = [mesh_neutral_pose, mesh_wo, joint_mats, pose_offset, env["smplx_expr_offset"], env["pose"][0]]
    loss = (outs[0] * w[0]).sum() + (outs[2] * w[1]).sum() + (outs[4] * w[2]).sum()
    loss.backward()
    grads = [hg.shape_param.grad, hg.joint_offset.grad,
             torch.cat([smplx_param[k].grad.reshape(-1, 3) for k, _ in POSE_KEYS]), smplx_param["expr"].grad]
    out = {f"out:{k}": v.detach().numpy() for k, v in zip(OUTPUTS, outs)}
    out.update({f"grad:{k}": v.detach().numpy() for k, v in zip(GRADS, grads)})
    dst = os.path.join(HERE, "rig.npz")
    np.savez_compressed(dst, **out)
    print(f"wrote {dst}: " + ", ".join(f"{k} {v.shape}" for k, v in out.items()))


if __name__ == "__main__":
    main(sys.argv[1])
