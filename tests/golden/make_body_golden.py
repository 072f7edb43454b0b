"""Generates tests/golden/body.npz from the original ExAvatar_RELEASE's own `Model.get_smplx_outputs`.

    python tests/golden/make_body_golden.py /path/to/ExAvatar_RELEASE

The synthetic SMPL-X model file and the golden mesh are make_rig_golden.py's (`rig_case`, `write_model_file`: 86 base
vertices, SMPL-X's 55-joint tree, non-zero hand means).  The vendored `smplx` package's `SMPLX` is instantiated from
that file with ExAvatar's `layer_arg`, in float64, and `Model.get_smplx_outputs` (avatar/main/model.py) is executed from
its source against a stub `self` (the layer and a `human_gaussian` holding shape_param and joint_offset) and a stub
`smpl_x` (joint_part, expr_param_dim, face_offset).  `.cuda()` is the identity and every tensor is float64.

The inputs are not stored: `body_case` rebuilds them from seeds.  The joint_offset has a non-zero root row (the call
passes it raw, without get_joint_offset) and the camera is a non-identity rotation with a translation.  Stored
(float64): the world mesh (`out:world`), the camera-space mesh (`out:camera`, the same call with R = I, t = 0) and the
gradients of a seeded weighted sum of both with respect to shape_param, joint_offset, the (55,3) pose in
`cat_full_pose` order, expr and trans.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import make_rig_golden as RG  # noqa: E402

GRADS = ("shape_param", "joint_offset", "full_pose", "expr", "trans")


def body_case():
    """(mesh, model, inputs, camera, weights) from seeds: make_rig_golden's model and pose keys, shape_param (100),
    joint_offset (55,3) with a root row of a few cm, the seven pose entries, expr (50), trans (3); camera {R, t};
    weights of the world and camera-space meshes (V,3) each."""
    mesh, model, _, _ = RG.rig_case()
    V = model["v_template"].shape[0]
    g = torch.Generator().manual_seed(41)
    d = torch.float64
    ins = {"shape_param": torch.randn(100, generator=g, dtype=d),
           "joint_offset": 0.01 * torch.randn(55, 3, generator=g, dtype=d)}
    ins["joint_offset"][0] = torch.tensor([0.03, -0.02, 0.05], dtype=d)
    for k, n in RG.POSE_KEYS:
        ins[k] = 0.4 * torch.randn(n, 3, generator=g, dtype=d)
    ins["expr"] = torch.randn(50, generator=g, dtype=d)
    ins["trans"] = torch.tensor([0.1, -0.2, 3.0], dtype=d) + 0.05 * torch.randn(3, generator=g, dtype=d)
    a = torch.tensor([0.3, -0.5, 0.2], dtype=d)
    th = a.norm()
    k = a / th
    K = torch.tensor([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]], dtype=d)
    R = torch.eye(3, dtype=d) + torch.sin(th) * K + (1 - torch.cos(th)) * K @ K
    cam = {"R": R, "t": torch.tensor([0.2, 0.1, -0.4], dtype=d)}
    w = [torch.randn(V, 3, generator=g, dtype=d) for _ in range(2)]
    return mesh, model, ins, cam, w


def full_pose(ins):
    return RG.full_pose(ins)


def main(ref_root):
    torch.set_default_dtype(torch.float64)
    torch.Tensor.cuda = lambda self, *a, **k: self
    sys.path.insert(0, os.path.join(ref_root, "avatar", "common", "utils", "smplx"))
    import smplx  # the reference's vendored copy

    _, model, ins, cam, w = body_case()
    V = model["v_template"].shape[0]
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "smplx"))
        RG.write_model_file(model, os.path.join(tmp, "smplx", "SMPLX_NEUTRAL.npz"))
        layer_arg = {"create_global_orient": False, "create_body_pose": False, "create_left_hand_pose": False,
                     "create_right_hand_pose": False, "create_jaw_pose": False, "create_leye_pose": False,
                     "create_reye_pose": False, "create_betas": False, "create_expression": False,
                     "create_transl": False}
        layer = smplx.create(tmp, "smplx", gender="neutral", num_betas=100, num_expression_coeffs=50, use_pca=False,
                             use_face_contour=True, dtype=torch.float64, **layer_arg)
    ej = layer.vertex_joint_selector.extra_joints_idxs
    layer.vertex_joint_selector.extra_joints_idxs = ej % V  # real SMPL-X vertex ids onto the small mesh: joints only

    mpath = os.path.join(ref_root, "avatar", "main", "model.py")
    smpl_x = types.SimpleNamespace(
        expr_param_dim=50, face_offset=model["face_offset"].double(),
        joint_part={"body": range(0, 22), "face": range(22, 25), "lhand": range(25, 40), "rhand": range(40, 55)})
    ns = {"torch": torch, "smpl_x": smpl_x}
    exec(compile(RG._method(mpath, "Model", "get_smplx_outputs"), mpath, "exec"), ns)
    hg = types.SimpleNamespace(shape_param=ins["shape_param"].clone().requires_grad_(),
                               joint_offset=ins["joint_offset"].clone().requires_grad_())
    this = types.SimpleNamespace(smplx_layer=layer, human_gaussian=hg)
    smplx_param = {k: ins[k].clone().requires_grad_() for k, _ in RG.POSE_KEYS}
    smplx_param["expr"] = ins["expr"].clone().requires_grad_()
    smplx_param["trans"] = ins["trans"].clone().requires_grad_()
    world = ns["get_smplx_outputs"](this, smplx_param, cam)
    camera = ns["get_smplx_outputs"](this, smplx_param, {"R": torch.eye(3), "t": torch.zeros(3)})
    ((world * w[0]).sum() + (camera * w[1]).sum()).backward()
    grads = [hg.shape_param.grad, hg.joint_offset.grad,
             torch.cat([smplx_param[k].grad.reshape(-1, 3) for k, _ in RG.POSE_KEYS]), smplx_param["expr"].grad,
             smplx_param["trans"].grad]
    out = {"out:world": world.detach().numpy(), "out:camera": camera.detach().numpy()}
    out.update({f"grad:{k}": v.detach().numpy() for k, v in zip(GRADS, grads)})
    dst = os.path.join(HERE, "body.npz")
    np.savez_compressed(dst, **out)
    print(f"wrote {dst}: " + ", ".join(f"{k} {v.shape}" for k, v in out.items()))


if __name__ == "__main__":
    main(sys.argv[1])
