"""Generates tests/golden/regs.npz from the original ExAvatar_RELEASE's own regulariser code.

    python tests/golden/make_regs_golden.py /path/to/ExAvatar_RELEASE

`LaplacianReg`, `HandMeanReg`, `HandRGBReg`, `ArmRGBReg` and `JointOffsetSymmetricReg` (avatar/common/nets/loss.py) are
executed verbatim, class sources only (the module itself imports lpips and pytorch3d), and so is `SMPLX.get_arm`
(avatar/common/utils/smpl_x.py).  `.cuda()` is patched to the identity, `smpl_x` is a stub carrying the reference's
`joints_name`, and pytorch3d's `Meshes` is a shim over `geometry.vertex_normals_reference(flip=None)` in the vertices'
dtype.  The block of avatar/main/model.py:217-257 is executed from its source lines against a stub `self`, once with
cfg.is_warmup False and once True.

The inputs are not stored: `regs_inputs` rebuilds them from `make_human_mesh(rings=7, segments=12)` (1 346 vertices;
the poles keep 12 neighbours, so LaplacianReg truncates them to 10), `make_regs_labels` and seeded generators.
Every input is float64 (mesh_neutral_pose holds float32 values), so the golden pins the float64 restatement; the
restatement makes the arm split and selection in fp32, which agrees with the reference's float64 ones on this case.
`pin_kinks` puts exact zeros at abs's and clamp's kinks.  Stored: the ten term values, the warm-up's
gaussian_scale_reg, each input's gradient of the sum of the ten means (train.py:43-46) at seeded elements with its
absolute sum (the zero-offset hand row's mean_offset gradient on its own), the reference's SMPL-X joint names, the five
weight columns, and a digest of LaplacianReg's table on the synthetic C4 mesh (167 618 vertices, 108-neighbour poles) with its two pole rows.
"""
import ast
import hashlib
import math
import os
import sys
import textwrap
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from exavatar_release_b200.geometry import vertex_normals_reference  # noqa: E402
from exavatar_release_b200.synthetic import make_human_mesh, make_regs_labels  # noqa: E402

MESH = {"rings": 7, "segments": 12}
SAMPLES = 64
INPUTS = ("mean_offset", "mean_offset_offset", "scale_offset", "scale", "scale_refined", "rgb", "rgb_refined",
          "joint_offset", "scale_wo_clamp")
ARM_JOINTS = ("R_Shoulder", "R_Elbow", "L_Shoulder", "L_Elbow")


def joints_name(ref_root):
    src = open(os.path.join(ref_root, "avatar", "common", "utils", "smpl_x.py")).read()
    for node in ast.walk(ast.parse(src)):
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Attribute) and t.attr == "joints_name"
                                                for t in node.targets):
            return ast.literal_eval(node.value)
    raise RuntimeError("joints_name not found")


def table_digest(idx, w):
    return hashlib.sha256(np.ascontiguousarray(idx, dtype=np.int64).tobytes()
                          + np.ascontiguousarray(w, dtype=np.float32).tobytes()).hexdigest()


def pin_kinks(ins, labels, names):
    """Puts exact zeros where the backward has a kink, so that its one-sided choice is pinned against autograd:
    R_Elbow / L_Elbow get x_L = -x_R and y_L = y_R, so two of JointOffsetSymmetricReg's abs arguments are exactly 0
    (abs's gradient there is 0), and the first right-hand row gets a zero mean_offset, so HandMeanReg's dot product is
    exactly 0 (clamp(min=0) passes the gradient there, through F.normalize's eps branch: n / 1e-12).  Returns that
    row, whose mean_offset gradient is ~1e12 times the others' and is compared on its own."""
    jo = ins["joint_offset"]
    r, l = names.index("R_Elbow"), names.index("L_Elbow")
    jo[l, 0] = -jo[r, 0]
    jo[l, 1] = jo[r, 1]
    row = int(torch.nonzero(labels["is_rhand"])[0])
    ins["mean_offset"][..., row, :] = 0.0
    return row


def regs_inputs(names):
    """(mesh, labels, inputs, joint_target, hand_joints, sym_pairs): the golden case, from seeds only."""
    mesh = make_human_mesh(**MESH)
    labels = make_regs_labels(mesh)
    P = mesh["verts"].shape[0]
    J = len(names)
    g = torch.Generator().manual_seed(17)
    d = torch.float64
    ins = {"mean_offset": 1e-3 * torch.randn(1, P, 3, generator=g, dtype=d),
           "mean_offset_offset": 5e-4 * torch.randn(1, P, 3, generator=g, dtype=d),
           "scale_offset": 1e-2 * torch.randn(1, P, 1, generator=g, dtype=d),
           "scale": torch.exp(math.log(4e-3) + 0.3 * torch.randn(1, P, 3, generator=g, dtype=d)),
           "scale_refined": torch.exp(math.log(4e-3) + 0.3 * torch.randn(1, P, 3, generator=g, dtype=d)),
           "rgb": torch.rand(1, P, 3, generator=g, dtype=d),
           "rgb_refined": torch.rand(1, P, 3, generator=g, dtype=d),
           "joint_offset": 1e-2 * torch.randn(J, 3, generator=g, dtype=d),
           "scale_wo_clamp": torch.exp(math.log(4e-3) + 0.3 * torch.randn(1, P, 3, generator=g, dtype=d))}
    pin_kinks(ins, labels, names)
    target = 1e-2 * torch.randn(J, 3, generator=g, dtype=d)
    lh = [i for i, n in enumerate(names) if n.startswith("L_") and n[2:].split("_")[0] in
          ("Index", "Middle", "Pinky", "Ring", "Thumb")]
    rh = [i for i, n in enumerate(names) if n.startswith("R_") and n[2:].split("_")[0] in
          ("Index", "Middle", "Pinky", "Ring", "Thumb")]
    right = [j for j in range(J) if names[j][:2] == "R_"]
    left = [names.index("L_" + names[j][2:]) for j in right]
    return mesh, labels, ins, target, lh + rh, (right, left)


def main(ref_root):
    torch.Tensor.cuda = lambda self, *a, **k: self
    names = joints_name(ref_root)
    mesh, labels, ins, target, hand_joints, _ = regs_inputs(names)
    P = mesh["verts"].shape[0]
    faces = mesh["faces"].numpy()

    class Meshes:
        def __init__(self, verts, faces):
            self.v, self.f = verts[0], faces[0]

        def verts_normals_packed(self):
            return vertex_normals_reference(self.v, self.f, dtype=self.v.dtype)

    smpl_x = types.SimpleNamespace(face_upsampled=faces, vertex_num_upsampled=P, joint_num=len(names),
                                   joints_name=names, joint_offset=target,
                                   joint_part={"lhand": hand_joints[:len(hand_joints) // 2],
                                               "rhand": hand_joints[len(hand_joints) // 2:]})
    ns = {"torch": torch, "nn": torch.nn, "F": torch.nn.functional, "math": math, "np": np, "Meshes": Meshes,
          "smpl_x": smpl_x}
    path = os.path.join(ref_root, "avatar", "common", "nets", "loss.py")
    src = open(path).read()
    wanted = ("LaplacianReg", "HandMeanReg", "HandRGBReg", "ArmRGBReg", "JointOffsetSymmetricReg")
    for cls in (n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name in wanted):
        exec(compile(ast.get_source_segment(src, cls), path, "exec"), ns)
    spath = os.path.join(ref_root, "avatar", "common", "utils", "smpl_x.py")
    ssrc = open(spath).read()
    smplx_cls = next(n for n in ast.parse(ssrc).body if isinstance(n, ast.ClassDef) and n.name == "SMPLX")
    fn = next(n for n in smplx_cls.body if isinstance(n, ast.FunctionDef) and n.name == "get_arm")
    exec(compile(textwrap.dedent(ast.get_source_segment(ssrc, fn)), spath, "exec"), ns)
    smpl_x.get_arm = types.MethodType(ns["get_arm"], smpl_x)

    skinning_weight = torch.zeros(P, len(names))
    skinning_weight[:, 0] = 1.0
    skinning_weight[labels["is_arm"], 0] = 0.0
    skinning_weight[labels["is_arm"], names.index(ARM_JOINTS[0])] = 1.0
    joint_offset = ins["joint_offset"].clone().requires_grad_()
    hg = types.SimpleNamespace(skinning_weight=skinning_weight, joint_offset=joint_offset,
                               **{k: labels[k] for k in ("is_rhand", "is_lhand", "is_face", "is_face_expr",
                                                         "is_cavity")})
    lap_reg = ns["LaplacianReg"](P, faces)
    stub = types.SimpleNamespace(human_gaussian=hg, hand_mean_reg=ns["HandMeanReg"](), lap_reg=lap_reg,
                                 hand_rgb_reg=ns["HandRGBReg"](), arm_rgb_reg=ns["ArmRGBReg"](),
                                 joint_offset_sym_reg=ns["JointOffsetSymmetricReg"]())
    mpath = os.path.join(ref_root, "avatar", "main", "model.py")
    lines = open(mpath).read().split("\n")
    block = textwrap.dedent("\n".join(lines[216:257]))  # model.py:217-257
    weight_blocks = [(217, 221), (224, 228), (234, 236), (239, 242), (244, 246)]

    out = {}
    mesh_np = mesh["verts"].double()  # float64 like every input: the golden pins the float64 restatement
    for warm in (False, True):
        leaves = {k: v.clone().requires_grad_() for k, v in ins.items() if k != "joint_offset"}
        human_offsets = {k: leaves[k] for k in ("mean_offset", "mean_offset_offset", "scale_offset")}
        human_assets = {"scale": leaves["scale"], "rgb": leaves["rgb"], "scale_wo_clamp": leaves["scale_wo_clamp"]}
        human_assets_refined = {"scale": leaves["scale_refined"], "rgb": leaves["rgb_refined"]}
        joint_offset.grad = None
        env = dict(ns, self=stub, cfg=types.SimpleNamespace(is_warmup=warm), human_offsets=human_offsets,
                   human_assets=human_assets, human_assets_refined=human_assets_refined, mesh_neutral_pose=mesh_np,
                   loss={})
        exec(compile(block, mpath, "exec"), env)
        loss = env["loss"]
        if warm:
            out["warmup_gaussian_scale_reg"] = loss["gaussian_scale_reg"].mean().detach().numpy()
            loss["gaussian_scale_reg"].mean().backward()
            gr = leaves["scale_wo_clamp"].grad.reshape(-1)
            g = torch.Generator().manual_seed(5)
            idx = torch.randperm(gr.numel(), generator=g)[:SAMPLES]
            out.update({"grad_idx:scale_wo_clamp": idx.numpy(), "grad_val:scale_wo_clamp": gr[idx].numpy(),
                        "grad_abs:scale_wo_clamp": gr.abs().sum().numpy()})
            continue
        for k, v in loss.items():
            out[f"term:{k}"] = v.mean().detach().numpy()
        sum(v.mean() for v in loss.values()).backward()
        g = torch.Generator().manual_seed(5)
        row = int(torch.nonzero(labels["is_rhand"])[0])
        for k in INPUTS[:-1]:
            gr = (joint_offset if k == "joint_offset" else leaves[k]).grad.reshape(-1).clone()
            if k == "mean_offset":
                out["kink_grad:mean_offset"] = gr[3 * row:3 * row + 3].numpy().copy()
                gr[3 * row:3 * row + 3] = 0.0  # stored above; kept out of the samples and the abs sum
            nz = torch.nonzero(gr).reshape(-1)
            idx = torch.cat((nz[torch.randperm(nz.numel(), generator=g)[:SAMPLES]],
                             torch.randperm(gr.numel(), generator=g)[:SAMPLES])).unique()
            out.update({f"grad_idx:{k}": idx.numpy(), f"grad_val:{k}": gr[idx].numpy(),
                        f"grad_abs:{k}": gr.abs().sum().numpy()})
    weights = []
    for a, b in weight_blocks:
        env = dict(ns, self=stub, smpl_x=smpl_x)
        exec(compile(textwrap.dedent("\n".join(lines[a - 1:b])), mpath, "exec"), env)
        weights.append(env["weight"].reshape(-1).numpy())
    out["weights"] = np.stack(weights).astype(np.float32)
    out["joints_name"] = np.array(names)
    lower = smpl_x.get_arm(mesh_np, skinning_weight)[1]
    out["n_lower"] = np.array(int(lower.sum()))

    c4 = make_human_mesh()
    Pc = c4["verts"].shape[0]
    idx, w = (t.numpy() for t in ns["LaplacianReg"](Pc, c4["faces"].numpy()).get_neighbor(Pc, c4["faces"].numpy()))
    out["c4_table_sha256"] = np.array(table_digest(idx, w))
    deg = np.bincount(c4["faces"].numpy().reshape(-1), minlength=Pc)
    poles = np.nonzero(deg == deg.max())[0]  # the two poles: 108 faces each
    out["c4_pole_rows"] = poles
    out["c4_pole_idx"] = idx[poles]
    out["c4_pole_w"] = w[poles]
    np.savez_compressed(os.path.join(HERE, "regs.npz"), **out)
    print("wrote regs.npz", {k: float(v) for k, v in out.items() if k.startswith("term:")})


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
