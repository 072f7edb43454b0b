"""Generates tests/golden/human_nets.npz from the original ExAvatar_RELEASE's own network code.

    python tests/golden/make_human_nets_golden.py /path/to/ExAvatar_RELEASE

`make_linear_layers` (avatar/common/nets/layer.py) and `HumanGaussian.extract_tri_feature` /
`forward_geo_network`-style wiring (avatar/common/nets/module.py) are executed from their own source, extracted with
`ast` (the modules import pytorch3d).  Everything runs in float64 on the CPU.  The case: P rows of a synthetic
`pos_enc_mesh`, some of them outside the [-1, 1] square of a plane, a face subset, small (3,C,H,W) triplanes, the four
stacks with a 1-joint pose block (6 columns) in the middle of the concatenation and a normal block at the end.

Nothing but the results is stored: `case_inputs` rebuilds the positions, planes, pose, normals and every parameter
from integer arithmetic, so the tests rebuild identical float64 inputs on any machine.  Stored: tri_feat, the four
outputs, and the gradients of a fixed weighted sum of all outputs with respect to both triplanes and every parameter
(sampled, plus abs-sums).
"""
import ast
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
P, CH, PH, PW = 300, 4, 8, 12       # rows, triplane channels, plane height and width
POSE = 6                            # one joint's 6D rotation
SHAPE_3D, FACE_SHAPE_3D = (2.0, 2.0, 2.0), (0.3, 0.3, 0.3)
NETS = ("geo_net", "mean_offset_net", "scale_net", "geo_offset_net", "mean_offset_offset_net", "scale_offset_net",
        "rgb_net", "rgb_offset_net")
OUTPUTS = ("tri_feat", "geo", "geo_offset", "rgb", "rgb_offset")
SAMPLES = 64

_M32 = 0xFFFFFFFF


def _hash(*keys):
    """32-bit integer hash of broadcastable int64 tensors (every intermediate below 2**63: exact)."""
    h = torch.zeros((), dtype=torch.int64)
    for k, p in zip(keys, (0x9E3779B1, 0x85EBCA77, 0xC2B2AE3D)):
        h = (h ^ ((k * p) & _M32)) & _M32
        h = ((h ^ (h >> 15)) * 0x5BD1E995) & _M32
    return h ^ (h >> 13)


def _uniform(shape, salt, scale):
    """float64 values in [-scale, scale] on a grid of 1/1024 steps, from the hash of (element, salt)."""
    n = int(np.prod(shape)) if shape else 1
    i = torch.arange(n, dtype=torch.int64)
    return ((_hash(i, torch.tensor(salt)) % 2049 - 1024).double() / 1024 * scale).reshape(shape)


def layer_dims():
    """make_linear_layers arguments of the eight modules (HumanGaussian.__init__, module.py:280-287) at this size."""
    t = CH * 3
    return {"geo_net": ([t, 128, 128, 128], True), "mean_offset_net": ([128, 3], False),
            "scale_net": ([128, 1], False), "geo_offset_net": ([t + POSE, 128, 128, 128], True),
            "mean_offset_offset_net": ([128, 3], False), "scale_offset_net": ([128, 1], False),
            "rgb_net": ([t, 128, 128, 128, 3], False), "rgb_offset_net": ([t + POSE + 3, 128, 128, 128, 3], False)}


def set_parameters(nets):
    """Every parameter from integer arithmetic: weights ~ U(1/sqrt(fan_in)), GroupNorm gamma around 1."""
    for k, name in enumerate(NETS):
        for j, (pname, p) in enumerate(nets[name].named_parameters()):
            salt = 1000 * k + j
            with torch.no_grad():
                if p.dim() == 2:
                    p.copy_(_uniform(tuple(p.shape), salt, 1.0 / np.sqrt(p.shape[1])))
                elif "weight" in pname:  # GroupNorm gamma
                    p.copy_(1.0 + _uniform(tuple(p.shape), salt, 0.5))
                else:
                    p.copy_(_uniform(tuple(p.shape), salt, 0.2))


def case_inputs(dtype=torch.float64):
    """(pos_enc_mesh, is_face, triplane, triplane_face, pose6d, normal) of the case."""
    i = torch.arange(P, dtype=torch.int64)
    pos = torch.stack([(_hash(i, torch.tensor(a)) % 2001 - 1000).double() / 1000 * (1.3 if a < 2 else 0.9)
                       for a in range(3)], 1)                                    # some rows beyond |x| = 1
    is_face = (i % 5 == 2)
    pos[is_face] = pos[is_face] * 0.12 + 0.4                                     # a small head, off-centre
    tp = _uniform((3, CH, PH, PW), 77, 1.0)
    tpf = _uniform((3, CH, PH, PW), 78, 1.0)
    pose = _uniform((POSE,), 79, 1.0)
    n = torch.stack([_uniform((P,), 80 + a, 1.0) for a in range(3)], 1)
    n = n / n.norm(dim=1, keepdim=True)
    return pos.to(dtype), is_face, tp.to(dtype), tpf.to(dtype), pose.to(dtype), n.to(dtype)


def output_weights(name, shape):
    """The fixed weights of the scalar whose gradients are stored: sum over outputs of w * out."""
    return _uniform(shape, 500 + OUTPUTS.index(name), 1.0)


def load_reference(ref_root):
    """make_linear_layers and extract_tri_feature from the reference's own source."""
    ns = {"torch": torch, "nn": nn, "F": F, "np": np}
    path = os.path.join(ref_root, "avatar", "common", "nets", "layer.py")
    src = open(path).read()
    fn = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "make_linear_layers")
    exec(compile(ast.get_source_segment(src, fn), path, "exec"), ns)
    path = os.path.join(ref_root, "avatar", "common", "nets", "module.py")
    src = open(path).read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "HumanGaussian")
    meth = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "extract_tri_feature")
    ns["cfg"] = types.SimpleNamespace(triplane_shape_3d=SHAPE_3D, triplane_face_shape_3d=FACE_SHAPE_3D)
    exec(compile(ast.get_source_segment(src, meth), path, "exec"), ns)
    return ns["make_linear_layers"], ns["extract_tri_feature"]


def main(ref_root):
    make_linear_layers, extract_tri_feature = load_reference(ref_root)
    nets = {k: make_linear_layers(d, relu_final=r, use_gn=k in ("geo_net", "geo_offset_net", "rgb_net",
                                                                   "rgb_offset_net")).double()
            for k, (d, r) in layer_dims().items()}
    set_parameters(nets)
    pos, is_face, tp, tpf, pose, normal = case_inputs()
    tp.requires_grad_()
    tpf.requires_grad_()
    obj = types.SimpleNamespace(pos_enc_mesh=pos, is_face=is_face, triplane=tp, triplane_face=tpf)
    tri = extract_tri_feature(obj)
    # the wiring of HumanGaussian.forward / forward_geo_network / forward_rgb_network (module.py:460-586)
    posep = pose.view(1, POSE).repeat(P, 1)
    geo_feat = nets["geo_net"](tri)
    goff = nets["geo_offset_net"](torch.cat((tri, posep.detach()), 1))
    outs = {"tri_feat": tri,
            "geo": torch.cat((nets["mean_offset_net"](geo_feat), nets["scale_net"](geo_feat)), 1),
            "geo_offset": torch.cat((nets["mean_offset_offset_net"](goff), nets["scale_offset_net"](goff)), 1),
            "rgb": nets["rgb_net"](tri),
            "rgb_offset": nets["rgb_offset_net"](torch.cat((tri, posep.detach(), normal.detach()), 1))}
    loss = sum((output_weights(k, tuple(v.shape)) * v).sum() for k, v in outs.items())
    loss.backward()
    out = {f"out_{k}": v.detach().numpy() for k, v in outs.items()}
    grads = {"triplane": tp.grad, "triplane_face": tpf.grad}
    for name in NETS:
        for pname, p in nets[name].named_parameters():
            grads[f"{name}.{pname}"] = p.grad
    g = torch.Generator().manual_seed(5)
    for k, v in grads.items():
        flat = v.reshape(-1)
        idx = torch.randperm(flat.numel(), generator=g)[:SAMPLES].sort().values
        out[f"grad_idx:{k}"] = idx.numpy().astype(np.int32)
        out[f"grad_val:{k}"] = flat[idx].numpy()
        out[f"grad_abs:{k}"] = flat.abs().sum().numpy()
    np.savez_compressed(os.path.join(HERE, "human_nets.npz"), **out)
    print("wrote human_nets.npz")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
