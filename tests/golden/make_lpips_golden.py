"""Generates tests/golden/lpips.npz from the original ExAvatar_RELEASE's own LPIPS wrapper.

    python tests/golden/make_lpips_golden.py /path/to/ExAvatar_RELEASE

`LPIPS` (avatar/common/nets/loss.py:77-95) is executed verbatim, class source only (the module itself imports pytorch3d).
Its `lpips` import is a shim: `lpips.LPIPS(net='vgg')` is restated from the lpips package (version 0.1: ScalingLayer,
the vgg16 slices [0:4] [4:9] [9:16] [16:23] [23:30] of torchvision's own `vgg16().features`, normalize_tensor,
Dropout + 1x1 lin convs without bias, spatial means, summed), in eval mode as ExAvatar's `eval_modules` puts it, and in
float64.  `.cuda()` is patched to the identity.

Nothing but the results is stored.  `lpips_weights` builds the 13 convs and the 5 lin weights from integer arithmetic
(fp32 values, He-scaled), and the images are `make_loss_golden.loss_images` at 72 x 96, so the tests rebuild the same
inputs on any machine.  Each case stores the loss, and the image gradient at a seeded sample of elements with its
abs-sum and non-zero count.
"""
import ast
import importlib.util
import math
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))

SIZE = (72, 96)  # H, W
# (name, bbox or None): negative corners, past the edge, fractional (47 wide: every pool floors in x), a 37 x 53 crop,
# exactly 16 px, the whole image
LPIPS_CASES = [
    ("neg_xy", (-10.7, -5.3, 60.9, 50.4)),
    ("past_edge", (50.5, 30.2, 80.0, 70.0)),
    ("frac", (13.6, 7.9, 47.3, 41.8)),
    ("odd_37x53", (20.2, 15.9, 53.9, 37.99)),
    ("exact_16", (30.0, 20.0, 16.0, 16.9)),
    ("whole", None),
]
SAMPLES = 256
CHANNELS = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
TAP_CHANNELS = (64, 128, 256, 512, 512)


def _loss_golden():
    spec = importlib.util.spec_from_file_location("make_loss_golden", os.path.join(HERE, "make_loss_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def lpips_images():
    """(img, target) float32 (3,72,96) in [0,1], from integer arithmetic only."""
    img, target, _ = _loss_golden().loss_images(*SIZE)
    return img.float() / 255, target.float() / 255


def lpips_weights():
    """(features, lins): torchvision's `vgg16().features` with fp32 weights from integer arithmetic (uniform, He-scaled
    conv weights, small biases), and the five (1,C,1,1) non-negative lin weights."""
    import torchvision
    h = _loss_golden()._hash
    features = torchvision.models.vgg16(weights=None).features
    convs = [m for m in features if isinstance(m, nn.Conv2d)]
    with torch.no_grad():
        for k, m in enumerate(convs):
            co, ci = m.weight.shape[:2]
            i = torch.arange(m.weight.numel(), dtype=torch.int64).reshape(m.weight.shape)
            a = math.sqrt(6.0 / (9 * ci))
            m.weight.copy_(((h(i, torch.tensor(k), torch.tensor(1)) % 2001 - 1000).double() / 1000 * a).float())
            j = torch.arange(co, dtype=torch.int64)
            m.bias.copy_(((h(j, torch.tensor(k), torch.tensor(2)) % 201 - 100).double() / 2000).float())
        lins = []
        for t, c in enumerate(TAP_CHANNELS):
            j = torch.arange(c, dtype=torch.int64)
            lins.append(((h(j, torch.tensor(t), torch.tensor(3)) % 1000 + 1).double() / 16000).float().reshape(1, c, 1, 1))
    return features.eval(), lins


class _ScalingLayer(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer("shift", torch.tensor([-.030, -.088, -.188])[None, :, None, None])
        self.register_buffer("scale", torch.tensor([.458, .448, .450])[None, :, None, None])

    def forward(self, inp):
        return (inp - self.shift) / self.scale


class _NetLinLayer(nn.Module):
    def __init__(self, chn_in):
        super().__init__()
        self.model = nn.Sequential(nn.Dropout(), nn.Conv2d(chn_in, 1, 1, stride=1, padding=0, bias=False))

    def forward(self, x):
        return self.model(x)


class _Vgg16(nn.Module):
    def __init__(self, features):
        super().__init__()
        for k, (a, b) in enumerate(((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))):
            s = nn.Sequential()
            for x in range(a, b):
                s.add_module(str(x), features[x])
            setattr(self, f"slice{k + 1}", s)

    def forward(self, x):
        out = []
        for k in range(5):
            x = getattr(self, f"slice{k + 1}")(x)
            out.append(x)
        return out


class _LpipsShim(nn.Module):
    """lpips.LPIPS(net='vgg', version='0.1') restated, weights from `lpips_weights`, eval mode, float64."""

    def __init__(self, net="vgg"):
        super().__init__()
        assert net == "vgg"
        features, lins = lpips_weights()
        self.scaling_layer = _ScalingLayer()
        self.net = _Vgg16(features)
        for k, (c, w) in enumerate(zip(TAP_CHANNELS, lins)):
            lin = _NetLinLayer(c)
            with torch.no_grad():
                lin.model[-1].weight.copy_(w)
            setattr(self, f"lin{k}", lin)
        self.double().eval()

    def forward(self, in0, in1):
        outs0, outs1 = self.net(self.scaling_layer(in0)), self.net(self.scaling_layer(in1))
        val = 0
        for k in range(5):
            f0 = outs0[k] / (torch.sqrt(torch.sum(outs0[k] ** 2, dim=1, keepdim=True)) + 1e-10)
            f1 = outs1[k] / (torch.sqrt(torch.sum(outs1[k] ** 2, dim=1, keepdim=True)) + 1e-10)
            val = val + getattr(self, f"lin{k}")((f0 - f1) ** 2).mean([2, 3], keepdim=True)
        return val


def load_lpips_class(ref_root):
    nn.Module.cuda = lambda self, *a, **k: self
    path = os.path.join(ref_root, "avatar", "common", "nets", "loss.py")
    src = open(path).read()
    shim = type(sys)("lpips")
    shim.LPIPS = _LpipsShim
    ns = {"torch": torch, "nn": nn, "lpips": shim}
    for cls in (n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "LPIPS"):
        exec(compile(ast.get_source_segment(src, cls), path, "exec"), ns)
    return ns["LPIPS"]()


def main(ref_root):
    ref = load_lpips_class(ref_root)
    g = torch.Generator().manual_seed(17)
    img, target = lpips_images()
    out = {}
    for name, box in LPIPS_CASES:
        x = img.double()[None].requires_grad_()
        bbox = None if box is None else torch.tensor([box], dtype=torch.float32)
        loss = ref(x, target.double()[None], bbox)
        loss.sum().backward()
        grad = x.grad[0].reshape(-1)
        nz = torch.nonzero(grad).reshape(-1)
        idx = torch.cat((nz[torch.randperm(nz.numel(), generator=g)[:SAMPLES]],
                         torch.randperm(grad.numel(), generator=g)[:SAMPLES])).unique()
        out.update({f"{name}_loss": loss.detach().reshape(()).numpy(), f"{name}_grad_idx": idx.numpy().astype(np.int32),
                    f"{name}_grad_val": grad[idx].numpy(), f"{name}_grad_abs_sum": grad.abs().sum().numpy(),
                    f"{name}_grad_nonzero": np.array(nz.numel())})
        print(f"{name}: loss {float(loss.detach()):.10f}  nonzero grads {nz.numel()}")
    np.savez_compressed(os.path.join(HERE, "lpips.npz"), **out)
    print("wrote lpips.npz")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
