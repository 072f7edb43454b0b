"""Shared helpers for the test-suite."""
from __future__ import annotations

import contextlib
import importlib.util
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
HEADER = os.path.join(ROOT, "include", "b200raster.h")
GOLDEN = os.path.join(ROOT, "tests", "golden")

from exavatar_release_b200.camera import look_at_cam_param  # noqa: E402
from exavatar_release_b200.renderer import render_settings  # noqa: E402
from exavatar_release_b200.synthetic import WORKLOADS, make_assets, make_grad_image  # noqa: E402
from benchkit import capture  # noqa: E402,F401 -- the one warm-up-then-capture protocol, shared with the tools
from oracle.oracle import OracleSettings  # noqa: E402


@pytest.fixture(scope="module")
def dev():
    """cuda:0, or a skip without a CUDA device.  Import it (`from util import dev  # noqa: F401`): one per module."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


@contextlib.contextmanager
def no_host_sync():
    """Any host synchronisation inside the block raises (torch's sync debug mode "error").  The device is synchronised
    before and after, and the mode that was set before is restored."""
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        yield
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()


def golden_generator(name):
    """tests/golden/<name>.py as a module: the generator of a golden file, whose functions restate the reference."""
    spec = importlib.util.spec_from_file_location(name, os.path.join(GOLDEN, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def assert_close(a, b, rel, name):
    """max|a - b| <= rel * max|b| (floored at 1e-30), in float64; an empty tensor passes.  Prints the measured error."""
    a, b = torch.as_tensor(a).detach().double(), torch.as_tensor(b).detach().double()
    if b.numel() == 0:
        return
    err = float((a - b).abs().max())
    scale = max(float(b.abs().max()), 1e-30)
    print(f"{name}: max|d| = {err:.3e}  rel {err / scale:.3e}  (limit {rel:.0e})")
    assert err <= rel * scale, f"{name}: max|d| = {err:.3e} > {rel:.1e} * {scale:.3e}"


def kat_settings(W=32, H=32, f=32.0, bg=(0.0, 0.0, 0.0), R=None, t=None, device="cpu", settings_cls=OracleSettings):
    """App. B camera: R = I, t = 0, fx = fy = f (tanfov = W / 2f)."""
    cam = {
        "R": torch.eye(3) if R is None else R,
        "t": torch.zeros(3) if t is None else t,
        "focal": torch.tensor([f, f], dtype=torch.float32),
        "princpt": torch.tensor([W / 2.0, H / 2.0], dtype=torch.float32),
    }
    cam = {k: v.to(device) for k, v in cam.items()}
    return render_settings((H, W), cam, torch.tensor(bg, dtype=torch.float32, device=device), settings_cls)


def workload_settings(name, yaw=0.0, bg=(1.0, 1.0, 1.0), device="cpu", settings_cls=OracleSettings):
    wl = WORKLOADS[name]
    cam = look_at_cam_param(yaw, (wl.height, wl.width), device=device)
    return render_settings((wl.height, wl.width), cam, torch.tensor(bg, dtype=torch.float32, device=device), settings_cls)


def splat(p, scale=0.1, q=(1.0, 0.0, 0.0, 0.0), o=0.5, rgb=(1.0, 0.0, 0.0)):
    s = (scale, scale, scale) if np.isscalar(scale) else scale
    return dict(p=p, s=s, q=q, o=o, rgb=rgb)


def pack(splats, device="cpu", dtype=torch.float32):
    t = lambda k, n: torch.tensor([list(s[k]) if n > 1 else [s[k]] for s in splats], dtype=dtype, device=device).reshape(-1, n)
    return dict(means3D=t("p", 3), scales=t("s", 3), rotations=t("q", 4), opacities=t("o", 1), colors_precomp=t("rgb", 3))


def rel_err(x, y, floor):
    """max |x-y| / max(|y|, floor)  (SURVEY section 8c tolerance form)."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    if x.size == 0:
        return 0.0
    return float(np.max(np.abs(x - y) / np.maximum(np.abs(y), floor)))


def settings_on(st, device, settings_cls):
    """The SAME settings (bit for bit) with their tensors on `device`, as another settings class.  Camera matrices built
    on different devices can differ in the last bit (atan / tan / inverse / mm), which flips radius and tile-rect
    decisions for a few of 10^5 Gaussians; parity tests therefore build them once (CPU) and hand both paths the same bits."""
    import torch
    d = st._asdict()
    for k, v in d.items():
        if isinstance(v, torch.Tensor):
            d[k] = v.to(device)
    return settings_cls(**d)


def _header_source():
    """include/b200raster.h without its comments."""
    with open(HEADER) as f:
        return re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)


def header_structs():
    """{name: field names in declaration order} of every typedef'd struct of the header.  A declaration may name several
    fields (`int32_t P, J, reserved[2]`); the type, a nested struct's included, and array sizes are dropped."""
    return {name: [re.findall(r"\w+", re.sub(r"\[.*?\]", "", d))[-1]
                   for decl in body.split(";") if decl.strip() for d in decl.split(",")]
            for name, body in re.findall(r"typedef struct (\w+) \{(.*?)\} \1;", _header_source(), re.S)}


def header_symbols():
    """The b2r_* functions the header declares, sorted."""
    return sorted(set(re.findall(r"\b(b2r_\w+)\s*\(", _header_source())))


def header_defines():
    """{name: value as written} of the header's #defines."""
    return dict(re.findall(r"^#define[ \t]+(\w+)[ \t]*(.*?)[ \t]*$", _header_source(), re.M))
