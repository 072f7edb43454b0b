"""Python surface of the drop-in (no GPU needed): names, settings tuple, validation, alias packages, no CPU fallback,
and this package's `GaussianRenderer` against what the original ExAvatar `GaussianRenderer.forward` source computed
with the same rasteriser behind it (tests/golden/renderer.npz)."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from exavatar_release_b200 import GaussianRasterizationSettings, GaussianRasterizer
from util import kat_settings, pack, splat

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "renderer.npz")


def test_settings_tuple_matches_call_site():
    # field names and order of module.py:609-622
    assert GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix", "projmatrix", "sh_degree",
        "campos", "prefiltered", "debug")
    st = kat_settings(settings_cls=GaussianRasterizationSettings)
    assert isinstance(st, tuple) and st.image_height == 32 and st.debug is False


def test_alias_packages_resolve_to_the_same_classes():
    import diff_gaussian_rasterization as vanilla
    import diff_gaussian_rasterization_depth as depth
    assert depth.GaussianRasterizer is GaussianRasterizer and vanilla.GaussianRasterizer is GaussianRasterizer
    assert depth.GaussianRasterizationSettings is GaussianRasterizationSettings


def test_argument_validation_same_messages_as_upstream():
    st = kat_settings(settings_cls=GaussianRasterizationSettings)
    a = pack([splat((0, 0, 2.0))])
    m2 = torch.zeros(1, 3)
    r = GaussianRasterizer(raster_settings=st)
    with pytest.raises(Exception, match="Please provide excatly one of either SHs or precomputed colors!"):
        r(means3D=a["means3D"], means2D=m2, opacities=a["opacities"], scales=a["scales"], rotations=a["rotations"])
    with pytest.raises(Exception, match="Please provide excatly one of either SHs or precomputed colors!"):
        r(means3D=a["means3D"], means2D=m2, opacities=a["opacities"], shs=torch.zeros(1, 16, 3),
          colors_precomp=a["colors_precomp"], scales=a["scales"], rotations=a["rotations"])
    with pytest.raises(Exception, match="exactly one of either scale/rotation pair or precomputed 3D covariance"):
        r(means3D=a["means3D"], means2D=m2, opacities=a["opacities"], colors_precomp=a["colors_precomp"])
    with pytest.raises(Exception, match="exactly one of either scale/rotation pair or precomputed 3D covariance"):
        r(means3D=a["means3D"], means2D=m2, opacities=a["opacities"], colors_precomp=a["colors_precomp"],
          scales=a["scales"], rotations=a["rotations"], cov3D_precomp=torch.zeros(1, 6))


def test_product_path_has_no_cpu_fallback():
    st = kat_settings(settings_cls=GaussianRasterizationSettings)
    a = pack([splat((0, 0, 2.0))])
    r = GaussianRasterizer(raster_settings=st)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        r(means3D=a["means3D"], means2D=torch.zeros(1, 3), opacities=a["opacities"], colors_precomp=a["colors_precomp"],
          scales=a["scales"], rotations=a["rotations"])


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "exavatar_release_b200")
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(root, f)).read()
                assert "import oracle" not in src and "from oracle" not in src and "gs_oracle" not in src, f


def test_missing_library_raises(monkeypatch):
    from exavatar_release_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libb200raster.so")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _lib.load()


def test_reference_renderer_outputs_match_golden():
    """The original `GaussianRenderer` class source, executed verbatim with the CPU oracle as its rasteriser
    (tests/golden/make_golden.py), left its inputs, outputs and gradients in the fixture; this package's renderer with the
    same rasteriser must reproduce them bit for bit."""
    from exavatar_release_b200.renderer import GaussianRenderer
    from oracle import oracle as O

    z = np.load(GOLDEN)
    assets = {k: torch.from_numpy(z["asset_" + k]).requires_grad_() for k in ("mean_3d", "scale", "rotation", "opacity", "rgb")}
    cam = {k: torch.from_numpy(z["cam_" + k]) for k in ("R", "t", "focal", "princpt")}
    mine = GaussianRenderer(rasterizer_cls=O.OracleRasterizer, settings_cls=O.OracleSettings)
    out = mine(assets, (int(z["H"]), int(z["W"])), cam, torch.from_numpy(z["bg"]))
    for k in ("img", "depthmap", "mask", "radius", "is_vis"):
        assert np.array_equal(out[k].detach().numpy(), z[k]), k
    out["img"].sum().backward()
    assert np.array_equal(out["mean_2d"].grad.numpy(), z["grad_mean_2d"])
    assert np.array_equal(assets["mean_3d"].grad.numpy(), z["grad_mean_3d"])
