"""Import-compatible alias: `from diff_gaussian_rasterization_depth import GaussianRasterizationSettings,
GaussianRasterizer` (ExAvatar's avatar/common/nets/module.py:11) resolves to this package's rasteriser."""
from exavatar_release_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer,  # noqa: F401
                                              rasterize_gaussians)
