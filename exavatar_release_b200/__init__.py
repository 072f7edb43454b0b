"""exavatar_release_b200 -- H100-native (sm_90a) differentiable Gaussian rasteriser for ExAvatar's render path.

Public surface (mirrors what /root/reference/avatar/common/nets/module.py:11 imports):
    GaussianRasterizationSettings, GaussianRasterizer
plus the host-side mirror of the caller (`GaussianRenderer`, module.py:588-647), `device_render_settings` (its render
settings computed on the device from a CUDA camera, no host read), `TrainingFrameRenderer` (the five
renders of a training frame, avatar/main/model.py:117-162, as one autograd call), `skin_gaussians` (both human sets
posed by one rig), `l1_ssim` (the L1 + SSIM terms of the loss block, model.py:196-215), `nearest_rows` and
`VertexNormals` (the nearest-vertex rows and mesh normals in front of the posing, module.py:501-504,541-546),
`FaceMeshRenderer` (the textured face render, model.py:170-175), `ShadedMeshRenderer` (the animation scripts' shaded
SMPL-X mesh panel, utils/vis.py:73-109), `HumanRegularizers` (the regulariser block,
model.py:217-257), `SmplxRig` (the SMPL-X rig of HumanGaussian.forward, module.py:517-518,533,537,549, and with
`.body_mesh` the frame's body mesh of get_smplx_outputs, model.py:37-58), `Adam` (ExAvatar's optimizer
step in one launch, base.py:83-85), `LPIPS` (the LPIPS-VGG terms, model.py:199,206), `NeumanScores` (the test-set
PSNR / SSIM / LPIPS-AlexNet of tools/eval_neuman.py), `face_composite` and `test_outputs` (the face composite of the
rgb_face terms, model.py:200-201,207-208, and the test-time composites and image bytes, model.py:268-276 and
main/test.py), `OrbitCamera`, `orbit_points` and `animation_panel` (the orbit camera, the recentred avatar and the
three-panel video frame of the animation scripts, animate.py and animate_view_rot.py), `scene_assets` (the scene
Gaussians' asset dict of SceneGaussian.forward, module.py:253-272), `decode_smplx_pose` (SMPLXParamDict.forward,
module.py:673-684), `SmplxParamTable` (every frame's SMPL-X parameters in one table, the frame picked on the device),
`IterationGraph` (a whole training iteration, forward, backward and Adam, as one CUDA graph per key for every frame),
`FrameTable` (every training frame's image, mask, box and camera on the device, the frame picked by the same slot),
`HumanAssets` (HumanGaussian's geometry and colour code around its networks, module.py:524-539,561-565
and model.py:92-96), synthetic workloads and the frame-sharding helper used by bench.py.
"""
from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer, rasterize_gaussians  # noqa: F401
from .renderer import GaussianRenderer, device_render_settings, render_settings  # noqa: F401
from .skinning import skin_gaussians  # noqa: F401
from .losses import l1_ssim  # noqa: F401
from .geometry import VertexNormals, nearest_rows  # noqa: F401
from .mesh_render import FaceMeshRenderer, ShadedMeshRenderer  # noqa: F401
from .regularizers import HumanRegularizers  # noqa: F401
from .smplx_rig import SmplxRig, cat_full_pose  # noqa: F401
from .optim import Adam  # noqa: F401
from .scene_assets import scene_assets  # noqa: F401
from .perceptual import LPIPS  # noqa: F401
from .metrics import NeumanScores  # noqa: F401
from .compose import face_composite, test_outputs  # noqa: F401
from .animation import OrbitCamera, animation_panel, orbit_points  # noqa: F401
from .human_assets import HumanAssets, SmplxParamTable, decode_smplx_pose  # noqa: F401
from .iteration import IterationGraph  # noqa: F401
from .frames import FrameTable  # noqa: F401


def __getattr__(name):  # TrainingFrameRenderer pulls in the plan machinery; loaded on first use
    if name == "TrainingFrameRenderer":
        from .fused import TrainingFrameRenderer
        return TrainingFrameRenderer
    raise AttributeError(name)


__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians", "GaussianRenderer",
           "render_settings", "device_render_settings", "TrainingFrameRenderer", "skin_gaussians", "l1_ssim", "nearest_rows", "VertexNormals",
           "FaceMeshRenderer", "ShadedMeshRenderer", "HumanRegularizers", "SmplxRig", "cat_full_pose", "Adam",
           "scene_assets", "LPIPS", "NeumanScores", "face_composite", "test_outputs", "OrbitCamera", "orbit_points", "animation_panel",
           "decode_smplx_pose", "SmplxParamTable", "HumanAssets", "IterationGraph", "FrameTable"]
