"""SURVEY.md section 8f-2: `SkinnedGaussianRasterizer`, linear-blend skinning in front of the rasteriser.

The unfused path is ExAvatar's own sequence of PyTorch ops (`get_transform_mat_vertex`, `lbs`, camera->world:
avatar/common/nets/module.py:413-422, 555-557; restated op for op in `renderer.lbs_reference`) followed by the
rasteriser.  `SkinnedGaussianRasterizer` poses with the skinning op (`skinning.skin_gaussians`) and returns gradients
with respect to the canonical positions, the joint transforms and the root translation.  The two paths round the
posed positions differently (a (P,55)x(55,16) GEMM vs. a sparse in-register blend), so discrete per-(pixel, splat)
decisions that sit on a threshold may flip; the comparison therefore allows a small fraction of outliers, like the
oracle parity tests do.
"""
import math

import numpy as np
import pytest
import torch

from util import workload_settings  # noqa: F401  (path setup)
from exavatar_release_b200.camera import look_at_cam_param
from exavatar_release_b200.renderer import lbs_reference
from exavatar_release_b200.renderer import render_settings
from exavatar_release_b200.synthetic import make_grad_image, make_population_assets


def _rig(P, J, dtype, device, seed=5):
    g = torch.Generator().manual_seed(seed)
    w = torch.zeros(P, J)
    idx = torch.rand(P, J, generator=g).topk(4, dim=1).indices  # four distinct joints per Gaussian
    val = torch.rand(P, 4, generator=g) + 0.05
    w.scatter_(1, idx, val / val.sum(1, keepdim=True))  # four joints per Gaussian, weights sum to one
    ax = torch.randn(J, 3, generator=g)
    ax = ax / ax.norm(dim=1, keepdim=True)
    ang = 0.15 * torch.rand(J, generator=g)
    K = torch.zeros(J, 3, 3)
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 0], K[:, 1, 2], K[:, 2, 0], K[:, 2, 1] = -ax[:, 2], ax[:, 1], ax[:, 2], -ax[:, 0], -ax[:, 1], ax[:, 0]
    Rj = torch.eye(3)[None] + torch.sin(ang)[:, None, None] * K + (1 - torch.cos(ang))[:, None, None] * (K @ K)
    A = torch.eye(4)[None].repeat(J, 1, 1)
    A[:, :3, :3] = Rj
    A[:, :3, 3] = 0.02 * torch.randn(J, 3, generator=g)
    trans = torch.tensor([0.01, -0.02, 0.03])
    return w.to(device=device, dtype=dtype), A.to(device=device, dtype=dtype), trans.to(device=device, dtype=dtype)


def test_lbs_reference_is_the_blend_formula():
    """posed_i = (sum_j w_ij A_j) [x_i, 1] + trans, then world = R^-1 (posed - t): restated per element in float64."""
    P, J = 64, 55
    w, A, trans = _rig(P, J, torch.float64, "cpu")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(P, 3, generator=g, dtype=torch.float64)
    cam = look_at_cam_param(10.0, (96, 128))
    R, t = cam["R"].double(), cam["t"].double()
    got = lbs_reference(x, w, A, trans, R, t).numpy()
    Rinv = np.linalg.inv(R.numpy())
    for i in range(0, P, 7):
        M = sum(w[i, j].item() * A[j].numpy() for j in range(J))
        posed = M[:3, :3] @ x[i].numpy() + M[:3, 3] + trans.numpy()
        assert np.allclose(got[i], Rinv @ (posed - t.numpy()), atol=1e-12)


def _close(name, x, y, outliers=2e-3, rel=1e-4):
    d = (x - y).abs()
    lim = rel * float(y.abs().max()) + 1e-12
    frac = float((d > lim).float().mean())
    assert frac <= outliers, f"{name}: {frac:.2e} of the elements differ by more than {lim:.3e} (max {float(d.max()):.3e})"
    assert float(d.max()) <= 0.05 * float(y.abs().max()) + 1e-12, f"{name}: max difference {float(d.max()):.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("world", [True, False])
def test_fused_skinning_matches_the_unfused_path(world):
    from exavatar_release_b200 import rasterizer as RZ
    dev = torch.device("cuda:0")
    H, W = 96, 128
    _, human, _ = make_population_assets("T1", seed=0, device=dev)
    P, J = human["mean_3d"].shape[0], 55
    cam = look_at_cam_param(7.0, (H, W), device=dev)
    st = render_settings((H, W), cam, torch.tensor([0.2, 0.4, 0.9], device=dev))
    w, A, trans = _rig(P, J, torch.float32, dev)
    # canonical positions: where the synthetic avatar sits, expressed in the frame the skinning works in
    xyz0 = (human["mean_3d"] @ cam["R"].t() + cam["t"].view(1, 3)) if world else human["mean_3d"].clone()
    R, t = (cam["R"], cam["t"]) if world else (None, None)
    gi = make_grad_image("T1", 2).to(dev)

    def leaves():
        return {"xyz": xyz0.clone().requires_grad_(), "A": A.clone().requires_grad_(), "trans": trans.clone().requires_grad_(),
                "scale": human["scale"].clone().requires_grad_(), "rgb": human["rgb"].clone().requires_grad_(),
                "opacity": human["opacity"].clone().requires_grad_()}

    a = leaves()
    posed_a = lbs_reference(a["xyz"], w, a["A"], a["trans"], R, t)
    m2a = torch.zeros(P, 3, device=dev, requires_grad=True)
    img_a, rad_a, _, _ = RZ.GaussianRasterizer(st)(means3D=posed_a, means2D=m2a, opacities=a["opacity"], colors_precomp=a["rgb"],
                                                  scales=a["scale"], rotations=human["rotation"])
    (img_a * gi).sum().backward()

    b = leaves()
    m2b = torch.zeros(P, 3, device=dev, requires_grad=True)
    img_b, rad_b, _, _, posed_b = RZ.SkinnedGaussianRasterizer(st)(b["xyz"], w, b["A"], b["trans"], R, t, m2b, b["opacity"],
                                                                  b["rgb"], b["scale"], human["rotation"])
    (img_b * gi).sum().backward()
    torch.cuda.synchronize()

    assert float((posed_a.detach() - posed_b).abs().max()) < 5e-6
    assert float((rad_a != rad_b).float().mean()) < 2e-3 and int((rad_a > 0).sum()) > P // 2
    _close("image", img_b.detach(), img_a.detach())
    for k in ("xyz", "A", "trans", "scale", "rgb", "opacity"):
        assert a[k].grad is not None and float(a[k].grad.abs().max()) > 0, k
        _close(k, b[k].grad, a[k].grad)
    _close("means2D", m2b.grad, m2a.grad)
    assert float(a["A"].grad[:, 3, :].abs().max()) == 0.0 and float(b["A"].grad[:, 3, :].abs().max()) == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("only_posed", [False, True])
def test_posed_positions_of_the_fused_path_are_differentiable(only_posed):
    """ExAvatar reads the posed mean_3d outside the rasteriser too (face_mesh_renderer, avatar/main/model.py:172-173; the
    cat(scene.detach(), human) renders, model.py:117-125).  A loss that touches `posed` must reach xyz, the joint
    transforms and the translation through SkinnedGaussianRasterizer exactly as through the unfused ops -- for Gaussians
    the render culled as well, and also when the image is not used at all."""
    from exavatar_release_b200 import rasterizer as RZ
    dev = torch.device("cuda:0")
    H, W = 96, 128
    _, human, _ = make_population_assets("T1", seed=0, device=dev)
    P, J = human["mean_3d"].shape[0], 55
    cam = look_at_cam_param(7.0, (H, W), device=dev)
    st = render_settings((H, W), cam, torch.tensor([0.2, 0.4, 0.9], device=dev))
    w, A, trans = _rig(P, J, torch.float32, dev)
    xyz0 = human["mean_3d"] @ cam["R"].t() + cam["t"].view(1, 3)
    xyz0[:50, 2] -= 100.0  # behind the camera after posing: culled by the render, still read by the second loss term
    gi = make_grad_image("T1", 2).to(dev)
    gp = torch.randn(P, 3, generator=torch.Generator().manual_seed(3)).to(dev)

    def leaves():
        return {"xyz": xyz0.clone().requires_grad_(), "A": A.clone().requires_grad_(), "trans": trans.clone().requires_grad_()}

    def loss_of(img, posed):
        extra = (posed * gp).sum()
        return extra if only_posed else (img * gi).sum() + extra

    a = leaves()
    posed_a = lbs_reference(a["xyz"], w, a["A"], a["trans"], cam["R"], cam["t"])
    img_a = RZ.GaussianRasterizer(st)(means3D=posed_a, means2D=torch.zeros(P, 3, device=dev), opacities=human["opacity"],
                                      colors_precomp=human["rgb"], scales=human["scale"], rotations=human["rotation"])[0]
    loss_of(img_a, posed_a).backward()
    b = leaves()
    img_b, rad_b, _, _, posed_b = RZ.SkinnedGaussianRasterizer(st)(b["xyz"], w, b["A"], b["trans"], cam["R"], cam["t"],
                                                                  torch.zeros(P, 3, device=dev), human["opacity"],
                                                                  human["rgb"], human["scale"], human["rotation"])
    assert posed_b.requires_grad
    loss_of(img_b, posed_b).backward()
    torch.cuda.synchronize()
    assert int((rad_b[:50] == 0).sum()) == 50 and int((rad_b > 0).sum()) > P // 2
    for k in ("xyz", "A", "trans"):
        assert float(a[k].grad.abs().max()) > 0, k
        _close(k, b[k].grad, a[k].grad)
    assert float(b["xyz"].grad[:50].abs().max()) > 0  # the culled Gaussians received the posed-position gradient


def test_host_helpers_of_the_skinning_backward():
    """`_inv3` (graph-capturable 3x3 inverse) against torch.inverse."""
    from exavatar_release_b200.camera import _inv3
    g = torch.Generator().manual_seed(11)
    for _ in range(5):
        R = torch.randn(3, 3, generator=g, dtype=torch.float64) + 2 * torch.eye(3, dtype=torch.float64)
        assert torch.allclose(_inv3(R), torch.inverse(R), rtol=1e-10, atol=1e-12)
