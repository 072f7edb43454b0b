"""The backward projection (K6, `b2r_backward_project`) row by row, through the C ABI: after one forward and one backward
composite of a small scene, K6 runs on the composite's scratch with every combination of output layout the kernel's
warp-staged row I/O has to get right -- a Gaussian count that is no multiple of 32 or 256, a detached prefix that
starts at row 0, inside a warp and on a 256-row block, write and accumulate, the densification statistics, each output
left out in turn and outputs that are not 16-byte aligned.  Every output lives inside a guard band: nothing outside
rows [0, P - first_row) may change.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from parity import compare
from util import workload_settings
from exavatar_release_b200.synthetic import WORKLOADS, make_assets, make_grad_image
from oracle import oracle as O

pytestmark = pytest.mark.gpu

WIDTHS = {"means3D": 3, "means2D": 3, "colors": 3, "opacities": 1, "scales": 3, "rotations": 4}
ORACLE_KEY = {"means3D": "means3D", "means2D": "means2D", "colors": "colors", "opacities": "opacities",
              "scales": "scales", "rotations": "rotations"}
P_ROWS = 3997  # no multiple of 32 or 256: the last warp and the last CTA are partial
GUARD = 37     # floats of guard band on either side of every output
SENTINEL = 1234.5


@pytest.fixture(scope="module")
def frame():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from exavatar_release_b200 import _lib as L
    from exavatar_release_b200 import rasterizer as rz
    from exavatar_release_b200.plan import FramePlan
    dev = torch.device("cuda:0")
    wl = WORKLOADS["T1"]
    assets = {k: v[:P_ROWS].contiguous() for k, v in make_assets("T1", seed=3).items()}
    st_c = workload_settings("T1", yaw=15.0, bg=(0.2, 0.6, 0.9))
    st_g = workload_settings("T1", yaw=15.0, bg=(0.2, 0.6, 0.9), device=dev, settings_cls=rz.GaussianRasterizationSettings)
    _, orad, _, _, octx = O.forward(st_c, assets["mean_3d"], assets["opacity"], scales=assets["scale"],
                                    rotations=assets["rotation"], colors_precomp=assets["rgb"])
    gi = make_grad_image("T1", 5)
    og = O.backward(octx, gi.numpy(), None, None)
    _, gm = O.fragility(octx)
    a = {k: v.to(dev) for k, v in assets.items()}
    plan = FramePlan(P_ROWS, wl.width, wl.height, 1_000_000, dev)
    sc = plan.scene(0, st_g, a)
    plan.forward(sc)
    g_color = gi.to(dev).contiguous()
    args = L.B2RBackwardArgs(g_color.data_ptr(), None, None)
    args.flags, args.first_row = 0, 0
    st = torch.cuda.current_stream(dev).cuda_stream
    L.check(plan.lib.b2r_backward_composite(C.byref(sc), C.byref(plan.ws), None, C.byref(args), plan.bwd_scratch.data_ptr(),
                                            plan.bwd_bytes, st), "b2r_backward_composite")
    torch.cuda.synchronize()
    radii = plan.radii.cpu().numpy()
    assert np.array_equal(radii, orad)
    return dict(L=L, plan=plan, sc=sc, dev=dev, og=og, gm=gm, radii=radii, keep=(a, g_color))


def _guarded(dev, rows, width, misalign, fill=None):
    """(buffer, view): a (rows, width) view inside a buffer with GUARD sentinel floats on both sides; `misalign` shifts the
    view by one float, so it is not 16-byte aligned."""
    off = GUARD + (1 if misalign else 0)
    buf = torch.full((off + rows * width + GUARD,), SENTINEL, dtype=torch.float32, device=dev)
    view = buf[off:off + rows * width].view(rows, width)
    if fill is not None:
        view.copy_(fill)
    return buf, view, off


def _run(fr, first_row, accumulate=False, skip=None, misalign=False, prior=None, densify=None, zero_scratch=False):
    L, plan, dev = fr["L"], fr["plan"], fr["dev"]
    rows = P_ROWS - first_row
    outs = {}
    for k, w in WIDTHS.items():
        if k == skip:
            continue
        outs[k] = _guarded(dev, rows, w, misalign, None if prior is None else prior[k])
    ptr = lambda k: outs[k][1].data_ptr() if k in outs else None
    a = L.B2RBackwardArgs(None, None, None, ptr("means3D"), ptr("means2D"), None, ptr("colors"), ptr("opacities"),
                          ptr("scales"), ptr("rotations"), None)
    a.flags = (L.B2R_BWD_ACCUMULATE if accumulate else 0) | (L.B2R_BWD_SCRATCH_ZEROED if zero_scratch else 0)
    a.first_row = first_row
    if densify is not None:
        a.densify_grad_accum, a.densify_count = densify["grad_accum"].data_ptr(), densify["count"].data_ptr()
        a.densify_radius_max = densify["radius_max"].data_ptr()
    st = torch.cuda.current_stream(dev).cuda_stream
    L.check(plan.lib.b2r_backward_project(C.byref(fr["sc"]), C.byref(plan.ws), C.byref(a), plan.bwd_scratch.data_ptr(),
                                          plan.bwd_bytes, st), "b2r_backward_project")
    torch.cuda.synchronize()
    for k, (buf, view, off) in outs.items():
        n = view.numel()
        assert torch.all(buf[:off] == SENTINEL) and torch.all(buf[off + n:] == SENTINEL), f"{k}: guard band written"
    return {k: v[1] for k, v in outs.items()}


FIRST_ROWS = [0, 16, 512, 1040]  # row 0, inside a warp, on a 256-row block, inside a warp of a later block


@pytest.mark.parametrize("first_row", FIRST_ROWS)
def test_rows_match_the_oracle(frame, first_row):
    out = _run(frame, first_row)
    gm = frame["gm"][first_row:]
    for k, t in out.items():
        y = np.asarray(frame["og"][ORACLE_KEY[k]], np.float64).reshape(P_ROWS, -1)[first_row:]
        x = t.cpu().numpy().reshape(y.shape)
        if np.abs(y).max() == 0:
            assert np.abs(x).max() <= 1e-6, k
            continue
        compare(f"k6_rows/first_row={first_row}", "d_" + k, x, y, np.broadcast_to(gm[:, None], y.shape))
    assert torch.all(out["means2D"][:, 2] == 0)
    culled = torch.from_numpy(frame["radii"][first_row:] <= 0).to(frame["dev"])
    for k, t in out.items():  # write mode: a culled Gaussian's rows are written, as zeros
        assert torch.all(t[culled] == 0), k


@pytest.mark.parametrize("first_row", FIRST_ROWS)
def test_accumulate_adds_the_fresh_gradient_exactly(frame, first_row):
    fresh = _run(frame, first_row)
    gen = torch.Generator(device=frame["dev"]).manual_seed(first_row)
    prior = {k: torch.rand(P_ROWS - first_row, w, generator=gen, device=frame["dev"]) + 0.5 for k, w in WIDTHS.items()}
    acc = _run(frame, first_row, accumulate=True, prior=prior)
    for k in WIDTHS:
        assert torch.equal(acc[k], prior[k] + fresh[k]), k


@pytest.mark.parametrize("skip", list(WIDTHS))
@pytest.mark.parametrize("accumulate", [False, True])
def test_each_output_can_be_left_out(frame, skip, accumulate):
    prior = {k: torch.full((P_ROWS - 16, w), 0.25, device=frame["dev"]) for k, w in WIDTHS.items()}
    full = _run(frame, 16, accumulate=accumulate, prior=prior)
    part = _run(frame, 16, accumulate=accumulate, prior=prior, skip=skip)
    assert skip not in part
    for k, t in part.items():
        assert torch.equal(t, full[k]), k


@pytest.mark.parametrize("first_row", [0, 16, 1040])
@pytest.mark.parametrize("accumulate", [False, True])
def test_unaligned_outputs(frame, first_row, accumulate):
    prior = {k: torch.full((P_ROWS - first_row, w), -0.75, device=frame["dev"]) for k, w in WIDTHS.items()}
    aligned = _run(frame, first_row, accumulate=accumulate, prior=prior)
    shifted = _run(frame, first_row, accumulate=accumulate, prior=prior, misalign=True)
    for k in WIDTHS:
        assert torch.equal(shifted[k], aligned[k]), k


@pytest.mark.parametrize("first_row", [0, 1040])
def test_densification_sums(frame, first_row):
    dev, rows = frame["dev"], P_ROWS - first_row
    gen = torch.Generator(device=dev).manual_seed(11)
    d0 = {"grad_accum": torch.rand(rows, generator=gen, device=dev), "count": torch.randint(0, 5, (rows,), generator=gen,
                                                                                           device=dev).float(),
          "radius_max": torch.randint(0, 9, (rows,), generator=gen, device=dev).float()}
    d = {k: v.clone() for k, v in d0.items()}
    out = _run(frame, first_row, accumulate=True, prior={k: torch.zeros(rows, w, device=dev) for k, w in WIDTHS.items()},
               densify=d)
    radii = torch.from_numpy(frame["radii"][first_row:]).to(dev)
    vis = radii > 0
    m2 = out["means2D"]
    norm = torch.sqrt(m2[:, 0] * m2[:, 0] + m2[:, 1] * m2[:, 1])
    assert torch.equal(d["count"], d0["count"] + vis.float())
    assert torch.equal(d["radius_max"], torch.where(vis, torch.maximum(d0["radius_max"], radii.float()), d0["radius_max"]))
    assert torch.equal(d["grad_accum"][~vis], d0["grad_accum"][~vis])
    torch.testing.assert_close(d["grad_accum"][vis], d0["grad_accum"][vis] + norm[vis], rtol=1e-6, atol=1e-7)


def test_scratch_is_left_zero(frame):
    """B2R_BWD_SCRATCH_ZEROED: the kernel clears every visible Gaussian's scratch row (run last: it consumes the
    scratch the other tests read)."""
    out = _run(frame, 0)
    again = _run(frame, 0, zero_scratch=True)
    for k in WIDTHS:
        assert torch.equal(again[k], out[k]), k
    assert torch.count_nonzero(frame["plan"].bwd_scratch) == 0
