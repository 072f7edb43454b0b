"""The C-ABI shared library: loads without a GPU, exports every symbol include/b200raster.h declares, struct layouts
agree with the ctypes mirror, argument validation returns the documented codes before any CUDA call."""
import ctypes as C
import os

import pytest

from util import header_structs, header_symbols
from exavatar_release_b200 import _lib as L


def test_library_exports_every_declared_symbol():
    lib = C.CDLL(L.LIB_PATH)
    names = header_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in b200raster.h but not exported"
    # and the binding knows all of them
    bound = {s[0] for s in L.SYMBOLS}
    assert set(names) <= bound, set(names) - bound


def test_struct_layouts_and_version():
    """Every ctypes mirror against the header's typedef and the library's b2r_sizeof: size, field names in order, and
    one mirror per index the library reports, without a device."""
    lib = L.load()
    assert lib.b2r_abi_version() == 4 == L.ABI_VERSION
    mirrors = [c for c in vars(L).values() if isinstance(c, type) and issubclass(c, C.Structure) and hasattr(c, "ID")]
    structs = header_structs()
    for cls in mirrors:
        assert lib.b2r_sizeof(cls.ID) == C.sizeof(cls), cls.__name__
        assert [n for n, _ in cls._fields_] == structs[cls.__name__], cls.__name__
    ids = sorted(c.ID for c in mirrors)
    assert len(set(ids)) == len(ids), ids
    assert ids == [i for i in range(64) if lib.b2r_sizeof(i)]
    assert lib.b2r_sizeof(7) == lib.b2r_sizeof(9) == lib.b2r_sizeof(30) == lib.b2r_sizeof(99) == 0
    assert sorted(c.__name__ for c in mirrors) == sorted(structs)  # and every struct of the header has a mirror
    assert C.sizeof(L.B2RStatus) == 64


def test_status_block_decodes_every_field():
    import torch
    s = L.B2RStatus(num_dups=7, dup_capacity=9, overflow=1, num_visible=5, consumed_fwd=80, consumed_bwd=40, token=3)
    ctx = torch.tensor(list(bytes(s)) + [0xAB] * 64, dtype=torch.uint8)  # the rest of a ctx buffer follows the block
    assert L.read_status(ctx) == {"num_dups": 7, "dup_capacity": 9, "overflow": 1, "num_visible": 5, "consumed_fwd": 80,
                                  "consumed_bwd": 40, "consumed_fwd_div": float(L.CONSUMED_FWD_DIV),
                                  "consumed_bwd_div": float(L.CONSUMED_BWD_DIV)}


def test_size_queries():
    lib = L.load()
    a = lib.b2r_ctx_bytes(1000, 64, 64)
    b = lib.b2r_ctx_bytes(2000, 64, 64)
    c = lib.b2r_ctx_bytes(1000, 128, 128)
    assert 0 < a < b and a < c and a % 256 == 0
    assert lib.b2r_scratch_bytes(1000, 64, 64, 0) >= 8
    assert lib.b2r_scratch_bytes(1000, 64, 64, 1 << 20) >= 8 << 20
    assert lib.b2r_backward_scratch_bytes(1000) >= 48000
    assert lib.b2r_ctx_bytes(0, 16, 16) > 0
    # checkpoint store: a segment table + 6 KB per 512-entry cut; grows with the duplicate capacity and the tile count
    c0 = lib.b2r_checkpoint_bytes(64, 64, 0)
    c1 = lib.b2r_checkpoint_bytes(64, 64, 1 << 20)
    assert 0 < c0 < c1 and c1 >= (1 << 20) // 512 * 6144
    assert lib.b2r_checkpoint_bytes(512, 512, 0) > c0


def test_error_codes_without_touching_cuda():
    lib = L.load()
    assert lib.b2r_strerror(0) == b"ok"
    assert b"invalid" in lib.b2r_strerror(-1)
    assert b"workspace" in lib.b2r_strerror(-2)
    sc = L.B2RScene()
    ws = L.B2RWorkspace()
    out = L.B2RForwardOutputs()
    # null scene / zero-sized image
    assert lib.b2r_forward(None, C.byref(ws), C.byref(out), None) == -1
    sc.P, sc.width, sc.height = 10, 0, 32
    assert lib.b2r_forward(C.byref(sc), C.byref(ws), C.byref(out), None) == -1
    sc.width, sc.tanfovx, sc.tanfovy = 32, 0.5, 0.5
    assert lib.b2r_forward(C.byref(sc), C.byref(ws), C.byref(out), None) == -1  # matrices missing
    fake = 0x1000  # never dereferenced on the host
    sc.bg = sc.viewmatrix = sc.projmatrix = sc.campos = fake
    sc.means3D = sc.opacities = fake
    assert lib.b2r_forward(C.byref(sc), C.byref(ws), C.byref(out), None) == -1  # neither shs nor colours
    sc.colors_precomp = fake
    sc.shs = fake
    assert lib.b2r_forward(C.byref(sc), C.byref(ws), C.byref(out), None) == -1  # both
    sc.shs = None
    assert lib.b2r_forward(C.byref(sc), C.byref(ws), C.byref(out), None) == -1  # no covariance source
    sc.scales = sc.rotations = fake
    assert lib.b2r_forward(C.byref(sc), C.byref(ws), C.byref(out), None) == -1  # ctx missing
    ws.ctx, ws.ctx_bytes = fake, 16
    assert lib.b2r_forward(C.byref(sc), C.byref(ws), C.byref(out), None) == -2  # ctx too small
    assert lib.b2r_mark_visible(-1, None, None, None, None) == -1
    assert lib.b2r_launch_count() == 0  # nothing was launched by any of the above


def test_kernel_names():
    lib = L.load()
    names = [lib.b2r_kernel_name(i).decode() for i in range(9)]
    assert names[0] == "project" and names[5] == "composite_fwd" and names[6] == "composite_bwd"
    assert lib.b2r_kernel_name(99) == b"?"


def test_error_codes_of_the_round1_additions_without_touching_cuda():
    """Validation of means3D, the detached prefix, the SH row limit and the id width happens on the host before any
    launch, so it is testable without a GPU."""
    lib = L.load()
    fake = 0x1000
    sc = L.B2RScene()
    sc.P, sc.width, sc.height, sc.tanfovx, sc.tanfovy = 10, 32, 32, 0.5, 0.5
    sc.bg = sc.viewmatrix = sc.projmatrix = sc.campos = fake
    sc.opacities = sc.colors_precomp = sc.scales = sc.rotations = fake
    ws = L.B2RWorkspace()
    ws.ctx, ws.ctx_bytes = fake, 16  # too small on purpose: a scene that validates reaches the workspace check (-2)
    out = L.B2RForwardOutputs()
    fwd = lambda: lib.b2r_forward(C.byref(sc), C.byref(ws), C.byref(out), None)
    assert fwd() == -1                      # no means3D
    sc.means3D = fake
    assert fwd() == -2
    # SH rows are staged through shared memory: at most 16 coefficients, degree <= 3, enough coefficients for the degree
    sc.colors_precomp = None
    sc.shs = fake
    sc.sh_degree, sc.sh_coeffs = 3, 16
    assert fwd() == -2
    sc.sh_coeffs = 9
    assert fwd() == -1
    sc.sh_degree, sc.sh_coeffs = 1, 17
    assert fwd() == -1
    sc.sh_degree, sc.sh_coeffs = 4, 25
    assert fwd() == -1
    sc.shs, sc.colors_precomp, sc.sh_degree, sc.sh_coeffs = None, fake, 0, 0
    # the splat record carries the Gaussian id in 29 bits
    sc.P = 1 << 29
    assert fwd() == -1
    sc.P = 10
    # backward: colour gradient and scratch are mandatory, the detached prefix cannot exceed P
    args = L.B2RBackwardArgs()
    ws.ctx_bytes = lib.b2r_ctx_bytes(10, 32, 32)
    bwd = lambda scratch, nbytes: lib.b2r_backward(C.byref(sc), C.byref(ws), C.byref(args), scratch, nbytes, None)
    assert bwd(fake, 1 << 20) == -1         # no dL_dcolor
    args.dL_dcolor = fake
    assert bwd(None, 1 << 20) == -1
    assert bwd(fake, 8) == -2               # scratch too small
    args.first_row = 11
    assert bwd(fake, 1 << 20) == -1


def test_error_codes_of_the_abi_v3_entry_points_without_touching_cuda():
    """Views, the split pipeline stages and the checkpoint store are validated on the host."""
    lib = L.load()
    fake = 0x1000
    sc = L.B2RScene()
    sc.P, sc.width, sc.height, sc.tanfovx, sc.tanfovy = 10, 32, 32, 0.5, 0.5
    sc.bg = sc.viewmatrix = sc.projmatrix = sc.campos = fake
    sc.means3D = sc.opacities = sc.colors_precomp = sc.scales = sc.rotations = fake
    ws = L.B2RWorkspace()
    ws.ctx, ws.ctx_bytes = fake, lib.b2r_ctx_bytes(10, 32, 32)
    ws.dup_ids, ws.dup_capacity = fake, 1000
    out = L.B2RForwardOutputs()
    view = L.B2RView()
    comp = lambda: lib.b2r_forward_composite(C.byref(sc), C.byref(ws), C.byref(view), C.byref(out), None)
    assert comp() == -1                      # no output images
    out.color = out.depth = out.alpha = fake
    view.id_begin, view.id_end = 4, 2
    assert comp() == -1                      # empty / inverted Gaussian range
    view.id_begin, view.id_end = 0, 11
    assert comp() == -1                      # range beyond P
    view.id_begin, view.id_end = 2, 10
    view.final_T = fake
    assert comp() == -1                      # final_T and n_contrib come as a pair
    view.final_T = None
    # an undersized checkpoint store is rejected before anything is launched
    ws.checkpoints, ws.checkpoint_bytes = fake, 16
    assert comp() == -2
    ws.checkpoint_bytes = lib.b2r_checkpoint_bytes(32, 32, 1000)
    view.checkpoints, view.checkpoint_bytes = fake, 16
    assert comp() == -2                      # ... and so is a view's own store
    # binning needs the scratch
    assert lib.b2r_forward_bin(C.byref(sc), C.byref(ws), None) == -1
    ws.scratch, ws.scratch_bytes = fake, 8
    assert lib.b2r_forward_bin(C.byref(sc), C.byref(ws), None) == -2
    # backward stages
    args = L.B2RBackwardArgs()
    view = L.B2RView()
    view.id_begin, view.id_end = 0, 10
    bc = lambda scratch, n: lib.b2r_backward_composite(C.byref(sc), C.byref(ws), C.byref(view), C.byref(args), scratch, n, None)
    bp = lambda scratch, n: lib.b2r_backward_project(C.byref(sc), C.byref(ws), C.byref(args), scratch, n, None)
    assert bc(fake, 1 << 20) == -1           # no dL_dcolor
    args.dL_dcolor = fake
    assert bc(fake, 8) == -2 and bp(fake, 8) == -2
    assert bp(None, 1 << 20) == -1
    args.first_row = 11
    assert bc(fake, 1 << 20) == -1 and bp(fake, 1 << 20) == -1
    # split pass: the own sorted ids ride behind the keys, 4 bytes per duplicate slot, aligned like every other region
    for cap in (0, 1, 64, 1000, 1 << 20):
        extra = -(-4 * max(cap, 1) // 256) * 256
        assert lib.b2r_split_scratch_bytes(10, 32, 32, cap) == lib.b2r_scratch_bytes(10, 32, 32, cap) + extra > 0
    # each call below is valid but for the one field under test: every rejection happens before a launch
    launches = lib.b2r_launch_count()
    ps = lambda first_row, radii: lib.b2r_forward_project_split(C.byref(sc), C.byref(ws), first_row, radii, None)
    assert ps(11, fake) == -1                # the split row lies beyond P
    ws.dup_capacity = 0
    assert ps(10, fake) == -1                # the split pass bins with the capacity it was given
    ws.dup_capacity = 1000
    assert ps(0, None) == -1                 # P > 0 rows need radii
    base = L.B2RWorkspace()
    base.ctx, base.ctx_bytes, base.dup_ids, base.dup_capacity = fake, lib.b2r_ctx_bytes(10, 32, 32), fake, 1000
    bs = lambda b, first_row=10: lib.b2r_forward_bin_split(C.byref(sc), C.byref(ws), b, first_row, fake, None)
    ws.scratch_bytes = lib.b2r_scratch_bytes(10, 32, 32, 1000)  # enough for a whole pass, not for the own ids
    assert bs(C.byref(base)) == -2
    ws.scratch_bytes = lib.b2r_split_scratch_bytes(10, 32, 32, 1000)
    assert bs(None) == -1                    # no base pass
    assert bs(C.byref(ws)) == -1             # the base pass is this pass
    base.ctx = None
    assert bs(C.byref(base)) == -1
    base.ctx, base.dup_ids = fake, None
    assert bs(C.byref(base)) == -1
    base.dup_ids, base.ctx_bytes = fake, lib.b2r_ctx_bytes(10, 32, 32) - 1
    assert bs(C.byref(base)) == -2           # the base ctx cannot hold P rows
    base.ctx_bytes = lib.b2r_ctx_bytes(10, 32, 32)
    assert bs(C.byref(base), 11) == -1       # the split row lies beyond P
    assert lib.b2r_forward_bin_split(C.byref(sc), C.byref(ws), C.byref(base), 10, None, None) == -1  # no radii
    ws.dup_capacity, ws.scratch_bytes = 0, lib.b2r_split_scratch_bytes(10, 32, 32, 0)
    assert bs(C.byref(base)) == -1           # no capacity
    assert lib.b2r_launch_count() == launches


def test_compiled_torch_binding_builds_loads_and_refuses_cpu_tensors():
    """csrc_torch/b2r_torch.cpp (the public call's host as a C++ autograd Function) builds in-tree against this
    interpreter's torch, links to libb200raster.so, reports the same ABI version and refuses CPU tensors with adaptive
    and with fixed capacity.  No compute here (no GPU)."""
    from exavatar_release_b200 import build_ext, rasterizer
    path = build_ext.build_torch_ext()
    assert os.path.exists(path)
    ext = rasterizer._compiled_binding()
    assert ext and ext.abi_version() == L.ABI_VERSION
    import torch
    a = torch.zeros(4, 3)
    for fixed_capacity in (-1, 1000):  # no CPU fallback in either capacity mode
        with pytest.raises(RuntimeError, match="CUDA tensor"):
            ext.rasterize(a, a, None, a, torch.zeros(4, 1), a, torch.zeros(4, 4), None, 16, 16, 1.0, 1.0, torch.zeros(3),
                          1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), True, 1.25, fixed_capacity, False)
