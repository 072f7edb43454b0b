"""`SmplxParamTable` (csrc/smplx_pose.cu b2r_param_table_*): every frame's SMPL-X parameters in one table, the frame
chosen by a slot read on the device.  CPU: the C ABI's refusals and the host checks of the
class.  GPU: forward and gradients bit-identical to `decode_smplx_pose` on the frame's
ParameterDict for every slot, as an int and as a CUDA tensor; zeros in every other row; NaN outputs and zero gradients
for an out-of-range device slot with the guards around the tables intact; the dict round trip bit for bit."""
import ctypes as C

import pytest
import torch
import torch.nn as nn

from exavatar_release_b200 import _lib as L
from exavatar_release_b200.human_assets import POSE_KEYS, POSE_ROWS, SmplxParamTable, decode_smplx_pose

NE = 50


# ---------------------------------------------------------------------------------------------------------- CPU tests

def test_abi_refusals_without_touching_cuda():
    lib = L.load()
    fake = 0x1000  # never dereferenced: every call below fails on the host
    launches = lib.b2r_launch_count()
    t = L.B2RSmplxParamTable(n_frames=4, n_joints=55, n_expr=NE, host_slot=0, pose=fake, expr=fake, trans=fake)
    g = L.B2RSmplxParamTableGrads(pose=fake, expr=fake, trans=fake)
    fwd = lambda: lib.b2r_param_table_forward(C.byref(t), fake, fake, fake, None)  # noqa: E731
    bwd = lambda: lib.b2r_param_table_backward(C.byref(t), C.byref(g), None)  # noqa: E731
    assert lib.b2r_param_table_forward(None, fake, fake, fake, None) == -1
    assert lib.b2r_param_table_backward(C.byref(t), None, None) == -1
    for field, bad in (("n_frames", 0), ("n_joints", 0), ("n_joints", 65), ("n_expr", -1), ("pose", None),
                       ("trans", None), ("expr", None)):
        good = getattr(t, field)
        setattr(t, field, bad)
        assert fwd() == -1 and bwd() == -1, field
        setattr(t, field, good)
    assert lib.b2r_param_table_forward(C.byref(t), None, fake, fake, None) == -1   # no full_pose
    assert lib.b2r_param_table_forward(C.byref(t), fake, None, fake, None) == -1   # no expr with n_expr > 0
    g.expr = None
    assert bwd() == -1
    assert lib.b2r_launch_count() == launches


def test_host_checks():
    with pytest.raises(RuntimeError, match="CUDA"):
        SmplxParamTable(torch.zeros(2, 55, 6), torch.zeros(2, NE), torch.zeros(2, 3))
    with pytest.raises(ValueError, match="no frames"):
        SmplxParamTable.from_param_dict({})
    d = {k: torch.zeros((6,) if n == 1 else (n, 6)) for k, n in zip(POSE_KEYS, POSE_ROWS)}
    d.update(expr=torch.zeros(NE), trans=torch.zeros(3))
    with pytest.raises(ValueError, match="lacks"):
        SmplxParamTable.from_param_dict({"0": {k: v for k, v in d.items() if k != "trans"}})
    with pytest.raises(ValueError, match="body_pose"):
        SmplxParamTable.from_param_dict({"0": dict(d, body_pose=torch.zeros(20, 6))})
    with pytest.raises(ValueError, match="trans"):
        SmplxParamTable.from_param_dict({"0": dict(d, trans=torch.zeros(4))})


# ---------------------------------------------------------------------------------------------------------- GPU tests

def frame_dicts(F, dev, seed=0):
    """ExAvatar's SMPLXParamDict.smplx_params: F frames of nine leaves, some 6D rows at the identity."""
    g = torch.Generator(device=dev).manual_seed(seed)
    out = {}
    for f in range(F):
        d = {}
        for k, n in zip(POSE_KEYS, POSE_ROWS):
            v = torch.randn((n, 6), generator=g, device=dev)
            if f % 3 == 0:
                v[0] = torch.tensor([1.0, 0, 0, 0, 1, 0], device=dev)
            d[k] = nn.Parameter(v[0] if n == 1 else v)
        d["expr"] = nn.Parameter(torch.randn(NE, generator=g, device=dev))
        d["trans"] = nn.Parameter(torch.randn(3, generator=g, device=dev))
        out[str(10 * f + 3)] = nn.ParameterDict(d)
    return nn.ParameterDict(out)


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def assert_bits(a, b, what):
    assert a.shape == b.shape and torch.equal(bits(a), bits(b)), what


@pytest.mark.gpu
@pytest.mark.parametrize("F", [1, 7, 1000])
def test_forward_and_gradients_match_decode_for_every_slot(F):
    dev = torch.device("cuda")
    params = frame_dicts(F, dev)
    table = SmplxParamTable.from_param_dict(params)
    gen = torch.Generator(device=dev).manual_seed(1)
    slot_t = torch.zeros(1, dtype=torch.int32, device=dev)
    for slot in range(F):
        key = table.frames[slot]
        assert table.slot_of(key) == slot == table.slot_of(int(key))
        ref = decode_smplx_pose(params[key])
        gf = torch.randn((55, 3), generator=gen, device=dev)
        ge = torch.randn(NE, generator=gen, device=dev)
        gt = torch.randn(3, generator=gen, device=dev)
        for p in params[key].values():
            p.grad = None
        torch.autograd.backward([ref["full_pose"], ref["expr"], ref["trans"]], [gf, ge, gt])
        want_pose = torch.cat([params[key][k].grad.reshape(-1, 6) for k in POSE_KEYS])
        for how in ("int", "tensor"):
            if how == "tensor":
                slot_t.fill_(slot)
            out = table(slot if how == "int" else slot_t)
            assert set(out) == set(ref)
            for k in ref:
                assert_bits(out[k], ref[k], f"F={F} slot={slot} {how} {k}")
            assert out["body_pose"].data_ptr() == out["full_pose"][1].data_ptr()  # views of full_pose
            for p in table.parameters():
                p.grad = None
            torch.autograd.backward([out["full_pose"], out["expr"], out["trans"]], [gf, ge, gt])
            for name, p, want in (("pose", table.pose, want_pose), ("expr", table.expr, params[key]["expr"].grad),
                                  ("trans", table.trans, params[key]["trans"].grad)):
                assert_bits(p.grad[slot], want.reshape(p.grad[slot].shape), f"F={F} slot={slot} {how} d{name}")
                rest = torch.cat([p.grad[:slot].reshape(-1), p.grad[slot + 1:].reshape(-1)])
                assert torch.equal(bits(rest), torch.zeros_like(bits(rest))), f"F={F} slot={slot} {how} d{name} rest"


@pytest.mark.gpu
def test_out_of_range_device_slot_reads_and_writes_no_row():
    dev = torch.device("cuda")
    F, guard = 5, 4096
    src = SmplxParamTable.from_param_dict(frame_dicts(F, dev, seed=2))
    sentinel = torch.tensor([0x7f800123], dtype=torch.int32).view(torch.float32).item()  # a NaN pattern
    sizes = [t.numel() for t in src.parameters()]
    store = torch.full((sum(sizes) + guard * (len(sizes) + 1),), sentinel, device=dev)
    views, off = [], guard
    for t, n in zip(src.parameters(), sizes):
        v = store[off:off + n].view(t.shape)
        v.copy_(t.detach())
        views.append(v.requires_grad_())
        off += n + guard
    table = SmplxParamTable(*views)
    before = store.detach().clone()
    slot_t = torch.zeros(1, dtype=torch.int32, device=dev)
    for bad in (-1, F, F + 7, 2 ** 31 - 1, -2 ** 31):
        slot_t.fill_(bad)
        out = table(slot_t)
        for k in ("full_pose", "expr", "trans"):
            assert torch.isnan(out[k]).all(), (bad, k)
        for p in table.parameters():
            p.grad = None
        torch.autograd.backward([out["full_pose"], out["expr"], out["trans"]],
                                [torch.ones_like(out["full_pose"]), torch.ones_like(out["expr"]),
                                 torch.ones_like(out["trans"])])
        for p in table.parameters():
            assert torch.equal(bits(p.grad), torch.zeros_like(bits(p.grad))), bad
        assert torch.equal(bits(store), bits(before)), bad  # tables and guards untouched
    with pytest.raises(IndexError):
        table(F)
    with pytest.raises(IndexError):
        table(-1)
    with pytest.raises(ValueError, match="int32"):
        table(torch.zeros(1, dtype=torch.int64, device=dev))


@pytest.mark.gpu
def test_param_dict_round_trip_is_bit_exact():
    dev = torch.device("cuda")
    params = frame_dicts(6, dev, seed=3)
    table = SmplxParamTable.from_param_dict(params)
    for f, key in enumerate(table.frames):
        r0 = 0
        for k, n in zip(POSE_KEYS, POSE_ROWS):
            assert_bits(table.pose[f, r0:r0 + n].reshape(params[key][k].shape), params[key][k], k)
            r0 += n
        assert_bits(table.expr[f], params[key]["expr"], "expr")
        assert_bits(table.trans[f], params[key]["trans"], "trans")
    with torch.no_grad():
        for p in table.parameters():
            p.mul_(1.5).add_(0.25)
    want = {key: {k: v.detach().clone() for k, v in params[key].items()} for key in table.frames}
    table.write_to(params)
    back = SmplxParamTable.from_param_dict(params)
    for a, b in zip(back.parameters(), table.parameters()):
        assert_bits(a, b, "round trip")
    for key in table.frames:
        for k, v in params[key].items():
            assert v.shape == want[key][k].shape and v.is_leaf
