"""`SmplxRig`, `SmplxRig.body_mesh` and `skin_gaussians` (csrc/smplx_rig.cu, csrc/skin.cu) at the model shapes the
C4-sized tests in test_smplx_rig.py, test_smplx_body.py and test_skin_pair.py never reach (those run the SMPL-X tree,
J = 55, NB = 100, NE = 50, V = 10 478 and P = 167 618 Gaussians with dense 4-sparse weight rows).

The kernels change behaviour at these boundaries, and these cases reach them:
  lanes over joints     the rig's LBS and backward vertex kernels, the body's LBS and backward vertex kernels and
                        skinning's stage_weight_rows and its two ballots put joint j on lane j and j + 32: J = 32
                        leaves the second trip empty (rig "j32_star", skin J = 32), J = 33 puts one joint in it
                        ("j33_random", skin J = 33), J = 64 fills it ("j64_chain", "j64_random", skin J = 64).
  coefficients per lane NB and NE four per lane (aB[4], aE[4], wpart[warp][lane + 32 k], RIG_CMAX = 128): widths 1, 32,
                        33, 97 and 128 of both, and NB = 128 with NE = 1 ("j64_chain"), NB = 1 with NE = 32.
  tree walk             the single-CTA chain kernels walk the tree level by level (a barrier per level, two chains
                        per 128-thread CTA, grp = tid / 64, RIG_JMAX = 64) and run the adjoints in reverse level
                        order: a 64-joint linear chain walks 63 levels ("j64_chain"), a star 1 ("j32_star"), SMPL-X's
                        tree cut to 5 joints or grown to 63 ("j5_tet", "j63_smplx") and seeded random trees
                        ("j33_random", "j64_random") the levels between.
  fixed-grid strides    the backward vertex loops stride by RIG_PART_BLOCKS x 8 warps = BODY_PART_BLOCKS x 4 warps
                        = 1024 vertices: V = 4 leaves 127 of the rig's 128 CTAs (and 255 of the body's 256) without a
                        vertex ("j5_tet"), V = 86 is not a multiple of 8 ("j32_star"), V = 1023, 1024 and 1025 sit at
                        the first stride's end and V = 2102 takes three strides ("j64_random").  Those CTAs must
                        still write a zero partial: the C ABI test runs every buffer poisoned with NaN.
  subdivision tables    the two-level tables (upT CSR, rig_level2) built from a tetrahedron (V = 4, P = 34) and
                        from a mesh with one vertex in no face ("j33_random", V = 1023), besides the tube meshes.
  skinning grid         blocks of SKIN_THREADS = 256 Gaussians in warps of 32 rows (nrows = min(32, P - row0)):
                        P = 1, 31, 32, 33, 255, 256, 257 and 2049; skin_reduce_kernel's eight warps over every eighth
                        block get unequal block counts at P = 2049 (nine blocks); P = 0 runs only the reduce, over
                        zero blocks.  Weight rows sparse, dense (both ballots full), all zero (M = 0) and with
                        negative weights; rows None, reversed, heavily duplicated and pointing at the table's last
                        row; one set and two, with and without the camera.

These tests pin
  * without a device: the test's synthetic models pass validate_model at every case; for small meshes on every
    tree and width, smplx_rig_reference's "contract at V, then subdivide" route equals ExAvatar's "subdivide the
    tables, then contract" route in float64; the appended-vertex model keeps the first V rows of every derived table;
    and the host refusals (validate_model and the three C ABIs) sit exactly at J = 64 / 65, n_body + 4 = J, NB and
    NE = 128 / 129 and the skinning's J = 1..64, with nothing launched;
  * on the GPU: every output and the gradients of a seeded loss against float64 (smplx_rig_reference,
    smplx_body_reference, renderer.lbs_reference) with zero, tiny (1e-8), ordinary and near-pi joints in one pose
    (the body mesh also at batch_rodrigues' shift point r = -1e-8 (1, 1, 1), rounded to fp32); exact zeros;
    bit-identical runs; per-vertex results that do not depend on V; skinning's gradient subsets; and all three ops
    through their C ABI into buffers of NaN padded with a sentinel, then into zeroed buffers, with the same bits.

Bounds: those the C4 tests hold (rig: 1e-6 of max for the meshes and joint transforms, 1e-5 for the offsets and the
gradients; body mesh: 1e-6 for the mesh, 2e-6 for the gradients; skinning: 1e-6 for the positions, 1e-5 for the
gradients), except the body mesh's gradients on the tetrahedron (BODY_GRAD_V4 below).  At J = 64 the pose feature has
9 (J - 1) = 567 terms against 486 at C4; the fp32 contraction's error grows with the square root of the term count
(about 8 % more), far inside 1e-5, so the offsets keep their bound.  `-s` prints every measured error.
"""
import ctypes as C
import functools
import math

import numpy as np
import pytest
import torch

from util import assert_close
from util import dev  # noqa: F401
from exavatar_release_b200 import _lib as L
from exavatar_release_b200.camera import _inv3
from exavatar_release_b200.renderer import lbs_reference
from exavatar_release_b200.smplx_rig import (batch_rodrigues, smplx_body_reference, smplx_rig_reference,
                                             subdivision_tables, validate_model)
from exavatar_release_b200.synthetic import SMPLX_PARENTS, make_human_mesh

FAKE = 0x1000  # never dereferenced: validation fails before any launch
SENTINEL = 1234.5  # finite, written past the end of every output buffer of the C ABI tests
PAD = 64
BODY_GRAD = 2e-6  # the body mesh's gradients, as at C4
# On the tetrahedron (V = 4) d full_pose is a sum of four vertices' terms taken at fp32 points 4.3 m from the origin,
# and its largest component is only about 0.3: the fp32 rounding of those points alone moves it by a few 1e-6 of its
# max.
# ExAvatar's own fp32 route (smplx_body_reference with dtype=float32, root pose 0.1 rad) is 3.1e-6 of max away from
# float64 there, in camera coordinates.  Measured for the op on an NVIDIA H100 80GB HBM3 at a 700 W power limit: 3.4e-6
# (camera) and 1.5e-6 (world); in every other case at most 1.1e-6, inside BODY_GRAD.
BODY_GRAD_V4 = 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# Synthetic models of any shape
# ---------------------------------------------------------------------------------------------------------------------

def _tree(kind, J, seed=0):
    """parents (J,) of a topological tree: "smplx" SMPL-X's tree cut at J joints, or grown past 55 by a chain under
    the last joint (a longer finger); "chain" parents[i] = i - 1 (depth J - 1); "star" every joint under the root
    (depth 1); "random" parents[i] uniform in [0, i), seeded."""
    if kind == "smplx":
        return list(SMPLX_PARENTS[:J]) + [i - 1 for i in range(len(SMPLX_PARENTS), J)]
    if kind == "chain":
        return [-1] + list(range(J - 1))
    if kind == "star":
        return [-1] + [0] * (J - 1)
    if kind == "random":
        g = np.random.default_rng(100 + seed)
        return [-1] + [int(g.integers(0, i)) for i in range(1, J)]
    raise ValueError(kind)


def _depth(parents):
    d = [0] * len(parents)
    for i in range(1, len(parents)):
        d[i] = d[parents[i]] + 1
    return max(d)


def _f32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))


def _tetrahedron():
    """V = 4, four outward faces: two subdivisions give P = 34."""
    v = np.array([[0.0, 0.3, 4.24], [0.2, -0.2, 4.1], [-0.2, -0.2, 4.1], [0.0, -0.1, 4.4]])
    faces = np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]], dtype=np.int64)
    return {"targets": _f32(v), "base_faces": torch.from_numpy(faces)}


def _tube(rings, segments):
    m = make_human_mesh(rings=rings, segments=segments)
    return {"targets": m["targets"], "base_faces": m["base_faces"]}


def _with_isolated_vertex(mesh):
    """One more vertex, in no face: subdivision keeps it as a row of its own and no edge reaches it."""
    extra = mesh["targets"].mean(0, keepdim=True) + torch.tensor([[0.0, 0.05, 0.0]])
    return {"targets": torch.cat([mesh["targets"], extra]), "base_faces": mesh["base_faces"]}


MESHES = {  # name: (builder, V)
    "tet": (_tetrahedron, 4),
    "v86": (lambda: _tube(7, 12), 86),
    "v1023": (lambda: _with_isolated_vertex(_tube(30, 34)), 1023),
    "v1024": (lambda: _tube(14, 73), 1024),
    "v1025": (lambda: _tube(31, 33), 1025),
    "v2102": (lambda: _tube(30, 70), 2102),
}


@functools.lru_cache(maxsize=None)
def _mesh(name):
    mesh = MESHES[name][0]()
    assert mesh["targets"].shape[0] == MESHES[name][1], name
    return mesh


def _masks(P):
    """is_rhand / is_lhand / is_face_expr as fixed patterns over the P rows: about half the rows in the mask."""
    p = torch.arange(P)
    return {"is_rhand": p % 7 == 0, "is_lhand": p % 7 == 1, "is_face_expr": p % 5 == 2}


def make_model(parents, NB, NE, n_body, mesh, seed=0, jreg_vertices=None):
    """A seeded SMPL-X-shaped body model of any shape on `mesh` ({"targets": (V,3), "base_faces": (F,3)}), as
    validate_model takes it: dense shapedirs / expr_dirs / posedirs, lbs_weights with min(J, 4) joints per vertex
    (rows summing to 1), a J_regressor over min(8, n) of the first n = jreg_vertices (default V) vertices per joint
    (rows summing to 1), pose_mean non-zero past the face joints, the 大 pose on the first two body joints, and the
    masks of `_masks`."""
    g = np.random.default_rng(7000 + seed)
    v = mesh["targets"].numpy().astype(np.float64)
    V, J = len(v), len(parents)
    nj = V if jreg_vertices is None else jreg_vertices
    jreg = np.zeros((J, V))
    for j in range(J):
        k = min(8, nj)
        cols = np.sort(g.choice(nj, k, replace=False))
        w = g.uniform(0.5, 1.5, k)
        jreg[j, cols] = w / w.sum()
    k = min(4, J)
    idx = np.argsort(g.random((V, J)), axis=1)[:, :k]
    val = g.uniform(0.1, 1.0, (V, k))
    W = np.zeros((V, J))
    W[np.arange(V)[:, None], idx] = val / val.sum(1, keepdims=True)
    pose_mean = np.zeros(3 * J)
    pose_mean[3 * (n_body + 4):] = 0.2 * g.standard_normal(3 * max(0, J - n_body - 4))
    nbp = np.zeros((n_body, 3))
    nbp[0] = [0, 0, 1]
    if n_body > 1:
        nbp[1] = [0, 0, -1]
    faces = mesh["base_faces"].numpy()
    P = subdivision_tables(faces, V)[3]
    return {"v_template": _f32(v), "face_offset": _f32(0.003 * g.standard_normal((V, 3))),
            "shapedirs": _f32(0.01 * g.standard_normal((V, 3, NB))),
            "expr_dirs": _f32(0.002 * g.standard_normal((V, 3, NE))),
            "posedirs": _f32(0.002 * g.standard_normal((9 * (J - 1), 3 * V))),
            "J_regressor": _f32(jreg), "lbs_weights": _f32(W), "parents": torch.tensor(parents, dtype=torch.int64),
            "pose_mean": _f32(pose_mean), "neutral_body_pose": _f32(nbp), "faces": torch.from_numpy(faces.copy()),
            **_masks(P)}


def _first_vertices(model, V):
    """The model restricted to its first V vertices and the faces among them: every per-vertex table's first V rows
    unchanged (the J_regressor must already be zero past them)."""
    assert float(model["J_regressor"][:, V:].abs().max()) == 0
    f = model["faces"]
    f = f[(f < V).all(1)].contiguous()
    P = subdivision_tables(f.numpy(), V)[3]
    return dict(model, v_template=model["v_template"][:V], face_offset=model["face_offset"][:V],
                shapedirs=model["shapedirs"][:V], expr_dirs=model["expr_dirs"][:V],
                posedirs=model["posedirs"][:, :3 * V].contiguous(),
                J_regressor=model["J_regressor"][:, :V].contiguous(), lbs_weights=model["lbs_weights"][:V], faces=f, **_masks(P))


RIG_CASES = {  # name: (tree, J, NB, NE, n_body, mesh)
    "j5_tet": ("smplx", 5, 1, 1, 1, "tet"),
    "j32_star": ("star", 32, 32, 33, 21, "v86"),
    "j33_random": ("random", 33, 33, 97, 21, "v1023"),
    "j64_chain": ("chain", 64, 128, 1, 21, "v1024"),
    "j63_smplx": ("smplx", 63, 97, 128, 21, "v1025"),
    "j64_random": ("random", 64, 1, 32, 60, "v2102"),
}
# shape independence: SMPL-X's tree on the first 1 + 18 x 55 = 991 vertices of a 1102-vertex tube (both sides of
# the 1024-vertex stride), the J_regressor on those 991 alone
APPEND = {"tree": "smplx", "J": 55, "NB": 100, "NE": 50, "n_body": 21, "rings": 20, "segments": 55, "V": 991}


@functools.lru_cache(maxsize=None)
def _case_model(name):
    tree, J, NB, NE, n_body, mesh = RIG_CASES[name]
    return make_model(_tree(tree, J), NB, NE, n_body, _mesh(mesh))


@functools.lru_cache(maxsize=None)
def _append_models():
    a = APPEND
    ext = make_model(_tree(a["tree"], a["J"]), a["NB"], a["NE"], a["n_body"], _tube(a["rings"], a["segments"]),
                     jreg_vertices=a["V"])
    return _first_vertices(ext, a["V"]), ext


def _pose(J, seed):
    """(J,3): joint i >= 1 cycles through ordinary (0.3 N(0,1)), zero, tiny (1e-8 along a random axis) and near-pi
    (pi - 1e-4) rotations, so every regime sits in one call and every joint of the deepest chain takes one."""
    g = torch.Generator().manual_seed(seed)
    pose = 0.3 * torch.randn(J, 3, generator=g)
    axis = torch.randn(J, 3, generator=g)
    axis = axis / axis.norm(dim=1, keepdim=True)
    for i in range(1, J):
        k = i % 4
        if k == 1:
            pose[i] = 0
        elif k == 2:
            pose[i] = 1e-8 * axis[i]
        elif k == 3:
            pose[i] = (math.pi - 1e-4) * axis[i]
    return pose


def _rig_inputs(J, NB, NE, seed):
    g = torch.Generator().manual_seed(seed)
    beta = torch.randn(NB, generator=g)
    jo = 0.01 * torch.randn(J, 3, generator=g)
    expr = torch.randn(NE, generator=g)
    return [beta, jo, _pose(J, seed + 1), expr]


def _body_inputs(J, NB, NE, seed):
    beta, jo, pose, expr = _rig_inputs(J, NB, NE, seed)
    jo[0] += torch.tensor([0.02, -0.03, 0.01])  # the body mesh takes the root row too
    # batch_rodrigues' shift point -1e-8 (1, 1, 1) in fp32 (pose_mean is zero at the root): the op's fp64 angle is
    # |r + 1e-8| = 1e-16, where ExAvatar's fp32 route divides 0 by 0 (fl(-1e-8) + 1e-8 = 0 in fp32)
    pose[0] = -1e-8
    trans = torch.tensor([0.1, -0.2, 3.0]) + 0.05 * torch.randn(3, generator=torch.Generator().manual_seed(seed + 2))
    return [beta, jo, pose, expr, trans]


def _camera(device="cpu", dtype=torch.float32):
    R = batch_rodrigues(torch.tensor([[0.3, -0.5, 0.2]], dtype=torch.float64))[0]
    return R.to(device, dtype), torch.tensor([0.2, 0.1, -0.4], dtype=dtype, device=device)


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(RIG_CASES))
def test_builder_models_pass_validation(name):
    tree, J, NB, NE, n_body, mesh = RIG_CASES[name]
    m = validate_model(**_case_model(name))
    assert (m["J"], m["NB"], m["NE"], m["n_body"], m["V"]) == (J, NB, NE, n_body, MESHES[mesh][1])
    assert torch.allclose(m["lbs_weights"].sum(1), torch.ones(m["V"], dtype=torch.float64), atol=1e-6)
    assert torch.allclose(m["J_regressor"].sum(1), torch.ones(J, dtype=torch.float64), atol=1e-6)
    assert bool(m["mask"].any()) and not bool(m["mask"].all())
    depth = _depth(m["parents"].tolist())
    if tree == "chain":
        assert depth == J - 1 == 63
    if tree == "star":
        assert depth == 1
    if mesh == "tet":
        assert (m["V1"], m["P"]) == (10, 34)
    if mesh == "v1023":  # the isolated vertex: no subdivision edge reaches it
        assert not bool(((torch.as_tensor(m["sub1"]) == 1022).any()))


def test_appended_vertices_keep_the_first_rows_of_every_table():
    base, ext = (validate_model(**m) for m in _append_models())
    V = APPEND["V"]
    assert (base["V"], ext["V"]) == (V, 1102) and base["V"] < 1024 < ext["V"]
    for k in ("v_template", "face_offset", "shapedirs", "expr_dirs", "lbs_weights"):
        assert torch.equal(base[k], ext[k][:V]), k
    assert torch.equal(base["J_regressor"], ext["J_regressor"][:, :V])
    assert torch.equal(base["posedirs"], ext["posedirs"][:, :3 * V])
    # the corrective offsets of the 大 pose are per vertex: their fp32 rows are the ones the op reads
    assert torch.equal(base["pose_offset0"].float(), ext["pose_offset0"][:V].float())


SMALL = {name: (tree, J, NB, NE, n_body) for name, (tree, J, NB, NE, n_body, _) in RIG_CASES.items()}


@pytest.mark.parametrize("name", list(SMALL))
@pytest.mark.parametrize("mesh", ["tet", "v86"])
def test_contract_at_V_equals_exavatars_route_in_float64(name, mesh):
    tree, J, NB, NE, n_body = SMALL[name]
    m = validate_model(**make_model(_tree(tree, J), NB, NE, n_body, _mesh(mesh)))
    ins = [t.double() for t in _rig_inputs(J, NB, NE, seed=3)]
    a = smplx_rig_reference(m, *ins, route="upsample")
    b = smplx_rig_reference(m, *ins, route="contract")
    for k in ("pose_offset", "expr_offset"):
        x, y = getattr(a, k), getattr(b, k)
        assert float(x.abs().max()) > 0, k
        torch.testing.assert_close(x, y, rtol=0, atol=1e-12 * float(x.abs().max()), msg=k)


def test_validate_model_refuses_exactly_past_the_limits():
    mesh = _mesh("tet")
    ok = lambda **kw: validate_model(**make_model(**kw))  # noqa: E731
    for J, n_body in ((64, 60), (5, 1)):
        assert ok(parents=_tree("chain", J), NB=8, NE=8, n_body=n_body, mesh=mesh)["J"] == J
    with pytest.raises(ValueError, match="joints"):
        ok(parents=_tree("chain", 65), NB=8, NE=8, n_body=21, mesh=mesh)
    with pytest.raises(ValueError, match="body joints"):
        ok(parents=_tree("chain", 4), NB=8, NE=8, n_body=1, mesh=mesh)
    with pytest.raises(ValueError, match="body joints"):
        ok(parents=_tree("chain", 5), NB=8, NE=8, n_body=2, mesh=mesh)
    m = ok(parents=_tree("star", 5), NB=128, NE=128, n_body=1, mesh=mesh)
    assert (m["NB"], m["NE"]) == (128, 128)
    with pytest.raises(ValueError, match="shapedirs"):
        ok(parents=_tree("star", 5), NB=129, NE=8, n_body=1, mesh=mesh)
    with pytest.raises(ValueError, match="expr_dirs"):
        ok(parents=_tree("star", 5), NB=8, NE=129, n_body=1, mesh=mesh)


def _fake_rig(**kw):
    r = L.B2RRig(V=100, V1=300, P=900, J=55, NB=100, NE=50, n_body=21)
    for name, _ in L.B2RRig._fields_[8:]:
        setattr(r, name, FAKE)
    for k, v in kw.items():
        setattr(r, k, v)
    return r


def _fake_body(rig):
    b = L.B2RSmplxBody(rig=rig)
    for name in ("pose_mean", "shape_param", "joint_offset", "full_pose", "expr", "trans", "cam_R", "cam_t"):
        setattr(b, name, FAKE)
    return b


def test_cabi_refusals_sit_exactly_at_the_limits():
    """-1 (invalid) past each limit; at the limit the call passes validation and stops at the scratch size (-2), so
    no case launches anything."""
    lib = L.load()
    n0 = lib.b2r_launch_count()
    rg = L.B2RRigGrads(FAKE, FAKE, FAKE, FAKE)
    bg = L.B2RSmplxBodyGrads(FAKE, FAKE, FAKE, FAKE, FAKE)
    cases = [({"J": 65}, -1), ({"J": 64, "n_body": 60}, -2), ({"J": 64, "n_body": 61}, -1), ({"J": 4, "n_body": 1}, -1),
             ({"J": 5, "n_body": 1}, -2), ({"J": 5, "n_body": 2}, -1), ({"NB": 129}, -1), ({"NE": 129}, -1),
             ({"NB": 128, "NE": 128}, -2), ({"NB": 1, "NE": 1}, -2), ({"NB": 0}, -1), ({"NE": 0}, -1)]
    for kw, rc in cases:
        r = _fake_rig(**kw)
        assert lib.b2r_rig_forward(C.byref(r), *[FAKE] * 6, FAKE, 0, None) == rc, kw
        assert lib.b2r_rig_backward(C.byref(r), None, None, None, C.byref(rg), FAKE, 0, None) == rc, kw
        b = _fake_body(_fake_rig(**kw))
        assert lib.b2r_smplx_body_forward(C.byref(b), FAKE, FAKE, 0, None) == rc, kw
        assert lib.b2r_smplx_body_backward(C.byref(b), None, C.byref(bg), FAKE, 0, None) == rc, kw
    g = (C.c_void_p * 2)(FAKE, FAKE)
    d = (C.c_void_p * 2)(FAKE, FAKE)
    for J, rc in ((0, -1), (65, -1), (1, -2), (64, -2)):
        s = L.B2RSkin()
        s.P, s.J, s.V = 64, J, 100
        s.weights = s.rows = s.joint_mats = s.trans = s.cam_Rinv = s.cam_t = FAKE
        s.xyz[0] = s.xyz[1] = s.posed[0] = s.posed[1] = FAKE
        assert lib.b2r_skin_backward(C.byref(s), g, d, FAKE, FAKE, FAKE, 8, None) == rc, J
        if rc == -1:
            assert lib.b2r_skin_forward(C.byref(s), None) == -1, J
    assert lib.b2r_launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------------
# GPU: SmplxRig and SmplxRig.body_mesh
# ---------------------------------------------------------------------------------------------------------------------

_RIGS = {}


def _rig(name, device):
    """(SmplxRig, reference cache) of a case, built once per module."""
    from exavatar_release_b200.smplx_rig import SmplxRig
    if name not in _RIGS:
        model = _append_models()[0 if name == "append_base" else 1] if name.startswith("append") \
            else _case_model(name)
        _RIGS[name] = (SmplxRig(**model, device=device), {})
    return _RIGS[name]


def _leaves(ins, dtype=torch.float32):
    return [t.detach().to("cuda", dtype).requires_grad_(True) for t in ins]


def _rig_weights(rig, seed=3):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g).cuda() for s in ((rig.P, 3), (rig.J, 4, 4), (rig.P, 3))]


def _rig_loss(out, w, use=(True, True, True)):
    terms = [(out.mesh_neutral_pose * w[0]).sum(), (out.joint_mats * w[1]).sum(), (out.expr_offset * w[2]).sum()]
    return sum(t for t, u in zip(terms, use) if u)


def _rig_run(rig, ins, w, use=(True, True, True)):
    a = _leaves(ins)
    out = rig(*a)
    _rig_loss(out, w, use).backward()
    return out, a


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(RIG_CASES))
def test_rig_against_float64(name, dev):
    rig, cache = _rig(name, dev)
    tree, J, NB, NE, n_body, mesh = RIG_CASES[name]
    assert (rig.J, rig.NB, rig.NE, rig.n_body, rig.V) == (J, NB, NE, n_body, MESHES[mesh][1])
    ins = _rig_inputs(J, NB, NE, seed=11)
    w = _rig_weights(rig)
    out, a = _rig_run(rig, ins, w)
    b = _leaves(ins, torch.float64)
    ref = rig.reference(*b, dtype=torch.float64, device=dev, cache=cache)
    for k in ("mesh_neutral_pose", "mesh_neutral_pose_wo_upsample", "joint_mats"):
        assert_close(getattr(out, k), getattr(ref, k), 1e-6, f"{name} {k}")
    # fp32 contractions of 9 (J - 1) <= 567 and NE <= 128 signed terms
    for k in ("pose_offset", "expr_offset"):
        assert_close(getattr(out, k), getattr(ref, k), 1e-5, f"{name} {k}")
    assert float((out.pose_6d.double() - ref.pose_6d).abs().max()) <= 1e-6
    _rig_loss(ref, [x.double() for x in w]).backward()
    for k, x, y in zip(("shape_param", "joint_offset", "full_pose", "expr"), a, b):
        assert bool(torch.isfinite(x.grad).all()), k
        assert float(y.grad.abs().max()) > 0, k
        assert_close(x.grad, y.grad, 1e-5, f"{name} d{k}")
    # exact zeros: the root's joint offset (get_joint_offset), pose_offset outside the mask
    assert bool((a[1].grad[0] == 0).all())
    outside = ~rig.mask.bool()
    assert int(outside.sum()) > 0 and bool((out.pose_offset[outside] == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(RIG_CASES))
def test_rig_pose_and_expr_gradients_are_exactly_zero_without_joint_mats(name, dev):
    rig, _ = _rig(name, dev)
    _, a = _rig_run(rig, _rig_inputs(rig.J, rig.NB, rig.NE, seed=12), _rig_weights(rig), use=(True, False, False))
    assert bool((a[2].grad == 0).all()) and bool((a[3].grad == 0).all())
    assert float(a[0].grad.abs().max()) > 0 and float(a[1].grad.abs().max()) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(RIG_CASES))
def test_rig_and_body_runs_are_bit_identical(name, dev):
    rig, _ = _rig(name, dev)
    ins = _rig_inputs(rig.J, rig.NB, rig.NE, seed=13)
    w = _rig_weights(rig)
    bins = _body_inputs(rig.J, rig.NB, rig.NE, seed=14)
    wb = torch.randn((rig.V, 3), generator=torch.Generator().manual_seed(15)).cuda()
    cam = _camera("cuda")

    def run():
        out, a = _rig_run(rig, ins, w)
        lb = _leaves(bins)
        mesh = rig.body_mesh(*lb, *cam)
        (mesh * wb).sum().backward()
        return [t.clone() for t in out] + [x.grad.clone() for x in a] + [mesh.detach().clone()] + [x.grad for x in lb]

    for x, y in zip(run(), run()):
        assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [False, True])
@pytest.mark.parametrize("name", list(RIG_CASES))
def test_body_mesh_against_float64(name, world, dev):
    rig, _ = _rig(name, dev)
    ins = _body_inputs(rig.J, rig.NB, rig.NE, seed=21)
    cam = _camera("cuda") if world else (None, None)
    cam64 = [None if c is None else c.double() for c in cam]
    w = torch.randn((rig.V, 3), generator=torch.Generator().manual_seed(22)).cuda()
    a = _leaves(ins)
    mesh, joints = rig.body_mesh(*a, *cam, joints=True)
    (mesh * w).sum().backward()
    b = _leaves(ins, torch.float64)
    ref, ref_joints = smplx_body_reference(rig.model, *b, *cam64, joints=True)
    tag = f"{name} {'world' if world else 'camera'}"
    assert mesh.shape == (rig.V, 3) and joints.shape == (rig.J, 3)
    assert_close(mesh, ref, 1e-6, f"{tag} mesh")
    assert_close(joints, ref_joints, 1e-6, f"{tag} joints")
    (ref * w.double()).sum().backward()
    bound = BODY_GRAD_V4 if rig.V == 4 else BODY_GRAD
    for k, x, y in zip(("shape_param", "joint_offset", "full_pose", "expr", "trans"), a, b):
        assert bool(torch.isfinite(x.grad).all()), k
        assert float(y.grad.abs().max()) > 0, k
        assert_close(x.grad, y.grad, bound, f"{tag} d{k}")
    # joints=True adds a launch that reads the forward's saved joints: the mesh and gradients stay the same bits
    a2 = _leaves(ins)
    mesh2 = rig.body_mesh(*a2, *cam)
    (mesh2 * w).sum().backward()
    assert torch.equal(mesh2, mesh)
    for x, y in zip(a, a2):
        assert torch.equal(x.grad, y.grad)


@pytest.mark.gpu
def test_per_vertex_results_do_not_depend_on_V(dev):
    """The same tables with 111 vertices appended (991 -> 1102, across the 1024-vertex stride) and the J_regressor
    zero on them: the joints keep their bits, so the first 991 rows of mesh_neutral_pose_wo_upsample and of the
    body mesh keep theirs, as do joint_mats, pose_6d and the body's joints."""
    (base, _), (ext, _) = _rig("append_base", dev), _rig("append_ext", dev)
    V = base.V
    assert (V, ext.V) == (991, 1102)
    ins = [t.cuda() for t in _rig_inputs(base.J, base.NB, base.NE, seed=31)]
    ob, oe = base(*ins), ext(*ins)
    assert torch.equal(ob.mesh_neutral_pose_wo_upsample, oe.mesh_neutral_pose_wo_upsample[:V])
    assert torch.equal(ob.joint_mats, oe.joint_mats) and torch.equal(ob.pose_6d, oe.pose_6d)
    bins = [t.cuda() for t in _body_inputs(base.J, base.NB, base.NE, seed=32)]
    for cam in ((None, None), _camera("cuda")):
        mb, jb = base.body_mesh(*bins, *cam, joints=True)
        me, je = ext.body_mesh(*bins, *cam, joints=True)
        assert torch.equal(mb, me[:V]) and torch.equal(jb, je)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: skin_gaussians
# ---------------------------------------------------------------------------------------------------------------------

SKIN_CASES = [  # (J, P, weight rows, row index, two sets, camera)
    (1, 257, "dense", "none", False, True),
    (2, 2049, "sparse", "dup", True, False),
    (31, 33, "negative", "reversed", True, True),
    (32, 256, "dense", "last", False, False),
    (33, 31, "dense", "dup", True, True),
    (33, 2049, "zero", "reversed", True, True),
    (63, 255, "sparse", "reversed", False, True),
    (64, 2049, "dense", "none", True, True),
    (64, 257, "negative", "last", True, False),
    (64, 32, "sparse", "dup", False, True),
    (64, 1, "negative", "last", True, False),
    (2, 0, "dense", "none", True, True),
    (64, 0, "sparse", "reversed", False, False),
]


def _skin_id(c):
    return f"J{c[0]}-P{c[1]}-{c[2]}-{c[3]}-{'two' if c[4] else 'one'}-{'cam' if c[5] else 'nocam'}"


def _skin_case(case, device):
    J, P, kind, rows_kind, two, cam = case
    g = torch.Generator().manual_seed(1000 * J + P)
    V = max(P, 1) if rows_kind == "none" else P + 7
    if kind == "sparse":
        k = min(J, 4)
        table = torch.zeros(V, J)
        idx = torch.rand(V, J, generator=g).argsort(1)[:, :k]
        val = torch.rand(V, k, generator=g) + 0.05
        table.scatter_(1, idx, val / val.sum(1, keepdim=True))
    elif kind == "dense":  # every joint non-zero: both ballots full at J > 32
        table = torch.rand(V, J, generator=g) + 0.05
        table = table / table.sum(1, keepdim=True)
    elif kind == "zero":  # M = 0: the posed position is trans
        table = torch.zeros(V, J)
    else:  # every joint non-zero, signs mixed
        table = torch.randn(V, J, generator=g)
        assert bool((table < 0).any()) and bool((table != 0).all())
    if rows_kind == "none":
        rows = None
    elif rows_kind == "reversed":
        rows = torch.arange(P - 1, -1, -1)
    elif rows_kind == "dup":  # most Gaussians on three rows, the rest on the first
        rows = torch.randint(0, 3, (P,), generator=g)
        rows[::5] = 0
    else:  # every third Gaussian on the table's last row
        rows = torch.randint(0, V, (P,), generator=g)
        rows[::3] = V - 1
    R, t = (batch_rodrigues(torch.tensor([[0.2, -0.4, 0.1]], dtype=torch.float64))[0].float(),
            torch.tensor([0.1, -0.3, 2.0])) if cam else (None, None)
    axes = 0.3 * torch.randn(J, 3, generator=g)
    A = torch.eye(4).repeat(J, 1, 1)
    A[:, :3, :3] = batch_rodrigues(axes.double()).float()
    A[:, :3, 3] = 0.05 * torch.randn(J, 3, generator=g)
    xyz = torch.randn(P, 3, generator=g) * torch.tensor([0.25, 0.85, 0.15]) + torch.tensor([0.0, 0.0, 4.24])
    xyz_r = xyz + 0.002 * torch.randn(P, 3, generator=g) if two else None
    trans = torch.tensor([0.01, -0.02, 0.03])
    gp, gq = torch.randn(P, 3, generator=g), torch.randn(P, 3, generator=g)
    to = lambda x: None if x is None else x.to(device)  # noqa: E731
    return dict(table=to(table), rows=to(rows), A=to(A), trans=to(trans), R=to(R), t=to(t), xyz=to(xyz),
                xyz_r=to(xyz_r), gp=to(gp), gq=to(gq))


def _skin_grads(c, want_x, want_rig):
    from exavatar_release_b200.skinning import skin_gaussians
    x = c["xyz"].clone().requires_grad_(want_x)
    xr = None if c["xyz_r"] is None else c["xyz_r"].clone().requires_grad_(want_x)
    A = c["A"].clone().requires_grad_(want_rig)
    tr = c["trans"].clone().requires_grad_(want_rig)
    posed, posed_r = skin_gaussians(x, xr, c["table"], c["rows"], A, tr, c["R"], c["t"])
    loss = (posed * c["gp"]).sum() + ((posed_r * c["gq"]).sum() if xr is not None else 0.0)
    loss.backward()
    return [posed.detach(), None if posed_r is None else posed_r.detach()], \
        {"xyz": x.grad, "xyz_r": None if xr is None else xr.grad, "A": A.grad, "trans": tr.grad}


@pytest.mark.gpu
@pytest.mark.parametrize("case", SKIN_CASES, ids=_skin_id)
def test_skin_against_float64(case, dev):
    J, P, kind, _, two, cam = case
    c = _skin_case(case, dev)
    posed, got = _skin_grads(c, True, True)
    tag = _skin_id(case)
    lx = [c["xyz"].double().requires_grad_()] + ([c["xyz_r"].double().requires_grad_()] if two else [])
    lA, lt = c["A"].double().requires_grad_(), c["trans"].double().requires_grad_()
    w = c["table"].double() if c["rows"] is None else c["table"].double()[c["rows"]]
    w = w[:P]
    R = None if c["R"] is None else c["R"].double()
    t = None if c["t"] is None else c["t"].double()
    ref = [lbs_reference(x, w, lA, lt, R, t) for x in lx]
    for name, x, y in zip(("posed", "posed_refined"), posed, ref):
        assert x.shape == (P, 3)
        assert_close(x, y, 1e-6, f"{tag} {name}")
    assert posed[1] is None if not two else posed[1] is not None
    sum((y * g.double()).sum() for y, g in zip(ref, (c["gp"], c["gq"]))).backward()
    refs = {"xyz": lx[0].grad, "xyz_r": lx[1].grad if two else None, "A": lA.grad, "trans": lt.grad}
    for k, r in refs.items():
        if r is None:
            assert got[k] is None, k
            continue
        assert bool(torch.isfinite(got[k]).all()), k
        assert_close(got[k], r, 1e-5, f"{tag} d{k}")  # an all-zero reference is met exactly (the floor is 1e-30)
    assert float(got["A"][:, 3, :].abs().max()) == 0.0
    if P == 0:
        assert float(got["A"].abs().max()) == 0.0 and float(got["trans"].abs().max()) == 0.0
        assert got["A"].shape == (J, 4, 4) and got["trans"].shape == (3,)
    if kind == "zero" and P > 0:
        assert float(got["A"].abs().max()) == 0.0 and float(got["xyz"].abs().max()) == 0.0
        assert float(got["trans"].abs().max()) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("case", SKIN_CASES, ids=_skin_id)
def test_skin_gradient_subsets_and_runs_are_bit_identical(case, dev):
    """Every gradient, then dxyz alone (no reduce), then joint and translation alone (no dxyz written): each
    requested gradient the bits of the full request, and a second full request the same bits again."""
    c = _skin_case(case, dev)
    _, full = _skin_grads(c, True, True)
    _, again = _skin_grads(c, True, True)
    _, xs = _skin_grads(c, True, False)
    _, rig = _skin_grads(c, False, True)
    for k in ("xyz", "xyz_r", "A", "trans"):
        if full[k] is not None:
            assert torch.equal(full[k], again[k]), k
    for k in ("xyz", "xyz_r"):
        assert (xs[k] is None) == (full[k] is None) and rig[k] is None, k
        if full[k] is not None:
            assert torch.equal(xs[k], full[k]), k
    assert xs["A"] is None and xs["trans"] is None
    assert torch.equal(rig["A"], full["A"]) and torch.equal(rig["trans"], full["trans"])


# ---------------------------------------------------------------------------------------------------------------------
# GPU: through the C ABI, every value written and nothing past the end
# ---------------------------------------------------------------------------------------------------------------------

def _poisoned(n, device, fill=float("nan")):
    """n values of `fill` followed by PAD sentinels."""
    buf = torch.full((n + PAD,), fill, dtype=torch.float32, device=device)
    buf[n:] = SENTINEL
    return buf


def _scratch(nbytes, device, fill):
    """The scratch with PAD sentinel floats after its end; fill 0xFF is NaN as float and as double."""
    buf = torch.full((nbytes + 4 * PAD,), fill, dtype=torch.uint8, device=device)
    buf[nbytes:].view(torch.float32).fill_(SENTINEL)
    return buf


def _assert_written(what, buf, n, expect=None):
    """The first n values finite (and equal to `expect` bit for bit), the sentinels past them untouched."""
    got = buf[:n]
    assert bool(torch.isfinite(got).all()), (what, int((~torch.isfinite(got)).sum()), n)
    if expect is not None:
        assert torch.equal(got, expect.reshape(-1)), what
    assert bool((buf[n:] == SENTINEL).all()), what


def _assert_scratch_end(what, buf, nbytes):
    assert bool((buf[nbytes:].view(torch.float32) == SENTINEL).all()), what


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["j5_tet", "j64_chain", "j63_smplx", "j64_random"])
def test_rig_and_body_abi_write_every_value_and_nothing_past_the_end(name, dev):
    """b2r_rig_* and b2r_smplx_body_* (with the camera, and the joints) into outputs, gradients and scratch of NaN
    with a sentinel past their ends, then into zeroed buffers: every value finite and the Python route's bits, and
    no sentinel touched.  At V = 4 (j5_tet) 127 of the rig's 128 backward CTAs and 255 of the body's 256 own no
    vertex: they must still write their partials."""
    rig, _ = _rig(name, dev)
    lib = L.load()
    stream = torch.cuda.current_stream(dev).cuda_stream
    P, V, J, NB, NE, nb = rig.P, rig.V, rig.J, rig.NB, rig.NE, rig.n_body
    ins = _rig_inputs(J, NB, NE, seed=41)
    w = _rig_weights(rig, seed=42)
    out, a = _rig_run(rig, ins, w)
    py_out = list(out)
    py_grads = [x.grad for x in a]
    bins = _body_inputs(J, NB, NE, seed=43)
    R, t = _camera("cuda")
    wb = torch.randn((V, 3), generator=torch.Generator().manual_seed(44)).cuda()
    lb = _leaves(bins)
    py_mesh, py_joints = rig.body_mesh(*lb, R, t, joints=True)
    (py_mesh * wb).sum().backward()
    py_bgrads = [x.grad for x in lb]
    torch.cuda.synchronize()
    flat = [rig._input(x.detach(), n, k) for x, n, k in zip(a, (NB, 3 * J, 3 * J, NE), "bjpe")]
    st = rig._struct(flat)
    bflat = [rig._input(x.detach(), n, k) for x, n, k in zip(lb, (NB, 3 * J, 3 * J, NE, 3), "bjpet")]
    bst = rig._body_struct(bflat, [rig._input(R, 9, "R"), rig._input(t, 3, "t")])
    sizes = (P * 3, V * 3, J * 16, P * 3, P * 3, 6 * nb)
    gsizes = (NB, 3 * J, 3 * J, NE)
    bgsizes = (NB, 3 * J, 3 * J, NE, 3)
    for fill, sfill in ((float("nan"), 0xFF), (0.0, 0)):
        outs = [_poisoned(n, dev, fill) for n in sizes]
        grads = [_poisoned(n, dev, fill) for n in gsizes]
        scratch = _scratch(rig.scratch_bytes, dev, sfill)
        L.check(lib.b2r_rig_forward(C.byref(st), *[o.data_ptr() for o in outs], scratch.data_ptr(), rig.scratch_bytes,
                                    stream), "b2r_rig_forward")
        L.check(lib.b2r_rig_backward(C.byref(st), w[0].data_ptr(), w[1].data_ptr(), w[2].data_ptr(),
                                     C.byref(L.B2RRigGrads(*[g.data_ptr() for g in grads])), scratch.data_ptr(),
                                     rig.scratch_bytes, stream), "b2r_rig_backward")
        mesh = _poisoned(V * 3, dev, fill)
        joints = _poisoned(J * 3, dev, fill)
        bgrads = [_poisoned(n, dev, fill) for n in bgsizes]
        bscratch = _scratch(rig.body_scratch_bytes, dev, sfill)
        L.check(lib.b2r_smplx_body_forward(C.byref(bst), mesh.data_ptr(), bscratch.data_ptr(), rig.body_scratch_bytes,
                                           stream), "b2r_smplx_body_forward")
        L.check(lib.b2r_smplx_body_joints(C.byref(bst), bscratch.data_ptr(), rig.body_scratch_bytes, joints.data_ptr(),
                                          stream), "b2r_smplx_body_joints")
        L.check(lib.b2r_smplx_body_backward(C.byref(bst), wb.data_ptr(),
                                            C.byref(L.B2RSmplxBodyGrads(*[g.data_ptr() for g in bgrads])),
                                            bscratch.data_ptr(), rig.body_scratch_bytes, stream),
                "b2r_smplx_body_backward")
        torch.cuda.synchronize()
        tag = f"{name} fill {fill}"
        for k, buf, n, ref in zip(("mesh", "mesh_wo", "joint_mats", "pose_offset", "expr_offset", "pose_6d"), outs,
                                  sizes, py_out):
            _assert_written(f"{tag} {k}", buf, n, ref)
        for k, buf, n, ref in zip(("shape_param", "joint_offset", "full_pose", "expr"), grads, gsizes, py_grads):
            _assert_written(f"{tag} d{k}", buf, n, ref)
        _assert_written(f"{tag} body mesh", mesh, V * 3, py_mesh)
        _assert_written(f"{tag} body joints", joints, J * 3, py_joints)
        for k, buf, n, ref in zip(("shape_param", "joint_offset", "full_pose", "expr", "trans"), bgrads, bgsizes,
                                  py_bgrads):
            _assert_written(f"{tag} body d{k}", buf, n, ref)
        _assert_scratch_end(f"{tag} rig scratch", scratch, rig.scratch_bytes)
        _assert_scratch_end(f"{tag} body scratch", bscratch, rig.body_scratch_bytes)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in SKIN_CASES if c[1] in (33, 2049, 257) and c[4]], ids=_skin_id)
def test_skin_abi_writes_every_value_and_nothing_past_the_end(case, dev):
    """b2r_skin_forward / _backward into posed positions, dxyz, joint and translation gradients and a scratch of NaN
    with a sentinel past their ends, then into zeroed buffers: the Python route's bits, no sentinel touched."""
    J, P, _, _, _, cam = case
    c = _skin_case(case, dev)
    posed, got = _skin_grads(c, True, True)
    lib = L.load()
    stream = torch.cuda.current_stream(dev).cuda_stream
    rows = None if c["rows"] is None else c["rows"].to(torch.int32).contiguous()
    Rinv = _inv3(c["R"]).contiguous() if cam else None
    A = c["A"].reshape(J, 16).contiguous()
    nbytes = int(lib.b2r_skin_scratch_bytes(P, J))
    for fill, sfill in ((float("nan"), 0xFF), (0.0, 0)):
        out = [_poisoned(P * 3, dev, fill) for _ in range(2)]
        dx = [_poisoned(P * 3, dev, fill) for _ in range(2)]
        dj, dt = _poisoned(J * 12, dev, fill), _poisoned(3, dev, fill)
        scratch = _scratch(nbytes, dev, sfill)
        s = L.B2RSkin()
        s.P, s.J, s.V = P, J, c["table"].shape[0]
        s.weights, s.rows, s.joint_mats, s.trans = L.ptr(c["table"]), L.ptr(rows), L.ptr(A), L.ptr(c["trans"])
        s.cam_Rinv, s.cam_t = L.ptr(Rinv), L.ptr(c["t"])
        s.xyz[0], s.xyz[1] = L.ptr(c["xyz"]), L.ptr(c["xyz_r"])
        s.posed[0], s.posed[1] = out[0].data_ptr(), out[1].data_ptr()
        L.check(lib.b2r_skin_forward(C.byref(s), stream), "b2r_skin_forward")
        dposed = (C.c_void_p * 2)(c["gp"].data_ptr(), c["gq"].data_ptr())
        dxyz = (C.c_void_p * 2)(dx[0].data_ptr(), dx[1].data_ptr())
        L.check(lib.b2r_skin_backward(C.byref(s), dposed, dxyz, dj.data_ptr(), dt.data_ptr(), scratch.data_ptr(),
                                      nbytes, stream), "b2r_skin_backward")
        torch.cuda.synchronize()
        tag = f"{_skin_id(case)} fill {fill}"
        _assert_written(f"{tag} posed", out[0], P * 3, posed[0])
        _assert_written(f"{tag} posed_refined", out[1], P * 3, posed[1])
        _assert_written(f"{tag} dxyz", dx[0], P * 3, got["xyz"])
        _assert_written(f"{tag} dxyz_refined", dx[1], P * 3, got["xyz_r"])
        _assert_written(f"{tag} djoint", dj, J * 12, got["A"][:, :3, :])
        _assert_written(f"{tag} dtrans", dt, 3, got["trans"])
        _assert_scratch_end(f"{tag} scratch", scratch, nbytes)
