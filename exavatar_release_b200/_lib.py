"""ctypes binding of libb200raster.so (the C ABI in include/b200raster.h).

There is NO CPU fallback: if the shared library is missing or cannot be loaded, `load()` raises.  The library is built
in-tree by `exavatar_release_b200.build_ext.build()` (nvcc, sm_90a).
"""
from __future__ import annotations

import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libb200raster.so")
LIB_PATH = os.environ.get("B2R_LIB", LIB_PATH)  # tuning experiments: an alternative build of the same library

ABI_VERSION = 4
B2R_OK = 0
B2R_FLAG_NO_TILE_CULL = 1
B2R_FLAG_DEBUG = 2
B2R_FLAG_CTX_CLEAN = 4

_fp = C.c_void_p  # device pointers travel as plain addresses


class B2RScene(C.Structure):
    _fields_ = [
        ("P", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("sh_degree", C.c_int32),
        ("sh_coeffs", C.c_int32), ("flags", C.c_uint32),
        ("scale_modifier", C.c_float), ("tanfovx", C.c_float), ("tanfovy", C.c_float),
        ("bg", _fp), ("viewmatrix", _fp), ("projmatrix", _fp), ("campos", _fp),
        ("means3D", _fp), ("shs", _fp), ("colors_precomp", _fp), ("opacities", _fp),
        ("scales", _fp), ("rotations", _fp), ("cov3D_precomp", _fp),
        # mixed colour source: rows [0, sh_rows) from `shs`, the rest from `colors_precomp`; 0 = one source
        ("sh_rows", C.c_int32),
    ]


class B2RStatus(C.Structure):
    _fields_ = [
        ("num_dups", C.c_uint64), ("dup_capacity", C.c_uint64), ("overflow", C.c_uint32), ("num_visible", C.c_uint32),
        ("consumed_fwd", C.c_uint64), ("consumed_bwd", C.c_uint64), ("token", C.c_uint64), ("reserved", C.c_uint64 * 2),
    ]


class B2RWorkspace(C.Structure):
    _fields_ = [
        ("ctx", _fp), ("ctx_bytes", C.c_size_t), ("dup_ids", _fp), ("dup_capacity", C.c_uint64),
        ("scratch", _fp), ("scratch_bytes", C.c_size_t), ("status_mirror", _fp), ("status_token", C.c_uint64),
        ("checkpoints", _fp), ("checkpoint_bytes", C.c_size_t),  # ABI v3: segment table + blend-state checkpoints
    ]


class B2RView(C.Structure):
    _fields_ = [
        ("id_begin", C.c_uint32), ("id_end", C.c_uint32), ("bg", _fp), ("final_T", _fp), ("n_contrib", _fp),
        ("checkpoints", _fp), ("checkpoint_bytes", C.c_size_t), ("skip_below", C.c_uint32), ("reserved", C.c_uint32),
    ]


class B2RSkin(C.Structure):
    """Standalone skinning of one or two Gaussian sets sharing a rig (b2r_skin_forward / b2r_skin_backward)."""
    _fields_ = [
        ("P", C.c_int32), ("J", C.c_int32), ("V", C.c_int32), ("reserved", C.c_int32),
        ("weights", _fp), ("rows", _fp), ("joint_mats", _fp), ("trans", _fp), ("cam_Rinv", _fp), ("cam_t", _fp),
        ("xyz", _fp * 2), ("posed", _fp * 2),
    ]


class B2RMeshRender(C.Structure):
    """Textured mesh render (b2r_mesh_render_forward / b2r_mesh_render_backward): ExAvatar's face render."""
    _fields_ = [
        ("V", C.c_int32), ("F", C.c_int32), ("Vt", C.c_int32), ("C", C.c_int32),
        ("tex_height", C.c_int32), ("tex_width", C.c_int32), ("height", C.c_int32), ("width", C.c_int32),
        ("mesh", _fp), ("faces", _fp), ("vertex_uv", _fp), ("face_uv", _fp), ("texture", _fp),
        ("cam_R", _fp), ("cam_t", _fp), ("focal", _fp), ("princpt", _fp), ("keys", _fp),
        ("vf_offsets", _fp), ("vf_entries", _fp),
    ]


class B2RGnMlp(C.Structure):
    """One GroupNorm MLP stack (b2r_gn_mlp_forward / b2r_gn_mlp_backward): HumanGaussian's networks."""
    _fields_ = [
        ("P", C.c_int32), ("K", C.c_int32), ("H", C.c_int32), ("reserved", C.c_int32),
        ("x", _fp), ("w", _fp * 3), ("b", _fp * 3), ("gamma", _fp * 3), ("beta", _fp * 3),
        ("w_head", _fp), ("b_head", _fp),
    ]


class B2RRegs(C.Structure):
    """ExAvatar's human regularisers (b2r_regs_forward / b2r_regs_backward): the inputs and the model's tables."""
    _fields_ = [
        ("P", C.c_int32), ("J", C.c_int32), ("n_arm", C.c_int32), ("n_pairs", C.c_int32), ("n_hand", C.c_int32),
        ("n_rhand", C.c_int32), ("reserved", C.c_int32 * 2),
        ("mesh", _fp), ("mean_offset", _fp), ("mean_offset_offset", _fp), ("scale_offset", _fp), ("scale", _fp),
        ("scale_refined", _fp), ("rgb", _fp), ("rgb_refined", _fp), ("scale_reg", _fp), ("joint_offset", _fp),
        ("faces", _fp), ("vf_offsets", _fp), ("vf_entries", _fp), ("nbr_idx", _fp), ("nbr_w", _fp),
        ("lapT_offsets", _fp), ("lapT_src", _fp), ("lapT_w", _fp), ("weights", _fp), ("hand", _fp), ("arm_idx", _fp),
        ("arm_slot", _fp), ("joint_target", _fp), ("joint_weight", _fp), ("sym_pairs", _fp),
    ]


class B2RRegsGrads(C.Structure):
    _fields_ = [(n, _fp) for n in ("mean_offset", "mean_offset_offset", "scale_offset", "scale", "scale_refined", "rgb",
                                   "rgb_refined", "scale_reg", "joint_offset")]


class B2RRig(C.Structure):
    """ExAvatar's SMPL-X rig (b2r_rig_forward / b2r_rig_backward): the per-call inputs and the model's tables."""
    _fields_ = [
        ("V", C.c_int32), ("V1", C.c_int32), ("P", C.c_int32), ("J", C.c_int32), ("NB", C.c_int32), ("NE", C.c_int32),
        ("n_body", C.c_int32), ("reserved", C.c_int32),
        *[(n, _fp) for n in ("shape_param", "joint_offset", "full_pose", "expr", "template_", "shapedirs", "expr_dirs",
                             "posedirs_t", "pose_offset0", "lbs_weights", "jreg_offsets", "jreg_cols", "jreg_vals",
                             "jregT_offsets", "jregT_rows", "jregT_vals", "parents", "rot_neutral", "rot_zero",
                             "rot_inv", "sub1", "sub2", "upT_offsets", "upT_rows", "upT_w", "mask")],
    ]


class B2RRigGrads(C.Structure):
    _fields_ = [(n, _fp) for n in ("shape_param", "joint_offset", "full_pose", "expr")]


class B2RSmplxBody(C.Structure):
    """The frame's SMPL-X body mesh (b2r_smplx_body_forward / b2r_smplx_body_backward): the rig's tables, pose_mean,
    the five per-call inputs and the optional camera."""
    _fields_ = [("rig", B2RRig), *[(n, _fp) for n in ("pose_mean", "shape_param", "joint_offset", "full_pose", "expr",
                                                      "trans", "cam_R", "cam_t")]]


class B2RSmplxBodyGrads(C.Structure):
    _fields_ = [(n, _fp) for n in ("shape_param", "joint_offset", "full_pose", "expr", "trans")]


class B2RAdamSegment(C.Structure):
    """One tensor of an Adam step (b2r_adam_step): its four device pointers, numel, first chunk, the param's row layout
    and the fp32 scalars."""
    _fields_ = [
        ("param", _fp), ("grad", _fp), ("exp_avg", _fp), ("exp_avg_sq", _fp), ("numel", C.c_int64),
        ("first_chunk", C.c_int64), ("row_len", C.c_int64), ("row_stride", C.c_int64), ("lerp_weight", C.c_float), ("beta2", C.c_float), ("one_minus_beta2", C.c_float),
        ("bc2_sqrt", C.c_float), ("eps", C.c_float), ("step_size", C.c_float),
    ]


class B2RLpips(C.Structure):
    """ExAvatar's LPIPS-VGG terms (b2r_lpips_forward / b2r_lpips_backward): the images, the box and the weights in the
    kernels' layouts."""
    _fields_ = [
        ("width", C.c_int32), ("height", C.c_int32), ("n_images", C.c_int32), ("reserved", C.c_int32),
        ("img", _fp), ("target", _fp), ("bbox", _fp), ("w_fwd", _fp * 13), ("w_bwd", _fp * 13), ("bias", _fp * 13),
        ("lin", _fp * 5),
    ]


class B2RSceneAssets(C.Structure):
    """ExAvatar's scene Gaussian assets (b2r_scene_assets_forward / b2r_scene_assets_backward): the parameters, their
    row strides, the device degree buffer and the camera (NULL: shs mode)."""
    _fields_ = [
        ("P", C.c_int32), ("M", C.c_int32), ("dc_stride", C.c_int64), ("rest_stride", C.c_int64),
        *[(n, _fp) for n in ("mean", "opacity_logit", "log_scale", "rotation6d", "feature_dc", "feature_rest",
                             "active_sh_degree", "cam_R", "cam_t")],
    ]


class B2RSceneAssetsGrads(C.Structure):
    _fields_ = [(n, _fp) for n in ("opacity", "scale", "dL_dopacity", "dL_dscale", "dL_drotation", "dL_dcolor",
                                   "dL_dlogit", "dL_dlog_scale", "dL_drotation6d", "dL_dfeature_dc",
                                   "dL_dfeature_rest", "dL_dmean")]


class B2RSmplxPose(C.Structure):
    """One frame's seven 6D pose parameters (b2r_decode_pose_forward / b2r_decode_pose_backward): pointers and rows."""
    _fields_ = [("param", _fp * 7), ("rows", C.c_int32 * 7), ("reserved", C.c_int32)]


class B2RSmplxPoseGrads(C.Structure):
    _fields_ = [("param", _fp * 7)]


class B2RHumanAssets(C.Structure):
    """HumanGaussian's geometry around its networks (b2r_human_geometry_forward / b2r_human_geometry_backward)."""
    _fields_ = [
        ("P", C.c_int32), ("warmup", C.c_int32), ("geo_stride", C.c_int64), ("geo_offset_stride", C.c_int64),
        *[(n, _fp) for n in ("mesh", "pose_offset", "expr_offset", "geo", "geo_offset", "mask")],
    ]


class B2RHumanAssetsGrads(C.Structure):
    _fields_ = [(n, _fp) for n in ("dL_dmean_3d", "dL_dmean_3d_refined", "dL_dscale", "dL_dscale_refined",
                                   "dL_dmean_offset_offset", "dL_dscale_wo_clamp", "dL_dscale_refined_wo_clamp",
                                   "dL_dmesh", "dL_dexpr_offset", "dL_dgeo", "dL_dgeo_offset")]


class B2RForwardOutputs(C.Structure):
    _fields_ = [("color", _fp), ("depth", _fp), ("alpha", _fp), ("radii", _fp)]


class B2RBackwardArgs(C.Structure):
    _fields_ = [
        ("dL_dcolor", _fp), ("dL_ddepth", _fp), ("dL_dalpha", _fp),
        ("dL_dmeans3D", _fp), ("dL_dmeans2D", _fp), ("dL_dshs", _fp), ("dL_dcolors", _fp), ("dL_dopacities", _fp),
        ("dL_dscales", _fp), ("dL_drotations", _fp), ("dL_dcov3D", _fp),
        ("flags", C.c_uint32), ("first_row", C.c_uint32),
        ("densify_grad_accum", _fp), ("densify_count", _fp), ("densify_radius_max", _fp),
        ("densify_rows", C.c_uint32), ("reserved", C.c_uint32),
    ]


# B2RStatus.consumed_fwd / consumed_bwd: list entries staged per tile, x 8 (forward) / x 4 (backward) -- b200raster.h
CONSUMED_FWD_DIV = 8
CONSUMED_BWD_DIV = 4

B2R_BWD_ACCUMULATE = 1
B2R_BWD_SCRATCH_ZEROED = 2


def read_status(ctx_buf) -> dict:
    """Decodes the B2RStatus block at the head of a ctx buffer (uint8 tensor).  Copies it to the host, which synchronises
    with the device: for tests, bench accounting and debugging."""
    s = B2RStatus.from_buffer_copy(ctx_buf[: C.sizeof(B2RStatus)].cpu().numpy().tobytes())
    return {"num_dups": int(s.num_dups), "dup_capacity": int(s.dup_capacity), "overflow": int(s.overflow),
            "num_visible": int(s.num_visible), "consumed_fwd": int(s.consumed_fwd), "consumed_bwd": int(s.consumed_bwd),
            # the composites count staged list entries per CTA; these divisors turn the sums into entries per TILE
            "consumed_fwd_div": float(CONSUMED_FWD_DIV), "consumed_bwd_div": float(CONSUMED_BWD_DIV)}


# every symbol include/b200raster.h declares: (name, restype, argtypes)
SYMBOLS = [
    ("b2r_abi_version", C.c_int, []),
    ("b2r_strerror", C.c_char_p, [C.c_int]),
    ("b2r_last_cuda_error", C.c_int, []),
    ("b2r_sizeof", C.c_size_t, [C.c_int]),
    ("b2r_ctx_bytes", C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    ("b2r_scratch_bytes", C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_uint64]),
    ("b2r_backward_scratch_bytes", C.c_size_t, [C.c_int32]),
    ("b2r_checkpoint_bytes", C.c_size_t, [C.c_int32, C.c_int32, C.c_uint64]),
    ("b2r_forward_bin", C.c_int, [C.POINTER(B2RScene), C.POINTER(B2RWorkspace), _fp]),
    ("b2r_forward_composite", C.c_int, [C.POINTER(B2RScene), C.POINTER(B2RWorkspace), C.POINTER(B2RView),
                                        C.POINTER(B2RForwardOutputs), _fp]),
    ("b2r_backward_composite", C.c_int, [C.POINTER(B2RScene), C.POINTER(B2RWorkspace), C.POINTER(B2RView),
                                         C.POINTER(B2RBackwardArgs), _fp, C.c_size_t, _fp]),
    ("b2r_backward_project", C.c_int, [C.POINTER(B2RScene), C.POINTER(B2RWorkspace), C.POINTER(B2RBackwardArgs), _fp,
                                       C.c_size_t, _fp]),
    ("b2r_forward_project", C.c_int, [C.POINTER(B2RScene), C.POINTER(B2RWorkspace), _fp, _fp]),
    ("b2r_split_scratch_bytes", C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_uint64]),
    ("b2r_forward_project_split", C.c_int, [C.POINTER(B2RScene), C.POINTER(B2RWorkspace), C.c_uint32, _fp, _fp]),
    ("b2r_forward_bin_split", C.c_int, [C.POINTER(B2RScene), C.POINTER(B2RWorkspace), C.POINTER(B2RWorkspace),
                                        C.c_uint32, _fp, _fp]),
    ("b2r_forward_render", C.c_int, [C.POINTER(B2RScene), C.POINTER(B2RWorkspace), C.POINTER(B2RForwardOutputs), _fp]),
    ("b2r_forward", C.c_int, [C.POINTER(B2RScene), C.POINTER(B2RWorkspace), C.POINTER(B2RForwardOutputs), _fp]),
    ("b2r_backward", C.c_int, [C.POINTER(B2RScene), C.POINTER(B2RWorkspace), C.POINTER(B2RBackwardArgs), _fp,
                               C.c_size_t, _fp]),
    ("b2r_mark_visible", C.c_int, [C.c_int32, _fp, _fp, _fp, _fp]),
    ("b2r_skin_forward", C.c_int, [C.POINTER(B2RSkin), _fp]),
    ("b2r_skin_backward", C.c_int, [C.POINTER(B2RSkin), C.POINTER(_fp), C.POINTER(_fp), _fp, _fp, _fp, C.c_size_t, _fp]),
    ("b2r_skin_scratch_bytes", C.c_size_t, [C.c_int32, C.c_int32]),
    ("b2r_l1ssim_scratch_bytes", C.c_size_t, [C.c_int32, C.c_int32]),
    ("b2r_l1ssim_forward", C.c_int, [C.c_int32, C.c_int32, _fp, _fp, _fp, _fp, C.c_int32, _fp, _fp, C.c_size_t, _fp]),
    ("b2r_l1ssim_backward", C.c_int, [C.c_int32, C.c_int32, _fp, _fp, _fp, _fp, C.c_int32, _fp, _fp, _fp, C.c_size_t,
                                      _fp]),
    ("b2r_nearest_scratch_bytes", C.c_size_t, [C.c_int32, C.c_int32]),
    ("b2r_nearest_rows", C.c_int, [C.c_int32, _fp, C.c_int32, _fp, _fp, _fp, _fp, C.c_size_t, _fp]),
    ("b2r_vertex_normals", C.c_int, [C.c_int32, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    ("b2r_mesh_render_scratch_bytes", C.c_size_t, [C.c_int32]),
    ("b2r_mesh_render_forward", C.c_int, [C.POINTER(B2RMeshRender), _fp, _fp, _fp, C.c_size_t, _fp]),
    ("b2r_mesh_render_backward", C.c_int, [C.POINTER(B2RMeshRender), _fp, _fp, _fp, _fp, C.c_size_t, _fp]),
    ("b2r_triplane_forward", C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    ("b2r_triplane_backward", C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, _fp, _fp, _fp, _fp, _fp, _fp,
                                        _fp]),
    ("b2r_gn_mlp_scratch_bytes", C.c_size_t, [C.c_int32]),
    ("b2r_gn_mlp_grads_count", C.c_size_t, [C.c_int32, C.c_int32]),
    ("b2r_gn_mlp_forward", C.c_int, [C.POINTER(B2RGnMlp), _fp, _fp, _fp]),
    ("b2r_gn_mlp_backward", C.c_int, [C.POINTER(B2RGnMlp), _fp, _fp, _fp, _fp, _fp, C.c_size_t, _fp]),
    ("b2r_regs_scratch_bytes", C.c_size_t, [C.c_int32, C.c_int32]),
    ("b2r_regs_forward", C.c_int, [C.POINTER(B2RRegs), _fp, _fp, C.c_size_t, _fp]),
    ("b2r_regs_backward", C.c_int, [C.POINTER(B2RRegs), _fp, C.POINTER(B2RRegsGrads), _fp, C.c_size_t, _fp]),
    ("b2r_rig_scratch_bytes", C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    ("b2r_rig_forward", C.c_int, [C.POINTER(B2RRig), _fp, _fp, _fp, _fp, _fp, _fp, _fp, C.c_size_t, _fp]),
    ("b2r_rig_backward", C.c_int, [C.POINTER(B2RRig), _fp, _fp, _fp, C.POINTER(B2RRigGrads), _fp, C.c_size_t, _fp]),
    ("b2r_smplx_body_scratch_bytes", C.c_size_t, [C.c_int32, C.c_int32]),
    ("b2r_smplx_body_forward", C.c_int, [C.POINTER(B2RSmplxBody), _fp, _fp, C.c_size_t, _fp]),
    ("b2r_smplx_body_backward", C.c_int, [C.POINTER(B2RSmplxBody), _fp, C.POINTER(B2RSmplxBodyGrads), _fp, C.c_size_t,
                                          _fp]),
    ("b2r_adam_chunk_elems", C.c_int64, []),
    ("b2r_adam_step", C.c_int, [_fp, C.c_int32, C.c_int64, _fp]),
    ("b2r_lpips_saved_bytes", C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    ("b2r_lpips_scratch_bytes", C.c_size_t, [C.c_int32, C.c_int32]),
    ("b2r_lpips_forward", C.c_int, [C.POINTER(B2RLpips), _fp, _fp, C.c_size_t, _fp, C.c_size_t, _fp]),
    ("b2r_lpips_backward", C.c_int, [C.POINTER(B2RLpips), _fp, C.c_size_t, _fp, _fp, _fp, C.c_size_t, _fp]),
    ("b2r_scene_assets_forward", C.c_int, [C.POINTER(B2RSceneAssets), _fp, _fp, _fp, _fp, _fp]),
    ("b2r_scene_assets_backward", C.c_int, [C.POINTER(B2RSceneAssets), C.POINTER(B2RSceneAssetsGrads), _fp]),
    ("b2r_decode_pose_forward", C.c_int, [C.POINTER(B2RSmplxPose), _fp, _fp]),
    ("b2r_decode_pose_backward", C.c_int, [C.POINTER(B2RSmplxPose), _fp, C.POINTER(B2RSmplxPoseGrads), _fp]),
    ("b2r_human_geometry_forward", C.c_int, [C.POINTER(B2RHumanAssets), _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    ("b2r_human_geometry_backward", C.c_int, [C.POINTER(B2RHumanAssets), C.POINTER(B2RHumanAssetsGrads), _fp]),
    ("b2r_human_colors_forward", C.c_int, [C.c_int32, _fp, _fp, _fp, _fp, _fp]),
    ("b2r_human_colors_backward", C.c_int, [C.c_int32, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    ("b2r_profile_enable", None, [C.c_int]),
    ("b2r_profile_read", C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.c_int]),
    ("b2r_launch_count", C.c_uint64, []),
    ("b2r_kernel_name", C.c_char_p, [C.c_int]),
    ("b2r_ctx_geom", _fp, [C.POINTER(B2RWorkspace), C.c_int32, C.c_int32, C.c_int32]),
    ("b2r_ctx_aux", _fp, [C.POINTER(B2RWorkspace), C.c_int32, C.c_int32, C.c_int32]),
    ("b2r_ctx_ranges", _fp, [C.POINTER(B2RWorkspace), C.c_int32, C.c_int32, C.c_int32]),
    ("b2r_ctx_final_T", _fp, [C.POINTER(B2RWorkspace), C.c_int32, C.c_int32, C.c_int32]),
    ("b2r_ctx_n_contrib", _fp, [C.POINTER(B2RWorkspace), C.c_int32, C.c_int32, C.c_int32]),
]

_lib = None


def load():
    """Loads the shared library (once).  Raises if it is absent -- the product path never falls back to CPU code."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"b200raster: {LIB_PATH} not found. Build it with `python -m exavatar_release_b200.build_ext` "
            "(nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, restype, argtypes in SYMBOLS:
        fn = getattr(lib, name)  # AttributeError if the .so is stale
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.b2r_abi_version() != ABI_VERSION:
        raise RuntimeError("b200raster: ABI version mismatch between the Python binding and libb200raster.so")
    # index 7 is unused (b2r_sizeof reports 0 there); B2RMeshRender is 8, B2RGnMlp 10 (9 unused too), B2RRegs 11,
    # B2RRegsGrads 12, B2RRig 13, B2RRigGrads 14, B2RAdamSegment 15, B2RLpips 16, B2RSceneAssets 17,
    # B2RSceneAssetsGrads 18, B2RSmplxPose 19, B2RSmplxPoseGrads 20, B2RHumanAssets 21, B2RHumanAssetsGrads 22,
    # B2RSmplxBody 23, B2RSmplxBodyGrads 24
    for idx, cls in ((0, B2RScene), (1, B2RStatus), (2, B2RWorkspace), (3, B2RForwardOutputs), (4, B2RBackwardArgs),
                     (5, B2RView), (6, B2RSkin), (8, B2RMeshRender), (10, B2RGnMlp), (11, B2RRegs),
                     (12, B2RRegsGrads), (13, B2RRig), (14, B2RRigGrads), (15, B2RAdamSegment),
                     (16, B2RLpips), (17, B2RSceneAssets), (18, B2RSceneAssetsGrads), (19, B2RSmplxPose),
                     (20, B2RSmplxPoseGrads), (21, B2RHumanAssets), (22, B2RHumanAssetsGrads), (23, B2RSmplxBody),
                     (24, B2RSmplxBodyGrads)):
        if lib.b2r_sizeof(idx) != C.sizeof(cls):
            raise RuntimeError(f"b200raster: struct layout drift for {cls.__name__}: "
                               f"{lib.b2r_sizeof(idx)} (C) vs {C.sizeof(cls)} (ctypes)")
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != B2R_OK:
        lib = load()
        msg = lib.b2r_strerror(rc).decode()
        raise RuntimeError(f"b200raster: {what} failed: {msg} (code {rc}, cudaError {lib.b2r_last_cuda_error()})")
