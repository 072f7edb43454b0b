// api.cu -- the extern "C" boundary declared in include/b200raster.h.
#include <cmath>

#include "common.cuh"

using namespace b2r;

namespace {

int validate_scene(const B2RScene* sc) {
  if (!sc) return B2R_E_INVALID;
  if (sc->P < 0 || sc->width <= 0 || sc->height <= 0) return B2R_E_INVALID;
  if (sc->P >= (1 << 29)) return B2R_E_INVALID;  // the splat record carries id in 29 bits (common.cuh Geom)
  if (sc->width > 65535 * TILE || sc->height > 32767 * TILE) return B2R_E_INVALID;
  // a device tan(fov) is checked by the kernels that read it (gaussian_math.cuh load_cam)
  if (!sc->tanfov && (!(sc->tanfovx > 0.f) || !(sc->tanfovy > 0.f))) return B2R_E_INVALID;
  if (!sc->bg || !sc->viewmatrix || !sc->projmatrix || !sc->campos) return B2R_E_INVALID;
  if (sc->sh_rows < 0 || sc->sh_rows > sc->P) return B2R_E_INVALID;
  if (sc->P > 0) {
    if (!sc->opacities || !sc->means3D) return B2R_E_INVALID;
    if (sc->sh_rows > 0) {  // mixed: SH rows first, then colour rows -- both sources required
      if (!sc->shs || !sc->colors_precomp) return B2R_E_INVALID;
    } else if ((sc->shs != nullptr) == (sc->colors_precomp != nullptr)) {
      return B2R_E_INVALID;  // exactly one colour source
    }
    const bool sr = sc->scales != nullptr && sc->rotations != nullptr;
    if (sr == (sc->cov3D_precomp != nullptr)) return B2R_E_INVALID;                      // exactly one covariance source
    if ((sc->scales != nullptr) != (sc->rotations != nullptr)) return B2R_E_INVALID;
    if (sc->shs) {
      if (sc->sh_degree < 0 || sc->sh_degree > 3) return B2R_E_INVALID;
      if (sc->sh_coeffs < (sc->sh_degree + 1) * (sc->sh_degree + 1)) return B2R_E_INVALID;
      if (sc->sh_coeffs > 16) return B2R_E_INVALID;  // rows are staged through shared memory (project.cu)
    }
  }
  return B2R_OK;
}

int validate_ws(const B2RScene* sc, const B2RWorkspace* ws, bool need_scratch) {
  if (!ws || !ws->ctx) return B2R_E_INVALID;
  if (ws->ctx_bytes < b2r_ctx_bytes(sc->P, sc->width, sc->height)) return B2R_E_WORKSPACE;
  if (ws->dup_capacity > 0xfffffff0ull) return B2R_E_INVALID;  // list positions are 32-bit
  if (need_scratch) {
    if (!ws->scratch) return B2R_E_INVALID;
    if (ws->scratch_bytes < b2r_scratch_bytes(sc->P, sc->width, sc->height, ws->dup_capacity)) return B2R_E_WORKSPACE;
  }
  if (ws->dup_capacity > 0 && !ws->dup_ids) return B2R_E_INVALID;
  if (ws->checkpoints && ws->checkpoint_bytes < b2r_checkpoint_bytes(sc->width, sc->height, ws->dup_capacity)) return B2R_E_WORKSPACE;
  return B2R_OK;
}

// dL_dshs is required whenever the backward projection writes SH rows: every row of an SH scene, or, in a mixed scene,
// the SH rows at or above first_row (a detached SH prefix -- cat(scene.detach(), human) -- has none).
bool missing_dshs(const B2RScene* sc, const B2RBackwardArgs* a) {
  if (!sc->shs || a->dL_dshs || sc->P == 0) return false;
  return sc->sh_rows == 0 || (int64_t)a->first_row < (int64_t)sc->sh_rows;
}

// skin.cu stages a weight row as at most two floats per lane: J <= 64
int validate_skin(const B2RSkin* s) {
  if (!s) return B2R_E_INVALID;
  if (s->P < 0 || s->V <= 0) return B2R_E_INVALID;
  if (s->J <= 0 || s->J > 64) return B2R_E_INVALID;
  if (s->cam_Rinv && !s->cam_t) return B2R_E_INVALID;
  if (s->posed[1] && !s->xyz[1]) return B2R_E_INVALID;
  if (s->P > 0) {
    if (!s->weights || !s->joint_mats || !s->trans || !s->xyz[0]) return B2R_E_INVALID;
    if (!s->rows && s->V < s->P) return B2R_E_INVALID;  // row i of the table for Gaussian i
  }
  return B2R_OK;
}

// l1ssim.cu: 16-pixel tiles on a 2-D grid (grid.y <= 65535); the 9 per-pixel partial planes stay addressable
bool valid_l1ssim_size(int32_t width, int32_t height) {
  return width > 0 && height > 0 && height <= 65535 * 16 && (int64_t)width * height <= (int64_t)1 << 31;
}

// sizes, strides and the pointers the mode reads (shs mode: no camera, mean or degree); the degree's value is checked
// on the device
int validate_scene_assets(const B2RSceneAssets* s) {
  if (!s || s->P < 0 || s->M < 1 || s->M > B2R_SCENE_MAX_COEFFS) return B2R_E_INVALID;
  if ((s->cam_R != nullptr) != (s->cam_t != nullptr)) return B2R_E_INVALID;
  if (s->P == 0) return B2R_OK;
  if (!s->opacity_logit || !s->log_scale || !s->rotation6d || !s->feature_dc) return B2R_E_INVALID;
  if (s->dc_stride < 3) return B2R_E_INVALID;
  if (s->M > 1 && (!s->feature_rest || s->rest_stride < 3 * (s->M - 1))) return B2R_E_INVALID;
  if (s->cam_R && (!s->mean || !s->active_sh_degree)) return B2R_E_INVALID;
  return B2R_OK;
}

// row counts (1 <= J <= 64 joints, one thread each) and the parameters that have rows
int validate_pose(const B2RSmplxPose* p) {
  if (!p) return B2R_E_INVALID;
  int J = 0;
  for (int k = 0; k < B2R_POSE_PARAMS; ++k) {
    if (p->rows[k] < 0 || p->rows[k] > B2R_POSE_MAX_JOINTS) return B2R_E_INVALID;
    if (p->rows[k] > 0 && !p->param[k]) return B2R_E_INVALID;
    J += p->rows[k];
  }
  return J >= 1 && J <= B2R_POSE_MAX_JOINTS ? B2R_OK : B2R_E_INVALID;
}

// a parameter table's sizes (one thread per joint, at least one frame) and its tables
int validate_param_table(const B2RSmplxParamTable* t) {
  if (!t || !t->pose || !t->trans) return B2R_E_INVALID;
  if (t->n_frames < 1 || t->n_joints < 1 || t->n_joints > B2R_POSE_MAX_JOINTS || t->n_expr < 0) return B2R_E_INVALID;
  if (t->n_expr > 0 && !t->expr) return B2R_E_INVALID;
  return B2R_OK;
}

// a frame table's sizes and arrays, and the host slot when no device slot is given
int validate_frame_table(const B2RFrameTable* t) {
  if (!t || !t->pixels || !t->bbox || !t->R || !t->t || !t->focal || !t->princpt || !t->frame_idx || !t->slot_row)
    return B2R_E_INVALID;
  if (t->n_rows < 1 || t->n_slots < 1 || t->height < 1 || t->width < 1) return B2R_E_INVALID;
  if (!t->slot && (t->host_slot < 0 || t->host_slot >= t->n_slots)) return B2R_E_INVALID;
  return B2R_OK;
}

// a segmentation table's sizes and arrays, and the host slot when no device slot is given (as a frame table's)
int validate_segmentation(const B2RSegmentation* s) {
  if (!s || !s->pixels || !s->slot_row) return B2R_E_INVALID;
  if (s->n_rows < 1 || s->n_slots < 1 || s->height < 1 || s->width < 1) return B2R_E_INVALID;
  if (!s->slot && (s->host_slot < 0 || s->host_slot >= s->n_slots)) return B2R_E_INVALID;
  return B2R_OK;
}

// sizes, row strides and every input pointer (an empty set reads nothing)
int validate_human_assets(const B2RHumanAssets* h) {
  if (!h || h->P < 0 || (h->warmup != 0 && h->warmup != 1)) return B2R_E_INVALID;
  if (h->P == 0) return B2R_OK;
  if (!h->mesh || !h->pose_offset || !h->expr_offset || !h->geo || !h->geo_offset || !h->mask) return B2R_E_INVALID;
  if (h->geo_stride < 4 || h->geo_offset_stride < 4) return B2R_E_INVALID;
  return B2R_OK;
}

// sizes and the pointers both directions read: every weight a layer uses, the images; the box may be NULL.  The conv
// grids put H / 8 tiles in grid.y, and NHWC offsets of 64 x W x H floats stay in size_t.
int validate_lpips(const B2RLpips* p) {
  if (!p || p->width < 16 || p->height < 16 || p->n_images < 1) return B2R_E_INVALID;
  if (p->height > 65535 * 8 || (int64_t)p->width * p->height > (int64_t)1 << 28) return B2R_E_INVALID;
  if (!p->img || !p->target || !p->w_fwd[0] || !p->bias[0]) return B2R_E_INVALID;
  for (int l = 1; l < 13; l++)
    if (!p->w_fwd[l] || !p->w_bwd[l] || !p->bias[l]) return B2R_E_INVALID;
  for (int t = 0; t < 5; t++)
    if (!p->lin[t]) return B2R_E_INVALID;
  return B2R_OK;
}

// metrics.cu: sizes (the second pool needs 31 px; SSIM tiles put H / 16 in grid.y and 3 N in grid.z, the convs 2 N;
// per-image offsets of W x H x 4 floats stay in int32 pixel indices), the mask's channel count with the mask, and
// every pointer the op reads
int validate_neuman(const B2RNeumanScores* p) {
  if (!p || p->width < 31 || p->height < 31 || p->n_images < 1 || p->n_images > 16384) return B2R_E_INVALID;
  if (p->height > 65535 * 16 || (int64_t)p->width * p->height > (int64_t)1 << 28) return B2R_E_INVALID;
  if (p->mask ? (p->mask_channels != 1 && p->mask_channels != 3) : p->mask_channels != 0) return B2R_E_INVALID;
  if (!p->render || !p->target) return B2R_E_INVALID;
  for (int l = 0; l < 5; l++)
    if (!p->w[l] || !p->bias[l] || !p->lin[l]) return B2R_E_INVALID;
  return B2R_OK;
}

// compose.cu: sizes (a grid of N H W / 1024 CTAs stays far inside grid.x) and every image the calls read
int validate_compose_size(int32_t W, int32_t H, int32_t N) {
  if (W <= 0 || H <= 0 || N <= 0 || (int64_t)W * H * N >= (int64_t)1 << 36) return B2R_E_INVALID;
  return B2R_OK;
}

int validate_test_outputs(const B2RTestOutputs* p) {
  if (!p) return B2R_E_INVALID;
  const int rc = validate_compose_size(p->width, p->height, p->n_images);
  if (rc) return rc;
  for (int i = 0; i < 5; i++)
    if (!p->render[i]) return B2R_E_INVALID;
  for (int k = 0; k < 2; k++)
    if (!p->mask[k] || !p->face[k]) return B2R_E_INVALID;
  return B2R_OK;
}

// sizes and the pointers both directions read; the index tables' contents are the caller's (see b200raster.h)
int validate_mesh_render(const B2RMeshRender* m) {
  if (!m) return B2R_E_INVALID;
  if (m->V < 0 || m->F < 0 || m->Vt < 0 || m->C < 1 || m->C > 4) return B2R_E_INVALID;
  if (m->width <= 0 || m->height <= 0 || (int64_t)m->width * m->height >= ((int64_t)1 << 31)) return B2R_E_INVALID;
  if (m->F >= (1 << 29) || m->V >= (1 << 29)) return B2R_E_INVALID;  // 9 F floats and 3 V indices stay in int32
  if (!m->cam_R || !m->cam_t || !m->focal || !m->princpt) return B2R_E_INVALID;
  if (m->F > 0) {
    if (m->V < 1 || m->Vt < 1 || m->tex_height < 1 || m->tex_width < 1) return B2R_E_INVALID;
    if ((int64_t)m->C * m->tex_height * m->tex_width >= ((int64_t)1 << 31)) return B2R_E_INVALID;
    if (!m->mesh || !m->faces || !m->vertex_uv || !m->face_uv || !m->texture) return B2R_E_INVALID;
  }
  return B2R_OK;
}

// the shaded render reads the geometry, camera and keys fields only (the texture fields are ignored)
int validate_mesh_shade(const B2RMeshRender* m) {
  if (!m) return B2R_E_INVALID;
  if (m->V < 0 || m->F < 0 || m->F >= (1 << 29) || m->V >= (1 << 29)) return B2R_E_INVALID;
  if (m->width <= 0 || m->height <= 0 || (int64_t)m->width * m->height >= ((int64_t)1 << 31)) return B2R_E_INVALID;
  if (!m->cam_R || !m->cam_t || !m->focal || !m->princpt || !m->keys) return B2R_E_INVALID;
  if (m->F > 0 && (m->V < 1 || !m->mesh || !m->faces)) return B2R_E_INVALID;
  return B2R_OK;
}

// triplane.cu: P * 3C output elements and 6 H W CSR keys (x 32 lanes) stay addressable in int32 / the grid
bool valid_triplane(int32_t P, int32_t C, int32_t height, int32_t width) {
  return P >= 0 && C >= 1 && height >= 1 && width >= 1 && (int64_t)P * 3 * C < ((int64_t)1 << 31) &&
         (int64_t)height * width * 6 * 32 < ((int64_t)1 << 31);
}

// gn_mlp.cu: ExAvatar's shapes only (hidden width 128 is fixed by the kernels); P * 128 stays in int32
int validate_gn_mlp(const B2RGnMlp* m) {
  if (!m) return B2R_E_INVALID;
  if (m->P < 1 || m->P >= (1 << 24) || m->K < 1 || m->K > 128 || m->H < 1 || m->H > 4) return B2R_E_INVALID;
  if (!m->x || !m->w_head || !m->b_head) return B2R_E_INVALID;
  for (int l = 0; l < 3; l++)
    if (!m->w[l] || !m->b[l] || !m->gamma[l] || !m->beta[l]) return B2R_E_INVALID;
  return B2R_OK;
}

// regularizers.cu: the joint gradients are written by the threads of one CTA (J <= 256); every table is required,
// and the means need at least one vertex, one joint and one symmetric pair
int validate_regs(const B2RRegs* r) {
  if (!r) return B2R_E_INVALID;
  if (r->P < 1 || r->P >= (1 << 28) || r->J < 1 || r->J > 256 || r->n_arm < 0 || r->n_arm > r->P) return B2R_E_INVALID;
  if (r->n_pairs < 1 || r->n_hand < 0 || r->n_rhand < 0 || r->n_hand > r->P) return B2R_E_INVALID;
  if (!r->mesh || !r->mean_offset || !r->mean_offset_offset || !r->scale_offset || !r->scale || !r->scale_refined ||
      !r->rgb || !r->rgb_refined || !r->joint_offset)
    return B2R_E_INVALID;
  if (!r->faces || !r->vf_offsets || !r->vf_entries || !r->nbr_idx || !r->nbr_w || !r->lapT_offsets || !r->lapT_src ||
      !r->lapT_w || !r->weights || !r->hand || !r->arm_slot || (r->n_arm > 0 && !r->arm_idx) || !r->joint_target ||
      !r->joint_weight || !r->sym_pairs)
    return B2R_E_INVALID;
  return B2R_OK;
}

// smplx_rig.cu: one thread per joint in a 128-thread CTA (J <= 64), NB / NE <= 128 (four coefficients per lane), the
// pose_6d of the body joints needs 1 + n_body + 3 face joints <= J, and every table and input is required
int validate_rig(const B2RRig* r) {
  if (!r) return B2R_E_INVALID;
  if (r->V < 1 || r->V1 < r->V || r->P < r->V1 || r->P >= (1 << 28) || r->J < 2 || r->J > 64 || r->NB < 1 ||
      r->NB > 128 || r->NE < 1 || r->NE > 128 || r->n_body < 1 || r->n_body + 4 > r->J)
    return B2R_E_INVALID;
  if (!r->shape_param || !r->joint_offset || !r->full_pose || !r->expr) return B2R_E_INVALID;
  if (!r->template_ || !r->shapedirs || !r->expr_dirs || !r->posedirs_t || !r->pose_offset0 || !r->lbs_weights ||
      !r->jreg_offsets || !r->jreg_cols || !r->jreg_vals || !r->jregT_offsets || !r->jregT_rows || !r->jregT_vals ||
      !r->parents || !r->rot_neutral || !r->rot_zero || !r->rot_inv || (r->V1 > r->V && !r->sub1) ||
      (r->P > r->V1 && !r->sub2) || !r->upT_offsets || !r->upT_rows || !r->upT_w || !r->mask)
    return B2R_E_INVALID;
  return B2R_OK;
}

// smplx_rig.cu's body mesh: the rig's checks on its tables with the body's inputs, the camera both or neither
int validate_body(const B2RSmplxBody* b) {
  if (!b || !b->pose_mean || !b->trans || (b->cam_R != nullptr) != (b->cam_t != nullptr)) return B2R_E_INVALID;
  const B2RSmplxBody o = with_body_inputs(*b);
  return validate_rig(&o.rig);
}

}  // namespace

extern "C" {

int b2r_abi_version(void) { return B2R_ABI_VERSION; }

const char* b2r_strerror(int code) {
  switch (code) {
    case B2R_OK: return "ok";
    case B2R_E_INVALID: return "invalid argument";
    case B2R_E_WORKSPACE: return "workspace buffer too small";
    case B2R_E_CUDA: return "CUDA launch failed";
    case B2R_E_DUP_OVERFLOW: return "duplicate capacity exceeded";
    default: return "unknown error";
  }
}

int b2r_last_cuda_error(void) { return g_last_cuda_error; }

size_t b2r_sizeof(int which) {
  switch (which) {
    case 0: return sizeof(B2RScene);
    case 1: return sizeof(B2RStatus);
    case 2: return sizeof(B2RWorkspace);
    case 3: return sizeof(B2RForwardOutputs);
    case 4: return sizeof(B2RBackwardArgs);
    case 5: return sizeof(B2RView);
    case 6: return sizeof(B2RSkin);
    case 8: return sizeof(B2RMeshRender);  // 7 stays unused
    case 10: return sizeof(B2RGnMlp);  // 9 stays unused
    case 11: return sizeof(B2RRegs);
    case 12: return sizeof(B2RRegsGrads);
    case 13: return sizeof(B2RRig);
    case 14: return sizeof(B2RRigGrads);
    case 15: return sizeof(B2RAdamSegment);
    case 16: return sizeof(B2RLpips);
    case 17: return sizeof(B2RSceneAssets);
    case 18: return sizeof(B2RSceneAssetsGrads);
    case 19: return sizeof(B2RSmplxPose);
    case 20: return sizeof(B2RSmplxPoseGrads);
    case 21: return sizeof(B2RHumanAssets);
    case 22: return sizeof(B2RHumanAssetsGrads);
    case 23: return sizeof(B2RSmplxBody);
    case 24: return sizeof(B2RSmplxBodyGrads);
    case 25: return sizeof(B2RNeumanScores);
    case 26: return sizeof(B2RFaceComposite);
    case 27: return sizeof(B2RTestOutputs);
    case 28: return sizeof(B2ROrbitCamera);
    case 29: return sizeof(B2RAnimationPanel);
    case 31: return sizeof(B2RSmplxParamTable);  // 30 stays unused
    case 32: return sizeof(B2RSmplxParamTableGrads);
    case 33: return sizeof(B2RFrameTable);
    case 34: return sizeof(B2RSegmentation);
    default: return 0;
  }
}

size_t b2r_ctx_bytes(int32_t P, int32_t width, int32_t height) { return ctx_layout(P, width, height).total; }

size_t b2r_scratch_bytes(int32_t P, int32_t width, int32_t height, uint64_t dup_capacity) {
  return scratch_layout(P, width, height, dup_capacity).total;
}

size_t b2r_backward_scratch_bytes(int32_t P) { return align_up((size_t)(P > 0 ? P : 1) * 12 * sizeof(float)); }

size_t b2r_checkpoint_bytes(int32_t width, int32_t height, uint64_t dup_capacity) {
  const CtxLayout L = ctx_layout(0, width, height);
  const uint32_t ms = max_segments(L.tiles, dup_capacity);
  return seg_table_bytes(ms) + (size_t)ms * CK_REC_BYTES;
}

int b2r_forward_project(const B2RScene* scene, const B2RWorkspace* ws, int32_t* radii, void* stream) {
  int rc = validate_scene(scene);
  if (rc) return rc;
  rc = validate_ws(scene, ws, false);
  if (rc) return rc;
  if (scene->P > 0 && !radii) return B2R_E_INVALID;
  const Ctx cx = resolve(ws, scene->P, scene->width, scene->height);
  return launch_project(*scene, cx, radii, (cudaStream_t)stream);
}

static int forward_render(const B2RScene* scene, const B2RWorkspace* ws, const B2RForwardOutputs* out, bool rescan,
                          void* stream) {
  int rc = validate_scene(scene);
  if (rc) return rc;
  rc = validate_ws(scene, ws, true);
  if (rc) return rc;
  if (!out || !out->color || !out->depth || !out->alpha) return B2R_E_INVALID;
  const Ctx cx = resolve(ws, scene->P, scene->width, scene->height);
  rc = launch_binning(*scene, cx, rescan, (cudaStream_t)stream);
  if (rc) return rc;
  return launch_composite_fwd(*scene, cx, *out, (cudaStream_t)stream);
}

// a view narrows the Gaussian range, swaps the background and redirects the per-pixel state / checkpoint records
static int apply_view(Ctx& cx, const B2RScene* scene, const B2RWorkspace* ws, const B2RView* v) {
  if (!v) return B2R_OK;
  if (v->id_end < v->id_begin || (int64_t)v->id_end > (int64_t)scene->P) return B2R_E_INVALID;
  if ((v->final_T != nullptr) != (v->n_contrib != nullptr)) return B2R_E_INVALID;
  cx.id_begin = v->id_begin;
  cx.id_span = v->id_end - v->id_begin;
  cx.bg = v->bg;
  cx.skip_below = v->skip_below;
  if (v->final_T) { cx.final_T = v->final_T; cx.n_contrib = v->n_contrib; }
  if (v->checkpoints && cx.ckpt) {  // records only; the segment table is the workspace's (one per binned scene)
    const size_t need = seg_table_bytes(cx.max_segs) + (size_t)cx.max_segs * CK_REC_BYTES;
    if (v->checkpoint_bytes < need) return B2R_E_WORKSPACE;
    cx.ckpt = (float*)((char*)v->checkpoints + seg_table_bytes(cx.max_segs));
  }
  (void)ws;
  return B2R_OK;
}

int b2r_forward_bin(const B2RScene* scene, const B2RWorkspace* ws, void* stream) {
  int rc = validate_scene(scene);
  if (rc) return rc;
  rc = validate_ws(scene, ws, true);
  if (rc) return rc;
  const Ctx cx = resolve(ws, scene->P, scene->width, scene->height);
  return launch_binning(*scene, cx, false, (cudaStream_t)stream);
}

size_t b2r_split_scratch_bytes(int32_t P, int32_t width, int32_t height, uint64_t dup_capacity) {
  return split_scratch_bytes(P, width, height, dup_capacity);
}

int b2r_forward_project_split(const B2RScene* scene, const B2RWorkspace* ws, uint32_t first_row, int32_t* radii,
                              void* stream) {
  int rc = validate_scene(scene);
  if (rc) return rc;
  rc = validate_ws(scene, ws, false);
  if (rc) return rc;
  if ((int64_t)first_row > (int64_t)scene->P) return B2R_E_INVALID;
  if (ws->dup_capacity == 0) return B2R_E_INVALID;  // the split pass bins with the capacity it was given
  if (scene->P > 0 && !radii) return B2R_E_INVALID;
  const Ctx cx = resolve(ws, scene->P, scene->width, scene->height);
  return launch_project(*scene, cx, radii, (cudaStream_t)stream, (int)first_row);
}

int b2r_forward_bin_split(const B2RScene* scene, const B2RWorkspace* ws, const B2RWorkspace* base, uint32_t first_row,
                          int32_t* radii, void* stream) {
  int rc = validate_scene(scene);
  if (rc) return rc;
  rc = validate_ws(scene, ws, true);
  if (rc) return rc;
  if ((int64_t)first_row > (int64_t)scene->P) return B2R_E_INVALID;
  if (ws->dup_capacity == 0 || (scene->P > 0 && !radii)) return B2R_E_INVALID;
  if (ws->scratch_bytes < split_scratch_bytes(scene->P, scene->width, scene->height, ws->dup_capacity))
    return B2R_E_WORKSPACE;
  if (!base || base == ws || !base->ctx || !base->dup_ids) return B2R_E_INVALID;
  if (base->ctx_bytes < b2r_ctx_bytes(scene->P, scene->width, scene->height)) return B2R_E_WORKSPACE;
  Ctx cx = resolve(ws, scene->P, scene->width, scene->height);
  cx.sort_len = (uint32_t*)((char*)ws->ctx + ctx_layout(scene->P, scene->width, scene->height).split_len);
  const Ctx bx = resolve(base, scene->P, scene->width, scene->height);
  uint32_t* own_ids = (uint32_t*)((char*)ws->scratch + scratch_layout(scene->P, scene->width, scene->height,
                                                                      ws->dup_capacity).total);
  return launch_binning_split(*scene, cx, bx, own_ids, (int)first_row, radii, (cudaStream_t)stream);
}

int b2r_forward_composite(const B2RScene* scene, const B2RWorkspace* ws, const B2RView* view,
                          const B2RForwardOutputs* out, void* stream) {
  int rc = validate_scene(scene);
  if (rc) return rc;
  rc = validate_ws(scene, ws, false);
  if (rc) return rc;
  if (!out || !out->color || !out->depth || !out->alpha) return B2R_E_INVALID;
  Ctx cx = resolve(ws, scene->P, scene->width, scene->height);
  rc = apply_view(cx, scene, ws, view);
  if (rc) return rc;
  return launch_composite_fwd(*scene, cx, *out, (cudaStream_t)stream);
}

int b2r_forward_render(const B2RScene* scene, const B2RWorkspace* ws, const B2RForwardOutputs* out, void* stream) {
  return forward_render(scene, ws, out, true, stream);
}

int b2r_forward(const B2RScene* scene, const B2RWorkspace* ws, const B2RForwardOutputs* out, void* stream) {
  if (!out) return B2R_E_INVALID;
  int rc = b2r_forward_project(scene, ws, out->radii, stream);
  if (rc) return rc;
  return forward_render(scene, ws, out, false, stream);
}

int b2r_backward(const B2RScene* scene, const B2RWorkspace* ws, const B2RBackwardArgs* args, void* bwd_scratch,
                 size_t bwd_scratch_bytes, void* stream) {
  int rc = validate_scene(scene);
  if (rc) return rc;
  rc = validate_ws(scene, ws, false);
  if (rc) return rc;
  if (!args || !args->dL_dcolor || !bwd_scratch) return B2R_E_INVALID;
  if (bwd_scratch_bytes < b2r_backward_scratch_bytes(scene->P)) return B2R_E_WORKSPACE;
  if (missing_dshs(scene, args)) return B2R_E_INVALID;
  if ((int64_t)args->first_row > (int64_t)scene->P) return B2R_E_INVALID;
  const Ctx cx = resolve(ws, scene->P, scene->width, scene->height);
  float* gacc = (float*)bwd_scratch;
  rc = launch_composite_bwd(*scene, cx, *args, gacc, (cudaStream_t)stream);
  if (rc) return rc;
  return launch_project_bwd(*scene, cx, *args, gacc, (cudaStream_t)stream);
}

int b2r_backward_composite(const B2RScene* scene, const B2RWorkspace* ws, const B2RView* view, const B2RBackwardArgs* args,
                           void* bwd_scratch, size_t bwd_scratch_bytes, void* stream) {
  int rc = validate_scene(scene);
  if (rc) return rc;
  rc = validate_ws(scene, ws, false);
  if (rc) return rc;
  if (!args || !args->dL_dcolor || !bwd_scratch) return B2R_E_INVALID;
  if (bwd_scratch_bytes < b2r_backward_scratch_bytes(scene->P)) return B2R_E_WORKSPACE;
  if ((int64_t)args->first_row > (int64_t)scene->P) return B2R_E_INVALID;
  Ctx cx = resolve(ws, scene->P, scene->width, scene->height);
  rc = apply_view(cx, scene, ws, view);
  if (rc) return rc;
  return launch_composite_bwd(*scene, cx, *args, (float*)bwd_scratch, (cudaStream_t)stream);
}

int b2r_backward_project(const B2RScene* scene, const B2RWorkspace* ws, const B2RBackwardArgs* args, void* bwd_scratch,
                         size_t bwd_scratch_bytes, void* stream) {
  int rc = validate_scene(scene);
  if (rc) return rc;
  rc = validate_ws(scene, ws, false);
  if (rc) return rc;
  if (!args || !bwd_scratch) return B2R_E_INVALID;
  if (bwd_scratch_bytes < b2r_backward_scratch_bytes(scene->P)) return B2R_E_WORKSPACE;
  if (missing_dshs(scene, args)) return B2R_E_INVALID;
  if ((int64_t)args->first_row > (int64_t)scene->P) return B2R_E_INVALID;
  const Ctx cx = resolve(ws, scene->P, scene->width, scene->height);
  return launch_project_bwd(*scene, cx, *args, (const float*)bwd_scratch, (cudaStream_t)stream);
}

size_t b2r_skin_scratch_bytes(int32_t P, int32_t J) { return skin_scratch_bytes(P, J); }

int b2r_skin_forward(const B2RSkin* skin, void* stream) {
  const int rc = validate_skin(skin);
  if (rc) return rc;
  if (skin->P > 0 && !skin->posed[0]) return B2R_E_INVALID;
  return launch_skin_forward(*skin, (cudaStream_t)stream);
}

int b2r_skin_backward(const B2RSkin* skin, const float* const dL_dpos[2], float* const dL_dxyz[2], float* dL_djoint,
                      float* dL_dtrans, void* scratch, size_t scratch_bytes, void* stream) {
  const int rc = validate_skin(skin);
  if (rc) return rc;
  if (dL_dpos && dL_dpos[1] && !skin->xyz[1]) return B2R_E_INVALID;
  if ((dL_djoint || dL_dtrans) && skin->P > 0) {
    if (!scratch) return B2R_E_INVALID;
    if (scratch_bytes < skin_scratch_bytes(skin->P, skin->J)) return B2R_E_WORKSPACE;
  }
  return launch_skin_backward(*skin, dL_dpos, dL_dxyz, dL_djoint, dL_dtrans, scratch, (cudaStream_t)stream);
}

size_t b2r_l1ssim_scratch_bytes(int32_t width, int32_t height) { return l1ssim_scratch_bytes(width, height); }

int b2r_l1ssim_forward(int32_t width, int32_t height, const float* img, const float* target, const float* mask,
                       const float* bbox, int32_t with_ssim, float* out, void* scratch, size_t scratch_bytes,
                       void* stream) {
  if (!valid_l1ssim_size(width, height) || !img || !target || !out || !scratch) return B2R_E_INVALID;
  if (scratch_bytes < l1ssim_scratch_bytes(width, height)) return B2R_E_WORKSPACE;
  return launch_l1ssim_forward(width, height, img, target, mask, bbox, with_ssim != 0, out, scratch,
                               (cudaStream_t)stream);
}

int b2r_l1ssim_backward(int32_t width, int32_t height, const float* img, const float* target, const float* mask,
                        const float* bbox, int32_t with_ssim, const float* dL_dout, float* dL_dimg, const void* scratch,
                        size_t scratch_bytes, void* stream) {
  if (!valid_l1ssim_size(width, height) || !img || !target || !dL_dout || !dL_dimg) return B2R_E_INVALID;
  if (with_ssim) {  // the forward's per-pixel SSIM partials
    if (!scratch) return B2R_E_INVALID;
    if (scratch_bytes < l1ssim_scratch_bytes(width, height)) return B2R_E_WORKSPACE;
  }
  return launch_l1ssim_backward(width, height, img, target, mask, bbox, with_ssim != 0, dL_dout, dL_dimg, scratch,
                                (cudaStream_t)stream);
}

size_t b2r_nearest_scratch_bytes(int32_t P, int32_t V) {
  (void)P;  // the grid is sized from the targets alone
  return nearest_scratch_bytes(V);
}

int b2r_nearest_rows(int32_t P, const float* queries, int32_t V, const float* targets, const uint8_t* self_map,
                     int32_t* rows, void* scratch, size_t scratch_bytes, void* stream) {
  if (P < 0 || V < 0 || V >= (1 << 29)) return B2R_E_INVALID;  // cell counts 2V + 64 stay in int32
  if (P == 0) return B2R_OK;
  if (V < 1 || !queries || !targets || !rows || !scratch) return B2R_E_INVALID;
  if (scratch_bytes < nearest_scratch_bytes(V)) return B2R_E_WORKSPACE;
  return launch_nearest_rows(P, queries, V, targets, self_map, rows, scratch, (cudaStream_t)stream);
}

int b2r_vertex_normals(int32_t P, const float* xyz, const int32_t* faces, const int32_t* vf_offsets,
                       const int32_t* vf_entries, const uint8_t* flip, float* normals, void* stream) {
  if (P < 0) return B2R_E_INVALID;
  if (P == 0) return B2R_OK;
  if (!xyz || !faces || !vf_offsets || !vf_entries || !normals) return B2R_E_INVALID;
  return launch_vertex_normals(P, xyz, faces, vf_offsets, vf_entries, flip, normals, (cudaStream_t)stream);
}

size_t b2r_mesh_render_scratch_bytes(int32_t F) { return mesh_render_scratch_bytes(F); }

int b2r_mesh_render_forward(const B2RMeshRender* mr, float* image, int32_t* pix_to_face, void* scratch,
                            size_t scratch_bytes, void* stream) {
  const int rc = validate_mesh_render(mr);
  if (rc) return rc;
  if (!mr->keys || !image || !pix_to_face || !scratch) return B2R_E_INVALID;
  if (scratch_bytes < mesh_render_scratch_bytes(mr->F)) return B2R_E_WORKSPACE;
  return launch_mesh_render_forward(*mr, image, pix_to_face, scratch, (cudaStream_t)stream);
}

int b2r_mesh_render_backward(const B2RMeshRender* mr, const int32_t* pix_to_face, const float* dL_dimage,
                             float* dL_dmesh, void* scratch, size_t scratch_bytes, void* stream) {
  const int rc = validate_mesh_render(mr);
  if (rc) return rc;
  if (!pix_to_face || !dL_dimage || !scratch) return B2R_E_INVALID;
  if (mr->V > 0 && (!dL_dmesh || !mr->vf_offsets || !mr->vf_entries)) return B2R_E_INVALID;
  if (scratch_bytes < mesh_render_scratch_bytes(mr->F)) return B2R_E_WORKSPACE;
  return launch_mesh_render_backward(*mr, pix_to_face, dL_dimage, dL_dmesh, scratch, (cudaStream_t)stream);
}

int b2r_mesh_shade_forward(const B2RMeshRender* mr, const float* normals, const float* bkg, float blend,
                           float blend_complement, float* out, void* scratch, size_t scratch_bytes, void* stream) {
  const int rc = validate_mesh_shade(mr);
  if (rc) return rc;
  if (mr->F > 0 && !normals) return B2R_E_INVALID;
  if (!bkg || !out || !scratch || !std::isfinite(blend) || !std::isfinite(blend_complement)) return B2R_E_INVALID;
  if (scratch_bytes < mesh_render_scratch_bytes(mr->F)) return B2R_E_WORKSPACE;
  return launch_mesh_shade_forward(*mr, normals, bkg, blend, blend_complement, out, scratch, (cudaStream_t)stream);
}

int b2r_triplane_forward(int32_t P, int32_t C, int32_t height, int32_t width, const float* planes,
                         const float* planes_face, const uint8_t* is_face, const int32_t* corners, const float* weights,
                         float* feat, void* stream) {
  if (!valid_triplane(P, C, height, width)) return B2R_E_INVALID;
  if (P == 0) return B2R_OK;
  if (!planes || !planes_face || !corners || !weights || !feat) return B2R_E_INVALID;
  return launch_triplane_forward(P, C, height, width, planes, planes_face, is_face, corners, weights, feat,
                                 (cudaStream_t)stream);
}

int b2r_triplane_backward(int32_t P, int32_t C, int32_t height, int32_t width, const float* dfeat,
                          const int32_t* offsets, const int32_t* rows, const float* w, float* dplanes,
                          float* dplanes_face, void* stream) {
  if (!valid_triplane(P, C, height, width)) return B2R_E_INVALID;
  if (!offsets || !dplanes || !dplanes_face || (P > 0 && (!dfeat || !rows || !w))) return B2R_E_INVALID;
  return launch_triplane_backward(C, height, width, dfeat, offsets, rows, w, dplanes, dplanes_face,
                                  (cudaStream_t)stream);
}

size_t b2r_gn_mlp_scratch_bytes(int32_t P) { return gn_mlp_scratch_bytes(P); }
size_t b2r_gn_mlp_grads_count(int32_t K, int32_t H) { return gn_mlp_grads_count(K, H); }

int b2r_gn_mlp_forward(const B2RGnMlp* m, float* out, float* saved, void* stream) {
  const int rc = validate_gn_mlp(m);
  if (rc) return rc;
  if (!out) return B2R_E_INVALID;
  return launch_gn_mlp_forward(*m, out, saved, (cudaStream_t)stream);
}

int b2r_gn_mlp_backward(const B2RGnMlp* m, const float* saved, const float* dL_dout, float* dL_dx, float* grads,
                        void* scratch, size_t scratch_bytes, void* stream) {
  const int rc = validate_gn_mlp(m);
  if (rc) return rc;
  if (!saved || !dL_dout || !grads || !scratch) return B2R_E_INVALID;
  if (scratch_bytes < gn_mlp_scratch_bytes(m->P)) return B2R_E_WORKSPACE;
  return launch_gn_mlp_backward(*m, saved, dL_dout, dL_dx, grads, scratch, (cudaStream_t)stream);
}

size_t b2r_regs_scratch_bytes(int32_t P, int32_t n_arm) { return regs_scratch_bytes(P, n_arm); }

int b2r_regs_forward(const B2RRegs* r, float* out, void* scratch, size_t scratch_bytes, void* stream) {
  const int rc = validate_regs(r);
  if (rc) return rc;
  if (!out || !scratch) return B2R_E_INVALID;
  if (scratch_bytes < regs_scratch_bytes(r->P, r->n_arm)) return B2R_E_WORKSPACE;
  return launch_regs_forward(*r, out, scratch, (cudaStream_t)stream);
}

int b2r_regs_backward(const B2RRegs* r, const float* dL_dout, const B2RRegsGrads* grads, const void* scratch,
                      size_t scratch_bytes, void* stream) {
  const int rc = validate_regs(r);
  if (rc) return rc;
  if (!dL_dout || !grads || !scratch) return B2R_E_INVALID;
  if (!grads->mean_offset || !grads->mean_offset_offset || !grads->scale_offset || !grads->scale ||
      !grads->scale_refined || !grads->rgb || !grads->rgb_refined || !grads->joint_offset ||
      (r->scale_reg && !grads->scale_reg))
    return B2R_E_INVALID;
  if (scratch_bytes < regs_scratch_bytes(r->P, r->n_arm)) return B2R_E_WORKSPACE;
  return launch_regs_backward(*r, dL_dout, *grads, scratch, (cudaStream_t)stream);
}

size_t b2r_rig_scratch_bytes(int32_t V, int32_t J, int32_t NB, int32_t NE) { return rig_scratch_bytes(V, J, NB, NE); }

int b2r_rig_forward(const B2RRig* r, float* mesh, float* mesh_wo, float* joint_mats, float* pose_offset,
                    float* expr_offset, float* pose_6d, void* scratch, size_t scratch_bytes, void* stream) {
  const int rc = validate_rig(r);
  if (rc) return rc;
  if (!mesh || !mesh_wo || !joint_mats || !pose_offset || !expr_offset || !pose_6d || !scratch) return B2R_E_INVALID;
  if (scratch_bytes < rig_scratch_bytes(r->V, r->J, r->NB, r->NE)) return B2R_E_WORKSPACE;
  return launch_rig_forward(*r, mesh, mesh_wo, joint_mats, pose_offset, expr_offset, pose_6d, scratch,
                            (cudaStream_t)stream);
}

int b2r_rig_backward(const B2RRig* r, const float* dL_dmesh, const float* dL_djoint_mats, const float* dL_dexpr_offset,
                     const B2RRigGrads* grads, void* scratch, size_t scratch_bytes, void* stream) {
  const int rc = validate_rig(r);
  if (rc) return rc;
  if (!grads || !grads->shape_param || !grads->joint_offset || !grads->full_pose || !grads->expr || !scratch)
    return B2R_E_INVALID;
  if (scratch_bytes < rig_scratch_bytes(r->V, r->J, r->NB, r->NE)) return B2R_E_WORKSPACE;
  return launch_rig_backward(*r, dL_dmesh, dL_djoint_mats, dL_dexpr_offset, *grads, scratch, (cudaStream_t)stream);
}

size_t b2r_smplx_body_scratch_bytes(int32_t V, int32_t J) {
  (void)J;  // the joint buffers are sized for 64 joints
  return smplx_body_scratch_bytes(V);
}

int b2r_smplx_body_forward(const B2RSmplxBody* b, float* mesh, void* scratch, size_t scratch_bytes, void* stream) {
  const int rc = validate_body(b);
  if (rc) return rc;
  if (!mesh || !scratch) return B2R_E_INVALID;
  if (scratch_bytes < smplx_body_scratch_bytes(b->rig.V)) return B2R_E_WORKSPACE;
  return launch_smplx_body_forward(*b, mesh, scratch, (cudaStream_t)stream);
}

int b2r_smplx_body_backward(const B2RSmplxBody* b, const float* dL_dmesh, const B2RSmplxBodyGrads* grads,
                            void* scratch, size_t scratch_bytes, void* stream) {
  const int rc = validate_body(b);
  if (rc) return rc;
  if (!grads || !grads->shape_param || !grads->joint_offset || !grads->full_pose || !grads->expr || !grads->trans ||
      !scratch)
    return B2R_E_INVALID;
  if (scratch_bytes < smplx_body_scratch_bytes(b->rig.V)) return B2R_E_WORKSPACE;
  return launch_smplx_body_backward(*b, dL_dmesh, *grads, scratch, (cudaStream_t)stream);
}

int64_t b2r_adam_chunk_elems(void) { return B2R_ADAM_CHUNK; }

int b2r_adam_step(const B2RAdamSegment* table, int32_t n_segments, int64_t n_chunks, void* stream) {
  if (n_segments < 0 || n_chunks < 0 || n_chunks > 0x7fffffff) return B2R_E_INVALID;  // one CTA per chunk: grid.x
  if (n_segments > 0 && !table) return B2R_E_INVALID;
  if (n_chunks > 0 && n_segments == 0) return B2R_E_INVALID;
  if (n_chunks == 0) return B2R_OK;
  return launch_adam_step(table, n_segments, n_chunks, (cudaStream_t)stream);
}

size_t b2r_lpips_saved_bytes(int32_t width, int32_t height, int32_t n_images) {
  return lpips_saved_bytes(width > 0 ? width : 1, height > 0 ? height : 1, n_images > 0 ? n_images : 1);
}
size_t b2r_lpips_scratch_bytes(int32_t width, int32_t height) {
  return lpips_scratch_bytes(width > 0 ? width : 1, height > 0 ? height : 1);
}

int b2r_lpips_forward(const B2RLpips* p, float* out, void* saved, size_t saved_bytes, void* scratch,
                      size_t scratch_bytes, void* stream) {
  const int rc = validate_lpips(p);
  if (rc) return rc;
  if (!out || !saved || !scratch) return B2R_E_INVALID;
  if (saved_bytes < lpips_saved_bytes(p->width, p->height, p->n_images) ||
      scratch_bytes < lpips_scratch_bytes(p->width, p->height))
    return B2R_E_WORKSPACE;
  return launch_lpips_forward(*p, out, (float*)saved, scratch, (cudaStream_t)stream);
}

int b2r_lpips_backward(const B2RLpips* p, const void* saved, size_t saved_bytes, const float* dL_dout, float* dL_dimg,
                       void* scratch, size_t scratch_bytes, void* stream) {
  const int rc = validate_lpips(p);
  if (rc) return rc;
  if (!saved || !dL_dout || !dL_dimg || !scratch) return B2R_E_INVALID;
  if (saved_bytes < lpips_saved_bytes(p->width, p->height, p->n_images) ||
      scratch_bytes < lpips_scratch_bytes(p->width, p->height))
    return B2R_E_WORKSPACE;
  return launch_lpips_backward(*p, (const float*)saved, dL_dout, dL_dimg, scratch, (cudaStream_t)stream);
}

size_t b2r_neuman_scratch_bytes(int32_t width, int32_t height, int32_t n_images) {
  return neuman_scratch_bytes(width > 31 ? width : 31, height > 31 ? height : 31, n_images > 0 ? n_images : 1);
}

int b2r_neuman_scores(const B2RNeumanScores* p, float* out, void* scratch, size_t scratch_bytes, void* stream) {
  const int rc = validate_neuman(p);
  if (rc) return rc;
  if (!out || !scratch) return B2R_E_INVALID;
  if (scratch_bytes < neuman_scratch_bytes(p->width, p->height, p->n_images)) return B2R_E_WORKSPACE;
  return launch_neuman_scores(*p, out, scratch, (cudaStream_t)stream);
}

int b2r_face_composite_forward(const B2RFaceComposite* p, float* out, void* stream) {
  if (!p || !p->img || !p->face || !out) return B2R_E_INVALID;
  const int rc = validate_compose_size(p->width, p->height, p->n_images);
  if (rc) return rc;
  return launch_face_composite_forward(*p, out, (cudaStream_t)stream);
}

int b2r_face_composite_backward(const B2RFaceComposite* p, const float* dout, float* dimg, float* dface, void* stream) {
  if (!p || !p->face || !dout || (!dimg && !dface)) return B2R_E_INVALID;
  const int rc = validate_compose_size(p->width, p->height, p->n_images);
  if (rc) return rc;
  return launch_face_composite_backward(*p, dout, dimg, dface, (cudaStream_t)stream);
}

int b2r_test_outputs(const B2RTestOutputs* p, float* const composite[4], uint8_t* png, void* stream) {
  const int rc = validate_test_outputs(p);
  if (rc) return rc;
  if (!composite) return B2R_E_INVALID;
  for (int k = 0; k < 4; k++)
    if (!composite[k]) return B2R_E_INVALID;
  return launch_test_outputs(*p, composite, png, (cudaStream_t)stream);
}

int b2r_orbit_camera(const B2ROrbitCamera* p, void* stream) {
  if (!p || !p->index || !p->state || p->k <= 0 || p->n_frames <= 0 || p->anchor < 0 || p->anchor > 2)
    return B2R_E_INVALID;
  const bool any_cam = p->cam_R || p->cam_t || p->root_cam, all_cam = p->cam_R && p->cam_t && p->root_cam;
  if (any_cam != all_cam || (p->anchor != 0 && !all_cam)) return B2R_E_INVALID;
  return launch_orbit_camera(*p, (cudaStream_t)stream);
}

int b2r_orbit_points(int32_t n, const float* points, const float* state, int32_t view, float* out, void* stream) {
  if (n <= 0 || !points || !state || !out) return B2R_E_INVALID;
  return launch_orbit_points(n, points, state, view != 0, out, (cudaStream_t)stream);
}

int b2r_animation_panel(const B2RAnimationPanel* p, uint8_t* out, void* stream) {
  if (!p || !p->frame || !p->mesh_panel || !p->render || !out) return B2R_E_INVALID;
  if (p->width <= 0 || p->height <= 0 || (int64_t)p->width * p->height >= (int64_t)1 << 31) return B2R_E_INVALID;
  return launch_animation_panel(*p, out, (cudaStream_t)stream);
}

int b2r_smplx_body_joints(const B2RSmplxBody* b, const void* scratch, size_t scratch_bytes, float* joints,
                          void* stream) {
  const int rc = validate_body(b);
  if (rc) return rc;
  if (!joints || !scratch) return B2R_E_INVALID;
  if (scratch_bytes < smplx_body_scratch_bytes(b->rig.V)) return B2R_E_WORKSPACE;
  return launch_smplx_body_joints(*b, scratch, joints, (cudaStream_t)stream);
}

int b2r_scene_assets_forward(const B2RSceneAssets* s, float* opacity, float* scale, float* rotation, float* color,
                             void* stream) {
  const int rc = validate_scene_assets(s);
  if (rc) return rc;
  if (s->P > 0 && (!opacity || !scale || !rotation || !color)) return B2R_E_INVALID;
  return launch_scene_assets_forward(*s, opacity, scale, rotation, color, (cudaStream_t)stream);
}

int b2r_scene_assets_backward(const B2RSceneAssets* s, const B2RSceneAssetsGrads* g, void* stream) {
  const int rc = validate_scene_assets(s);
  if (rc) return rc;
  if (!g) return B2R_E_INVALID;
  if (s->P > 0) {
    if (!g->opacity || !g->scale || !g->dL_dlogit || !g->dL_dlog_scale || !g->dL_drotation6d || !g->dL_dfeature_dc)
      return B2R_E_INVALID;
    if (s->M > 1 && !g->dL_dfeature_rest) return B2R_E_INVALID;
    if ((s->cam_R != nullptr) != (g->dL_dmean != nullptr)) return B2R_E_INVALID;  // d mean exactly in rgb mode
  }
  return launch_scene_assets_backward(*s, *g, (cudaStream_t)stream);
}

int b2r_decode_pose_forward(const B2RSmplxPose* p, float* full_pose, void* stream) {
  const int rc = validate_pose(p);
  if (rc) return rc;
  if (!full_pose) return B2R_E_INVALID;
  return launch_decode_pose_forward(*p, full_pose, (cudaStream_t)stream);
}

int b2r_decode_pose_backward(const B2RSmplxPose* p, const float* dL_dfull_pose, const B2RSmplxPoseGrads* grads,
                             void* stream) {
  const int rc = validate_pose(p);
  if (rc) return rc;
  if (!dL_dfull_pose || !grads) return B2R_E_INVALID;
  for (int k = 0; k < B2R_POSE_PARAMS; ++k)
    if (p->rows[k] > 0 && !grads->param[k]) return B2R_E_INVALID;
  return launch_decode_pose_backward(*p, dL_dfull_pose, *grads, (cudaStream_t)stream);
}

int b2r_param_table_forward(const B2RSmplxParamTable* t, float* full_pose, float* expr, float* trans, void* stream) {
  const int rc = validate_param_table(t);
  if (rc) return rc;
  if (!full_pose || !trans || (t->n_expr > 0 && !expr)) return B2R_E_INVALID;
  return launch_param_table_forward(*t, full_pose, expr, trans, (cudaStream_t)stream);
}

int b2r_param_table_backward(const B2RSmplxParamTable* t, const B2RSmplxParamTableGrads* g, void* stream) {
  const int rc = validate_param_table(t);
  if (rc) return rc;
  if (!g || !g->pose || !g->trans || (t->n_expr > 0 && !g->expr)) return B2R_E_INVALID;
  return launch_param_table_backward(*t, *g, (cudaStream_t)stream);
}

int b2r_frame_unpack(const B2RFrameTable* table, float* img, float* mask, float* bbox, float* R, float* t,
                     float* focal, float* princpt, int64_t* frame_idx, void* stream) {
  const int rc = validate_frame_table(table);
  if (rc) return rc;
  if (!img || !mask || !bbox || !R || !t || !focal || !princpt || !frame_idx) return B2R_E_INVALID;
  return launch_frame_unpack(*table, img, mask, bbox, R, t, focal, princpt, frame_idx, (cudaStream_t)stream);
}

int b2r_segmentation_unpack(const B2RSegmentation* seg, float* mask, void* stream) {
  const int rc = validate_segmentation(seg);
  if (rc) return rc;
  if (!mask) return B2R_E_INVALID;
  return launch_segmentation_unpack(*seg, mask, (cudaStream_t)stream);
}

int b2r_human_geometry_forward(const B2RHumanAssets* h, float* mean_3d, float* mean_3d_refined, float* scale,
                               float* scale_refined, float* mean_offset_offset, float* scale_wo_clamp,
                               float* scale_refined_wo_clamp, void* stream) {
  const int rc = validate_human_assets(h);
  if (rc) return rc;
  if (h->P > 0) {
    if (!mean_3d || !mean_3d_refined || !scale || !scale_refined || !mean_offset_offset) return B2R_E_INVALID;
    if (h->warmup && (!scale_wo_clamp || !scale_refined_wo_clamp)) return B2R_E_INVALID;
  }
  return launch_human_geometry_forward(*h, mean_3d, mean_3d_refined, scale, scale_refined, mean_offset_offset,
                                       scale_wo_clamp, scale_refined_wo_clamp, (cudaStream_t)stream);
}

int b2r_human_geometry_backward(const B2RHumanAssets* h, const B2RHumanAssetsGrads* g, void* stream) {
  const int rc = validate_human_assets(h);
  if (rc) return rc;
  if (!g) return B2R_E_INVALID;
  if (h->P > 0 && (!g->dL_dmesh || !g->dL_dexpr_offset || !g->dL_dgeo || !g->dL_dgeo_offset)) return B2R_E_INVALID;
  return launch_human_geometry_backward(*h, *g, (cudaStream_t)stream);
}

int b2r_human_colors_forward(int32_t P, const float* rgb, const float* rgb_offset, float* rgb_out, float* rgb_refined,
                             void* stream) {
  if (P < 0 || (P > 0 && (!rgb || !rgb_offset || !rgb_out || !rgb_refined))) return B2R_E_INVALID;
  return launch_human_colors_forward(P, rgb, rgb_offset, rgb_out, rgb_refined, (cudaStream_t)stream);
}

int b2r_human_colors_backward(int32_t P, const float* rgb, const float* rgb_offset, const float* dL_drgb_out,
                              const float* dL_drgb_refined, float* dL_drgb, float* dL_drgb_offset, void* stream) {
  if (P < 0 || (P > 0 && (!rgb || !rgb_offset || !dL_drgb || !dL_drgb_offset))) return B2R_E_INVALID;
  return launch_human_colors_backward(P, rgb, rgb_offset, dL_drgb_out, dL_drgb_refined, dL_drgb, dL_drgb_offset,
                                      (cudaStream_t)stream);
}

int b2r_camera_setup(const float* R, const float* t, const float* focal, int32_t width, int32_t height, float* out,
                     void* stream) {
  if (!R || !t || !focal || !out || width <= 0 || height <= 0) return B2R_E_INVALID;
  return launch_camera_setup(R, t, focal, width, height, out, (cudaStream_t)stream);
}

int b2r_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, uint8_t* present, void* stream) {
  if (P < 0 || (P > 0 && (!means3D || !present)) || !viewmatrix) return B2R_E_INVALID;
  return launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)stream);
}

const float* b2r_ctx_geom(const B2RWorkspace* ws, int32_t P, int32_t width, int32_t height) {
  return (const float*)((const char*)ws->ctx + ctx_layout(P, width, height).geom);
}
const int32_t* b2r_ctx_aux(const B2RWorkspace* ws, int32_t P, int32_t width, int32_t height) {
  return (const int32_t*)((const char*)ws->ctx + ctx_layout(P, width, height).aux);
}
const uint32_t* b2r_ctx_ranges(const B2RWorkspace* ws, int32_t P, int32_t width, int32_t height) {
  return (const uint32_t*)((const char*)ws->ctx + ctx_layout(P, width, height).ranges);
}
const float* b2r_ctx_final_T(const B2RWorkspace* ws, int32_t P, int32_t width, int32_t height) {
  return (const float*)((const char*)ws->ctx + ctx_layout(P, width, height).final_T);
}
const uint32_t* b2r_ctx_n_contrib(const B2RWorkspace* ws, int32_t P, int32_t width, int32_t height) {
  return (const uint32_t*)((const char*)ws->ctx + ctx_layout(P, width, height).n_contrib);
}

}  // extern "C"
