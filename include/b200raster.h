/*
 * b200raster.h -- C ABI of the H100-native (sm_90a) differentiable 3D-Gaussian rasteriser.
 *
 * Drop-in boundary for the one hot path of mks0601/ExAvatar_RELEASE: the rasteriser that
 * `GaussianRenderer.forward` reaches through `GaussianRasterizer(raster_settings)(...)`
 * (avatar/common/nets/module.py:609-640).  The reference binds that path through a third-party
 * pybind module (`diff_gaussian_rasterization_depth._C`, module.py:11, not vendored); the entry
 * points below are what that binding would call instead:
 *
 *   reference interface (file:line / upstream symbol)                    replaced by
 *   ------------------------------------------------------------------   -------------------------
 *   _C.rasterize_gaussians(...)        <- module.py:632-640 forward      b2r_forward_project +
 *                                                                        b2r_forward_render (or b2r_forward)
 *   _C.rasterize_gaussians_backward(.) <- loss.backward(), train.py:46   b2r_backward
 *   _C.mark_visible(...)               <- GaussianRasterizer.markVisible b2r_mark_visible
 *   geom/binning/img byte arenas owned by the autograd ctx               B2RWorkspace (caller-owned)
 *
 * Rules of the boundary: plain pointers and sizes only (no torch / STL types); every pointer is a
 * DEVICE pointer unless its comment says host; the library never allocates device memory, never
 * synchronises the stream and never throws -- it returns 0 or a negative B2R_E_* code.  All work is
 * enqueued on the caller's `stream` (a cudaStream_t passed as void*).
 *
 * Matrix layout (what ExAvatar hands over, module.py:605-607): `viewmatrix` / `projmatrix` are 16
 * floats with element (r,c) of the mathematical matrix at [4*c + r].
 */
#ifndef B200RASTER_H_
#define B200RASTER_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2R_ABI_VERSION 4

#define B2R_OK 0
#define B2R_E_INVALID (-1)      /* bad argument (null pointer, negative size, both / neither colour source, sh_rows > P ...) */
#define B2R_E_WORKSPACE (-2)    /* ctx / scratch buffer smaller than b2r_*_bytes() reports */
#define B2R_E_CUDA (-3)         /* a CUDA launch failed; b2r_last_cuda_error() has the cudaError_t */
#define B2R_E_DUP_OVERFLOW (-4) /* only ever reported through B2RStatus.overflow (device side) */

/* flags */
#define B2R_FLAG_NO_TILE_CULL 1u /* keep every tile of the 3-sigma rect (reference list membership, for list parity tests) */
#define B2R_FLAG_DEBUG 2u        /* reference `debug=True` (module.py:621): the host wrapper syncs and checks after the call */
#define B2R_FLAG_CTX_CLEAN 4u    /* the ctx buffer's counters are zero: its last use was a b2r_forward / b2r_forward_project
                                    with dup_capacity > 0 (or b2r_forward_render) of this library, which leave them zero
                                    again -- the projection then skips its reset launch.  Never set it for a fresh buffer. */

/* Scene description shared by forward and backward: the fields of GaussianRasterizationSettings
 * (module.py:609-622) plus the per-Gaussian inputs of the call (module.py:632-640). */
typedef struct B2RScene {
  int32_t P;              /* number of Gaussians */
  int32_t width, height;  /* image_width, image_height */
  int32_t sh_degree;      /* active SH degree (0..3); ignored when only colors_precomp is set */
  int32_t sh_coeffs;      /* M: coefficients per Gaussian in `shs` (0 when shs == NULL) */
  uint32_t flags;         /* B2R_FLAG_* */
  float scale_modifier;
  float tanfovx, tanfovy;
  const float* bg;            /* (3) */
  const float* viewmatrix;    /* (16) world->view, [4c+r] */
  const float* projmatrix;    /* (16) full projection (proj*view), [4c+r] */
  const float* campos;        /* (3) */
  const float* means3D;       /* (P,3) */
  const float* shs;           /* (P,M,3) or NULL; (sh_rows,M,3) when sh_rows > 0 */
  const float* colors_precomp;/* (P,3) or NULL  (exactly one of shs / colors_precomp, unless sh_rows > 0) */
  const float* opacities;     /* (P) */
  const float* scales;        /* (P,3) or NULL */
  const float* rotations;     /* (P,4) (r,x,y,z), used un-normalised, or NULL */
  const float* cov3D_precomp; /* (P,6) or NULL  (exactly one of scales+rotations / cov3D_precomp) */
  /* Mixed colour source.  0: exactly one of shs / colors_precomp colours every Gaussian.  0 < sh_rows <= P: BOTH are
   * required; Gaussians [0, sh_rows) are coloured from `shs`, which then holds sh_rows rows of sh_coeffs coefficients
   * (sh_degree / sh_coeffs rules as above), and Gaussians [sh_rows, P) read colors_precomp[i] -- the global index, so
   * colors_precomp keeps P rows and its first sh_rows are never read.  This is ExAvatar's cat(scene, human) with the
   * scene coloured from SH and the human from RGB (avatar/main/model.py:117-125).  Backward: dL_dshs has
   * sh_rows - first_row rows (none, and it may be NULL, when first_row >= sh_rows); dL_dcolors is zero on SH rows. */
  int32_t sh_rows;
} B2RScene;

/* Device-side status block; lives at offset 0 of the ctx buffer (read it back with a 64-byte D2H copy). */
typedef struct B2RStatus {
  uint64_t num_dups;      /* (tile, Gaussian) pairs the binning wants to emit */
  uint64_t dup_capacity;  /* capacity the render phase ran with */
  uint32_t overflow;      /* 1 if num_dups > dup_capacity: outputs are truncated, re-run with more room */
  uint32_t num_visible;   /* Gaussians with radii > 0 */
  uint64_t consumed_fwd;  /* list entries staged by the forward composite per tile (C_f of the roofline model), x 8 */
  uint64_t consumed_bwd;  /* list entries staged by the backward composite per tile (C_b), x 4 (one count per quarter tile) */
  uint64_t token;         /* B2RWorkspace.status_token of the project phase that filled this block */
  uint64_t reserved[2];
} B2RStatus; /* 64 bytes */

/* Caller-owned memory for one forward->backward context. */
typedef struct B2RWorkspace {
  void* ctx;             /* >= b2r_ctx_bytes(P,W,H); saved until backward */
  size_t ctx_bytes;
  uint32_t* dup_ids;     /* dup_capacity sorted per-tile Gaussian ids; saved until backward */
  uint64_t dup_capacity;
  void* scratch;         /* >= b2r_scratch_bytes(P,W,H,dup_capacity); free after the call returns + stream order */
  size_t scratch_bytes;
  uint64_t* status_mirror; /* optional device-accessible pointer to 2 x uint64 in pinned HOST memory: the project
                              phase stores {num_dups, status_token} there (in that order) so the host can learn the
                              duplicate count by polling, without a stream synchronisation */
  uint64_t status_token;   /* caller-chosen, e.g. a call counter */
  /* Optional (ABI v3): room for the segment table + per-pixel blend-state checkpoints the forward composite stores at
   * every 512-entry cut of a tile's list, >= b2r_checkpoint_bytes(width, height, dup_capacity); saved until backward.
   * With it the backward composite replays every (quarter tile, 512-entry segment) as an independent work item instead
   * of walking a 2000-entry list on one warp.  NULL: lists are not cut (same results, longer serial chains). */
  void* checkpoints;
  size_t checkpoint_bytes;
} B2RWorkspace;

/* A VIEW of a binned scene (ABI v3; SURVEY section 8f-3).  ExAvatar renders one camera five times per training frame
 * (avatar/main/model.py:130-162): the scene Gaussians, the human Gaussians, and cat(scene, human) -- the same
 * projections, tile lists and depth order every time.  Project + bin cat(scene, human) ONCE (b2r_forward_project,
 * b2r_forward_bin) and composite it several times, each view keeping only the Gaussians of an index range, with its own
 * background and its own per-pixel state; b2r_backward_composite accumulates every view's screen-space gradients into
 * one scratch, b2r_backward_project turns them into parameter gradients once. */
typedef struct B2RView {
  uint32_t id_begin, id_end; /* Gaussians [id_begin, id_end) take part; the others are skipped as if absent */
  const float* bg;           /* (3) background of this view; NULL = scene->bg */
  float* final_T;            /* (H*W) per-pixel final transmittance of this view, saved until its backward; NULL = in ctx */
  uint32_t* n_contrib;       /* (H*W) per-pixel position of the last applied list entry; NULL = in ctx */
  void* checkpoints;         /* this view's checkpoint store (see B2RWorkspace.checkpoints); NULL = the workspace's */
  size_t checkpoint_bytes;
  uint32_t skip_below;       /* != 0: tiles whose list holds no Gaussian of index >= skip_below are SKIPPED -- the forward
                                leaves their pixels of `out` (and of final_T / n_contrib) untouched, the backward adds
                                nothing for them.  For cat(scene.detach(), human) with skip_below = #scene: where no human
                                Gaussian reaches a tile the combined render equals the scene-only view (copy its image
                                into `out` first) and nothing of it carries gradient (model.py:117-125). */
  uint32_t reserved;
} B2RView;

typedef struct B2RForwardOutputs {
  float* color;   /* (3,H,W) */
  float* depth;   /* (H,W)  sum z*alpha*T, no background term */
  float* alpha;   /* (H,W)  sum alpha*T */
  int32_t* radii; /* (P)    3-sigma pixel radius, 0 when culled */
} B2RForwardOutputs;

typedef struct B2RBackwardArgs {
  const float* dL_dcolor; /* (3,H,W) */
  const float* dL_ddepth; /* (H,W) or NULL */
  const float* dL_dalpha; /* (H,W) or NULL */
  /* outputs; every element is written (zeros for culled Gaussians).  Any may be NULL. */
  float* dL_dmeans3D;   /* (P,3) */
  float* dL_dmeans2D;   /* (P,3) NDC-scaled screen gradient, z = 0 (module.py:626-629 reads its .grad) */
  float* dL_dshs;       /* (P,M,3); (sh_rows - first_row, M, 3) in a mixed scene (B2RScene.sh_rows) */
  float* dL_dcolors;    /* (P,3); zero on the SH rows of a mixed scene */
  float* dL_dopacities; /* (P) */
  float* dL_dscales;    /* (P,3) */
  float* dL_drotations; /* (P,4) */
  float* dL_dcov3D;     /* (P,6) */
  uint32_t flags;       /* B2R_BWD_ACCUMULATE: outputs += gradient instead of outputs = gradient, so the frames a rank
                           renders in one step sum into a single bucket that is all-reduced once (SURVEY section 8e) */
  uint32_t first_row;   /* Gaussians [0, first_row) are a DETACHED PREFIX: no gradient is written for them and Gaussian i
                           goes to row i - first_row of every output (outputs then have P - first_row rows).  This is
                           ExAvatar's "scene + human" render, cat(scene.detach(), human) (avatar/main/model.py:117-125):
                           the human part of the gradient lands directly in the human bucket.  0 = off.  The backward
                           projection does not visit whole 256-row blocks below first_row, so (B2R_BWD_SCRATCH_ZEROED)
                           the views composited into its scratch must not accumulate there: their first_row >= this one. */
  /* Optional fused densification bookkeeping (SURVEY section 8f-1), each (P) or NULL, updated IN PLACE for Gaussians
   * with radii > 0 exactly as ExAvatar does after backward (avatar/common/nets/module.py:155-157,
   * avatar/main/model.py:283-285):  grad_accum += ||dL/dmeans2D.xy||,  count += 1,  radius_max = max(radius_max, radii). */
  float* densify_grad_accum;
  float* densify_count;
  float* densify_radius_max;
  /* (ABI v3) the densification statistics above are updated for Gaussians [0, densify_rows) only; 0 = all.  A merged
   * cat(scene, human) pass keeps ExAvatar's bookkeeping to the scene Gaussians this way (model.py:193). */
  uint32_t densify_rows;
  uint32_t reserved;
} B2RBackwardArgs;
/* Standalone linear-blend skinning of one or two Gaussian sets that share a rig (SURVEY section 8f-2).  ExAvatar poses
 * `mean_3d` and `mean_3d_refined` of its human Gaussians with the same weight rows, joint transforms, translation and
 * camera (avatar/common/nets/module.py:549-557):  M_i = sum_j W[rows[i], j] A_j,  posed_s,i = M_i [xyz_s,i, 1] + trans,
 * then Rinv (posed - t) with a camera.  b2r_skin_forward blends M_i once per Gaussian and writes both posed sets, which
 * the caller's normal / colour networks and the renders then read as B2RScene.means3D.  It poses ahead of the render
 * rather than inside its projection because those networks need the posed positions before anything is rendered. */
typedef struct B2RSkin {
  int32_t P;                /* Gaussians per set */
  int32_t J;                /* joints (55 for SMPL-X); 1..64 */
  int32_t V;                /* rows of the weight table */
  int32_t reserved;
  const float* weights;     /* (V,J) skinning weight table */
  const int32_t* rows;      /* (P) row of `weights` for each Gaussian (nn_vertex_idxs, module.py:414; every value in
                               [0, V)), or NULL: row i (then V >= P) */
  const float* joint_mats;  /* (J,16) row-major 4x4 transform per joint; rows 0..2 are read */
  const float* trans;       /* (3) root translation added after blending */
  const float* cam_Rinv;    /* (9) row-major inverse camera rotation, or NULL to stay in the posed frame */
  const float* cam_t;       /* (3) camera translation (required with cam_Rinv) */
  const float* xyz[2];      /* (P,3) canonical positions of set 0 / set 1 (set 1 may be NULL) */
  float* posed[2];          /* (P,3) OUTPUT posed positions; posed[1] requires xyz[1] (NULL: set 1 is not posed) */
} B2RSkin;

#define B2R_BWD_ACCUMULATE 1u
/* The caller guarantees `bwd_scratch` is all zero on entry; b2r_backward then skips its memset and leaves the scratch
 * all zero again on return (the backward projection kernel clears each row after consuming it).  For callers that
 * keep one scratch buffer alive across steps (plan.py): one graph node and one 48 B/Gaussian memset less per render. */
#define B2R_BWD_SCRATCH_ZEROED 2u

int b2r_abi_version(void);
const char* b2r_strerror(int code);
int b2r_last_cuda_error(void);
/* sizeof() of the ABI structs, for bindings to verify their mirror: 0 B2RScene, 1 B2RStatus, 2 B2RWorkspace,
 * 3 B2RForwardOutputs, 4 B2RBackwardArgs, 5 B2RView, 6 B2RSkin, 8 B2RMeshRender, 10 B2RGnMlp, 11 B2RRegs,
 * 12 B2RRegsGrads, 13 B2RRig, 14 B2RRigGrads, 15 B2RAdamSegment, 16 B2RLpips, 17 B2RSceneAssets,
 * 18 B2RSceneAssetsGrads, 19 B2RSmplxPose, 20 B2RSmplxPoseGrads, 21 B2RHumanAssets, 22 B2RHumanAssetsGrads,
 * 23 B2RSmplxBody, 24 B2RSmplxBodyGrads; 0 for anything else
 * (7 and 9 are unused and report 0). */
size_t b2r_sizeof(int which);

size_t b2r_ctx_bytes(int32_t P, int32_t width, int32_t height);
size_t b2r_scratch_bytes(int32_t P, int32_t width, int32_t height, uint64_t dup_capacity);
size_t b2r_backward_scratch_bytes(int32_t P);
size_t b2r_checkpoint_bytes(int32_t width, int32_t height, uint64_t dup_capacity);

/* Phase A: projection, tile counting, tile scan.  Writes radii and B2RStatus.num_dups.  With ws->dup_capacity == 0 it
 * only counts (two-phase use: size the lists from num_dups, then b2r_forward_render).  With a capacity it also prepares
 * the binning (b2r_forward_bin may follow directly); if that capacity then turns out too small (B2RStatus.overflow), run
 * the whole forward again with more room -- the tile counters are consumed. */
int b2r_forward_project(const B2RScene* scene, const B2RWorkspace* ws, int32_t* radii, void* stream);
/* Phase B: duplicate-with-keys, per-tile sort, forward composite (needs phase A on the same ws).  After a count-only
 * phase A it re-derives the per-tile ranges for ws->dup_capacity; after a phase A that was given a capacity it uses the
 * ranges that phase prepared (same capacity expected). */
int b2r_forward_render(const B2RScene* scene, const B2RWorkspace* ws, const B2RForwardOutputs* out, void* stream);
/* Both phases with a capacity chosen up front. */
int b2r_forward(const B2RScene* scene, const B2RWorkspace* ws, const B2RForwardOutputs* out, void* stream);

/* Backward composite + backward projection.  `ws` is the forward's; `bwd_scratch` >= b2r_backward_scratch_bytes(P). */
int b2r_backward(const B2RScene* scene, const B2RWorkspace* ws, const B2RBackwardArgs* args, void* bwd_scratch,
                 size_t bwd_scratch_bytes, void* stream);

/* The same pipeline in separately callable stages (ABI v3), for several views of one binned scene:
 *   b2r_forward_project -> b2r_forward_bin -> b2r_forward_composite (once per view)
 *   b2r_backward_composite (once per view, same scratch) -> b2r_backward_project (once).
 * b2r_forward_render == bin + composite(view = NULL); b2r_backward == composite(view = NULL) + project.
 * b2r_backward_composite reads only dL_dcolor / dL_ddepth / dL_dalpha, `flags` (B2R_BWD_SCRATCH_ZEROED: the caller zeroed
 * the scratch before the FIRST view; later views must pass it too, so nothing is cleared in between) and `first_row`
 * (Gaussians below it receive nothing from this view: the detached prefix of cat(scene.detach(), human)). */
int b2r_forward_bin(const B2RScene* scene, const B2RWorkspace* ws, void* stream);
int b2r_forward_composite(const B2RScene* scene, const B2RWorkspace* ws, const B2RView* view,
                          const B2RForwardOutputs* out, void* stream);
int b2r_backward_composite(const B2RScene* scene, const B2RWorkspace* ws, const B2RView* view, const B2RBackwardArgs* args,
                           void* bwd_scratch, size_t bwd_scratch_bytes, void* stream);
int b2r_backward_project(const B2RScene* scene, const B2RWorkspace* ws, const B2RBackwardArgs* args, void* bwd_scratch,
                         size_t bwd_scratch_bytes, void* stream);

/* Split pass (ABI v3 addition).  Two passes that share the rows [0, first_row) -- same inputs, same camera -- need not
 * project, bin and sort them twice.  ExAvatar's merged frame bins cat(scene, human) (the BASE pass) and
 * cat(scene, human_refined); the second pass then covers its own rows [first_row, P) only:
 *   b2r_forward_project_split  projects rows [first_row, P) (radii, records, tile counts of those rows); no scan yet.
 *   b2r_forward_bin_split      after the base pass's b2r_forward_bin (stream order is the caller's): copies the base's
 *                              records and radii of rows [0, first_row) into this pass (a view gathers them; their aux
 *                              rows are not copied and never read), then builds a list ONLY in the tiles the own rows
 *                              reach -- the base list of the tile filtered to ids < first_row, merged with the own rows'
 *                              sorted entries on the (depth, id) key: entry for entry the list the whole pass would have
 *                              built there.  Every other tile gets an empty list, so a view of this pass must skip the
 *                              tiles without own rows (B2RView.skip_below >= first_row).  B2RStatus.num_dups counts the
 *                              entries of these lists; `ws` needs a capacity and scratch >= b2r_split_scratch_bytes().
 * Ids keep the numbering of the whole scene.  `base` must be a workspace of the same P, width and height whose lists
 * stay unchanged until this call's work has run.  The composites and the backward stages take the pass as usual. */
size_t b2r_split_scratch_bytes(int32_t P, int32_t width, int32_t height, uint64_t dup_capacity);
int b2r_forward_project_split(const B2RScene* scene, const B2RWorkspace* ws, uint32_t first_row, int32_t* radii,
                              void* stream);
int b2r_forward_bin_split(const B2RScene* scene, const B2RWorkspace* ws, const B2RWorkspace* base, uint32_t first_row,
                          int32_t* radii, void* stream);

/* Skinning (B2RSkin).  Forward: writes posed[0] and, when given, posed[1].  Backward: dL_dpos (host array of two
 * device pointers, the gradients at posed[0] / posed[1]; either may be NULL = no gradient reaches that set, dL_dpos[1]
 * requires xyz[1]) ->
 *   dL_dxyz[s]  (P,3) = M_i[:3,:3]^T g_cam,s,i  with  g_cam = Rinv^T dL/dposed  (zeros when dL_dpos[s] is NULL);
 *   dL_djoint (J,3,4) = sum_i W[rows[i], j] sum_s g_cam,s,i [xyz_s,i, 1]^T   (row 3 of each 4x4 has no gradient);
 *   dL_dtrans (3)     = sum_i sum_s g_cam,s,i.
 * dL_dxyz (host array) and each output may be NULL.  The joint / translation sums are deterministic (block partials
 * added in a fixed order, no float atomics): bit-identical from run to run.  `scratch` >= b2r_skin_scratch_bytes(P, J)
 * when dL_djoint or dL_dtrans is given.  No gradient for the weights or the camera.  Neither call allocates or syncs. */
int b2r_skin_forward(const B2RSkin* skin, void* stream);
int b2r_skin_backward(const B2RSkin* skin, const float* const dL_dpos[2], float* const dL_dxyz[2], float* dL_djoint,
                      float* dL_dtrans, void* scratch, size_t scratch_bytes, void* stream);
size_t b2r_skin_scratch_bytes(int32_t P, int32_t J);

/* Photometric L1 + SSIM of one (3,H,W) image against a target (avatar/common/nets/loss.py RGBLoss / SSIM, reduced with
 * .mean() as avatar/main/model.py:196-215 does).  `mask` (H,W) or NULL multiplies both images first; `bbox` is a DEVICE
 * float[4] {xmin, ymin, width, height} or NULL (the whole image), read on the device with the reference's integer rules:
 * x0 = max(trunc(xmin), 0), x1 = min(x0 + trunc(width), W), likewise for y, crop [y0:y1, x0:x1].  The SSIM window
 * (11 taps, sigma 1.5) runs over the crop with zero padding at the crop's border.  Forward writes out[0] = mean |x - y|
 * and, with with_ssim != 0, out[1] = mean SSIM, both over 3 h w (NaN for an empty crop).  Backward reads dL_dout[2]
 * (device) and writes every element of dL_dimg (3,H,W): zero outside the crop.  `scratch` >= b2r_l1ssim_scratch_bytes
 * (W, H) holds the forward's per-pixel SSIM partials until the backward (the backward without SSIM does not read it,
 * and it may then be NULL).  Fixed-order reductions, no float atomics: bit-identical runs.  Neither call allocates or
 * syncs. */
size_t b2r_l1ssim_scratch_bytes(int32_t width, int32_t height);
int b2r_l1ssim_forward(int32_t width, int32_t height, const float* img, const float* target, const float* mask,
                       const float* bbox, int32_t with_ssim, float* out, void* scratch, size_t scratch_bytes,
                       void* stream);
int b2r_l1ssim_backward(int32_t width, int32_t height, const float* img, const float* target, const float* mask,
                        const float* bbox, int32_t with_ssim, const float* dL_dout, float* dL_dimg, const void* scratch,
                        size_t scratch_bytes, void* stream);

/* Nearest mesh vertex of every human Gaussian (avatar/common/nets/module.py:541-546: knn_points(K=1) and the
 * hand / face self-map).  rows[i] = i where self_map[i] != 0 (self_map (P) may be NULL: none); otherwise the smallest j
 * minimising d(i,j) = dx*dx + dy*dy + dz*dz (dx = queries[i].x - targets[j].x ..., fp32, left to right, no fma), which
 * is torch.argmin's answer, ties included; a query with a non-finite coordinate gets row 0.  queries (P,3), targets
 * (V,3) must be finite (other targets give unspecified rows, never an out-of-bounds access); rows (P) int32 is what
 * B2RSkin.rows reads.  Every call builds a uniform grid over the targets in `scratch` (>= b2r_nearest_scratch_bytes(P,
 * V), which depends on V only) and searches it exactly.  P = 0 launches nothing.  No allocation, no sync. */
size_t b2r_nearest_scratch_bytes(int32_t P, int32_t V);
int b2r_nearest_rows(int32_t P, const float* queries, int32_t V, const float* targets, const uint8_t* self_map,
                     int32_t* rows, void* scratch, size_t scratch_bytes, void* stream);

/* Area-weighted vertex normals of a triangle mesh with P vertices (module.py:501-504: verts_normals_packed and the
 * cavity flip).  xyz (P,3); faces (F,3) int32, every index in [0, P).  The vertex -> face CSR: vf_offsets (P+1) int32,
 * vf_offsets[0] = 0, non-decreasing, vf_offsets[P] = 3F; vf_entries (3F) int32 face indices, the incident faces of
 * vertex v at [vf_offsets[v], vf_offsets[v+1]) in ascending order, one entry per corner (a face that repeats v lists it
 * twice).  normals[v] = n / max(|n|, 1e-6) with n the fp32 sum, in CSR order, of (x1 - x0) x (x2 - x0) over v's
 * entries (0 for a vertex in no face), negated where flip (P, may be NULL) is set.  No float atomics: bit-identical
 * runs.  P = 0 launches nothing.  No allocation, no sync. */
int b2r_vertex_normals(int32_t P, const float* xyz, const int32_t* faces, const int32_t* vf_offsets,
                       const int32_t* vf_entries, const uint8_t* flip, float* normals, void* stream);

/* Textured render of a triangle mesh: ExAvatar's face render (avatar/main/model.py:170-175 -> MeshRenderer,
 * avatar/common/nets/layer.py:23-68: pytorch3d's MeshRasterizer with blur_radius 0, faces_per_pixel 1, perspective-
 * correct barycentrics, no culling or clipping, then TexturesUV), restated from pytorch3d's implementation:
 *   camera   p_c = R p + t;  u = fx x_c / z_c + cx,  v = fy y_c / z_c + cy;  x_ndc = (W/2 - u) / s, y_ndc = (H/2 - v) / s
 *            with s = min(H, W) / 2; a corner's z is z_c.
 *   pixel    (row r, col c) sits at NDC (PixToNonSquareNdc(W-1-c, W, H), PixToNonSquareNdc(H-1-r, H, W)), the point
 *            u = c + 0.5, v = r + 0.5.
 *   coverage a face is skipped if max z < 0, |E(v0,v1,v2)| <= 1e-8, or a corner is not finite.  A pixel centre p is
 *            covered if it lies in the face's closed NDC xy box (pytorch3d's CheckPointOutsideBoundingBox), pz = b.z >= 0
 *            and all three perspective-corrected barycentrics b are > 0, where
 *            b0 = (E(p,v1,v2), E(p,v2,v0), E(p,v0,v1)) / (E(v2,v0,v1) + 1e-8),
 *            b = (b0.x z1 z2, z0 b0.y z2, z0 z1 b0.z) / max(sum, 1e-8),  E(p,a,b) = (p.x-a.x)(b.y-a.y) - (p.y-a.y)(b.x-a.x).
 *            The covering face of least pz wins, equal pz to the lowest index.
 *   texture  uv = sum_k b_k (a_k, 1 - b_k) over the corners' vertex_uv rows (a_k, b_k) chosen by face_uv; the texture
 *            flipped vertically is sampled at grid 2 uv - 1 (bilinear, align_corners, border padding).
 *   output   image (C,H,W), -1 in every channel where no face covers the pixel; pix_to_face (H*W) int32, -1 there.
 * The backward gives dL/dmesh only (texture and uv are constants), the derivative of the above with the per-pixel face
 * held fixed.  All arithmetic is fp32; the per-pixel face is computed exactly as a float32 restatement with no fma. */
typedef struct B2RMeshRender {
  int32_t V;                    /* mesh vertices */
  int32_t F;                    /* faces */
  int32_t Vt;                   /* rows of vertex_uv */
  int32_t C;                    /* texture channels, 1..4 */
  int32_t tex_height, tex_width;
  int32_t height, width;        /* output size; height * width < 2^31 */
  const float* mesh;            /* (V,3) world positions */
  const int32_t* faces;         /* (F,3) vertex indices in [0, V) (a face with an index outside is skipped) */
  const float* vertex_uv;       /* (Vt,2) */
  const int32_t* face_uv;       /* (F,3) rows of vertex_uv, every one in [0, Vt) */
  const float* texture;         /* (C, tex_height, tex_width), row 0 at the top (the map is NOT pre-flipped) */
  const float* cam_R;           /* (9) row-major, read on the device */
  const float* cam_t;           /* (3) */
  const float* focal;           /* (2) fx, fy */
  const float* princpt;         /* (2) cx, cy */
  uint64_t* keys;               /* forward: (height * width) per-pixel depth keys, all ~0 on entry and left all ~0 */
  const int32_t* vf_offsets;    /* backward: the vertex -> face CSR of b2r_vertex_normals over (V, faces) */
  const int32_t* vf_entries;
} B2RMeshRender;

/* `scratch` >= b2r_mesh_render_scratch_bytes(F): per-face records the forward writes and the backward reads (keep it
 * until the backward), plus the backward's per-face gradients.  Forward: writes every element of image (C,H,W) and
 * pix_to_face (H*W).  Backward: reads the forward's pix_to_face and scratch and dL_dimage (C,H,W), writes every element
 * of dL_dmesh (V,3) -- the per-face sums walk each face's pixels in raster order and each vertex sums its corners in
 * CSR order, no float atomics: bit-identical runs.  Neither allocates, syncs or reads device data on the host, so a
 * captured graph replays with new mesh and camera contents. */
size_t b2r_mesh_render_scratch_bytes(int32_t F);
int b2r_mesh_render_forward(const B2RMeshRender* mr, float* image, int32_t* pix_to_face, void* scratch,
                            size_t scratch_bytes, void* stream);
int b2r_mesh_render_backward(const B2RMeshRender* mr, const int32_t* pix_to_face, const float* dL_dimage,
                             float* dL_dmesh, void* scratch, size_t scratch_bytes, void* stream);

/* Triplane features of the human Gaussians (avatar/common/nets/module.py:424-457 extract_tri_feature).  planes and
 * planes_face are (3,C,height,width); corners (P,3,4) int32 holds, per row and plane (xy, xz, yz), the texels
 * y * width + x of F.grid_sample's four bilinear corners in its order (nw, ne, sw, se), -1 for a corner outside the
 * plane (zero padding), and weights (P,3,4) their weights.  Forward: feat (P,3C)[r][p*C + c] = sum over the corners of
 * w T[p][c][texel], T = planes_face where is_face[r] != 0 (is_face (P) may be NULL: none), else planes.  Backward:
 * writes every element of dplanes and dplanes_face (both (3,C,height,width)) from dfeat (P,3C) and the texel -> row
 * CSR of the same corners: key (s * 3 + p) * height * width + texel with s = 1 for face rows, offsets (6 * height *
 * width + 1), rows / w the entries' rows (ascending within a key) and weights.  Sums in CSR order, no float atomics:
 * bit-identical runs.  No allocation, no sync. */
int b2r_triplane_forward(int32_t P, int32_t C, int32_t height, int32_t width, const float* planes,
                         const float* planes_face, const uint8_t* is_face, const int32_t* corners, const float* weights,
                         float* feat, void* stream);
int b2r_triplane_backward(int32_t P, int32_t C, int32_t height, int32_t width, const float* dfeat,
                          const int32_t* offsets, const int32_t* rows, const float* w, float* dplanes,
                          float* dplanes_face, void* stream);

/* One of HumanGaussian's GroupNorm MLP stacks (avatar/common/nets/layer.py make_linear_layers(use_gn=True)):
 *   z_l = a_{l-1} W_l^T + b_l,  a_l = relu(GroupNorm(4, 128, eps 1e-5)(z_l) * gamma_l + beta_l),  l = 0, 1, 2,
 *   out = a_2 Wh^T + bh,  with a_{-1} = x.
 * A first-layer input block that is the same for every row is the caller's to fold into b[0].  Products are taken as
 * 3xTF32 on the tensor cores (fp32-accurate), sums in fp32. */
typedef struct B2RGnMlp {
  int32_t P;              /* rows, >= 1 */
  int32_t K;              /* per-row first-layer inputs, 1..128 */
  int32_t H;              /* head outputs, 1..4 */
  int32_t reserved;
  const float* x;         /* (P,K) */
  const float* w[3];      /* w[0] (128,K), w[1], w[2] (128,128), row-major [out][in] */
  const float* b[3];      /* (128) each */
  const float* gamma[3];  /* (128) each: the GroupNorm affine */
  const float* beta[3];
  const float* w_head;    /* (H,128) */
  const float* b_head;    /* (H) */
} B2RGnMlp;

/* Forward: writes out (P,H) and, when saved is not NULL, the pre-GroupNorm z_0, z_1, z_2 into saved (3,P,128), which
 * the backward reads.  Backward: from saved and dL_dout (P,H) writes dL_dx (P,K) when not NULL, and every element of
 * grads (b2r_gn_mlp_grads_count(K, H) floats) = [dW_0 (128,K) | dW_1 (128,128) | dW_2 (128,128) | dgamma (3,128) |
 * dbeta (3,128) | db (3,128) | dWh (H,128) | dbh (H)].  The parameter gradients are summed into fixed per-CTA and
 * per-1024-row partials, then over those in a fixed order: no float atomics, bit-identical runs.  `scratch` >=
 * b2r_gn_mlp_scratch_bytes(P).  Neither call allocates or syncs. */
size_t b2r_gn_mlp_scratch_bytes(int32_t P);
size_t b2r_gn_mlp_grads_count(int32_t K, int32_t H);
int b2r_gn_mlp_forward(const B2RGnMlp* m, float* out, float* saved, void* stream);
int b2r_gn_mlp_backward(const B2RGnMlp* m, const float* saved, const float* dL_dout, float* dL_dx, float* grads,
                        void* scratch, size_t scratch_bytes, void* stream);

/* ExAvatar's per-frame human regularisers (avatar/main/model.py:217-257 with avatar/common/nets/loss.py:97-197 and
 * smpl_x.get_arm) as ten means, out[10] = {gaussian_mean_reg, gaussian_mean_hand_reg, gaussian_scale_reg, lap_mean,
 * lap_scale, lap_rgb, hand_rgb_reg, arm_rgb_reg, joint_offset_reg, joint_offset_sym_reg}, each equal to the mean of the
 * reference's map with its constant factor (1e5 for lap_mean / lap_scale, 0.01 hand_rgb_reg, 0.1 arm_rgb_reg).
 * Per-vertex inputs are (P,3) float, scale_offset (P); the tables are constants of the model (built once by the caller):
 *   lap      nbr_idx / nbr_w (P,10): LaplacianReg's neighbour table; lapT_* its transpose as a CSR over the entries of
 *            non-zero weight, each vertex's entries in ascending source order (the backward's adjoint gather).
 *   weights  (5,P): the weight columns of gaussian_mean_reg, gaussian_scale_reg, lap_mean, lap_scale, lap_rgb.
 *   hand     (P): bit 0 is_rhand, bit 1 is_lhand; n_hand = #(rhand | lhand) rows, n_rhand = #rhand = #lhand.
 *   arm      arm_idx (n_arm): the is_arm rows ascending; arm_slot (P): position in arm_idx or -1.
 *   joints   joint_target (J,3), joint_weight (J), sym_pairs (n_pairs,2) = (right, left) joint ids; J <= 256.
 * The normals of `mesh` come from the b2r_vertex_normals kernel over faces / vf_offsets / vf_entries (no flip).  An arm
 * row is upper when n_y > 0.5f, else lower; a lower row's target is the mean rgb of the k upper rows nearest in fp32
 * distance among those with |fl(l_x - u_x)| < 0.01f, k = min(50, smallest such count), distance ties to the lower
 * vertex index; k = 0 or no lower row gives NaN for arm_rgb_reg.  scale_reg (P,3) or NULL replaces `scale` in
 * gaussian_scale_reg (the warm-up's scale_wo_clamp).  `scratch` >= b2r_regs_scratch_bytes(P, n_arm) is kept from the
 * forward until the backward.  The backward reads dL_dout[10] on the device and writes every element of each gradient
 * in B2RRegsGrads (scale_reg required iff given); mesh gets none.  No float atomics (bit-identical runs), no
 * allocation, no sync: both calls can be captured in a CUDA graph. */
typedef struct B2RRegs {
  int32_t P, J, n_arm, n_pairs, n_hand, n_rhand, reserved[2];
  const float* mesh;                /* (P,3) mesh_neutral_pose */
  const float* mean_offset;         /* (P,3) */
  const float* mean_offset_offset;  /* (P,3) */
  const float* scale_offset;        /* (P) */
  const float* scale;               /* (P,3) */
  const float* scale_refined;       /* (P,3) */
  const float* rgb;                 /* (P,3) */
  const float* rgb_refined;         /* (P,3) */
  const float* scale_reg;           /* (P,3) or NULL */
  const float* joint_offset;        /* (J,3) */
  const int32_t* faces;             /* (F,3) and the vertex -> face CSR of b2r_vertex_normals */
  const int32_t* vf_offsets;
  const int32_t* vf_entries;
  const int32_t* nbr_idx;
  const float* nbr_w;
  const int32_t* lapT_offsets;      /* (P+1) */
  const int32_t* lapT_src;
  const float* lapT_w;
  const float* weights;
  const uint8_t* hand;
  const int32_t* arm_idx;
  const int32_t* arm_slot;
  const float* joint_target;
  const float* joint_weight;
  const int32_t* sym_pairs;
} B2RRegs;

typedef struct B2RRegsGrads {
  float* mean_offset;
  float* mean_offset_offset;
  float* scale_offset;
  float* scale;
  float* scale_refined;
  float* rgb;
  float* rgb_refined;
  float* scale_reg;    /* required iff B2RRegs.scale_reg is given */
  float* joint_offset;
} B2RRegsGrads;

size_t b2r_regs_scratch_bytes(int32_t P, int32_t n_arm);
int b2r_regs_forward(const B2RRegs* r, float* out, void* scratch, size_t scratch_bytes, void* stream);
int b2r_regs_backward(const B2RRegs* r, const float* dL_dout, const B2RRegsGrads* grads, const void* scratch,
                      size_t scratch_bytes, void* stream);

/* ExAvatar's SMPL-X rig (HumanGaussian.forward, avatar/common/nets/module.py:517-518, 533, 537, 549): the 大-pose and
 * zero-pose body-model forwards with identity information, the inverse-neutral and the frame's forward kinematics, the
 * pose-corrective and expression offsets, and two midpoint subdivisions -- one forward and one backward call.
 * Sizes: V base vertices, V1 after one subdivision, P after two; J joints (22 + 3 <= n_body + 4 <= J <= 64, parents
 * topological: parents[0] = -1, 0 <= parents[i] < i), NB shape and NE expression coefficients (<= 128 each); the pose
 * feature has 9 (J-1) entries.  Per-call inputs (float, device): shape_param (NB), joint_offset (J,3) before the root
 * is zeroed (its row 0 is ignored), full_pose (J,3) axis-angle in the model's joint order, expr (NE).  Tables (constants
 * of the model, built once by the caller):
 *   template      (V,3)  v_template + face_offset, rounded as one fp32 add;  shapedirs (V,3,NB), expr_dirs (V,3,NE)
 *   posedirs_t    (V,3,9(J-1)) posedirs per vertex row;  pose_offset0 (V,3) the 大 pose's corrective offsets
 *   lbs_weights   (V,J);  jreg_* J_regressor as a per-joint CSR (offsets J+1, cols, vals) and jregT_* its transpose
 *                 per vertex (offsets V+1, rows ascending, vals)
 *   rot_neutral / rot_zero / rot_inv  (J,9) double: the rotations of the 大-pose, zero-pose and inverse-neutral chains
 *   sub1 (V1-V,2), sub2 (P-V1,2): each new vertex is the midpoint fl(fl(a + b) * 0.5f) of two of the level below
 *   upT_*         the composed two-level subdivision transposed per base vertex (offsets V+1, rows ascending, weights)
 *   mask          (P) uint8: rows of pose_offset kept (is_rhand | is_lhand | is_face_expr); the others are written 0.
 * Forward outputs: mesh (P,3) mesh_neutral_pose, mesh_wo (V,3) before subdivision, joint_mats (J,4,4), pose_offset
 * (P,3), expr_offset (P,3), pose_6d (6 n_body): the first two rows of each body joint's rotation.  `scratch` >=
 * b2r_rig_scratch_bytes(V, J, NB, NE) is kept from the forward until the backward.  The backward reads the gradients of
 * mesh, joint_mats and expr_offset (any may be NULL: zero) and writes every element of the four B2RRigGrads buffers;
 * the root row of joint_offset's gradient is exactly 0.  Parents that are not topological are found on the device:
 * no chain is walked and joint_mats, the meshes and the joint and pose gradients are NaN.  No float atomics (bit-identical runs), no allocation, no sync:
 * both calls can be captured in a CUDA graph. */
typedef struct B2RRig {
  int32_t V, V1, P, J, NB, NE, n_body, reserved;
  const float* shape_param;
  const float* joint_offset;
  const float* full_pose;
  const float* expr;
  const float* template_;
  const float* shapedirs;
  const float* expr_dirs;
  const float* posedirs_t;
  const float* pose_offset0;
  const float* lbs_weights;
  const int32_t* jreg_offsets;
  const int32_t* jreg_cols;
  const float* jreg_vals;
  const int32_t* jregT_offsets;
  const int32_t* jregT_rows;
  const float* jregT_vals;
  const int32_t* parents;
  const double* rot_neutral;
  const double* rot_zero;
  const double* rot_inv;
  const int32_t* sub1;
  const int32_t* sub2;
  const int32_t* upT_offsets;
  const int32_t* upT_rows;
  const float* upT_w;
  const uint8_t* mask;
} B2RRig;

typedef struct B2RRigGrads {
  float* shape_param;
  float* joint_offset;
  float* full_pose;
  float* expr;
} B2RRigGrads;

size_t b2r_rig_scratch_bytes(int32_t V, int32_t J, int32_t NB, int32_t NE);
int b2r_rig_forward(const B2RRig* r, float* mesh, float* mesh_wo, float* joint_mats, float* pose_offset,
                    float* expr_offset, float* pose_6d, void* scratch, size_t scratch_bytes, void* stream);
int b2r_rig_backward(const B2RRig* r, const float* dL_dmesh, const float* dL_djoint_mats, const float* dL_dexpr_offset,
                     const B2RRigGrads* grads, void* scratch, size_t scratch_bytes, void* stream);

/* The frame's SMPL-X body mesh (ExAvatar's get_smplx_outputs, avatar/main/model.py:37-58: smplx's SMPLX.forward and
 * lbs.lbs, then the world transform) for one frame, over the rig's tables.  `rig` is the model's B2RRig as
 * b2r_rig_forward takes it (its four input pointers are not read; the body's are).  Per-call inputs (float, device):
 * shape_param (NB), joint_offset (J,3) used as given, every row including the root, full_pose (J,3) axis-angle in the
 * model's joint order, expr (NE), trans (3); pose_mean (J,3) is the model's.  With v_shaped = template + shapedirs .
 * shape_param + expr_dirs . expr, J = J_regressor . v_shaped + joint_offset, rot = smplx batch_rodrigues(full_pose +
 * pose_mean) (angle = |r + 1e-8|), v_posed = v_shaped + (rot[1:] - I) . posedirs, the forward writes mesh (V,3) =
 * LBS(v_posed, batch_rigid_transform(rot, J)) + trans and, when cam_R (3,3) row-major and cam_t (3) are given (both or
 * neither), R^-1 (mesh - t) with R^-1 by cofactors.  Landmarks and joints are not computed.  `scratch` >=
 * b2r_smplx_body_scratch_bytes(V, J) is kept from the forward until the backward.  The backward reads dL_dmesh (NULL:
 * zero) and writes every element of the five B2RSmplxBodyGrads buffers; the camera gets no gradient.  Parents that are
 * not topological give NaN meshes and joint / pose gradients.  No float atomics (bit-identical runs), no allocation, no
 * sync: both calls can be captured in a CUDA graph. */
typedef struct B2RSmplxBody {
  B2RRig rig;
  const float* pose_mean;
  const float* shape_param;
  const float* joint_offset;
  const float* full_pose;
  const float* expr;
  const float* trans;
  const float* cam_R;
  const float* cam_t;
} B2RSmplxBody;

typedef struct B2RSmplxBodyGrads {
  float* shape_param;
  float* joint_offset;
  float* full_pose;
  float* expr;
  float* trans;
} B2RSmplxBodyGrads;

size_t b2r_smplx_body_scratch_bytes(int32_t V, int32_t J);
int b2r_smplx_body_forward(const B2RSmplxBody* b, float* mesh, void* scratch, size_t scratch_bytes, void* stream);
int b2r_smplx_body_backward(const B2RSmplxBody* b, const float* dL_dmesh, const B2RSmplxBodyGrads* grads,
                            void* scratch, size_t scratch_bytes, void* stream);

/* One Adam step over many fp32 tensors in one launch: ExAvatar's torch.optim.Adam(params, lr, eps=1e-15)
 * (avatar/common/base.py:83-85), element for element the arithmetic of torch's default foreach path (weight_decay 0,
 * no amsgrad, no maximize).  `table` (device) holds one segment per tensor with a gradient; grad, exp_avg and
 * exp_avg_sq are numel contiguous floats, and param is numel / row_len rows of row_len contiguous floats, row_stride
 * floats apart (row_stride >= row_len; row_stride == row_len: contiguous).  The strided form is a view such as
 * ExAvatar's feature_dc / feature_rest, slices of one (P,16,3) tensor.  param / exp_avg / exp_avg_sq are updated in
 * place.  The segments split into chunks of b2r_adam_chunk_elems() elements: first_chunk is the sum of
 * ceil(numel / chunk) over the segments before it, and n_chunks that sum over all of them (the launch has one CTA per
 * chunk).  The scalars are torch's, evaluated in double on the host and rounded to fp32 once: lerp_weight 1-beta1,
 * beta2, one_minus_beta2 1-beta2, bc2_sqrt (1-beta2^t)^0.5, eps, step_size (lr / (1-beta1^t)) * -1.  Tensors may start
 * anywhere (float4 I/O when a segment is contiguous and all four pointers are 16-byte aligned).  No atomics, no
 * allocation, no sync; n_chunks == 0 launches nothing. */
typedef struct B2RAdamSegment {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  int64_t numel;
  int64_t first_chunk;
  int64_t row_len;
  int64_t row_stride;
  float lerp_weight, beta2, one_minus_beta2, bc2_sqrt, eps, step_size;
} B2RAdamSegment;

#define B2R_ADAM_CHUNK 16384
int64_t b2r_adam_chunk_elems(void);
int b2r_adam_step(const B2RAdamSegment* table, int32_t n_segments, int64_t n_chunks, void* stream);

/* ExAvatar's LPIPS-VGG terms (avatar/common/nets/loss.py LPIPS over lpips.LPIPS(net='vgg'), version 0.1, eval mode) of
 * n_images (3,H,W) images `img` against one (3,H,W) `target`.  `bbox` is a DEVICE float[4] {xmin, ymin, width, height}
 * or NULL (the whole image), read on the device by b2r_l1ssim_forward's crop rules.  Per image: crop, x*2-1, lpips's
 * ScalingLayer, VGG-16 features through relu5_3 (3x3 zero padding at the crop's border, 2x2 floor max pools), and the
 * sum over the taps relu1_2, relu2_2, relu3_3, relu4_3, relu5_3 of mean_p sum_c lin[t]_c (n_c(img) - n_c(target))^2,
 * n(f) = f / (|f| + 1e-10).  Convolutions run as TF32 (round to nearest) on the tensor cores with fp32 accumulation.
 * Weights (fp32, device): w_fwd[0] is conv1_1's (64,3,3,3) torch tensor and w_bwd[0] is not read; for l >= 1 w_fwd[l]
 * is (3,3,C_in,C_out) (torch's (C_out,C_in,3,3) permuted 2,3,1,0) and w_bwd[l] is (3,3,C_out,C_in) (flipped in both
 * taps, permuted 2,3,0,1); bias[l] (C_out); lin[t] (C) of tap t.  Weight and activation pointers are 16-byte aligned.
 * Forward writes out[n] (NaN when the crop is narrower or shorter than 16 px) and fills `saved`
 * (>= b2r_lpips_saved_bytes(W, H, N): the 13 ReLU outputs per image and the target's normalised taps), which the
 * backward reads.  Backward reads dL_dout[n] (device) and writes every element of dL_dimg (N,3,H,W): zero outside the
 * crop, and zero everywhere for a crop under 16 px.  No gradient for the target or the weights.  `scratch` >=
 * b2r_lpips_scratch_bytes(W, H) is free between the calls.  W, H >= 16.  Fixed-order reductions, no float atomics:
 * bit-identical runs; every grid is sized from W x H, never from the box.  Neither call allocates or syncs. */
typedef struct B2RLpips {
  int32_t width, height, n_images, reserved;
  const float* img;
  const float* target;
  const float* bbox;
  const float* w_fwd[13];
  const float* w_bwd[13];
  const float* bias[13];
  const float* lin[5];
} B2RLpips;

size_t b2r_lpips_saved_bytes(int32_t width, int32_t height, int32_t n_images);
size_t b2r_lpips_scratch_bytes(int32_t width, int32_t height);
int b2r_lpips_forward(const B2RLpips* p, float* out, void* saved, size_t saved_bytes, void* scratch,
                      size_t scratch_bytes, void* stream);
int b2r_lpips_backward(const B2RLpips* p, const void* saved, size_t saved_bytes, const float* dL_dout, float* dL_dimg,
                       void* scratch, size_t scratch_bytes, void* stream);

/* ExAvatar's scene Gaussian assets (avatar/common/nets/module.py:253-272, SceneGaussian.forward) from the stored
 * parameters of P Gaussians with M SH coefficients (1 <= M <= B2R_SCENE_MAX_COEFFS): opacity = sigmoid(logit) (P,1),
 * scale = exp(log_scale) (P,3), rotation = pytorch3d 0.7.5's matrix_to_quaternion(rotation_6d_to_matrix(rotation6d))
 * (P,4), and one colour output:
 *   shs mode (cam_R == NULL): shs (P,M,3) = cat(feature_dc, feature_rest, 1);
 *   rgb mode (cam_R, cam_t set): rgb (P,3) = clamp_min(eval_sh(deg, sh, normalize(mean - campos)) + 0.5, 0) with
 *   campos = -R^-1 t (R (3,3) row-major and t (3) on the device; the camera gets no gradient) and deg the DEVICE float
 *   `active_sh_degree`, compared as ExAvatar's eval_sh compares it.  A degree outside 0..3, or one needing more than M
 *   coefficients, writes NaN colours and NaN colour gradients; no coefficient beyond M is read.
 * rotation6d, log_scale, opacity_logit and mean are contiguous rows; feature_dc's row p (3 floats) starts at
 * feature_dc + p * dc_stride and feature_rest's (3 (M-1) contiguous floats) at feature_rest + p * rest_stride, so the
 * (P,1,3) / (P,M-1,3) views of one (P,M,3) tensor are read in place.  feature_rest may be NULL when M == 1.
 * Backward: g's upstream gradients may be NULL (zero); it writes d logit (P,1), d log_scale (P,3), d rotation6d (P,6),
 * d feature_dc (P,1,3) and d feature_rest (P,M-1,3) contiguous (exact zeros above the degree in rgb mode) and, in rgb
 * mode, the view-direction term of d mean (P,3).  Each output element is written once; no atomics, no allocation, no
 * sync. */
#define B2R_SCENE_MAX_COEFFS 16
typedef struct B2RSceneAssets {
  int32_t P, M;
  int64_t dc_stride, rest_stride;
  const float* mean;
  const float* opacity_logit;
  const float* log_scale;
  const float* rotation6d;
  const float* feature_dc;
  const float* feature_rest;
  const float* active_sh_degree;
  const float* cam_R;
  const float* cam_t;
} B2RSceneAssets;

typedef struct B2RSceneAssetsGrads {
  const float* opacity;       /* the forward's opacity (P,1) */
  const float* scale;         /* the forward's scale (P,3) */
  const float* dL_dopacity;   /* (P,1) or NULL */
  const float* dL_dscale;     /* (P,3) or NULL */
  const float* dL_drotation;  /* (P,4) or NULL */
  const float* dL_dcolor;     /* shs mode (P,M,3), rgb mode (P,3), or NULL */
  float* dL_dlogit;
  float* dL_dlog_scale;
  float* dL_drotation6d;
  float* dL_dfeature_dc;
  float* dL_dfeature_rest;    /* NULL when M == 1 */
  float* dL_dmean;            /* rgb mode only */
} B2RSceneAssetsGrads;

int b2r_scene_assets_forward(const B2RSceneAssets* s, float* opacity, float* scale, float* rotation, float* color,
                             void* stream);
int b2r_scene_assets_backward(const B2RSceneAssets* s, const B2RSceneAssetsGrads* g, void* stream);

/* ExAvatar's SMPLXParamDict.forward (avatar/common/nets/module.py:673-684) for one frame: each of the seven 6D pose
 * parameters (root, body, jaw, leye, reye, lhand, rhand) through pytorch3d 0.7.5's
 * matrix_to_axis_angle(rotation_6d_to_matrix(x)) -- Gram-Schmidt with the 1e-12 floor, the first largest q_abs with
 * the 0.1 floor, the sign standardisation, atan2 and the |angle| < 1e-6 branch -- evaluated in fp64 from the fp32
 * rows and rounded once.  param[k] holds rows[k] contiguous 6-float rows; full_pose (J,3), J = sum rows[k] (1 <= J <=
 * B2R_POSE_MAX_JOINTS), takes them in order (ExAvatar's cat_full_pose order).  Backward: autograd's derivative through
 * the branches the forward took (zero through sqrt where its argument is <= 0, through the selected branch of each
 * `where`, norm's zero at a zero vector; finite at the identity), written to grads->param[k] (rows[k] x 6,
 * contiguous).  One CTA of one thread per joint each way; no atomics, no allocation, no sync. */
#define B2R_POSE_PARAMS 7
#define B2R_POSE_MAX_JOINTS 64
typedef struct B2RSmplxPose {
  const float* param[B2R_POSE_PARAMS];
  int32_t rows[B2R_POSE_PARAMS];
  int32_t reserved;
} B2RSmplxPose;

typedef struct B2RSmplxPoseGrads {
  float* param[B2R_POSE_PARAMS];
} B2RSmplxPoseGrads;

int b2r_decode_pose_forward(const B2RSmplxPose* p, float* full_pose, void* stream);
int b2r_decode_pose_backward(const B2RSmplxPose* p, const float* dL_dfull_pose, const B2RSmplxPoseGrads* grads,
                             void* stream);

/* HumanGaussian's geometry around its networks (avatar/common/nets/module.py:524-539 with get_mean_offset_offset's
 * mask, :489-493, and model.py:92-96's warm-up clamp), per Gaussian p of P, in ExAvatar's fp32 operations and order:
 *   m = mesh + geo[0:3];  mmo = geo_offset[0:3] * (1 - mask);  mean_3d = m + expr_offset;
 *   mean_3d_refined = (m + (mmo + pose_offset)) + expr_offset;  scale = exp(geo[3]) x3;
 *   scale_refined = exp(geo[3] + geo_offset[3]) x3;  mean_offset_offset = mmo.
 * warmup != 0: scale_wo_clamp / scale_refined_wo_clamp receive the unclamped scales and scale / scale_refined
 * torch.clamp(x, max=0.001) (NaN stays NaN; the gradient passes where x <= 0.001).  mesh, pose_offset, expr_offset are
 * (P,3) contiguous; geo / geo_offset rows are 4 contiguous floats, geo_stride / geo_offset_stride floats apart (the
 * column views of a wider head output are read in place); mask (P) holds 0 or 1.  Outputs (P,3) contiguous.
 * Backward: upstream gradients may be NULL (zero); it writes d mesh, d expr_offset (P,3) and d geo, d geo_offset (P,4)
 * contiguous; pose_offset gets none (ExAvatar detaches the pose there).  One thread per Gaussian, each output element
 * written once: no atomics, no allocation, no sync. */
typedef struct B2RHumanAssets {
  int32_t P, warmup;
  int64_t geo_stride, geo_offset_stride;
  const float* mesh;
  const float* pose_offset;
  const float* expr_offset;
  const float* geo;
  const float* geo_offset;
  const float* mask;
} B2RHumanAssets;

typedef struct B2RHumanAssetsGrads {
  const float* dL_dmean_3d;               /* each (P,3) or NULL */
  const float* dL_dmean_3d_refined;
  const float* dL_dscale;
  const float* dL_dscale_refined;
  const float* dL_dmean_offset_offset;
  const float* dL_dscale_wo_clamp;        /* warmup only */
  const float* dL_dscale_refined_wo_clamp;
  float* dL_dmesh;                        /* (P,3) */
  float* dL_dexpr_offset;                 /* (P,3) */
  float* dL_dgeo;                         /* (P,4) */
  float* dL_dgeo_offset;                  /* (P,4) */
} B2RHumanAssetsGrads;

int b2r_human_geometry_forward(const B2RHumanAssets* h, float* mean_3d, float* mean_3d_refined, float* scale,
                               float* scale_refined, float* mean_offset_offset, float* scale_wo_clamp,
                               float* scale_refined_wo_clamp, void* stream);
int b2r_human_geometry_backward(const B2RHumanAssets* h, const B2RHumanAssetsGrads* g, void* stream);

/* HumanGaussian's colours (module.py:561): rgb_out = (tanh(rgb) + 1) / 2, rgb_refined = (tanh(rgb + rgb_offset) + 1) / 2,
 * (P,3) contiguous fp32, in torch's operations.  Backward: dL_drgb_out / dL_drgb_refined may be NULL (zero); writes
 * dL_drgb and dL_drgb_offset (P,3). */
int b2r_human_colors_forward(int32_t P, const float* rgb, const float* rgb_offset, float* rgb_out, float* rgb_refined,
                             void* stream);
int b2r_human_colors_backward(int32_t P, const float* rgb, const float* rgb_offset, const float* dL_drgb_out,
                              const float* dL_drgb_refined, float* dL_drgb, float* dL_drgb_offset, void* stream);

/* present[i] = 1 iff Gaussian i passes the near-plane test (z_view > 0.2). */
int b2r_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, uint8_t* present, void* stream);

/* Measurement hooks (host side).  Kernel ids: 0 project, 1 tile_scan, 2 scatter, 3 sort (all lists, long ones in chunks), 4 sort_merge (chunks of the long lists),
 * 5 composite_fwd, 6 composite_bwd, 7 project_bwd, 8 misc (status reset, the b2r_skin_*, b2r_l1ssim_*, b2r_nearest_rows, b2r_vertex_normals, b2r_mesh_render_*, b2r_triplane_*, b2r_gn_mlp_*, b2r_regs_*, b2r_rig_*, b2r_smplx_body_*, b2r_adam_step, b2r_lpips_*, b2r_scene_assets_*, b2r_decode_pose_* and b2r_human_* kernels).  With profiling on, every kernel launch
 * is bracketed by CUDA events on the caller's stream; b2r_profile_read() waits for them and returns the summed
 * milliseconds and launch counts per kernel id (arrays of B2R_NUM_KERNELS).  b2r_launch_count() counts kernel
 * launches made by this library since it was loaded, profiling or not. */
#define B2R_NUM_KERNELS 9
void b2r_profile_enable(int on);
int b2r_profile_read(double* ms_sum, uint64_t* counts, int reset);
uint64_t b2r_launch_count(void);
const char* b2r_kernel_name(int id);

/* Stage-level introspection for parity tests (device pointers into ctx; valid until ctx is reused).
 * geom: P x 12 floats {px, py, A2, B2 | C2, opacity, depth, thr2 | r, g, b, bits};  A2,B2,C2 are the conic
 * pre-scaled for exp2: A2 = -0.5*log2(e)*conic.x, B2 = -log2(e)*conic.y, C2 = -0.5*log2(e)*conic.z.
 * aux: P x 4 int32 {rect_min (x | y<<16), rect_max (x | y<<16), radius, tiles_kept}.
 * ranges: Tn x 2 uint32 [start,end) into dup_ids.  pixel_state: per pixel {final_T (float), n_contrib (uint32)}. */
const float* b2r_ctx_geom(const B2RWorkspace* ws, int32_t P, int32_t width, int32_t height);
const int32_t* b2r_ctx_aux(const B2RWorkspace* ws, int32_t P, int32_t width, int32_t height);
const uint32_t* b2r_ctx_ranges(const B2RWorkspace* ws, int32_t P, int32_t width, int32_t height);
const float* b2r_ctx_final_T(const B2RWorkspace* ws, int32_t P, int32_t width, int32_t height);
const uint32_t* b2r_ctx_n_contrib(const B2RWorkspace* ws, int32_t P, int32_t width, int32_t height);

#ifdef __cplusplus
}
#endif
#endif /* B200RASTER_H_ */
