// common.cuh -- shared constants, buffer layouts and device helpers of the rasteriser.
// Algorithm constants follow SURVEY.md App. A (the published 3DGS rasteriser the reference imports at
// avatar/common/nets/module.py:11); the kernel design is this repository's own.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200raster.h"

namespace b2r {

constexpr int TILE = 16;           // pixels per tile edge (App. A constants)
constexpr int TILE_PIX = TILE * TILE;
constexpr float K_NEAR = 0.2f;
constexpr float K_DILATE = 0.3f;
constexpr float K_ALPHA_MAX = 0.99f;
constexpr float K_ALPHA_MIN = 1.0f / 255.0f;
constexpr float K_T_MIN = 0.0001f;
constexpr float K_FRUSTUM = 1.3f;
constexpr float K_EPS_W = 0.0000001f;
constexpr float K_EIG_FLOOR = 0.1f;
constexpr float LOG2E = 1.4426950408889634f;
constexpr float INV_LOG2E = 0.6931471805599453f;
// slack (in log2 units) added to the "can this splat reach alpha >= 1/255 anywhere in this pixel rect" test so
// that rounding in the per-pixel evaluation can never disagree with a cull decision
constexpr float CULL_MARGIN2 = 0.02f;

#ifndef SORT_CTA_SHIFT
#define SORT_CTA_SHIFT 9  // log2 of the shortest list that gets a CTA of its own in the per-tile sort (tuning hook)
#endif
constexpr int SORT_CHUNK = 2048;  // per-tile sort: lists are sorted in chunks of this many entries (binning.cu)
// Segmented composites (composite_fwd4.cu / composite_bwd4.cu).  A tile's depth-sorted list is cut every SEG entries;
// the forward stores the per-pixel blend state at every cut (a "checkpoint record"), which lets the backward replay
// each (quarter tile, segment) as an independent work item.  SEG is a multiple of the forward's staging batch, so cuts are
// batch boundaries.
#ifndef SEG_SHIFT
#define SEG_SHIFT 9  // log2 of the segment length; tuning hook (build_ext.py B2R_NVCC_EXTRA).  Every work item pays ~6
                     // dependent global loads before its first batch, so fewer, longer items win until the longest chain
                     // becomes the tail
#endif
constexpr int SEG = 1 << SEG_SHIFT;
constexpr int CK_PLANE0 = TILE_PIX * 4;              // floats: per pixel (T, C_r, C_g, C_b)
constexpr int CK_REC_FLOATS = TILE_PIX * 4 + TILE_PIX * 2;  // + per pixel (depth sum, alpha sum)
constexpr size_t CK_REC_BYTES = (size_t)CK_REC_FLOATS * 4;  // 6144
// slots of Ctx::classes (written by tile_scan_kernel; positions refer to tile_order, which is sorted longest first)
enum { CLS_N_LARGE = 0,   // tiles with >= 2048 entries (sorted in chunks)
       CLS_N_GE512 = 1,   // tiles with >= 512 entries  (CTA-class sort; "heavy" tiles of the forward composite)
       CLS_N_MULTI = 2,   // tiles cut into segments (>= SEG entries), 0 when the caller gave no checkpoint buffer
       CLS_N_CHUNKS = 3,  // sort chunks of the large tiles
       CLS_TOTAL_SEGS = 4,  // segments of the multi-segment tiles
       CLS_N_GE1024 = 5,    // tiles with >= 1024 entries
       CLS_VIS_ACC = 6,     // visible-Gaussian accumulator of the projection kernel (published to B2RStatus by the scan)
       CLS_SCAN_FINAL = 7,  // 1 once a final scan has consumed the tile counters of the current projection
       CLS_COUNT = 8 };
constexpr size_t ALIGN = 256;
__host__ __device__ inline size_t align_up(size_t v) { return (v + ALIGN - 1) / ALIGN * ALIGN; }

struct Geom {  // 48 bytes per Gaussian, three 16-byte vectors
  float4 g0;   // px, py, A2, B2
  float4 g1;   // C2, opacity, depth, thr2
  float4 g2;   // r, g, b, id | SH clamp mask << 29 (uint bits)
};
static_assert(sizeof(Geom) == 48, "Geom must be 48 bytes");

struct CtxLayout {
  size_t status, geom, aux, ranges, tile_count, tile_cursor, tile_order, chunk_start, seg_start, classes, tile_maxid,
      split_len, final_T, n_contrib, total;
  int gx, gy, tiles;
};
__host__ __device__ inline CtxLayout ctx_layout(int P, int W, int H) {
  CtxLayout L;
  L.gx = (W + TILE - 1) / TILE;
  L.gy = (H + TILE - 1) / TILE;
  L.tiles = L.gx * L.gy;
  size_t Pn = P > 0 ? (size_t)P : 1, N = (size_t)W * H;
  size_t o = 0;
  L.status = o; o += align_up(sizeof(B2RStatus));
  L.geom = o; o += align_up(Pn * sizeof(Geom));
  L.aux = o; o += align_up(Pn * 16);
  L.ranges = o; o += align_up((size_t)L.tiles * 8);
  L.tile_count = o; o += align_up((size_t)L.tiles * 4);
  L.tile_cursor = o; o += align_up((size_t)L.tiles * 4);
  L.tile_order = o; o += align_up((size_t)L.tiles * 4);
  L.chunk_start = o; o += align_up((size_t)L.tiles * 4);
  L.seg_start = o; o += align_up((size_t)L.tiles * 4);
  L.classes = o; o += align_up((size_t)CLS_COUNT * 4);
  L.tile_maxid = o; o += align_up((size_t)L.tiles * 4);
  L.split_len = o; o += align_up((size_t)L.tiles * 4);
  L.final_T = o; o += align_up(N * 4);
  L.n_contrib = o; o += align_up(N * 4);
  L.total = o;
  return L;
}

struct ScratchLayout {
  size_t keys, total;
};
__host__ __device__ inline ScratchLayout scratch_layout(int P, int W, int H, uint64_t cap) {
  (void)P; (void)W; (void)H;
  ScratchLayout S;
  size_t o = 0;
  S.keys = o; o += align_up((size_t)(cap > 0 ? cap : 1) * 8);
  S.total = o;
  return S;
}
// a split pass (b2r_forward_bin_split) also keeps the sorted ids of its own rows in the scratch, behind the keys
__host__ __device__ inline size_t split_scratch_bytes(int P, int W, int H, uint64_t cap) {
  return scratch_layout(P, W, H, cap).total + align_up((size_t)(cap > 0 ? cap : 1) * 4);
}

// Resolved device pointers of one context.
struct Ctx {
  B2RStatus* status;
  Geom* geom;
  int4* aux;
  uint2* ranges;
  float* final_T;
  uint32_t* n_contrib;
  uint32_t* dup_ids;
  uint64_t dup_capacity;
  uint32_t* tile_count;
  uint32_t* tile_cursor;
  uint32_t* tile_order;  // tiles sorted longest list first (see tile_scan_kernel)
  uint32_t* chunk_start; // first sort chunk of the t-th tile of tile_order, for the tiles of >= 2048 entries
  uint2* keys;
  uint64_t* status_mirror;
  uint64_t status_token;
  int gx, gy, tiles;
  // segmentation (all null / 0 when the workspace carries no checkpoint buffer: every list is then one segment)
  uint32_t* seg_start;   // by position in tile_order, multi-segment tiles: segments (= checkpoint records) of all earlier ones
  uint32_t* classes;     // CLS_* counters
  uint2* seg_table;      // one (tile_order position, segment index) per segment of the multi-segment tiles
  float* ckpt;           // checkpoint records, CK_REC_FLOATS each
  uint32_t max_segs;     // capacity of seg_table / ckpt in segments
  // view (B2RView): which Gaussians take part, with which background, and where the per-pixel state lives
  uint32_t id_begin, id_span;  // Gaussian i takes part iff i - id_begin < id_span (unsigned)
  const float* bg;
  uint32_t* tile_maxid;  // per tile: largest Gaussian index in its list (written by the per-tile sort)
  uint32_t skip_below;   // != 0: the composites skip tiles whose tile_maxid < skip_below (B2RView.skip_below)
  // split pass only (b2r_forward_bin_split), else null: per tile, how many entries of its range the per-tile sort covers
  // (the pass's own rows; the rest of the range is filled by the merge with the base pass's list)
  uint32_t* sort_len;
};
// entries of the tile's range the per-tile sort orders
__device__ __forceinline__ int sort_length(const Ctx& cx, int tile, uint2 r) {
  const int n = (int)(r.y - r.x);
  return cx.sort_len ? min(n, (int)cx.sort_len[tile]) : n;
}

// capacity of the segment table / checkpoint store for a given duplicate capacity
__host__ __device__ inline uint32_t max_segments(int tiles, uint64_t cap) { return (uint32_t)(cap / SEG) + (uint32_t)tiles; }
__host__ __device__ inline size_t seg_table_bytes(uint32_t max_segs) { return align_up((size_t)max_segs * 8); }

inline Ctx resolve(const B2RWorkspace* ws, int P, int W, int H) {
  CtxLayout L = ctx_layout(P, W, H);
  ScratchLayout S = scratch_layout(P, W, H, ws->dup_capacity);
  char* c = (char*)ws->ctx;
  char* s = (char*)ws->scratch;
  Ctx x;
  x.status = (B2RStatus*)(c + L.status);
  x.geom = (Geom*)(c + L.geom);
  x.aux = (int4*)(c + L.aux);
  x.ranges = (uint2*)(c + L.ranges);
  x.final_T = (float*)(c + L.final_T);
  x.n_contrib = (uint32_t*)(c + L.n_contrib);
  x.dup_ids = ws->dup_ids;
  x.dup_capacity = ws->dup_capacity;
  x.tile_count = (uint32_t*)(c + L.tile_count);
  x.tile_cursor = (uint32_t*)(c + L.tile_cursor);
  x.tile_order = (uint32_t*)(c + L.tile_order);
  x.chunk_start = (uint32_t*)(c + L.chunk_start);
  x.keys = s ? (uint2*)(s + S.keys) : nullptr;
  x.status_mirror = ws->status_mirror;
  x.status_token = ws->status_token;
  x.gx = L.gx; x.gy = L.gy; x.tiles = L.tiles;
  x.seg_start = (uint32_t*)(c + L.seg_start);
  x.classes = (uint32_t*)(c + L.classes);
  x.seg_table = nullptr; x.ckpt = nullptr; x.max_segs = 0;
  if (ws->checkpoints) {
    const uint32_t ms = max_segments(L.tiles, ws->dup_capacity);
    if (ws->checkpoint_bytes >= seg_table_bytes(ms) + (size_t)ms * CK_REC_BYTES) {
      x.seg_table = (uint2*)ws->checkpoints;
      x.ckpt = (float*)((char*)ws->checkpoints + seg_table_bytes(ms));
      x.max_segs = ms;
    }
  }
  x.id_begin = 0; x.id_span = 0xffffffffu;
  x.bg = nullptr;
  x.tile_maxid = (uint32_t*)(c + L.tile_maxid);
  x.skip_below = 0;
  x.sort_len = nullptr;
  return x;
}

// ---------------------------------------------------------------------------------------------
// Region test shared by the binning (16x16 tile) and the composites (8x4 warp sub-tile).
// The splat's exponent in log2 units is  p2(dx,dy) = A2 dx^2 + B2 dx dy + C2 dy^2  with d = centre - pixel,
// concave when A2 < 0, C2 < 0, 4 A2 C2 > B2^2.  Returns an upper bound of p2 over all pixel centres of the
// inclusive rect [x0,x1] x [y0,y1]: exact maximum over the continuous rect (a superset of the pixel centres).
// A splat can pass the alpha >= 1/255 test somewhere in the rect only if  bound >= thr2 (geom.g1.w).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float region_max_p2(float sx, float sy, float A2, float B2, float C2, float x0, float y0,
                                               float x1, float y1) {
  const float lx = sx - x1, hx = sx - x0;  // dx range
  const float ly = sy - y1, hy = sy - y0;  // dy range
  const bool in_x = (lx <= 0.f) && (hx >= 0.f);
  const bool in_y = (ly <= 0.f) && (hy >= 0.f);
  if (in_x && in_y) return 0.f;
  float best = -INFINITY;
  if (!in_x) {  // nearest vertical edge; maximise over dy on it
    const float ex = lx > 0.f ? lx : hx;
    float dy = __fdividef(-B2 * ex, 2.f * C2);
    dy = fminf(fmaxf(dy, ly), hy);
    best = fmaxf(best, A2 * ex * ex + B2 * ex * dy + C2 * dy * dy);
  }
  if (!in_y) {
    const float ey = ly > 0.f ? ly : hy;
    float dx = __fdividef(-B2 * ey, 2.f * A2);
    dx = fminf(fmaxf(dx, lx), hx);
    best = fmaxf(best, A2 * dx * dx + B2 * dx * ey + C2 * ey * ey);
  }
  return best;
}

// ---------------------------------------------------------------------------------------------------------------
// Tile culling by ROWS.  The tiles a splat keeps are those whose pixel-centre rectangle intersects the ellipse
// E = { p2(d) >= thr2 }.  Round 1 / 2 tested every tile of the 3-sigma rect with region_max_p2 (~45 instructions per tile,
// and a warp pays the largest rect among its lanes: the projection spent ~45 % of its instructions there).  For one tile
// ROW the kept tiles form an interval: the band y in [y0, y1] cuts E in a convex set whose x-extent [xl, xr] has a closed
// form -- the right end of the chord at height dy,  dx(dy) = (-B2 dy - sqrt(D dy^2 + 4 A2 thr2)) / (2 A2)  with
// D = B2^2 - 4 A2 C2 < 0, is concave in dy, so its maximum over the band is at the clamped apex
// dy* = -B2 dx_top / (2 C2), dx_top = sqrt(4 C2 thr2 / -D); the left end is its mirror image -- and a tile of the row is
// kept iff its pixel-centre range meets [xl, xr].  Same set as the per-tile test (the rect spans the whole band, so
// "rect meets E" <=> "x-range of the rect meets the x-extent of E in the band"), ~40 instructions per row instead of ~45
// per tile.  The interval is padded by 0.01 px against the rounding of the closed form (a superset is always allowed:
// the composites cull again per 8x4 pixel rect); a numpy restatement checked it on 2.7 M (splat, tile) pairs: no kept tile
// missed, 0.03 % more pairs (tests/test_tile_rows.py).
// ---------------------------------------------------------------------------------------------------------------
struct RowCull {  // per-splat constants of the row test
  float sx, sy, A2, B2, nD4, fA4t, dy_ext, dys, inv2A;
  int mode;       // 0: closed form, 1: keep every tile (culling off / degenerate conic), 2: keep none
};
__device__ __forceinline__ RowCull row_cull_setup(float sx, float sy, float A2, float B2, float C2, float thr2, bool no_cull) {
  RowCull rc;
  rc.sx = sx; rc.sy = sy; rc.A2 = A2; rc.B2 = B2;
  rc.mode = (no_cull || thr2 == -INFINITY) ? 1 : 0;
  const float D = B2 * B2 - 4.f * A2 * C2;      // < 0 for a concave conic
  const float k = __fdividef(4.f * thr2, -D);   // dy_ext^2 = A2 k, dx_top^2 = C2 k  (A2, C2 < 0 and thr2 < 0 => both > 0)
  rc.dy_ext = sqrtf(A2 * k);                    // NaN when thr2 > 0 or +inf: the splat reaches 1/255 nowhere
  const float dx_top = sqrtf(C2 * k);
  rc.dys = __fdividef(-B2, 2.f * C2) * dx_top;  // dy at the rightmost point of the ellipse
  rc.nD4 = D;
  rc.fA4t = 4.f * A2 * thr2;
  rc.inv2A = __fdividef(1.f, 2.f * A2);
  if (rc.mode == 0 && !(rc.dy_ext >= 0.f)) rc.mode = 2;
  return rc;
}
constexpr float ROW_PAD = 0.01f;
// Kept tile columns [tlo, thi] (inclusive; empty when tlo > thi) of tile row `ty` inside the rect columns [x0, x1).
__device__ __forceinline__ void row_kept_columns(const RowCull& rc, int ty, int x0, int x1, int W, int H, int& tlo, int& thi) {
  tlo = x0; thi = x1 - 1;
  if (rc.mode == 1) return;
  if (rc.mode == 2) { thi = tlo - 1; return; }
  const float y0 = (float)(ty * TILE), y1 = fminf(y0 + (float)(TILE - 1), (float)(H - 1));
  const float lo = fmaxf(rc.sy - y1, -rc.dy_ext), hi = fminf(rc.sy - y0, rc.dy_ext);
  if (!(lo <= hi)) { thi = tlo - 1; return; }
  const float dyr = fminf(fmaxf(rc.dys, lo), hi), dyl = fminf(fmaxf(-rc.dys, lo), hi);
  const float disc_r = fmaxf(rc.nD4 * dyr * dyr + rc.fA4t, 0.f), disc_l = fmaxf(rc.nD4 * dyl * dyl + rc.fA4t, 0.f);
  const float dx_hi = (-rc.B2 * dyr - sqrtf(disc_r)) * rc.inv2A;  // largest dx = centre - x  => smallest x
  const float dx_lo = (-rc.B2 * dyl + sqrtf(disc_l)) * rc.inv2A;
  const float xl = rc.sx - dx_hi - ROW_PAD, xr = rc.sx - dx_lo + ROW_PAD;
  if (!(xl <= (float)(W - 1))) { thi = tlo - 1; return; }  // every tile's last pixel centre is <= W - 1
  // tile tx spans pixel centres [16 tx, min(16 tx + 15, W - 1)]: kept iff xl <= its last and xr >= its first centre
  tlo = max(x0, (int)ceilf((xl - (float)(TILE - 1)) * (1.f / TILE)));
  thi = min(x1 - 1, (int)floorf(xr * (1.f / TILE)));
}

// tile index t (row-major inside a rect of width w) -> row; exact for the sizes that occur: (t + 0.5) / w is at least
// 0.5 / w away from an integer, far more than the rounding of the reciprocal and the product
__device__ __forceinline__ int rect_row(int t, float inv_w) { return (int)(((float)t + 0.5f) * inv_w); }

// Warp-cooperative enumeration of the tiles a Gaussian keeps (rect minus culled tiles).  Every lane brings one
// Gaussian (or active = false).  A lane walks the rows of its own rect, or -- when few lanes carry tall rects -- a rect is
// broadcast and its rows are spread over the 32 lanes.  Must be called by full warps.
constexpr int KEPT_SMALL = 4;
#ifndef WALK_ROW_COST_N
#define WALK_ROW_COST_N 40  // tuning hooks (build_ext.py B2R_NVCC_EXTRA): modelled instructions per row / per kept tile
#endif
constexpr unsigned WALK_ROW_COST = WALK_ROW_COST_N, WALK_TILE_COST = 10u, WALK_BCAST_COST = 30u;

// bits [pos, pos + cnt) of a 32-bit mask (cnt >= 1, pos + cnt <= 32)
__device__ __forceinline__ uint32_t bit_run(int pos, int cnt) { return (cnt >= 32 ? 0xffffffffu : ((1u << cnt) - 1u)) << pos; }

// The counting walk (projection): table[ty * gx + tx] += 1 once per kept tile.  Returns, to the owner lane, the KEPT MASK
// of a rect of at most 32 tiles (bit t = tile t in row-major order); the scatter replays it instead of repeating the walk.
__device__ __forceinline__ uint32_t warp_count_kept_tiles(bool active, int x0, int y0, int x1, int y1, float px, float py,
                                                          float A2, float B2, float C2, float thr2, bool no_cull, int W,
                                                          int H, int gx, uint32_t* table) {
  const int lane = threadIdx.x & 31;
  const int w = x1 - x0, h = y1 - y0;
  const int area = active ? w * h : 0;
  uint32_t kept = 0u;
  // Schedule (warp-uniform), by modelled cost: every lane walks its own rect (the warp pays the most expensive lane), or
  // the rects of more than KEPT_SMALL tiles are broadcast one after the other and their rows spread over the lanes.
  const bool big = area > KEPT_SMALL;
  const unsigned own_cost = area ? (unsigned)h * WALK_ROW_COST + (unsigned)area * WALK_TILE_COST : 0u;
  const unsigned coop_cost = big ? WALK_BCAST_COST + (unsigned)((h + 31) >> 5) * (WALK_ROW_COST + (unsigned)w * WALK_TILE_COST) : 0u;
  const unsigned max_own = __reduce_max_sync(0xffffffffu, own_cost);
  const unsigned sum_coop = __reduce_add_sync(0xffffffffu, coop_cost);
  const bool all_private = max_own <= sum_coop + 64u;
  if (area > 0 && (all_private || !big)) {
    const RowCull rc = row_cull_setup(px, py, A2, B2, C2, thr2, no_cull);
    for (int ty = y0; ty < y1; ty++) {
      int tlo, thi;
      row_kept_columns(rc, ty, x0, x1, W, H, tlo, thi);
      if (tlo <= thi) {
        if (area <= 32) kept |= bit_run((ty - y0) * w + (tlo - x0), thi - tlo + 1);
        uint32_t* row = table + ty * gx;
        for (int tx = tlo; tx <= thi; tx++) atomicAdd(row + tx, 1u);
      }
    }
  }
  unsigned mask = all_private ? 0u : __ballot_sync(0xffffffffu, big);
  while (mask) {
    const int src = __ffs(mask) - 1;
    mask &= mask - 1;
    const int bx0 = __shfl_sync(0xffffffffu, x0, src), by0 = __shfl_sync(0xffffffffu, y0, src);
    const int bx1 = __shfl_sync(0xffffffffu, x1, src), by1 = __shfl_sync(0xffffffffu, y1, src);
    const float spx = __shfl_sync(0xffffffffu, px, src), spy = __shfl_sync(0xffffffffu, py, src);
    const float sA = __shfl_sync(0xffffffffu, A2, src), sB = __shfl_sync(0xffffffffu, B2, src);
    const float sC = __shfl_sync(0xffffffffu, C2, src), sT = __shfl_sync(0xffffffffu, thr2, src);
    const RowCull rc = row_cull_setup(spx, spy, sA, sB, sC, sT, no_cull);
    const int bw = bx1 - bx0;
    const bool small = bw * (by1 - by0) <= 32;
    uint32_t bits = 0u;
    for (int ty = by0 + lane; ty < by1; ty += 32) {
      int tlo, thi;
      row_kept_columns(rc, ty, bx0, bx1, W, H, tlo, thi);
      if (tlo <= thi) {
        if (small) bits |= bit_run((ty - by0) * bw + (tlo - bx0), thi - tlo + 1);
        uint32_t* row = table + ty * gx;
        for (int tx = tlo; tx <= thi; tx++) atomicAdd(row + tx, 1u);
      }
    }
    bits = __reduce_or_sync(0xffffffffu, bits);
    if (lane == src) kept = bits;
  }
  return kept;
}

// The replay (scatter): the same (splat, tile) pairs as warp_count_kept_tiles produced.  Per pair: old = table[tile]++,
// then post(old, tile, u0, u1) with the owner's two payload words.  A rect of <= 32 tiles is replayed by its own lane from
// the stored mask (a loop over the set bits: no shuffles, no geometry; the warp pays the largest pair count among its
// lanes, a handful).  Larger rects repeat the row walk (the same row_kept_columns on the same inputs in a unit compiled
// with the same flags, so the pairs are identical), privately or with their rows spread over the lanes; px..thr2 need to
// be valid on lanes whose rect has more than 32 tiles only.  Must be called by full warps.
template <typename F>
__device__ __forceinline__ void warp_replay_kept_tiles(bool active, int x0, int y0, int x1, int y1, uint32_t kept, float px,
                                                       float py, float A2, float B2, float C2, float thr2, uint32_t u0,
                                                       uint32_t u1, bool no_cull, int W, int H, int gx, uint32_t* table,
                                                       F&& post) {
  const int lane = threadIdx.x & 31;
  const int w = x1 - x0, h = y1 - y0;
  const int area = active ? w * h : 0;
  if (area > 0 && area <= 32) {
    const float inv_w = __frcp_rn((float)w);
    const int tile0 = y0 * gx + x0;
    for (uint32_t m = kept; m; m &= m - 1u) {
      const int t = __ffs(m) - 1;
      const int r = rect_row(t, inv_w);
      const int tile = tile0 + r * gx + (t - r * w);
      post(atomicAdd(table + tile, 1u), tile, u0, u1);
    }
  }
  const bool big = area > 32;
  const unsigned own_cost = big ? (unsigned)h * WALK_ROW_COST + (unsigned)area * WALK_TILE_COST : 0u;
  const unsigned coop_cost = big ? WALK_BCAST_COST + (unsigned)((h + 31) >> 5) * (WALK_ROW_COST + (unsigned)w * WALK_TILE_COST) : 0u;
  const unsigned sum_coop = __reduce_add_sync(0xffffffffu, coop_cost);
  if (sum_coop == 0u) return;
  const unsigned max_own = __reduce_max_sync(0xffffffffu, own_cost);
  if (max_own <= sum_coop) {
    if (big) {
      const RowCull rc = row_cull_setup(px, py, A2, B2, C2, thr2, no_cull);
      for (int ty = y0; ty < y1; ty++) {
        int tlo, thi;
        row_kept_columns(rc, ty, x0, x1, W, H, tlo, thi);
        for (int tx = tlo; tx <= thi; tx++) {
          const int tile = ty * gx + tx;
          post(atomicAdd(table + tile, 1u), tile, u0, u1);
        }
      }
    }
    return;
  }
  unsigned mask = __ballot_sync(0xffffffffu, big);
  while (mask) {
    const int src = __ffs(mask) - 1;
    mask &= mask - 1;
    const int bx0 = __shfl_sync(0xffffffffu, x0, src), by0 = __shfl_sync(0xffffffffu, y0, src);
    const int bx1 = __shfl_sync(0xffffffffu, x1, src), by1 = __shfl_sync(0xffffffffu, y1, src);
    const uint32_t s0 = __shfl_sync(0xffffffffu, u0, src), s1 = __shfl_sync(0xffffffffu, u1, src);
    const float spx = __shfl_sync(0xffffffffu, px, src), spy = __shfl_sync(0xffffffffu, py, src);
    const float sA = __shfl_sync(0xffffffffu, A2, src), sB = __shfl_sync(0xffffffffu, B2, src);
    const float sC = __shfl_sync(0xffffffffu, C2, src), sT = __shfl_sync(0xffffffffu, thr2, src);
    const RowCull rc = row_cull_setup(spx, spy, sA, sB, sC, sT, no_cull);
    for (int ty = by0 + lane; ty < by1; ty += 32) {
      int tlo, thi;
      row_kept_columns(rc, ty, bx0, bx1, W, H, tlo, thi);
      for (int tx = tlo; tx <= thi; tx++) {
        const int tile = ty * gx + tx;
        post(atomicAdd(table + tile, 1u), tile, s0, s1);
      }
    }
  }
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// 16-byte vector reduction to global memory (sm_90+): one L2 atomic transaction instead of four.
__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// ---------------------------------------------------------------------------------------------------------------
// Warp-cooperative staging of 32 consecutive rows of L floats (SH coefficients / their gradients) between global and
// shared memory.  Global side: the rows are one contiguous block, moved with full-line accesses and all loads of a
// lane in flight together.  Shared side: row stride S = L | 1 (odd), so "every lane reads its own row" is conflict-free.
// mode 0: shared <- global;  1: global <- shared;  2: global += shared.  `row_mask` (modes 1, 2) selects rows.
// ---------------------------------------------------------------------------------------------------------------
template <int MODE>
__device__ __forceinline__ void stage_rows(float* __restrict__ wstage, float* __restrict__ gptr, const int L, const int nrows,
                                           const unsigned row_mask) {
  const int lane = threadIdx.x & 31;
  const int S = L | 1;
  if (L == 48 && (reinterpret_cast<uintptr_t>(gptr) & 15) == 0) {  // degree-3 layout: 12 float4 per row
    float4* g4 = reinterpret_cast<float4*>(gptr);
    const int n4 = nrows * 12;
    float4 v[12];
    if (MODE != 1) {
#pragma unroll
      for (int u = 0; u < 12; u++) {
        const int j = lane + 32 * u;
        // masked rows are never touched, not even read: with a detached prefix they lie before the output buffer
        const bool rd = j < n4 && (MODE == 0 || ((row_mask >> (j / 12)) & 1u));
        v[u] = rd ? (MODE == 0 ? __ldg(g4 + j) : g4[j]) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int u = 0; u < 12; u++) {
      const int j = lane + 32 * u;
      const int r = j / 12, c = (j - r * 12) * 4;
      float* w = wstage + r * S + c;
      if (j < n4) {
        if (MODE == 0) {
          w[0] = v[u].x; w[1] = v[u].y; w[2] = v[u].z; w[3] = v[u].w;
        } else if ((row_mask >> r) & 1u) {
          if (MODE == 1) g4[j] = make_float4(w[0], w[1], w[2], w[3]);
          else g4[j] = make_float4(v[u].x + w[0], v[u].y + w[1], v[u].z + w[2], v[u].w + w[3]);
        }
      }
    }
    return;
  }
  const int total = nrows * L;
  for (int e0 = lane; e0 < total; e0 += 32 * 8) {
    float v[8];
    if (MODE != 1) {
#pragma unroll
      for (int u = 0; u < 8; u++) {
        const int e = e0 + 32 * u;
        v[u] = (e < total && (MODE == 0 || ((row_mask >> (e / L)) & 1u))) ? gptr[e] : 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < 8; u++) {
      const int e = e0 + 32 * u;
      if (e < total) {
        const int r = e / L, c = e - r * L;
        float* w = wstage + r * S + c;
        if (MODE == 0) *w = v[u];
        else if ((row_mask >> r) & 1u) gptr[e] = MODE == 1 ? *w : v[u] + *w;
      }
    }
  }
}

// Crop box of ExAvatar's image losses (l1ssim.cu, lpips.cu), read on the device.
struct Crop {
  int x0, y0, x1, y1;  // [y0, y1) x [x0, x1), x1 >= x0, y1 >= y0
  __device__ bool has(int x, int y) const { return x >= x0 && x < x1 && y >= y0 && y < y1; }
  __device__ float count3() const { return 3.f * (float)(x1 - x0) * (float)(y1 - y0); }
};

// the reference's integer rules: int() truncates, the CLAMPED start is added to the width (a box with negative xmin
// moves right instead of being clipped), the end is clamped to the image
__device__ __forceinline__ int trunc_i(float v) { return __float2int_rz(fminf(fmaxf(v, -1e9f), 1e9f)); }
__device__ __forceinline__ Crop read_crop(const float* bbox, int W, int H) {
  Crop c{0, 0, W, H};
  if (bbox) {
    c.x0 = max(trunc_i(bbox[0]), 0);
    c.y0 = max(trunc_i(bbox[1]), 0);
    c.x1 = max(min(c.x0 + trunc_i(bbox[2]), W), c.x0);
    c.y1 = max(min(c.y0 + trunc_i(bbox[3]), H), c.y0);
  }
  return c;
}

// TF32 tensor-core helpers (gn_mlp.cu, lpips.cu): round to TF32 with cvt.rna, d += a.b on one m16n8k8 tile
__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ---------------------------------------------------------------------------------------------------------------
// Fixed-order sums, behind every op's "bit-identical run to run" and "no float atomics".  A warp sums by an xor
// butterfly (16, 8, 4, 2, 1); a block stores one value per warp in shared memory and thread 0 folds them in warp order,
// starting from zero (so a zero sum keeps its sign).  They only add: --fmad=false does not change them.
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {  // every lane ends with the same bits
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// v[0..N) already the same across each warp of a THREADS-thread block -> thread 0's v holds the block's N sums (the
// other threads' v is unchanged).  wsum: THREADS / 32 x N values in shared memory, warp-major.  Every thread of the
// block calls it; the barrier in front lets the next call reuse wsum.
template <int THREADS, typename T, int N>
__device__ __forceinline__ void block_fold(T (&v)[N], T* wsum) {
  __syncthreads();
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int i = 0; i < N; i++) wsum[(threadIdx.x >> 5) * N + i] = v[i];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int i = 0; i < N; i++) {
      T s = T(0);
      for (int w = 0; w < THREADS / 32; w++) s += wsum[w * N + i];
      v[i] = s;
    }
}

// the block's N sums of v[0..N), in thread 0 (block_fold after warp_sum)
template <int THREADS, typename T, int N>
__device__ __forceinline__ void block_sum(T (&v)[N], T* wsum) {
#pragma unroll
  for (int i = 0; i < N; i++) v[i] = warp_sum(v[i]);
  block_fold<THREADS>(v, wsum);
}

// the column sums of n rows of N partials at p (row-major) into v, in thread 0: thread t adds rows t, t + THREADS, ...
// and then block_sum runs
template <int THREADS, typename T, int N>
__device__ __forceinline__ void block_sum_strided(const T* p, int n, T (&v)[N], T* wsum) {
#pragma unroll
  for (int i = 0; i < N; i++) v[i] = T(0);
  for (int r = threadIdx.x; r < n; r += THREADS)
#pragma unroll
    for (int i = 0; i < N; i++) v[i] += p[r * N + i];
  block_sum<THREADS>(v, wsum);
}

// The byte ExAvatar's test.py stores for an fp32 value p: cv2.imwrite(path, img * 255) of a float32 array converts with
// saturate_cast<uchar>, i.e. v = fl(p * 255), then 0 if v is NaN or |v| >= 2^31 (cvRound's out-of-range result
// saturates to 0), else clamp(rint(v), 0, 255) with ties to even.  The PNG stores that byte losslessly.  Callers are
// compiled with --fmad=false (metrics.cu, compose.cu), though the product is rounded on its own either way.
__device__ __forceinline__ int png_u8(float p) {
  const float v = p * 255.f;
  if (isnan(v) || fabsf(v) >= 2147483648.f) return 0;  // cvRound's out-of-range result saturates to 0
  return min(max(__float2int_rn(v), 0), 255);          // an integer: rint(-0.4) = -0 reads back as +0
}

// launch wrappers (one per translation unit)
int launch_project(const B2RScene& sc, const Ctx& cx, int32_t* radii, cudaStream_t st, int first_row = 0);
int launch_binning(const B2RScene& sc, const Ctx& cx, bool rescan, cudaStream_t st);
int launch_binning_split(const B2RScene& sc, const Ctx& cx, const Ctx& base, uint32_t* own_ids, int first_row,
                         int32_t* radii, cudaStream_t st);
void launch_tile_scan(const Ctx& cx, cudaStream_t st, int final = 2);  // final: see tile_scan_kernel
int launch_composite_fwd(const B2RScene& sc, const Ctx& cx, const B2RForwardOutputs& out, cudaStream_t st);
int launch_composite_bwd(const B2RScene& sc, const Ctx& cx, const B2RBackwardArgs& a, float* gacc, cudaStream_t st);

int launch_project_bwd(const B2RScene& sc, const Ctx& cx, const B2RBackwardArgs& a, const float* gacc, cudaStream_t st);
int launch_mark_visible(int P, const float* means3D, const float* view, uint8_t* present, cudaStream_t st);
int launch_skin_forward(const B2RSkin& s, cudaStream_t st);
int launch_skin_backward(const B2RSkin& s, const float* const dposed[2], float* const dxyz[2], float* djoint,
                         float* dtrans, void* scratch, cudaStream_t st);
size_t skin_scratch_bytes(int P, int J);
int launch_l1ssim_forward(int W, int H, const float* img, const float* target, const float* mask, const float* bbox,
                          bool with_ssim, float* out, void* scratch, cudaStream_t st);
int launch_l1ssim_backward(int W, int H, const float* img, const float* target, const float* mask, const float* bbox,
                           bool with_ssim, const float* dout, float* dimg, const void* scratch, cudaStream_t st);
size_t l1ssim_scratch_bytes(int W, int H);
int launch_nearest_rows(int P, const float* queries, int V, const float* targets, const uint8_t* self_map,
                        int32_t* rows, void* scratch, cudaStream_t st);
size_t nearest_scratch_bytes(int V);
int launch_vertex_normals(int P, const float* xyz, const int32_t* faces, const int32_t* vf_offsets,
                          const int32_t* vf_entries, const uint8_t* flip, float* normals, cudaStream_t st);
size_t mesh_render_scratch_bytes(int F);
int launch_mesh_render_forward(const B2RMeshRender& m, float* image, int32_t* pix_to_face, void* scratch,
                               cudaStream_t st);
int launch_mesh_render_backward(const B2RMeshRender& m, const int32_t* pix_to_face, const float* dimage, float* dmesh,
                                void* scratch, cudaStream_t st);
int launch_mesh_shade_forward(const B2RMeshRender& m, const float* normals, const float* bkg, float blend,
                              float blend_complement, float* out, void* scratch, cudaStream_t st);
int launch_triplane_forward(int P, int C, int H, int W, const float* planes, const float* planes_face,
                            const uint8_t* is_face, const int32_t* corners, const float* weights, float* feat,
                            cudaStream_t st);
int launch_triplane_backward(int C, int H, int W, const float* dfeat, const int32_t* offsets, const int32_t* rows,
                             const float* w, float* dplanes, float* dplanes_face, cudaStream_t st);
size_t gn_mlp_scratch_bytes(int P);
size_t gn_mlp_grads_count(int K, int H);
int launch_gn_mlp_forward(const B2RGnMlp& m, float* out, float* saved, cudaStream_t st);
int launch_gn_mlp_backward(const B2RGnMlp& m, const float* saved, const float* dout, float* dx, float* grads,
                           void* scratch, cudaStream_t st);
size_t regs_scratch_bytes(int P, int n_arm);
int launch_regs_forward(const B2RRegs& r, float* out, void* scratch, cudaStream_t st);
int launch_regs_backward(const B2RRegs& r, const float* dout, const B2RRegsGrads& g, const void* scratch,
                         cudaStream_t st);
size_t rig_scratch_bytes(int V, int J, int NB, int NE);
int launch_rig_forward(const B2RRig& r, float* mesh, float* mesh_wo, float* joint_mats, float* pose_offset,
                       float* expr_offset, float* pose_6d, void* scratch, cudaStream_t st);
int launch_rig_backward(const B2RRig& r, const float* dmesh, const float* djm, const float* dexpr, const B2RRigGrads& g,
                        void* scratch, cudaStream_t st);
// the body with its B2RRig's four input pointers set to the body's (the rig's validation and shape pass read them)
inline B2RSmplxBody with_body_inputs(const B2RSmplxBody& b) {
  B2RSmplxBody o = b;
  o.rig.shape_param = b.shape_param;
  o.rig.joint_offset = b.joint_offset;
  o.rig.full_pose = b.full_pose;
  o.rig.expr = b.expr;
  return o;
}
size_t smplx_body_scratch_bytes(int V);
int launch_smplx_body_forward(const B2RSmplxBody& b, float* mesh, void* scratch, cudaStream_t st);
int launch_smplx_body_backward(const B2RSmplxBody& b, const float* dmesh, const B2RSmplxBodyGrads& g, void* scratch,
                               cudaStream_t st);
int launch_smplx_body_joints(const B2RSmplxBody& b, const void* scratch, float* joints, cudaStream_t st);
int launch_orbit_camera(const B2ROrbitCamera& p, cudaStream_t st);
int launch_orbit_points(int n, const float* points, const float* state, int view, float* out, cudaStream_t st);
int launch_animation_panel(const B2RAnimationPanel& p, uint8_t* out, cudaStream_t st);
int launch_adam_step(const B2RAdamSegment* table, int n_segments, int64_t n_chunks, cudaStream_t st);
size_t lpips_saved_bytes(int W, int H, int N);
size_t lpips_scratch_bytes(int W, int H);
int launch_lpips_forward(const B2RLpips& p, float* out, float* saved, void* scratch, cudaStream_t st);
int launch_lpips_backward(const B2RLpips& p, const float* saved, const float* dout, float* dimg, void* scratch,
                          cudaStream_t st);
size_t neuman_scratch_bytes(int W, int H, int N);
int launch_neuman_scores(const B2RNeumanScores& p, float* out, void* scratch, cudaStream_t st);
int launch_face_composite_forward(const B2RFaceComposite& p, float* out, cudaStream_t st);
int launch_face_composite_backward(const B2RFaceComposite& p, const float* dout, float* dimg, float* dface,
                                   cudaStream_t st);
int launch_test_outputs(const B2RTestOutputs& p, float* const composite[4], uint8_t* png, cudaStream_t st);
int launch_scene_assets_forward(const B2RSceneAssets& s, float* opacity, float* scale, float* rotation, float* color,
                                cudaStream_t st);
int launch_scene_assets_backward(const B2RSceneAssets& s, const B2RSceneAssetsGrads& g, cudaStream_t st);
int launch_decode_pose_forward(const B2RSmplxPose& p, float* full_pose, cudaStream_t st);
int launch_decode_pose_backward(const B2RSmplxPose& p, const float* dfull, const B2RSmplxPoseGrads& g, cudaStream_t st);
int launch_param_table_forward(const B2RSmplxParamTable& t, float* full_pose, float* expr, float* trans,
                               cudaStream_t st);
int launch_param_table_backward(const B2RSmplxParamTable& t, const B2RSmplxParamTableGrads& g, cudaStream_t st);
int launch_frame_unpack(const B2RFrameTable& t, float* img, float* mask, float* bbox, float* R, float* tr, float* focal,
                        float* princpt, int64_t* frame_idx, cudaStream_t st);
int launch_segmentation_unpack(const B2RSegmentation& s, float* mask, cudaStream_t st);
int launch_human_geometry_forward(const B2RHumanAssets& h, float* mean, float* mean_r, float* scale, float* scale_r,
                                  float* mmo, float* scale_wo, float* scale_r_wo, cudaStream_t st);
int launch_human_geometry_backward(const B2RHumanAssets& h, const B2RHumanAssetsGrads& g, cudaStream_t st);
int launch_human_colors_forward(int P, const float* rgb, const float* off, float* out, float* out_r, cudaStream_t st);
int launch_human_colors_backward(int P, const float* rgb, const float* off, const float* g, const float* g_r,
                                 float* d_rgb, float* d_off, cudaStream_t st);
int launch_camera_setup(const float* R, const float* t, const float* focal, int W, int H, float* out, cudaStream_t st);

// RAII bracket around one kernel launch: counts it and, when profiling is on, records CUDA events around it.
enum KernelId { K_PROJECT = 0, K_TILE_SCAN, K_SCATTER, K_SORT_SMALL, K_SORT_LARGE, K_COMPOSITE_FWD, K_COMPOSITE_BWD,
                K_PROJECT_BWD, K_MISC };
struct ProfScope {
  int id;
  cudaStream_t st;
  bool on;
  cudaEvent_t a;
  ProfScope(int id, cudaStream_t st, int launches = 1);
  ~ProfScope();
};

// Optional per-CTA timeline (compile with -DB2R_CTA_TRACE; tools/cta_trace.py): every composite CTA records
// {start ns, end ns, smid, list length} so the schedule (tail, per-SM balance, longest chain) can be reconstructed.
#ifdef B2R_CTA_TRACE
static __device__ unsigned long long* g_cta_trace;  // one copy per translation unit, set by b2r_debug_trace_*()
__device__ __forceinline__ unsigned long long trace_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void trace_end(unsigned long long t0, int n) {
  if (threadIdx.x == 0 && g_cta_trace) {
    unsigned smid;
    asm volatile("mov.u32 %0, %smid;" : "=r"(smid));
    unsigned long long* d = g_cta_trace + 4ull * blockIdx.x;
    d[0] = t0; d[1] = trace_now(); d[2] = smid; d[3] = (unsigned long long)n;
  }
}
#define B2R_TRACE_BEGIN() const unsigned long long trace_t0 = trace_now()
#define B2R_TRACE_END(n) trace_end(trace_t0, (n))
#else
#define B2R_TRACE_BEGIN()
#define B2R_TRACE_END(n)
#endif

// Kernel launch with an execution priority (a launch attribute; captured into CUDA-graph kernel nodes as well).
// When several frames are in flight on different streams (plan.py FrameLanes) the block scheduler hands freed SM
// resources to pending CTAs in launch order, so a 1-CTA scan or a few-hundred-CTA projection of frame B would wait
// behind the thousands of composite CTAs frame A still has queued (tools/lanes_timeline.py shows such gaps).  The
// short, latency-bound kernels of the chain therefore run at high priority and the two composites at the default.
int launch_priority(bool high);
int device_sm_count();
template <typename... KArgs, typename... Args>
inline void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool high,
                     Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributePriority;
  attr[0].val.priority = launch_priority(high);
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

extern int g_last_cuda_error;
inline int check_launch() {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    g_last_cuda_error = (int)e;
    return B2R_E_CUDA;
  }
  return B2R_OK;
}

}  // namespace b2r
