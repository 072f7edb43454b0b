// composite_fwd4.cu -- K4: forward alpha-composite (App. A.3) with blend-state checkpoints and views.
//
// Replaces the reference rasteriser's forward render kernel for ExAvatar's render path
// (avatar/common/nets/module.py:632 -> render_img, render_depthmap, render_mask).
//
// Design.  The kernel is issue- and latency-bound, not HBM-bound (SURVEY.md section 7.2; DESIGN.md section 5), so
// the structure removes per-pixel work and idle SMs rather than bytes:
//   * work unit = one 8x8 quarter of a 16x16 tile, one 64-thread CTA (2 warps, each an 8x4 pixel rect), launched
//     longest-list-first (cx.tile_order).  A quarter retires as soon as its own 64 pixels are saturated, and only two
//     warps meet at the per-batch barrier;
//   * the tile's depth-sorted id list is streamed in batches of 128; each thread gathers two 48-byte splat records
//     (three 16-byte cp.async = LDGSTS each, no register staging) into a double-buffered shared-memory stage while the
//     previous batch is composited;
//   * for every 32 staged splats a warp runs ONE lane-parallel test "can this splat reach alpha >= 1/255 anywhere in my
//     8x4 rect" (region_max_p2), ballots, and the survivors are appended to a warp-private queue that the hit loop
//     walks four splats per trip (their exponent evaluations overlap; only the short T recurrence is serial);
//   * CHECKPOINTS: at every 512-entry cut of a list the per-pixel blend state (T, C, depth sum, alpha sum) is stored
//     (when the workspace has room: B2RWorkspace.checkpoints).  Alpha compositing can be re-entered at any list position
//     once the state there is known, which is what lets composite_bwd4.cu replay every 512-entry segment as an
//     independent work item instead of walking 2000 entries on one warp;
//   * VIEWS (B2RView): Gaussians outside the view's index range are dropped when a batch is staged (no gather for
//     them); tiles whose list holds nothing of the view's own (tile_maxid < skip_below) are skipped altogether.
// Not done here: splitting the long lists of the forward over eight warps per pixel rect (local blends from T = 1, a
// prefix walk over the segments' transmittance products, replay of the one segment in which a pixel stops).  It is exact
// and shortens the kernel ALONE on long-list workloads, but spends more warp-time (speculative segments, replays, CTA
// barriers), which costs throughput with other kernels in flight -- and that is how the training step runs.
#include "common.cuh"

namespace b2r {

#ifndef FL_BATCH_N
#define FL_BATCH_N 128  // entries staged per batch (tuning hook)
#endif
constexpr int F4_BATCH = 2 * FL_BATCH_N;  // capacity of the two-half staging buffer
#ifndef F4_GROUP_N
#define F4_GROUP_N 4
#endif
constexpr int F4_GROUP = F4_GROUP_N;  // splats blended per trip of the hit loop (their evaluations overlap: ILP 4)
constexpr int F4_CQ = 32 + F4_GROUP;  // circular survivor queue: < F4_GROUP left over + 32 new per chunk; a multiple of
                                      // F4_GROUP, so a group never straddles the wrap

struct F4Stage {
  float4 a[F4_BATCH];  // px, py, A2, B2
  float4 b[F4_BATCH];  // C2, opacity, depth, thr2
  float4 c[F4_BATCH];  // r, g, b, id bits
};
struct F4Queue {          // warp-private circular queue of cull survivors in list order
  float4 r[3][F4_CQ];     // [0] px,py,A2,B2  [1] C2,opacity,depth,1-based list position (int bits)  [2] r,g,b,-
};
// Per-pixel blend state.  T is the RUNNING PRODUCT of (1 - alpha) over every splat the pixel accepted or was stopped by:
// it is multiplied unconditionally, so the only serial dependency between consecutive splats is one FMUL (round 1 carried
// "finished" in the sign of T, which put a compare, a predicate combine and a select on that chain: ~18 cycles per splat
// for a warp that runs alone).  A pixel is alive while T >= 1e-4; the first accepted splat that takes the product below
// 1e-4 finishes the pixel without being applied (App. A.3), and because the product can only shrink, nothing after it
// passes `T_next >= 1e-4` again.  Tf trails T: the transmittance after the last APPLIED splat = App. A.3's final_T.
struct Blend {
  float T, Tf, Cr, Cg, Cb, Dp, Aa;
  uint32_t last;
};
__device__ __forceinline__ bool alive(const Blend& s) { return s.T >= K_T_MIN; }

__device__ __forceinline__ void store4v(float* base, bool vec_ok, int lane, float v, bool inside) {
  if (vec_ok) {
    const float v1 = __shfl_down_sync(0xffffffffu, v, 1);
    const float v2 = __shfl_down_sync(0xffffffffu, v, 2);
    const float v3 = __shfl_down_sync(0xffffffffu, v, 3);
    if ((lane & 3) == 0 && inside) *reinterpret_cast<float4*>(base) = make_float4(v, v1, v2, v3);
  } else if (inside) {
    *base = v;
  }
}

// One trip = F4_GROUP queued splats.  Their exponent evaluations are independent of the blend state and of each other,
// so they overlap (shared loads, FMA chain, MUFU); only the short T recurrence that follows is serial.  Branch-free
// (App. A.3): a splat is skipped unless the pixel is alive, power <= 0 and alpha >= 1/255; a splat that would drop the
// transmittance below 1e-4 finishes the pixel WITHOUT being applied.
__device__ __forceinline__ void blend_group4(const F4Queue& cw, const int k, Blend& s, const float pxf, const float pyf) {
  float al[F4_GROUP], om[F4_GROUP];
  bool ok[F4_GROUP];
  float4 col[F4_GROUP];
  float dep[F4_GROUP];
  uint32_t pos[F4_GROUP];
#pragma unroll
  for (int u = 0; u < F4_GROUP; u++) {
    const float4 a = cw.r[0][k + u], bb = cw.r[1][k + u];
    col[u] = cw.r[2][k + u];
    const float dx = a.x - pxf, dy = a.y - pyf;
    const float p2 = a.z * dx * dx + bb.x * dy * dy + a.w * dx * dy;
    const float ar = bb.y * ex2_approx(p2);
    al[u] = fminf(K_ALPHA_MAX, ar);
    ok[u] = (ar >= K_ALPHA_MIN) & (p2 <= 0.f);
    om[u] = ok[u] ? 1.f - al[u] : 1.f;  // a splat the pixel skips leaves the product alone
    dep[u] = bb.z;
    pos[u] = (uint32_t)__float_as_int(bb.w);
  }
#pragma unroll
  for (int u = 0; u < F4_GROUP; u++) {
    const float w = al[u] * s.T;
    const float Tn = s.T * om[u];              // the whole serial chain: one multiply per splat
    const bool use = ok[u] & (Tn >= K_T_MIN);  // false for ever once the product has dropped below 1e-4
    s.Cr = use ? fmaf(col[u].x, w, s.Cr) : s.Cr;  // predicated accumulates: a skipped splat must not touch the sums at all
    s.Cg = use ? fmaf(col[u].y, w, s.Cg) : s.Cg;
    s.Cb = use ? fmaf(col[u].z, w, s.Cb) : s.Cb;
    s.Dp = use ? fmaf(dep[u], w, s.Dp) : s.Dp;
    s.Aa = use ? s.Aa + w : s.Aa;
    s.last = use ? pos[u] : s.last;
    s.Tf = use ? Tn : s.Tf;
    s.T = Tn;
  }
}

// 32 staged entries (one per lane; `in_range` false past the end): sub-tile cull against the warp's 8x4 rect, survivors
// appended to the circular queue in list order, whole groups blended.  `head` = slot of the oldest queued survivor (a
// multiple of F4_GROUP), `fill` = survivors queued; what does not fill a group simply stays where it is (round 1 moved
// the leftovers to the front after every chunk: 19 instructions and two warp barriers per chunk).  `pos1` = 1-based list
// position of this lane's entry.
__device__ __forceinline__ void cull_and_blend(const F4Stage& st, const int idx, const bool in_range, const int pos1,
                                               F4Queue& cw, int& head, int& fill, Blend& s, const float rx0, const float ry0,
                                               const float rx1, const float ry1, const float pxf, const float pyf) {
  const int lane = threadIdx.x & 31;
  bool hit = false;
  float4 a, bb;
  if (in_range) {
    a = st.a[idx];
    bb = st.b[idx];
    hit = !(region_max_p2(a.x, a.y, a.z, a.w, bb.x, rx0, ry0, rx1, ry1) < bb.w);
  }
  const unsigned mask = __ballot_sync(0xffffffffu, hit);
  if (mask == 0u) return;
  if (hit) {
    int slot = head + fill + __popc(mask & ((1u << lane) - 1u));
    slot -= slot >= F4_CQ ? F4_CQ : 0;
    cw.r[0][slot] = a;
    cw.r[1][slot] = make_float4(bb.x, bb.y, bb.z, __int_as_float(pos1));
    cw.r[2][slot] = st.c[idx];
  }
  fill += __popc(mask);
  __syncwarp();
  for (; fill >= F4_GROUP; fill -= F4_GROUP) {
    blend_group4(cw, head, s, pxf, pyf);
    head = head + F4_GROUP == F4_CQ ? 0 : head + F4_GROUP;
  }
  __syncwarp();  // orders the queue reads before the next append
}

// blends what is still queued: the last group is padded with splats of opacity 0 (alpha 0 < 1/255 => skipped)
__device__ __forceinline__ void flush_queue(F4Queue& cw, int& head, int& fill, Blend& s, const float pxf, const float pyf) {
  if (fill > 0) {
    const int lane = threadIdx.x & 31;
    if (lane >= fill && lane < F4_GROUP) {  // head is a multiple of F4_GROUP: the group does not wrap
      cw.r[0][head + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
      cw.r[1][head + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
      cw.r[2][head + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncwarp();
    blend_group4(cw, head, s, pxf, pyf);
    __syncwarp();
    head = head + F4_GROUP == F4_CQ ? 0 : head + F4_GROUP;
    fill = 0;
  }
}

__device__ __forceinline__ void store_checkpoint(float* rec, const int pix_in_tile, const Blend& s) {
  reinterpret_cast<float4*>(rec)[pix_in_tile] = make_float4(s.Tf, s.Cr, s.Cg, s.Cb);
  reinterpret_cast<float2*>(rec + CK_PLANE0)[pix_in_tile] = make_float2(s.Dp, s.Aa);
}

__device__ __forceinline__ void write_outputs(const B2RScene& sc, const Ctx& cx, const B2RForwardOutputs& out, const int vec_ok,
                                              const Blend& S, const int px, const int py, const bool inside, const int lane) {
  const float T = S.Tf;
  const size_t N = (size_t)sc.width * sc.height;
  const size_t pix = (size_t)py * sc.width + px;
  const float* bgp = cx.bg ? cx.bg : sc.bg;
  const float bg0 = __ldg(bgp), bg1 = __ldg(bgp + 1), bg2 = __ldg(bgp + 2);
  const bool v = vec_ok != 0;
  store4v(out.color + pix, v, lane, fmaf(T, bg0, S.Cr), inside);
  store4v(out.color + N + pix, v, lane, fmaf(T, bg1, S.Cg), inside);
  store4v(out.color + 2 * N + pix, v, lane, fmaf(T, bg2, S.Cb), inside);
  store4v(out.depth + pix, v, lane, S.Dp, inside);
  store4v(out.alpha + pix, v, lane, S.Aa, inside);
  store4v(cx.final_T + pix, v, lane, T, inside);
  store4v(reinterpret_cast<float*>(cx.n_contrib) + pix, v, lane, __uint_as_float(S.last), inside);
}

constexpr int FL_THREADS = 64;
constexpr int FL_BATCH = FL_BATCH_N;
static_assert(SEG % FL_BATCH == 0, "checkpoint cuts fall on batch boundaries");

#ifndef F4_MIN_BLOCKS
#define F4_MIN_BLOCKS 14  // = the shared-memory limit (15.7 KB per CTA): keeps the kernel at 72 registers; 16 forces 64 (measured)
#endif
__global__ void __launch_bounds__(FL_THREADS, F4_MIN_BLOCKS) composite_fwd_kernel(const B2RScene sc, const Ctx cx,
                                                                          const B2RForwardOutputs out, const int vec_ok) {
  __shared__ F4Stage stage_raw;          // used as two 128-entry halves: [0,128) and [128,256) of every array
  __shared__ F4Queue queue[2];
  B2R_TRACE_BEGIN();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int W = sc.width, H = sc.height;
  const int t_pos = blockIdx.x >> 2;
  const int tile = (int)cx.tile_order[t_pos];
  if (cx.skip_below && cx.tile_maxid[tile] < cx.skip_below) return;  // nothing of this view's own here (B2RView.skip_below)
  const int quad = blockIdx.x & 3;
  const int tx = tile % cx.gx, ty = tile / cx.gx;
  const int wx0 = tx * TILE + (quad & 1) * 8, wy0 = ty * TILE + (quad >> 1) * 8 + warp * 4;
  if (wx0 >= W || ty * TILE + (quad >> 1) * 8 >= H) return;  // quarter entirely outside the image (CTA-uniform)
  const int px = wx0 + (lane & 7), py = wy0 + (lane >> 3);
  const bool inside = px < W && py < H;
  const float pxf = (float)px, pyf = (float)py;
  const float rx0 = (float)wx0, ry0 = (float)wy0;
  const float rx1 = fminf((float)(wx0 + 7), (float)(W - 1)), ry1 = fminf((float)(wy0 + 3), (float)(H - 1));
  const int pix_in_tile = (py - ty * TILE) * TILE + (px - tx * TILE);

  const uint2 range = cx.ranges[tile];
  const int n = (int)(range.y - range.x);
  const uint32_t* ids = cx.dup_ids + range.x;
  const int nb = (n + FL_BATCH - 1) / FL_BATCH;
  const int nrec = (n + SEG - 1) / SEG;
  float* ck = nullptr;  // checkpoint records of this tile: record j = state at list position min(SEG (j+1), n)
  if (cx.ckpt && t_pos < (int)cx.classes[CLS_N_MULTI]) ck = cx.ckpt + (size_t)cx.seg_start[t_pos] * CK_REC_FLOATS;

  const uint32_t id_begin = cx.id_begin, id_span = cx.id_span;
  // The gather of a batch is two dependent global loads (list entry -> record).  The list entries of batch b+2 are
  // fetched into registers while batch b is composited, so that issue(b+1) starts its record gathers without waiting for
  // them (otherwise the gathers of a batch, and the partner warp at the batch barrier, stall on that wait).
  constexpr int FL_PER_THREAD = FL_BATCH / FL_THREADS;
  uint32_t next_id[FL_PER_THREAD];
  auto prefetch = [&](int b) {
#pragma unroll
    for (int u = 0; u < FL_PER_THREAD; u++) {
      const int idx = b * FL_BATCH + threadIdx.x + u * FL_THREADS;
      next_id[u] = idx < n ? __ldg(ids + idx) : 0u;
    }
  };
  auto issue = [&](int b) {  // consumes next_id (= the entries of batch b)
    const int half = (b & 1) * FL_BATCH;
#pragma unroll
    for (int u = 0; u < FL_PER_THREAD; u++) {
      const int slot = half + threadIdx.x + u * FL_THREADS;
      const int idx = b * FL_BATCH + threadIdx.x + u * FL_THREADS;
      if (idx < n) {
        const uint32_t id = next_id[u];
        if (id - id_begin < id_span) {
          const float4* src = reinterpret_cast<const float4*>(cx.geom + id);
          cp_async16(&stage_raw.a[slot], src);
          cp_async16(&stage_raw.b[slot], src + 1);
          cp_async16(&stage_raw.c[slot], src + 2);
        } else {  // not part of this view: a record that can never pass the sub-tile cull (thr2 = +inf)
          stage_raw.a[slot] = make_float4(0.f, 0.f, -1.f, 0.f);
          stage_raw.b[slot] = make_float4(-1.f, 0.f, 0.f, INFINITY);
        }
      }
    }
    cp_async_commit();
  };

  Blend S;
  S.T = S.Tf = inside ? 1.f : 0.f;
  S.Cr = S.Cg = S.Cb = S.Dp = S.Aa = 0.f;
  S.last = 0;
  F4Queue& cw = queue[warp];
  int head = 0, fill = 0, staged = 0;
  if (nb > 0) {
    prefetch(0);
    issue(0);
    if (nb > 1) prefetch(1);
  }
  for (int b = 0; b < nb; b++) {
    cp_async_wait<0>();
    if (__syncthreads_and(!alive(S))) break;  // batch b visible; everyone is past batch b-1
    if (b + 1 < nb) {
      issue(b + 1);
      if (b + 2 < nb) prefetch(b + 2);
    }
    const int count = min(FL_BATCH, n - b * FL_BATCH);
    staged += count;
    const int half = (b & 1) * FL_BATCH;
    bool warp_live = __any_sync(0xffffffffu, alive(S));
    for (int c0 = 0; c0 < count && warp_live; c0 += 32) {
      const int idx = c0 + lane;
      cull_and_blend(stage_raw, half + idx, idx < count, b * FL_BATCH + idx + 1, cw, head, fill, S, rx0, ry0, rx1, ry1, pxf, pyf);
      warp_live = __any_sync(0xffffffffu, alive(S));
    }
    if (ck && ((b + 1) * FL_BATCH) % SEG == 0 && b + 1 < nb) {  // a cut (multiple of SEG): the state must be exact there
      flush_queue(cw, head, fill, S, pxf, pyf);
      if (inside) store_checkpoint(ck + (size_t)((b + 1) * FL_BATCH / SEG - 1) * CK_REC_FLOATS, pix_in_tile, S);
    }
  }
  flush_queue(cw, head, fill, S, pxf, pyf);
  cp_async_wait<0>();
  if (ck && nrec >= 2 && inside) store_checkpoint(ck + (size_t)(nrec - 1) * CK_REC_FLOATS, pix_in_tile, S);
  // consumed_fwd counts list entries per TILE x 8: four quarter-CTAs each add twice what they staged
  if (threadIdx.x == 0 && staged)
    atomicAdd(reinterpret_cast<unsigned long long*>(&cx.status->consumed_fwd), 2ull * (unsigned long long)staged);
  write_outputs(sc, cx, out, vec_ok, S, px, py, inside, lane);
  B2R_TRACE_END(n);
}

int launch_composite_fwd(const B2RScene& sc, const Ctx& cx, const B2RForwardOutputs& out, cudaStream_t st) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  const int vec_ok = (sc.width % 4 == 0) && al16(out.color) && al16(out.depth) && al16(out.alpha) && al16(cx.final_T) &&
                     al16(cx.n_contrib);
  ProfScope p(K_COMPOSITE_FWD, st);
  launch_k(composite_fwd_kernel, (unsigned)(cx.tiles * 4), FL_THREADS, 0, st, false, sc, cx, out, vec_ok);
  return check_launch();
}

}  // namespace b2r

#ifdef B2R_CTA_TRACE
extern "C" int b2r_debug_trace_fwd(unsigned long long* buf) {
  return (int)cudaMemcpyToSymbol(b2r::g_cta_trace, &buf, sizeof(buf));
}
#endif
