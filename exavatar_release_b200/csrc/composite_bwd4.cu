// composite_bwd4.cu -- K5: backward alpha-composite (App. A.4), one work item per (quarter tile, 512-entry segment).
//
// Replaces the reference rasteriser's backward render kernel (SURVEY.md section 2.3 row 8).  The per-hit machinery is
// round 1's composite_bwd3 (64-thread CTA per 8x8 quarter tile, cp.async staging, 8x4 sub-tile cull with a compacted
// survivor queue, back to front; phase A lanes = pixels replays the blend state and writes (q, w) per pixel into a warp
// queue; phase B lanes = splats sums nine moments in registers and leaves with three 16-byte vector reductions per
// (splat, warp); scalar colour recurrence; one MUFU.RCP for 1/(1-alpha)).  What changed: the list is no longer walked
// by one CTA from its last contributor to its first.  The backward recurrences can be ENTERED at any list position p
// once the state there is known -- T(p), and the colour composited behind p,  (C_final - C_prefix(p)) / T(p) -- and
// the forward (composite_fwd4.cu) stores exactly that, per pixel, at every 512-entry cut of a list.  So every
// (quarter tile, segment) is an independent CTA: the longest serial chain drops from ~1200 hits to <= ~170, the eight
// CTAs that used to run alone for the last third of the kernel disappear, and no combine pass is needed because the
// per-Gaussian sums are accumulated atomically anyway.  Error of the subtraction: <= 1 ulp of C (~1e-7) entering
// dL/dalpha_k scaled by T_k / (T(p) (1 - alpha_k)) <= 100 -- inside the 1e-4 tolerance, measured in tests/.
// Without a checkpoint buffer in the workspace every list is a single segment (the round-1 behaviour).
// Conventions (App. A.6): the 0.99 clamp is ignored on the way back; masks are constants.
#include "common.cuh"

namespace b2r {

constexpr int B4_THREADS = 64;
constexpr int B4_BATCH = 64;
#ifndef B4_QUEUE_DEPTH
#define B4_QUEUE_DEPTH 16
#endif
#ifndef B4_MIN_BLOCKS
#define B4_MIN_BLOCKS 10
#endif
constexpr int B4_QUEUE = B4_QUEUE_DEPTH;  // queued splats per warp before phase B runs (32 / B4_QUEUE lanes share a splat)

struct B4Stage {
  float4 a[B4_BATCH];  // px, py, A2, B2
  float4 b[B4_BATCH];  // C2, opacity, depth, thr2
  float4 c[B4_BATCH];  // r, g, b, id | clamp bits << 29
};
// splats replayed per trip of the hit loop (their evaluations overlap).  2 rather than 4 or 8: measured on an H100,
// the C2 backward composite takes 82 / 100 / 170 us with groups of 2 / 4 / 8, although a group of 2 issues the most
// instructions per splat (DESIGN.md section 3.3)
constexpr int B4_GROUP = 2;
// Circular survivor queue.  A replayed survivor keeps its slot until phase B has read its record from there, so the queue
// holds < B4_QUEUE replayed-but-not-drained survivors, < B4_GROUP left over and 32 new per chunk.  A multiple of B4_GROUP.
constexpr int B4_CQ = 32 + B4_QUEUE;
struct B4Compact {            // warp-private circular queue of cull survivors, back to front
  float4 r[3][B4_CQ];         // [0] px,py,A2,B2  [1] C2,opacity,depth,list position (int bits)  [2] r,g,b,id bits
};
static_assert(B4_QUEUE % B4_GROUP == 0, "phase B runs when whole groups fill the transposition queue");
static_assert(B4_CQ % B4_GROUP == 0, "a group never straddles the wrap of the survivor queue");

__device__ __forceinline__ float rcp_approx4(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct B4Smem {
  B4Stage stage[2];
  B4Compact compact[2];
  float2 tb[2][B4_QUEUE][33];  // [warp][queued splat][pixel], padded rows: conflict-free both ways
  float4 gpix[2][32];          // per pixel of the warp: g_r, g_g, g_b, g_depth
  int warp_max_s[2];
};

// one work item: quarter `quad` of segment `seg` of the tile at position `t_pos` of cx.tile_order
template <bool HAS_DA>
__device__ __forceinline__ void bwd4_item(const B2RScene& sc, const Ctx& cx, const B2RBackwardArgs& args,
                                          float* __restrict__ gacc, B4Smem& sm, const int t_pos, const int seg,
                                          const int quad, const int n_multi) {
  B4Stage (&stage)[2] = sm.stage;
  B4Compact (&compact)[2] = sm.compact;
  float2 (&tb)[2][B4_QUEUE][33] = sm.tb;
  float4 (&gpix)[2][32] = sm.gpix;
  int (&warp_max_s)[2] = sm.warp_max_s;
  B2R_TRACE_BEGIN();
  const bool multi = t_pos < n_multi;
  const int tile = (int)cx.tile_order[t_pos];
  // a view whose own Gaussians (index >= skip_below) do not occur in this tile has nothing to accumulate here: in
  // ExAvatar's cat(scene.detach(), human) renders that is every tile the human does not touch
  if (cx.skip_below && cx.tile_maxid[tile] < cx.skip_below) return;
  const int tx = tile % cx.gx, ty = tile / cx.gx;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int W = sc.width, H = sc.height;
  const int wx0 = tx * TILE + (quad & 1) * 8, wy0 = ty * TILE + (quad >> 1) * 8 + warp * 4;
  if (wx0 >= W || ty * TILE + (quad >> 1) * 8 >= H) return;  // quarter entirely outside the image (CTA-uniform)
  const int px = wx0 + (lane & 7), py = wy0 + (lane >> 3);
  const bool inside = px < W && py < H;
  const float pxf = (float)px, pyf = (float)py;
  const float rx0 = (float)wx0, ry0 = (float)wy0;
  const float rx1 = fminf((float)(wx0 + 7), (float)(W - 1)), ry1 = fminf((float)(wy0 + 3), (float)(H - 1));
  const size_t N = (size_t)W * H;
  const size_t pix = (size_t)py * W + px;

  const uint2 range = cx.ranges[tile];
  const int n = (int)(range.y - range.x);
  const int lo = multi ? seg * SEG : 0;               // this item replays list positions [lo, hi)
  const int hi = multi ? min(n, lo + SEG) : n;
  const uint32_t* ids = cx.dup_ids + range.x + lo;

  const int my_n = inside ? (int)cx.n_contrib[pix] : 0;  // 1-based position of the pixel's last applied entry
  const int my_hi = min(my_n, hi) - lo;                 // entries of this segment the pixel reaches (<= 0: none)
  const bool cont = my_n > hi;                          // the pixel's walk started behind this segment
  const float T_final = inside ? cx.final_T[pix] : 0.f;
  const float g_r = inside ? __ldg(args.dL_dcolor + pix) : 0.f;
  const float g_g = inside ? __ldg(args.dL_dcolor + N + pix) : 0.f;
  const float g_b = inside ? __ldg(args.dL_dcolor + 2 * N + pix) : 0.f;
  float g_d = 0.f, g_a = 0.f;
  if (HAS_DA && inside) {
    if (args.dL_ddepth) g_d = __ldg(args.dL_ddepth + pix);
    if (args.dL_dalpha) g_a = __ldg(args.dL_dalpha + pix);
  }
  const float* bgp = cx.bg ? cx.bg : sc.bg;
  const float Tfb = T_final * (__ldg(bgp) * g_r + __ldg(bgp + 1) * g_g + __ldg(bgp + 2) * g_b);
  gpix[warp][lane] = make_float4(g_r, g_g, g_b, g_d);

  const int warp_n = __reduce_max_sync(0xffffffffu, max(my_hi, 0));
  if (lane == 0) warp_max_s[warp] = warp_n;
  __syncthreads();
  const int nmax = max(warp_max_s[0], warp_max_s[1]);
  if (nmax == 0) {
    B2R_TRACE_END(0);
    return;
  }
  const int nb = (nmax + B4_BATCH - 1) / B4_BATCH;

  // ---- blend state at the back end of the segment ----
  // A pixel whose last contributor lies in this segment starts from its final state (nothing behind it).  A pixel that
  // continues behind the segment enters at the cut `hi`: T(hi) and the prefix sums there come from the forward's
  // checkpoint record, the state behind the cut is  (final sums - prefix sums) / T(hi)  dotted with the pixel's gradient.
  float T = T_final, B = 0.f;
  if (cont) {  // only possible in a multi-segment tile, whose records exist
    const int pit = (py - ty * TILE) * TILE + (px - tx * TILE);
    const int nrec = (n + SEG - 1) / SEG;
    const float* rec = cx.ckpt + (size_t)(cx.seg_start[t_pos] + seg) * CK_REC_FLOATS;
    const float* fin = cx.ckpt + (size_t)(cx.seg_start[t_pos] + nrec - 1) * CK_REC_FLOATS;
    const float4 c = __ldg(reinterpret_cast<const float4*>(rec) + pit);
    const float4 f = __ldg(reinterpret_cast<const float4*>(fin) + pit);
    float num = (f.y - c.y) * g_r + (f.z - c.z) * g_g + (f.w - c.w) * g_b;
    if (HAS_DA) {
      const float2 c2 = __ldg(reinterpret_cast<const float2*>(rec + CK_PLANE0) + pit);
      const float2 f2 = __ldg(reinterpret_cast<const float2*>(fin + CK_PLANE0) + pit);
      num += (f2.x - c2.x) * g_d + (f2.y - c2.y) * g_a;
    }
    T = c.x;
    B = __fdividef(num, c.x);
  }
  float la = 0.f, olm = 1.f, lv = 0.f;
  int qpos = 0, qbase = 0;  // warp-uniform: queued splats in the transposition queue, survivor-queue slot of the first
  B4Compact& cw = compact[warp];
  const unsigned lanes_above = 0xfffffffeu << lane;  // lanes with a higher index (= later list entries)
  const uint32_t first_grad = args.first_row;        // Gaussians below it are detached in this view: no accumulation

  // phase B: 32 / B4_QUEUE lanes share a queued splat, each walks its pixel rows; combined with shuffles.  The splat's
  // record is read from its survivor-queue slot, which phase A left in place.
  auto drain = [&](const int count) {
    constexpr int SHARE = 32 / B4_QUEUE;  // lanes per queued splat
    constexpr int ROWS = 4 / SHARE;       // pixel rows (of eight) per lane
    static_assert(B4_QUEUE == 8 || B4_QUEUE == 16 || B4_QUEUE == 32, "queue depth");
    __syncwarp();
    const int h = lane & (B4_QUEUE - 1), part = lane / B4_QUEUE;
    const bool live = h < count;
    float Sx = 0.f, Sy = 0.f, Sxx = 0.f, Sxy = 0.f, Syy = 0.f, Sq = 0.f, Sr = 0.f, Sg = 0.f, Sb = 0.f, Sd = 0.f;
    float4 m0 = make_float4(0.f, 0.f, 0.f, 0.f), m1 = make_float4(0.f, 1.f, 0.f, 0.f);
    if (live) {
      const int slot = qbase + h < B4_CQ ? qbase + h : qbase + h - B4_CQ;
      m0 = cw.r[0][slot];
      const float4 r1 = cw.r[1][slot];
      m1 = make_float4(r1.x, r1.y, cw.r[2][slot].w, 0.f);
      // ROWS pixel rows of eight per lane.  Within a row dy is constant, so only q, q dx and q dx^2 are summed per
      // pixel; the dy moments are formed once per row from the row sums.
      const float mx = m0.x - rx0, my = m0.y - ry0;
      float dxs[8];
#pragma unroll
      for (int c = 0; c < 8; c++) dxs[c] = mx - (float)c;
#pragma unroll
      for (int r = 0; r < ROWS; r++) {
        const float dy = my - (float)(part * ROWS + r);
        float Rq = 0.f, Rx = 0.f, Rxx = 0.f;
#pragma unroll
        for (int c = 0; c < 8; c++) {
          const int p = (part * ROWS + r) * 8 + c;
          const float2 t = tb[warp][h][p];
          const float4 g = gpix[warp][p];
          const float hx = t.x * dxs[c];
          Rq += t.x;
          Rx += hx;
          Rxx = fmaf(hx, dxs[c], Rxx);
          Sr = fmaf(t.y, g.x, Sr);
          Sg = fmaf(t.y, g.y, Sg);
          Sb = fmaf(t.y, g.z, Sb);
          if (HAS_DA) Sd = fmaf(t.y, g.w, Sd);
        }
        const float hy = Rq * dy;
        Sq += Rq;
        Sx += Rx;
        Sxx += Rxx;
        Sy += hy;
        Syy = fmaf(hy, dy, Syy);
        Sxy = fmaf(Rx, dy, Sxy);
      }
    }
#pragma unroll
    for (int o = B4_QUEUE; o < 32; o <<= 1) {  // combine the lanes that share a splat
      Sx += __shfl_xor_sync(0xffffffffu, Sx, o);
      Sy += __shfl_xor_sync(0xffffffffu, Sy, o);
      Sxx += __shfl_xor_sync(0xffffffffu, Sxx, o);
      Sxy += __shfl_xor_sync(0xffffffffu, Sxy, o);
      Syy += __shfl_xor_sync(0xffffffffu, Syy, o);
      Sq += __shfl_xor_sync(0xffffffffu, Sq, o);
      Sr += __shfl_xor_sync(0xffffffffu, Sr, o);
      Sg += __shfl_xor_sync(0xffffffffu, Sg, o);
      Sb += __shfl_xor_sync(0xffffffffu, Sb, o);
      if (HAS_DA) Sd += __shfl_xor_sync(0xffffffffu, Sd, o);
    }
    const uint32_t gid = __float_as_uint(m1.z) & 0x1fffffffu;
    if (live && part == 0 && gid >= first_grad) {
      // accumulator row convention of project_bwd.cu
      float* dst = gacc + (size_t)gid * 12;
      red_add_v4(dst, 2.f * m0.z * Sx + m0.w * Sy, 2.f * m1.x * Sy + m0.w * Sx, Sxx, Sxy);
      red_add_v4(dst + 4, Syy, __fdividef(Sq, m1.y), Sd, 0.f);
      red_add_v4(dst + 8, Sr, Sg, Sb, 0.f);
    }
    __syncwarp();
  };

  const uint32_t id_begin = cx.id_begin, id_span = cx.id_span;
  // list entry -> record is two dependent global loads: the entry of the batch after next is fetched into a register while
  // the current batch is replayed (see composite_fwd4.cu)
  uint32_t next_id = 0u;
  auto prefetch = [&](int b) {
    const int idx = b * B4_BATCH + threadIdx.x;
    next_id = idx < nmax ? __ldg(ids + idx) : 0u;
  };
  auto issue = [&](int b) {  // consumes next_id (= the entry of batch b)
    B4Stage& s = stage[b & 1];
    const int idx = b * B4_BATCH + threadIdx.x;
    if (idx < nmax) {
      const uint32_t id = next_id;
      if (id - id_begin < id_span) {
        const float4* src = reinterpret_cast<const float4*>(cx.geom + id);
        cp_async16(&s.a[threadIdx.x], src);
        cp_async16(&s.b[threadIdx.x], src + 1);
        cp_async16(&s.c[threadIdx.x], src + 2);
      } else {  // not part of this view: can never pass the sub-tile cull
        s.a[threadIdx.x] = make_float4(0.f, 0.f, -1.f, 0.f);
        s.b[threadIdx.x] = make_float4(-1.f, 0.f, 0.f, INFINITY);
      }
    }
    cp_async_commit();
  };

  // One trip = B4_GROUP queued survivors.  Stage 1 (independent per splat, so the four overlap): exponent, alpha,
  // validity and the scalar "colour" v = c . g.  Stage 2: the short serial recurrences (T, B) and the two numbers per
  // pixel that go to the transposition queue.  No branches inside a trip; a splat no pixel of the warp accepts still
  // takes a queue slot (all-zero column).  The splats' records stay in their survivor-queue slots for phase B.
  auto replay_group = [&](const int k) {
    float araw[B4_GROUP], vv[B4_GROUP];
    bool valid[B4_GROUP];
#pragma unroll
    for (int u = 0; u < B4_GROUP; u++) {
      const float4 a = cw.r[0][k + u], bb = cw.r[1][k + u], col = cw.r[2][k + u];
      const float dx = a.x - pxf, dy = a.y - pyf;
      const float p2 = a.z * dx * dx + bb.x * dy * dy + a.w * dx * dy;
      araw[u] = bb.y * ex2_approx(p2);
      valid[u] = (__float_as_int(bb.w) < my_hi) && (p2 <= 0.f) && (araw[u] >= K_ALPHA_MIN);
      float v = fmaf(col.z, g_b, fmaf(col.y, g_g, col.x * g_r));
      if (HAS_DA) v += fmaf(bb.z, g_d, g_a);
      vv[u] = v;
    }
    if (qpos == 0) qbase = k;
#pragma unroll
    for (int u = 0; u < B4_GROUP; u++) {
      const float ae = valid[u] ? fminf(K_ALPHA_MAX, araw[u]) : 0.f;  // a skipped splat enters with alpha = 0 (identity)
      const float om = 1.f - ae;
      const float rcp = rcp_approx4(om);
      const float Tn = T * rcp;
      B = fmaf(la, lv, olm * B);
      const float dLda = fmaf(vv[u] - B, Tn, -Tfb * rcp);
      la = ae; olm = om; lv = vv[u]; T = Tn;
      tb[warp][qpos + u][lane] = make_float2(valid[u] ? araw[u] * dLda : 0.f, ae * Tn);  // q = dL/dG * G (clamp ignored), w
    }
    qpos += B4_GROUP;
    if (qpos == B4_QUEUE) {
      drain(B4_QUEUE);
      qpos = 0;
    }
  };

  int head = 0, fill = 0;  // warp-uniform: slot of the oldest queued survivor (a multiple of B4_GROUP); survivors queued
  prefetch(nb - 1);
  issue(nb - 1);
  if (nb > 1) prefetch(nb - 2);
  for (int b = nb - 1; b >= 0; b--) {
    cp_async_wait<0>();
    __syncthreads();  // batch b staged; both warps are done with batch b+1
    if (b > 0) {
      issue(b - 1);
      if (b > 1) prefetch(b - 2);
    }
    const int count = min(B4_BATCH, nmax - b * B4_BATCH);
    const B4Stage& s = stage[b & 1];
    if (warp_n <= b * B4_BATCH) continue;  // warp-uniform: none of my pixels reaches this batch
    for (int c0 = ((count - 1) >> 5) << 5; c0 >= 0; c0 -= 32) {
      const int idx = c0 + lane;
      const int pos = b * B4_BATCH + idx;  // position inside the segment
      bool hit = false;
      float4 a, bb;
      if (idx < count && pos < warp_n) {
        a = s.a[idx];
        bb = s.b[idx];
        hit = !(region_max_p2(a.x, a.y, a.z, a.w, bb.x, rx0, ry0, rx1, ry1) < bb.w);
      }
      const unsigned mask = __ballot_sync(0xffffffffu, hit);
      if (mask == 0u) continue;
      if (hit) {  // back to front: the highest surviving list position is queued first
        int slot = head + fill + __popc(mask & lanes_above);
        slot -= slot >= B4_CQ ? B4_CQ : 0;
        cw.r[0][slot] = a;
        cw.r[1][slot] = make_float4(bb.x, bb.y, bb.z, __int_as_float(pos));
        cw.r[2][slot] = s.c[idx];
      }
      fill += __popc(mask);
      __syncwarp();
      for (; fill >= B4_GROUP; fill -= B4_GROUP) {  // what does not fill a group stays queued where it is
        replay_group(head);
        head = head + B4_GROUP == B4_CQ ? 0 : head + B4_GROUP;
      }
      __syncwarp();  // queue reads before the next append
    }
  }
  if (fill > 0) {  // flush: pad the last group with splats that can never be valid (list position INT_MAX); their
                   // opacity is 1 because phase B divides by it
    if (lane >= fill && lane < B4_GROUP) {  // head is a multiple of B4_GROUP: the group does not wrap
      cw.r[0][head + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
      cw.r[1][head + lane] = make_float4(0.f, 1.f, 0.f, __int_as_float(0x7fffffff));
      cw.r[2][head + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncwarp();
    replay_group(head);
  }
  if (qpos > 0) drain(qpos);
  if (threadIdx.x == 0) atomicAdd(reinterpret_cast<unsigned long long*>(&cx.status->consumed_bwd), (unsigned long long)nmax);
  B2R_TRACE_END(nmax);
}

// The number of work items -- 4 quarter tiles x (segments of the multi-segment tiles + one per remaining tile) -- is only
// known on the device, so the grid is a fixed number of CTAs that stride over the items (heaviest first: the item order
// follows cx.tile_order).  A grid sized for the host-side worst case (capacity / SEG segments) would be mostly CTAs that
// read two counters and exit -- most of them with a generously sized workspace.
template <bool HAS_DA>
__global__ void __launch_bounds__(B4_THREADS, B4_MIN_BLOCKS) composite_bwd4_kernel(const B2RScene sc, const Ctx cx,
                                                                    const B2RBackwardArgs args, float* __restrict__ gacc) {
  __shared__ B4Smem sm;
  // the two counters are re-read per item rather than kept live across the item loop: held in registers they spill
  for (int item = blockIdx.x;; item += gridDim.x) {
    const int n_multi = cx.ckpt ? (int)cx.classes[CLS_N_MULTI] : 0;
    const int total_segs = cx.ckpt ? (int)cx.classes[CLS_TOTAL_SEGS] : 0;
    if (item >= 4 * (total_segs + (cx.tiles - n_multi))) break;
    const int s_item = item >> 2;
    int t_pos, seg;
    if (s_item < total_segs) {
      const uint2 e = cx.seg_table[s_item];
      t_pos = (int)e.x;
      seg = (int)e.y;
    } else {
      t_pos = n_multi + (s_item - total_segs);
      seg = 0;
    }
    bwd4_item<HAS_DA>(sc, cx, args, gacc, sm, t_pos, seg, item & 3, n_multi);
    __syncthreads();  // shared memory is reused by the next item
  }
}

int launch_composite_bwd(const B2RScene& sc, const Ctx& cx, const B2RBackwardArgs& a, float* gacc, cudaStream_t st) {
  if (!(a.flags & B2R_BWD_SCRATCH_ZEROED)) cudaMemsetAsync(gacc, 0, (size_t)(sc.P > 0 ? sc.P : 1) * 12 * sizeof(float), st);
  // host-side bound on the item count (every segment beyond a tile's first covers SEG list entries), capped at a few
  // waves of resident CTAs: the kernel strides over the items
  const uint64_t extra = cx.ckpt ? cx.dup_capacity / SEG : 0;
  const uint64_t bound = 4ull * ((uint64_t)cx.tiles + extra);
  const uint64_t cap = (uint64_t)device_sm_count() * B4_MIN_BLOCKS * 4;
  const unsigned grid = (unsigned)(bound < cap ? bound : cap);
  ProfScope p(K_COMPOSITE_BWD, st);
  if (a.dL_ddepth || a.dL_dalpha)
    launch_k(composite_bwd4_kernel<true>, grid, B4_THREADS, 0, st, false, sc, cx, a, gacc);
  else
    launch_k(composite_bwd4_kernel<false>, grid, B4_THREADS, 0, st, false, sc, cx, a, gacc);
  return check_launch();
}

}  // namespace b2r

#ifdef B2R_CTA_TRACE
extern "C" int b2r_debug_trace_bwd(unsigned long long* buf) {
  return (int)cudaMemcpyToSymbol(b2r::g_cta_trace, &buf, sizeof(buf));
}
#endif
