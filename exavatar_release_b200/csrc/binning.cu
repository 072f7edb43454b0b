// binning.cu -- K2: duplicate-with-keys scattered straight into per-tile segments; K3: per-tile depth sort.
//
// Replaces the reference rasteriser's duplicateWithKeys + global 64-bit cub::DeviceRadixSort (5-6 passes over
// every duplicate in HBM) + identifyTileRanges (SURVEY.md section 2.3 rows 4-6; App. A.2).  Here every tile owns a
// contiguous segment (offsets from project.cu's tile scan), K2 drops (depth, id) pairs into it, and K3 sorts each
// segment inside one CTA's shared memory: each key crosses HBM once in and its id once out.
//
// Order contract (App. A.2): ascending view depth, ties by ascending Gaussian index.  The 64-bit sort key
// (depth_bits << 32 | id) gives exactly that for positive floats and makes the result independent of the order in
// which the scatter's atomics landed, i.e. the pipeline is deterministic.
#include <cstdlib>

#include "common.cuh"

namespace b2r {

__global__ void __launch_bounds__(256) scatter_kernel(const B2RScene sc, const Ctx cx, const int first_row) {
  const int i = first_row + blockIdx.x * blockDim.x + threadIdx.x;
  int4 aux = make_int4(0, 0, 0, 0);
  float4 g0 = make_float4(0.f, 0.f, 0.f, 0.f), g1 = g0;
  uint32_t depth_bits = 0u;
  if (i < sc.P) {
    aux = cx.aux[i];
    if (aux.z > 0) {
      const int area = ((aux.y & 0xffff) - (aux.x & 0xffff)) * ((aux.y >> 16) - (aux.x >> 16));
      depth_bits = __float_as_uint(cx.geom[i].g1.z);
      if (area > 32) {  // only these repeat the region test (warp_replay_kept_tiles)
        g0 = reinterpret_cast<const float4*>(cx.geom + i)[0];
        g1 = reinterpret_cast<const float4*>(cx.geom + i)[1];
      }
    }
  }
  const uint64_t cap = cx.dup_capacity;
  const int gx = cx.gx;
  uint32_t* cursor = cx.tile_cursor;
  uint2* keys = cx.keys;
  // The slot-claiming atomics (ATOMG with a ~700-cycle round trip; 2/3 of this kernel's stall samples in the first
  // profile) overlap: a pair is stored one claim late, when its slot number has had time to come back.
  constexpr uint32_t NONE = 0xffffffffu;
  uint32_t pend_pos = NONE, pend_depth = 0, pend_id = 0;
  warp_replay_kept_tiles(aux.z > 0, aux.x & 0xffff, aux.x >> 16, aux.y & 0xffff, aux.y >> 16, (uint32_t)aux.w, g0.x, g0.y,
                         g0.z, g0.w, g1.x, g1.w, depth_bits, (uint32_t)i, (sc.flags & B2R_FLAG_NO_TILE_CULL) != 0, sc.width,
                         sc.height, gx, cursor, [&](uint32_t p, int, uint32_t d, uint32_t id) {
                           if (pend_pos < cap) keys[pend_pos] = make_uint2(pend_depth, pend_id);  // NONE >= cap always
                           pend_pos = p; pend_depth = d; pend_id = id;
                         });
  if (pend_pos < cap) keys[pend_pos] = make_uint2(pend_depth, pend_id);
}

// K2, aggregated variant (default when the per-tile counters fit in shared memory).  Atomics from different warps to
// the same global address serialise in L2 (the hot avatar tiles receive thousands), so a CTA
// claims its slots of a tile with ONE global atomic: (1) count the CTA's pairs per tile in shared memory, (2) one
// atomicAdd per touched tile reserves a contiguous run of the tile's segment, (3) enumerate again and drop each pair
// at run base + its rank inside the CTA (shared-memory atomic).  Both enumerations replay the projection's kept masks.
__global__ void __launch_bounds__(256) scatter_agg_kernel(const B2RScene sc, const Ctx cx, const int first_row) {
  extern __shared__ uint32_t s_mem[];
  uint32_t* s_cnt = s_mem;              // [tiles] pairs of this CTA per tile, then the running rank
  uint32_t* s_base = s_mem + cx.tiles;  // [tiles] first slot of this CTA's run
  for (int t = threadIdx.x; t < cx.tiles; t += blockDim.x) s_cnt[t] = 0u;
  __syncthreads();
  const int i = first_row + blockIdx.x * blockDim.x + threadIdx.x;
  int4 aux = make_int4(0, 0, 0, 0);
  float4 g0 = make_float4(0.f, 0.f, 0.f, 0.f), g1 = g0;
  uint32_t depth_bits = 0u;
  if (i < sc.P) {
    aux = cx.aux[i];
    if (aux.z > 0) {
      const int area = ((aux.y & 0xffff) - (aux.x & 0xffff)) * ((aux.y >> 16) - (aux.x >> 16));
      depth_bits = __float_as_uint(cx.geom[i].g1.z);
      if (area > 32) {  // only these repeat the region test (warp_replay_kept_tiles)
        g0 = reinterpret_cast<const float4*>(cx.geom + i)[0];
        g1 = reinterpret_cast<const float4*>(cx.geom + i)[1];
      }
    }
  }
  const int gx = cx.gx;
  const bool no_cull = (sc.flags & B2R_FLAG_NO_TILE_CULL) != 0;
  const int x0 = aux.x & 0xffff, y0 = aux.x >> 16, x1 = aux.y & 0xffff, y1 = aux.y >> 16;
  const uint32_t kept = (uint32_t)aux.w;
  warp_replay_kept_tiles(aux.z > 0, x0, y0, x1, y1, kept, g0.x, g0.y, g0.z, g0.w, g1.x, g1.w, 0u, 0u, no_cull, sc.width,
                         sc.height, gx, s_cnt, [](uint32_t, int, uint32_t, uint32_t) {});
  __syncthreads();
  for (int t = threadIdx.x; t < cx.tiles; t += blockDim.x) {
    const uint32_t c = s_cnt[t];
    if (c) {
      s_base[t] = atomicAdd(cx.tile_cursor + t, c);
      s_cnt[t] = 0u;
    }
  }
  __syncthreads();
  const uint64_t cap = cx.dup_capacity;
  uint2* keys = cx.keys;
  warp_replay_kept_tiles(aux.z > 0, x0, y0, x1, y1, kept, g0.x, g0.y, g0.z, g0.w, g1.x, g1.w, depth_bits, (uint32_t)i,
                         no_cull, sc.width, sc.height, gx, s_cnt, [&](uint32_t rank, int t, uint32_t d, uint32_t id) {
                           const uint32_t pos = s_base[t] + rank;
                           if (pos < cap) keys[pos] = make_uint2(d, id);
                         });
}

// ---------------------------------------------------------------------------------------------------------------
// K3: per-tile sort.  Order contract (App. A.2): ascending view depth, ties by ascending Gaussian index.
//
// One CTA per tile (CTAs stride over cx.tile_order, longest list first).  Lists of <= 32 entries are rank-sorted in registers.  Longer lists use an LSD radix sort in shared memory on the 32-bit depth bits
// (positive floats order like unsigned integers) carrying a 16-bit local index:
//   * 8-bit digits; a digit position on which every key of the tile agrees is skipped (the exponent byte almost
//     always is), so most tiles need 3 passes;
//   * each warp owns a contiguous chunk; MATCH.ANY groups equal digits inside a 32-key row, so a pass is a
//     warp-private histogram (no atomics), one 256-digit scan, and a stable scatter;
//   * ids are fetched once at the end; runs of bit-identical depths (rare: cloned Gaussians) are put in id order by
//     an odd-even fix-up, which makes the result independent of the scatter's atomic arrival order.
// Lists of >= 2048 entries are sorted in chunks of SORT_CHUNK and merged (merge_chunks_kernel): no length limit.
// ---------------------------------------------------------------------------------------------------------------

// Lanes holding the same 8-bit digit (invalid lanes match nobody), from eight ballots instead of MATCH.ANY (the sort
// kernel's CTA timeline, tools/cta_trace.py, compares the two).
__device__ __forceinline__ unsigned match_digit(const uint32_t d, const bool valid) {
  unsigned peers = __ballot_sync(0xffffffffu, valid);
#pragma unroll
  for (int bit = 0; bit < 8; bit++) {
    const bool on = (d >> bit) & 1u;
    const unsigned b = __ballot_sync(0xffffffffu, on);
    peers &= on ? b : ~b;
  }
  return valid ? peers : 0u;
}

template <int CAP, int THREADS>
struct RadixSmem {
  static constexpr int W = THREADS / 32;
  static constexpr size_t bytes = (size_t)CAP * 12 + (size_t)W * 256 * 2 + 64;
};

// PAIRS = false: dst[i] = id of the i-th entry in (depth, id) order.  PAIRS = true (one chunk of a long list): the sorted
// (depth, id) pairs are written back over the chunk itself, to be merged with the other chunks by merge_chunks_kernel.
// `maxid` (global, zeroed per render) receives the largest Gaussian index of the list (Ctx::tile_maxid).
template <int CAP, int THREADS, bool PAIRS = false>
__device__ __forceinline__ void radix_sort_tile(const uint2* src, uint32_t* dst, const int n, unsigned char* smem_raw,
                                                uint32_t* maxid) {
  constexpr int W = THREADS / 32;
  constexpr int ROWS = CAP / (W * 32);  // 32-key rows of a warp's share of a full chunk
  static_assert(CAP % (W * 32) == 0, "a warp's share must be whole rows");
  uint32_t* keyA = reinterpret_cast<uint32_t*>(smem_raw);
  uint32_t* keyB = keyA + CAP;
  uint16_t* idxA = reinterpret_cast<uint16_t*>(keyB + CAP);
  uint16_t* idxB = idxA + CAP;
  uint16_t* hist = idxB + CAP;  // [W][256]
  uint32_t* misc = reinterpret_cast<uint32_t*>(hist + W * 256);  // [0] OR, [1] AND, [2..9] warp totals of the digit scan
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) { misc[0] = 0u; misc[1] = 0xffffffffu; }
  __syncthreads();
  uint32_t vor = 0u, vand = 0xffffffffu;
  for (int i = tid; i < n; i += THREADS) {
    const uint32_t k = src[i].x;
    keyA[i] = k;
    idxA[i] = (uint16_t)i;
    vor |= k;
    vand &= k;
  }
  vor = __reduce_or_sync(0xffffffffu, vor);
  vand = __reduce_and_sync(0xffffffffu, vand);
  if (lane == 0) { atomicOr(&misc[0], vor); atomicAnd(&misc[1], vand); }
  __syncthreads();
  const uint32_t differ = misc[0] ^ misc[1];

  const int chunk = (((n + W - 1) / W) + 31) & ~31;  // keys per warp, a multiple of 32
  const int c_begin = min(warp * chunk, n), c_end = min(c_begin + chunk, n);
  uint32_t* kin = keyA; uint32_t* kout = keyB;
  uint16_t* iin = idxA; uint16_t* iout = idxB;
  for (int pass = 0; pass < 4; pass++) {
    const int shift = 8 * pass;
    if (((differ >> shift) & 0xffu) == 0u) continue;  // CTA-uniform
    for (int i = tid; i < W * 256; i += THREADS) hist[i] = 0;
    __syncthreads();
    uint16_t* myhist = hist + warp * 256;
    // pass 1: warp-private digit histogram; the peer masks (lanes of the row with the same digit) are kept in registers
    // for the scatter below, which sees the same rows -- the nine ballots of match_digit are a third of a pass
    unsigned row_peers[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
      const int base = c_begin + 32 * r;
      row_peers[r] = 0u;
      if (base < c_end) {  // warp-uniform
        const int i = base + lane;
        const bool valid = i < c_end;
        const uint32_t d = valid ? ((kin[i] >> shift) & 0xffu) : (256u + lane);
        const unsigned peers = match_digit(d, valid);
        row_peers[r] = peers;
        if (valid && (peers & ((1u << lane) - 1u)) == 0u) myhist[d] = (uint16_t)(myhist[d] + __popc(peers));
        __syncwarp();
      }
    }
    __syncthreads();
    // scan: hist[w][d] <- first output slot of (digit d, warp w)
    // each of the first 256 / DPT threads owns DPT consecutive digits (DPT = 2 for the 128-thread class)
    constexpr int DPT = THREADS >= 256 ? 1 : 256 / THREADS;
    constexpr int SCAN_THREADS = 256 / DPT;
    uint32_t tot[DPT];
    uint32_t total = 0;
    if (tid < SCAN_THREADS) {
#pragma unroll
      for (int r = 0; r < DPT; r++) {
        const int d = tid * DPT + r;
        uint32_t run = 0;
        for (int w = 0; w < W; w++) {
          const uint32_t t = hist[w * 256 + d];
          hist[w * 256 + d] = (uint16_t)run;
          run += t;
        }
        tot[r] = run;
        total += run;
      }
    }
    uint32_t incl = total;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (tid < SCAN_THREADS && lane == 31) misc[2 + warp] = incl;
    __syncthreads();
    if (tid < SCAN_THREADS) {
      uint32_t base = incl - total;
      for (int w = 0; w < warp; w++) base += misc[2 + w];
#pragma unroll
      for (int r = 0; r < DPT; r++) {
        const int d = tid * DPT + r;
        for (int w = 0; w < W; w++) hist[w * 256 + d] = (uint16_t)(hist[w * 256 + d] + base);
        base += tot[r];
      }
    }
    __syncthreads();
    // pass 2: stable scatter
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
      const int base = c_begin + 32 * r;
      if (base < c_end) {  // warp-uniform
        const int i = base + lane;
        const bool valid = i < c_end;
        const uint32_t k = valid ? kin[i] : 0u;
        const uint32_t d = (k >> shift) & 0xffu;
        const unsigned peers = row_peers[r];
        const unsigned below = peers & ((1u << lane) - 1u);
        uint32_t start = 0;
        if (valid && below == 0u) {
          start = myhist[d];
          myhist[d] = (uint16_t)(start + __popc(peers));
        }
        start = __shfl_sync(0xffffffffu, start, valid ? __ffs(peers) - 1 : lane);
        if (valid) {
          const uint32_t o = start + __popc(below);
          kout[o] = k;
          iout[o] = iin[i];
        }
        __syncwarp();
      }
    }
    __syncthreads();
    { uint32_t* t = kin; kin = kout; kout = t; }
    { uint16_t* t = iin; iin = iout; iout = t; }
  }
  // ids of the sorted entries (kout is free now)
  uint32_t* ids = kout;
  uint32_t vmax = 0u;
  for (int i = tid; i < n; i += THREADS) {
    const uint32_t id = src[iin[i]].y;
    ids[i] = id;
    vmax = max(vmax, id);
  }
  vmax = __reduce_max_sync(0xffffffffu, vmax);
  if (lane == 0 && vmax) atomicMax(maxid, vmax);
  __syncthreads();
  // equal depths: ascending id (odd-even transposition restricted to runs of identical keys)
  for (;;) {
    int changed = 0;
#pragma unroll
    for (int phase = 0; phase < 2; phase++) {
      for (int i = 2 * tid + phase; i + 1 < n; i += 2 * THREADS) {
        if (kin[i] == kin[i + 1]) {
          const uint32_t a = ids[i], b = ids[i + 1];
          if (a > b) { ids[i] = b; ids[i + 1] = a; changed = 1; }
        }
      }
      __syncthreads();
    }
    if (!__syncthreads_or(changed)) break;
  }
  if (PAIRS) {
    uint2* out = const_cast<uint2*>(src);  // every read of the chunk happened before the barriers above
    for (int i = tid; i < n; i += THREADS) out[i] = make_uint2(kin[i], ids[i]);
  } else {
    for (int i = tid; i < n; i += THREADS) dst[i] = ids[i];
  }
  __syncthreads();  // shared memory is reused by the next tile of this CTA
}

// ---------------------------------------------------------------------------------------------------------------
// Warp-class sort: one WARP per tile for lists shorter than 512 entries (88 % of the tiles of workload C2, median
// 165 entries).  Same order contract and the same LSD radix scheme as radix_sort_tile, but warp-synchronous: no CTA
// barriers, 6.6 KB of shared memory per warp, eight tiles per 256-thread CTA.  The CTA-wide version spent most of its
// time in ~20 barriers per tile with seven of eight warps idle, while holding all 64 warp slots of the SM.
// ---------------------------------------------------------------------------------------------------------------
constexpr int WSORT_CAP = 1 << SORT_CTA_SHIFT;  // warp-class lists are shorter than the CTA-class boundary
constexpr size_t WSORT_BYTES = (size_t)WSORT_CAP * 12 + 256 * 2;  // keyA, keyB (u32), idxA, idxB (u16), hist (u16)

__device__ __forceinline__ void warp_sort_tile(const uint2* __restrict__ src, uint32_t* __restrict__ dst, const int n,
                                               unsigned char* smem_warp, uint32_t* __restrict__ maxid) {
  const int lane = threadIdx.x & 31;
  const unsigned below_mask = (1u << lane) - 1u;
  if (n <= 0) return;
  if (n <= 32) {  // rank sort in registers: position = number of entries with a smaller (depth, id)
    const uint2 kv = lane < n ? src[lane] : make_uint2(0xffffffffu, 0xffffffffu);
    const uint32_t m = __reduce_max_sync(0xffffffffu, lane < n ? kv.y : 0u);
    if (lane == 0) *maxid = m;
    const unsigned long long me = ((unsigned long long)kv.x << 32) | kv.y;
    int rank = 0;
    for (int j = 0; j < n; j++) {
      const unsigned long long o = __shfl_sync(0xffffffffu, me, j);
      rank += (o < me) ? 1 : 0;
    }
    if (lane < n) dst[rank] = kv.y;
    return;
  }
  uint32_t* keyA = reinterpret_cast<uint32_t*>(smem_warp);
  uint32_t* keyB = keyA + WSORT_CAP;
  uint16_t* idxA = reinterpret_cast<uint16_t*>(keyB + WSORT_CAP);
  uint16_t* idxB = idxA + WSORT_CAP;
  uint16_t* hist = idxB + WSORT_CAP;  // [256]
  uint32_t vor = 0u, vand = 0xffffffffu;
  for (int i = lane; i < n; i += 32) {
    const uint32_t k = src[i].x;
    keyA[i] = k;
    idxA[i] = (uint16_t)i;
    vor |= k;
    vand &= k;
  }
  const uint32_t differ = __reduce_or_sync(0xffffffffu, vor) ^ __reduce_and_sync(0xffffffffu, vand);
  __syncwarp();
  uint32_t* kin = keyA; uint32_t* kout = keyB;
  uint16_t* iin = idxA; uint16_t* iout = idxB;
  for (int pass = 0; pass < 4; pass++) {
    const int shift = 8 * pass;
    if (((differ >> shift) & 0xffu) == 0u) continue;  // warp-uniform: the whole tile agrees on this digit
    reinterpret_cast<uint4*>(hist)[lane] = make_uint4(0u, 0u, 0u, 0u);  // 32 lanes x 16 bytes = 256 x u16
    __syncwarp();
    constexpr int CACHED = 8;  // rows whose peer masks stay in registers (see radix_sort_tile): lists up to 256 entries
    unsigned row_peers[CACHED];
#pragma unroll
    for (int r = 0; r < CACHED; r++) {
      const int base = 32 * r;
      row_peers[r] = 0u;
      if (base < n) {
        const int i = base + lane;
        const bool valid = i < n;
        const uint32_t d = valid ? ((kin[i] >> shift) & 0xffu) : (256u + lane);
        const unsigned peers = match_digit(d, valid);
        row_peers[r] = peers;
        if (valid && (peers & below_mask) == 0u) hist[d] = (uint16_t)(hist[d] + __popc(peers));
        __syncwarp();
      }
    }
    for (int base = 32 * CACHED; base < n; base += 32) {
      const int i = base + lane;
      const bool valid = i < n;
      const uint32_t d = valid ? ((kin[i] >> shift) & 0xffu) : (256u + lane);
      const unsigned peers = match_digit(d, valid);
      if (valid && (peers & below_mask) == 0u) hist[d] = (uint16_t)(hist[d] + __popc(peers));
      __syncwarp();
    }
    // exclusive scan of the 256 counters: lane owns digits 8*lane .. 8*lane+7
    uint32_t c[8], total = 0;
#pragma unroll
    for (int r = 0; r < 8; r++) { c[r] = hist[8 * lane + r]; total += c[r]; }
    uint32_t incl = total;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    uint32_t run = incl - total;
#pragma unroll
    for (int r = 0; r < 8; r++) { hist[8 * lane + r] = (uint16_t)run; run += c[r]; }
    __syncwarp();
    auto place_row = [&](const int base, const bool cached, const unsigned cached_peers) {  // stable scatter of one row
        const int i = base + lane;
        const bool valid = i < n;
        const uint32_t k = valid ? kin[i] : 0u;
        const uint32_t d = valid ? ((k >> shift) & 0xffu) : (256u + lane);
        const unsigned peers = cached ? cached_peers : match_digit(d, valid);
        const unsigned below = peers & below_mask;
        uint32_t start = 0;
        if (valid && below == 0u) {
          start = hist[d];
          hist[d] = (uint16_t)(start + __popc(peers));
        }
        start = __shfl_sync(0xffffffffu, start, valid ? __ffs(peers) - 1 : lane);
        if (valid) {
          const uint32_t o = start + __popc(below);
          kout[o] = k;
          iout[o] = iin[i];
        }
        __syncwarp();
    };
#pragma unroll
    for (int r = 0; r < CACHED; r++)
      if (32 * r < n) place_row(32 * r, true, row_peers[r]);
    for (int base = 32 * CACHED; base < n; base += 32) place_row(base, false, 0u);
    { uint32_t* t = kin; kin = kout; kout = t; }
    { uint16_t* t = iin; iin = iout; iout = t; }
  }
  uint32_t* ids = kout;  // free now
  uint32_t vmax = 0u;
  for (int i = lane; i < n; i += 32) {
    const uint32_t id = src[iin[i]].y;
    ids[i] = id;
    vmax = max(vmax, id);
  }
  vmax = __reduce_max_sync(0xffffffffu, vmax);
  if (lane == 0) *maxid = vmax;
  __syncwarp();
  // equal depths: ascending id (odd-even transposition restricted to runs of identical keys)
  for (;;) {
    bool changed = false;
#pragma unroll
    for (int phase = 0; phase < 2; phase++) {
      for (int i = 2 * lane + phase; i + 1 < n; i += 64) {
        if (kin[i] == kin[i + 1]) {
          const uint32_t a = ids[i], b = ids[i + 1];
          if (a > b) { ids[i] = b; ids[i + 1] = a; changed = true; }
        }
      }
      __syncwarp();
    }
    if (!__any_sync(0xffffffffu, changed)) break;
  }
  for (int i = lane; i < n; i += 32) dst[i] = ids[i];
  __syncwarp();
}

// One launch sorts every list.  tile_order is sorted by floor(log2 n) descending and the scan kernel publishes how many
// tiles have n >= 2048 and n >= 512 plus a chunk table for the long ones (B2RStatus.reserved), so a CTA finds its work
// items without searching.  Work items, heaviest first:
//   1. one SORT_CHUNK-entry chunk of a list of >= 2048 entries: CTA-wide radix sort, sorted pairs written back in place
//      (merged by merge_chunks_kernel);
//   2. one list of 512..2047 entries: CTA-wide radix sort, ids written to their final place;
//   3. eight lists shorter than 512 entries, one per warp.
// The grid is the tile count; CTAs stride over the items and surplus CTAs exit at once.
template <int CAP, int THREADS>
__global__ void __launch_bounds__(THREADS) sort_mixed_kernel(const Ctx cx) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  B2R_TRACE_BEGIN();
  const unsigned long long cls = cx.status->reserved[0];
  const int n_large = (int)(cls & 0xffffffffull), n_ge512 = (int)(cls >> 32);
  const int n_chunks = (int)cx.status->reserved[1];
  const int n_cta = n_ge512 - n_large;
  const int n_warp_items = (cx.tiles - n_ge512 + (THREADS / 32) - 1) / (THREADS / 32);
  const int items = n_chunks + n_cta + n_warp_items;
  int last_n = 0;
  for (int b = blockIdx.x; b < items; b += gridDim.x) {
    if (b < n_chunks) {
      int lo = 0, hi = n_large - 1;  // the long list this chunk belongs to: last t with chunk_start[t] <= b
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if ((int)cx.chunk_start[mid] <= b) lo = mid; else hi = mid - 1;
      }
      const uint32_t tile = cx.tile_order[lo];
      const uint2 r = cx.ranges[tile];
      const int off = (b - (int)cx.chunk_start[lo]) * SORT_CHUNK;
      const int len = min(SORT_CHUNK, sort_length(cx, (int)tile, r) - off);
      if (len > 1) radix_sort_tile<CAP, THREADS, true>(cx.keys + r.x + off, nullptr, len, smem_raw, cx.tile_maxid + tile);
      else if (len == 1 && threadIdx.x == 0) atomicMax(cx.tile_maxid + tile, cx.keys[r.x + off].y);
      last_n = len;
    } else if (b < n_chunks + n_cta) {
      const uint32_t tile = cx.tile_order[n_large + (b - n_chunks)];
      const uint2 r = cx.ranges[tile];
      const int n = sort_length(cx, (int)tile, r);  // < 2048; can be below 512 when the duplicate capacity clamped the range
      const uint2* src = cx.keys + r.x;
      uint32_t* dst = cx.dup_ids + r.x;
      if (n > 32) {
        radix_sort_tile<CAP, THREADS>(src, dst, n, smem_raw, cx.tile_maxid + tile);
      } else {
        if (threadIdx.x < 32) warp_sort_tile(src, dst, n, smem_raw, cx.tile_maxid + tile);
        __syncthreads();
      }
      last_n = n;
    } else {
      const int warp = threadIdx.x >> 5;
      const int t = n_ge512 + (b - n_chunks - n_cta) * (THREADS / 32) + warp;
      if (t < cx.tiles) {
        const uint32_t tile = cx.tile_order[t];
        const uint2 r = cx.ranges[tile];
        const int n = sort_length(cx, (int)tile, r);
        last_n = -n;
        warp_sort_tile(cx.keys + r.x, cx.dup_ids + r.x, n, smem_raw + (size_t)warp * WSORT_BYTES, cx.tile_maxid + tile);
      }
    }
  }
  B2R_TRACE_END(last_n);
}

// Merge of the sorted chunks of the long lists: an entry's final position is its position in its own chunk plus, for
// every other chunk of the list, the number of entries that precede it -- one binary search per other chunk on the
// 64-bit (depth, id) key, which is unique, so the positions are a permutation.
// One work item = one chunk (2048 entries, eight per thread).  The other chunk is staged in shared memory with one round
// of coalesced loads and searched there (11 branch-free steps, the eight searches of a thread interleaved), and the
// chunk -> list look-up runs on a staged copy of the chunk table.  Searching in global memory instead would cost per entry
// ~40 DEPENDENT L2 accesses (7 for the look-up, 11 per other chunk) -- pure latency, and that much register-file-time
// taken from the frames in flight.  Exits at once when no list
// is that long (the common case at ExAvatar's single-render sizes).
constexpr int MERGE_TABLE = 1024;  // staged entries of chunk_start (lists of >= 2048 entries; more fall back to global loads)
__global__ void __launch_bounds__(256) merge_chunks_kernel(const Ctx cx) {
  const int n_large = (int)(cx.status->reserved[0] & 0xffffffffull);
  const int n_chunks = (int)cx.status->reserved[1];
  if ((int)blockIdx.x >= n_chunks) return;
  __shared__ uint2 other[SORT_CHUNK];
  __shared__ uint32_t table[MERGE_TABLE];
  const int tid = threadIdx.x;
  const int n_tab = min(n_large, MERGE_TABLE);
  for (int i = tid; i < n_tab; i += 256) table[i] = cx.chunk_start[i];
  __syncthreads();
  constexpr int PER = SORT_CHUNK / 256;  // entries per thread
  for (int b = blockIdx.x; b < n_chunks; b += gridDim.x) {
    int lo = 0, hi = n_large - 1;  // the long list chunk b belongs to: last t with chunk_start[t] <= b
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      const int cs = mid < n_tab ? (int)table[mid] : (int)cx.chunk_start[mid];
      if (cs <= b) lo = mid; else hi = mid - 1;
    }
    const uint32_t tile = cx.tile_order[lo];
    const uint2 r = cx.ranges[tile];
    const int n = sort_length(cx, (int)tile, r);
    const int c = b - (int)(lo < n_tab ? table[lo] : cx.chunk_start[lo]);
    const uint2* pairs = cx.keys + r.x;
    const int chunks = (n + SORT_CHUNK - 1) / SORT_CHUNK;
    const int len = min(SORT_CHUNK, n - c * SORT_CHUNK);  // entries of my chunk (<= 0: past a split pass's own entries)
    unsigned long long key[PER];
    uint32_t id[PER];
    int rank[PER];
#pragma unroll
    for (int j = 0; j < PER; j++) {
      const int i = j * 256 + tid;
      const uint2 me = i < len ? pairs[c * SORT_CHUNK + i] : make_uint2(0u, 0u);
      key[j] = ((unsigned long long)me.x << 32) | me.y;
      id[j] = me.y;
      rank[j] = i;
    }
    for (int c2 = 0; c2 < chunks; c2++) {
      if (c2 == c) continue;  // CTA-uniform
      const uint2* q = pairs + c2 * SORT_CHUNK;
      const int len2 = min(SORT_CHUNK, n - c2 * SORT_CHUNK);
      __syncthreads();  // the previous chunk's searches are done
#pragma unroll
      for (int j = 0; j < PER; j++) {
        const int i = j * 256 + tid;
        if (i < len2) other[i] = q[i];
      }
      __syncthreads();
      int l[PER];
#pragma unroll
      for (int j = 0; j < PER; j++) l[j] = 0;
#pragma unroll
      for (int step = SORT_CHUNK / 2; step >= 1; step >>= 1) {  // l = number of entries of chunk c2 below `key`
#pragma unroll
        for (int j = 0; j < PER; j++) {
          const int probe = l[j] + step;  // entries [0, probe) all below key  <=>  other[probe - 1] < key
          if (probe <= len2) {
            const uint2 v = other[probe - 1];
            if ((((unsigned long long)v.x << 32) | v.y) < key[j]) l[j] = probe;
          }
        }
      }
      // `step` runs over the powers of two below 2048, so l can reach 2047 at most; the one remaining case is "all 2048
      // entries are below key"
      if (len2 == SORT_CHUNK) {
#pragma unroll
        for (int j = 0; j < PER; j++) {
          if (l[j] == SORT_CHUNK - 1) {
            const uint2 v = other[SORT_CHUNK - 1];
            if ((((unsigned long long)v.x << 32) | v.y) < key[j]) l[j] = SORT_CHUNK;
          }
        }
      }
#pragma unroll
      for (int j = 0; j < PER; j++) rank[j] += l[j];
    }
#pragma unroll
    for (int j = 0; j < PER; j++)
      if (j * 256 + tid < len) cx.dup_ids[r.x + rank[j]] = id[j];
  }
}

constexpr int SORT_SMALL = SORT_CHUNK;  // capacity of the CTA-wide sort = chunk size of the long lists
void launch_sort(const Ctx& cx, cudaStream_t st);

int launch_binning(const B2RScene& sc, const Ctx& cx, bool rescan, cudaStream_t st) {
  // the two-phase entry re-derives ranges and cursors for the capacity the caller finally chose
  // (never re-published to the host mirror: the count there belongs to the project phase that produced it, and another
  // stream's render may be waiting on its own token in the same mirror)
  if (rescan) {
    Ctx quiet = cx;
    quiet.status_mirror = nullptr;
    launch_tile_scan(quiet, st);
  }
  if (sc.P > 0) {
    ProfScope p(K_SCATTER, st);
    const size_t smem = (size_t)cx.tiles * 8;
    // worth it while the per-CTA zero / flush sweeps over the tile table stay small (at 8160 tiles they cost more than
    // the direct atomics save)
    if (cx.tiles <= 2048) {
      cudaFuncSetAttribute(scatter_agg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
      launch_k(scatter_agg_kernel, (sc.P + 255) / 256, 256, smem, st, true, sc, cx, 0);
    } else {
      launch_k(scatter_kernel, (sc.P + 255) / 256, 256, 0, st, true, sc, cx, 0);
    }
  }
  launch_sort(cx, st);
  return check_launch();
}

void launch_sort(const Ctx& cx, cudaStream_t st) {
  const int sms = device_sm_count();
  constexpr int ST = 256;
  constexpr size_t cta_bytes = RadixSmem<SORT_SMALL, ST>::bytes, warp_bytes = (ST / 32) * WSORT_BYTES;
  constexpr size_t small_bytes = cta_bytes > warp_bytes ? cta_bytes : warp_bytes;
  // function attributes are per device: set on every launch (cheap), so a process that drives several GPUs works
  cudaFuncSetAttribute(sort_mixed_kernel<SORT_SMALL, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)small_bytes);
  {
    ProfScope p(K_SORT_SMALL, st);
    launch_k(sort_mixed_kernel<SORT_SMALL, ST>, cx.tiles, ST, small_bytes, st, true, cx);
  }
  {
    ProfScope p(K_SORT_LARGE, st);
    launch_k(merge_chunks_kernel, 2 * sms, 256, 0, st, true, cx);  // strides over the chunks; surplus CTAs exit at once
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Split pass (b2r_forward_project_split / b2r_forward_bin_split).  Rows [0, split) of this pass are the rows [0, split) of
// a BASE pass that projected and binned them with the same camera and inputs (ExAvatar: the scene Gaussians of
// cat(scene, human) and of cat(scene, human_refined)), so their records, their tile pairs and their depth order are the
// base pass's.  This pass projects, scatters and sorts only its own rows [split, P), and only tiles its own rows reach get
// a list: the base list of the tile filtered to ids < split (filtering keeps the order) merged with the own sorted
// entries on the unique 64-bit (depth_bits, id) key -- the order the joint sort gives, entry for entry.  Other tiles get
// empty lists (tile_maxid 0).
// ---------------------------------------------------------------------------------------------------------------

// Copies the base pass's records and radii of rows [0, split) (a view gathers them) and turns every tile count of the own
// rows into the length of the merged list: own entries + base entries with id < split.  sort_len keeps the own count.
__global__ void __launch_bounds__(256) split_prepare_kernel(const Ctx cx, const Ctx base, const int split,
                                                            int32_t* __restrict__ radii) {
  const int tid = threadIdx.x;
  const float4* gsrc = reinterpret_cast<const float4*>(base.geom);
  float4* gdst = reinterpret_cast<float4*>(cx.geom);
  for (size_t k = (size_t)blockIdx.x * 256 + tid; k < (size_t)split * 3; k += (size_t)gridDim.x * 256) gdst[k] = gsrc[k];
  for (int k = blockIdx.x * 256 + tid; k < split; k += gridDim.x * 256) radii[k] = base.aux[k].z;
  for (int t = blockIdx.x; t < cx.tiles; t += gridDim.x) {
    const uint32_t own = cx.tile_count[t];  // CTA-uniform
    uint32_t s = 0;
    if (own) {
      const uint2 rb = base.ranges[t];
      for (uint32_t k = rb.x; k < rb.y; k += 256)
        s += (uint32_t)__syncthreads_count(k + tid < rb.y && base.dup_ids[k + tid] < (uint32_t)split);
    }
    if (tid == 0) {
      cx.sort_len[t] = own;
      cx.tile_count[t] = own + s;
    }
    __syncthreads();
  }
}

// One CTA per tile of tile_order (the tiles with a list come first).  The own sorted ids and the filtered base list are
// written as (depth_bits, id) keys into the tile's key range -- own entries first, then base entries -- and every entry
// goes to its position in the merged order: its index in its own sequence plus the number of entries of the other
// sequence below it (binary searches in shared-memory chunks of the other sequence).
constexpr int SPLIT_CHUNK = 2048;
constexpr int SPLIT_PER = 8;  // entries per thread and round
__global__ void __launch_bounds__(256) split_merge_kernel(const Ctx cx, const Ctx base, const uint32_t* __restrict__ own_ids,
                                                          const int split) {
  __shared__ uint2 other[SPLIT_CHUNK];
  __shared__ uint32_t wtot[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t tile = cx.tile_order[blockIdx.x];
  const uint2 r = cx.ranges[tile];
  const int n = (int)(r.y - r.x);
  if (n == 0) return;
  const int n_own = sort_length(cx, (int)tile, r);
  uint2* keys = cx.keys + r.x;
  for (int i = tid; i < n_own; i += 256) {
    const uint32_t id = own_ids[r.x + i];
    keys[i] = make_uint2(__float_as_uint(cx.geom[id].g1.z), id);
  }
  // ordered compaction of the base list's entries below the split behind the own entries (guarded: with an overflowed
  // capacity the range can be shorter than both sequences)
  const uint2 rb = base.ranges[tile];
  int n_base = 0;
  for (uint32_t k0 = rb.x; k0 < rb.y; k0 += 256) {
    const uint32_t k = k0 + tid;
    const uint32_t id = k < rb.y ? base.dup_ids[k] : 0xffffffffu;
    const bool take = id < (uint32_t)split;
    const unsigned b = __ballot_sync(0xffffffffu, take);
    if (lane == 0) wtot[warp] = __popc(b);
    __syncthreads();
    int off = n_base, tot = 0;
    for (int w = 0; w < 8; w++) {
      off += w < warp ? (int)wtot[w] : 0;
      tot += (int)wtot[w];
    }
    off += __popc(b & ((1u << lane) - 1u));
    if (take && n_own + off < n) keys[n_own + off] = make_uint2(__float_as_uint(cx.geom[id].g1.z), id);
    n_base += tot;
    __syncthreads();  // wtot is rewritten by the next round
  }
  __syncthreads();  // the keys above are visible to the whole CTA
  if (n_own + n_base != n) {  // capacity overflow (reported in B2RStatus): keep every entry a valid id, order is moot
    for (int i = tid; i < n; i += 256) cx.dup_ids[r.x + i] = keys[i].y;
    return;
  }
  for (int side = 0; side < 2; side++) {  // 0: own entries against the base sequence, 1: the other way round
    const uint2* mine = side ? keys + n_own : keys;
    const uint2* oth = side ? keys : keys + n_own;
    const int n_mine = side ? n_base : n_own, n_oth = side ? n_own : n_base;
    for (int x0 = 0; x0 < n_mine; x0 += 256 * SPLIT_PER) {  // CTA-uniform
      unsigned long long key[SPLIT_PER];
      int rank[SPLIT_PER];
#pragma unroll
      for (int j = 0; j < SPLIT_PER; j++) {
        const int i = x0 + j * 256 + tid;
        const uint2 v = i < n_mine ? mine[i] : make_uint2(0u, 0u);
        key[j] = ((unsigned long long)v.x << 32) | v.y;
        rank[j] = i;
      }
      for (int c0 = 0; c0 < n_oth; c0 += SPLIT_CHUNK) {
        const int len2 = min(SPLIT_CHUNK, n_oth - c0);
        __syncthreads();  // the previous chunk's searches are done
        for (int i = tid; i < len2; i += 256) other[i] = oth[c0 + i];
        __syncthreads();
#pragma unroll
        for (int j = 0; j < SPLIT_PER; j++) {
          int l = 0;  // entries of the chunk below key
          for (int step = SPLIT_CHUNK; step >= 1; step >>= 1) {
            const int probe = l + step;
            if (probe <= len2) {
              const uint2 v = other[probe - 1];
              if ((((unsigned long long)v.x << 32) | v.y) < key[j]) l = probe;
            }
          }
          rank[j] += l;
        }
      }
#pragma unroll
      for (int j = 0; j < SPLIT_PER; j++)
        if (x0 + j * 256 + tid < n_mine) cx.dup_ids[r.x + rank[j]] = (uint32_t)(key[j] & 0xffffffffull);
    }
  }
}

int launch_binning_split(const B2RScene& sc, const Ctx& cx_in, const Ctx& base, uint32_t* own_ids, const int first_row,
                         int32_t* radii, cudaStream_t st) {
  const Ctx& cx = cx_in;
  {
    ProfScope p(K_MISC, st);
    launch_k(split_prepare_kernel, cx.tiles, 256, 0, st, true, cx, base, first_row, radii);
  }
  launch_tile_scan(cx, st, cx.dup_capacity > 0 ? 1 : 0);
  if (sc.P > first_row) {
    ProfScope p(K_SCATTER, st);
    const unsigned grid = (unsigned)((sc.P - first_row + 255) / 256);
    if (cx.tiles <= 2048) {
      cudaFuncSetAttribute(scatter_agg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
      launch_k(scatter_agg_kernel, grid, 256, (size_t)cx.tiles * 8, st, true, sc, cx, first_row);
    } else {
      launch_k(scatter_kernel, grid, 256, 0, st, true, sc, cx, first_row);
    }
  }
  Ctx own = cx;  // the own entries are sorted into the scratch; the merge writes the lists
  own.dup_ids = own_ids;
  launch_sort(own, st);
  {
    ProfScope p(K_SORT_LARGE, st);
    launch_k(split_merge_kernel, cx.tiles, 256, 0, st, true, cx, base, own_ids, first_row);
  }
  return check_launch();
}

}  // namespace b2r

#ifdef B2R_CTA_TRACE
extern "C" int b2r_debug_trace_sort(unsigned long long* buf) {
  return (int)cudaMemcpyToSymbol(b2r::g_cta_trace, &buf, sizeof(buf));
}
#endif
