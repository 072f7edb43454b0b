// regularizers.cu -- ExAvatar's per-frame human regularisers (avatar/main/model.py:217-257 with LaplacianReg,
// HandMeanReg, HandRGBReg, ArmRGBReg and JointOffsetSymmetricReg of avatar/common/nets/loss.py:97-197 and
// smpl_x.get_arm) as ten means, with no host synchronisation and no float atomics.
//
// Forward (all launches on the caller's stream, counted under kernel id 8 misc):
//   vertex_normals_kernel (geometry.cu) on mesh_neutral_pose: HandMeanReg and the arm split share it.
//   regs_hand_partial_kernel  fp64 partial sums of rgb / rgb_refined over the right- and left-hand rows (grid-stride,
//                             fixed row -> thread map, block_sum of common.cuh).
//   regs_split_kernel         ONE CTA: the hand means from those partials; the arm rows classified upper (n_y > 0.5f)
//                             or lower and compacted in vertex order with device-side counts; k reset to 50.
//   regs_rank_kernel          rank of every upper row by (x, vertex index): integer counts, integer atomics.
//   regs_scatter_kernel       upper rows in x order, padded to the arm capacity with +inf.
//   regs_window_kernel        per lower row l: the window |fl(l_x - u_x)| < 0.01f is a contiguous range of the sorted
//                             list (fl(l - u) is monotone in u); two binary searches with that predicate give it, and
//                             k = min(50, min_i c_i) by an integer atomicMin.
//   regs_select_kernel        one warp per lower row: the k smallest keys (fp32 distance bits, vertex index) of its
//                             window by a bitwise search on the 64-bit key, the means of rgb AND rgb_refined over them
//                             (one selection serves both terms) and the row's arm term.
//   regs_terms_kernel         one thread per vertex: every per-row contribution, the six Laplacians kept for the
//                             backward; fp64 per-CTA partials.
//   regs_reduce_kernel        ONE CTA: partials in a fixed order, the arm terms, the two joint terms; out[10].
// Backward: regs_backward_kernel, one thread per vertex, closed forms; the Laplacian adjoint is a gather over the
// transposed table (CSR).  The joint gradients are written by the first CTA.
//
// The arm predicates (fp32 x-difference against 0.01f, fp32 distance sqrt((dx*dx + dy*dy) + dz*dz)) must be the
// reference's bits: this unit is compiled with --fmad=false (build_ext.py).
#include <float.h>
#include <limits.h>
#include <math.h>

#include "common.cuh"

namespace b2r {

constexpr int RG_THREADS = 256;
constexpr int RG_HAND_BLOCKS = 128;  // fixed: the hand sums' row -> thread map, and so their bits, never change
constexpr int RG_SPLIT_THREADS = 1024;
constexpr int RG_NBR = 10;           // LaplacianReg's neighbor_max_num
constexpr int RG_KMAX = 50;          // ArmRGBReg's top_k cap
constexpr int RG_NTERMS = 7;         // per-row terms summed by regs_terms_kernel
constexpr float RG_DIST_X_THR = 0.01f;
constexpr float RG_COS60 = 0.5f;     // math.cos(math.pi / 3) compared against an fp32 tensor: rounded to fp32
constexpr float RG_NORMALIZE_EPS = 1e-12f;

struct RegsLayout {
  size_t normals, lap, hand_part, hand_mean, counters, up_key, rank, sorted_x, sorted_idx, lo_idx, arm_lo, win, arm_tgt,
      arm_term, term_part, total;
  int nb;  // CTAs of the per-vertex kernels
};

inline RegsLayout regs_layout(int P, int n_arm) {
  const size_t p = P > 0 ? (size_t)P : 1, a = n_arm > 0 ? (size_t)n_arm : 1;
  RegsLayout L;
  L.nb = (int)((p + RG_THREADS - 1) / RG_THREADS);
  size_t o = 0;
  L.normals = o; o += align_up(p * 3 * sizeof(float));
  L.lap = o; o += align_up(6 * p * 3 * sizeof(float));  // A mo, A (mo + moo), A s, A s', A rgb, A rgb'
  L.hand_part = o; o += align_up((size_t)RG_HAND_BLOCKS * 12 * sizeof(double));
  L.hand_mean = o; o += align_up(12 * sizeof(float));
  L.counters = o; o += align_up(4 * sizeof(int));  // n_up, n_lo, k
  L.up_key = o; o += align_up(a * sizeof(unsigned long long));
  L.rank = o; o += align_up(a * sizeof(int));
  L.sorted_x = o; o += align_up(a * sizeof(float));
  L.sorted_idx = o; o += align_up(a * sizeof(int));
  L.lo_idx = o; o += align_up(a * sizeof(int));
  L.arm_lo = o; o += align_up(a * sizeof(int));
  L.win = o; o += align_up(a * sizeof(int2));
  L.arm_tgt = o; o += align_up(a * 6 * sizeof(float));
  L.arm_term = o; o += align_up(a * sizeof(double));
  L.term_part = o; o += align_up((size_t)L.nb * RG_NTERMS * sizeof(double));
  L.total = o;
  return L;
}

struct RegsPtrs {
  float* normals;
  float* lap;
  double* hand_part;
  float* hand_mean;  // [set][hand][c]: set 0 rgb, 1 rgb_refined; hand 0 right, 1 left
  int* counters;
  unsigned long long* up_key;
  int* rank;
  float* sorted_x;
  int* sorted_idx;
  int* lo_idx;
  int* arm_lo;
  int2* win;
  float* arm_tgt;
  double* arm_term;
  double* term_part;
};

inline RegsPtrs regs_ptrs(const B2RRegs& r, void* scratch) {
  const RegsLayout L = regs_layout(r.P, r.n_arm);
  char* s = (char*)scratch;
  return RegsPtrs{(float*)(s + L.normals), (float*)(s + L.lap), (double*)(s + L.hand_part),
                  (float*)(s + L.hand_mean), (int*)(s + L.counters), (unsigned long long*)(s + L.up_key),
                  (int*)(s + L.rank), (float*)(s + L.sorted_x), (int*)(s + L.sorted_idx), (int*)(s + L.lo_idx),
                  (int*)(s + L.arm_lo), (int2*)(s + L.win), (float*)(s + L.arm_tgt), (double*)(s + L.arm_term),
                  (double*)(s + L.term_part)};
}

// x -> an unsigned key with the float order (negative values reversed), for the (x, index) sort of the upper rows
__device__ __forceinline__ unsigned ordered_bits(float x) {
  const unsigned u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(RG_THREADS) regs_hand_partial_kernel(const B2RRegs r, double* __restrict__ part) {
  __shared__ double wsum[RG_THREADS / 32 * 12];
  double v[12];
#pragma unroll
  for (int t = 0; t < 12; t++) v[t] = 0.0;
  for (int i = blockIdx.x * RG_THREADS + threadIdx.x; i < r.P; i += RG_HAND_BLOCKS * RG_THREADS) {
    const uint8_t h = r.hand[i];
    if (!h) continue;
#pragma unroll
    for (int hand = 0; hand < 2; hand++) {
      if (!((h >> hand) & 1)) continue;
#pragma unroll
      for (int c = 0; c < 3; c++) {
        v[hand * 3 + c] += (double)r.rgb[3 * i + c];
        v[6 + hand * 3 + c] += (double)r.rgb_refined[3 * i + c];
      }
    }
  }
  block_sum<RG_THREADS>(v, wsum);
  if (threadIdx.x == 0)
    for (int t = 0; t < 12; t++) part[blockIdx.x * 12 + t] = v[t];
}

// exclusive block scan of one int per thread (1024 threads); returns the block total to every thread
__device__ __forceinline__ int block_excl_scan(int x, int& total, int* wsum) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = x;
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += y;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = wsum[lane];
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += y;
    }
    wsum[lane] = w;
  }
  __syncthreads();
  total = wsum[31];
  const int r = incl - x + (warp > 0 ? wsum[warp - 1] : 0);
  __syncthreads();  // wsum is reused by the next call
  return r;
}

__global__ void __launch_bounds__(RG_SPLIT_THREADS) regs_split_kernel(const B2RRegs r, const RegsPtrs s) {
  __shared__ int wsum[32];
  const int tid = threadIdx.x;
  if (tid < 12) {  // hand means: the partials in block order, over the (equal) hand counts
    double a = 0.0;
    for (int b = 0; b < RG_HAND_BLOCKS; b++) a += s.hand_part[b * 12 + tid];
    s.hand_mean[tid] = (float)(a / (double)r.n_rhand);
  }
  int n_up = 0, n_lo = 0;
  for (int c0 = 0; c0 < r.n_arm; c0 += RG_SPLIT_THREADS) {
    const int t = c0 + tid;
    int v = -1;
    bool up = false;
    if (t < r.n_arm) {
      v = r.arm_idx[t];
      up = s.normals[3 * v + 1] > RG_COS60;
    }
    int tot_up, tot_lo;
    const int pu = block_excl_scan(t < r.n_arm && up, tot_up, wsum);
    const int pl = block_excl_scan(t < r.n_arm && !up, tot_lo, wsum);
    if (t < r.n_arm) {
      if (up) {
        s.up_key[n_up + pu] = ((unsigned long long)ordered_bits(r.mesh[3 * v]) << 32) | (unsigned)v;
        s.arm_lo[t] = -1;
      } else {
        s.lo_idx[n_lo + pl] = v;
        s.arm_lo[t] = n_lo + pl;
      }
    }
    n_up += tot_up;
    n_lo += tot_lo;
  }
  for (int t = tid; t < r.n_arm; t += RG_SPLIT_THREADS) s.rank[t] = 0;
  if (tid == 0) {
    s.counters[0] = n_up;
    s.counters[1] = n_lo;
    s.counters[2] = RG_KMAX;
  }
}

// rank[i] = #{ j < n_up : key[j] < key[i] }: CTA (x, y) counts the keys of tile y below each key of tile x
__global__ void __launch_bounds__(RG_THREADS) regs_rank_kernel(const RegsPtrs s) {
  __shared__ unsigned long long kt[RG_THREADS];
  const int n_up = s.counters[0];
  const int i0 = blockIdx.x * RG_THREADS, j0 = blockIdx.y * RG_THREADS;
  if (i0 >= n_up || j0 >= n_up) return;  // CTA-uniform
  const int j = j0 + threadIdx.x;
  kt[threadIdx.x] = j < n_up ? s.up_key[j] : ~0ull;
  __syncthreads();
  const int i = i0 + threadIdx.x;
  if (i >= n_up) return;
  const unsigned long long k = s.up_key[i];
  int c = 0;
  for (int q = 0; q < RG_THREADS; q++) c += kt[q] < k;
  if (c) atomicAdd(s.rank + i, c);  // integer sums: the same result in any order
}

__global__ void __launch_bounds__(RG_THREADS) regs_scatter_kernel(const B2RRegs r, const RegsPtrs s) {
  const int i = blockIdx.x * RG_THREADS + threadIdx.x;
  if (i >= r.n_arm) return;
  const int n_up = s.counters[0];
  if (i < n_up) {
    const int v = (int)(unsigned)(s.up_key[i] & 0xffffffffull);
    const int q = s.rank[i];
    s.sorted_x[q] = r.mesh[3 * v];
    s.sorted_idx[q] = v;
  } else {
    s.sorted_x[i] = INFINITY;  // the ranks fill [0, n_up): the padding is never overwritten
    s.sorted_idx[i] = -1;
  }
}

__global__ void __launch_bounds__(RG_THREADS) regs_window_kernel(const B2RRegs r, const RegsPtrs s) {
  const int p = blockIdx.x * RG_THREADS + threadIdx.x;
  const int n_up = s.counters[0], n_lo = s.counters[1];
  int c = INT_MAX;
  if (p < n_lo) {
    const float l = r.mesh[3 * s.lo_idx[p]];
    // fl(l - u) falls as u grows: [a, b) = { u : -0.01f < fl(l - u) < 0.01f } = { u : |fl(l - u)| < 0.01f }
    int lo = 0, hi = n_up;
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if (l - s.sorted_x[m] < RG_DIST_X_THR) hi = m; else lo = m + 1;
    }
    const int a = lo;
    hi = n_up;
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if (l - s.sorted_x[m] <= -RG_DIST_X_THR) hi = m; else lo = m + 1;
    }
    s.win[p] = make_int2(a, lo);
    c = lo - a;
  }
  c = __reduce_min_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c < RG_KMAX) atomicMin(s.counters + 2, c);
}

// distance key of upper row q of the window for the lower vertex (lx, ly, lz): fp32 sqrt((dx*dx + dy*dy) + dz*dz)
// (torch.sqrt(torch.sum((lower - upper) ** 2, 2))) in the high word, the upper vertex index in the low word
__device__ __forceinline__ unsigned long long arm_key(const B2RRegs& r, const RegsPtrs& s, int q, float lx, float ly,
                                                      float lz, int& v) {
  v = s.sorted_idx[q];
  const float dx = lx - r.mesh[3 * v], dy = ly - r.mesh[3 * v + 1], dz = lz - r.mesh[3 * v + 2];
  const float d = sqrtf((dx * dx + dy * dy) + dz * dz);
  return ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)v;
}

__global__ void __launch_bounds__(RG_THREADS) regs_select_kernel(const B2RRegs r, const RegsPtrs s) {
  const int lane = threadIdx.x & 31;
  const int p = (blockIdx.x * RG_THREADS + threadIdx.x) >> 5;
  if (p >= s.counters[1]) return;  // warp-uniform
  const int k = s.counters[2];
  const int2 w = s.win[p];
  const int lv = s.lo_idx[p];
  const float lx = r.mesh[3 * lv], ly = r.mesh[3 * lv + 1], lz = r.mesh[3 * lv + 2];
  // the k-th smallest key K: the largest value with fewer than k keys below it, built bit by bit.  Keys are distinct
  // (vertex index in the low word), so exactly k keys are <= K: distance ties at the k-th place go to the lowest index.
  unsigned long long K = 0ull;
  if (k > 0) {
    for (int b = 62; b >= 0; b--) {
      const unsigned long long t = K | (1ull << b);
      int c = 0;
      for (int q = w.x + lane; q < w.y; q += 32) {
        int v;
        c += arm_key(r, s, q, lx, ly, lz, v) < t;
      }
      c = __reduce_add_sync(0xffffffffu, c);
      if (c < k) K = t;
    }
  }
  float a[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (k > 0)
    for (int q = w.x + lane; q < w.y; q += 32) {
      int v;
      if (arm_key(r, s, q, lx, ly, lz, v) <= K)
        for (int c = 0; c < 3; c++) {
          a[c] += r.rgb[3 * v + c];
          a[3 + c] += r.rgb_refined[3 * v + c];
        }
    }
#pragma unroll
  for (int c = 0; c < 6; c++) a[c] = warp_sum(a[c]);
  if (lane == 0) {
    double term = 0.0;
    for (int c = 0; c < 6; c++) {
      const float t = a[c] / (float)k;  // k = 0: 0 / 0 = NaN, the mean over an empty axis
      s.arm_tgt[6 * p + c] = t;
      const float x = c < 3 ? r.rgb[3 * lv + c] : r.rgb_refined[3 * lv + c - 3];
      const double d = (double)x - (double)t;
      term += d * d;
    }
    s.arm_term[p] = term;
  }
}

// lap(x)_v = x_v + sum_j x[n_vj] w_vj (LaplacianReg.compute_laplacian), fp32, neighbours in table order
__device__ __forceinline__ float3 laplacian(const float* __restrict__ x, const int* __restrict__ nbr,
                                            const float* __restrict__ nw, int v) {
  float sx = 0.f, sy = 0.f, sz = 0.f;
#pragma unroll
  for (int j = 0; j < RG_NBR; j++) {
    const int n = nbr[RG_NBR * v + j];
    const float w = nw[RG_NBR * v + j];
    sx += x[3 * n] * w;
    sy += x[3 * n + 1] * w;
    sz += x[3 * n + 2] * w;
  }
  return make_float3(x[3 * v] + sx, x[3 * v + 1] + sy, x[3 * v + 2] + sz);
}

__device__ __forceinline__ double sq3(float3 a) {
  return (double)a.x * a.x + (double)a.y * a.y + (double)a.z * a.z;
}

// clamp(n . normalize(o), min=0) with F.normalize's max(|o|, 1e-12)
__device__ __forceinline__ float hand_dot(const float* n, const float* o) {
  const float nrm = sqrtf(o[0] * o[0] + o[1] * o[1] + o[2] * o[2]);
  const float den = fmaxf(nrm, RG_NORMALIZE_EPS);
  return fmaxf(n[0] * (o[0] / den) + n[1] * (o[1] / den) + n[2] * (o[2] / den), 0.f);
}

__global__ void __launch_bounds__(RG_THREADS) regs_terms_kernel(const B2RRegs r, const RegsPtrs s) {
  __shared__ double wsum[RG_THREADS / 32 * RG_NTERMS];
  const int v = blockIdx.x * RG_THREADS + threadIdx.x;
  double t[RG_NTERMS];
#pragma unroll
  for (int q = 0; q < RG_NTERMS; q++) t[q] = 0.0;
  if (v < r.P) {
    const size_t P = (size_t)r.P;
    const float* W = r.weights;  // (5,P)
    const float w1 = W[v], w2 = W[P + v], w3 = W[2 * P + v], w4 = W[3 * P + v], w5 = W[4 * P + v];
    float mo[3], moo[3], su[3], mm[3];
    double a = 0.0, b = 0.0;
    const float so = r.scale_offset[v];
    const float* sused = r.scale_reg ? r.scale_reg : r.scale;
    for (int c = 0; c < 3; c++) {
      mo[c] = r.mean_offset[3 * v + c];
      moo[c] = r.mean_offset_offset[3 * v + c];
      mm[c] = mo[c] + moo[c];
      su[c] = sused[3 * v + c];
      a += (double)mo[c] * mo[c] + (double)moo[c] * moo[c];
      b += (double)su[c] * su[c] + (double)so * so;
    }
    t[0] = a * w1;
    t[2] = b * w2;
    const uint8_t h = r.hand[v];
    if (h) {
      const float* n = s.normals + 3 * v;
      t[1] = (double)hand_dot(n, mo) + (double)hand_dot(n, moo);
      for (int set = 0; set < 2; set++) {
        const float* x = (set ? r.rgb_refined : r.rgb) + 3 * v;
        for (int hand = 0; hand < 2; hand++) {
          if (!((h >> hand) & 1)) continue;
          for (int c = 0; c < 3; c++) {
            const double d = (double)x[c] - (double)s.hand_mean[set * 6 + hand * 3 + c];
            t[6] += d * d;
          }
        }
      }
    }
    // lap_mean: lap(mnp + mo) - lap(mnp) = lap(mo) and likewise for mo + moo -- the Laplacian is linear, and taking it of
    // the offsets avoids subtracting two Laplacians of metre-scale coordinates in fp32
    const float3 l1 = laplacian(r.mean_offset, r.nbr_idx, r.nbr_w, v);
    float3 l2;
    {
      float sx = 0.f, sy = 0.f, sz = 0.f;
#pragma unroll
      for (int j = 0; j < RG_NBR; j++) {
        const int n = r.nbr_idx[RG_NBR * v + j];
        const float w = r.nbr_w[RG_NBR * v + j];
        sx += (r.mean_offset[3 * n] + r.mean_offset_offset[3 * n]) * w;
        sy += (r.mean_offset[3 * n + 1] + r.mean_offset_offset[3 * n + 1]) * w;
        sz += (r.mean_offset[3 * n + 2] + r.mean_offset_offset[3 * n + 2]) * w;
      }
      l2 = make_float3(mm[0] + sx, mm[1] + sy, mm[2] + sz);
    }
    const float3 l3 = laplacian(r.scale, r.nbr_idx, r.nbr_w, v);
    const float3 l4 = laplacian(r.scale_refined, r.nbr_idx, r.nbr_w, v);
    const float3 l5 = laplacian(r.rgb, r.nbr_idx, r.nbr_w, v);
    const float3 l6 = laplacian(r.rgb_refined, r.nbr_idx, r.nbr_w, v);
    t[3] = (sq3(l1) + sq3(l2)) * w3;
    t[4] = (sq3(l3) + sq3(l4)) * w4;
    t[5] = (sq3(l5) + sq3(l6)) * w5;
    const float3 ls[6] = {l1, l2, l3, l4, l5, l6};
    for (int q = 0; q < 6; q++) {
      float* o = s.lap + (size_t)q * P * 3 + 3 * v;
      o[0] = ls[q].x; o[1] = ls[q].y; o[2] = ls[q].z;
    }
  }
  block_sum<RG_THREADS>(t, wsum);
  if (threadIdx.x == 0)
    for (int q = 0; q < RG_NTERMS; q++) s.term_part[(size_t)blockIdx.x * RG_NTERMS + q] = t[q];
}

__global__ void __launch_bounds__(RG_THREADS) regs_reduce_kernel(const B2RRegs r, const RegsPtrs s, const int nb,
                                                                 float* __restrict__ out) {
  __shared__ double wsum[RG_THREADS / 32 * (RG_NTERMS + 1)];
  double t[RG_NTERMS + 1];
#pragma unroll
  for (int q = 0; q <= RG_NTERMS; q++) t[q] = 0.0;
  for (int b = threadIdx.x; b < nb; b += RG_THREADS)
    for (int q = 0; q < RG_NTERMS; q++) t[q] += s.term_part[(size_t)b * RG_NTERMS + q];
  const int n_lo = s.counters[1];
  for (int p = threadIdx.x; p < n_lo; p += RG_THREADS) t[RG_NTERMS] += s.arm_term[p];
  block_sum<RG_THREADS>(t, wsum);
  if (threadIdx.x != 0) return;
  const double n3 = 3.0 * r.P;
  double jreg = 0.0, jsym = 0.0;
  for (int j = 0; j < r.J; j++)
    for (int c = 0; c < 3; c++) {
      const double d = (double)r.joint_offset[3 * j + c] - (double)r.joint_target[3 * j + c];
      jreg += d * d * r.joint_weight[j];
    }
  for (int q = 0; q < r.n_pairs; q++) {
    const float* a = r.joint_offset + 3 * r.sym_pairs[2 * q];
    const float* b = r.joint_offset + 3 * r.sym_pairs[2 * q + 1];
    jsym += fabs((double)a[0] + b[0]) + fabs((double)a[1] - b[1]) + fabs((double)a[2] - b[2]);
  }
  out[0] = (float)(t[0] / n3);                                 // gaussian_mean_reg
  out[1] = (float)(t[1] / r.n_hand);                           // gaussian_mean_hand_reg
  out[2] = (float)(t[2] / n3);                                 // gaussian_scale_reg
  out[3] = (float)(t[3] * 100000.0 / n3);                      // lap_mean
  out[4] = (float)(t[4] * 100000.0 / n3);                      // lap_scale
  out[5] = (float)(t[5] / n3);                                 // lap_rgb
  out[6] = (float)(t[6] * 0.01 / (3.0 * r.n_rhand));           // hand_rgb_reg
  out[7] = (float)(t[RG_NTERMS] * 0.1 / (3.0 * n_lo));         // arm_rgb_reg: NaN without lower rows (0 / 0)
  out[8] = (float)(jreg / (3.0 * r.J));                        // joint_offset_reg
  out[9] = (float)(jsym / r.n_pairs);                          // joint_offset_sym_reg
}

// d/do clamp(n . o / max(|o|, eps), 0): passes where the clamped value is >= 0 (clamp's gradient at exactly 0)
__device__ __forceinline__ void hand_grad(const float* n, const float* o, float g, float* d) {
  const float nrm = sqrtf(o[0] * o[0] + o[1] * o[1] + o[2] * o[2]);
  const float den = fmaxf(nrm, RG_NORMALIZE_EPS);
  const float dot = n[0] * (o[0] / den) + n[1] * (o[1] / den) + n[2] * (o[2] / den);
  if (!(dot >= 0.f)) return;
  if (nrm >= RG_NORMALIZE_EPS) {  // the norm's own gradient passes clamp_min where |o| >= eps
    const float nu = dot;  // n . u with u = o / |o|
    for (int c = 0; c < 3; c++) d[c] += g * (n[c] - nu * (o[c] / nrm)) / nrm;
  } else {
    for (int c = 0; c < 3; c++) d[c] += g * n[c] / den;
  }
}

// A^T y at vertex i for y_v = w(v) lap_v: y_i + sum over the transposed entries (v, w_vj) of i of w_vj y_v
__device__ __forceinline__ float3 lap_adjoint(const B2RRegs& r, const float* __restrict__ lap, const float* __restrict__ w,
                                              int i) {
  float x = w[i] * lap[3 * i], y = w[i] * lap[3 * i + 1], z = w[i] * lap[3 * i + 2];
  const int e1 = r.lapT_offsets[i + 1];
  for (int e = r.lapT_offsets[i]; e < e1; e++) {
    const int v = r.lapT_src[e];
    const float a = r.lapT_w[e] * w[v];
    x += a * lap[3 * v];
    y += a * lap[3 * v + 1];
    z += a * lap[3 * v + 2];
  }
  return make_float3(x, y, z);
}

__global__ void __launch_bounds__(RG_THREADS) regs_backward_kernel(const B2RRegs r, const RegsPtrs s,
                                                                   const float* __restrict__ dout,
                                                                   const B2RRegsGrads gr) {
  const float g0 = dout[0], g1 = dout[1], g2 = dout[2], g3 = dout[3], g4 = dout[4], g5 = dout[5], g6 = dout[6],
              g7 = dout[7];
  const float n3 = 3.f * (float)r.P;
  if (blockIdx.x == 0 && threadIdx.x < r.J) {
    const int j = threadIdx.x;
    const float cj = 2.f * dout[8] * r.joint_weight[j] / (3.f * (float)r.J), cs = dout[9] / (float)r.n_pairs;
    float d[3];
    for (int c = 0; c < 3; c++) d[c] = cj * (r.joint_offset[3 * j + c] - r.joint_target[3 * j + c]);
    for (int q = 0; q < r.n_pairs; q++) {  // pairs in table order: one fixed sum per joint
      const int a = r.sym_pairs[2 * q], b = r.sym_pairs[2 * q + 1];
      if (a != j && b != j) continue;
      const float* ja = r.joint_offset + 3 * a;
      const float* jb = r.joint_offset + 3 * b;
      const float e[3] = {ja[0] + jb[0], ja[1] - jb[1], ja[2] - jb[2]};
      for (int c = 0; c < 3; c++) {
        const float sg = (float)((e[c] > 0.f) - (e[c] < 0.f));  // sign(0) = 0, as abs's gradient
        if (a == j) d[c] += cs * sg;
        if (b == j) d[c] += cs * (c == 0 ? sg : -sg);
      }
    }
    for (int c = 0; c < 3; c++) gr.joint_offset[3 * j + c] = d[c];
  }
  const int v = blockIdx.x * RG_THREADS + threadIdx.x;
  if (v >= r.P) return;
  const size_t P = (size_t)r.P;
  const float* W = r.weights;
  const float w1 = W[v], w2 = W[P + v];
  const float* L = s.lap;
  const float* lap_of[6] = {L, L + 3 * P, L + 6 * P, L + 9 * P, L + 12 * P, L + 15 * P};
  const float c3 = 2.f * g3 * 100000.f / n3, c4 = 2.f * g4 * 100000.f / n3, c5 = 2.f * g5 / n3;
  const float3 a1 = lap_adjoint(r, lap_of[0], W + 2 * P, v), a2 = lap_adjoint(r, lap_of[1], W + 2 * P, v);
  const float3 a3 = lap_adjoint(r, lap_of[2], W + 3 * P, v), a4 = lap_adjoint(r, lap_of[3], W + 3 * P, v);
  const float3 a5 = lap_adjoint(r, lap_of[4], W + 4 * P, v), a6 = lap_adjoint(r, lap_of[5], W + 4 * P, v);
  float dmo[3] = {c3 * (a1.x + a2.x), c3 * (a1.y + a2.y), c3 * (a1.z + a2.z)};
  float dmoo[3] = {c3 * a2.x, c3 * a2.y, c3 * a2.z};
  float dsc[3] = {c4 * a3.x, c4 * a3.y, c4 * a3.z};
  const float dsr[3] = {c4 * a4.x, c4 * a4.y, c4 * a4.z};
  float drgb[3] = {c5 * a5.x, c5 * a5.y, c5 * a5.z};
  float drgbr[3] = {c5 * a6.x, c5 * a6.y, c5 * a6.z};
  const float c0 = 2.f * g0 * w1 / n3, c2 = 2.f * g2 * w2 / n3;
  float mo[3], moo[3];
  for (int c = 0; c < 3; c++) {
    mo[c] = r.mean_offset[3 * v + c];
    moo[c] = r.mean_offset_offset[3 * v + c];
    dmo[c] += c0 * mo[c];
    dmoo[c] += c0 * moo[c];
  }
  const float so = r.scale_offset[v];
  gr.scale_offset[v] = 3.f * c2 * so;
  if (r.scale_reg) {  // the warm-up's scale_wo_clamp carries gaussian_scale_reg; `scale` keeps lap_scale only
    for (int c = 0; c < 3; c++) gr.scale_reg[3 * v + c] = c2 * r.scale_reg[3 * v + c];
  } else {
    for (int c = 0; c < 3; c++) dsc[c] += c2 * r.scale[3 * v + c];
  }
  const uint8_t h = r.hand[v];
  if (h) {
    const float* n = s.normals + 3 * v;
    const float gh = g1 / (float)r.n_hand;
    hand_grad(n, mo, gh, dmo);
    hand_grad(n, moo, gh, dmoo);
    const float ch = 2.f * g6 * 0.01f / (3.f * (float)r.n_rhand);
    for (int hand = 0; hand < 2; hand++) {
      if (!((h >> hand) & 1)) continue;
      for (int c = 0; c < 3; c++) {
        drgb[c] += ch * (r.rgb[3 * v + c] - s.hand_mean[hand * 3 + c]);
        drgbr[c] += ch * (r.rgb_refined[3 * v + c] - s.hand_mean[6 + hand * 3 + c]);
      }
    }
  }
  const int slot = r.arm_slot[v];
  if (slot >= 0) {
    const int p = s.arm_lo[slot];
    if (p >= 0) {  // a lower arm row: its targets are detached
      const float ca = 2.f * g7 * 0.1f / (3.f * (float)s.counters[1]);
      for (int c = 0; c < 3; c++) {
        drgb[c] += ca * (r.rgb[3 * v + c] - s.arm_tgt[6 * p + c]);
        drgbr[c] += ca * (r.rgb_refined[3 * v + c] - s.arm_tgt[6 * p + 3 + c]);
      }
    }
  }
  for (int c = 0; c < 3; c++) {
    gr.mean_offset[3 * v + c] = dmo[c];
    gr.mean_offset_offset[3 * v + c] = dmoo[c];
    gr.scale[3 * v + c] = dsc[c];
    gr.scale_refined[3 * v + c] = dsr[c];
    gr.rgb[3 * v + c] = drgb[c];
    gr.rgb_refined[3 * v + c] = drgbr[c];
  }
}

size_t regs_scratch_bytes(int P, int n_arm) { return regs_layout(P, n_arm).total; }

int launch_regs_forward(const B2RRegs& r, float* out, void* scratch, cudaStream_t st) {
  const RegsLayout L = regs_layout(r.P, r.n_arm);
  const RegsPtrs s = regs_ptrs(r, scratch);
  int rc = launch_vertex_normals(r.P, r.mesh, r.faces, r.vf_offsets, r.vf_entries, nullptr, s.normals, st);
  if (rc) return rc;
  const int cap = r.n_arm > 0 ? r.n_arm : 1;
  const int tiles = (cap + RG_THREADS - 1) / RG_THREADS;
  {
    ProfScope p(K_MISC, st);
    launch_k(regs_hand_partial_kernel, RG_HAND_BLOCKS, RG_THREADS, 0, st, true, r, s.hand_part);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(regs_split_kernel, 1, RG_SPLIT_THREADS, 0, st, true, r, s);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(regs_rank_kernel, dim3(tiles, tiles), RG_THREADS, 0, st, true, s);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(regs_scatter_kernel, tiles, RG_THREADS, 0, st, true, r, s);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(regs_window_kernel, tiles, RG_THREADS, 0, st, true, r, s);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(regs_select_kernel, (cap + RG_THREADS / 32 - 1) / (RG_THREADS / 32), RG_THREADS, 0, st, true, r, s);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(regs_terms_kernel, L.nb, RG_THREADS, 0, st, true, r, s);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(regs_reduce_kernel, 1, RG_THREADS, 0, st, true, r, s, L.nb, out);
  }
  return check_launch();
}

int launch_regs_backward(const B2RRegs& r, const float* dout, const B2RRegsGrads& g, const void* scratch,
                         cudaStream_t st) {
  const RegsLayout L = regs_layout(r.P, r.n_arm);
  const RegsPtrs s = regs_ptrs(r, const_cast<void*>(scratch));
  const int nb = max(L.nb, (r.J + RG_THREADS - 1) / RG_THREADS);
  ProfScope p(K_MISC, st);
  launch_k(regs_backward_kernel, nb, RG_THREADS, 0, st, true, r, s, dout, g);
  return check_launch();
}

}  // namespace b2r
