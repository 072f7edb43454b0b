// gn_mlp.cu -- ExAvatar's GroupNorm MLP stacks (avatar/common/nets/layer.py make_linear_layers(use_gn=True), used by
// HumanGaussian's geo / geo_offset / rgb / rgb_offset networks) on the tensor cores:
//   z_l = a_{l-1} W_l^T + b_l,  a_l = relu(GroupNorm(4, 128)(z_l))  for l = 0, 1, 2;  out = a_2 Wh^T + bh  (H <= 4).
//
// Arithmetic: every product of the three 128-wide layers goes through mma.sync.m16n8k8 TF32 as 3xTF32 -- each fp32
// operand x is split into hi = tf32(x) and lo = tf32(x - hi) and a.b is accumulated as a_lo b_hi + a_hi b_lo + a_hi b_hi
// (the lo.lo term, below 2^-22 |a b|, is dropped) -- so the layers are fp32-accurate, not TF32-accurate.
//
// Forward (gn_mlp_fwd_kernel): persistent CTAs hold W_0..W_2 in shared memory (3 x 68 KB); each warp runs whole 16-row
// tiles through all layers with the activations in registers.  The accumulator fragment of one layer is the A fragment
// of the next under the k-permutation {t -> 2t, t + 4 -> 2t + 1} inside each 8-column block, which the B fragment loads
// mirror, so no activation is moved between layers.  GroupNorm statistics come from quad shuffles (a 32-column group of
// a row lives in the 4 lanes of a quad).  With `saved` the pre-GN z_l are written for the backward (3 x P x 128 fp32).
//
// Backward:
//   gn_mlp_bwd_chain_kernel  per 16-row tile, from the saved z_l: GN / ReLU recomputed, dz_l through the chain
//                            (da_{l-1} = dz_l W_l on the tensor cores, W_1 and W_2 transposed in shared memory), dz_l and
//                            a_0, a_1 written out; dgamma, dbeta, dWh (fp32) and db, dbh (fp64) summed into per-warp
//                            shared partials, the warps added in order into one partial per CTA.
//   gn_mlp_dx_kernel         dX = dz_0 W_0 (only when a per-row input block needs its gradient).
//   gn_mlp_dw_kernel         dW_l = dz_l^T a_{l-1} (a_{-1} = X) over fixed 1024-row chunks, one partial per chunk.
//   gn_mlp_reduce_kernel     every gradient summed over its partials in a fixed order (runs, then a binary tree).
// No float atomics anywhere: two runs are bit-identical.  Nothing is allocated and the host reads no device data.
#include "common.cuh"

namespace b2r {

constexpr int GN_W = 128;           // hidden width
constexpr int GN_LD = 136;          // shared row stride in floats: conflict-free float2 B-fragment and A-column loads
constexpr int GN_WARPS = 8;
constexpr int GN_THREADS = GN_WARPS * 32;
constexpr int GN_CTAS = 132;        // persistent CTAs; fixed, so the partials and their sum order do not depend on the GPU
constexpr int GN_CHUNK = 1024;      // rows per weight-gradient partial
constexpr int GN_STAGE = 32;        // rows staged in shared memory per step of gn_mlp_dw_kernel
constexpr int GN_HMAX = 4;
// per-CTA partials of the chain kernel, fp32: dgamma[3][128] | dbeta[3][128] | dWh[4][128]; fp64: db[3][128] | dbh[4].
// The bias gradients are plain sums of dL/dz (dL/dout) over the rows, where large terms of both signs cancel: their
// partials are kept in double so the result does not depend on the order of the cancellation.
constexpr int GN_ACC_DGAMMA = 0, GN_ACC_DBETA = 3 * GN_W, GN_ACC_DWH = 6 * GN_W, GN_ACC = GN_ACC_DWH + GN_HMAX * GN_W;
constexpr int GN_ACCD_DB = 0, GN_ACCD_DBH = 3 * GN_W, GN_ACCD = GN_ACCD_DBH + GN_HMAX;
constexpr float GN_EPS = 1e-5f;

struct GnScratch {
  size_t dz, act, pchain, pchain_d, pw, total;
};
inline int gn_chunks(int P) { return (P + GN_CHUNK - 1) / GN_CHUNK; }
inline GnScratch gn_scratch_layout(int P) {
  GnScratch L;
  size_t o = 0;
  const size_t rows = (size_t)(P > 0 ? P : 1) * GN_W * sizeof(float);
  L.dz = o; o += align_up(3 * rows);
  L.act = o; o += align_up(2 * rows);
  L.pchain = o; o += align_up((size_t)GN_CTAS * GN_ACC * sizeof(float));
  L.pchain_d = o; o += align_up((size_t)GN_CTAS * GN_ACCD * sizeof(double));
  L.pw = o; o += align_up((size_t)3 * (gn_chunks(P) > 0 ? gn_chunks(P) : 1) * GN_W * GN_W * sizeof(float));
  L.total = o;
  return L;
}

__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = to_tf32(x);
  lo = to_tf32(x - __uint_as_float(hi));
}
// d += a.b as 3xTF32: the two small cross terms first, then the large one, into a zeroed fragment that is then added
// to d in fp32 with round-to-nearest.  The tensor core's own accumulation does not round to nearest; chained over
// every k-step of a layer (or over the rows of a weight gradient) its error would grow with the chain and exceed the
// fp32 GEMM's.
__device__ __forceinline__ void mma3(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], float b0, float b1) {
  uint32_t bh0, bl0, bh1, bl1;
  split_tf32(b0, bh0, bl0);
  split_tf32(b1, bh1, bl1);
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  mma_tf32(s, al, bh0, bh1);
  mma_tf32(s, ah, bl0, bl1);
  mma_tf32(s, ah, bh0, bh1);
#pragma unroll
  for (int i = 0; i < 4; i++) d[i] += s[i];
}

// acc[j] (16 x 8 block j of a 16 x 8nt tile) += A (16 x 8) B_j over one k-step.  `a` holds the A fragment under the
// permutation: a[0] / a[1] = rows g / g + 8 at column k0 + 2t, a[2] / a[3] the same rows at k0 + 2t + 1.  B_j[k][n] is
// M[(8j + n) * GN_LD + k] (M stored [n][k]); the float2 at column k0 + 2t serves both halves of the permuted k.
template <int NT>
__device__ __forceinline__ void mma_step(float (&acc)[NT][4], const float (&a)[4], const float* __restrict__ M, int k0,
                                         int nt, int g, int t) {
  uint32_t ah[4], al[4];
#pragma unroll
  for (int i = 0; i < 4; i++) split_tf32(a[i], ah[i], al[i]);
#pragma unroll
  for (int j = 0; j < NT; j++) {
    if (j < nt) {
      const float2 b = *reinterpret_cast<const float2*>(M + (8 * j + g) * GN_LD + k0 + 2 * t);
      mma3(acc[j], ah, al, b.x, b.y);
    }
  }
}

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// GroupNorm(4, 128) statistics of a 16 x 128 accumulator tile: mean / rstd of row g (s = 0) and g + 8 (s = 1) in group
// q.  Each sum is a balanced tree over 2^5 values, so a group of equal values has exactly that value as its mean and a
// variance of exactly 0 (rstd = 1 / sqrt(eps), as the reference's Welford update gives).
__device__ __forceinline__ void gn_stats(const float (&v)[16][4], float (&mean)[2][4], float (&rstd)[2][4]) {
#pragma unroll
  for (int s = 0; s < 2; s++) {
#pragma unroll
    for (int q = 0; q < 4; q++) {
      float p[4];
#pragma unroll
      for (int jj = 0; jj < 4; jj++) p[jj] = v[4 * q + jj][2 * s] + v[4 * q + jj][2 * s + 1];
      const float m = quad_sum((p[0] + p[1]) + (p[2] + p[3])) * (1.f / 32.f);
#pragma unroll
      for (int jj = 0; jj < 4; jj++) {
        const float d0 = v[4 * q + jj][2 * s] - m, d1 = v[4 * q + jj][2 * s + 1] - m;
        p[jj] = d0 * d0 + d1 * d1;
      }
      const float var = quad_sum((p[0] + p[1]) + (p[2] + p[3])) * (1.f / 32.f);
      mean[s][q] = m;
      rstd[s][q] = rsqrtf(var + GN_EPS);
    }
  }
}

// the GroupNorm affine of one normalised value: the forward and the backward's recomputation use this expression
__device__ __forceinline__ float gn_affine(float zhat, float gam, float bet) { return zhat * gam + bet; }

// Sums f(j, i) of a C-fragment tile over its 16 rows and adds the column sums to acc[0..128) (lanes 0..3 write, in
// tile order: deterministic).
template <class F, class T>
__device__ __forceinline__ void col_sums_add(F f, T* acc, int g, int t) {
#pragma unroll
  for (int j = 0; j < 16; j++) {
    float s0 = f(j, 0) + f(j, 2), s1 = f(j, 1) + f(j, 3);
#pragma unroll
    for (int d = 4; d < 32; d <<= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, d);
      s1 += __shfl_xor_sync(0xffffffffu, s1, d);
    }
    if (g == 0) {
      acc[8 * j + 2 * t] += s0;
      acc[8 * j + 2 * t + 1] += s1;
    }
  }
}

// rows ra (s = 0) and rb (s = 1) of a (P,128) fp32 array into / out of the C-fragment layout
__device__ __forceinline__ void load_tile(float (&v)[16][4], const float* __restrict__ src, int ra, int rb, bool va,
                                          bool vb, int t) {
#pragma unroll
  for (int j = 0; j < 16; j++) {
    const float2 x = va ? *reinterpret_cast<const float2*>(src + (size_t)ra * GN_W + 8 * j + 2 * t) : make_float2(0.f, 0.f);
    const float2 y = vb ? *reinterpret_cast<const float2*>(src + (size_t)rb * GN_W + 8 * j + 2 * t) : make_float2(0.f, 0.f);
    v[j][0] = x.x; v[j][1] = x.y; v[j][2] = y.x; v[j][3] = y.y;
  }
}
__device__ __forceinline__ void store_tile(const float (&v)[16][4], float* __restrict__ dst, int ra, int rb, bool va,
                                           bool vb, int t) {
#pragma unroll
  for (int j = 0; j < 16; j++) {
    if (va) *reinterpret_cast<float2*>(dst + (size_t)ra * GN_W + 8 * j + 2 * t) = make_float2(v[j][0], v[j][1]);
    if (vb) *reinterpret_cast<float2*>(dst + (size_t)rb * GN_W + 8 * j + 2 * t) = make_float2(v[j][2], v[j][3]);
  }
}

size_t gn_fwd_smem() { return ((size_t)3 * GN_W * GN_LD + 9 * GN_W + GN_HMAX * GN_W + GN_HMAX) * sizeof(float); }

__global__ void __launch_bounds__(GN_THREADS, 1) gn_mlp_fwd_kernel(const B2RGnMlp m, float* __restrict__ out,
                                                                   float* __restrict__ saved) {
  extern __shared__ float4 gn_smem4[];
  float* Ws = reinterpret_cast<float*>(gn_smem4);  // W_l [o][i], stride GN_LD
  float* bs = Ws + 3 * GN_W * GN_LD;                // b[3][128]
  float* gs = bs + 3 * GN_W;                        // gamma[3][128]
  float* es = gs + 3 * GN_W;                        // beta[3][128]
  float* hs = es + 3 * GN_W;                        // w_head[4][128], zero rows past H
  float* hb = hs + GN_HMAX * GN_W;                  // b_head[4]
  const int tid = threadIdx.x, P = m.P, K = m.K, H = m.H;
  for (int e = tid; e < GN_W * GN_W; e += GN_THREADS) {
    const int o = e >> 7, i = e & 127;
    Ws[o * GN_LD + i] = i < K ? m.w[0][o * K + i] : 0.f;
    Ws[GN_W * GN_LD + o * GN_LD + i] = m.w[1][e];
    Ws[2 * GN_W * GN_LD + o * GN_LD + i] = m.w[2][e];
  }
  for (int e = tid; e < 3 * GN_W; e += GN_THREADS) {
    const int l = e >> 7, c = e & 127;
    bs[e] = m.b[l][c];
    gs[e] = m.gamma[l][c];
    es[e] = m.beta[l][c];
  }
  for (int e = tid; e < GN_HMAX * GN_W; e += GN_THREADS) hs[e] = (e >> 7) < H ? m.w_head[e] : 0.f;
  if (tid < GN_HMAX) hb[tid] = tid < H ? m.b_head[tid] : 0.f;
  __syncthreads();

  const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int ntile = (P + 15) / 16, KT = (K + 7) / 8;
  for (int tile = blockIdx.x * GN_WARPS + warp; tile < ntile; tile += gridDim.x * GN_WARPS) {
    const int ra = tile * 16 + g, rb = ra + 8;
    const bool va = ra < P, vb = rb < P;
    float h[16][4], acc[16][4];
#pragma unroll
    for (int j = 0; j < 16; j++) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    for (int kk = 0; kk < KT; kk++) {
      const int c0 = 8 * kk + 2 * t, c1 = c0 + 1;
      float a[4];
      a[0] = va && c0 < K ? __ldg(m.x + (size_t)ra * K + c0) : 0.f;
      a[1] = vb && c0 < K ? __ldg(m.x + (size_t)rb * K + c0) : 0.f;
      a[2] = va && c1 < K ? __ldg(m.x + (size_t)ra * K + c1) : 0.f;
      a[3] = vb && c1 < K ? __ldg(m.x + (size_t)rb * K + c1) : 0.f;
      mma_step<16>(acc, a, Ws, 8 * kk, 16, g, t);
    }
#pragma unroll 1
    for (int l = 0; l < 3; l++) {
      if (l > 0) {
#pragma unroll
        for (int j = 0; j < 16; j++) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
        const float* Wl = Ws + l * GN_W * GN_LD;
#pragma unroll
        for (int kk = 0; kk < 16; kk++) {
          const float a[4] = {h[kk][0], h[kk][2], h[kk][1], h[kk][3]};
          mma_step<16>(acc, a, Wl, 8 * kk, 16, g, t);
        }
      }
      const float* bl = bs + l * GN_W;
#pragma unroll
      for (int j = 0; j < 16; j++) {
        const float b0 = bl[8 * j + 2 * t], b1 = bl[8 * j + 2 * t + 1];
        acc[j][0] += b0; acc[j][1] += b1; acc[j][2] += b0; acc[j][3] += b1;
      }
      if (saved) store_tile(acc, saved + (size_t)l * P * GN_W, ra, rb, va, vb, t);
      float mean[2][4], rstd[2][4];
      gn_stats(acc, mean, rstd);
      const float* gl = gs + l * GN_W;
      const float* el = es + l * GN_W;
#pragma unroll
      for (int j = 0; j < 16; j++) {
#pragma unroll
        for (int i = 0; i < 4; i++) {
          const int c = 8 * j + 2 * t + (i & 1), s = i >> 1;
          h[j][i] = fmaxf(gn_affine((acc[j][i] - mean[s][j >> 2]) * rstd[s][j >> 2], gl[c], el[c]), 0.f);
        }
      }
    }
#pragma unroll
    for (int hh = 0; hh < GN_HMAX; hh++) {
      if (hh < H) {
        float sa = 0.f, sb = 0.f;
#pragma unroll
        for (int j = 0; j < 16; j++) {
          const float w0 = hs[hh * GN_W + 8 * j + 2 * t], w1 = hs[hh * GN_W + 8 * j + 2 * t + 1];
          sa += h[j][0] * w0 + h[j][1] * w1;
          sb += h[j][2] * w0 + h[j][3] * w1;
        }
        sa = quad_sum(sa);
        sb = quad_sum(sb);
        if (t == 0) {
          if (va) out[(size_t)ra * H + hh] = sa + hb[hh];
          if (vb) out[(size_t)rb * H + hh] = sb + hb[hh];
        }
      }
    }
  }
}

size_t gn_chain_smem() {
  return (size_t)GN_WARPS * GN_ACCD * sizeof(double) +
         ((size_t)2 * GN_W * GN_LD + 6 * GN_W + GN_HMAX * GN_W + (size_t)GN_WARPS * GN_ACC) * sizeof(float);
}

__global__ void __launch_bounds__(GN_THREADS, 1) gn_mlp_bwd_chain_kernel(const B2RGnMlp m, const float* __restrict__ saved,
                                                                         const float* __restrict__ dout,
                                                                         float* __restrict__ dz_out,
                                                                         float* __restrict__ act_out,
                                                                         float* __restrict__ partial,
                                                                         double* __restrict__ partial_d) {
  extern __shared__ float4 gn_smem4[];
  double* accds = reinterpret_cast<double*>(gn_smem4);                   // [GN_WARPS][GN_ACCD]
  float* WT = reinterpret_cast<float*>(accds + GN_WARPS * GN_ACCD);     // W_1^T, W_2^T: [i][o], stride GN_LD
  float* gs = WT + 2 * GN_W * GN_LD;                // gamma[3][128]
  float* es = gs + 3 * GN_W;                        // beta[3][128]
  float* hs = es + 3 * GN_W;                        // w_head[4][128]
  float* accs = hs + GN_HMAX * GN_W;                // [GN_WARPS][GN_ACC]
  const int tid = threadIdx.x, P = m.P, H = m.H;
  for (int e = tid; e < GN_W * GN_W; e += GN_THREADS) {
    const int o = e >> 7, i = e & 127;
    WT[i * GN_LD + o] = m.w[1][e];
    WT[GN_W * GN_LD + i * GN_LD + o] = m.w[2][e];
  }
  for (int e = tid; e < 3 * GN_W; e += GN_THREADS) {
    gs[e] = m.gamma[e >> 7][e & 127];
    es[e] = m.beta[e >> 7][e & 127];
  }
  for (int e = tid; e < GN_HMAX * GN_W; e += GN_THREADS) hs[e] = (e >> 7) < H ? m.w_head[e] : 0.f;
  for (int e = tid; e < GN_WARPS * GN_ACC; e += GN_THREADS) accs[e] = 0.f;
  for (int e = tid; e < GN_WARPS * GN_ACCD; e += GN_THREADS) accds[e] = 0.0;
  __syncthreads();

  const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  float* acc_w = accs + warp * GN_ACC;
  double* accd_w = accds + warp * GN_ACCD;
  const int ntile = (P + 15) / 16;
  for (int tile = blockIdx.x * GN_WARPS + warp; tile < ntile; tile += gridDim.x * GN_WARPS) {
    const int ra = tile * 16 + g, rb = ra + 8;
    const bool va = ra < P, vb = rb < P;
    float d[16][4], v[16][4];
#pragma unroll 1
    for (int l = 2; l >= 0; l--) {
      load_tile(v, saved + (size_t)l * P * GN_W, ra, rb, va, vb, t);
      float mean[2][4], rstd[2][4];
      gn_stats(v, mean, rstd);
#pragma unroll
      for (int j = 0; j < 16; j++)
#pragma unroll
        for (int i = 0; i < 4; i++) v[j][i] = (v[j][i] - mean[i >> 1][j >> 2]) * rstd[i >> 1][j >> 2];  // zhat
      const float* gl = gs + l * GN_W;
      const float* el = es + l * GN_W;
      auto act = [&](int j, int i) {
        const int c = 8 * j + 2 * t + (i & 1);
        return fmaxf(gn_affine(v[j][i], gl[c], el[c]), 0.f);
      };
      if (l == 2) {  // head: dbh, dWh, and da_2 = dout Wh (dL/dout is live in this branch only)
        float go[2][GN_HMAX];  // dL/dout of rows ra, rb (0 past P or H)
#pragma unroll
        for (int hh = 0; hh < GN_HMAX; hh++) {
          go[0][hh] = va && hh < H ? dout[(size_t)ra * H + hh] : 0.f;
          go[1][hh] = vb && hh < H ? dout[(size_t)rb * H + hh] : 0.f;
          float s = go[0][hh] + go[1][hh];
#pragma unroll
          for (int dd = 4; dd < 32; dd <<= 1) s += __shfl_xor_sync(0xffffffffu, s, dd);
          if (lane == 0) accd_w[GN_ACCD_DBH + hh] += (double)s;
        }
#pragma unroll
        for (int hh = 0; hh < GN_HMAX; hh++) {
          if (hh < H)
            col_sums_add([&](int j, int i) { return go[i >> 1][hh] * act(j, i); }, acc_w + GN_ACC_DWH + hh * GN_W, g,
                         t);
        }
#pragma unroll
        for (int j = 0; j < 16; j++) {
#pragma unroll
          for (int i = 0; i < 4; i++) {
            const int c = 8 * j + 2 * t + (i & 1);
            float s = 0.f;
#pragma unroll
            for (int hh = 0; hh < GN_HMAX; hh++) s += go[i >> 1][hh] * hs[hh * GN_W + c];
            d[j][i] = s;
          }
        }
      } else {
        float* dst = act_out + (size_t)l * P * GN_W;
#pragma unroll
        for (int j = 0; j < 16; j++) {
          if (va) *reinterpret_cast<float2*>(dst + (size_t)ra * GN_W + 8 * j + 2 * t) = make_float2(act(j, 0), act(j, 1));
          if (vb) *reinterpret_cast<float2*>(dst + (size_t)rb * GN_W + 8 * j + 2 * t) = make_float2(act(j, 2), act(j, 3));
        }
      }
      // ReLU (relu'(0) = 0) and the affine
#pragma unroll
      for (int j = 0; j < 16; j++)
#pragma unroll
        for (int i = 0; i < 4; i++) {
          const int c = 8 * j + 2 * t + (i & 1);
          if (!(gn_affine(v[j][i], gl[c], el[c]) > 0.f)) d[j][i] = 0.f;
        }
      col_sums_add([&](int j, int i) { return d[j][i] * v[j][i]; }, acc_w + GN_ACC_DGAMMA + l * GN_W, g, t);
      col_sums_add([&](int j, int i) { return d[j][i]; }, acc_w + GN_ACC_DBETA + l * GN_W, g, t);
      // GroupNorm backward: dz = rstd (dzhat - mean(dzhat) - zhat mean(dzhat zhat)) over the row's group
#pragma unroll
      for (int j = 0; j < 16; j++)
#pragma unroll
        for (int i = 0; i < 4; i++) d[j][i] *= gl[8 * j + 2 * t + (i & 1)];
#pragma unroll
      for (int s = 0; s < 2; s++) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
          float p1[4], p2[4];
#pragma unroll
          for (int jj = 0; jj < 4; jj++) {
            const int j = 4 * q + jj;
            p1[jj] = d[j][2 * s] + d[j][2 * s + 1];
            p2[jj] = d[j][2 * s] * v[j][2 * s] + d[j][2 * s + 1] * v[j][2 * s + 1];
          }
          const float m1 = quad_sum((p1[0] + p1[1]) + (p1[2] + p1[3])) * (1.f / 32.f);
          const float m2 = quad_sum((p2[0] + p2[1]) + (p2[2] + p2[3])) * (1.f / 32.f);
#pragma unroll
          for (int jj = 0; jj < 4; jj++) {
            const int j = 4 * q + jj;
            d[j][2 * s] = rstd[s][q] * (d[j][2 * s] - m1 - v[j][2 * s] * m2);
            d[j][2 * s + 1] = rstd[s][q] * (d[j][2 * s + 1] - m1 - v[j][2 * s + 1] * m2);
          }
        }
      }
      col_sums_add([&](int j, int i) { return d[j][i]; }, accd_w + GN_ACCD_DB + l * GN_W, g, t);
      store_tile(d, dz_out + (size_t)l * P * GN_W, ra, rb, va, vb, t);
      if (l > 0) {  // da_{l-1} = dz_l W_l
        float acc[16][4];
#pragma unroll
        for (int j = 0; j < 16; j++) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
        const float* Ml = WT + (l - 1) * GN_W * GN_LD;
#pragma unroll
        for (int kk = 0; kk < 16; kk++) {
          const float a[4] = {d[kk][0], d[kk][2], d[kk][1], d[kk][3]};
          mma_step<16>(acc, a, Ml, 8 * kk, 16, g, t);
        }
#pragma unroll
        for (int j = 0; j < 16; j++)
#pragma unroll
          for (int i = 0; i < 4; i++) d[j][i] = acc[j][i];
      }
    }
  }
  __syncthreads();
  for (int e = tid; e < GN_ACC; e += GN_THREADS) {
    float s = 0.f;
    for (int w = 0; w < GN_WARPS; w++) s += accs[w * GN_ACC + e];
    partial[(size_t)blockIdx.x * GN_ACC + e] = s;
  }
  for (int e = tid; e < GN_ACCD; e += GN_THREADS) {
    double s = 0.0;
    for (int w = 0; w < GN_WARPS; w++) s += accds[w * GN_ACCD + e];
    partial_d[(size_t)blockIdx.x * GN_ACCD + e] = s;
  }
}

size_t gn_dx_smem() { return (size_t)GN_W * GN_LD * sizeof(float); }

__global__ void __launch_bounds__(GN_THREADS, 1) gn_mlp_dx_kernel(const int P, const int K, const float* __restrict__ w0,
                                                                  const float* __restrict__ dz0, float* __restrict__ dx) {
  extern __shared__ float4 gn_smem4[];
  float* W0T = reinterpret_cast<float*>(gn_smem4);  // W_0^T [i][o], rows K.. zero
  const int tid = threadIdx.x;
  for (int e = tid; e < GN_W * GN_W; e += GN_THREADS) {
    const int i = e >> 7, o = e & 127;
    W0T[i * GN_LD + o] = i < K ? w0[o * K + i] : 0.f;
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int ntile = (P + 15) / 16, NT = (K + 7) / 8;
  for (int tile = blockIdx.x * GN_WARPS + warp; tile < ntile; tile += gridDim.x * GN_WARPS) {
    const int ra = tile * 16 + g, rb = ra + 8;
    const bool va = ra < P, vb = rb < P;
    float acc[16][4];
#pragma unroll
    for (int j = 0; j < 16; j++) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll 4
    for (int kk = 0; kk < 16; kk++) {
      const float2 x = va ? *reinterpret_cast<const float2*>(dz0 + (size_t)ra * GN_W + 8 * kk + 2 * t) : make_float2(0.f, 0.f);
      const float2 y = vb ? *reinterpret_cast<const float2*>(dz0 + (size_t)rb * GN_W + 8 * kk + 2 * t) : make_float2(0.f, 0.f);
      const float a[4] = {x.x, y.x, x.y, y.y};
      mma_step<16>(acc, a, W0T, 8 * kk, NT, g, t);
    }
#pragma unroll
    for (int j = 0; j < 16; j++) {
      const int c = 8 * j + 2 * t;
      if (j < NT) {
        if (va && c < K) dx[(size_t)ra * K + c] = acc[j][0];
        if (va && c + 1 < K) dx[(size_t)ra * K + c + 1] = acc[j][1];
        if (vb && c < K) dx[(size_t)rb * K + c] = acc[j][2];
        if (vb && c + 1 < K) dx[(size_t)rb * K + c + 1] = acc[j][3];
      }
    }
  }
}

// dW_l[o][i] = sum over the chunk's rows of dz_l[r][o] a_{l-1}[r][i]: M = o (16 per warp), N = i, K = rows
__global__ void __launch_bounds__(GN_THREADS) gn_mlp_dw_kernel(const int P, const int K, const float* __restrict__ x,
                                                               const float* __restrict__ dz,
                                                               const float* __restrict__ act, float* __restrict__ pw) {
  __shared__ __align__(16) float zs[GN_STAGE * GN_LD];
  __shared__ __align__(16) float as[GN_STAGE * GN_LD];
  const int L = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
  const float* A = dz + (size_t)L * P * GN_W;
  const float* B = L == 0 ? x : act + (size_t)(L - 1) * P * GN_W;
  const int KB = L == 0 ? K : GN_W, NT = (KB + 7) / 8;
  const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3, o0 = warp * 16;
  float acc[16][4];
#pragma unroll
  for (int j = 0; j < 16; j++) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  const int r_end = min(P, (chunk + 1) * GN_CHUNK);
  for (int r0 = chunk * GN_CHUNK; r0 < r_end; r0 += GN_STAGE) {
    __syncthreads();
    for (int e = tid; e < GN_STAGE * GN_W; e += GN_THREADS) {
      const int r = e >> 7, c = e & 127, rr = r0 + r;
      zs[r * GN_LD + c] = rr < r_end ? A[(size_t)rr * GN_W + c] : 0.f;
      as[r * GN_LD + c] = rr < r_end && c < KB ? B[(size_t)rr * KB + c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k0 = 0; k0 < GN_STAGE; k0 += 8) {
      const float a[4] = {zs[(k0 + t) * GN_LD + o0 + g], zs[(k0 + t) * GN_LD + o0 + g + 8],
                          zs[(k0 + t + 4) * GN_LD + o0 + g], zs[(k0 + t + 4) * GN_LD + o0 + g + 8]};
      uint32_t ah[4], al[4];
#pragma unroll
      for (int i = 0; i < 4; i++) split_tf32(a[i], ah[i], al[i]);
#pragma unroll
      for (int j = 0; j < 16; j++)
        if (j < NT) mma3(acc[j], ah, al, as[(k0 + t) * GN_LD + 8 * j + g], as[(k0 + t + 4) * GN_LD + 8 * j + g]);
    }
  }
  float* dst = pw + ((size_t)L * gridDim.x + chunk) * GN_W * GN_W;
#pragma unroll
  for (int j = 0; j < 16; j++) {
    const int c = 8 * j + 2 * t;
    *reinterpret_cast<float2*>(dst + (o0 + g) * GN_W + c) = make_float2(acc[j][0], acc[j][1]);
    *reinterpret_cast<float2*>(dst + (o0 + g + 8) * GN_W + c) = make_float2(acc[j][2], acc[j][3]);
  }
}

// sum of p[0], p[stride], ..., p[(n-1) stride] in a fixed order: at most 32 runs of consecutive terms added in order,
// the run sums added as a binary tree, so the rounding error grows with n / 32 + log2(32) additions instead of n
template <class T>
__device__ T pairwise_sum(const T* __restrict__ p, int n, size_t stride) {
  T run[32];
  const int len = max(8, (n + 31) / 32);
  int nr = 0;
  for (int c0 = 0; c0 < n; c0 += len) {
    T s = 0;
    for (int c = c0; c < min(n, c0 + len); c++) s += p[(size_t)c * stride];
    run[nr++] = s;
  }
  for (int w = 1; w < nr; w <<= 1)
    for (int i = 0; i + w < nr; i += 2 * w) run[i] += run[i + w];
  return nr ? run[0] : T(0);
}

// grads = [dW_0 (128,K) | dW_1 | dW_2 (128,128) | dgamma (3,128) | dbeta (3,128) | db (3,128) | dWh (H,128) | dbh (H)]
__global__ void gn_mlp_reduce_kernel(const int K, const int H, const int nchunk, const float* __restrict__ pw,
                                     const float* __restrict__ pchain, const double* __restrict__ pchain_d,
                                     float* __restrict__ grads) {
  const int n_w = GN_W * K + 2 * GN_W * GN_W, n_all = n_w + 9 * GN_W + H * GN_W + H;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_all) return;
  if (e < n_w) {
    int L, o, i;
    if (e < GN_W * K) { L = 0; o = e / K; i = e % K; }
    else { const int f = e - GN_W * K; L = 1 + f / (GN_W * GN_W); o = (f / GN_W) % GN_W; i = f % GN_W; }
    grads[e] = pairwise_sum(pw + (size_t)L * nchunk * GN_W * GN_W + o * GN_W + i, nchunk, (size_t)GN_W * GN_W);
  } else {
    // dgamma | dbeta (fp32 partials), db (fp64), dWh (fp32), dbh (fp64)
    const int f = e - n_w;
    if (f < 6 * GN_W) grads[e] = pairwise_sum(pchain + GN_ACC_DGAMMA + f, GN_CTAS, GN_ACC);
    else if (f < 9 * GN_W) grads[e] = (float)pairwise_sum(pchain_d + GN_ACCD_DB + (f - 6 * GN_W), GN_CTAS, GN_ACCD);
    else if (f < 9 * GN_W + H * GN_W) grads[e] = pairwise_sum(pchain + GN_ACC_DWH + (f - 9 * GN_W), GN_CTAS, GN_ACC);
    else grads[e] = (float)pairwise_sum(pchain_d + GN_ACCD_DBH + (f - 9 * GN_W - H * GN_W), GN_CTAS, GN_ACCD);
  }
}

size_t gn_mlp_scratch_bytes(int P) { return gn_scratch_layout(P).total; }
size_t gn_mlp_grads_count(int K, int H) { return (size_t)GN_W * K + 2 * GN_W * GN_W + 9 * GN_W + (size_t)H * GN_W + H; }

static int gn_ctas(int P) {
  const int tiles = (P + 15) / 16;
  return min(GN_CTAS, (tiles + GN_WARPS - 1) / GN_WARPS);
}

int launch_gn_mlp_forward(const B2RGnMlp& m, float* out, float* saved, cudaStream_t st) {
  ProfScope p(K_MISC, st);
  cudaFuncSetAttribute(gn_mlp_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gn_fwd_smem());
  launch_k(gn_mlp_fwd_kernel, gn_ctas(m.P), GN_THREADS, gn_fwd_smem(), st, false, m, out, saved);
  return check_launch();
}

int launch_gn_mlp_backward(const B2RGnMlp& m, const float* saved, const float* dout, float* dx, float* grads,
                           void* scratch, cudaStream_t st) {
  const GnScratch L = gn_scratch_layout(m.P);
  char* s = (char*)scratch;
  float* dz = (float*)(s + L.dz);
  float* act = (float*)(s + L.act);
  float* pchain = (float*)(s + L.pchain);
  double* pchain_d = (double*)(s + L.pchain_d);
  float* pw = (float*)(s + L.pw);
  const int nchunk = gn_chunks(m.P);
  {
    // every CTA of the fixed grid writes its partial, also those without a tile
    ProfScope p(K_MISC, st);
    cudaFuncSetAttribute(gn_mlp_bwd_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gn_chain_smem());
    launch_k(gn_mlp_bwd_chain_kernel, GN_CTAS, GN_THREADS, gn_chain_smem(), st, false, m, saved, dout, dz, act,
             pchain, pchain_d);
  }
  if (dx) {
    ProfScope p(K_MISC, st);
    cudaFuncSetAttribute(gn_mlp_dx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gn_dx_smem());
    launch_k(gn_mlp_dx_kernel, gn_ctas(m.P), GN_THREADS, gn_dx_smem(), st, false, m.P, m.K, m.w[0], (const float*)dz,
             dx);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(gn_mlp_dw_kernel, dim3(nchunk, 3), GN_THREADS, 0, st, false, m.P, m.K, m.x, (const float*)dz,
             (const float*)act, pw);
  }
  {
    ProfScope p(K_MISC, st);
    const int n = (int)gn_mlp_grads_count(m.K, m.H);
    launch_k(gn_mlp_reduce_kernel, (n + 255) / 256, 256, 0, st, false, m.K, m.H, nchunk, (const float*)pw,
             (const float*)pchain, (const double*)pchain_d, grads);
  }
  return check_launch();
}

}  // namespace b2r
