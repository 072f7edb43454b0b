// lpips.cu -- ExAvatar's perceptual terms (avatar/common/nets/loss.py LPIPS over lpips.LPIPS(net='vgg'), version 0.1,
// eval mode) for N images against one target, in an op that never reads the crop box on the host.
//
// Per image: crop [y0:y1, x0:x1] by l1_ssim's rules, x*2-1, ScalingLayer, VGG-16 features through relu5_3 with 3x3 zero
// padding at the CROP's border and 2x2 floor max pools, and per tap k (relu1_2, relu2_2, relu3_3, relu4_3, relu5_3)
//   L_k = mean_p sum_c w_kc (n_c(f_img) - n_c(f_tgt))^2,  n(f) = f / (sqrt(sum_c f_c^2) + 1e-10);   out = sum_k L_k.
//
// Static grids: every launch is sized from the image capacity W x H (level l has capacity (H >> l) x (W >> l)) and
// activations are stored relative to the crop origin, NHWC fp32 with row stride W >> l.  A CTA whose tile lies outside
// the level's valid extent ((y1 - y0) >> l) x ((x1 - x0) >> l), derived on the device from the box, exits.  Nothing
// reads outside a valid extent, so no buffer is cleared.
//   forward   target: conv1_1 (CUDA cores) and 12 implicit-GEMM convs (mma.sync m16n8k8 TF32) ping-ponging through the
//             scratch, each tap normalised into `saved`.  Each image: the same convs into `saved` (the 13 ReLU outputs
//             the backward masks with), the pools into the scratch, one head kernel per tap (fp64 per-CTA partials)
//             and one reduce (fixed order, divided by each tap's extent).
//   backward  per image, level 4 down to 0: one boundary kernel (the head gradient of the tap plus the max-pool gradient
//             of the level above, routed to the first maximum of its window, a gather) and the input gradients of the
//             level's convs -- the same GEMM kernel on flipped, transposed weights, its load masked by ReLU output > 0 --
//             then conv1_1's input gradient with the ScalingLayer's chain rule, zero outside the crop.
// No float atomics, no allocation, no host sync: bit-identical runs, CUDA-graph capturable.
#include "common.cuh"

namespace b2r {

constexpr float LP_EPS = 1e-10f;  // lpips normalize_tensor
__constant__ float c_lp_shift[3] = {-.030f, -.088f, -.188f};
__constant__ float c_lp_scale[3] = {.458f, .448f, .450f};

__host__ __device__ constexpr int lp_cout(int l) { return l < 2 ? 64 : l < 4 ? 128 : l < 7 ? 256 : 512; }
__host__ __device__ constexpr int lp_cin(int l) { return l == 0 ? 3 : lp_cout(l - 1); }
__host__ __device__ constexpr int lp_level(int l) { return l < 2 ? 0 : l < 4 ? 1 : l < 7 ? 2 : l < 10 ? 3 : 4; }
__host__ __device__ constexpr int lp_tap_layer(int t) { return t == 0 ? 1 : t == 1 ? 3 : 3 * t; }  // 1 3 6 9 12

struct LpExt {
  int h, w;
};
// valid extent of `level` for the box on the device
__device__ __forceinline__ LpExt lp_extent(const float* bbox, int W, int H, int level) {
  const Crop c = read_crop(bbox, W, H);
  return {(c.y1 - c.y0) >> level, (c.x1 - c.x0) >> level};
}

// ---------------------------------------------------------------------------------------------------------------------
// Buffer layouts.  saved: per image the 13 ReLU outputs, then the target's 5 normalised taps.  scratch: two ping-pong
// planes of 64 x H x W floats (target activations, then the backward's gradients; an image's pools), then the heads'
// fp64 per-CTA partials.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int HD_WARPS = 8, HD_PPW = 4, HD_PIX = HD_WARPS * HD_PPW;  // head kernels: a warp per pixel, 32 pixels a CTA

static size_t lp_plane(int W, int H, int level, int C) {
  return align_up((size_t)C * (size_t)(H >> level) * (size_t)(W >> level) * sizeof(float));
}
static int lp_head_ctas(int W, int H, int level) {
  return (int)(((size_t)(H >> level) * (size_t)(W >> level) + HD_PIX - 1) / HD_PIX);
}
struct LpSaved {
  size_t act[13], image, tap[5], total;
};
static LpSaved lp_saved_layout(int W, int H, int N) {
  LpSaved s;
  size_t o = 0;
  for (int l = 0; l < 13; l++) { s.act[l] = o; o += lp_plane(W, H, lp_level(l), lp_cout(l)); }
  s.image = o;
  o = (size_t)N * s.image;
  for (int t = 0; t < 5; t++) { s.tap[t] = o; o += lp_plane(W, H, t, lp_cout(lp_tap_layer(t))); }
  s.total = o;
  return s;
}
struct LpScratch {
  size_t a, b, part[5], total;
};
static LpScratch lp_scratch_layout(int W, int H) {
  LpScratch s;
  size_t o = 0;
  s.a = o; o += lp_plane(W, H, 0, 64);
  s.b = o; o += lp_plane(W, H, 0, 64);
  for (int t = 0; t < 5; t++) { s.part[t] = o; o += align_up((size_t)lp_head_ctas(W, H, t) * sizeof(double)); }
  s.total = o;
  return s;
}
size_t lpips_saved_bytes(int W, int H, int N) { return lp_saved_layout(W, H, N).total; }
size_t lpips_scratch_bytes(int W, int H) { return lp_scratch_layout(W, H).total; }

// ---------------------------------------------------------------------------------------------------------------------
// conv1_1 (C_in = 3) on the CUDA cores: x*2-1, ScalingLayer, 3x3 conv + bias, ReLU.  One thread per pixel, 64 outputs.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int C0_T = 16;
__global__ void __launch_bounds__(C0_T * C0_T) lp_conv0_fwd_kernel(const float* __restrict__ img, const float* bbox,
                                                                   int W, int H, const float* __restrict__ w,
                                                                   const float* __restrict__ bias,
                                                                   float* __restrict__ out) {
  __shared__ float sw[64 * 27], sb[64];
  const Crop cr = read_crop(bbox, W, H);
  const int h = cr.y1 - cr.y0, wd = cr.x1 - cr.x0;
  const int tx0 = blockIdx.x * C0_T, ty0 = blockIdx.y * C0_T;
  if (tx0 >= wd || ty0 >= h) return;  // block-uniform
  for (int e = threadIdx.x; e < 64 * 27; e += C0_T * C0_T) sw[e] = __ldg(w + e);
  if (threadIdx.x < 64) sb[threadIdx.x] = __ldg(bias + threadIdx.x);
  __syncthreads();
  const int x = tx0 + threadIdx.x % C0_T, y = ty0 + threadIdx.x / C0_T;
  if (x >= wd || y >= h) return;
  const size_t HW = (size_t)W * H;
  float in[27];  // [ci][ky][kx] of the scaled input, zero outside the crop
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int ky = 0; ky < 3; ky++)
#pragma unroll
      for (int kx = 0; kx < 3; kx++) {
        const int yy = y + ky - 1, xx = x + kx - 1;
        float v = 0.f;
        if (yy >= 0 && yy < h && xx >= 0 && xx < wd) {
          const float p = __ldg(img + c * HW + (size_t)(cr.y0 + yy) * W + cr.x0 + xx);
          v = ((p * 2.f - 1.f) - c_lp_shift[c]) / c_lp_scale[c];
        }
        in[(c * 3 + ky) * 3 + kx] = v;
      }
  float4* dst = reinterpret_cast<float4*>(out + ((size_t)y * W + x) * 64);
  for (int c4 = 0; c4 < 16; c4++) {
    float r[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const float* wc = sw + (4 * c4 + u) * 27;
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < 27; k++) s = fmaf(wc[k], in[k], s);
      r[u] = fmaxf(s + sb[4 * c4 + u], 0.f);
    }
    dst[c4] = make_float4(r[0], r[1], r[2], r[3]);
  }
}

// dL/dimg: conv1_1's input gradient (masked by relu1_1 > 0) times the chain rule 2 / scale_c.  Every pixel of the
// image is written: exact zeros outside the crop.
__global__ void __launch_bounds__(C0_T * C0_T) lp_conv0_bwd_kernel(const float* __restrict__ grad,
                                                                   const float* __restrict__ act, const float* bbox,
                                                                   int W, int H, const float* __restrict__ w,
                                                                   float* __restrict__ dimg) {
  __shared__ float sw[64 * 27];
  const Crop cr = read_crop(bbox, W, H);
  const int h = cr.y1 - cr.y0, wd = cr.x1 - cr.x0;
  for (int e = threadIdx.x; e < 64 * 27; e += C0_T * C0_T) sw[e] = __ldg(w + e);
  __syncthreads();
  const int px = blockIdx.x * C0_T + threadIdx.x % C0_T, py = blockIdx.y * C0_T + threadIdx.x / C0_T;
  if (px >= W || py >= H) return;
  const size_t HW = (size_t)W * H, o = (size_t)py * W + px;
  if (!cr.has(px, py)) {
    for (int c = 0; c < 3; c++) dimg[c * HW + o] = 0.f;
    return;
  }
  const int x = px - cr.x0, y = py - cr.y0;
  float d[3] = {0.f, 0.f, 0.f};
  for (int ky = 0; ky < 3; ky++)
    for (int kx = 0; kx < 3; kx++) {
      const int yy = y - ky + 1, xx = x - kx + 1;  // the output pixel this tap reads us from
      if (yy < 0 || yy >= h || xx < 0 || xx >= wd) continue;
      const float4* g4 = reinterpret_cast<const float4*>(grad + ((size_t)yy * W + xx) * 64);
      const float4* a4 = reinterpret_cast<const float4*>(act + ((size_t)yy * W + xx) * 64);
      for (int c4 = 0; c4 < 16; c4++) {
        const float4 g = __ldg(g4 + c4), a = __ldg(a4 + c4);
        const float gm[4] = {a.x > 0.f ? g.x : 0.f, a.y > 0.f ? g.y : 0.f, a.z > 0.f ? g.z : 0.f,
                             a.w > 0.f ? g.w : 0.f};
#pragma unroll
        for (int u = 0; u < 4; u++)
#pragma unroll
          for (int c = 0; c < 3; c++) d[c] = fmaf(sw[(4 * c4 + u) * 27 + (c * 3 + ky) * 3 + kx], gm[u], d[c]);
      }
    }
  for (int c = 0; c < 3; c++) dimg[c * HW + o] = d[c] / c_lp_scale[c] * 2.f;
}

// ---------------------------------------------------------------------------------------------------------------------
// 3x3 convolution as an implicit GEMM on the tensor cores: M = the 8 x 16 pixels of a tile, N = 64 output channels a CTA,
// K = 9 x C_in in stages of 8 channels.  Each stage puts the tile's input + 1-pixel halo (zero outside the valid extent)
// and the 9 x 8 x 64 weights in shared memory, rounded to TF32 (cvt.rna) once; a warp owns two tile rows (two m16
// tiles) and all eight n8 tiles.  Strides 12 and 72 words make the A and B fragment reads conflict-free.
//   FWD:  y = relu(conv(x, W) + b),                weights (3,3,C_in,C_out)
//   !FWD: y = conv(x * [mask > 0], W_flipped^T),   weights (3,3,C_out,C_in) -- the input gradient, with x the gradient
//         at this conv's output and mask its saved ReLU output (a select, as threshold_backward)
// ---------------------------------------------------------------------------------------------------------------------
constexpr int CV_TW = 16, CV_TH = 8, CV_N = 64, CV_KC = 8, CV_THREADS = 128;
constexpr int CV_HW = CV_TW + 2, CV_HH = CV_TH + 2;
constexpr int CV_IS = CV_KC + 4;  // words per staged pixel
constexpr int CV_WS = CV_N + 8;   // words per staged weight row

struct ConvArgs {
  const float* x;     // (h, w, K) NHWC
  const float* mask;  // !FWD: (h, w, K) saved ReLU output
  const float* wt;    // (9, K, N)
  const float* bias;  // FWD: (N)
  float* y;           // (h, w, N)
  const float* bbox;
  int W, H, level, K, N;
};

template <bool FWD>
__global__ void __launch_bounds__(CV_THREADS) lp_conv_kernel(const ConvArgs a) {
  __shared__ __align__(16) uint32_t s_in[CV_HH * CV_HW * CV_IS];
  __shared__ __align__(16) uint32_t s_w[9 * CV_KC * CV_WS];
  const LpExt ex = lp_extent(a.bbox, a.W, a.H, a.level);
  const int tx0 = blockIdx.x * CV_TW, ty0 = blockIdx.y * CV_TH, n0 = blockIdx.z * CV_N;
  if (tx0 >= ex.w || ty0 >= ex.h) return;  // block-uniform
  const int ld = a.W >> a.level;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  float acc[2][8][4];
#pragma unroll
  for (int j = 0; j < 2; j++)
#pragma unroll
    for (int n = 0; n < 8; n++) acc[j][n][0] = acc[j][n][1] = acc[j][n][2] = acc[j][n][3] = 0.f;

  for (int k0 = 0; k0 < a.K; k0 += CV_KC) {
    __syncthreads();  // the previous stage is consumed
    for (int e = threadIdx.x; e < CV_HH * CV_HW * 2; e += CV_THREADS) {
      const int p = e >> 1, q = e & 1;
      const int hy = p / CV_HW, hx = p - hy * CV_HW;
      const int gy = ty0 - 1 + hy, gx = tx0 - 1 + hx;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gy >= 0 && gy < ex.h && gx >= 0 && gx < ex.w) {
        const size_t o = ((size_t)gy * ld + gx) * a.K + k0 + 4 * q;
        v = __ldg(reinterpret_cast<const float4*>(a.x + o));
        if (!FWD) {
          const float4 m = __ldg(reinterpret_cast<const float4*>(a.mask + o));
          v.x = m.x > 0.f ? v.x : 0.f;
          v.y = m.y > 0.f ? v.y : 0.f;
          v.z = m.z > 0.f ? v.z : 0.f;
          v.w = m.w > 0.f ? v.w : 0.f;
        }
      }
      *reinterpret_cast<uint4*>(s_in + p * CV_IS + 4 * q) = make_uint4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z),
                                                                       to_tf32(v.w));
    }
    for (int e = threadIdx.x; e < 9 * CV_KC * (CV_N / 4); e += CV_THREADS) {
      const int r = e >> 4, c4 = e & 15;  // r = tap * 8 + k
      const int tap = r >> 3, k = r & 7;
      const float4 v = __ldg(reinterpret_cast<const float4*>(a.wt + ((size_t)tap * a.K + k0 + k) * a.N + n0 + 4 * c4));
      *reinterpret_cast<uint4*>(s_w + r * CV_WS + 4 * c4) = make_uint4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z),
                                                                       to_tf32(v.w));
    }
    __syncthreads();
#pragma unroll
    for (int tap = 0; tap < 9; tap++) {
      const int ky = tap / 3, kx = tap - 3 * (tap / 3);
      uint32_t af[2][4];
#pragma unroll
      for (int j = 0; j < 2; j++) {
        const uint32_t* p0 = s_in + ((2 * warp + j + ky) * CV_HW + g + kx) * CV_IS + t;
        const uint32_t* p1 = p0 + 8 * CV_IS;
        af[j][0] = p0[0];
        af[j][1] = p1[0];
        af[j][2] = p0[4];
        af[j][3] = p1[4];
      }
#pragma unroll
      for (int n = 0; n < 8; n++) {
        const uint32_t b0 = s_w[(tap * CV_KC + t) * CV_WS + 8 * n + g];
        const uint32_t b1 = s_w[(tap * CV_KC + t + 4) * CV_WS + 8 * n + g];
        mma_tf32(acc[0][n], af[0], b0, b1);
        mma_tf32(acc[1][n], af[1], b0, b1);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 2; j++) {
    const int py = ty0 + 2 * warp + j;
    if (py >= ex.h) continue;
#pragma unroll
    for (int half = 0; half < 2; half++) {
      const int px = tx0 + g + 8 * half;
      if (px >= ex.w) continue;
      float* dst = a.y + ((size_t)py * ld + px) * a.N + n0;
#pragma unroll
      for (int n = 0; n < 8; n++) {
        const int co = 8 * n + 2 * t;
        float v0 = acc[j][n][2 * half], v1 = acc[j][n][2 * half + 1];
        if (FWD) {
          v0 = fmaxf(v0 + __ldg(a.bias + n0 + co), 0.f);
          v1 = fmaxf(v1 + __ldg(a.bias + n0 + co + 1), 0.f);
        }
        *reinterpret_cast<float2*>(dst + co) = make_float2(v0, v1);
      }
    }
  }
}

// 2x2 stride-2 max pool with floor: level l - 1 -> l, one thread per (pixel, 4 channels)
__global__ void __launch_bounds__(256) lp_pool_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                      const float* bbox, int W, int H, int level, int C) {
  const LpExt ex = lp_extent(bbox, W, H, level);
  const int ldo = W >> level, ldi = W >> (level - 1), C4 = C / 4;
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= (size_t)(H >> level) * ldo * C4) return;
  const int c4 = (int)(i % C4);
  const int p = (int)(i / C4);
  const int y = p / ldo, x = p - y * ldo;
  if (y >= ex.h || x >= ex.w) return;
  const float4* s = reinterpret_cast<const float4*>(in) + ((size_t)(2 * y) * ldi + 2 * x) * C4 + c4;
  const float4 v[4] = {__ldg(s), __ldg(s + C4), __ldg(s + (size_t)ldi * C4), __ldg(s + (size_t)ldi * C4 + C4)};
  float4 m = v[0];
#pragma unroll
  for (int k = 1; k < 4; k++) {
    m.x = v[k].x > m.x ? v[k].x : m.x;
    m.y = v[k].y > m.y ? v[k].y : m.y;
    m.z = v[k].z > m.z ? v[k].z : m.z;
    m.w = v[k].w > m.w ? v[k].w : m.w;
  }
  reinterpret_cast<float4*>(out)[(size_t)p * C4 + c4] = m;
}

// ---------------------------------------------------------------------------------------------------------------------
// Heads: a warp per pixel, lane l holds channels 4 (l + 32 i) .. + 3.  Sums over channels are warp_sum (every lane ends
// with the same value).
// ---------------------------------------------------------------------------------------------------------------------
template <int C>
struct HeadVec {
  static constexpr int NV = C >= 128 ? C / 128 : 1;
  float4 v[NV];
  __device__ __forceinline__ void load(const float* p, int lane) {
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c4 = lane + 32 * i;
      v[i] = c4 < C / 4 ? __ldg(reinterpret_cast<const float4*>(p) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  __device__ __forceinline__ void store(float* p, int lane) const {
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c4 = lane + 32 * i;
      if (c4 < C / 4) reinterpret_cast<float4*>(p)[c4] = v[i];
    }
  }
};
template <int C>
__device__ __forceinline__ float sum_sq(const HeadVec<C>& f) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < HeadVec<C>::NV; i++) s += f.v[i].x * f.v[i].x + f.v[i].y * f.v[i].y + f.v[i].z * f.v[i].z + f.v[i].w * f.v[i].w;
  return warp_sum(s);
}

// the target's normalised tap
template <int C>
__global__ void __launch_bounds__(HD_WARPS * 32) lp_head_target_kernel(const float* __restrict__ f,
                                                                       float* __restrict__ nrm, const float* bbox,
                                                                       int W, int H, int level) {
  const LpExt ex = lp_extent(bbox, W, H, level);
  const int ld = W >> level, lane = threadIdx.x & 31;
  for (int k = 0; k < HD_PPW; k++) {
    const int p = blockIdx.x * HD_PIX + (threadIdx.x >> 5) * HD_PPW + k;
    const int y = p / ld, x = p - y * ld;
    if (y >= ex.h || x >= ex.w) continue;  // warp-uniform
    HeadVec<C> v;
    v.load(f + (size_t)p * C, lane);
    const float s = sqrtf(sum_sq(v)) + LP_EPS;
#pragma unroll
    for (int i = 0; i < HeadVec<C>::NV; i++) v.v[i] = make_float4(v.v[i].x / s, v.v[i].y / s, v.v[i].z / s, v.v[i].w / s);
    v.store(nrm + (size_t)p * C, lane);
  }
}

// sum over the CTA's pixels of sum_c w_c (n_c(f) - nt_c)^2, in fp64, into part[blockIdx.x]
template <int C>
__global__ void __launch_bounds__(HD_WARPS * 32) lp_head_fwd_kernel(const float* __restrict__ f,
                                                                    const float* __restrict__ nt,
                                                                    const float* __restrict__ lw,
                                                                    double* __restrict__ part, const float* bbox, int W,
                                                                    int H, int level) {
  __shared__ double wsum[HD_WARPS];
  const LpExt ex = lp_extent(bbox, W, H, level);
  const int ld = W >> level, lane = threadIdx.x & 31;
  HeadVec<C> w;
  w.load(lw, lane);
  double acc[1] = {0.0};
  for (int k = 0; k < HD_PPW; k++) {
    const int p = blockIdx.x * HD_PIX + (threadIdx.x >> 5) * HD_PPW + k;
    const int y = p / ld, x = p - y * ld;
    if (y >= ex.h || x >= ex.w) continue;  // warp-uniform
    HeadVec<C> v, n;
    v.load(f + (size_t)p * C, lane);
    n.load(nt + (size_t)p * C, lane);
    const float s = sqrtf(sum_sq(v)) + LP_EPS;
    float d = 0.f;
#pragma unroll
    for (int i = 0; i < HeadVec<C>::NV; i++) {
      const float a0 = v.v[i].x / s - n.v[i].x, a1 = v.v[i].y / s - n.v[i].y;
      const float a2 = v.v[i].z / s - n.v[i].z, a3 = v.v[i].w / s - n.v[i].w;
      d += w.v[i].x * (a0 * a0) + w.v[i].y * (a1 * a1) + w.v[i].z * (a2 * a2) + w.v[i].w * (a3 * a3);
    }
    acc[0] += (double)warp_sum(d);
  }
  block_fold<HD_WARPS * 32>(acc, wsum);
  if (threadIdx.x == 0) part[blockIdx.x] = acc[0];
}

struct LpParts {
  const double* p[5];
  int n[5];
};
// out = sum_k (sum of tap k's partials) / (h_k w_k): fixed order; an empty extent gives 0 / 0 = NaN
__global__ void __launch_bounds__(256) lp_reduce_kernel(const LpParts parts, const float* bbox, int W, int H,
                                                        float* __restrict__ out) {
  __shared__ double ws[8];
  double total = 0.0;
  for (int t = 0; t < 5; t++) {
    double s[1];
    block_sum_strided<256>(parts.p[t], parts.n[t], s, ws);
    if (threadIdx.x == 0) {
      const LpExt ex = lp_extent(bbox, W, H, t);
      total += s[0] / ((double)ex.h * (double)ex.w);
    }
  }
  if (threadIdx.x == 0) out[0] = (float)total;
}

// The gradient at a tap's ReLU output: the head's closed form plus, below relu5_3, the max-pool gradient of the next
// level (dq, the gradient at the pool's output), routed to the first maximum of the window in scan order.
//   n = f / s, s = r + eps, r = |f|:  dn_c = G 2 w_c (n_c - nt_c),  df_c = dn_c / s + f_c (-(sum_k dn_k f_k) / s^2) / r
// with G = dL/dout / (h w); r = 0 gives NaN as autograd does (masked out by the ReLU select below it).  A crop whose
// level-4 extent is empty has a NaN loss and gets G = 0: a zero gradient.
template <int C>
__global__ void __launch_bounds__(HD_WARPS * 32) lp_boundary_kernel(const float* __restrict__ f,
                                                                    const float* __restrict__ nt,
                                                                    const float* __restrict__ lw,
                                                                    const float* __restrict__ dq,
                                                                    const float* __restrict__ dout,
                                                                    float* __restrict__ gout, const float* bbox,
                                                                    int W, int H, int level) {
  const LpExt ex = lp_extent(bbox, W, H, level);
  const LpExt e4 = lp_extent(bbox, W, H, 4);
  const LpExt eq = lp_extent(bbox, W, H, level + 1);
  const int ld = W >> level, ldq = W >> (level + 1), lane = threadIdx.x & 31;
  const float G = (e4.h > 0 && e4.w > 0) ? __ldg(dout) / ((float)ex.h * (float)ex.w) : 0.f;
  HeadVec<C> w;
  w.load(lw, lane);
  for (int k = 0; k < HD_PPW; k++) {
    const int p = blockIdx.x * HD_PIX + (threadIdx.x >> 5) * HD_PPW + k;
    const int y = p / ld, x = p - y * ld;
    if (y >= ex.h || x >= ex.w) continue;  // warp-uniform
    HeadVec<C> v, out;
    v.load(f + (size_t)p * C, lane);
#pragma unroll
    for (int i = 0; i < HeadVec<C>::NV; i++) out.v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (G != 0.f) {
      HeadVec<C> n;
      n.load(nt + (size_t)p * C, lane);
      const float r = sqrtf(sum_sq(v)), s = r + LP_EPS;
      float td = 0.f;
#pragma unroll
      for (int i = 0; i < HeadVec<C>::NV; i++) {
        float4& o = out.v[i];
        o.x = G * 2.f * w.v[i].x * (v.v[i].x / s - n.v[i].x);
        o.y = G * 2.f * w.v[i].y * (v.v[i].y / s - n.v[i].y);
        o.z = G * 2.f * w.v[i].z * (v.v[i].z / s - n.v[i].z);
        o.w = G * 2.f * w.v[i].w * (v.v[i].w / s - n.v[i].w);
        td += o.x * v.v[i].x + o.y * v.v[i].y + o.z * v.v[i].z + o.w * v.v[i].w;
      }
      const float gr = (-warp_sum(td) / (s * s)) / r;
#pragma unroll
      for (int i = 0; i < HeadVec<C>::NV; i++) {
        float4& o = out.v[i];
        o = make_float4(o.x / s + v.v[i].x * gr, o.y / s + v.v[i].y * gr, o.z / s + v.v[i].z * gr,
                        o.w / s + v.v[i].w * gr);
      }
    }
    const int qy = y >> 1, qx = x >> 1;
    if (dq && qy < eq.h && qx < eq.w) {
      const int me = (y & 1) * 2 + (x & 1);
      const float* w0 = f + ((size_t)(2 * qy) * ld + 2 * qx) * C;
#pragma unroll
      for (int i = 0; i < HeadVec<C>::NV; i++) {
        const int c4 = lane + 32 * i;
        if (c4 >= C / 4) continue;
        float4 win[4];
        win[0] = __ldg(reinterpret_cast<const float4*>(w0) + c4);
        win[1] = __ldg(reinterpret_cast<const float4*>(w0 + C) + c4);
        win[2] = __ldg(reinterpret_cast<const float4*>(w0 + (size_t)ld * C) + c4);
        win[3] = __ldg(reinterpret_cast<const float4*>(w0 + (size_t)ld * C + C) + c4);
        int ax = 0, ay = 0, az = 0, aw = 0;
#pragma unroll
        for (int k2 = 1; k2 < 4; k2++) {
          if (win[k2].x > win[ax].x) ax = k2;
          if (win[k2].y > win[ay].y) ay = k2;
          if (win[k2].z > win[az].z) az = k2;
          if (win[k2].w > win[aw].w) aw = k2;
        }
        const float4 g = __ldg(reinterpret_cast<const float4*>(dq + ((size_t)qy * ldq + qx) * C) + c4);
        float4& o = out.v[i];
        o.x += ax == me ? g.x : 0.f;
        o.y += ay == me ? g.y : 0.f;
        o.z += az == me ? g.z : 0.f;
        o.w += aw == me ? g.w : 0.f;
      }
    }
    out.store(gout + (size_t)p * C, lane);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------------------------------
static void lp_conv(bool fwd, const B2RLpips& P, int l, const float* x, const float* mask, float* y, cudaStream_t st) {
  const int lev = lp_level(l);
  ConvArgs a{x, mask, fwd ? P.w_fwd[l] : P.w_bwd[l], P.bias[l], y, P.bbox, P.width, P.height, lev,
             fwd ? lp_cin(l) : lp_cout(l), fwd ? lp_cout(l) : lp_cin(l)};
  const dim3 grid(((P.width >> lev) + CV_TW - 1) / CV_TW, ((P.height >> lev) + CV_TH - 1) / CV_TH, a.N / CV_N);
  ProfScope ps(K_MISC, st);
  if (fwd) launch_k(lp_conv_kernel<true>, grid, CV_THREADS, 0, st, false, a);
  else launch_k(lp_conv_kernel<false>, grid, CV_THREADS, 0, st, false, a);
}

static void lp_pool(const B2RLpips& P, int level, int C, const float* in, float* out, cudaStream_t st) {
  const size_t n = (size_t)(P.height >> level) * (P.width >> level) * (C / 4);
  ProfScope ps(K_MISC, st);
  launch_k(lp_pool_kernel, (unsigned)((n + 255) / 256), 256, 0, st, false, in, out, P.bbox, P.width, P.height, level, C);
}

template <template <int> class K, typename... Args>
static void lp_head_launch(int C, int ctas, cudaStream_t st, Args... args) {
  ProfScope ps(K_MISC, st);
  switch (C) {
    case 64: launch_k(K<64>::fn, ctas, HD_WARPS * 32, 0, st, false, args...); break;
    case 128: launch_k(K<128>::fn, ctas, HD_WARPS * 32, 0, st, false, args...); break;
    case 256: launch_k(K<256>::fn, ctas, HD_WARPS * 32, 0, st, false, args...); break;
    default: launch_k(K<512>::fn, ctas, HD_WARPS * 32, 0, st, false, args...); break;
  }
}
template <int C> struct HeadTarget { static constexpr auto fn = lp_head_target_kernel<C>; };
template <int C> struct HeadFwd { static constexpr auto fn = lp_head_fwd_kernel<C>; };
template <int C> struct Boundary { static constexpr auto fn = lp_boundary_kernel<C>; };

// the 13 convs and 4 pools of one image; act(l, in) is where layer l's ReLU output goes, pool(in) the output of the pool
// reading `in`, tap(t, f) runs after each tapped layer
template <typename Act, typename Pool, typename Tap>
static void lp_features(const B2RLpips& P, const float* img, Act act, Pool pool, Tap tap, cudaStream_t st) {
  const int W = P.width, H = P.height;
  {
    ProfScope ps(K_MISC, st);
    launch_k(lp_conv0_fwd_kernel, dim3((W + C0_T - 1) / C0_T, (H + C0_T - 1) / C0_T), C0_T * C0_T, 0, st, false, img,
             P.bbox, W, H, P.w_fwd[0], P.bias[0], act(0, nullptr));
  }
  const float* cur = act(0, nullptr);
  for (int l = 1; l < 13; l++) {
    if (lp_level(l) != lp_level(l - 1)) {
      float* y = pool(cur);
      lp_pool(P, lp_level(l), lp_cin(l), cur, y, st);
      cur = y;
    }
    float* y = act(l, cur);
    lp_conv(true, P, l, cur, nullptr, y, st);
    cur = y;
    if (l == lp_tap_layer(lp_level(l))) tap(lp_level(l), cur);
  }
}

int launch_lpips_forward(const B2RLpips& P, float* out, float* saved, void* scratch, cudaStream_t st) {
  const int W = P.width, H = P.height;
  const LpSaved S = lp_saved_layout(W, H, P.n_images);
  const LpScratch R = lp_scratch_layout(W, H);
  char* sv = (char*)saved;
  char* sc = (char*)scratch;
  float* A = (float*)(sc + R.a);
  float* B = (float*)(sc + R.b);
  // target: layer outputs ping-pong between A and B (never onto the layer's input); the pools write the other one
  auto other = [&](const float* in) { return in == A ? B : A; };
  lp_features(P, P.target, [&](int, const float* in) { return other(in); }, other, [&](int t, const float* f) {
                lp_head_launch<HeadTarget>(lp_cout(lp_tap_layer(t)), lp_head_ctas(W, H, t), st, f,
                                           (float*)(sv + S.tap[t]), P.bbox, W, H, t);
              }, st);
  LpParts parts;
  for (int t = 0; t < 5; t++) { parts.p[t] = (const double*)(sc + R.part[t]); parts.n[t] = lp_head_ctas(W, H, t); }
  for (int n = 0; n < P.n_images; n++) {
    char* im = sv + (size_t)n * S.image;
    lp_features(P, P.img + (size_t)n * 3 * W * H, [&](int l, const float*) { return (float*)(im + S.act[l]); },
                [&](const float*) { return A; },
                [&](int t, const float* f) {
                  lp_head_launch<HeadFwd>(lp_cout(lp_tap_layer(t)), lp_head_ctas(W, H, t), st, f,
                                          (const float*)(sv + S.tap[t]), P.lin[t], (double*)(sc + R.part[t]), P.bbox,
                                          W, H, t);
                }, st);
    ProfScope ps(K_MISC, st);
    launch_k(lp_reduce_kernel, 1, 256, 0, st, false, parts, P.bbox, W, H, out + n);
  }
  return check_launch();
}

int launch_lpips_backward(const B2RLpips& P, const float* saved, const float* dout, float* dimg, void* scratch,
                          cudaStream_t st) {
  const int W = P.width, H = P.height;
  const LpSaved S = lp_saved_layout(W, H, P.n_images);
  const LpScratch R = lp_scratch_layout(W, H);
  const char* sv = (const char*)saved;
  char* sc = (char*)scratch;
  float* A = (float*)(sc + R.a);
  float* B = (float*)(sc + R.b);
  for (int n = 0; n < P.n_images; n++) {
    const char* im = sv + (size_t)n * S.image;
    auto act = [&](int l) { return (const float*)(im + S.act[l]); };
    float* cur = nullptr;  // the gradient at the input of the level above (the pool's output)
    for (int t = 4; t >= 0; t--) {
      const int L = lp_tap_layer(t);
      float* g = cur == A ? B : A;
      lp_head_launch<Boundary>(lp_cout(L), lp_head_ctas(W, H, t), st, act(L), (const float*)(sv + S.tap[t]), P.lin[t],
                               (const float*)cur, dout + n, g, P.bbox, W, H, t);
      cur = g;
      for (int l = L; l >= 0 && lp_level(l) == t; l--) {
        if (l == 0) {
          ProfScope ps(K_MISC, st);
          launch_k(lp_conv0_bwd_kernel, dim3((W + C0_T - 1) / C0_T, (H + C0_T - 1) / C0_T), C0_T * C0_T, 0, st, false,
                   (const float*)cur, act(0), P.bbox, W, H, P.w_fwd[0], dimg + (size_t)n * 3 * W * H);
          break;
        }
        float* y = cur == A ? B : A;
        lp_conv(false, P, l, cur, act(l), y, st);
        cur = y;
      }
    }
  }
  return check_launch();
}

}  // namespace b2r
