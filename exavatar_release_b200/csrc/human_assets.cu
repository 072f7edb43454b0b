// human_assets.cu -- HumanGaussian's code around its networks (avatar/common/nets/module.py:524-539, 561 with
// get_mean_offset_offset's mask, :489-493, and model.py:92-96's warm-up clamp), forward and backward, one thread per
// Gaussian (exavatar_release_b200/human_assets.py).
//
// Geometry, per Gaussian and coordinate, in the reference's operations and order:
//   m = mesh + mean_offset;  mmo = mean_offset_offset * (1 - mask);  mean_3d = m + expr_offset;
//   mean_3d_refined = (m + (mmo + pose_offset)) + expr_offset;
//   scale = exp(s) x3, scale_refined = exp(s + scale_offset) x3, warm-up: clamp(x, max=0.001) beside the unclamped x.
// The mask multiplies (NaN and inf in mean_offset_offset give NaN on masked rows, as in ExAvatar).  Colours:
//   rgb = (tanh(x) + 1) / 2, rgb_refined = (tanh(x + rgb_offset) + 1) / 2.
// The unit is compiled with --fmad=false and calls expf / tanhf as torch's CUDA kernels do, so every forward output is
// bit-identical to ExAvatar's fp32 torch expressions.  The backward recomputes the activations from the inputs and sums
// each gradient in a fixed order; every output element is written once.  No atomics, no allocation, no sync.
#include "common.cuh"

namespace b2r {

constexpr int HA_THREADS = 256;

__device__ __forceinline__ float ld_or0(const float* p, int64_t i) { return p ? __ldg(p + i) : 0.f; }

// torch.clamp(x, max=0.001): the Python float becomes the kernel's float scalar; NaN propagates
__device__ __forceinline__ float warmup_clamp(float x) {
  const float hi = static_cast<float>(0.001);
  return x > hi ? hi : x;
}

__global__ void __launch_bounds__(HA_THREADS) human_geometry_fwd_kernel(
    const B2RHumanAssets h, float* __restrict__ mean, float* __restrict__ mean_r, float* __restrict__ scale,
    float* __restrict__ scale_r, float* __restrict__ mmo_out, float* __restrict__ scale_wo,
    float* __restrict__ scale_r_wo) {
  const int64_t p = (int64_t)blockIdx.x * HA_THREADS + threadIdx.x;
  if (p >= h.P) return;
  const float* geo = h.geo + p * h.geo_stride;
  const float* go = h.geo_offset + p * h.geo_offset_stride;
  const float keep = 1.f - __ldg(h.mask + p);
  const float s = expf(__ldg(geo + 3)), sr = expf(__ldg(geo + 3) + __ldg(go + 3));
  for (int i = 0; i < 3; ++i) {
    const int64_t e = 3 * p + i;
    const float m = __ldg(h.mesh + e) + __ldg(geo + i);
    const float mmo = __ldg(go + i) * keep;
    const float x = __ldg(h.expr_offset + e);
    mean[e] = m + x;
    mean_r[e] = (m + (mmo + __ldg(h.pose_offset + e))) + x;
    mmo_out[e] = mmo;
    if (h.warmup) {
      scale_wo[e] = s;
      scale_r_wo[e] = sr;
      scale[e] = warmup_clamp(s);
      scale_r[e] = warmup_clamp(sr);
    } else {
      scale[e] = s;
      scale_r[e] = sr;
    }
  }
}

__global__ void __launch_bounds__(HA_THREADS) human_geometry_bwd_kernel(const B2RHumanAssets h,
                                                                        const B2RHumanAssetsGrads g) {
  const int64_t p = (int64_t)blockIdx.x * HA_THREADS + threadIdx.x;
  if (p >= h.P) return;
  const float* geo = h.geo + p * h.geo_stride;
  const float* go = h.geo_offset + p * h.geo_offset_stride;
  const float keep = 1.f - __ldg(h.mask + p);
  const float s = expf(__ldg(geo + 3)), sr = expf(__ldg(geo + 3) + __ldg(go + 3));
  const float hi = static_cast<float>(0.001);
  float gs = 0.f, gsr = 0.f;  // d of the repeated (P,3) scales, summed over the three columns (repeat's backward)
  for (int i = 0; i < 3; ++i) {
    const int64_t e = 3 * p + i;
    const float gm = ld_or0(g.dL_dmean_3d, e), gr = ld_or0(g.dL_dmean_3d_refined, e);
    const float gmr = gm + gr;  // m, mesh, mean_offset and expr_offset each feed both means
    g.dL_dmesh[e] = gmr;
    g.dL_dexpr_offset[e] = gmr;
    g.dL_dgeo[4 * p + i] = gmr;
    g.dL_dgeo_offset[4 * p + i] = (gr + ld_or0(g.dL_dmean_offset_offset, e)) * keep;
    float a = ld_or0(g.dL_dscale, e), b = ld_or0(g.dL_dscale_refined, e);
    if (h.warmup) {  // clamp's mask passes x <= max; the clone passes everything
      a = (s <= hi ? a : 0.f) + ld_or0(g.dL_dscale_wo_clamp, e);
      b = (sr <= hi ? b : 0.f) + ld_or0(g.dL_dscale_refined_wo_clamp, e);
    }
    gs = i == 0 ? a : gs + a;
    gsr = i == 0 ? b : gsr + b;
  }
  const float dsr = gsr * sr;
  g.dL_dgeo[4 * p + 3] = gs * s + dsr;
  g.dL_dgeo_offset[4 * p + 3] = dsr;
}

__device__ __forceinline__ float tanh_color(float x) { return (tanhf(x) + 1.f) * 0.5f; }

__global__ void __launch_bounds__(HA_THREADS) human_colors_fwd_kernel(int64_t n, const float* __restrict__ rgb,
                                                                      const float* __restrict__ off,
                                                                      float* __restrict__ out,
                                                                      float* __restrict__ out_r) {
  const int64_t e = (int64_t)blockIdx.x * HA_THREADS + threadIdx.x;
  if (e >= n) return;
  const float x = __ldg(rgb + e);
  out[e] = tanh_color(x);
  out_r[e] = tanh_color(x + __ldg(off + e));
}

__global__ void __launch_bounds__(HA_THREADS) human_colors_bwd_kernel(int64_t n, const float* __restrict__ rgb,
                                                                      const float* __restrict__ off,
                                                                      const float* __restrict__ g,
                                                                      const float* __restrict__ g_r,
                                                                      float* __restrict__ d_rgb,
                                                                      float* __restrict__ d_off) {
  const int64_t e = (int64_t)blockIdx.x * HA_THREADS + threadIdx.x;
  if (e >= n) return;
  const float x = __ldg(rgb + e);
  const float t = tanhf(x), tr = tanhf(x + __ldg(off + e));
  // (tanh(x) + 1) / 2: the division's 0.5, then tanh's 1 - y^2
  const float d = (ld_or0(g, e) * 0.5f) * (1.f - t * t);
  const float dr = (ld_or0(g_r, e) * 0.5f) * (1.f - tr * tr);
  d_rgb[e] = d + dr;
  d_off[e] = dr;
}

static unsigned blocks(int64_t n) { return (unsigned)((n + HA_THREADS - 1) / HA_THREADS); }

int launch_human_geometry_forward(const B2RHumanAssets& h, float* mean, float* mean_r, float* scale, float* scale_r,
                                  float* mmo, float* scale_wo, float* scale_r_wo, cudaStream_t st) {
  if (h.P == 0) return B2R_OK;
  ProfScope ps(K_MISC, st);
  launch_k(human_geometry_fwd_kernel, blocks(h.P), HA_THREADS, 0, st, false, h, mean, mean_r, scale, scale_r, mmo,
           scale_wo, scale_r_wo);
  return check_launch();
}

int launch_human_geometry_backward(const B2RHumanAssets& h, const B2RHumanAssetsGrads& g, cudaStream_t st) {
  if (h.P == 0) return B2R_OK;
  ProfScope ps(K_MISC, st);
  launch_k(human_geometry_bwd_kernel, blocks(h.P), HA_THREADS, 0, st, false, h, g);
  return check_launch();
}

int launch_human_colors_forward(int P, const float* rgb, const float* off, float* out, float* out_r, cudaStream_t st) {
  if (P == 0) return B2R_OK;
  ProfScope ps(K_MISC, st);
  launch_k(human_colors_fwd_kernel, blocks(3 * (int64_t)P), HA_THREADS, 0, st, false, 3 * (int64_t)P, rgb, off, out,
           out_r);
  return check_launch();
}

int launch_human_colors_backward(int P, const float* rgb, const float* off, const float* g, const float* g_r,
                                 float* d_rgb, float* d_off, cudaStream_t st) {
  if (P == 0) return B2R_OK;
  ProfScope ps(K_MISC, st);
  launch_k(human_colors_bwd_kernel, blocks(3 * (int64_t)P), HA_THREADS, 0, st, false, 3 * (int64_t)P, rgb, off, g,
           g_r, d_rgb, d_off);
  return check_launch();
}

}  // namespace b2r
