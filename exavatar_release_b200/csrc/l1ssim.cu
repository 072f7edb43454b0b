// l1ssim.cu -- ExAvatar's photometric L1 + SSIM terms (avatar/common/nets/loss.py RGBLoss / SSIM, as
// avatar/main/model.py:196-215 reduces them with .mean()) in one op that never reads the crop box on the host.
//
// The crop box lives on the device, so the grid covers the whole W x H image in 16x16 tiles and a tile outside the crop
// only writes a zero partial.  Inside, with x' = img * mask, y' = target * mask on the crop and ZERO outside it (the
// reference convolves the crop with zero padding 5, not the image):
//   forward   l1ssim_fwd_kernel<true>: stage x', y' of the tile + a 5-pixel halo, the five moments mu_x, mu_y, S_xx,
//             S_yy, S_xy by separable 11-tap passes (horizontal, then vertical), the SSIM map m = A B / (C D), and per
//             pixel / channel the three partials dm/dmu_x, dm/dS_xx, dm/dS_xy into the scratch for the backward; one
//             (sum |x' - y'|, sum m) partial per tile.  l1ssim_reduce_kernel adds the tile partials in a fixed order.
//   backward  l1ssim_bwd_kernel<true>: a gather -- stage the three partials of the tile + halo, window them by the same
//             separable passes (the window is symmetric), dL/dx'(p) = g [S1 + 2 x'(p) S2 + y'(p) S3]; times the mask,
//             plus the L1 term mask * sign(x' - y') dL/dl1 / (3hw).  Every pixel of dL/dimg is written (0 outside).
// No float atomics anywhere: two runs are bit-identical.  Nothing reads back to the host: CUDA-graph capturable.
#include "common.cuh"

namespace b2r {

constexpr int LS_T = 16;                 // output tile edge
constexpr int LS_R = 5;                  // window radius (11 taps)
constexpr int LS_S = LS_T + 2 * LS_R;    // staged edge with the halo
constexpr int LS_THREADS = LS_T * LS_T;  // one thread per output pixel
constexpr int LS_WARPS = LS_THREADS / 32;

// SSIM.gaussian(11, 1.5): exp(-(x-5)^2 / 4.5) rounded to fp32, divided by its fp32 sum (bit-exact fp32 values)
__constant__ float c_ssim_w[11] = {1.028380124e-03f, 7.598758209e-03f, 3.600077331e-02f, 1.093606874e-01f,
                                   2.130055279e-01f, 2.660117149e-01f, 2.130055279e-01f, 1.093606874e-01f,
                                   3.600077331e-02f, 7.598758209e-03f, 1.028380124e-03f};

struct L1SsimIn {
  int W, H;
  const float* img;
  const float* target;
  const float* mask;  // (H,W) or null
  const float* bbox;  // device {xmin, ymin, width, height} or null
};

__host__ __device__ inline int ls_tiles_x(int W) { return (W + LS_T - 1) / LS_T; }
__host__ __device__ inline int ls_tiles_y(int H) { return (H + LS_T - 1) / LS_T; }
static size_t ls_map_bytes(int W, int H) { return align_up((size_t)9 * W * H * sizeof(float)); }

// maps: 9 planes of H*W floats, plane 3*k + c = partial k (dm/dmu_x, dm/dS_xx, dm/dS_xy) of channel c
template <bool SSIM>
__global__ void __launch_bounds__(LS_THREADS) l1ssim_fwd_kernel(const L1SsimIn a, float* __restrict__ maps,
                                                                float2* __restrict__ tile_sums) {
  __shared__ float sx[LS_S * LS_S], sy[LS_S * LS_S];
  __shared__ float hm[5][LS_S * LS_T];  // horizontal pass: mu_x, mu_y, S_xx, S_yy, S_xy
  __shared__ float wsum[LS_WARPS * 2];
  const Crop cr = read_crop(a.bbox, a.W, a.H);
  const int tx0 = blockIdx.x * LS_T, ty0 = blockIdx.y * LS_T;
  const int tile = blockIdx.y * gridDim.x + blockIdx.x;
  if (tx0 >= cr.x1 || tx0 + LS_T <= cr.x0 || ty0 >= cr.y1 || ty0 + LS_T <= cr.y0) {  // block-uniform
    if (threadIdx.x == 0) tile_sums[tile] = make_float2(0.f, 0.f);
    return;
  }
  const int lx = threadIdx.x % LS_T, ly = threadIdx.x / LS_T;
  const int px = tx0 + lx, py = ty0 + ly;
  const bool inside = cr.has(px, py);
  const size_t HW = (size_t)a.W * a.H, o = (size_t)py * a.W + px;
  const float m_p = inside && a.mask ? __ldg(a.mask + o) : 1.f;
  float l1 = 0.f, ssum = 0.f;
  for (int c = 0; c < 3; c++) {
    if (!SSIM) {
      if (inside) l1 += fabsf(__ldg(a.img + c * HW + o) * m_p - __ldg(a.target + c * HW + o) * m_p);
      continue;
    }
    __syncthreads();  // the previous channel is done with the stage
    for (int e = threadIdx.x; e < LS_S * LS_S; e += LS_THREADS) {
      const int r = e / LS_S, q = e - r * LS_S;
      const int gx = tx0 - LS_R + q, gy = ty0 - LS_R + r;
      float xv = 0.f, yv = 0.f;
      if (cr.has(gx, gy)) {
        const size_t g = (size_t)gy * a.W + gx;
        const float m = a.mask ? __ldg(a.mask + g) : 1.f;
        xv = __ldg(a.img + c * HW + g) * m;
        yv = __ldg(a.target + c * HW + g) * m;
      }
      sx[e] = xv;
      sy[e] = yv;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < LS_S * LS_T; e += LS_THREADS) {
      const int r = e / LS_T, q = e - r * LS_T;
      const float* rx = sx + r * LS_S + q;
      const float* ry = sy + r * LS_S + q;
      float mx = 0.f, my = 0.f, xx = 0.f, yy = 0.f, xy = 0.f;
#pragma unroll
      for (int k = 0; k < 11; k++) {
        const float w = c_ssim_w[k], u = rx[k], v = ry[k];
        mx += w * u;
        my += w * v;
        xx += w * (u * u);
        yy += w * (v * v);
        xy += w * (u * v);
      }
      hm[0][e] = mx; hm[1][e] = my; hm[2][e] = xx; hm[3][e] = yy; hm[4][e] = xy;
    }
    __syncthreads();
    if (inside) {
      float mx = 0.f, my = 0.f, xx = 0.f, yy = 0.f, xy = 0.f;
#pragma unroll
      for (int k = 0; k < 11; k++) {
        const float w = c_ssim_w[k];
        const int e = (ly + k) * LS_T + lx;
        mx += w * hm[0][e];
        my += w * hm[1][e];
        xx += w * hm[2][e];
        yy += w * hm[3][e];
        xy += w * hm[4][e];
      }
      constexpr float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
      const float A = 2.f * mx * my + C1;
      const float B = 2.f * (xy - mx * my) + C2;
      const float Cc = mx * mx + my * my + C1;
      const float D = (xx - mx * mx) + (yy - my * my) + C2;
      const float inv = 1.f / (Cc * D);
      const float m = A * B * inv;
      const float xc = sx[(ly + LS_R) * LS_S + lx + LS_R], yc = sy[(ly + LS_R) * LS_S + lx + LS_R];
      l1 += fabsf(xc - yc);
      ssum += m;
      maps[(0 + c) * HW + o] = (2.f * my * (B - A) + 2.f * mx * m * (Cc - D)) * inv;  // dm/dmu_x
      maps[(3 + c) * HW + o] = -m / D;                                                 // dm/dS_xx
      maps[(6 + c) * HW + o] = 2.f * A * inv;                                          // dm/dS_xy
    }
  }
  float t[2] = {l1, ssum};
  block_sum<LS_THREADS>(t, wsum);
  if (threadIdx.x == 0) tile_sums[tile] = make_float2(t[0], t[1]);
}

// the tile partials (ntiles x 2 floats) in a fixed order; means over 3 h w
__global__ void __launch_bounds__(LS_THREADS) l1ssim_reduce_kernel(const float* __restrict__ tile_sums, const int ntiles,
                                                                   const float* __restrict__ bbox, const int W,
                                                                   const int H, const int with_ssim,
                                                                   float* __restrict__ out) {
  __shared__ float wsum[LS_WARPS * 2];
  float s[2];
  block_sum_strided<LS_THREADS>(tile_sums, ntiles, s, wsum);
  if (threadIdx.x == 0) {
    const float n = read_crop(bbox, W, H).count3();  // 0 for an empty crop: 0 / 0 = NaN, like mean() of nothing
    out[0] = s[0] / n;
    if (with_ssim) out[1] = s[1] / n;
  }
}

template <bool SSIM>
__global__ void __launch_bounds__(LS_THREADS) l1ssim_bwd_kernel(const L1SsimIn a, const float* __restrict__ maps,
                                                                const float* __restrict__ dout,
                                                                float* __restrict__ dimg) {
  __shared__ float sp[3][LS_S * LS_S];
  __shared__ float hp[3][LS_S * LS_T];
  const Crop cr = read_crop(a.bbox, a.W, a.H);
  const int tx0 = blockIdx.x * LS_T, ty0 = blockIdx.y * LS_T;
  const int lx = threadIdx.x % LS_T, ly = threadIdx.x / LS_T;
  const int px = tx0 + lx, py = ty0 + ly;
  const bool in_image = px < a.W && py < a.H;
  const size_t HW = (size_t)a.W * a.H, o = (size_t)py * a.W + px;
  if (tx0 >= cr.x1 || tx0 + LS_T <= cr.x0 || ty0 >= cr.y1 || ty0 + LS_T <= cr.y0) {  // block-uniform
    if (in_image)
      for (int c = 0; c < 3; c++) dimg[c * HW + o] = 0.f;
    return;
  }
  const bool inside = cr.has(px, py);
  const float n = cr.count3();  // > 0: this tile meets the crop
  const float g_l1 = __ldg(dout) / n;
  const float g_ss = SSIM ? __ldg(dout + 1) / n : 0.f;
  const float m_p = inside && a.mask ? __ldg(a.mask + o) : 1.f;
  for (int c = 0; c < 3; c++) {
    float d = 0.f, xc = 0.f, yc = 0.f;
    if (inside) {
      xc = __ldg(a.img + c * HW + o) * m_p;
      yc = __ldg(a.target + c * HW + o) * m_p;
    }
    if (SSIM) {
      __syncthreads();
      for (int e = threadIdx.x; e < LS_S * LS_S; e += LS_THREADS) {
        const int r = e / LS_S, q = e - r * LS_S;
        const int gx = tx0 - LS_R + q, gy = ty0 - LS_R + r;
        float v0 = 0.f, v1 = 0.f, v2 = 0.f;
        if (cr.has(gx, gy)) {  // q runs over the crop only: its partials are the ones the forward wrote
          const size_t g = (size_t)gy * a.W + gx;
          v0 = __ldg(maps + (0 + c) * HW + g);
          v1 = __ldg(maps + (3 + c) * HW + g);
          v2 = __ldg(maps + (6 + c) * HW + g);
        }
        sp[0][e] = v0; sp[1][e] = v1; sp[2][e] = v2;
      }
      __syncthreads();
      for (int e = threadIdx.x; e < LS_S * LS_T; e += LS_THREADS) {
        const int r = e / LS_T, q = e - r * LS_T;
        float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; k++) {
          const float w = c_ssim_w[k];
          const int s = r * LS_S + q + k;
          s0 += w * sp[0][s];
          s1 += w * sp[1][s];
          s2 += w * sp[2][s];
        }
        hp[0][e] = s0; hp[1][e] = s1; hp[2][e] = s2;
      }
      __syncthreads();
      if (inside) {
        float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; k++) {
          const float w = c_ssim_w[k];
          const int e = (ly + k) * LS_T + lx;
          s0 += w * hp[0][e];
          s1 += w * hp[1][e];
          s2 += w * hp[2][e];
        }
        d = g_ss * (s0 + 2.f * xc * s1 + yc * s2);
      }
    }
    if (inside) {
      const float diff = xc - yc;
      d += g_l1 * (float)((diff > 0.f) - (diff < 0.f));  // sign(0) = 0, as torch.abs's gradient
    }
    if (in_image) dimg[c * HW + o] = inside ? m_p * d : 0.f;
  }
}

size_t l1ssim_scratch_bytes(int W, int H) {
  const int w = W > 0 ? W : 1, h = H > 0 ? H : 1;
  return ls_map_bytes(w, h) + align_up((size_t)ls_tiles_x(w) * ls_tiles_y(h) * sizeof(float2));
}

int launch_l1ssim_forward(int W, int H, const float* img, const float* target, const float* mask, const float* bbox,
                          bool with_ssim, float* out, void* scratch, cudaStream_t st) {
  const L1SsimIn a{W, H, img, target, mask, bbox};
  const dim3 grid(ls_tiles_x(W), ls_tiles_y(H));
  float* maps = (float*)scratch;
  float2* tiles = (float2*)((char*)scratch + ls_map_bytes(W, H));
  {
    ProfScope p(K_MISC, st);
    if (with_ssim) launch_k(l1ssim_fwd_kernel<true>, grid, LS_THREADS, 0, st, true, a, maps, tiles);
    else launch_k(l1ssim_fwd_kernel<false>, grid, LS_THREADS, 0, st, true, a, maps, tiles);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(l1ssim_reduce_kernel, 1, LS_THREADS, 0, st, true, (const float*)tiles, (int)(grid.x * grid.y), bbox, W,
             H, with_ssim ? 1 : 0, out);
  }
  return check_launch();
}

int launch_l1ssim_backward(int W, int H, const float* img, const float* target, const float* mask, const float* bbox,
                           bool with_ssim, const float* dout, float* dimg, const void* scratch, cudaStream_t st) {
  const L1SsimIn a{W, H, img, target, mask, bbox};
  const dim3 grid(ls_tiles_x(W), ls_tiles_y(H));
  ProfScope p(K_MISC, st);
  if (with_ssim) launch_k(l1ssim_bwd_kernel<true>, grid, LS_THREADS, 0, st, true, a, (const float*)scratch, dout, dimg);
  else launch_k(l1ssim_bwd_kernel<false>, grid, LS_THREADS, 0, st, true, a, (const float*)nullptr, dout, dimg);
  return check_launch();
}

}  // namespace b2r
