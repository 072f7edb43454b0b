// metrics.cu -- the test-set scores of ExAvatar's NeuMan protocol (avatar/tools/eval_neuman.py) for N frames, each a
// render against its own target, in one op that never reads anything back on the host.
//
// Per frame n and image (render x, target y), the 8-bit PNG round trip of test.py's cv2.imwrite and eval's imread / 255:
//   v = fl(p * 255);  u8 = 0 if v is NaN or |v| >= 2^31, else clamp(rint(v), 0, 255);  q = fl((double)u8 / 255)
// then, with a mask m (1 = human), eval's white background fl(fl(q m) + fl(1 - m)).  Then
//   psnr  = 10 log10(1 / mse), the mean of (x - y)^2 over the 3 H W elements in fp64, rounded once;
//   ssim  = torchmetrics' SSIM (Gaussian 11 x 11, sigma 1.5, c1 = 0.01^2, c2 = 0.03^2, variances clamped at 0) averaged
//           over the 3 (H - 10) (W - 10) window centres that reflect padding never reaches; the window sums run in fp64;
//   lpips = lpips.LPIPS(net='alex') version 0.1 on x*2-1: ScalingLayer, torchvision's alexnet().features[0:12] (conv
//           11x11/4 pad 2, pool 3/2, conv 5x5 pad 2, pool 3/2, conv 3x3 pad 1 x3, ReLU after each conv), and per tap
//           relu1..relu5  mean_p sum_c w_c (n_c(f_x) - n_c(f_y))^2,  n(f) = f / (sqrt(sum_c f_c^2) + 1e-10).
// out[n] = {psnr, ssim, lpips}.
//
// The file is compiled with --fmad=false: the round trip, the composite and the ScalingLayer are torch's fp32
// expressions rounded operation by operation, and identical images give SSIM terms whose numerator and denominator are
// the same bits.
//
// Launches (every grid sized from W, H, N; no allocation, no float atomics, no host sync):
//   nm_prep_kernel      the round trip and composite of all 2N images into `q`, and the trunk's input into `in0`
//   nm_ssim_kernel      per (frame, channel, 32 x 16 tile): fp64 partials of the squared error and the SSIM sum
//   nm_conv_kernel x5   the AlexNet convs of all 2N images, TF32 implicit GEMMs (mma.sync m16n8k8, both operands
//                       rounded with cvt.rna), bias + ReLU fused, into `act`
//   nm_pool_kernel x2   3x3 stride-2 floor max pools
//   nm_head_kernel x5   per tap: fp64 per-CTA partials of the head sum for every frame
//   nm_reduce_kernel    one CTA per frame: every partial in a fixed order, into out
//
// Scratch layout (byte offsets of nm_layout, every region 256-byte aligned; image i < N is render i, image N + i
// target i):
//   q        (2N, 3, H, W)        the quantised, composited images
//   in0      (2N, H, W, 4)        ((q*2 - 1) - shift) / scale, channel 3 zero
//   act[l]   (2N, H_l, W_l, C_l)  relu(l+1), C = 64 192 384 256 256; H_0 = (H - 7) / 4 + 1, H_1 = H_0 pooled,
//                                  H_2..4 = H_1 pooled; pooling is (h - 3) / 2 + 1
//   pool[p]  (2N, ..., C)         pool 1 (64 channels at H_1 x W_1) and pool 2 (192 at H_2 x W_2)
//   sse, ssim (N, 3, ctas) double the pixel kernels' partials, ctas = ceil(W / 32) ceil(H / 16)
//   part[t]  (N, ceil(H_t W_t / 32)) double   the heads' partials
//
// The AlexNet trunk does not reuse lpips.cu's VGG kernels: those are 3x3 stride-1 convs over power-of-two levels of a
// crop (W >> level), with heads whose lane layout covers 64, 128, 256 and 512 channels, and AlexNet needs 11x11 / 5x5
// kernels, stride 4 and 192 / 384 channels.  Sharing them would need a branch on which network calls.
#include "common.cuh"

namespace b2r {

// torchmetrics' 1D window: exp(-(d / 1.5)^2 / 2), d = -5 .. 5, divided by its sum, in fp32 as torch builds it on a
// CUDA device, where eval_neuman's images live (the CPU build differs by up to 8 ulps; metrics.SSIM_WINDOW)
__constant__ float c_nm_gauss[11] = {0x1.0d956p-10f, 0x1.f1fdfcp-8f, 0x1.26eb18p-5f, 0x1.bff1p-4f,   0x1.b43c4p-3f,
                                     0x1.106562p-2f, 0x1.b43c4p-3f,  0x1.bff1p-4f,   0x1.26eb18p-5f, 0x1.f1fdfcp-8f,
                                     0x1.0d956p-10f};
__constant__ float c_nm_shift[3] = {-.030f, -.088f, -.188f};  // lpips ScalingLayer
__constant__ float c_nm_scale[3] = {.458f, .448f, .450f};
constexpr float NM_EPS = 1e-10f;
constexpr double NM_C1 = 0.01 * 0.01, NM_C2 = 0.03 * 0.03;

constexpr int NM_CIN[5] = {4, 64, 192, 384, 256};  // conv1's input is padded to 4 channels
constexpr int NM_COUT[5] = {64, 192, 384, 256, 256};
constexpr int NM_KS[5] = {11, 5, 3, 3, 3};
constexpr int NM_STRIDE[5] = {4, 1, 1, 1, 1};
constexpr int NM_PAD[5] = {2, 2, 1, 1, 1};

struct Dim {
  int h, w;
};
// spatial size of act[l] (l = 0..4) and of the pools
static Dim nm_act_dim(int W, int H, int l) {
  Dim d{(H - 7) / 4 + 1, (W - 7) / 4 + 1};
  const int pools = l == 0 ? 0 : l == 1 ? 1 : 2;
  for (int p = 0; p < pools; p++) d = {(d.h - 3) / 2 + 1, (d.w - 3) / 2 + 1};
  return d;
}

constexpr int SS_TW = 32, SS_TH = 16;                  // nm_ssim_kernel's output tile
constexpr int HD_WARPS = 8, HD_PPW = 4, HD_PIX = HD_WARPS * HD_PPW;  // heads: a warp per pixel, 32 pixels a CTA

static int nm_ssim_ctas(int W, int H) { return ((W + SS_TW - 1) / SS_TW) * ((H + SS_TH - 1) / SS_TH); }
static int nm_head_ctas(int W, int H, int t) {
  const Dim d = nm_act_dim(W, H, t);
  return (d.h * d.w + HD_PIX - 1) / HD_PIX;
}
static int nm_kpad(int l) { return (NM_KS[l] * NM_KS[l] * NM_CIN[l] + 31) / 32 * 32; }

struct NmLayout {
  size_t q, in0, act[5], pool[2], sse, ssim, part[5], total;
};
static NmLayout nm_layout(int W, int H, int N) {
  NmLayout s;
  const size_t HW = (size_t)W * H, I = 2 * (size_t)N;
  size_t o = 0;
  s.q = o; o += align_up(I * 3 * HW * sizeof(float));
  s.in0 = o; o += align_up(I * 4 * HW * sizeof(float));
  for (int l = 0; l < 5; l++) {
    const Dim d = nm_act_dim(W, H, l);
    s.act[l] = o; o += align_up(I * d.h * d.w * NM_COUT[l] * sizeof(float));
  }
  for (int p = 0; p < 2; p++) {
    const Dim d = nm_act_dim(W, H, p + 1);
    s.pool[p] = o; o += align_up(I * d.h * d.w * NM_COUT[p] * sizeof(float));
  }
  const size_t ss = (size_t)N * 3 * nm_ssim_ctas(W, H) * sizeof(double);
  s.sse = o; o += align_up(ss);
  s.ssim = o; o += align_up(ss);
  for (int t = 0; t < 5; t++) { s.part[t] = o; o += align_up((size_t)N * nm_head_ctas(W, H, t) * sizeof(double)); }
  s.total = o;
  return s;
}

// ---------------------------------------------------------------------------------------------------------------------
// The round trip, the composite and the trunk's input: one thread per pixel of one of the 2N images.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int nm_png_u8(float p) {
  const float v = p * 255.f;
  if (isnan(v) || fabsf(v) >= 2147483648.f) return 0;  // cvRound's out-of-range result saturates to 0
  return min(max(__float2int_rn(v), 0), 255);          // an integer: rint(-0.4) = -0 reads back as +0
}

__global__ void __launch_bounds__(256) nm_prep_kernel(const float* __restrict__ render, const float* __restrict__ target,
                                                      const float* __restrict__ mask, int mc, int W, int H, int N,
                                                      float* __restrict__ q, float4* __restrict__ in0) {
  const size_t HW = (size_t)W * H;
  const size_t e = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (e >= 2 * (size_t)N * HW) return;
  const size_t i = e / HW, p = e - i * HW;
  const size_t n = i < (size_t)N ? i : i - N;
  const float* src = (i < (size_t)N ? render : target) + n * 3 * HW + p;
  float r[4];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    float v = (float)((double)nm_png_u8(__ldg(src + c * HW)) / 255.0);
    if (mask) {
      const float m = __ldg(mask + (n * mc + (mc == 3 ? c : 0)) * HW + p);
      v = v * m + (1.f - m);
    }
    q[(i * 3 + c) * HW + p] = v;
    r[c] = ((v * 2.f - 1.f) - c_nm_shift[c]) / c_nm_scale[c];
  }
  in0[i * HW + p] = make_float4(r[0], r[1], r[2], 0.f);
}

// ---------------------------------------------------------------------------------------------------------------------
// SSIM and the squared error: per (frame, channel) a 32 x 16 tile of window centres.  The tile and its 5-pixel halo of
// both images are staged in shared memory (zeros outside the image: they reach only centres that are not kept), the
// horizontal 11-tap sums of x, y, x^2, y^2, xy go to shared memory in fp64, and each thread finishes its centre with the
// vertical sums.  The CTA's two sums are reduced in a fixed order into sse / ssim.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int SS_HW = SS_TW + 10, SS_HH = SS_TH + 10;

__global__ void __launch_bounds__(SS_TW * SS_TH) nm_ssim_kernel(const float* __restrict__ q, int W, int H, int N,
                                                                double* __restrict__ sse, double* __restrict__ ssim) {
  __shared__ float sx[SS_HH * SS_HW], sy[SS_HH * SS_HW];
  __shared__ double hs[5][SS_HH * SS_TW];
  __shared__ double red[SS_TW * SS_TH / 32];
  const int n = blockIdx.z / 3, c = blockIdx.z - 3 * n;
  const size_t HW = (size_t)W * H;
  const float* x = q + ((size_t)n * 3 + c) * HW;
  const float* y = q + (((size_t)N + n) * 3 + c) * HW;
  const int tx0 = blockIdx.x * SS_TW, ty0 = blockIdx.y * SS_TH;
  for (int e = threadIdx.x; e < SS_HH * SS_HW; e += SS_TW * SS_TH) {
    const int r = e / SS_HW, col = e - r * SS_HW;
    const int gy = ty0 - 5 + r, gx = tx0 - 5 + col;
    const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
    sx[e] = in ? __ldg(x + (size_t)gy * W + gx) : 0.f;
    sy[e] = in ? __ldg(y + (size_t)gy * W + gx) : 0.f;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < SS_HH * SS_TW; e += SS_TW * SS_TH) {
    const int r = e / SS_TW, col = e - r * SS_TW;
    double a[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
    for (int k = 0; k < 11; k++) {
      const double g = c_nm_gauss[k];
      const double u = sx[r * SS_HW + col + k], v = sy[r * SS_HW + col + k];
      a[0] += g * u;
      a[1] += g * v;
      a[2] += g * (u * u);
      a[3] += g * (v * v);
      a[4] += g * (u * v);
    }
#pragma unroll
    for (int j = 0; j < 5; j++) hs[j][e] = a[j];
  }
  __syncthreads();
  const int lx = threadIdx.x % SS_TW, ly = threadIdx.x / SS_TW;
  const int px = tx0 + lx, py = ty0 + ly;
  double s = 0.0, d2 = 0.0;
  if (px < W && py < H) {
    const double d = (double)sx[(ly + 5) * SS_HW + lx + 5] - (double)sy[(ly + 5) * SS_HW + lx + 5];
    d2 = d * d;
    if (px >= 5 && px < W - 5 && py >= 5 && py < H - 5) {
      double a[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int k = 0; k < 11; k++) {
        const double g = c_nm_gauss[k];
#pragma unroll
        for (int j = 0; j < 5; j++) a[j] += g * hs[j][(ly + k) * SS_TW + lx];
      }
      const double mx = a[0], my = a[1];
      const double vx = fmax(a[2] - mx * mx, 0.0), vy = fmax(a[3] - my * my, 0.0), cxy = a[4] - mx * my;
      s = ((2.0 * mx * my + NM_C1) * (2.0 * cxy + NM_C2)) / ((mx * mx + my * my + NM_C1) * (vx + vy + NM_C2));
    }
  }
  const size_t slot = ((size_t)n * 3 + c) * (gridDim.x * gridDim.y) + blockIdx.y * gridDim.x + blockIdx.x;
  double ts[1] = {s}, td[1] = {d2};
  block_sum<SS_TW * SS_TH>(ts, red);
  if (threadIdx.x == 0) ssim[slot] = ts[0];
  block_sum<SS_TW * SS_TH>(td, red);
  if (threadIdx.x == 0) sse[slot] = td[0];
}

// ---------------------------------------------------------------------------------------------------------------------
// Convolution as an implicit GEMM on the tensor cores, for every image at once (grid.z): M = 128 output pixels of one
// image (row-major over the output plane), N = 64 output channels (grid.y), K = KS x KS x C_in in stages of 32, ordered
// (ky, kx, ci) so that a float4 of 4 consecutive channels never straddles a tap.  Weights (K_pad, C_out), rows past
// KS^2 C_in zero.  Each stage puts the 128 x 32 gathered inputs (zero outside the image) and the 32 x 64 weights in
// shared memory, rounded to TF32 (cvt.rna) once; a warp owns 32 pixels (two m16 tiles) and all eight n8 tiles.  Strides
// 36 and 72 words make the fragment reads conflict-free.  y = relu(conv(x, W) + b), NHWC.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int NC_M = 128, NC_N = 64, NC_K = 32, NC_THREADS = 128;
constexpr int NC_AS = NC_K + 4, NC_BS = NC_N + 8;

struct NmConv {
  const float* x;  // (I, hi, wi, cin)
  const float* w;  // (kpad, cout)
  const float* b;  // (cout)
  float* y;        // (I, ho, wo, cout)
  int hi, wi, cin, ho, wo, cout, ks, stride, pad, kpad;
};

__global__ void __launch_bounds__(NC_THREADS) nm_conv_kernel(const NmConv a) {
  __shared__ __align__(16) uint32_t s_a[NC_M * NC_AS];
  __shared__ __align__(16) uint32_t s_b[NC_K * NC_BS];
  const int M = a.ho * a.wo;
  const int m0 = blockIdx.x * NC_M, n0 = blockIdx.y * NC_N;
  const size_t img = blockIdx.z;
  const float* x = a.x + img * a.hi * a.wi * a.cin;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  // staging: this thread loads float4 q4 of the stage for the pixels (threadIdx.x >> 3) + 16 j
  const int q4 = threadIdx.x & 7;
  int iy0[8], ix0[8];
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int p = m0 + (threadIdx.x >> 3) + 16 * j;
    const int oy = p / a.wo, ox = p - oy * a.wo;
    iy0[j] = p < M ? oy * a.stride - a.pad : -(1 << 20);  // a pixel past the plane reads zeros
    ix0[j] = ox * a.stride - a.pad;
  }
  float acc[2][8][4];
#pragma unroll
  for (int j = 0; j < 2; j++)
#pragma unroll
    for (int n = 0; n < 8; n++) acc[j][n][0] = acc[j][n][1] = acc[j][n][2] = acc[j][n][3] = 0.f;

  for (int k0 = 0; k0 < a.kpad; k0 += NC_K) {
    __syncthreads();  // the previous stage is consumed
    {
      const int k = k0 + 4 * q4;
      const int tap = k / a.cin, ci = k - tap * a.cin;
      const int ky = tap / a.ks, kx = tap - ky * a.ks;
      const bool live = tap < a.ks * a.ks;
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int iy = iy0[j] + ky, ix = ix0[j] + kx;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live && iy >= 0 && iy < a.hi && ix >= 0 && ix < a.wi)
          v = __ldg(reinterpret_cast<const float4*>(x + ((size_t)iy * a.wi + ix) * a.cin + ci));
        *reinterpret_cast<uint4*>(s_a + ((threadIdx.x >> 3) + 16 * j) * NC_AS + 4 * q4) =
            make_uint4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w));
      }
    }
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int e = threadIdx.x + NC_THREADS * j;
      const int r = e >> 4, c4 = e & 15;
      const float4 v = __ldg(reinterpret_cast<const float4*>(a.w + (size_t)(k0 + r) * a.cout + n0 + 4 * c4));
      *reinterpret_cast<uint4*>(s_b + r * NC_BS + 4 * c4) = make_uint4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z),
                                                                      to_tf32(v.w));
    }
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < NC_K / 8; ks++) {
      uint32_t af[2][4];
#pragma unroll
      for (int j = 0; j < 2; j++) {
        const uint32_t* p0 = s_a + (32 * warp + 16 * j + g) * NC_AS + 8 * ks + t;
        af[j][0] = p0[0];
        af[j][1] = p0[8 * NC_AS];
        af[j][2] = p0[4];
        af[j][3] = p0[8 * NC_AS + 4];
      }
#pragma unroll
      for (int n = 0; n < 8; n++) {
        const uint32_t b0 = s_b[(8 * ks + t) * NC_BS + 8 * n + g];
        const uint32_t b1 = s_b[(8 * ks + t + 4) * NC_BS + 8 * n + g];
        mma_tf32(acc[0][n], af[0], b0, b1);
        mma_tf32(acc[1][n], af[1], b0, b1);
      }
    }
  }
  float* y = a.y + img * (size_t)M * a.cout;
#pragma unroll
  for (int j = 0; j < 2; j++)
#pragma unroll
    for (int half = 0; half < 2; half++) {
      const int p = m0 + 32 * warp + 16 * j + g + 8 * half;
      if (p >= M) continue;
      float* dst = y + (size_t)p * a.cout + n0;
#pragma unroll
      for (int n = 0; n < 8; n++) {
        const int co = 8 * n + 2 * t;
        const float v0 = fmaxf(acc[j][n][2 * half] + __ldg(a.b + n0 + co), 0.f);
        const float v1 = fmaxf(acc[j][n][2 * half + 1] + __ldg(a.b + n0 + co + 1), 0.f);
        *reinterpret_cast<float2*>(dst + co) = make_float2(v0, v1);
      }
    }
}

// 3x3 stride-2 max pool with floor, NHWC, every image at once: one thread per (image, pixel, 4 channels)
__global__ void __launch_bounds__(256) nm_pool_kernel(const float* __restrict__ in, float* __restrict__ out, int hi,
                                                      int wi, int ho, int wo, int C, int I) {
  const int C4 = C / 4;
  const size_t e = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (e >= (size_t)I * ho * wo * C4) return;
  const int c4 = (int)(e % C4);
  const size_t r = e / C4;
  const size_t img = r / ((size_t)ho * wo);
  const int p = (int)(r - img * ho * wo);
  const int oy = p / wo, ox = p - oy * wo;
  const float4* s = reinterpret_cast<const float4*>(in) + ((img * hi + 2 * oy) * wi + 2 * ox) * C4 + c4;
  float4 m = __ldg(s);
#pragma unroll
  for (int ky = 0; ky < 3; ky++)
#pragma unroll
    for (int kx = 0; kx < 3; kx++) {
      const float4 v = __ldg(s + ((size_t)ky * wi + kx) * C4);
      m.x = v.x > m.x ? v.x : m.x;
      m.y = v.y > m.y ? v.y : m.y;
      m.z = v.z > m.z ? v.z : m.z;
      m.w = v.w > m.w ? v.w : m.w;
    }
  reinterpret_cast<float4*>(out)[r * C4 + c4] = m;
}

// ---------------------------------------------------------------------------------------------------------------------
// Heads: a warp per pixel, lane l holds channels 4 (l + 32 i) .. + 3 of both images' taps.  Channel sums are warp_sum;
// the CTA's fp64 sum of sum_c w_c (n_c(f_x) - n_c(f_y))^2 goes to part[n][blockIdx.x].
// ---------------------------------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(HD_WARPS * 32) nm_head_kernel(const float* __restrict__ act,
                                                                const float* __restrict__ lw, int npix, int N,
                                                                double* __restrict__ part) {
  constexpr int NV = (C / 4 + 31) / 32;
  __shared__ double wsum[HD_WARPS];
  const int n = blockIdx.y, lane = threadIdx.x & 31;
  const float* fx = act + (size_t)n * npix * C;
  const float* fy = act + ((size_t)N + n) * npix * C;
  float4 w[NV];
#pragma unroll
  for (int i = 0; i < NV; i++) {
    const int c4 = lane + 32 * i;
    w[i] = c4 < C / 4 ? __ldg(reinterpret_cast<const float4*>(lw) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  double acc[1] = {0.0};
  for (int k = 0; k < HD_PPW; k++) {
    const int p = blockIdx.x * HD_PIX + (threadIdx.x >> 5) * HD_PPW + k;
    if (p >= npix) continue;  // warp-uniform
    float4 a[NV], b[NV];
    float sa = 0.f, sb = 0.f;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c4 = lane + 32 * i;
      const bool on = c4 < C / 4;
      a[i] = on ? __ldg(reinterpret_cast<const float4*>(fx + (size_t)p * C) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
      b[i] = on ? __ldg(reinterpret_cast<const float4*>(fy + (size_t)p * C) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
      sa += a[i].x * a[i].x + a[i].y * a[i].y + a[i].z * a[i].z + a[i].w * a[i].w;
      sb += b[i].x * b[i].x + b[i].y * b[i].y + b[i].z * b[i].z + b[i].w * b[i].w;
    }
    const float na = sqrtf(warp_sum(sa)) + NM_EPS, nb = sqrtf(warp_sum(sb)) + NM_EPS;
    float d = 0.f;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const float d0 = a[i].x / na - b[i].x / nb, d1 = a[i].y / na - b[i].y / nb;
      const float d2 = a[i].z / na - b[i].z / nb, d3 = a[i].w / na - b[i].w / nb;
      d += w[i].x * (d0 * d0) + w[i].y * (d1 * d1) + w[i].z * (d2 * d2) + w[i].w * (d3 * d3);
    }
    acc[0] += (double)warp_sum(d);
  }
  block_fold<HD_WARPS * 32>(acc, wsum);
  if (threadIdx.x == 0) part[(size_t)n * gridDim.x + blockIdx.x] = acc[0];
}

struct NmParts {
  const double* sse;
  const double* ssim;
  const double* tap[5];
  int ssim_ctas, tap_ctas[5], tap_pix[5];
};

// one CTA per frame: each run of partials in a fixed order
__global__ void __launch_bounds__(256) nm_reduce_kernel(const NmParts P, int W, int H, float* __restrict__ out) {
  __shared__ double ws[8];
  const int n = blockIdx.x;
  const int per = 3 * P.ssim_ctas;
  double sse[1], ss[1], tap[1], lp = 0.0;
  block_sum_strided<256>(P.sse + (size_t)n * per, per, sse, ws);
  block_sum_strided<256>(P.ssim + (size_t)n * per, per, ss, ws);
  for (int t = 0; t < 5; t++) {
    block_sum_strided<256>(P.tap[t] + (size_t)n * P.tap_ctas[t], P.tap_ctas[t], tap, ws);
    lp += tap[0] / (double)P.tap_pix[t];
  }
  if (threadIdx.x == 0) {
    const double mse = sse[0] / (3.0 * (double)W * (double)H);
    out[3 * n + 0] = (float)(10.0 * log10(1.0 / mse));
    out[3 * n + 1] = (float)(ss[0] / (3.0 * (double)(W - 10) * (double)(H - 10)));
    out[3 * n + 2] = (float)lp;
  }
}

template <int C>
static void nm_head(const float* act, const float* lw, int npix, int N, int ctas, double* part, cudaStream_t st) {
  ProfScope ps(K_MISC, st);
  launch_k(nm_head_kernel<C>, dim3(ctas, N), HD_WARPS * 32, 0, st, false, act, lw, npix, N, part);
}

size_t neuman_scratch_bytes(int W, int H, int N) { return nm_layout(W, H, N).total; }

int launch_neuman_scores(const B2RNeumanScores& p, float* out, void* scratch, cudaStream_t st) {
  const int W = p.width, H = p.height, N = p.n_images, I = 2 * N;
  const NmLayout S = nm_layout(W, H, N);
  char* sc = (char*)scratch;
  float* q = (float*)(sc + S.q);
  const size_t HW = (size_t)W * H;
  {
    ProfScope ps(K_MISC, st);
    launch_k(nm_prep_kernel, (unsigned)((I * HW + 255) / 256), 256, 0, st, false, p.render, p.target, p.mask,
             p.mask_channels, W, H, N, q, (float4*)(sc + S.in0));
  }
  {
    ProfScope ps(K_MISC, st);
    launch_k(nm_ssim_kernel, dim3((W + SS_TW - 1) / SS_TW, (H + SS_TH - 1) / SS_TH, 3 * N), SS_TW * SS_TH, 0, st,
             false, (const float*)q, W, H, N, (double*)(sc + S.sse), (double*)(sc + S.ssim));
  }
  const float* cur = (const float*)(sc + S.in0);
  Dim din{H, W};
  for (int l = 0; l < 5; l++) {
    if (l == 1 || l == 2) {  // pool 1 before conv 2, pool 2 before conv 3
      const Dim dp = nm_act_dim(W, H, l);
      float* y = (float*)(sc + S.pool[l - 1]);
      const size_t n = (size_t)I * dp.h * dp.w * (NM_COUT[l - 1] / 4);
      ProfScope ps(K_MISC, st);
      launch_k(nm_pool_kernel, (unsigned)((n + 255) / 256), 256, 0, st, false, cur, y, din.h, din.w, dp.h, dp.w,
               NM_COUT[l - 1], I);
      cur = y;
      din = dp;
    }
    const Dim d = nm_act_dim(W, H, l);
    float* y = (float*)(sc + S.act[l]);
    const NmConv a{cur, p.w[l], p.bias[l], y, din.h, din.w, NM_CIN[l], d.h, d.w, NM_COUT[l], NM_KS[l], NM_STRIDE[l],
                   NM_PAD[l], nm_kpad(l)};
    {
      ProfScope ps(K_MISC, st);
      launch_k(nm_conv_kernel, dim3((d.h * d.w + NC_M - 1) / NC_M, NM_COUT[l] / NC_N, I), NC_THREADS, 0, st, false, a);
    }
    cur = y;
    din = d;
  }
  NmParts parts;
  parts.sse = (const double*)(sc + S.sse);
  parts.ssim = (const double*)(sc + S.ssim);
  parts.ssim_ctas = nm_ssim_ctas(W, H);
  for (int t = 0; t < 5; t++) {
    const Dim d = nm_act_dim(W, H, t);
    const int ctas = nm_head_ctas(W, H, t), npix = d.h * d.w;
    const float* act = (const float*)(sc + S.act[t]);
    double* part = (double*)(sc + S.part[t]);
    switch (NM_COUT[t]) {
      case 64: nm_head<64>(act, p.lin[t], npix, N, ctas, part, st); break;
      case 192: nm_head<192>(act, p.lin[t], npix, N, ctas, part, st); break;
      case 384: nm_head<384>(act, p.lin[t], npix, N, ctas, part, st); break;
      default: nm_head<256>(act, p.lin[t], npix, N, ctas, part, st); break;
    }
    parts.tap[t] = part;
    parts.tap_ctas[t] = ctas;
    parts.tap_pix[t] = npix;
  }
  {
    ProfScope ps(K_MISC, st);
    launch_k(nm_reduce_kernel, N, 256, 0, st, false, parts, W, H, out);
  }
  return check_launch();
}

}  // namespace b2r
