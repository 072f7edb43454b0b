// frames.cu -- FrameTable's unpack (exavatar_release_b200/frames.py): every training frame of a split lives on the
// device as uint8 RGB + mask, and one launch expands the frame of a slot into the fp32 tensors ExAvatar's DataLoader
// would have collated, so the frame's data is read inside a captured training iteration instead of copied in from the
// host.  The slot is read on the device and mapped to a row through the table's slot -> row map.
//
// The image is fl(k / 255) per byte k, the IEEE-rounded quotient (__fdiv_rn): the fp32 value of ToTensor(img) / 255.
// in NeuMan / Custom __getitem__.  A product with the rounded reciprocal of 255 differs from it for 126 of the 256
// byte values.  The kernel is bandwidth-bound: 4 bytes in and 16 bytes out per pixel.
#include "common.cuh"

namespace b2r {

constexpr int FU_THREADS = 256;
constexpr int FU_META = 4 + 9 + 3 + 2 + 2;  // bbox, R, t, focal, princpt

// the row of the table's slot: *slot on the device, or host_slot; -1 for a slot outside [0, n_slots) or without a row
__device__ __forceinline__ int frame_row(const B2RFrameTable& t) {
  const int s = t.slot ? __ldg(t.slot) : t.host_slot;
  const int r = s >= 0 && s < t.n_slots ? __ldg(t.slot_row + s) : -1;
  return r >= 0 && r < t.n_rows ? r : -1;
}

__device__ __forceinline__ float unit(uint32_t k) { return __fdiv_rn((float)k, 255.f); }

// One thread per 4 pixels.  VEC: one 16-byte load of the 4 pixels and one float4 store per plane (H*W % 4 == 0 and
// 16-byte aligned arrays); otherwise byte loads and scalar stores, with the last quad cut at H*W.  Block 0's first
// FU_META + 1 threads also write the row's box, camera and frame index.
template <bool VEC>
__global__ void __launch_bounds__(FU_THREADS) frame_unpack_kernel(const B2RFrameTable t, float* __restrict__ img,
                                                                 float* __restrict__ mask, float* __restrict__ bbox,
                                                                 float* __restrict__ R, float* __restrict__ tr,
                                                                 float* __restrict__ focal,
                                                                 float* __restrict__ princpt,
                                                                 int64_t* __restrict__ frame_idx) {
  const int r = frame_row(t);
  const float nan = __int_as_float(0x7fc00000);
  if (blockIdx.x == 0 && threadIdx.x <= FU_META) {
    const int i = threadIdx.x;
    if (i == FU_META) {
      frame_idx[0] = r >= 0 ? __ldg(t.frame_idx + r) : -1;
    } else {
      const float* src;
      float* dst;
      int k, n;
      if (i < 4) src = t.bbox, dst = bbox, k = i, n = 4;
      else if (i < 13) src = t.R, dst = R, k = i - 4, n = 9;
      else if (i < 16) src = t.t, dst = tr, k = i - 13, n = 3;
      else if (i < 18) src = t.focal, dst = focal, k = i - 16, n = 2;
      else src = t.princpt, dst = princpt, k = i - 18, n = 2;
      dst[k] = r >= 0 ? __ldg(src + (int64_t)r * n + k) : nan;
    }
  }
  const int64_t HW = (int64_t)t.height * t.width;
  const int64_t q = (int64_t)blockIdx.x * FU_THREADS + threadIdx.x;
  if (4 * q >= HW) return;
  const uint8_t* px = t.pixels + (r >= 0 ? (int64_t)r * HW * 4 : 0);
  if (VEC) {
    float4 c[4];
    if (r >= 0) {
      const uint4 w = __ldg(reinterpret_cast<const uint4*>(px) + q);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const int s = 8 * ch;
        c[ch] = make_float4(unit((w.x >> s) & 255u), unit((w.y >> s) & 255u), unit((w.z >> s) & 255u),
                            unit((w.w >> s) & 255u));
      }
      c[3] = make_float4((float)(w.x >> 24), (float)(w.y >> 24), (float)(w.z >> 24), (float)(w.w >> 24));
    } else {
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) c[ch] = make_float4(nan, nan, nan, nan);
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) reinterpret_cast<float4*>(img + ch * HW)[q] = c[ch];
    reinterpret_cast<float4*>(mask)[q] = c[3];
  } else {
    const int64_t end = min(4 * q + 4, HW);
    for (int64_t p = 4 * q; p < end; ++p) {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) img[ch * HW + p] = r >= 0 ? unit(__ldg(px + 4 * p + ch)) : nan;
      mask[p] = r >= 0 ? (float)__ldg(px + 4 * p + 3) : nan;
    }
  }
}

static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

int launch_frame_unpack(const B2RFrameTable& t, float* img, float* mask, float* bbox, float* R, float* tr, float* focal,
                        float* princpt, int64_t* frame_idx, cudaStream_t st) {
  const int64_t HW = (int64_t)t.height * t.width;
  const unsigned blocks = (unsigned)((HW + 4 * FU_THREADS - 1) / (4 * FU_THREADS));
  const bool vec = HW % 4 == 0 && aligned16(t.pixels) && aligned16(img) && aligned16(mask);
  ProfScope ps(K_MISC, st);
  if (vec)
    launch_k(frame_unpack_kernel<true>, blocks, FU_THREADS, 0, st, false, t, img, mask, bbox, R, tr, focal, princpt,
             frame_idx);
  else
    launch_k(frame_unpack_kernel<false>, blocks, FU_THREADS, 0, st, false, t, img, mask, bbox, R, tr, focal, princpt,
             frame_idx);
  return check_launch();
}

}  // namespace b2r
