// compose.cu -- ExAvatar's image composites between the renders and their consumers, in ops that never read anything
// back on the host:
//   * the face composite in front of the rgb_face terms (avatar/main/model.py:200-201, 207-208), forward and backward;
//   * the test-time outputs of Model.forward(mode='test') (model.py:268-276) and, optionally, the bytes test.py's ten
//     cv2.imwrite calls store (main/test.py:40-64), in one launch.
//
// The file is compiled with --fmad=false: every output is torch's fp32 expression rounded operation by operation, so
// the results, signed zeros included, are torch's bits (include/b200raster.h states each expression).
//
// A thread owns CP_PIX = 4 consecutive pixels of the flattened (N, H, W) index, and every output of those pixels, so
// nothing is shared between threads and there are no atomics.  VEC (H W a multiple of 4, 16-byte aligned planes): the
// 4 pixels lie in one frame, every plane is read and written as float4, and each image's 12 bytes of BGR are stored as
// three 4-byte words.  Otherwise each pixel is addressed on its own and its bytes are stored one by one.
#include "common.cuh"

namespace b2r {

constexpr int CP_THREADS = 256;
constexpr int CP_PIX = 4;

// The 4 pixels of plane c of an (N, C, H, W) tensor that start at flattened pixel q; `cnt` of them exist.
template <bool VEC>
__device__ __forceinline__ void cp_load(const float* __restrict__ t, int C, int c, size_t q, size_t HW, int cnt,
                                        float (&v)[CP_PIX]) {
  if (VEC) {
    const size_t n = q / HW;
    const float4 x = __ldg(reinterpret_cast<const float4*>(t + (n * C + c) * HW + (q - n * HW)));
    v[0] = x.x, v[1] = x.y, v[2] = x.z, v[3] = x.w;
  } else {
#pragma unroll
    for (int j = 0; j < CP_PIX; j++) {
      const size_t qj = q + j, n = qj / HW;
      v[j] = j < cnt ? __ldg(t + (n * C + c) * HW + (qj - n * HW)) : 0.f;
    }
  }
}

template <bool VEC>
__device__ __forceinline__ void cp_store(float* __restrict__ t, int C, int c, size_t q, size_t HW, int cnt,
                                         const float (&v)[CP_PIX]) {
  if (VEC) {
    const size_t n = q / HW;
    *reinterpret_cast<float4*>(t + (n * C + c) * HW + (q - n * HW)) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
#pragma unroll
    for (int j = 0; j < CP_PIX; j++) {
      const size_t qj = q + j, n = qj / HW;
      if (j < cnt) t[(n * C + c) * HW + (qj - n * HW)] = v[j];
    }
  }
}

// test.py's bytes of the 4 pixels at q of one (N, H, W, 3) BGR image: pixel j is bytes 3j .. 3j + 2 = B, G, R.
template <bool VEC>
__device__ __forceinline__ void cp_png(uint8_t* __restrict__ img, size_t q, int cnt, const float (&rgb)[3][CP_PIX]) {
  uint32_t s[3 * CP_PIX];
#pragma unroll
  for (int j = 0; j < CP_PIX; j++)
#pragma unroll
    for (int c = 0; c < 3; c++) s[3 * j + c] = (uint32_t)png_u8(rgb[2 - c][j]);
  uint8_t* d = img + q * 3;
  if (VEC) {
    uint32_t* w = reinterpret_cast<uint32_t*>(d);  // q is a multiple of 4: 12-byte steps from a 4-byte aligned base
#pragma unroll
    for (int k = 0; k < 3; k++) w[k] = s[4 * k] | s[4 * k + 1] << 8 | s[4 * k + 2] << 16 | s[4 * k + 3] << 24;
  } else {
#pragma unroll
    for (int k = 0; k < 3 * CP_PIX; k++)
      if (k < 3 * cnt) d[k] = (uint8_t)s[k];
  }
}

// torch's is_face of the training composite: (face[c] != -1) * (face[3] == 1), a bool product cast to float
__device__ __forceinline__ float fc_mask(float f, float f3) { return (f != -1.f && f3 == 1.f) ? 1.f : 0.f; }

template <bool VEC>
__global__ void __launch_bounds__(CP_THREADS) fc_forward_kernel(const float* __restrict__ img,
                                                                const float* __restrict__ face, size_t HW, size_t NP,
                                                                float* __restrict__ out) {
  const size_t q = ((size_t)blockIdx.x * CP_THREADS + threadIdx.x) * CP_PIX;
  if (q >= NP) return;
  const int cnt = (int)min((size_t)CP_PIX, NP - q);
  float f3[CP_PIX];
  cp_load<VEC>(face, 4, 3, q, HW, cnt, f3);
#pragma unroll
  for (int c = 0; c < 3; c++) {
    float x[CP_PIX], f[CP_PIX], o[CP_PIX];
    cp_load<VEC>(img, 3, c, q, HW, cnt, x);
    cp_load<VEC>(face, 4, c, q, HW, cnt, f);
#pragma unroll
    for (int j = 0; j < CP_PIX; j++) {
      const float m = fc_mask(f[j], f3[j]);
      o[j] = x[j] * (1.f - m) + f[j] * m;
    }
    cp_store<VEC>(out, 3, c, q, HW, cnt, o);
  }
}

template <bool VEC>
__global__ void __launch_bounds__(CP_THREADS) fc_backward_kernel(const float* __restrict__ face,
                                                                 const float* __restrict__ dout, size_t HW, size_t NP,
                                                                 float* __restrict__ dimg, float* __restrict__ dface) {
  const size_t q = ((size_t)blockIdx.x * CP_THREADS + threadIdx.x) * CP_PIX;
  if (q >= NP) return;
  const int cnt = (int)min((size_t)CP_PIX, NP - q);
  float f3[CP_PIX];
  cp_load<VEC>(face, 4, 3, q, HW, cnt, f3);
#pragma unroll
  for (int c = 0; c < 3; c++) {
    float g[CP_PIX], f[CP_PIX], a[CP_PIX], b[CP_PIX];
    cp_load<VEC>(dout, 3, c, q, HW, cnt, g);
    cp_load<VEC>(face, 4, c, q, HW, cnt, f);
#pragma unroll
    for (int j = 0; j < CP_PIX; j++) {
      const float m = fc_mask(f[j], f3[j]);
      a[j] = g[j] * (1.f - m);
      b[j] = g[j] * m;
    }
    if (dimg) cp_store<VEC>(dimg, 3, c, q, HW, cnt, a);
    if (dface) cp_store<VEC>(dface, 4, c, q, HW, cnt, b);
  }
  if (dface) {  // face[:, 3:] only enters through `== 1`: torch leaves zeros there
    const float z[CP_PIX] = {0.f, 0.f, 0.f, 0.f};
    cp_store<VEC>(dface, 4, 3, q, HW, cnt, z);
  }
}

struct TestOut {
  float* composite[4];
  uint8_t* png;  // (K, N, H, W, 3) or nullptr
};

// One thread, 4 pixels, every output: the five renders' bytes, the two face composites, the two mask composites (fp32
// and bytes), and gt's bytes.  Inputs read twice (a human render feeds a face and a mask composite) come from L1.
template <bool VEC>
__global__ void __launch_bounds__(CP_THREADS) test_outputs_kernel(const B2RTestOutputs p, const TestOut o, size_t HW,
                                                                  size_t NP) {
  const size_t q = ((size_t)blockIdx.x * CP_THREADS + threadIdx.x) * CP_PIX;
  if (q >= NP) return;
  const int cnt = (int)min((size_t)CP_PIX, NP - q);
  const size_t plane = NP * 3;  // bytes of one image in `png`
  float v[3][CP_PIX];
  if (o.png) {
#pragma unroll
    for (int i = 0; i < 5; i++) {
#pragma unroll
      for (int c = 0; c < 3; c++) cp_load<VEC>(p.render[i], 3, c, q, HW, cnt, v[c]);
      cp_png<VEC>(o.png + i * plane, q, cnt, v);
    }
  }
#pragma unroll
  for (int k = 0; k < 2; k++) {  // human_face_img (k = 0), human_face_img_refined (k = 1)
    const float* human = p.render[1 + 2 * k];
    float f3[CP_PIX];
    cp_load<VEC>(p.face[k], 4, 3, q, HW, cnt, f3);
#pragma unroll
    for (int c = 0; c < 3; c++) {
      float x[CP_PIX], f[CP_PIX];
      cp_load<VEC>(human, 3, c, q, HW, cnt, x);
      cp_load<VEC>(p.face[k], 4, c, q, HW, cnt, f);
#pragma unroll
      for (int j = 0; j < CP_PIX; j++) {
        const float m = (f[j] != -1.f ? 1.f : 0.f) * f3[j];  // the soft mask: -0 where face[3] = -1
        v[c][j] = x[j] * (1.f - m) + f[j] * m;
      }
      cp_store<VEC>(o.composite[k], 3, c, q, HW, cnt, v[c]);
    }
    if (o.png) cp_png<VEC>(o.png + (5 + k) * plane, q, cnt, v);
  }
#pragma unroll
  for (int k = 0; k < 2; k++) {  // scene_human_img_composed (k = 0), scene_human_img_refined_composed (k = 1)
    const float* human = p.render[1 + 2 * k];
    const float* scene_human = p.render[2 + 2 * k];
    float fg[CP_PIX];
    cp_load<VEC>(p.mask[k], 1, 0, q, HW, cnt, fg);
#pragma unroll
    for (int j = 0; j < CP_PIX; j++) fg[j] = fg[j] > 0.9f ? 1.f : 0.f;  // `mask > 0.9` compares in fp32
#pragma unroll
    for (int c = 0; c < 3; c++) {
      float x[CP_PIX], s[CP_PIX];
      cp_load<VEC>(human, 3, c, q, HW, cnt, x);
      cp_load<VEC>(scene_human, 3, c, q, HW, cnt, s);
#pragma unroll
      for (int j = 0; j < CP_PIX; j++) v[c][j] = fg[j] * x[j] + (1.f - fg[j]) * s[j];
      cp_store<VEC>(o.composite[2 + k], 3, c, q, HW, cnt, v[c]);
    }
    if (o.png) cp_png<VEC>(o.png + (7 + k) * plane, q, cnt, v);
  }
  if (o.png && p.gt) {
#pragma unroll
    for (int c = 0; c < 3; c++) cp_load<VEC>(p.gt, 3, c, q, HW, cnt, v[c]);
    cp_png<VEC>(o.png + 9 * plane, q, cnt, v);
  }
}

static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }
static unsigned cp_grid(size_t NP) { return (unsigned)((NP + (size_t)CP_THREADS * CP_PIX - 1) / ((size_t)CP_THREADS * CP_PIX)); }

int launch_face_composite_forward(const B2RFaceComposite& p, float* out, cudaStream_t st) {
  const size_t HW = (size_t)p.width * p.height, NP = HW * p.n_images;
  const bool vec = HW % CP_PIX == 0 && aligned16(p.img) && aligned16(p.face) && aligned16(out);
  ProfScope ps(K_MISC, st);
  if (vec)
    launch_k(fc_forward_kernel<true>, cp_grid(NP), CP_THREADS, 0, st, false, p.img, p.face, HW, NP, out);
  else
    launch_k(fc_forward_kernel<false>, cp_grid(NP), CP_THREADS, 0, st, false, p.img, p.face, HW, NP, out);
  return check_launch();
}

int launch_face_composite_backward(const B2RFaceComposite& p, const float* dout, float* dimg, float* dface,
                                   cudaStream_t st) {
  const size_t HW = (size_t)p.width * p.height, NP = HW * p.n_images;
  const bool vec = HW % CP_PIX == 0 && aligned16(p.face) && aligned16(dout) && aligned16(dimg) && aligned16(dface);
  ProfScope ps(K_MISC, st);
  if (vec)
    launch_k(fc_backward_kernel<true>, cp_grid(NP), CP_THREADS, 0, st, false, p.face, dout, HW, NP, dimg, dface);
  else
    launch_k(fc_backward_kernel<false>, cp_grid(NP), CP_THREADS, 0, st, false, p.face, dout, HW, NP, dimg, dface);
  return check_launch();
}

int launch_test_outputs(const B2RTestOutputs& p, float* const composite[4], uint8_t* png, cudaStream_t st) {
  const size_t HW = (size_t)p.width * p.height, NP = HW * p.n_images;
  TestOut o;
  bool vec = HW % CP_PIX == 0 && aligned16(p.gt) && ((uintptr_t)png & 3) == 0;
  for (int i = 0; i < 5; i++) vec = vec && aligned16(p.render[i]);
  for (int k = 0; k < 2; k++) vec = vec && aligned16(p.mask[k]) && aligned16(p.face[k]);
  for (int k = 0; k < 4; k++) {
    o.composite[k] = composite[k];
    vec = vec && aligned16(composite[k]);
  }
  o.png = png;
  ProfScope ps(K_MISC, st);
  if (vec)
    launch_k(test_outputs_kernel<true>, cp_grid(NP), CP_THREADS, 0, st, false, p, o, HW, NP);
  else
    launch_k(test_outputs_kernel<false>, cp_grid(NP), CP_THREADS, 0, st, false, p, o, HW, NP);
  return check_launch();
}

}  // namespace b2r
