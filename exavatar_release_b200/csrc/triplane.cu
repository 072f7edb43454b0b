// triplane.cu -- HumanGaussian.extract_tri_feature (avatar/common/nets/module.py:424-457): three bilinear
// F.grid_sample reads (align_corners=False, zero padding) of a (3,C,H,W) triplane per row, with the face rows read from
// the face triplane instead.  The sample positions never change (pos_enc_mesh is a fixed buffer), so the caller
// computes every row's four corners and weights per plane once (exavatar_release_b200/human_nets.py TriplaneFeatures):
//   triplane_fwd_kernel  one thread per output element feat[r][p*C + c] = sum_k w[r][p][k] T[p][c][texel[r][p][k]]
//                        over the in-bounds corners in grid_sample's order (nw, ne, sw, se).
//   triplane_bwd_kernel  one warp per (triplane, plane, texel): the gradient of the texel's C channels is the sum, over
//                        the texel's CSR entries (rows ascending), of w dL/dfeat[row] -- a gather, no float atomics, so
//                        two runs are bit-identical.  Face rows are entries of the face triplane only.
#include "common.cuh"

namespace b2r {

constexpr int TP_THREADS = 256;

__global__ void __launch_bounds__(TP_THREADS) triplane_fwd_kernel(const int P, const int C, const int HW,
                                                                  const float* __restrict__ planes,
                                                                  const float* __restrict__ planes_face,
                                                                  const uint8_t* __restrict__ is_face,
                                                                  const int32_t* __restrict__ corners,
                                                                  const float* __restrict__ weights,
                                                                  float* __restrict__ feat) {
  const int64_t e = (int64_t)blockIdx.x * TP_THREADS + threadIdx.x;
  const int cols = 3 * C;
  if (e >= (int64_t)P * cols) return;
  const int r = (int)(e / cols), col = (int)(e % cols), p = col / C, c = col % C;
  const float* T = (is_face && is_face[r] ? planes_face : planes) + ((size_t)p * C + c) * HW;
  const int32_t* ci = corners + ((size_t)r * 3 + p) * 4;
  const float* wi = weights + ((size_t)r * 3 + p) * 4;
  float f = 0.f;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int idx = __ldg(ci + k);
    if (idx >= 0) f += __ldg(T + idx) * __ldg(wi + k);
  }
  feat[e] = f;
}

__global__ void __launch_bounds__(TP_THREADS) triplane_bwd_kernel(const int C, const int HW, const int cols,
                                                                  const float* __restrict__ dfeat,
                                                                  const int32_t* __restrict__ offsets,
                                                                  const int32_t* __restrict__ rows,
                                                                  const float* __restrict__ w,
                                                                  float* __restrict__ dplanes,
                                                                  float* __restrict__ dplanes_face) {
  const int64_t key = ((int64_t)blockIdx.x * TP_THREADS + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (key >= (int64_t)6 * HW) return;
  const int s = (int)(key / (3 * HW)), p = (int)((key / HW) % 3), texel = (int)(key % HW);
  float* out = (s ? dplanes_face : dplanes) + (size_t)p * C * HW + texel;
  const int e0 = offsets[key], e1 = offsets[key + 1];
  for (int c = lane; c < C; c += 32) {
    float acc = 0.f;
    for (int e = e0; e < e1; e++) acc += __ldg(w + e) * __ldg(dfeat + (size_t)__ldg(rows + e) * cols + p * C + c);
    out[(size_t)c * HW] = acc;
  }
}

int launch_triplane_forward(int P, int C, int H, int W, const float* planes, const float* planes_face,
                            const uint8_t* is_face, const int32_t* corners, const float* weights, float* feat,
                            cudaStream_t st) {
  ProfScope p(K_MISC, st);
  const int64_t n = (int64_t)P * 3 * C;
  launch_k(triplane_fwd_kernel, (unsigned)((n + TP_THREADS - 1) / TP_THREADS), TP_THREADS, 0, st, false, P, C, H * W,
           planes, planes_face, is_face, corners, weights, feat);
  return check_launch();
}

int launch_triplane_backward(int C, int H, int W, const float* dfeat, const int32_t* offsets, const int32_t* rows,
                             const float* w, float* dplanes, float* dplanes_face, cudaStream_t st) {
  ProfScope p(K_MISC, st);
  const int64_t n = (int64_t)6 * H * W * 32;
  launch_k(triplane_bwd_kernel, (unsigned)((n + TP_THREADS - 1) / TP_THREADS), TP_THREADS, 0, st, false, C, H * W,
           3 * C, dfeat, offsets, rows, w, dplanes, dplanes_face);
  return check_launch();
}

}  // namespace b2r
