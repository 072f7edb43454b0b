// adam.cu -- one Adam step over every parameter tensor of an optimizer in a single launch (exavatar_release_b200/optim.py
// Adam), element for element the arithmetic of torch.optim.Adam's default foreach path (torch/optim/adam.py
// _multi_tensor_adam with capturable=False, amsgrad=False, weight_decay=0).
//
// The caller's device table holds one B2RAdamSegment per tensor with a gradient: the four pointers, numel, the
// segment's first chunk, the param's row layout (contiguous, or the rows of a strided view such as ExAvatar's
// feature_dc / feature_rest) and its six fp32 scalars, computed on the host in double with torch's expressions and
// rounded once.  CTA b owns chunk b (ADAM_CHUNK elements) of the segment whose [first_chunk, first_chunk + chunks) holds b, found
// by a binary search over first_chunk; a 3-element tensor and a 7.9 M-element one share the launch, and there is no cap
// on the number of tensors.
//
// Per element, the seven foreach ops in their order and with their roundings (ATen/native/Lerp.h,
// ATen/native/cuda/ForeachFunctors.cuh, DeviceAddCmulCdiv.cuh, and the sm_90 SASS of those kernels in libtorch_cuda.so):
//   _foreach_lerp_(m, g, w)        |w| < 0.5: fma(w, g - m, m)        else: fma(-(g - m), 1 - w, g)    (FFMA in the SASS)
//   _foreach_mul_(v, beta2)        v * beta2
//   _foreach_addcmul_(v, g, g, c)  c == 1: fma(g, g, v)               else: fma(c, g * g, v)           (std::fma)
//   _foreach_sqrt                  s = sqrt(v)                                                          (IEEE)
//   _foreach_div_(s, bc2_sqrt)     s / bc2_sqrt                                                         (IEEE division)
//   _foreach_add_(s, eps)          s + eps
//   _foreach_addcdiv_(p, m, s, a)  fma(a, m / s, p); for a == 1 torch rounds p + m / s, which is the same value
// The unit is compiled with --fmad=false so that only the __fmaf_rn calls below are fused.
#include "common.cuh"

namespace b2r {

constexpr int ADAM_THREADS = 256;

__device__ __forceinline__ void adam_element(float& p, const float g, float& m, float& v, const B2RAdamSegment& s) {
  const float d = g - m;
  m = fabsf(s.lerp_weight) < 0.5f ? __fmaf_rn(s.lerp_weight, d, m) : __fmaf_rn(-d, 1.f - s.lerp_weight, g);
  v = v * s.beta2;
  v = s.one_minus_beta2 == 1.f ? __fmaf_rn(g, g, v) : __fmaf_rn(s.one_minus_beta2, g * g, v);
  float q = sqrtf(v);
  q = __fdiv_rn(q, s.bc2_sqrt);
  q = q + s.eps;
  p = __fmaf_rn(s.step_size, __fdiv_rn(m, q), p);
}

__global__ void __launch_bounds__(ADAM_THREADS) adam_step_kernel(const B2RAdamSegment* __restrict__ table, const int n) {
  __shared__ B2RAdamSegment seg;
  if (threadIdx.x == 0) {
    int lo = 0, hi = n - 1;  // the last segment whose first_chunk <= blockIdx.x (empty segments share it with the next)
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (table[mid].first_chunk <= (int64_t)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    seg = table[lo];
  }
  __syncthreads();
  const int64_t base = ((int64_t)blockIdx.x - seg.first_chunk) * B2R_ADAM_CHUNK;
  // a table whose first_chunk does not match its numel, or whose row layout is not one, writes nothing
  if (base < 0 || base >= seg.numel || seg.row_len <= 0 || seg.row_stride < seg.row_len) return;
  const int len = (int)min((int64_t)B2R_ADAM_CHUNK, seg.numel - base);
  float* __restrict__ p = seg.param + base;
  const float* __restrict__ g = seg.grad + base;
  float* __restrict__ m = seg.exp_avg + base;
  float* __restrict__ v = seg.exp_avg_sq + base;
  if (seg.row_stride != seg.row_len) {  // a strided param view: rows of row_len floats, row_stride apart
    for (int i = threadIdx.x; i < len; i += ADAM_THREADS) {
      const int64_t e = base + i;
      float* pe = seg.param + (e / seg.row_len) * seg.row_stride + e % seg.row_len;
      float P = *pe, M = m[i], V = v[i];
      adam_element(P, __ldcs(g + i), M, V, seg);
      *pe = P;
      m[i] = M;
      v[i] = V;
    }
    return;
  }
  // B2R_ADAM_CHUNK is a multiple of 4, so every chunk of an aligned segment starts on a 16-byte boundary
  const bool vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                     reinterpret_cast<uintptr_t>(v)) & 15) == 0;
  int done = 0;
  if (vec) {
    const int nv = len >> 2;
#pragma unroll 4
    for (int i = threadIdx.x; i < nv; i += ADAM_THREADS) {
      float4 P = reinterpret_cast<float4*>(p)[i];
      const float4 G = __ldcs(reinterpret_cast<const float4*>(g) + i);
      float4 M = reinterpret_cast<float4*>(m)[i];
      float4 V = reinterpret_cast<float4*>(v)[i];
      adam_element(P.x, G.x, M.x, V.x, seg);
      adam_element(P.y, G.y, M.y, V.y, seg);
      adam_element(P.z, G.z, M.z, V.z, seg);
      adam_element(P.w, G.w, M.w, V.w, seg);
      reinterpret_cast<float4*>(p)[i] = P;
      reinterpret_cast<float4*>(m)[i] = M;
      reinterpret_cast<float4*>(v)[i] = V;
    }
    done = nv << 2;
  }
  for (int i = done + threadIdx.x; i < len; i += ADAM_THREADS) {
    float P = p[i], M = m[i], V = v[i];
    adam_element(P, __ldcs(g + i), M, V, seg);
    p[i] = P;
    m[i] = M;
    v[i] = V;
  }
}

int launch_adam_step(const B2RAdamSegment* table, int n_segments, int64_t n_chunks, cudaStream_t st) {
  ProfScope ps(K_MISC, st);
  launch_k(adam_step_kernel, (unsigned)n_chunks, ADAM_THREADS, 0, st, false, table, n_segments);
  return check_launch();
}

}  // namespace b2r
