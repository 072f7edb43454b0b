// skin.cu -- standalone linear-blend skinning of one or two Gaussian sets that share a rig (B2RSkin; SURVEY section 8f-2).
//
// ExAvatar poses `mean_3d` and `mean_3d_refined` of its human Gaussians with the same weight rows, joint transforms,
// root translation and camera (avatar/common/nets/module.py:549-557), each through a (P,55) gather, a (P,55)x(55,16)
// matmul into (P,4,4), a bmm and a torch.inverse.  Here one thread per Gaussian blends M = sum_j w_j A_j once
// (skin_blend) and applies it to both canonical sets; the weight rows are read through the (P) row index straight from
// the (V,J) table, never gathered.
//
// Backward: per Gaussian, g_cam = Rinv^T dL/dposed and dL/dx = M3^T g_cam (skin_transpose); M is recomputed, not
// stored.  The joint gradient dL/dA_j[:3,:] = sum_i w_ij sum_s g_cam,s,i [x_s,i, 1]^T is reduced DETERMINISTICALLY:
// each warp accumulates its 32 Gaussians in lane order into a shared-memory (J,12) table (only the non-zero weights of a
// row are visited), the block adds its eight warp tables in warp order and writes one partial row to the scratch, and
// skin_reduce_kernel sums the partials in a fixed order -- no float atomics, bit-identical runs.
//
// Compiled WITHOUT fma contraction (build_ext.py PER_FILE_FLAGS): skin_apply rounds every product and sum on its own,
// so the posed positions the renders read do not move in the last bits.
#include "common.cuh"

namespace b2r {

// Linear-blend skinning (avatar/common/nets/module.py:413-422, 555-557):
//   M = sum_j w_j A_j (rows 0..2 of the 4x4),  posed = M [x,1] + trans,  world = Rinv (posed - t)
// `wrow` is the Gaussian's weight row in the warp's shared-memory stage, `A` the (J,16) row-major joint transforms in
// global memory (warp-uniform addresses: one broadcast line per load).
__device__ __forceinline__ void skin_blend(const float* __restrict__ A, const int J, const float* __restrict__ wrow,
                                           float* M) {
#pragma unroll
  for (int k = 0; k < 12; k++) M[k] = 0.f;
  for (int j = 0; j < J; j++) {
    const float w = wrow[j];
    if (w != 0.f) {  // SMPL-X skinning weights are sparse (a handful of joints per vertex)
#pragma unroll
      for (int k = 0; k < 12; k++) M[k] = fmaf(w, __ldg(A + 16 * j + k), M[k]);
    }
  }
}

// posed = M [x,1] + trans; then Rinv (posed - t) when Rinv is given
__device__ __forceinline__ float3 skin_apply(const float* M, const float3 x, const float* __restrict__ trans,
                                             const float* __restrict__ Rinv, const float* __restrict__ t) {
  float px = M[0] * x.x + M[1] * x.y + M[2] * x.z + M[3] + __ldg(trans);
  float py = M[4] * x.x + M[5] * x.y + M[6] * x.z + M[7] + __ldg(trans + 1);
  float pz = M[8] * x.x + M[9] * x.y + M[10] * x.z + M[11] + __ldg(trans + 2);
  if (Rinv) {
    const float dx = px - __ldg(t), dy = py - __ldg(t + 1), dz = pz - __ldg(t + 2);
    px = __ldg(Rinv) * dx + __ldg(Rinv + 1) * dy + __ldg(Rinv + 2) * dz;
    py = __ldg(Rinv + 3) * dx + __ldg(Rinv + 4) * dy + __ldg(Rinv + 5) * dz;
    pz = __ldg(Rinv + 6) * dx + __ldg(Rinv + 7) * dy + __ldg(Rinv + 8) * dz;
  }
  return make_float3(px, py, pz);
}

// Transpose of skin_apply for one Gaussian, `g` the gradient at the output position:
//   g_cam = Rinv^T g  (g itself without Rinv),  dL/dx = M3^T g_cam;
// the Gaussian's share of dL/dA_j[:3, :] is w_j g_cam [x, 1]^T and of dL/dtrans g_cam.  `gc` may alias `g`.
__device__ __forceinline__ void skin_transpose(const float* M, const float* __restrict__ Rinv, const float* g, float* gc,
                                               float* dx) {
  const float g0 = g[0], g1 = g[1], g2 = g[2];
  if (Rinv) {
    gc[0] = __ldg(Rinv) * g0 + __ldg(Rinv + 3) * g1 + __ldg(Rinv + 6) * g2;
    gc[1] = __ldg(Rinv + 1) * g0 + __ldg(Rinv + 4) * g1 + __ldg(Rinv + 7) * g2;
    gc[2] = __ldg(Rinv + 2) * g0 + __ldg(Rinv + 5) * g1 + __ldg(Rinv + 8) * g2;
  } else {
    gc[0] = g0; gc[1] = g1; gc[2] = g2;
  }
#pragma unroll
  for (int c = 0; c < 3; c++) dx[c] = M[c] * gc[0] + M[4 + c] * gc[1] + M[8 + c] * gc[2];
}

constexpr int SKIN_THREADS = 256;
constexpr int SKIN_WARPS = SKIN_THREADS / 32;
constexpr int SKIN_G_STRIDE = 13;  // per-lane G row in shared memory (12 floats, odd stride)

__host__ __device__ inline int skin_blocks(int P) { return (P + SKIN_THREADS - 1) / SKIN_THREADS; }
__host__ __device__ inline int skin_partial_stride(int J) { return J * 12 + 4; }  // (J,12) joint block + dL/dtrans + pad

// The warp's 32 weight rows into its shared-memory stage (row stride J | 1).  Row i of the Gaussians is row rows[i] of
// the (V,J) table, or row i when `rows` is null.  Row by row: a row is J <= 64 contiguous floats, two per lane, and
// eight rows are in flight at a time (no per-element index division: it dominated an element-wise copy).
__device__ __forceinline__ void stage_weight_rows(float* __restrict__ wstage, const float* __restrict__ W,
                                                  const int32_t* __restrict__ rows, const int J, const int row0,
                                                  const int nrows) {
  const int lane = threadIdx.x & 31;
  const int S = J | 1;
  const int src_row = lane < nrows ? (rows ? __ldg(rows + row0 + lane) : row0 + lane) : 0;
  const bool c0 = lane < J, c1 = lane + 32 < J;
  for (int r0 = 0; r0 < nrows; r0 += 8) {  // warp-uniform trip count: the shuffles need every lane
    float v0[8], v1[8];
#pragma unroll
    for (int u = 0; u < 8; u++) {
      const int r = r0 + u;
      const float* g = W + (size_t)__shfl_sync(0xffffffffu, src_row, r & 31) * J;
      v0[u] = (r < nrows && c0) ? __ldg(g + lane) : 0.f;
      v1[u] = (r < nrows && c1) ? __ldg(g + lane + 32) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 8; u++) {
      const int r = r0 + u;
      if (r < nrows) {
        if (c0) wstage[r * S + lane] = v0[u];
        if (c1) wstage[r * S + lane + 32] = v1[u];
      }
    }
  }
}

__device__ __forceinline__ float3 load3(const float* __restrict__ p, const int i) {
  return make_float3(__ldg(p + 3 * (size_t)i), __ldg(p + 3 * (size_t)i + 1), __ldg(p + 3 * (size_t)i + 2));
}

__global__ void __launch_bounds__(SKIN_THREADS) skin_pose_kernel(const B2RSkin s) {
  extern __shared__ float skin_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row0 = blockIdx.x * SKIN_THREADS + warp * 32;
  const int nrows = min(32, s.P - row0);
  if (nrows <= 0) return;  // warp-uniform
  const int S = s.J | 1;
  float* wstage = skin_smem + (size_t)warp * 32 * S;
  stage_weight_rows(wstage, s.weights, s.rows, s.J, row0, nrows);
  __syncwarp();
  if (lane >= nrows) return;
  const int i = row0 + lane;
  float M[12];
  skin_blend(s.joint_mats, s.J, wstage + lane * S, M);
#pragma unroll
  for (int set = 0; set < 2; set++) {
    float* out = s.posed[set];
    if (!out) continue;
    const float3 p = skin_apply(M, load3(s.xyz[set], i), s.trans, s.cam_Rinv, s.cam_t);
    out[3 * (size_t)i] = p.x;
    out[3 * (size_t)i + 1] = p.y;
    out[3 * (size_t)i + 2] = p.z;
  }
}

struct SkinGrads {
  const float* dposed[2];
  float* dxyz[2];
};

// One partial row per block: partial[block * stride + j*12 + k] = sum over the block's Gaussians of w_ij G_i[k],
// then the block's sum of g_cam at [J*12, J*12 + 3).
__global__ void __launch_bounds__(SKIN_THREADS) skin_pose_bwd_kernel(const B2RSkin s, const SkinGrads g,
                                                                     float* __restrict__ partial) {
  extern __shared__ float skin_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int J = s.J, S = J | 1, JK = J * 12;
  float* wstage = skin_smem + (size_t)warp * 32 * S;
  float* gstage = skin_smem + (size_t)SKIN_WARPS * 32 * S + (size_t)warp * 32 * SKIN_G_STRIDE;
  float* acc_all = skin_smem + (size_t)SKIN_WARPS * 32 * (S + SKIN_G_STRIDE);
  float* acc = acc_all + (size_t)warp * JK;
  for (int t = lane; t < JK; t += 32) acc[t] = 0.f;
  const int row0 = blockIdx.x * SKIN_THREADS + warp * 32;
  const int nrows = max(0, min(32, s.P - row0));
  if (nrows > 0) stage_weight_rows(wstage, s.weights, s.rows, J, row0, nrows);
  __syncwarp();

  float G[12];
#pragma unroll
  for (int k = 0; k < 12; k++) G[k] = 0.f;
  if (lane < nrows) {
    const int i = row0 + lane;
    float M[12];
    skin_blend(s.joint_mats, J, wstage + lane * S, M);
#pragma unroll
    for (int set = 0; set < 2; set++) {
      float dx[3] = {0.f, 0.f, 0.f};
      if (g.dposed[set]) {
        const float3 gp = load3(g.dposed[set], i);
        const float gw[3] = {gp.x, gp.y, gp.z};
        float gc[3];
        skin_transpose(M, s.cam_Rinv, gw, gc, dx);
        const float3 x = load3(s.xyz[set], i);
        const float xs[4] = {x.x, x.y, x.z, 1.f};
#pragma unroll
        for (int r = 0; r < 3; r++)
#pragma unroll
          for (int c = 0; c < 4; c++) G[4 * r + c] = fmaf(gc[r], xs[c], G[4 * r + c]);
      }
      if (float* d = g.dxyz[set]) {
        d[3 * (size_t)i] = dx[0];
        d[3 * (size_t)i + 1] = dx[1];
        d[3 * (size_t)i + 2] = dx[2];
      }
    }
  }
  if (!partial) return;  // no joint / translation gradient requested (block-uniform)

  // the warp's Gaussians one after the other (lane order), each over its non-zero weights: lane k < 12 owns column k
#pragma unroll
  for (int k = 0; k < 12; k++) gstage[lane * SKIN_G_STRIDE + k] = G[k];
  __syncwarp();
  for (int src = 0; src < nrows; src++) {
    const float* w = wstage + src * S;
    unsigned lo = __ballot_sync(0xffffffffu, lane < J && w[lane] != 0.f);
    unsigned hi = __ballot_sync(0xffffffffu, lane + 32 < J && w[lane + 32] != 0.f);
    const float gk = lane < 12 ? gstage[src * SKIN_G_STRIDE + lane] : 0.f;
    while (lo) {
      const int j = __ffs(lo) - 1;
      lo &= lo - 1;
      if (lane < 12) acc[j * 12 + lane] = fmaf(w[j], gk, acc[j * 12 + lane]);
    }
    while (hi) {
      const int j = 32 + __ffs(hi) - 1;
      hi &= hi - 1;
      if (lane < 12) acc[j * 12 + lane] = fmaf(w[j], gk, acc[j * 12 + lane]);
    }
  }
  // dL/dtrans: the block's sum of g_cam = G[:, 3], a warp_sum per warp
  float t3[3] = {G[3], G[7], G[11]};
#pragma unroll
  for (int c = 0; c < 3; c++) t3[c] = warp_sum(t3[c]);
  __shared__ float wtrans[SKIN_WARPS][3];
  if (lane == 0) { wtrans[warp][0] = t3[0]; wtrans[warp][1] = t3[1]; wtrans[warp][2] = t3[2]; }
  __syncthreads();
  float* prow = partial + (size_t)blockIdx.x * skin_partial_stride(J);
  for (int t = threadIdx.x; t < JK; t += SKIN_THREADS) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < SKIN_WARPS; w++) v += acc_all[(size_t)w * JK + t];
    prow[t] = v;
  }
  if (threadIdx.x < 3) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < SKIN_WARPS; w++) v += wtrans[w][threadIdx.x];
    prow[JK + threadIdx.x] = v;
  }
}

// Second stage: output o of the (J*12 + 3) joint / translation gradient = sum of the block partials, each warp over
// every eighth block, the eight warp sums in warp order.
__global__ void __launch_bounds__(SKIN_THREADS) skin_reduce_kernel(const float* __restrict__ partial, const int nblocks,
                                                                   const int J, float* __restrict__ djoint,
                                                                   float* __restrict__ dtrans) {
  __shared__ float wsum[SKIN_WARPS][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int JK = J * 12, n_out = JK + 3, stride = skin_partial_stride(J);
  const int o = blockIdx.x * 32 + lane;
  float v = 0.f;
  if (o < n_out)
    for (int b = warp; b < nblocks; b += SKIN_WARPS) v += __ldg(partial + (size_t)b * stride + o);
  wsum[warp][lane] = v;
  __syncthreads();
  if (warp == 0 && o < n_out) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < SKIN_WARPS; w++) t += wsum[w][lane];
    if (o < JK) {
      if (djoint) djoint[o] = t;
    } else if (dtrans) {
      dtrans[o - JK] = t;
    }
  }
}

size_t skin_scratch_bytes(int P, int J) {
  return align_up((size_t)(P > 0 ? skin_blocks(P) : 1) * skin_partial_stride(J > 0 ? J : 1) * sizeof(float));
}

static size_t stage_bytes(int J) { return (size_t)SKIN_WARPS * 32 * (J | 1) * sizeof(float); }

int launch_skin_forward(const B2RSkin& s, cudaStream_t st) {
  ProfScope p(K_MISC, st, s.P > 0 ? 1 : 0);
  if (s.P > 0) {
    cudaFuncSetAttribute(skin_pose_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);  // per device
    launch_k(skin_pose_kernel, skin_blocks(s.P), SKIN_THREADS, stage_bytes(s.J), st, true, s);
  }
  return check_launch();
}

int launch_skin_backward(const B2RSkin& s, const float* const dposed[2], float* const dxyz[2], float* djoint,
                         float* dtrans, void* scratch, cudaStream_t st) {
  const bool reduce = djoint != nullptr || dtrans != nullptr;
  SkinGrads g;
  for (int k = 0; k < 2; k++) {
    g.dposed[k] = dposed ? dposed[k] : nullptr;
    g.dxyz[k] = dxyz ? dxyz[k] : nullptr;
  }
  const int nb = s.P > 0 ? skin_blocks(s.P) : 0;
  if (nb > 0 && (reduce || g.dxyz[0] || g.dxyz[1])) {
    ProfScope p(K_MISC, st);
    const size_t smem = stage_bytes(s.J) + (size_t)SKIN_WARPS * 32 * SKIN_G_STRIDE * sizeof(float) +
                        (size_t)SKIN_WARPS * s.J * 12 * sizeof(float);
    cudaFuncSetAttribute(skin_pose_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024);
    launch_k(skin_pose_bwd_kernel, nb, SKIN_THREADS, smem, st, true, s, g, reduce ? (float*)scratch : nullptr);
  }
  if (reduce) {  // also for P == 0: the gradients are then zero
    ProfScope p(K_MISC, st);
    launch_k(skin_reduce_kernel, (s.J * 12 + 3 + 31) / 32, SKIN_THREADS, 0, st, true, (const float*)scratch, nb, s.J,
             djoint, dtrans);
  }
  return check_launch();
}

}  // namespace b2r
