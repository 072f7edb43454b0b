// scene_assets.cu -- the asset dict of ExAvatar's SceneGaussian.forward (avatar/common/nets/module.py:253-272) from the
// scene's stored parameters, forward and backward, one thread per Gaussian (exavatar_release_b200/scene_assets.py).
//
// Per Gaussian:
//   opacity  = sigmoid(logit) = 1 / (1 + exp(-logit))          backward: g * (1 - opacity) * opacity (torch's form)
//   scale    = exp(log_scale)                                   backward: g * scale
//   rotation = matrix_to_quaternion(rotation_6d_to_matrix(a))   pytorch3d 0.7.5, restated in smplx_rig.py
//   shs mode: shs = cat(feature_dc, feature_rest, 1)            (P,M,3)
//   rgb mode: rgb = clamp_min(eval_sh(deg, sh, normalize(mean - campos)) + 0.5, 0), campos = -R^-1 t by cofactors
// The backward is autograd's through those formulas: the quaternion's derivative runs through the selected candidate
// only (its q_abs in the denominator included, zero where 1 +- m00 +- m11 +- m22 <= 0), clamp_min passes the gradient
// where x >= 0, coefficients above the degree get exact zeros, and `mean` gets the view-direction term.
//
// A CTA stages its SA_THREADS rows of every array through shared memory, so global reads and writes walk consecutive
// floats (feature_dc / feature_rest are read through their row strides); each thread then works on its own row, with
// the row stride in shared memory odd so the per-thread accesses are free of bank conflicts.  The degree is read from
// the caller's float buffer on the device: one captured graph serves every degree.  A degree outside 0..3, or one that
// needs more than M coefficients, gives NaN colours (and NaN colour gradients) and reads no coefficient beyond M.
// No atomics, no allocation, no sync; the unit is compiled with --fmad=false, so every fp32 product and sum is rounded
// as torch rounds the same expression.  The rotation alone is evaluated in fp64 (rot6d.cuh).
#include "common.cuh"
#include "rot6d.cuh"

namespace b2r {

constexpr int SA_THREADS = 128;
constexpr int SA_SH = 3 * B2R_SCENE_MAX_COEFFS + 1;  // staged SH row: 3M floats, odd stride
constexpr float SH_C0 = 0.28209479177387814f;
constexpr float SH_C1 = 0.4886025119029199f;
__constant__ float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f,
                               0.5462742152960396f};
__constant__ float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                               -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

// rows [r0, r0 + n) of L floats, `stride` floats apart, into shared rows of Ls floats (a null source reads zeros)
__device__ __forceinline__ void load_rows(float* sm, int Ls, const float* __restrict__ g, int64_t stride, int L,
                                          int64_t r0, int n) {
  for (int i = threadIdx.x; i < n * L; i += SA_THREADS) {
    const int r = i / L, c = i - r * L;
    sm[r * Ls + c] = g ? __ldg(g + (r0 + r) * stride + c) : 0.f;
  }
}
// shared rows -> rows [r0, r0 + n) of a contiguous (rows, L) array
__device__ __forceinline__ void store_rows(float* __restrict__ g, int L, const float* sm, int Ls, int64_t r0, int n) {
  for (int i = threadIdx.x; i < n * L; i += SA_THREADS) {
    const int r = i / L, c = i - r * L;
    g[r0 * L + i] = sm[r * Ls + c];
  }
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// F.normalize's divisor max(|v|, 1e-12) and |v|
__device__ __forceinline__ float norm3(const float* v) { return sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

// basis functions used at degree `deg` (ExAvatar's eval_sh compares the float buffer: deg > 0, > 1, > 2), or 0 for a
// degree the op does not take (outside 0..3, NaN, or more coefficients than M -- a fractional degree such as 2.5 passes
// eval_sh's (deg + 1)^2 <= M assert and still reads 16)
__device__ __forceinline__ int sh_basis_count(float deg, int M) {
  if (!(deg >= 0.f && deg <= 3.f && (deg + 1.f) * (deg + 1.f) <= (float)M)) return 0;
  const int nb = deg > 2.f ? 16 : deg > 1.f ? 9 : deg > 0.f ? 4 : 1;
  return nb <= M ? nb : 0;
}

// basis value k at unit direction (x, y, z) and its gradient
__device__ __forceinline__ float sh_basis(int k, float x, float y, float z, float* g) {
  const float xx = x * x, yy = y * y, zz = z * z;
  switch (k) {
    case 0: g[0] = g[1] = g[2] = 0.f; return SH_C0;
    case 1: g[0] = 0.f; g[1] = -SH_C1; g[2] = 0.f; return -SH_C1 * y;
    case 2: g[0] = 0.f; g[1] = 0.f; g[2] = SH_C1; return SH_C1 * z;
    case 3: g[0] = -SH_C1; g[1] = 0.f; g[2] = 0.f; return -SH_C1 * x;
    case 4: g[0] = SH_C2[0] * y; g[1] = SH_C2[0] * x; g[2] = 0.f; return SH_C2[0] * (x * y);
    case 5: g[0] = 0.f; g[1] = SH_C2[1] * z; g[2] = SH_C2[1] * y; return SH_C2[1] * (y * z);
    case 6:
      g[0] = SH_C2[2] * (-2.f * x); g[1] = SH_C2[2] * (-2.f * y); g[2] = SH_C2[2] * (4.f * z);
      return SH_C2[2] * (2.f * zz - xx - yy);
    case 7: g[0] = SH_C2[3] * z; g[1] = 0.f; g[2] = SH_C2[3] * x; return SH_C2[3] * (x * z);
    case 8: g[0] = SH_C2[4] * (2.f * x); g[1] = SH_C2[4] * (-2.f * y); g[2] = 0.f; return SH_C2[4] * (xx - yy);
    case 9:
      g[0] = SH_C3[0] * (6.f * x * y); g[1] = SH_C3[0] * (3.f * xx - 3.f * yy); g[2] = 0.f;
      return SH_C3[0] * y * (3.f * xx - yy);
    case 10:
      g[0] = SH_C3[1] * (y * z); g[1] = SH_C3[1] * (x * z); g[2] = SH_C3[1] * (x * y);
      return SH_C3[1] * (x * y) * z;
    case 11:
      g[0] = SH_C3[2] * (-2.f * x * y); g[1] = SH_C3[2] * (4.f * zz - xx - 3.f * yy); g[2] = SH_C3[2] * (8.f * y * z);
      return SH_C3[2] * y * (4.f * zz - xx - yy);
    case 12:
      g[0] = SH_C3[3] * (-6.f * x * z); g[1] = SH_C3[3] * (-6.f * y * z); g[2] = SH_C3[3] * (6.f * zz - 3.f * xx - 3.f * yy);
      return SH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy);
    case 13:
      g[0] = SH_C3[4] * (4.f * zz - 3.f * xx - yy); g[1] = SH_C3[4] * (-2.f * x * y); g[2] = SH_C3[4] * (8.f * x * z);
      return SH_C3[4] * x * (4.f * zz - xx - yy);
    case 14:
      g[0] = SH_C3[5] * (2.f * x * z); g[1] = SH_C3[5] * (-2.f * y * z); g[2] = SH_C3[5] * (xx - yy);
      return SH_C3[5] * z * (xx - yy);
    default:
      g[0] = SH_C3[6] * (3.f * xx - 3.f * yy); g[1] = SH_C3[6] * (-6.f * x * y); g[2] = 0.f;
      return SH_C3[6] * x * (xx - 3.f * yy);
  }
}

// -R^-1 t by cofactors (rasterizer._inv3's expressions)
__device__ __forceinline__ void cam_position(const float* __restrict__ R, const float* __restrict__ t, float* c) {
  const float a = __ldg(R + 0), b = __ldg(R + 1), cc = __ldg(R + 2), d = __ldg(R + 3), e = __ldg(R + 4),
              f = __ldg(R + 5), g = __ldg(R + 6), h = __ldg(R + 7), i = __ldg(R + 8);
  const float adj[9] = {e * i - f * h, cc * h - b * i, b * f - cc * e, f * g - d * i, a * i - cc * g, cc * d - a * f,
                        d * h - e * g, b * g - a * h, a * e - b * d};
  const float det = a * (e * i - f * h) - b * (d * i - f * g) + cc * (d * h - e * g);
  const float t0 = __ldg(t + 0), t1 = __ldg(t + 1), t2 = __ldg(t + 2);
  for (int r = 0; r < 3; ++r) c[r] = -((adj[3 * r] / det) * t0 + (adj[3 * r + 1] / det) * t1 + (adj[3 * r + 2] / det) * t2);
}

struct FwdSmem {
  float rot[SA_THREADS * 7];  // rot6d in, quaternion out
  float op[SA_THREADS];       // logit in, opacity out
  float sc[SA_THREADS * 3];   // log_scale in, scale out
  float sh[SA_THREADS * SA_SH];
  float mean[SA_THREADS * 3];  // mean in, rgb out
};

__global__ void __launch_bounds__(SA_THREADS) scene_assets_fwd_kernel(const B2RSceneAssets s, float* __restrict__ opacity,
                                                                      float* __restrict__ scale,
                                                                      float* __restrict__ rotation,
                                                                      float* __restrict__ color) {
  __shared__ FwdSmem sm;
  const int64_t r0 = (int64_t)blockIdx.x * SA_THREADS;
  const int n = (int)min((int64_t)SA_THREADS, (int64_t)s.P - r0);
  const int M = s.M, Ls = 3 * M | 1;
  const bool rgb = s.cam_R != nullptr;
  load_rows(sm.rot, 7, s.rotation6d, 6, 6, r0, n);
  load_rows(sm.op, 1, s.opacity_logit, 1, 1, r0, n);
  load_rows(sm.sc, 3, s.log_scale, 3, 3, r0, n);
  load_rows(sm.sh, Ls, s.feature_dc, s.dc_stride, 3, r0, n);
  if (M > 1) load_rows(sm.sh + 3, Ls, s.feature_rest, s.rest_stride, 3 * (M - 1), r0, n);
  if (rgb) load_rows(sm.mean, 3, s.mean, 3, 3, r0, n);
  __syncthreads();
  const int j = threadIdx.x;
  if (j < n) {
    sm.op[j] = sigmoidf_(sm.op[j]);
    for (int i = 0; i < 3; ++i) sm.sc[3 * j + i] = expf(sm.sc[3 * j + i]);
    double a[6];
    for (int i = 0; i < 6; ++i) a[i] = sm.rot[7 * j + i];
    Rot6d r;
    rot6d_forward(a, r);
    Quat o;
    quat_forward(r, o);
    for (int i = 0; i < 4; ++i) sm.rot[7 * j + i] = (float)o.q[i];
    if (rgb) {
      float c[3], v[3];
      cam_position(s.cam_R, s.cam_t, c);
      for (int i = 0; i < 3; ++i) v[i] = sm.mean[3 * j + i] - c[i];
      const float dn = fmaxf(norm3(v), 1e-12f);
      const float x = v[0] / dn, y = v[1] / dn, z = v[2] / dn;
      const int nb = sh_basis_count(__ldg(s.active_sh_degree), M);
      float res[3] = {0.f, 0.f, 0.f}, g[3];
      const float* row = sm.sh + Ls * j;
      for (int k = 0; k < nb; ++k) {
        const float b = sh_basis(k, x, y, z, g);
        for (int ch = 0; ch < 3; ++ch) res[ch] = k == 0 ? b * row[ch] : res[ch] + b * row[3 * k + ch];
      }
      for (int ch = 0; ch < 3; ++ch) sm.mean[3 * j + ch] = nb ? fmaxf(res[ch] + 0.5f, 0.f) : __int_as_float(0x7fc00000);
    }
  }
  __syncthreads();
  store_rows(opacity, 1, sm.op, 1, r0, n);
  store_rows(scale, 3, sm.sc, 3, r0, n);
  store_rows(rotation, 4, sm.rot, 7, r0, n);
  if (rgb) store_rows(color, 3, sm.mean, 3, r0, n);
  else store_rows(color, 3 * M, sm.sh, Ls, r0, n);
}

struct BwdSmem {
  float rot[SA_THREADS * 7];  // rot6d in, d rot6d out
  float grot[SA_THREADS * 5];
  float op[SA_THREADS];       // opacity
  float gop[SA_THREADS];      // d opacity in, d logit out
  float sc[SA_THREADS * 3];   // scale
  float gsc[SA_THREADS * 3];  // d scale in, d log_scale out
  float sh[SA_THREADS * SA_SH];  // shs mode: d shs; rgb mode: sh in, d sh out
  float grgb[SA_THREADS * 3];
  float mean[SA_THREADS * 3];  // mean in, d mean out
};

__global__ void __launch_bounds__(SA_THREADS) scene_assets_bwd_kernel(const B2RSceneAssets s, B2RSceneAssetsGrads g) {
  __shared__ BwdSmem sm;
  const int64_t r0 = (int64_t)blockIdx.x * SA_THREADS;
  const int n = (int)min((int64_t)SA_THREADS, (int64_t)s.P - r0);
  const int M = s.M, Ls = 3 * M | 1;
  const bool rgb = s.cam_R != nullptr;
  load_rows(sm.rot, 7, s.rotation6d, 6, 6, r0, n);
  load_rows(sm.grot, 5, g.dL_drotation, 4, 4, r0, n);
  load_rows(sm.op, 1, g.opacity, 1, 1, r0, n);
  load_rows(sm.gop, 1, g.dL_dopacity, 1, 1, r0, n);
  load_rows(sm.sc, 3, g.scale, 3, 3, r0, n);
  load_rows(sm.gsc, 3, g.dL_dscale, 3, 3, r0, n);
  if (rgb) {
    load_rows(sm.sh, Ls, s.feature_dc, s.dc_stride, 3, r0, n);
    if (M > 1) load_rows(sm.sh + 3, Ls, s.feature_rest, s.rest_stride, 3 * (M - 1), r0, n);
    load_rows(sm.grgb, 3, g.dL_dcolor, 3, 3, r0, n);
    load_rows(sm.mean, 3, s.mean, 3, 3, r0, n);
  } else {
    load_rows(sm.sh, Ls, g.dL_dcolor, 3 * M, 3 * M, r0, n);
  }
  __syncthreads();
  const int j = threadIdx.x;
  if (j < n) {
    const float o = sm.op[j];
    sm.gop[j] = sm.gop[j] * (1.f - o) * o;
    for (int i = 0; i < 3; ++i) sm.gsc[3 * j + i] = sm.gsc[3 * j + i] * sm.sc[3 * j + i];
    float a[6], gq[4], ga[6];
    for (int i = 0; i < 6; ++i) a[i] = sm.rot[7 * j + i];
    for (int i = 0; i < 4; ++i) gq[i] = sm.grot[5 * j + i];
    rot_backward(a, gq, ga);
    for (int i = 0; i < 6; ++i) sm.rot[7 * j + i] = ga[i];
    if (rgb) {
      float c[3], v[3];
      cam_position(s.cam_R, s.cam_t, c);
      for (int i = 0; i < 3; ++i) v[i] = sm.mean[3 * j + i] - c[i];
      const float nv = norm3(v), dn = fmaxf(nv, 1e-12f);
      const float x = v[0] / dn, y = v[1] / dn, z = v[2] / dn;
      const int nb = sh_basis_count(__ldg(s.active_sh_degree), M);
      float* row = sm.sh + Ls * j;
      float gres[3], gb[3], gdir[3] = {0.f, 0.f, 0.f};
      if (nb) {
        float res[3] = {0.f, 0.f, 0.f};  // the forward's sum, for clamp_min's mask
        for (int k = 0; k < nb; ++k) {
          const float b = sh_basis(k, x, y, z, gb);
          for (int ch = 0; ch < 3; ++ch) res[ch] = k == 0 ? b * row[ch] : res[ch] + b * row[3 * k + ch];
        }
        for (int ch = 0; ch < 3; ++ch) gres[ch] = res[ch] + 0.5f >= 0.f ? sm.grgb[3 * j + ch] : 0.f;
        for (int k = 0; k < nb; ++k) {
          const float b = sh_basis(k, x, y, z, gb);
          const float w = gres[0] * row[3 * k] + gres[1] * row[3 * k + 1] + gres[2] * row[3 * k + 2];
          for (int i = 0; i < 3; ++i) gdir[i] += w * gb[i];
          for (int ch = 0; ch < 3; ++ch) row[3 * k + ch] = b * gres[ch];
        }
        for (int k = nb; k < M; ++k)
          for (int ch = 0; ch < 3; ++ch) row[3 * k + ch] = 0.f;
        // dir = v / max(|v|, eps)
        const float sv = nv >= 1e-12f ? (gdir[0] * v[0] + gdir[1] * v[1] + gdir[2] * v[2]) / (dn * dn) / nv : 0.f;
        for (int i = 0; i < 3; ++i) sm.mean[3 * j + i] = gdir[i] / dn - sv * v[i];
      } else {
        const float nan = __int_as_float(0x7fc00000);
        for (int k = 0; k < 3 * M; ++k) row[k] = nan;
        for (int i = 0; i < 3; ++i) sm.mean[3 * j + i] = nan;
      }
    }
  }
  __syncthreads();
  store_rows(g.dL_dlogit, 1, sm.gop, 1, r0, n);
  store_rows(g.dL_dlog_scale, 3, sm.gsc, 3, r0, n);
  store_rows(g.dL_drotation6d, 6, sm.rot, 7, r0, n);
  store_rows(g.dL_dfeature_dc, 3, sm.sh, Ls, r0, n);
  if (M > 1) store_rows(g.dL_dfeature_rest, 3 * (M - 1), sm.sh + 3, Ls, r0, n);
  if (rgb) store_rows(g.dL_dmean, 3, sm.mean, 3, r0, n);
}

int launch_scene_assets_forward(const B2RSceneAssets& s, float* opacity, float* scale, float* rotation, float* color,
                                cudaStream_t st) {
  if (s.P == 0) return B2R_OK;
  ProfScope ps(K_MISC, st);
  launch_k(scene_assets_fwd_kernel, (unsigned)((s.P + SA_THREADS - 1) / SA_THREADS), SA_THREADS, 0, st, false, s,
           opacity, scale, rotation, color);
  return check_launch();
}

int launch_scene_assets_backward(const B2RSceneAssets& s, const B2RSceneAssetsGrads& g, cudaStream_t st) {
  if (s.P == 0) return B2R_OK;
  ProfScope ps(K_MISC, st);
  launch_k(scene_assets_bwd_kernel, (unsigned)((s.P + SA_THREADS - 1) / SA_THREADS), SA_THREADS, 0, st, false, s, g);
  return check_launch();
}

}  // namespace b2r
