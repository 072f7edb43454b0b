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
// as torch rounds the same expression.  The rotation alone is evaluated in fp64 (below).
#include "common.cuh"

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

__device__ __forceinline__ double norm3d(const double* v) { return sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

// The rotation runs in fp64 from the fp32 inputs and is rounded to fp32 once: Gram-Schmidt's cancellation in
// a2 - (b1 . a2) b1 magnifies every rounding by about 1 / sin(a1, a2), so an fp32 evaluation loses digits on nearly
// parallel rows (a few in 10^5 random ones), and the quaternion's pick would then differ from an exact one near ties.
struct Rot6d {
  double b1[3], b2[3], b3[3], u[3];
  double n1, n2, dot;
};

__device__ __forceinline__ void rot6d_forward(const double* a, Rot6d& r) {
  r.n1 = norm3d(a);
  const double d1 = fmax(r.n1, 1e-12);
  for (int i = 0; i < 3; ++i) r.b1[i] = a[i] / d1;
  r.dot = r.b1[0] * a[3] + r.b1[1] * a[4] + r.b1[2] * a[5];
  for (int i = 0; i < 3; ++i) r.u[i] = a[3 + i] - r.dot * r.b1[i];
  r.n2 = norm3d(r.u);
  const double d2 = fmax(r.n2, 1e-12);
  for (int i = 0; i < 3; ++i) r.b2[i] = r.u[i] / d2;
  r.b3[0] = r.b1[1] * r.b2[2] - r.b1[2] * r.b2[1];
  r.b3[1] = r.b1[2] * r.b2[0] - r.b1[0] * r.b2[2];
  r.b3[2] = r.b1[0] * r.b2[1] - r.b1[1] * r.b2[0];
}

// matrix_to_quaternion of the rows (b1, b2, b3): the four 1 +- m00 +- m11 +- m22, the pick (first argmax of q_abs),
// the picked candidate over 2 max(q_abs, 0.1), and the sign (q0 < 0 -> -q)
struct Quat {
  double t[4], qa[4], cand[4], den, q[4];
  int k;
  bool flip;
};

__device__ __forceinline__ void quat_forward(const Rot6d& r, Quat& o) {
  const double m00 = r.b1[0], m01 = r.b1[1], m02 = r.b1[2], m10 = r.b2[0], m11 = r.b2[1], m12 = r.b2[2],
              m20 = r.b3[0], m21 = r.b3[1], m22 = r.b3[2];
  o.t[0] = 1. + m00 + m11 + m22;
  o.t[1] = 1. + m00 - m11 - m22;
  o.t[2] = 1. - m00 + m11 - m22;
  o.t[3] = 1. - m00 - m11 + m22;
  for (int i = 0; i < 4; ++i) o.qa[i] = o.t[i] > 0. ? sqrt(o.t[i]) : 0.;
  o.k = 0;
  for (int i = 1; i < 4; ++i)
    if (o.qa[i] > o.qa[o.k]) o.k = i;
  const double s = o.qa[o.k] * o.qa[o.k];
  switch (o.k) {
    case 0: o.cand[0] = s; o.cand[1] = m21 - m12; o.cand[2] = m02 - m20; o.cand[3] = m10 - m01; break;
    case 1: o.cand[0] = m21 - m12; o.cand[1] = s; o.cand[2] = m10 + m01; o.cand[3] = m02 + m20; break;
    case 2: o.cand[0] = m02 - m20; o.cand[1] = m10 + m01; o.cand[2] = s; o.cand[3] = m12 + m21; break;
    default: o.cand[0] = m10 - m01; o.cand[1] = m20 + m02; o.cand[2] = m21 + m12; o.cand[3] = s; break;
  }
  o.den = 2. * fmax(o.qa[o.k], 0.1);
  for (int i = 0; i < 4; ++i) o.q[i] = o.cand[i] / o.den;
  o.flip = o.q[0] < 0.;
  if (o.flip)
    for (int i = 0; i < 4; ++i) o.q[i] = -o.q[i];
}

// d rot6d (6) from d quaternion (4), through the forward's own branches
__device__ __forceinline__ void rot_backward(const float* af, const float* gq_in, float* ga) {
  double a[6];
  for (int i = 0; i < 6; ++i) a[i] = af[i];
  Rot6d r;
  rot6d_forward(a, r);
  Quat o;
  quat_forward(r, o);
  double gq[4];
  for (int i = 0; i < 4; ++i) gq[i] = o.flip ? -gq_in[i] : gq_in[i];
  // q = cand / den
  double gc[4], gden = 0.;
  for (int i = 0; i < 4; ++i) {
    gc[i] = gq[i] / o.den;
    gden -= gq[i] * o.cand[i] / (o.den * o.den);
  }
  const int k = o.k;
  // den = 2 max(qa_k, 0.1) (qa_k >= 1 for any input: the four t sum to 4); cand_kk = qa_k^2
  double gqa = (o.qa[k] > 0.1 ? 2. * gden : 0.) + 2. * o.qa[k] * gc[k];
  const double gt = o.t[k] > 0. ? gqa / (2. * o.qa[k]) : 0.;
  // dL/dm from t_k and the candidate's off-diagonal entries
  double gm[9] = {0., 0., 0., 0., 0., 0., 0., 0., 0.};  // m00 m01 m02 m10 m11 m12 m20 m21 m22
  const double sg[4][3] = {{1., 1., 1.}, {1., -1., -1.}, {-1., 1., -1.}, {-1., -1., 1.}};
  gm[0] += sg[k][0] * gt;
  gm[4] += sg[k][1] * gt;
  gm[8] += sg[k][2] * gt;
  // the three off-diagonal entries of the picked candidate: (index into cand, m_a, m_b, sign of m_b)
  switch (k) {
    case 0:
      gm[7] += gc[1]; gm[5] -= gc[1]; gm[2] += gc[2]; gm[6] -= gc[2]; gm[3] += gc[3]; gm[1] -= gc[3]; break;
    case 1:
      gm[7] += gc[0]; gm[5] -= gc[0]; gm[3] += gc[2]; gm[1] += gc[2]; gm[2] += gc[3]; gm[6] += gc[3]; break;
    case 2:
      gm[2] += gc[0]; gm[6] -= gc[0]; gm[3] += gc[1]; gm[1] += gc[1]; gm[5] += gc[3]; gm[7] += gc[3]; break;
    default:
      gm[3] += gc[0]; gm[1] -= gc[0]; gm[6] += gc[1]; gm[2] += gc[1]; gm[7] += gc[2]; gm[5] += gc[2]; break;
  }
  double gb1[3] = {gm[0], gm[1], gm[2]}, gb2[3] = {gm[3], gm[4], gm[5]};
  const double g3[3] = {gm[6], gm[7], gm[8]};
  // b3 = b1 x b2: gb1 += b2 x g3, gb2 += g3 x b1
  gb1[0] += r.b2[1] * g3[2] - r.b2[2] * g3[1];
  gb1[1] += r.b2[2] * g3[0] - r.b2[0] * g3[2];
  gb1[2] += r.b2[0] * g3[1] - r.b2[1] * g3[0];
  gb2[0] += g3[1] * r.b1[2] - g3[2] * r.b1[1];
  gb2[1] += g3[2] * r.b1[0] - g3[0] * r.b1[2];
  gb2[2] += g3[0] * r.b1[1] - g3[1] * r.b1[0];
  // b2 = u / max(|u|, eps): the norm's term only where the clamp passes (|u| >= eps) and |u| > 0
  const double d2 = fmax(r.n2, 1e-12);
  const double s2 = (r.n2 >= 1e-12) ? (gb2[0] * r.u[0] + gb2[1] * r.u[1] + gb2[2] * r.u[2]) / (d2 * d2) / r.n2 : 0.;
  double gu[3];
  for (int i = 0; i < 3; ++i) gu[i] = gb2[i] / d2 - s2 * r.u[i];
  // u = a2 - dot b1, dot = b1 . a2
  const double gdot = -(gu[0] * r.b1[0] + gu[1] * r.b1[1] + gu[2] * r.b1[2]);
  for (int i = 0; i < 3; ++i) {
    gb1[i] += -r.dot * gu[i] + gdot * a[3 + i];
    ga[3 + i] = (float)(gu[i] + gdot * r.b1[i]);
  }
  // b1 = a1 / max(|a1|, eps)
  const double d1 = fmax(r.n1, 1e-12);
  const double s1 = (r.n1 >= 1e-12) ? (gb1[0] * a[0] + gb1[1] * a[1] + gb1[2] * a[2]) / (d1 * d1) / r.n1 : 0.;
  for (int i = 0; i < 3; ++i) ga[i] = (float)(gb1[i] / d1 - s1 * a[i]);
}

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
