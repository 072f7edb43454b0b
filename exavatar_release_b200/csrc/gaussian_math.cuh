// gaussian_math.cuh -- per-Gaussian projection maths shared by the forward (project.cu) and backward
// (project_bwd.cu) kernels.  Follows SURVEY.md App. A.1 (steps 1-7) / A.5 / A.7.
#pragma once
#include "common.cuh"

namespace b2r {

struct Cam {
  float v[16];  // view, [4c+r]
  float p[16];  // full projection, [4c+r]
  float campos[3];
  float fx, fy, tanfovx, tanfovy;
  int W, H;
  bool valid;  // false: the device tan(fov) is not finite and > 0 -- the projection culls every Gaussian
};

// The one place the projection kernels read tan(fov): B2RScene.tanfov on the device when set, the by-value floats
// otherwise (checked > 0 on the host).  The host cannot check a device value, so one that is not finite and > 0 marks
// the camera invalid instead (the forward projection then culls every Gaussian, and nothing is visible to the backward).
// DEVICE_TANFOV = false compiles the by-value read alone: the forward projection kernel is instantiated both ways,
// because at its 64-register budget two loaded floats in place of two kernel parameters would spill.
template <bool DEVICE_TANFOV = true>
__device__ __forceinline__ Cam load_cam(const B2RScene& sc) {
  Cam c;
#pragma unroll
  for (int i = 0; i < 16; i++) {
    c.v[i] = __ldg(sc.viewmatrix + i);
    c.p[i] = __ldg(sc.projmatrix + i);
  }
#pragma unroll
  for (int i = 0; i < 3; i++) c.campos[i] = __ldg(sc.campos + i);
  c.W = sc.width;
  c.H = sc.height;
  c.tanfovx = sc.tanfovx;
  c.tanfovy = sc.tanfovy;
  c.valid = true;
  if (DEVICE_TANFOV && sc.tanfov) {
    const float tx = __ldg(sc.tanfov), ty = __ldg(sc.tanfov + 1);
    c.valid = tx > 0.f && tx < INFINITY && ty > 0.f && ty < INFINITY;
    c.tanfovx = tx;
    c.tanfovy = ty;
  }
  c.fx = (float)sc.width / (2.f * c.tanfovx);
  c.fy = (float)sc.height / (2.f * c.tanfovy);
  return c;
}

// View-space point.  Evaluated left to right WITHOUT fma contraction: view depth is the sort key and feeds the
// near-plane and frustum-clamp decisions, so it is kept bit-identical to the oracle's C expression (and to itself
// between the forward and backward kernels) -- per-tile list order is then exactly reproducible.
__device__ __forceinline__ float dot4_rn(float a, float x, float b, float y, float c, float z, float d) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, x), __fmul_rn(b, y)), __fmul_rn(c, z)), d);
}
__device__ __forceinline__ float3 xform4x3(const float3 p, const float* m) {
  return make_float3(dot4_rn(m[0], p.x, m[4], p.y, m[8], p.z, m[12]), dot4_rn(m[1], p.x, m[5], p.y, m[9], p.z, m[13]),
                     dot4_rn(m[2], p.x, m[6], p.y, m[10], p.z, m[14]));
}
__device__ __forceinline__ float4 xform4x4(const float3 p, const float* m) {
  return make_float4(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12], m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                     m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14], m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15]);
}

// R_std of an un-normalised quaternion (r,x,y,z), row-major R[row*3+col]
__device__ __forceinline__ void quat_to_R(const float4 q, float* R) {
  const float r = q.x, x = q.y, y = q.z, z = q.w;
  R[0] = 1.f - 2.f * (y * y + z * z);
  R[1] = 2.f * (x * y - r * z);
  R[2] = 2.f * (x * z + r * y);
  R[3] = 2.f * (x * y + r * z);
  R[4] = 1.f - 2.f * (x * x + z * z);
  R[5] = 2.f * (y * z - r * x);
  R[6] = 2.f * (x * z - r * y);
  R[7] = 2.f * (y * z + r * x);
  R[8] = 1.f - 2.f * (x * x + y * y);
}

// Sigma = R S^2 R^T, upper triangle (xx xy xz yy yz zz)
__device__ __forceinline__ void cov3d_from_scale_rot(const float3 scale, float mod, const float4 q, float* c6) {
  float R[9];
  quat_to_R(q, R);
  const float s[3] = {mod * scale.x, mod * scale.y, mod * scale.z};
  float M[9];  // M[i][j] = s_i * R[j][i]
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) M[i * 3 + j] = s[i] * R[j * 3 + i];
  auto S = [&](int a, int b) { return M[a] * M[b] + M[3 + a] * M[3 + b] + M[6 + a] * M[6 + b]; };
  c6[0] = S(0, 0); c6[1] = S(0, 1); c6[2] = S(0, 2);
  c6[3] = S(1, 1); c6[4] = S(1, 2); c6[5] = S(2, 2);
}

struct Ewa {
  float t[3];      // view-space position with frustum-clamped x,y
  float A0[3], A1[3];  // rows of J * Rv
  float xmul, ymul;
  float a, b, c;   // dilated 2D covariance
};

__device__ __forceinline__ void ewa_project(const float3 pview, const float* c6, const Cam& cam, Ewa& e) {
  const float limx = K_FRUSTUM * cam.tanfovx, limy = K_FRUSTUM * cam.tanfovy;
  const float txtz = pview.x / pview.z, tytz = pview.y / pview.z;
  e.xmul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
  e.ymul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
  e.t[0] = fminf(limx, fmaxf(-limx, txtz)) * pview.z;
  e.t[1] = fminf(limy, fmaxf(-limy, tytz)) * pview.z;
  e.t[2] = pview.z;
  const float J00 = cam.fx / e.t[2], J02 = -(cam.fx * e.t[0]) / (e.t[2] * e.t[2]);
  const float J11 = cam.fy / e.t[2], J12 = -(cam.fy * e.t[1]) / (e.t[2] * e.t[2]);
  const float* v = cam.v;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    e.A0[k] = J00 * v[4 * k + 0] + J02 * v[4 * k + 2];
    e.A1[k] = J11 * v[4 * k + 1] + J12 * v[4 * k + 2];
  }
  const float S[9] = {c6[0], c6[1], c6[2], c6[1], c6[3], c6[4], c6[2], c6[4], c6[5]};
  float B0[3], B1[3];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    B0[k] = e.A0[0] * S[k] + e.A0[1] * S[3 + k] + e.A0[2] * S[6 + k];
    B1[k] = e.A1[0] * S[k] + e.A1[1] * S[3 + k] + e.A1[2] * S[6 + k];
  }
  e.a = B0[0] * e.A0[0] + B0[1] * e.A0[1] + B0[2] * e.A0[2] + K_DILATE;
  e.b = B0[0] * e.A1[0] + B0[1] * e.A1[1] + B0[2] * e.A1[2];
  e.c = B1[0] * e.A1[0] + B1[1] * e.A1[1] + B1[2] * e.A1[2] + K_DILATE;
}

// SH basis constants (avatar/common/utils/transforms.py:82-110)
#define B2R_SH_C0 0.28209479177387814f
#define B2R_SH_C1 0.4886025119029199f
static __device__ __constant__ float c_SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                            -1.0925484305920792f, 0.5462742152960396f};
static __device__ __constant__ float c_SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                            0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                                            -0.5900435899266435f};

}  // namespace b2r
