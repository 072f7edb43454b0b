// rot6d.cuh -- pytorch3d 0.7.5's matrix_to_quaternion(rotation_6d_to_matrix(a)) for one 6D row, forward and backward,
// in fp64 (restated in smplx_rig.py).  Shared by scene_assets.cu (the scene Gaussians' rotations) and smplx_pose.cu
// (ExAvatar's SMPL-X pose parameters, which continue to axis-angle).
#pragma once

namespace b2r {

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

// d rot6d (6) from d quaternion (4, float or double), through the forward's own branches
template <typename G>
__device__ __forceinline__ void rot_backward(const float* af, const G* gq_in, float* ga) {
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

}  // namespace b2r
