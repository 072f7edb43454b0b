// smplx_pose.cu -- ExAvatar's SMPLXParamDict.forward (avatar/common/nets/module.py:673-684) for one frame: the seven 6D
// pose parameters to the (J,3) axis-angle pose, forward and backward, one CTA of one thread per joint
// (exavatar_release_b200/human_assets.py).  The same per-joint arithmetic serves SmplxParamTable: every frame's
// parameters in one table and the frame chosen by a slot read on the device, so one captured graph serves every frame.
//
// Per joint, pytorch3d 0.7.5 as smplx_rig.py restates it: q = matrix_to_quaternion(rotation_6d_to_matrix(a))
// (rot6d.cuh), then quaternion_to_axis_angle:
//   n = |q[1:]|, half = atan2(n, q0), angle = 2 half,
//   s = |angle| < 1e-6 ? 0.5 - angle^2 / 48 : sin(half) / angle,   axis_angle = q[1:] / s.
// Everything runs in fp64 from the fp32 rows and is rounded once.  The backward is autograd's through the branches the
// forward took: only the selected side of each `where` (the small-angle polynomial, or sin(half) / angle), norm's
// derivative zeroed at n == 0 (torch's norm backward), and rot_backward's rules for the quaternion.  At the identity
// q = (1, 0, 0, 0): s = 0.5, d q[1:] = 2 g, finite.
#include "common.cuh"
#include "rot6d.cuh"

namespace b2r {

constexpr int DP_THREADS = B2R_POSE_MAX_JOINTS;

// joint j's row: parameter k and row r within it (the loop unrolls, so the struct is indexed by constants only)
__device__ __forceinline__ bool pose_row(const B2RSmplxPose& p, int j, int& k, int& r) {
  r = j;
#pragma unroll
  for (int i = 0; i < B2R_POSE_PARAMS; ++i) {
    if (r < p.rows[i]) {
      k = i;
      return true;
    }
    r -= p.rows[i];
  }
  return false;
}

__device__ __forceinline__ const float* param_ptr(const B2RSmplxPose& p, int k) {
  const float* out = nullptr;
#pragma unroll
  for (int i = 0; i < B2R_POSE_PARAMS; ++i)
    if (i == k) out = p.param[i];
  return out;
}

__device__ __forceinline__ float* grad_ptr(const B2RSmplxPoseGrads& g, int k) {
  float* out = nullptr;
#pragma unroll
  for (int i = 0; i < B2R_POSE_PARAMS; ++i)
    if (i == k) out = g.param[i];
  return out;
}

// quaternion_to_axis_angle's intermediates
struct AxisAngle {
  double n, half, angle, s;
  bool small;
};

__device__ __forceinline__ void axis_angle_forward(const double* q, AxisAngle& x) {
  x.n = norm3d(q + 1);
  x.half = atan2(x.n, q[0]);
  x.angle = 2. * x.half;
  x.small = fabs(x.angle) < 1e-6;
  x.s = x.small ? 0.5 - x.angle * x.angle / 48. : sin(x.half) / x.angle;
}

// joint j of a frame: the 6D row to its axis-angle (3 floats)
__device__ __forceinline__ void decode_joint_forward(const float* __restrict__ row, float* __restrict__ out) {
  double a[6];
  for (int i = 0; i < 6; ++i) a[i] = __ldg(row + i);
  Rot6d rt;
  rot6d_forward(a, rt);
  Quat o;
  quat_forward(rt, o);
  AxisAngle x;
  axis_angle_forward(o.q, x);
  for (int i = 0; i < 3; ++i) out[i] = (float)(o.q[1 + i] / x.s);
}

// the gradient of the 6D row from the gradient of its axis-angle, dout (3 floats)
__device__ __forceinline__ void decode_joint_backward(const float* __restrict__ row, const float* __restrict__ dout,
                                                      float* __restrict__ out) {
  float af[6];
  double a[6];
  for (int i = 0; i < 6; ++i) a[i] = af[i] = __ldg(row + i);
  Rot6d rt;
  rot6d_forward(a, rt);
  Quat o;
  quat_forward(rt, o);
  AxisAngle x;
  axis_angle_forward(o.q, x);
  const double* v = o.q + 1;
  double gv[3], gs = 0.;
  for (int i = 0; i < 3; ++i) {
    const double gi = __ldg(dout + i);
    gv[i] = gi / x.s;  // axis_angle = v / s
    gs -= gi * v[i] / (x.s * x.s);
  }
  double ghalf = 0., gangle;
  if (x.small) {
    gangle = -gs * 2. * x.angle / 48.;
  } else {
    ghalf = gs * cos(x.half) / x.angle;
    gangle = -gs * sin(x.half) / (x.angle * x.angle);
  }
  ghalf += 2. * gangle;
  // half = atan2(n, q0)
  const double den = x.n * x.n + o.q[0] * o.q[0];
  const double gn = ghalf * o.q[0] / den;
  double gq[4];
  gq[0] = -ghalf * x.n / den;
  for (int i = 0; i < 3; ++i) gq[1 + i] = gv[i] + (x.n != 0. ? gn * v[i] / x.n : 0.);
  float ga[6];
  rot_backward(af, gq, ga);
  for (int i = 0; i < 6; ++i) out[i] = ga[i];
}

__global__ void __launch_bounds__(DP_THREADS) decode_pose_fwd_kernel(const B2RSmplxPose p, float* __restrict__ full_pose) {
  const int j = threadIdx.x;
  int k, r;
  if (!pose_row(p, j, k, r)) return;
  decode_joint_forward(param_ptr(p, k) + 6 * r, full_pose + 3 * j);
}

__global__ void __launch_bounds__(DP_THREADS) decode_pose_bwd_kernel(const B2RSmplxPose p,
                                                                     const float* __restrict__ dfull,
                                                                     const B2RSmplxPoseGrads g) {
  const int j = threadIdx.x;
  int k, r;
  if (!pose_row(p, j, k, r)) return;
  decode_joint_backward(param_ptr(p, k) + 6 * r, dfull + 3 * j, grad_ptr(g, k) + 6 * r);
}

// The frame of a parameter table: *slot on the device, or host_slot; -1 when it lies outside [0, n_frames)
__device__ __forceinline__ int table_frame(const B2RSmplxParamTable& t) {
  const int s = t.slot ? __ldg(t.slot) : t.host_slot;
  return s >= 0 && s < t.n_frames ? s : -1;
}

// one CTA: thread j < n_joints decodes joint j of the frame; the CTA copies the frame's expr and trans rows
__global__ void __launch_bounds__(DP_THREADS) param_table_fwd_kernel(const B2RSmplxParamTable t,
                                                                     float* __restrict__ full_pose,
                                                                     float* __restrict__ expr, float* __restrict__ trans) {
  const int f = table_frame(t);
  const int j = threadIdx.x;
  const float nan = __int_as_float(0x7fc00000);
  if (j < t.n_joints) {
    if (f >= 0) {
      decode_joint_forward(t.pose + ((int64_t)f * t.n_joints + j) * 6, full_pose + 3 * j);
    } else {
      for (int i = 0; i < 3; ++i) full_pose[3 * j + i] = nan;
    }
  }
  for (int i = j; i < t.n_expr; i += DP_THREADS) expr[i] = f >= 0 ? __ldg(t.expr + (int64_t)f * t.n_expr + i) : nan;
  if (j < 3) trans[j] = f >= 0 ? __ldg(t.trans + 3 * f + j) : nan;
}

// CTA f writes frame f's rows of the three gradients: the decode's backward and the two upstream gradients for the
// selected frame, zeros for every other frame
__global__ void __launch_bounds__(DP_THREADS) param_table_bwd_kernel(const B2RSmplxParamTable t,
                                                                     const B2RSmplxParamTableGrads g) {
  const int f = blockIdx.x;
  const bool sel = f == table_frame(t);
  const int j = threadIdx.x;
  float* dpose = g.pose + (int64_t)f * t.n_joints * 6;
  if (sel && g.dL_dfull_pose) {
    if (j < t.n_joints) decode_joint_backward(t.pose + ((int64_t)f * t.n_joints + j) * 6, g.dL_dfull_pose + 3 * j,
                                              dpose + 6 * j);
  } else {
    for (int i = j; i < 6 * t.n_joints; i += DP_THREADS) dpose[i] = 0.f;
  }
  for (int i = j; i < t.n_expr; i += DP_THREADS)
    g.expr[(int64_t)f * t.n_expr + i] = sel && g.dL_dexpr ? __ldg(g.dL_dexpr + i) : 0.f;
  if (j < 3) g.trans[3 * f + j] = sel && g.dL_dtrans ? __ldg(g.dL_dtrans + j) : 0.f;
}

int launch_decode_pose_forward(const B2RSmplxPose& p, float* full_pose, cudaStream_t st) {
  ProfScope ps(K_MISC, st);
  launch_k(decode_pose_fwd_kernel, 1, DP_THREADS, 0, st, true, p, full_pose);
  return check_launch();
}

int launch_decode_pose_backward(const B2RSmplxPose& p, const float* dfull, const B2RSmplxPoseGrads& g,
                                cudaStream_t st) {
  ProfScope ps(K_MISC, st);
  launch_k(decode_pose_bwd_kernel, 1, DP_THREADS, 0, st, true, p, dfull, g);
  return check_launch();
}

int launch_param_table_forward(const B2RSmplxParamTable& t, float* full_pose, float* expr, float* trans,
                               cudaStream_t st) {
  ProfScope ps(K_MISC, st);
  launch_k(param_table_fwd_kernel, 1, DP_THREADS, 0, st, true, t, full_pose, expr, trans);
  return check_launch();
}

int launch_param_table_backward(const B2RSmplxParamTable& t, const B2RSmplxParamTableGrads& g, cudaStream_t st) {
  ProfScope ps(K_MISC, st);
  launch_k(param_table_bwd_kernel, (unsigned)t.n_frames, DP_THREADS, 0, st, true, t, g);
  return check_launch();
}

}  // namespace b2r
