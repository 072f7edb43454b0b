// smplx_rig.cu -- ExAvatar's SMPL-X rig (HumanGaussian.forward, avatar/common/nets/module.py:517-518, 533, 537, 549):
// the 大-pose and zero-pose body-model forwards with identity information, the inverse-neutral and the frame's forward
// kinematics, the pose-corrective and expression offsets and the two midpoint subdivisions, with no host
// synchronisation and no float atomics.
//
// Contract at V, then upsample: subdivision is linear, so the pose and expression offsets are contracted with the base
// tables (posedirs 9(J-1) x 3V, expr_dirs V x 3 x NE) and the (V,3) results are subdivided; ExAvatar subdivides the
// tables first (P x 3 x 486 and P x 3 x 50) and contracts those.  The two agree in exact arithmetic.
//
// Forward (all launches on the caller's stream, counted under kernel id 8 misc):
//   rig_shape_kernel      one warp per vertex: v_shaped = template + shapedirs . beta and expr_V = expr_dirs . expr.
//   rig_chain_kernel      ONE CTA: the joints J_regressor . v_shaped (+ joint_offset, root zeroed) over the per-joint
//                         CSR in fp64; the frame's rotations from full_pose (pytorch3d's axis_angle_to_matrix); the
//                         four kinematic chains in fp64, two at a time, walked level by level over the tree (thread i
//                         = joint i): 大 pose and zero pose on the joints, then inverse-neutral on the 大-pose joints
//                         and the frame's on the zero-pose joints; joint_mats = frame . inverse-neutral; the pose
//                         feature (R - I of joints 1..J-1) and pose_6d.
//   rig_lbs_kernel        one warp per vertex: pose_V = feature . posedirs and mesh_wo = (W A_neutral) (v_shaped +
//                         pose_offset0, 1).
//   rig_upsample_kernel   one thread per output row: two midpoint levels fl(fl(a + b) * 0.5f) of mesh_wo, pose_V
//                         (masked after subdivision) and expr_V.
// Backward:
//   rig_bwd_vertex_kernel fixed grid, one warp per vertex: the transposed subdivision as a gather (upT CSR), the LBS
//                         adjoint (dv_shaped through W A_neutral), fp64 per-CTA partials of W^T g (the translation
//                         columns of dA_neutral; its rotations are constants) and of expr_dirs^T g_expr.
//   rig_bwd_chain_kernel  ONE CTA: the partials in a fixed order; the four chains recomputed and their adjoints run in
//                         reverse level order (children gathered in index order); d full_pose through the derivative
//                         of axis_angle_to_matrix; d joint_offset with an exactly-zero root row.
//   rig_bwd_shape_kernel  fixed grid, one warp per vertex: dv_shaped + J_regressor^T dJ (per-vertex CSR), fp64 per-CTA
//                         partials of shapedirs^T dv_shaped.
//   rig_bwd_reduce_kernel ONE CTA: d shape_param from those partials in a fixed order.
//
// The second half of the file is the frame's SMPL-X body mesh of get_smplx_outputs (b2r_smplx_body_*) over the same
// tables, reusing the shape pass, the chain steps and their adjoints.
//
// Compiled with --fmad=false (build_ext.py): each product and sum is rounded on its own, so the midpoints are
// fl(fl(a + b) * 0.5f) as in pytorch3d's SubdivideMeshes, and the vertex sums have one order whatever the compiler does.
#include <math.h>

#include "common.cuh"

namespace b2r {

constexpr int RIG_THREADS = 256;
constexpr int RIG_WARPS = RIG_THREADS / 32;
constexpr int RIG_PART_BLOCKS = 128;  // fixed: the partials' vertex -> warp map, and so their bits, never change
constexpr int RIG_JMAX = 64;
constexpr int RIG_CMAX = 128;         // NB, NE
constexpr int RIG_CHAIN_THREADS = 2 * RIG_JMAX;
constexpr double RIG_SMALL_ANGLE = 1e-6;  // pytorch3d axis_angle_to_quaternion's eps

struct RigLayout {
  size_t vs, ev, pv, feat, an, jn, dvs, djn, part_a, part_e, part_b, total;
};

inline RigLayout rig_layout(int V, int J, int NB, int NE) {
  (void)J; (void)NB; (void)NE;
  const size_t v = V > 0 ? (size_t)V : 1;
  RigLayout L;
  size_t o = 0;
  L.vs = o; o += align_up(v * 3 * sizeof(float));
  L.ev = o; o += align_up(v * 3 * sizeof(float));
  L.pv = o; o += align_up(v * 3 * sizeof(float));
  L.feat = o; o += align_up((size_t)9 * RIG_JMAX * sizeof(float));
  L.an = o; o += align_up((size_t)12 * RIG_JMAX * sizeof(float));
  L.jn = o; o += align_up((size_t)3 * RIG_JMAX * sizeof(double));
  L.dvs = o; o += align_up(v * 3 * sizeof(float));
  L.djn = o; o += align_up((size_t)3 * RIG_JMAX * sizeof(double));
  L.part_a = o; o += align_up((size_t)RIG_PART_BLOCKS * 3 * RIG_JMAX * sizeof(double));
  L.part_e = o; o += align_up((size_t)RIG_PART_BLOCKS * RIG_CMAX * sizeof(double));
  L.part_b = o; o += align_up((size_t)RIG_PART_BLOCKS * RIG_CMAX * sizeof(double));
  L.total = o;
  return L;
}

struct RigPtrs {
  float *vs, *ev, *pv, *feat, *an, *dvs;
  double *jn, *djn, *part_a, *part_e, *part_b;
};

inline RigPtrs rig_ptrs(const B2RRig& r, void* scratch) {
  const RigLayout L = rig_layout(r.V, r.J, r.NB, r.NE);
  char* s = (char*)scratch;
  RigPtrs p;
  p.vs = (float*)(s + L.vs);
  p.ev = (float*)(s + L.ev);
  p.pv = (float*)(s + L.pv);
  p.feat = (float*)(s + L.feat);
  p.an = (float*)(s + L.an);
  p.jn = (double*)(s + L.jn);
  p.dvs = (float*)(s + L.dvs);
  p.djn = (double*)(s + L.djn);
  p.part_a = (double*)(s + L.part_a);
  p.part_e = (double*)(s + L.part_e);
  p.part_b = (double*)(s + L.part_b);
  return p;
}

// ---------------------------------------------------------------------------------------------------------------------
// pytorch3d 0.7.5 axis_angle_to_matrix = quaternion_to_matrix(axis_angle_to_quaternion(a)), in fp64, and its adjoint.

__device__ __forceinline__ void aa_quat(const double a[3], double q[4], double& angle, double& s) {
  angle = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
  const double h = 0.5 * angle;
  s = fabs(angle) < RIG_SMALL_ANGLE ? 0.5 - angle * angle / 48.0 : sin(h) / angle;
  q[0] = cos(h);
  q[1] = a[0] * s;
  q[2] = a[1] * s;
  q[3] = a[2] * s;
}

__device__ void aa_to_matrix(const double a[3], double R[9]) {
  double q[4], angle, s;
  aa_quat(a, q, angle, s);
  const double r = q[0], i = q[1], j = q[2], k = q[3];
  const double ts = 2.0 / (r * r + i * i + j * j + k * k);
  R[0] = 1.0 - ts * (j * j + k * k); R[1] = ts * (i * j - k * r);       R[2] = ts * (i * k + j * r);
  R[3] = ts * (i * j + k * r);       R[4] = 1.0 - ts * (i * i + k * k); R[5] = ts * (j * k - i * r);
  R[6] = ts * (i * k - j * r);       R[7] = ts * (j * k + i * r);       R[8] = 1.0 - ts * (i * i + j * j);
}

// da = (dR/da)^T dR; zero angle takes torch's convention for the norm's gradient (0 at 0)
__device__ void aa_to_matrix_bwd(const double a[3], const double dR[9], double da[3]) {
  double q[4], angle, s;
  aa_quat(a, q, angle, s);
  const double r = q[0], i = q[1], j = q[2], k = q[3];
  const double ts = 2.0 / (r * r + i * i + j * j + k * k);
  const double N[9] = {-(j * j + k * k), i * j - k * r, i * k + j * r, i * j + k * r, -(i * i + k * k), j * k - i * r,
                       i * k - j * r, j * k + i * r, -(i * i + j * j)};
  double dts = 0.0, dN[9];
  for (int t = 0; t < 9; t++) {
    dts += dR[t] * N[t];
    dN[t] = ts * dR[t];
  }
  double dq[4];
  dq[0] = -k * dN[1] + j * dN[2] + k * dN[3] - i * dN[5] - j * dN[6] + i * dN[7];
  dq[1] = -2.0 * i * dN[4] - 2.0 * i * dN[8] + j * dN[1] + k * dN[2] + j * dN[3] - r * dN[5] + k * dN[6] + r * dN[7];
  dq[2] = -2.0 * j * dN[0] - 2.0 * j * dN[8] + i * dN[1] + r * dN[2] + i * dN[3] + k * dN[5] - r * dN[6] + k * dN[7];
  dq[3] = -2.0 * k * dN[0] - 2.0 * k * dN[4] - r * dN[1] + i * dN[2] + r * dN[3] + j * dN[5] + i * dN[6] + j * dN[7];
  const double dq_ts = -dts * ts * ts;  // d(2/|q|^2)/dq = -ts^2 q
  for (int t = 0; t < 4; t++) dq[t] += dq_ts * q[t];
  const double h = 0.5 * angle;
  const double ds = fabs(angle) < RIG_SMALL_ANGLE ? -angle / 24.0 : (0.5 * cos(h) * angle - sin(h)) / (angle * angle);
  const double dangle = dq[0] * (-0.5 * sin(h)) + (dq[1] * a[0] + dq[2] * a[1] + dq[3] * a[2]) * ds;
  const double inv = angle > 0.0 ? dangle / angle : 0.0;
  for (int t = 0; t < 3; t++) da[t] = dq[1 + t] * s + inv * a[t];
}

// ---------------------------------------------------------------------------------------------------------------------
// Kinematic chains (smplx lbs.batch_rigid_transform), fp64.  G (J,12): the global 3x4 transform of each joint, row-major.
// One thread per joint; the caller loops the levels of the tree with a barrier between them.

__device__ __forceinline__ void chain_step(int i, const int* __restrict__ parents, const double* R, const double* jt,
                                           double* G) {
  const double* Ri = R + 9 * i;
  const int p = parents[i];
  double tl[3];
  for (int c = 0; c < 3; c++) tl[c] = jt[3 * i + c] - (p >= 0 ? jt[3 * p + c] : 0.0);
  double* Gi = G + 12 * i;
  if (p < 0) {
    for (int a = 0; a < 3; a++) {
      for (int c = 0; c < 3; c++) Gi[4 * a + c] = Ri[3 * a + c];
      Gi[4 * a + 3] = tl[a];
    }
    return;
  }
  const double* Gp = G + 12 * p;
  for (int a = 0; a < 3; a++) {
    for (int c = 0; c < 3; c++) Gi[4 * a + c] = Gp[4 * a] * Ri[c] + Gp[4 * a + 1] * Ri[3 + c] + Gp[4 * a + 2] * Ri[6 + c];
    Gi[4 * a + 3] = Gp[4 * a] * tl[0] + Gp[4 * a + 1] * tl[1] + Gp[4 * a + 2] * tl[2] + Gp[4 * a + 3];
  }
}

// rel transform A_i = [G_i.R | G_i.t - G_i.R j_i] (batch_rigid_transform's second output)
__device__ __forceinline__ void chain_rel(int i, const double* jt, const double* G, double A[12]) {
  const double* Gi = G + 12 * i;
  for (int a = 0; a < 3; a++) {
    for (int c = 0; c < 3; c++) A[4 * a + c] = Gi[4 * a + c];
    A[4 * a + 3] = Gi[4 * a + 3] -
                   (Gi[4 * a] * jt[3 * i] + Gi[4 * a + 1] * jt[3 * i + 1] + Gi[4 * a + 2] * jt[3 * i + 2]);
  }
}

// the joint's own adjoint terms from dA_i (dAR may be null: zero) and d posed_i (may be null): dG_i and dj_i
__device__ __forceinline__ void chain_own(int i, const double* jt, const double* G, const double* dAR, const double* dAt,
                                          const double* dposed, double* dG, double* dj) {
  const double* Gi = G + 12 * i;
  double* g = dG + 12 * i;
  for (int a = 0; a < 3; a++) {
    for (int c = 0; c < 3; c++) g[4 * a + c] = (dAR ? dAR[3 * a + c] : 0.0) - dAt[a] * jt[3 * i + c];
    g[4 * a + 3] = dAt[a] + (dposed ? dposed[a] : 0.0);
  }
  for (int c = 0; c < 3; c++) dj[3 * i + c] = -(Gi[c] * dAt[0] + Gi[4 + c] * dAt[1] + Gi[8 + c] * dAt[2]);
}

// reverse level step of joint i: gather its children (index order), then d rotation (dR may be null) and d local
// translation; dj_i += dtl_i - sum_children dtl_c
__device__ __forceinline__ void chain_back_step(int i, int J, const int* __restrict__ parents, const double* R,
                                                const double* jt, const double* G, double* dG, double* dtl, double* dj,
                                                double* dR) {
  double* g = dG + 12 * i;
  for (int c = i + 1; c < J; c++) {
    if (parents[c] != i) continue;
    const double* gc = dG + 12 * c;
    const double* Rc = R + 9 * c;
    double tl[3];
    for (int t = 0; t < 3; t++) tl[t] = jt[3 * c + t] - jt[3 * i + t];
    for (int a = 0; a < 3; a++) {
      for (int b = 0; b < 3; b++)
        g[4 * a + b] += gc[4 * a] * Rc[3 * b] + gc[4 * a + 1] * Rc[3 * b + 1] + gc[4 * a + 2] * Rc[3 * b + 2] +
                        gc[4 * a + 3] * tl[b];
      g[4 * a + 3] += gc[4 * a + 3];
    }
    for (int t = 0; t < 3; t++) dj[3 * i + t] -= dtl[3 * c + t];
  }
  const int p = parents[i];
  double d[3];
  if (p < 0) {
    for (int a = 0; a < 3; a++) {
      d[a] = g[4 * a + 3];
      if (dR)
        for (int b = 0; b < 3; b++) dR[9 * i + 3 * a + b] = g[4 * a + b];
    }
  } else {
    const double* Gp = G + 12 * p;
    for (int a = 0; a < 3; a++) {
      d[a] = Gp[a] * g[3] + Gp[4 + a] * g[7] + Gp[8 + a] * g[11];
      if (dR)
        for (int b = 0; b < 3; b++) dR[9 * i + 3 * a + b] = Gp[a] * g[b] + Gp[4 + a] * g[4 + b] + Gp[8 + a] * g[8 + b];
    }
  }
  for (int t = 0; t < 3; t++) {
    dtl[3 * i + t] = d[t];
    dj[3 * i + t] += d[t];
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Shared state of the single-CTA kernels

struct RigChainSm {
  double jn[RIG_JMAX * 3], jnp[RIG_JMAX * 3], jzp[RIG_JMAX * 3], rf[RIG_JMAX * 9];
  double G[4][RIG_JMAX * 12];  // 0 neutral, 1 zero, 2 inverse-neutral, 3 frame
  int depth[RIG_JMAX];
  int maxd;
  int bad;  // parents not topological (the C ABI cannot check device data): no chain is walked, outputs are NaN
};
static_assert(sizeof(RigChainSm) <= 48 * 1024, "the forward's single CTA fits the default dynamic shared memory");

struct RigBackSm {
  RigChainSm c;
  double dG[2][RIG_JMAX * 12], dtl[2][RIG_JMAX * 3], dj[2][RIG_JMAX * 3], dR[RIG_JMAX * 9], dAt[RIG_JMAX * 3];
};

// the depth of each joint in the tree and the deepest level; parents that are not topological set `bad`, every depth
// to 0 and maxd to -1 (no level is walked)
__device__ void chain_depths(const int* __restrict__ parents, int J, int* depth, int& maxd, int& bad) {
  int m = 0, b = 0;
  for (int i = 0; i < J; i++) {
    const int p = parents[i];
    b |= i == 0 ? p != -1 : (p < 0 || p >= i);
    depth[i] = b ? 0 : (p < 0 ? 0 : depth[p] + 1);
    m = max(m, depth[i]);
  }
  maxd = b ? -1 : m;
  bad = b;
}

// joints, frame rotations, depths, then the four chains; leaves sm.G, sm.jnp, sm.jzp filled
__device__ void rig_chains(const B2RRig& r, const float* __restrict__ vs, RigChainSm& sm, bool from_vs,
                           const double* __restrict__ jn_saved) {
  const int tid = threadIdx.x, J = r.J;
  if (tid < J) {
    double acc[3] = {0.0, 0.0, 0.0};
    if (from_vs) {
      for (int q = r.jreg_offsets[tid]; q < r.jreg_offsets[tid + 1]; q++) {
        const int v = r.jreg_cols[q];
        const double w = (double)r.jreg_vals[q];
        for (int c = 0; c < 3; c++) acc[c] += w * (double)vs[3 * v + c];
      }
      for (int c = 0; c < 3; c++) sm.jn[3 * tid + c] = acc[c] + (tid > 0 ? (double)r.joint_offset[3 * tid + c] : 0.0);
    } else {
      for (int c = 0; c < 3; c++) sm.jn[3 * tid + c] = jn_saved[3 * tid + c];
    }
    const double a[3] = {(double)r.full_pose[3 * tid], (double)r.full_pose[3 * tid + 1], (double)r.full_pose[3 * tid + 2]};
    aa_to_matrix(a, sm.rf + 9 * tid);
  }
  if (tid == 0) chain_depths(r.parents, J, sm.depth, sm.maxd, sm.bad);
  __syncthreads();
  const int grp = tid / RIG_JMAX, i = tid % RIG_JMAX;
  for (int d = 0; d <= sm.maxd; d++) {
    if (i < J && sm.depth[i] == d)
      chain_step(i, r.parents, grp == 0 ? r.rot_neutral : r.rot_zero, sm.jn, sm.G[grp]);
    __syncthreads();
  }
  if (tid < J)
    for (int c = 0; c < 3; c++) {
      sm.jnp[3 * tid + c] = sm.G[0][12 * tid + 4 * c + 3];
      sm.jzp[3 * tid + c] = sm.G[1][12 * tid + 4 * c + 3];
    }
  __syncthreads();
  for (int d = 0; d <= sm.maxd; d++) {
    if (i < J && sm.depth[i] == d) {
      if (grp == 0) chain_step(i, r.parents, r.rot_inv, sm.jnp, sm.G[2]);
      else chain_step(i, r.parents, sm.rf, sm.jzp, sm.G[3]);
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Forward

__global__ void __launch_bounds__(RIG_THREADS) rig_shape_kernel(const B2RRig r, const RigPtrs s) {
  const int lane = threadIdx.x & 31;
  const int v = blockIdx.x * RIG_WARPS + (threadIdx.x >> 5);
  if (v >= r.V) return;
  float b[4], e[4];
  for (int k = 0; k < 4; k++) {
    const int n = lane + 32 * k;
    b[k] = n < r.NB ? r.shape_param[n] : 0.f;
    e[k] = n < r.NE ? r.expr[n] : 0.f;
  }
  for (int c = 0; c < 3; c++) {
    const float* S = r.shapedirs + ((size_t)v * 3 + c) * r.NB;
    const float* E = r.expr_dirs + ((size_t)v * 3 + c) * r.NE;
    float as = 0.f, ae = 0.f;
    for (int k = 0; k < 4; k++) {
      const int n = lane + 32 * k;
      if (n < r.NB) as += S[n] * b[k];
      if (n < r.NE) ae += E[n] * e[k];
    }
    as = warp_sum(as);
    ae = warp_sum(ae);
    if (lane == 0) {
      s.vs[3 * v + c] = r.template_[3 * v + c] + as;
      s.ev[3 * v + c] = ae;
    }
  }
}

__global__ void __launch_bounds__(RIG_CHAIN_THREADS) rig_chain_kernel(const B2RRig r, const RigPtrs s,
                                                                      float* __restrict__ joint_mats,
                                                                      float* __restrict__ pose_6d) {
  extern __shared__ __align__(16) unsigned char rig_smem[];
  RigChainSm& sm = *reinterpret_cast<RigChainSm*>(rig_smem);
  rig_chains(r, s.vs, sm, true, nullptr);
  const int tid = threadIdx.x, J = r.J;
  if (tid >= J) return;
  for (int c = 0; c < 3; c++) s.jn[3 * tid + c] = sm.jn[3 * tid + c];
  double An[12], Ai[12], Af[12];
  chain_rel(tid, sm.jn, sm.G[0], An);
  chain_rel(tid, sm.jnp, sm.G[2], Ai);
  chain_rel(tid, sm.jzp, sm.G[3], Af);
  if (sm.bad)
    for (int t = 0; t < 12; t++) An[t] = Ai[t] = Af[t] = nan("");
  for (int t = 0; t < 12; t++) s.an[12 * tid + t] = (float)An[t];
  float* M = joint_mats + 16 * tid;
  for (int a = 0; a < 3; a++) {
    for (int c = 0; c < 3; c++) M[4 * a + c] = (float)(Af[4 * a] * Ai[c] + Af[4 * a + 1] * Ai[4 + c] + Af[4 * a + 2] * Ai[8 + c]);
    M[4 * a + 3] = (float)(Af[4 * a] * Ai[3] + Af[4 * a + 1] * Ai[7] + Af[4 * a + 2] * Ai[11] + Af[4 * a + 3]);
  }
  M[12] = 0.f; M[13] = 0.f; M[14] = 0.f; M[15] = 1.f;
  if (tid >= 1) {
    const double* Rf = sm.rf + 9 * tid;  // from full_pose alone: finite even with bad parents
    for (int t = 0; t < 9; t++) s.feat[9 * (tid - 1) + t] = (float)(Rf[t] - ((t % 4) == 0 ? 1.0 : 0.0));
    if (tid <= r.n_body)
      for (int t = 0; t < 6; t++) pose_6d[6 * (tid - 1) + t] = (float)Rf[t];
  }
}

__global__ void __launch_bounds__(RIG_THREADS) rig_lbs_kernel(const B2RRig r, const RigPtrs s, float* __restrict__ mesh_wo) {
  __shared__ float feat[9 * RIG_JMAX];
  __shared__ float an[12 * RIG_JMAX];
  const int K = 9 * (r.J - 1);
  for (int t = threadIdx.x; t < K; t += RIG_THREADS) feat[t] = s.feat[t];
  for (int t = threadIdx.x; t < 12 * r.J; t += RIG_THREADS) an[t] = s.an[t];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int v = blockIdx.x * RIG_WARPS + (threadIdx.x >> 5);
  if (v >= r.V) return;
  float po[3];
  for (int c = 0; c < 3; c++) {
    const float* D = r.posedirs_t + ((size_t)v * 3 + c) * K;
    float a = 0.f;
    for (int k = lane; k < K; k += 32) a += feat[k] * D[k];
    po[c] = warp_sum(a);
  }
  float T[12];
  for (int t = 0; t < 12; t++) T[t] = 0.f;
  for (int j = lane; j < r.J; j += 32) {
    const float w = r.lbs_weights[(size_t)v * r.J + j];
    for (int t = 0; t < 12; t++) T[t] += w * an[12 * j + t];
  }
  for (int t = 0; t < 12; t++) T[t] = warp_sum(T[t]);
  if (lane == 0) {
    float x[3];
    for (int c = 0; c < 3; c++) x[c] = s.vs[3 * v + c] + r.pose_offset0[3 * v + c];
    for (int c = 0; c < 3; c++) {
      mesh_wo[3 * v + c] = T[4 * c] * x[0] + T[4 * c + 1] * x[1] + T[4 * c + 2] * x[2] + T[4 * c + 3];
      s.pv[3 * v + c] = po[c];
    }
  }
}

__device__ __forceinline__ float3 rig_ld3(const float* p, int i) { return make_float3(p[3 * i], p[3 * i + 1], p[3 * i + 2]); }
__device__ __forceinline__ float3 rig_mid(float3 a, float3 b) {
  return make_float3((a.x + b.x) * 0.5f, (a.y + b.y) * 0.5f, (a.z + b.z) * 0.5f);
}

// row q of the first subdivision level
__device__ __forceinline__ float3 rig_level1(const B2RRig& r, const float* x, int q) {
  if (q < r.V) return rig_ld3(x, q);
  const int2 e = reinterpret_cast<const int2*>(r.sub1)[q - r.V];
  return rig_mid(rig_ld3(x, e.x), rig_ld3(x, e.y));
}

__device__ __forceinline__ float3 rig_level2(const B2RRig& r, const float* x, int p) {
  if (p < r.V1) return rig_level1(r, x, p);
  const int2 e = reinterpret_cast<const int2*>(r.sub2)[p - r.V1];
  return rig_mid(rig_level1(r, x, e.x), rig_level1(r, x, e.y));
}

__device__ __forceinline__ void rig_st3(float* p, int i, float3 v) {
  p[3 * i] = v.x;
  p[3 * i + 1] = v.y;
  p[3 * i + 2] = v.z;
}

__global__ void __launch_bounds__(RIG_THREADS) rig_upsample_kernel(const B2RRig r, const RigPtrs s,
                                                                   const float* __restrict__ mesh_wo,
                                                                   float* __restrict__ mesh, float* __restrict__ pose_offset,
                                                                   float* __restrict__ expr_offset) {
  const int p = blockIdx.x * RIG_THREADS + threadIdx.x;
  if (p >= r.P) return;
  rig_st3(mesh, p, rig_level2(r, mesh_wo, p));
  rig_st3(pose_offset, p, r.mask[p] ? rig_level2(r, s.pv, p) : make_float3(0.f, 0.f, 0.f));
  rig_st3(expr_offset, p, rig_level2(r, s.ev, p));
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward

constexpr int RIG_PART_A = 3 * RIG_JMAX;
constexpr int RIG_PART_W = RIG_PART_A + RIG_CMAX;  // per-warp partial: W^T g (J,3), then expr_dirs^T g_expr (NE)

__global__ void __launch_bounds__(RIG_THREADS) rig_bwd_vertex_kernel(const B2RRig r, const RigPtrs s,
                                                                     const float* __restrict__ dmesh,
                                                                     const float* __restrict__ dexpr) {
  __shared__ float an[12 * RIG_JMAX];
  __shared__ double wpart[RIG_WARPS][RIG_PART_W];
  for (int t = threadIdx.x; t < 12 * r.J; t += RIG_THREADS) an[t] = s.an[t];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double aA[2][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}}, aE[4] = {0.0, 0.0, 0.0, 0.0};
  for (int v = blockIdx.x * RIG_WARPS + warp; v < r.V; v += RIG_PART_BLOCKS * RIG_WARPS) {
    float g[3] = {0.f, 0.f, 0.f}, ge[3] = {0.f, 0.f, 0.f};
    for (int q = r.upT_offsets[v] + lane; q < r.upT_offsets[v + 1]; q += 32) {
      const int p = r.upT_rows[q];
      const float w = r.upT_w[q];
      for (int c = 0; c < 3; c++) {
        if (dmesh) g[c] += w * dmesh[3 * p + c];
        if (dexpr) ge[c] += w * dexpr[3 * p + c];
      }
    }
    for (int c = 0; c < 3; c++) {
      g[c] = warp_sum(g[c]);
      ge[c] = warp_sum(ge[c]);
    }
    float T[9];
    for (int t = 0; t < 9; t++) T[t] = 0.f;
    for (int k = 0; k < 2; k++) {
      const int j = lane + 32 * k;
      if (j >= r.J) continue;
      const float w = r.lbs_weights[(size_t)v * r.J + j];
      for (int c = 0; c < 3; c++) aA[k][c] += (double)w * (double)g[c];
      for (int a = 0; a < 3; a++)
        for (int c = 0; c < 3; c++) T[3 * a + c] += w * an[12 * j + 4 * a + c];
    }
    for (int t = 0; t < 9; t++) T[t] = warp_sum(T[t]);
    if (lane == 0)
      for (int c = 0; c < 3; c++) s.dvs[3 * v + c] = T[c] * g[0] + T[3 + c] * g[1] + T[6 + c] * g[2];
    for (int k = 0; k < 4; k++) {
      const int n = lane + 32 * k;
      if (n >= r.NE) continue;
      double a = 0.0;
      for (int c = 0; c < 3; c++) a += (double)r.expr_dirs[((size_t)v * 3 + c) * r.NE + n] * (double)ge[c];
      aE[k] += a;
    }
  }
  for (int k = 0; k < 2; k++)
    for (int c = 0; c < 3; c++) wpart[warp][3 * (lane + 32 * k) + c] = aA[k][c];
  for (int k = 0; k < 4; k++) wpart[warp][RIG_PART_A + lane + 32 * k] = aE[k];
  __syncthreads();
  for (int t = threadIdx.x; t < RIG_PART_W; t += RIG_THREADS) {
    double a = 0.0;
    for (int w = 0; w < RIG_WARPS; w++) a += wpart[w][t];
    if (t < RIG_PART_A) s.part_a[(size_t)blockIdx.x * RIG_PART_A + t] = a;
    else s.part_e[(size_t)blockIdx.x * RIG_CMAX + (t - RIG_PART_A)] = a;
  }
}

__global__ void __launch_bounds__(RIG_CHAIN_THREADS) rig_bwd_chain_kernel(const B2RRig r, const RigPtrs s,
                                                                          const float* __restrict__ djm,
                                                                          const B2RRigGrads gr) {
  extern __shared__ __align__(16) unsigned char rig_smem[];
  RigBackSm& sm = *reinterpret_cast<RigBackSm*>(rig_smem);
  const int tid = threadIdx.x, J = r.J;
  for (int t = tid; t < 3 * J; t += RIG_CHAIN_THREADS) {
    double a = 0.0;
    for (int b = 0; b < RIG_PART_BLOCKS; b++) a += s.part_a[(size_t)b * RIG_PART_A + t];
    sm.dAt[t] = a;
  }
  for (int n = tid; n < r.NE; n += RIG_CHAIN_THREADS) {
    double a = 0.0;
    for (int b = 0; b < RIG_PART_BLOCKS; b++) a += s.part_e[(size_t)b * RIG_CMAX + n];
    gr.expr[n] = (float)a;
  }
  rig_chains(r, nullptr, sm.c, false, s.jn);  // its barriers also publish sm.dAt
  // joint_mats = Af Ai: the adjoints of the frame (Af) and inverse-neutral (Ai) rel transforms
  if (tid < J) {
    double Ai[12], Af[12], dAfR[9], dAft[3], dAiR[9], dAit[3];
    chain_rel(tid, sm.c.jnp, sm.c.G[2], Ai);
    chain_rel(tid, sm.c.jzp, sm.c.G[3], Af);
    double dM[12];
    for (int t = 0; t < 12; t++) dM[t] = djm ? (double)djm[16 * tid + t] : 0.0;  // the last row has no path
    for (int a = 0; a < 3; a++) {
      for (int c = 0; c < 3; c++) {
        dAfR[3 * a + c] = dM[4 * a] * Ai[4 * c] + dM[4 * a + 1] * Ai[4 * c + 1] + dM[4 * a + 2] * Ai[4 * c + 2] +
                          dM[4 * a + 3] * Ai[4 * c + 3];
        dAiR[3 * a + c] = Af[a] * dM[c] + Af[4 + a] * dM[4 + c] + Af[8 + a] * dM[8 + c];
      }
      dAft[a] = dM[4 * a + 3];
      dAit[a] = Af[a] * dM[3] + Af[4 + a] * dM[7] + Af[8 + a] * dM[11];
    }
    chain_own(tid, sm.c.jzp, sm.c.G[3], dAfR, dAft, nullptr, sm.dG[0], sm.dj[0]);
    chain_own(tid, sm.c.jnp, sm.c.G[2], dAiR, dAit, nullptr, sm.dG[1], sm.dj[1]);
  }
  __syncthreads();
  const int grp = tid / RIG_JMAX, i = tid % RIG_JMAX;
  for (int d = sm.c.maxd; d >= 0; d--) {
    if (i < J && sm.c.depth[i] == d) {
      if (grp == 0) chain_back_step(i, J, r.parents, sm.c.rf, sm.c.jzp, sm.c.G[3], sm.dG[0], sm.dtl[0], sm.dj[0], sm.dR);
      else chain_back_step(i, J, r.parents, r.rot_inv, sm.c.jnp, sm.c.G[2], sm.dG[1], sm.dtl[1], sm.dj[1], nullptr);
    }
    __syncthreads();
  }
  // d full_pose; then the 大-pose chain (dA from the LBS partials, d posed from the inverse chain) and the zero-pose
  // chain (d posed from the frame chain) on the joints
  double djzp[3], djnp[3];
  if (tid < J) {
    double da[3] = {0.0, 0.0, 0.0};
    if (djm) {
      const double a[3] = {(double)r.full_pose[3 * tid], (double)r.full_pose[3 * tid + 1], (double)r.full_pose[3 * tid + 2]};
      aa_to_matrix_bwd(a, sm.dR + 9 * tid, da);
    }
    for (int c = 0; c < 3; c++) {
      gr.full_pose[3 * tid + c] = sm.c.bad ? nanf("") : (float)da[c];
      djzp[c] = sm.dj[0][3 * tid + c];
      djnp[c] = sm.dj[1][3 * tid + c];
    }
  }
  __syncthreads();
  if (tid < J) {
    chain_own(tid, sm.c.jn, sm.c.G[0], nullptr, sm.dAt + 3 * tid, djnp, sm.dG[0], sm.dj[0]);
    const double zero[3] = {0.0, 0.0, 0.0};
    chain_own(tid, sm.c.jn, sm.c.G[1], nullptr, zero, djzp, sm.dG[1], sm.dj[1]);
  }
  __syncthreads();
  for (int d = sm.c.maxd; d >= 0; d--) {
    if (i < J && sm.c.depth[i] == d)
      chain_back_step(i, J, r.parents, grp == 0 ? r.rot_neutral : r.rot_zero, sm.c.jn, sm.c.G[grp], sm.dG[grp],
                      sm.dtl[grp], sm.dj[grp], nullptr);
    __syncthreads();
  }
  if (tid < J)
    for (int c = 0; c < 3; c++) {
      const double d = sm.c.bad ? nan("") : sm.dj[0][3 * tid + c] + sm.dj[1][3 * tid + c];
      s.djn[3 * tid + c] = d;
      gr.joint_offset[3 * tid + c] = tid > 0 ? (float)d : 0.f;  // get_joint_offset zeroes the root
    }
}

__global__ void __launch_bounds__(RIG_THREADS) rig_bwd_shape_kernel(const B2RRig r, const RigPtrs s) {
  __shared__ double djn[3 * RIG_JMAX];
  __shared__ double wpart[RIG_WARPS][RIG_CMAX];
  for (int t = threadIdx.x; t < 3 * r.J; t += RIG_THREADS) djn[t] = s.djn[t];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double aB[4] = {0.0, 0.0, 0.0, 0.0};
  for (int v = blockIdx.x * RIG_WARPS + warp; v < r.V; v += RIG_PART_BLOCKS * RIG_WARPS) {
    double d[3];
    for (int c = 0; c < 3; c++) d[c] = (double)s.dvs[3 * v + c];
    for (int q = r.jregT_offsets[v]; q < r.jregT_offsets[v + 1]; q++) {  // every lane, same order
      const int k = r.jregT_rows[q];
      const double w = (double)r.jregT_vals[q];
      for (int c = 0; c < 3; c++) d[c] += w * djn[3 * k + c];
    }
    for (int k = 0; k < 4; k++) {
      const int n = lane + 32 * k;
      if (n >= r.NB) continue;
      double a = 0.0;
      for (int c = 0; c < 3; c++) a += (double)r.shapedirs[((size_t)v * 3 + c) * r.NB + n] * d[c];
      aB[k] += a;
    }
  }
  for (int k = 0; k < 4; k++) wpart[warp][lane + 32 * k] = aB[k];
  __syncthreads();
  for (int t = threadIdx.x; t < RIG_CMAX; t += RIG_THREADS) {
    double a = 0.0;
    for (int w = 0; w < RIG_WARPS; w++) a += wpart[w][t];
    s.part_b[(size_t)blockIdx.x * RIG_CMAX + t] = a;
  }
}

__global__ void __launch_bounds__(RIG_CMAX) rig_bwd_reduce_kernel(const B2RRig r, const RigPtrs s, float* __restrict__ dshape) {
  const int n = threadIdx.x;
  if (n >= r.NB) return;
  double a = 0.0;
  for (int b = 0; b < RIG_PART_BLOCKS; b++) a += s.part_b[(size_t)b * RIG_CMAX + n];
  dshape[n] = (float)a;
}

// ---------------------------------------------------------------------------------------------------------------------

size_t rig_scratch_bytes(int V, int J, int NB, int NE) { return rig_layout(V, J, NB, NE).total; }

int launch_rig_forward(const B2RRig& r, float* mesh, float* mesh_wo, float* joint_mats, float* pose_offset,
                       float* expr_offset, float* pose_6d, void* scratch, cudaStream_t st) {
  const RigPtrs s = rig_ptrs(r, scratch);
  const int vblocks = (r.V + RIG_WARPS - 1) / RIG_WARPS;
  {
    ProfScope p(K_MISC, st);
    launch_k(rig_shape_kernel, vblocks, RIG_THREADS, 0, st, true, r, s);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(rig_chain_kernel, 1, RIG_CHAIN_THREADS, sizeof(RigChainSm), st, true, r, s, joint_mats, pose_6d);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(rig_lbs_kernel, vblocks, RIG_THREADS, 0, st, true, r, s, mesh_wo);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(rig_upsample_kernel, (r.P + RIG_THREADS - 1) / RIG_THREADS, RIG_THREADS, 0, st, true, r, s,
             (const float*)mesh_wo, mesh, pose_offset, expr_offset);
  }
  return check_launch();
}

int launch_rig_backward(const B2RRig& r, const float* dmesh, const float* djm, const float* dexpr, const B2RRigGrads& g,
                        void* scratch, cudaStream_t st) {
  const RigPtrs s = rig_ptrs(r, scratch);
  // per device; a host-side attribute, not a stream operation, so it may be set while a graph is being captured
  const cudaError_t e = cudaFuncSetAttribute(rig_bwd_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)sizeof(RigBackSm));
  if (e != cudaSuccess) {
    g_last_cuda_error = (int)e;
    return B2R_E_CUDA;
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(rig_bwd_vertex_kernel, RIG_PART_BLOCKS, RIG_THREADS, 0, st, true, r, s, dmesh, dexpr);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(rig_bwd_chain_kernel, 1, RIG_CHAIN_THREADS, sizeof(RigBackSm), st, true, r, s, djm, g);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(rig_bwd_shape_kernel, RIG_PART_BLOCKS, RIG_THREADS, 0, st, true, r, s);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(rig_bwd_reduce_kernel, 1, RIG_CMAX, 0, st, true, r, s, g.shape_param);
  }
  return check_launch();
}

// =====================================================================================================================
// The frame's SMPL-X body mesh (get_smplx_outputs, avatar/main/model.py:37-58): smplx's SMPLX.forward + lbs with the
// frame's shape, expression, raw joint_offset, full_pose + pose_mean and transl, then optionally R^-1 (mesh - t).
//
// Forward:
//   rig_shape_kernel        (the rig's) vs = template + shapedirs . beta, ev = expr_dirs . expr; v_shaped = vs + ev.
//   body_chain_kernel       ONE CTA, fp64: J = J_regressor . v_shaped + joint_offset (every row) over the per-joint
//                           CSR; smplx's batch_rodrigues of full_pose + pose_mean; the pose feature (R - I of joints
//                           1..J-1); FK level by level; the rel transforms A; R^-1 by cofactors when a camera is given.
//   body_lbs_kernel         one warp per vertex: v_posed = v_shaped + feature . posedirs (kept for the backward),
//                           mesh = (W A) (v_posed, 1) + trans, then R^-1 (mesh - t).
// Backward:
//   body_bwd_vertex_kernel  fixed grid, one warp per vertex: g = R^-T dmesh; dv_posed = (W A)_R^T g; fp64 per-CTA
//                           partials of dA = W^T (g (v_posed, 1)^T), d feature = posedirs^T dv_posed and d trans.
//   body_bwd_reduce_kernel  one warp per partial entry: the CTAs' partials in a fixed order.
//   body_bwd_chain_kernel   ONE CTA: the chain recomputed from the saved joints, its adjoint in reverse level order,
//                           d rotation + d feature through batch_rodrigues' derivative (with its 1e-8 shift), d joints.
//   body_bwd_shape_kernel   fixed grid, one warp per vertex: dv_shaped = dv_posed + J_regressor^T dJ; fp64 per-CTA
//                           partials of shapedirs^T and expr_dirs^T dv_shaped.
//   body_bwd_coeff_kernel   ONE CTA: d shape_param and d expr from those partials in a fixed order.

constexpr int BODY_THREADS = 128;  // backward vertex kernel: four warps, so their fp64 partials fit static shared memory
constexpr int BODY_WARPS = BODY_THREADS / 32;
constexpr int BODY_PART_BLOCKS = 256;  // fixed, like RIG_PART_BLOCKS: the partials' bits never depend on the device
constexpr int BODY_PART_A = 12 * RIG_JMAX;  // dA (J,3,4)
constexpr int BODY_PART_F = 9 * RIG_JMAX;   // d feature (9 (J-1)), padded to whole lanes
constexpr int BODY_FEAT_PER_LANE = BODY_PART_F / 32;
constexpr int BODY_PART_W = BODY_PART_A + BODY_PART_F + 4;  // + d trans (3), padded
constexpr double BODY_RODRIGUES_SHIFT = 1e-8;               // lbs.batch_rodrigues: |r + 1e-8|

struct BodyLayout {
  size_t vs, ev, vp, dvs, feat, an, rinv, jn, djn, part_v, red, part_b, part_e, total;
};

inline BodyLayout body_layout(int V) {
  const size_t v = V > 0 ? (size_t)V : 1;
  BodyLayout L;
  size_t o = 0;
  L.vs = o; o += align_up(v * 3 * sizeof(float));
  L.ev = o; o += align_up(v * 3 * sizeof(float));
  L.vp = o; o += align_up(v * 3 * sizeof(float));
  L.dvs = o; o += align_up(v * 3 * sizeof(float));
  L.feat = o; o += align_up((size_t)9 * RIG_JMAX * sizeof(float));
  L.an = o; o += align_up((size_t)12 * RIG_JMAX * sizeof(float));
  L.rinv = o; o += align_up((size_t)9 * sizeof(float));
  L.jn = o; o += align_up((size_t)3 * RIG_JMAX * sizeof(double));
  L.djn = o; o += align_up((size_t)3 * RIG_JMAX * sizeof(double));
  L.part_v = o; o += align_up((size_t)BODY_PART_BLOCKS * BODY_PART_W * sizeof(double));
  L.red = o; o += align_up((size_t)BODY_PART_W * sizeof(double));
  L.part_b = o; o += align_up((size_t)RIG_PART_BLOCKS * RIG_CMAX * sizeof(double));
  L.part_e = o; o += align_up((size_t)RIG_PART_BLOCKS * RIG_CMAX * sizeof(double));
  L.total = o;
  return L;
}

struct BodyPtrs {
  float *vs, *ev, *vp, *dvs, *feat, *an, *rinv;
  double *jn, *djn, *part_v, *red, *part_b, *part_e;
};

inline BodyPtrs body_ptrs(const B2RSmplxBody& b, void* scratch) {
  const BodyLayout L = body_layout(b.rig.V);
  char* s = (char*)scratch;
  BodyPtrs p;
  p.vs = (float*)(s + L.vs);
  p.ev = (float*)(s + L.ev);
  p.vp = (float*)(s + L.vp);
  p.dvs = (float*)(s + L.dvs);
  p.feat = (float*)(s + L.feat);
  p.an = (float*)(s + L.an);
  p.rinv = (float*)(s + L.rinv);
  p.jn = (double*)(s + L.jn);
  p.djn = (double*)(s + L.djn);
  p.part_v = (double*)(s + L.part_v);
  p.red = (double*)(s + L.red);
  p.part_b = (double*)(s + L.part_b);
  p.part_e = (double*)(s + L.part_e);
  return p;
}

// smplx lbs.batch_rodrigues in fp64: angle = |r + 1e-8| (the shift on each component), d = r / angle, K = [d]x,
// R = I + sin(angle) K + (1 - cos(angle)) K K
__device__ __forceinline__ void rodrigues_terms(const double r[3], double e[3], double& angle, double K[9],
                                                double KK[9]) {
  for (int c = 0; c < 3; c++) e[c] = r[c] + BODY_RODRIGUES_SHIFT;
  angle = sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
  const double d0 = r[0] / angle, d1 = r[1] / angle, d2 = r[2] / angle;
  K[0] = 0.0; K[1] = -d2; K[2] = d1;
  K[3] = d2; K[4] = 0.0; K[5] = -d0;
  K[6] = -d1; K[7] = d0; K[8] = 0.0;
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) KK[3 * a + b] = K[3 * a] * K[b] + K[3 * a + 1] * K[3 + b] + K[3 * a + 2] * K[6 + b];
}

__device__ void rodrigues(const double r[3], double R[9]) {
  double e[3], angle, K[9], KK[9];
  rodrigues_terms(r, e, angle, K, KK);
  const double s = sin(angle), c1 = 1.0 - cos(angle);
  for (int t = 0; t < 9; t++) R[t] = ((t % 4) == 0 ? 1.0 : 0.0) + s * K[t] + c1 * KK[t];
}

// dr = (dR/dr)^T dR through the shift: angle > 0 unless r = -1e-8 (1, 1, 1) exactly; there the norm's gradient is 0
__device__ void rodrigues_bwd(const double r[3], const double dR[9], double dr[3]) {
  double e[3], angle, K[9], KK[9];
  rodrigues_terms(r, e, angle, K, KK);
  const double s = sin(angle), co = cos(angle), c1 = 1.0 - co;
  double ds = 0.0, dc1 = 0.0, dK[9];
  for (int t = 0; t < 9; t++) {
    ds += dR[t] * K[t];
    dc1 += dR[t] * KK[t];
  }
  for (int a = 0; a < 3; a++)  // d(K K) = dK K + K dK: dK += c1 (dR K^T + K^T dR)
    for (int b = 0; b < 3; b++) {
      double acc = 0.0;
      for (int t = 0; t < 3; t++) acc += dR[3 * a + t] * K[3 * b + t] + K[3 * t + a] * dR[3 * t + b];
      dK[3 * a + b] = s * dR[3 * a + b] + c1 * acc;
    }
  const double dd[3] = {dK[7] - dK[5], dK[2] - dK[6], dK[3] - dK[1]};
  double dangle = ds * co + dc1 * s;
  for (int c = 0; c < 3; c++) {
    dr[c] = dd[c] / angle;
    dangle -= dd[c] * r[c] / (angle * angle);
  }
  const double inv = angle > 0.0 ? dangle / angle : 0.0;
  for (int c = 0; c < 3; c++) dr[c] += inv * e[c];
}

struct BodyChainSm {
  double jn[RIG_JMAX * 3], rot[RIG_JMAX * 9], G[RIG_JMAX * 12];
  int depth[RIG_JMAX];
  int maxd;
  int bad;
};

struct BodyBackSm {
  BodyChainSm c;
  double dG[RIG_JMAX * 12], dtl[RIG_JMAX * 3], dj[RIG_JMAX * 3], dR[RIG_JMAX * 9];
};
static_assert(sizeof(BodyBackSm) <= 48 * 1024, "the backward's single CTA fits static shared memory");

// the joints (from v_shaped, or the forward's saved ones), the rotations of full_pose + pose_mean, the depths, then FK
__device__ void body_chain(const B2RSmplxBody& b, const BodyPtrs& s, BodyChainSm& sm, bool from_vs) {
  const B2RRig& r = b.rig;
  const int tid = threadIdx.x, J = r.J;
  if (tid < J) {
    if (from_vs) {
      double acc[3] = {0.0, 0.0, 0.0};
      for (int q = r.jreg_offsets[tid]; q < r.jreg_offsets[tid + 1]; q++) {
        const int v = r.jreg_cols[q];
        const double w = (double)r.jreg_vals[q];
        for (int c = 0; c < 3; c++) acc[c] += w * (double)(s.vs[3 * v + c] + s.ev[3 * v + c]);
      }
      for (int c = 0; c < 3; c++) sm.jn[3 * tid + c] = acc[c] + (double)b.joint_offset[3 * tid + c];
    } else {
      for (int c = 0; c < 3; c++) sm.jn[3 * tid + c] = s.jn[3 * tid + c];
    }
    double a[3];
    for (int c = 0; c < 3; c++) a[c] = (double)b.full_pose[3 * tid + c] + (double)b.pose_mean[3 * tid + c];
    rodrigues(a, sm.rot + 9 * tid);
  }
  if (tid == 0) chain_depths(r.parents, J, sm.depth, sm.maxd, sm.bad);
  __syncthreads();
  for (int d = 0; d <= sm.maxd; d++) {
    if (tid < J && sm.depth[tid] == d) chain_step(tid, r.parents, sm.rot, sm.jn, sm.G);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(RIG_JMAX) body_chain_kernel(const B2RSmplxBody b, const BodyPtrs s) {
  __shared__ BodyChainSm sm;
  body_chain(b, s, sm, true);
  const int tid = threadIdx.x;
  if (tid == 0 && b.cam_R) {  // R^-1 by cofactors (camera._inv3's expressions), fp32
    const float* R = b.cam_R;
    const float a = R[0], bb = R[1], c = R[2], d = R[3], e = R[4], f = R[5], g = R[6], h = R[7], i = R[8];
    const float adj[9] = {e * i - f * h, c * h - bb * i, bb * f - c * e, f * g - d * i, a * i - c * g,
                          c * d - a * f, d * h - e * g, bb * g - a * h, a * e - bb * d};
    const float det = a * (e * i - f * h) - bb * (d * i - f * g) + c * (d * h - e * g);
    for (int t = 0; t < 9; t++) s.rinv[t] = adj[t] / det;
  }
  if (tid >= b.rig.J) return;
  for (int c = 0; c < 3; c++) s.jn[3 * tid + c] = sm.jn[3 * tid + c];
  double A[12];
  chain_rel(tid, sm.jn, sm.G, A);
  for (int t = 0; t < 12; t++) s.an[12 * tid + t] = sm.bad ? nanf("") : (float)A[t];
  if (tid >= 1)
    for (int t = 0; t < 9; t++) s.feat[9 * (tid - 1) + t] = (float)(sm.rot[9 * tid + t] - ((t % 4) == 0 ? 1.0 : 0.0));
}

__global__ void __launch_bounds__(RIG_THREADS) body_lbs_kernel(const B2RSmplxBody b, const BodyPtrs s,
                                                               float* __restrict__ mesh) {
  __shared__ float feat[9 * RIG_JMAX];
  __shared__ float an[12 * RIG_JMAX];
  const B2RRig& r = b.rig;
  const int K = 9 * (r.J - 1);
  for (int t = threadIdx.x; t < K; t += RIG_THREADS) feat[t] = s.feat[t];
  for (int t = threadIdx.x; t < 12 * r.J; t += RIG_THREADS) an[t] = s.an[t];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int v = blockIdx.x * RIG_WARPS + (threadIdx.x >> 5);
  if (v >= r.V) return;
  float po[3];
  for (int c = 0; c < 3; c++) {
    const float* D = r.posedirs_t + ((size_t)v * 3 + c) * K;
    float a = 0.f;
    for (int k = lane; k < K; k += 32) a += feat[k] * D[k];
    po[c] = warp_sum(a);
  }
  float T[12];
  for (int t = 0; t < 12; t++) T[t] = 0.f;
  for (int j = lane; j < r.J; j += 32) {
    const float w = r.lbs_weights[(size_t)v * r.J + j];
    for (int t = 0; t < 12; t++) T[t] += w * an[12 * j + t];
  }
  for (int t = 0; t < 12; t++) T[t] = warp_sum(T[t]);
  if (lane == 0) {
    float x[3], m[3];
    for (int c = 0; c < 3; c++) {
      x[c] = po[c] + (s.vs[3 * v + c] + s.ev[3 * v + c]);  // v_posed = pose_offsets + v_shaped
      s.vp[3 * v + c] = x[c];
    }
    for (int c = 0; c < 3; c++) m[c] = (T[4 * c] * x[0] + T[4 * c + 1] * x[1] + T[4 * c + 2] * x[2] + T[4 * c + 3]) +
                                       b.trans[c];
    if (b.cam_R) {
      float d[3];
      for (int c = 0; c < 3; c++) d[c] = m[c] - b.cam_t[c];
      for (int c = 0; c < 3; c++) m[c] = s.rinv[3 * c] * d[0] + s.rinv[3 * c + 1] * d[1] + s.rinv[3 * c + 2] * d[2];
    }
    for (int c = 0; c < 3; c++) mesh[3 * v + c] = m[c];
  }
}

__global__ void __launch_bounds__(BODY_THREADS) body_bwd_vertex_kernel(const B2RSmplxBody b, const BodyPtrs s,
                                                                       const float* __restrict__ dmesh) {
  __shared__ float an[12 * RIG_JMAX];
  __shared__ double wpart[BODY_WARPS][BODY_PART_W];
  const B2RRig& r = b.rig;
  for (int t = threadIdx.x; t < 12 * r.J; t += BODY_THREADS) an[t] = s.an[t];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int K = 9 * (r.J - 1);
  float ri[9];
  for (int t = 0; t < 9; t++) ri[t] = b.cam_R ? s.rinv[t] : ((t % 4) == 0 ? 1.f : 0.f);
  double aA[2][12], aF[BODY_FEAT_PER_LANE], aT[3] = {0.0, 0.0, 0.0};
#pragma unroll
  for (int k = 0; k < 2; k++)
#pragma unroll
    for (int t = 0; t < 12; t++) aA[k][t] = 0.0;
#pragma unroll
  for (int i = 0; i < BODY_FEAT_PER_LANE; i++) aF[i] = 0.0;
  for (int v = blockIdx.x * BODY_WARPS + warp; v < r.V; v += BODY_PART_BLOCKS * BODY_WARPS) {
    float go[3], g[3], x[3];
    for (int c = 0; c < 3; c++) {
      go[c] = dmesh ? dmesh[3 * v + c] : 0.f;
      x[c] = s.vp[3 * v + c];
    }
    for (int c = 0; c < 3; c++) g[c] = b.cam_R ? ri[c] * go[0] + ri[3 + c] * go[1] + ri[6 + c] * go[2] : go[c];
    if (lane == 0)
      for (int c = 0; c < 3; c++) aT[c] += (double)g[c];
    float T[9];
    for (int t = 0; t < 9; t++) T[t] = 0.f;
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const int j = lane + 32 * k;
      if (j >= r.J) continue;
      const float w = r.lbs_weights[(size_t)v * r.J + j];
#pragma unroll
      for (int a = 0; a < 3; a++) {
        const double wg = (double)w * (double)g[a];
#pragma unroll
        for (int c = 0; c < 3; c++) aA[k][4 * a + c] += wg * (double)x[c];
        aA[k][4 * a + 3] += wg;
      }
      for (int a = 0; a < 3; a++)
        for (int c = 0; c < 3; c++) T[3 * a + c] += w * an[12 * j + 4 * a + c];
    }
    for (int t = 0; t < 9; t++) T[t] = warp_sum(T[t]);
    float dvp[3];
    for (int c = 0; c < 3; c++) dvp[c] = T[c] * g[0] + T[3 + c] * g[1] + T[6 + c] * g[2];
    if (lane == 0)
      for (int c = 0; c < 3; c++) s.dvs[3 * v + c] = dvp[c];
    const float* D = r.posedirs_t + (size_t)v * 3 * K;
#pragma unroll
    for (int i = 0; i < BODY_FEAT_PER_LANE; i++) {
      const int k = lane + 32 * i;
      if (k < K)
        aF[i] += ((double)D[k] * (double)dvp[0] + (double)D[K + k] * (double)dvp[1]) + (double)D[2 * K + k] * (double)dvp[2];
    }
  }
#pragma unroll
  for (int k = 0; k < 2; k++)
#pragma unroll
    for (int t = 0; t < 12; t++) wpart[warp][12 * (lane + 32 * k) + t] = aA[k][t];
#pragma unroll
  for (int i = 0; i < BODY_FEAT_PER_LANE; i++) wpart[warp][BODY_PART_A + lane + 32 * i] = aF[i];
  if (lane == 0)
    for (int c = 0; c < 4; c++) wpart[warp][BODY_PART_A + BODY_PART_F + c] = c < 3 ? aT[c] : 0.0;
  __syncthreads();
  for (int t = threadIdx.x; t < BODY_PART_W; t += BODY_THREADS) {
    double a = 0.0;
    for (int w = 0; w < BODY_WARPS; w++) a += wpart[w][t];
    s.part_v[(size_t)blockIdx.x * BODY_PART_W + t] = a;
  }
}

__global__ void __launch_bounds__(RIG_THREADS) body_bwd_reduce_kernel(const BodyPtrs s) {
  const int t = blockIdx.x * RIG_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= BODY_PART_W) return;
  double a = 0.0;
  for (int blk = lane; blk < BODY_PART_BLOCKS; blk += 32) a += s.part_v[(size_t)blk * BODY_PART_W + t];
  a = warp_sum(a);
  if (lane == 0) s.red[t] = a;
}

__global__ void __launch_bounds__(RIG_JMAX) body_bwd_chain_kernel(const B2RSmplxBody b, const BodyPtrs s,
                                                                  const B2RSmplxBodyGrads gr) {
  __shared__ BodyBackSm sm;
  const B2RRig& r = b.rig;
  const int tid = threadIdx.x, J = r.J;
  body_chain(b, s, sm.c, false);
  if (tid < J) {
    const double* dA = s.red + 12 * tid;
    double dAR[9], dAt[3];
    for (int a = 0; a < 3; a++) {
      for (int c = 0; c < 3; c++) dAR[3 * a + c] = dA[4 * a + c];
      dAt[a] = dA[4 * a + 3];
    }
    chain_own(tid, sm.c.jn, sm.c.G, dAR, dAt, nullptr, sm.dG, sm.dj);
  }
  if (tid < 3) gr.trans[tid] = (float)s.red[BODY_PART_A + BODY_PART_F + tid];
  __syncthreads();
  for (int d = sm.c.maxd; d >= 0; d--) {
    if (tid < J && sm.c.depth[tid] == d)
      chain_back_step(tid, J, r.parents, sm.c.rot, sm.c.jn, sm.c.G, sm.dG, sm.dtl, sm.dj, sm.dR);
    __syncthreads();
  }
  if (tid >= J) return;
  double dR[9], a[3], da[3];
  for (int t = 0; t < 9; t++) dR[t] = sm.dR[9 * tid + t] + (tid >= 1 ? s.red[BODY_PART_A + 9 * (tid - 1) + t] : 0.0);
  for (int c = 0; c < 3; c++) a[c] = (double)b.full_pose[3 * tid + c] + (double)b.pose_mean[3 * tid + c];
  rodrigues_bwd(a, dR, da);
  for (int c = 0; c < 3; c++) {
    const double dj = sm.c.bad ? nan("") : sm.dj[3 * tid + c];
    s.djn[3 * tid + c] = dj;
    gr.joint_offset[3 * tid + c] = (float)dj;
    gr.full_pose[3 * tid + c] = sm.c.bad ? nanf("") : (float)da[c];
  }
}

__global__ void __launch_bounds__(RIG_THREADS) body_bwd_shape_kernel(const B2RSmplxBody b, const BodyPtrs s) {
  __shared__ double djn[3 * RIG_JMAX];
  __shared__ double wpart[RIG_WARPS][2 * RIG_CMAX];
  const B2RRig& r = b.rig;
  for (int t = threadIdx.x; t < 3 * r.J; t += RIG_THREADS) djn[t] = s.djn[t];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double aB[4] = {0.0, 0.0, 0.0, 0.0}, aE[4] = {0.0, 0.0, 0.0, 0.0};
  for (int v = blockIdx.x * RIG_WARPS + warp; v < r.V; v += RIG_PART_BLOCKS * RIG_WARPS) {
    double d[3];
    for (int c = 0; c < 3; c++) d[c] = (double)s.dvs[3 * v + c];
    for (int q = r.jregT_offsets[v]; q < r.jregT_offsets[v + 1]; q++) {  // every lane, same order
      const int k = r.jregT_rows[q];
      const double w = (double)r.jregT_vals[q];
      for (int c = 0; c < 3; c++) d[c] += w * djn[3 * k + c];
    }
    for (int k = 0; k < 4; k++) {
      const int n = lane + 32 * k;
      if (n < r.NB) {
        double a = 0.0;
        for (int c = 0; c < 3; c++) a += (double)r.shapedirs[((size_t)v * 3 + c) * r.NB + n] * d[c];
        aB[k] += a;
      }
      if (n < r.NE) {
        double a = 0.0;
        for (int c = 0; c < 3; c++) a += (double)r.expr_dirs[((size_t)v * 3 + c) * r.NE + n] * d[c];
        aE[k] += a;
      }
    }
  }
  for (int k = 0; k < 4; k++) {
    wpart[warp][lane + 32 * k] = aB[k];
    wpart[warp][RIG_CMAX + lane + 32 * k] = aE[k];
  }
  __syncthreads();
  for (int t = threadIdx.x; t < 2 * RIG_CMAX; t += RIG_THREADS) {
    double a = 0.0;
    for (int w = 0; w < RIG_WARPS; w++) a += wpart[w][t];
    (t < RIG_CMAX ? s.part_b : s.part_e)[(size_t)blockIdx.x * RIG_CMAX + t % RIG_CMAX] = a;
  }
}

__global__ void __launch_bounds__(2 * RIG_CMAX) body_bwd_coeff_kernel(const B2RSmplxBody b, const BodyPtrs s,
                                                                      const B2RSmplxBodyGrads gr) {
  const int t = threadIdx.x, n = t % RIG_CMAX;
  const bool shape = t < RIG_CMAX;
  if (n >= (shape ? b.rig.NB : b.rig.NE)) return;
  const double* part = shape ? s.part_b : s.part_e;
  double a = 0.0;
  for (int blk = 0; blk < RIG_PART_BLOCKS; blk++) a += part[(size_t)blk * RIG_CMAX + n];
  (shape ? gr.shape_param : gr.expr)[n] = (float)a;
}

// smplx's output.joints[:J]: batch_rigid_transform's posed joints (the chain's translations) + transl, from the
// forward's saved rest joints -- the same chain the backward reruns
__global__ void __launch_bounds__(RIG_JMAX) body_joints_kernel(const B2RSmplxBody b, const BodyPtrs s,
                                                               float* __restrict__ joints) {
  __shared__ BodyChainSm sm;
  body_chain(b, s, sm, false);
  const int tid = threadIdx.x;
  if (tid >= b.rig.J) return;
  for (int c = 0; c < 3; c++) joints[3 * tid + c] = sm.bad ? nanf("") : (float)sm.G[12 * tid + 4 * c + 3] + b.trans[c];
}

size_t smplx_body_scratch_bytes(int V) { return body_layout(V).total; }

int launch_smplx_body_joints(const B2RSmplxBody& body, const void* scratch, float* joints, cudaStream_t st) {
  const B2RSmplxBody b = with_body_inputs(body);
  const BodyPtrs s = body_ptrs(b, const_cast<void*>(scratch));  // the kernel only reads the saved joints
  ProfScope p(K_MISC, st);
  launch_k(body_joints_kernel, 1, RIG_JMAX, 0, st, true, b, s, joints);
  return check_launch();
}

int launch_smplx_body_forward(const B2RSmplxBody& body, float* mesh, void* scratch, cudaStream_t st) {
  const B2RSmplxBody b = with_body_inputs(body);
  const BodyPtrs s = body_ptrs(b, scratch);
  RigPtrs shape = {};  // the rig's shape pass writes v_shaped's two parts into the body's scratch
  shape.vs = s.vs;
  shape.ev = s.ev;
  const int vblocks = (b.rig.V + RIG_WARPS - 1) / RIG_WARPS;
  {
    ProfScope p(K_MISC, st);
    launch_k(rig_shape_kernel, vblocks, RIG_THREADS, 0, st, true, b.rig, shape);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(body_chain_kernel, 1, RIG_JMAX, 0, st, true, b, s);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(body_lbs_kernel, vblocks, RIG_THREADS, 0, st, true, b, s, mesh);
  }
  return check_launch();
}

int launch_smplx_body_backward(const B2RSmplxBody& body, const float* dmesh, const B2RSmplxBodyGrads& g, void* scratch,
                               cudaStream_t st) {
  const B2RSmplxBody b = with_body_inputs(body);
  const BodyPtrs s = body_ptrs(b, scratch);
  {
    ProfScope p(K_MISC, st);
    launch_k(body_bwd_vertex_kernel, BODY_PART_BLOCKS, BODY_THREADS, 0, st, true, b, s, dmesh);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(body_bwd_reduce_kernel, (BODY_PART_W + RIG_WARPS - 1) / RIG_WARPS, RIG_THREADS, 0, st, true, s);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(body_bwd_chain_kernel, 1, RIG_JMAX, 0, st, true, b, s, g);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(body_bwd_shape_kernel, RIG_PART_BLOCKS, RIG_THREADS, 0, st, true, b, s);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(body_bwd_coeff_kernel, 1, 2 * RIG_CMAX, 0, st, true, b, s, g);
  }
  return check_launch();
}

}  // namespace b2r
