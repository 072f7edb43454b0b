// animate.cu -- the per-frame host work of ExAvatar's animation scripts (avatar/main/animate.py,
// animate_view_rot.py, get_neutral_pose.py) as device ops, so a video frame goes from the SMPL-X parameters and the
// source frame's bytes to one uint8 panel without a host synchronisation:
//   * orbit_camera_kernel  pytorch3d's look_at_view_transform and the script's torch.inverse of its R (one thread),
//                          with the frame-0 anchors of animate_view_rot.py:85-91;
//   * orbit_points_kernel  the x / z recentring of animate_view_rot.py:92,103 and the view transform of :97;
//   * panel_kernel         the (H, 3W, 3) BGR frame of animate.py:86,94 before the text.
//
// The file is compiled with --fmad=false: the camera and the points are the scripts' fp32 expressions rounded
// operation by operation (include/b200raster.h states each one), and the panel is numpy's truncating cast.
#include "common.cuh"

namespace b2r {

constexpr int OC_AT = 0, OC_ELEV = 3, OC_DIST = 4, OC_R = 5, OC_T = 14, OC_ROOT = 17;
static_assert(OC_ROOT + 3 == B2R_ORBIT_STATE, "the state block's layout");

// camera._inv3's cofactor expressions in fp32 (R row-major)
__device__ __forceinline__ void inv3(const float* R, float out[9]) {
  const float a = R[0], b = R[1], c = R[2], d = R[3], e = R[4], f = R[5], g = R[6], h = R[7], i = R[8];
  const float adj[9] = {e * i - f * h, c * h - b * i, b * f - c * e, f * g - d * i, a * i - c * g,
                        c * d - a * f, d * h - e * g, b * g - a * h, a * e - b * d};
  const float det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
  for (int t = 0; t < 9; t++) out[t] = adj[t] / det;
}

// torch.matmul of a 3x3 and a 3-vector, summed left to right
__device__ __forceinline__ void mul3(const float M[9], const float v[3], float out[3]) {
  for (int r = 0; r < 3; r++) out[r] = (M[3 * r] * v[0] + M[3 * r + 1] * v[1]) + M[3 * r + 2] * v[2];
}

// torch.cross(a, b, dim=1) of one row
__device__ __forceinline__ void cross3(const float a[3], const float b[3], float out[3]) {
  out[0] = a[1] * b[2] - a[2] * b[1];
  out[1] = a[2] * b[0] - a[0] * b[2];
  out[2] = a[0] * b[1] - a[1] * b[0];
}

// F.normalize(v, eps=1e-5): v / max(|v|_2, 1e-5)
__device__ __forceinline__ void normalize3(float v[3]) {
  const float n = fmaxf(sqrtf((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]), 1e-5f);
  for (int c = 0; c < 3; c++) v[c] = v[c] / n;
}

// sin and cos of an fp32 angle, rounded to fp32 from double sincospi(x / pi): within an ulp of torch's sinf / cosf,
// and sincospi's exact reduction keeps the thread off sinf's large-argument path and its local-memory stack
__device__ __forceinline__ void sincos_f(float x, float& s, float& c) {
  double sd, cd;
  sincospi((double)x / 3.141592653589793, &sd, &cd);
  s = (float)sd;
  c = (float)cd;
}

__global__ void __launch_bounds__(32) orbit_camera_kernel(const B2ROrbitCamera p) {
  if (threadIdx.x != 0) return;
  float* s = p.state;
  const int i = *p.index;
  float root_world[3];
  if (p.cam_R) {
    float Rinv[9], d[3], nt[3];
    inv3(p.cam_R, Rinv);
    for (int c = 0; c < 3; c++) d[c] = p.root_cam[c] - p.cam_t[c];
    mul3(Rinv, d, root_world);
    if (p.anchor == 2 || (p.anchor == 1 && i == 0)) {
      float cam_pos[3], v[3];
      for (int c = 0; c < 3; c++) nt[c] = -p.cam_t[c];
      mul3(Rinv, nt, cam_pos);
      for (int c = 0; c < 3; c++) {
        s[OC_AT + c] = root_world[c];
        v[c] = cam_pos[c] - root_world[c];
      }
      s[OC_ELEV] = atanf(fabsf(p.root_cam[1]) / fabsf(p.root_cam[2]));
      s[OC_DIST] = sqrtf((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
    }
  } else {
    for (int c = 0; c < 3; c++) root_world[c] = s[OC_AT + c];
  }
  float at[3];
  for (int c = 0; c < 3; c++) at[c] = s[OC_AT + c];
  const float elev = s[OC_ELEV], dist = s[OC_DIST];
  // Python's double arithmetic of `math.pi + math.pi*k*i/N`, then look_at_view_transform's float32 tensor of it
  const float azim = __double2float_rn(3.141592653589793 + ((3.141592653589793 * (double)p.k) * (double)i) /
                                                              (double)p.n_frames);
  float ce, se, sa, ca;
  sincos_f(elev, se, ce);
  sincos_f(azim, sa, ca);
  const float C[3] = {(dist * ce) * sa + at[0], dist * se + at[1], (dist * ce) * ca + at[2]};
  const float up[3] = {0.f, 1.f, 0.f};
  float z[3], x[3], y[3];
  for (int c = 0; c < 3; c++) z[c] = at[c] - C[c];
  normalize3(z);
  cross3(up, z, x);
  normalize3(x);
  cross3(z, x, y);
  normalize3(y);
  if (fabsf(x[0]) <= 5e-3f && fabsf(x[1]) <= 5e-3f && fabsf(x[2]) <= 5e-3f) {  // torch.isclose(x, 0, atol=5e-3)
    cross3(y, z, x);
    normalize3(x);
  }
  const float Rp[9] = {x[0], y[0], z[0], x[1], y[1], z[1], x[2], y[2], z[2]};
  float R[9];
  inv3(Rp, R);
  for (int t = 0; t < 9; t++) s[OC_R + t] = R[t];
  for (int j = 0; j < 3; j++) s[OC_T + j] = -((Rp[j] * C[0] + Rp[3 + j] * C[1]) + Rp[6 + j] * C[2]);
  for (int c = 0; c < 3; c++) s[OC_ROOT + c] = root_world[c];
}

constexpr int OP_THREADS = 256;

__global__ void __launch_bounds__(OP_THREADS) orbit_points_kernel(int n, const float* __restrict__ pts,
                                                                  const float* __restrict__ state, int view,
                                                                  float* __restrict__ out) {
  const int r = blockIdx.x * OP_THREADS + threadIdx.x;
  if (r >= n) return;
  const float* p = pts + 3 * (size_t)r;
  float q[3] = {(__ldg(p) - state[OC_ROOT]) + state[OC_AT], __ldg(p + 1),
                (__ldg(p + 2) - state[OC_ROOT + 2]) + state[OC_AT + 2]};
  if (view) {
    float v[3];
    mul3(state + OC_R, q, v);
    for (int c = 0; c < 3; c++) q[c] = v[c] + state[OC_T + c];
  }
  float* o = out + 3 * (size_t)r;
  for (int c = 0; c < 3; c++) o[c] = q[c];
}

// numpy's astype(np.uint8) on [0, 256): toward zero; below 0 and NaN give 0 (cvt.rzi.sat), above 255 gives 255
__device__ __forceinline__ uint32_t trunc_u8(float v) { return min(__float2uint_rz(v), 255u); }

constexpr int PN_THREADS = 256;
constexpr int PN_PIX = 8;  // pixels of one row per thread in the vector path: 24 bytes per panel, three 8-byte words

// VEC: W % 8 == 0 and aligned pointers; a thread owns pixels x0 .. x0 + 7 of row y.  Otherwise one pixel per thread.
template <bool VEC>
__global__ void __launch_bounds__(PN_THREADS) panel_kernel(const B2RAnimationPanel p, uint8_t* __restrict__ out) {
  const int W = p.width, H = p.height;
  const size_t HW = (size_t)W * H;
  if (VEC) {
    const int per_row = W / PN_PIX;
    const size_t g = (size_t)blockIdx.x * PN_THREADS + threadIdx.x;
    if (g >= (size_t)per_row * H) return;
    const int y = (int)(g / per_row), x0 = (int)(g - (size_t)y * per_row) * PN_PIX;
    const size_t pix = (size_t)y * W + x0;
    uint8_t* row = out + (size_t)y * 9 * W;
    // left: the frame's 24 bytes as they are
    const uint2* src = reinterpret_cast<const uint2*>(p.frame + 3 * pix);
    uint2* dst = reinterpret_cast<uint2*>(row + 3 * x0);
#pragma unroll
    for (int k = 0; k < 3; k++) dst[k] = __ldg(src + k);
    // middle: 24 floats, HWC
    const float4* m = reinterpret_cast<const float4*>(p.mesh_panel + 3 * pix);
    uint32_t b[3 * PN_PIX];
#pragma unroll
    for (int k = 0; k < 6; k++) {
      const float4 v = __ldg(m + k);
      b[4 * k] = trunc_u8(v.x), b[4 * k + 1] = trunc_u8(v.y), b[4 * k + 2] = trunc_u8(v.z), b[4 * k + 3] = trunc_u8(v.w);
    }
    unsigned long long* dm = reinterpret_cast<unsigned long long*>(row + 3 * W + 3 * x0);
#pragma unroll
    for (int k = 0; k < 3; k++) {
      unsigned long long w = 0;
#pragma unroll
      for (int j = 0; j < 8; j++) w |= (unsigned long long)b[8 * k + j] << (8 * j);
      dm[k] = w;
    }
    // right: the render's planes, channels reversed
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const float4* r = reinterpret_cast<const float4*>(p.render + (size_t)(2 - c) * HW + pix);
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const float4 v = __ldg(r + h);
        b[3 * (4 * h) + c] = trunc_u8(v.x * 255.f);
        b[3 * (4 * h + 1) + c] = trunc_u8(v.y * 255.f);
        b[3 * (4 * h + 2) + c] = trunc_u8(v.z * 255.f);
        b[3 * (4 * h + 3) + c] = trunc_u8(v.w * 255.f);
      }
    }
    unsigned long long* dr = reinterpret_cast<unsigned long long*>(row + 6 * W + 3 * x0);
#pragma unroll
    for (int k = 0; k < 3; k++) {
      unsigned long long w = 0;
#pragma unroll
      for (int j = 0; j < 8; j++) w |= (unsigned long long)b[8 * k + j] << (8 * j);
      dr[k] = w;
    }
  } else {
    const size_t q = (size_t)blockIdx.x * PN_THREADS + threadIdx.x;
    if (q >= HW) return;
    const size_t y = q / W, x = q - y * W;
    uint8_t* row = out + y * 9 * W;
#pragma unroll
    for (int c = 0; c < 3; c++) {
      row[3 * x + c] = p.frame[3 * q + c];
      row[3 * W + 3 * x + c] = (uint8_t)trunc_u8(p.mesh_panel[3 * q + c]);
      row[6 * W + 3 * x + c] = (uint8_t)trunc_u8(p.render[(2 - c) * HW + q] * 255.f);
    }
  }
}

int launch_orbit_camera(const B2ROrbitCamera& p, cudaStream_t st) {
  ProfScope ps(K_MISC, st);
  launch_k(orbit_camera_kernel, 1, 32, 0, st, true, p);
  return check_launch();
}

int launch_orbit_points(int n, const float* points, const float* state, int view, float* out, cudaStream_t st) {
  ProfScope ps(K_MISC, st);
  launch_k(orbit_points_kernel, (unsigned)((n + OP_THREADS - 1) / OP_THREADS), OP_THREADS, 0, st, false, n, points,
           state, view, out);
  return check_launch();
}

static bool aligned(const void* p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

int launch_animation_panel(const B2RAnimationPanel& p, uint8_t* out, cudaStream_t st) {
  const size_t HW = (size_t)p.width * p.height;
  const bool vec = p.width % PN_PIX == 0 && aligned(p.frame, 8) && aligned(out, 8) && aligned(p.mesh_panel, 16) &&
                   aligned(p.render, 16);
  ProfScope ps(K_MISC, st);
  if (vec)
    launch_k(panel_kernel<true>, (unsigned)((HW / PN_PIX + PN_THREADS - 1) / PN_THREADS), PN_THREADS, 0, st, false,
             p, out);
  else
    launch_k(panel_kernel<false>, (unsigned)((HW + PN_THREADS - 1) / PN_THREADS), PN_THREADS, 0, st, false, p, out);
  return check_launch();
}

}  // namespace b2r
