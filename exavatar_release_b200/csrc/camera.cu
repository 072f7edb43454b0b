// camera.cu -- b2r_camera_setup: the render settings of one camera, evaluated on the device (b200raster.h).
//
// ExAvatar's GaussianRenderer builds them per render from cam_param (avatar/common/nets/module.py:604-613,
// transforms.py:38-70); the host mirror renderer._device_camera reads the camera back to do the same on the CPU.  This
// kernel writes the 37-float block view | full projection | campos | tan(fov_x/2) | tan(fov_y/2) instead, so nothing of
// the camera ever reaches the host.  Compiled with --fmad=false: every product and sum below is rounded on its own, as
// the torch expressions it restates round them.
#include "common.cuh"

namespace b2r {

// One thread: 37 outputs from 14 inputs.  Expression by expression (matrices stored [4c+r], as B2RScene reads them):
//   fov    = 2 * atan(W / (2 f))   torch's CUDA kernels: `W / x` on a tensor is x.reciprocal() * W, then atanf, x 2
//   tanfov = tan(fov / 2)          torch.tan on the device: tanf
//   proj   = transforms.py:43-64   math.tan(float(fov) / 2) and the entries in fp64, each rounded to fp32 once
//   full   = view^T-stored x proj^T-stored, every entry summed left to right over k = 0..3 in rounded fp32 products
//   campos = -R^T t                fp64, rounded once (the rigid inverse, not an LU solve)
__global__ void camera_setup_kernel(const float* __restrict__ R, const float* __restrict__ t,
                                    const float* __restrict__ focal, const int W, const int H, float* __restrict__ out) {
  float r[9], tv[3];
#pragma unroll
  for (int k = 0; k < 9; k++) r[k] = R[k];
#pragma unroll
  for (int k = 0; k < 3; k++) tv[k] = t[k];
  const float fov_x = __fmul_rn(2.f, atanf(__fmul_rn(__frcp_rn(__fmul_rn(2.f, focal[0])), (float)W)));
  const float fov_y = __fmul_rn(2.f, atanf(__fmul_rn(__frcp_rn(__fmul_rn(2.f, focal[1])), (float)H)));

  // view (transposed: element (r, c) of [R t; 0 0 0 1] at [4c + r])
  float v[16];
#pragma unroll
  for (int row = 0; row < 3; row++) {
#pragma unroll
    for (int c = 0; c < 3; c++) v[4 * c + row] = r[3 * row + c];
    v[12 + row] = tv[row];
  }
  v[3] = v[7] = v[11] = 0.f;
  v[15] = 1.f;

  // projection, stored the same way (module.py permutes it too)
  const double znear = 0.01, zfar = 100.0;
  const double top = tan((double)fov_y / 2) * znear, bottom = -top;
  const double right = tan((double)fov_x / 2) * znear, left = -right;
  float p[16];
#pragma unroll
  for (int k = 0; k < 16; k++) p[k] = 0.f;
  p[0] = (float)(2.0 * znear / (right - left));   // (0,0)
  p[5] = (float)(2.0 * znear / (top - bottom));   // (1,1)
  p[8] = (float)((right + left) / (right - left)); // (0,2)
  p[9] = (float)((top + bottom) / (top - bottom)); // (1,2)
  p[11] = 1.f;                                     // (3,2): z_sign
  p[10] = (float)(1.0 * zfar / (zfar - znear));    // (2,2)
  p[14] = (float)(-(zfar * znear) / (zfar - znear)); // (2,3)

  // full = torch.mm(view^T, proj^T): row i, column j of the stored matrices is memory [4i + j]
#pragma unroll
  for (int i = 0; i < 4; i++) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
      float s = __fmul_rn(v[4 * i], p[j]);
#pragma unroll
      for (int k = 1; k < 4; k++) s = __fadd_rn(s, __fmul_rn(v[4 * i + k], p[4 * k + j]));
      out[16 + 4 * i + j] = s;
    }
  }
#pragma unroll
  for (int k = 0; k < 16; k++) out[k] = v[k];
#pragma unroll
  for (int c = 0; c < 3; c++)
    out[32 + c] = (float)(-((double)r[c] * (double)tv[0] + (double)r[3 + c] * (double)tv[1] +
                            (double)r[6 + c] * (double)tv[2]));
  out[35] = tanf(__fmul_rn(fov_x, 0.5f));
  out[36] = tanf(__fmul_rn(fov_y, 0.5f));
}

int launch_camera_setup(const float* R, const float* t, const float* focal, int W, int H, float* out, cudaStream_t st) {
  ProfScope ps(K_MISC, st);
  launch_k(camera_setup_kernel, 1, 1, 0, st, true, R, t, focal, W, H, out);
  return check_launch();
}

}  // namespace b2r
