// mesh_raster.cu -- ExAvatar's face render (avatar/main/model.py:170-175 -> MeshRenderer, avatar/common/nets/layer.py:
// 23-68): pytorch3d's MeshRasterizer (blur_radius 0, faces_per_pixel 1, perspective-correct barycentrics, no culling,
// no clipping) followed by TexturesUV's bilinear sample, restated from pytorch3d's implementation (the semantics are
// spelled out in include/b200raster.h B2RMeshRender and mesh_render.py).
//
//   mr_face_kernel     one thread per face: world -> camera -> NDC of the three corners, the skip rules, a conservative
//                      pixel box, then the box walked.  Boxes of more than MR_SMALL pixels are walked by the whole warp,
//                      one face after the other (a close-up face covers thousands of pixels, most C4 faces less than
//                      one).  Every covered pixel takes atomicMin of the key (float_bits(pz) << 32) | face: pz >= 0, so
//                      the bits order like the floats, and the minimum is the nearest face, ties to the lowest index,
//                      whatever order the faces arrive in.
//   mr_resolve_kernel  one thread per pixel: decode the key, recompute the barycentrics with the same device function,
//                      interpolate uv, sample the texture (ATen's bilinear expression order), write the image and the
//                      face id, and reset the key to ~0 -- the buffer is clean for the next call (no memset node).
//   mr_shade_kernel    (b2r_mesh_shade_forward, the animation scripts' untextured mesh panel) one thread per pixel:
//                      decode and reset the key like the resolve, interpolate position, vertex normal and the
//                      all-ones texture, Phong-shade with pytorch3d's default point light, composite over `bkg`.
//   mr_face_bwd_kernel one work item per face walks its box in raster order and sums, over the pixels whose face id is
//                      that face, dL/d(x_ndc, y_ndc, z) of its three corners (the big boxes again by the whole warp, each
//                      lane a fixed stride, combined by a fixed shuffle tree).  Every face's 9 values are written.
//   mr_vertex_bwd_kernel one thread per vertex sums its corners over the vertex -> face CSR (ascending faces, the
//                      table of VertexNormals) and applies NDC -> camera -> world once.
// No float atomics anywhere: two runs give identical bits.  This unit is compiled with --fmad=false (build_ext.py): the
// coverage test and pz are, operation for operation, the float32 restatement's (mesh_render.face_render_reference), so
// the per-pixel face is identical to it, not merely equal up to ulp ties.
#include <float.h>

#include "common.cuh"

namespace b2r {

constexpr int MR_THREADS = 128;
constexpr int MR_SMALL = 32;   // boxes of more pixels are walked by the whole warp
constexpr float MR_EPS = 1e-8f;  // pytorch3d's kEpsilon

// per-face record, written by the forward and read by the resolve and the backward
struct MRFace {
  float x[3], y[3], z[3];  // NDC x, y and view depth of the corners
  int c0, r0, c1, r1;      // inclusive pixel box; c0 > c1 when the face is skipped
  float pad[3];
};
static_assert(sizeof(MRFace) == 64, "MRFace must be 64 bytes");

struct MRLayout {
  size_t faces, grad, total;
};
inline MRLayout mr_layout(int F) {
  const size_t n = F > 0 ? (size_t)F : 1;
  MRLayout L;
  size_t o = 0;
  L.faces = o; o += align_up(n * sizeof(MRFace));
  L.grad = o; o += align_up(n * 9 * sizeof(float));
  L.total = o;
  return L;
}

struct MRCam {
  float R[9], t[3], fx, fy, cx, cy;
};

__device__ __forceinline__ MRCam mr_load_cam(const B2RMeshRender& m) {
  MRCam c;
#pragma unroll
  for (int i = 0; i < 9; i++) c.R[i] = m.cam_R[i];
#pragma unroll
  for (int i = 0; i < 3; i++) c.t[i] = m.cam_t[i];
  c.fx = m.focal[0]; c.fy = m.focal[1];
  c.cx = m.princpt[0]; c.cy = m.princpt[1];
  return c;
}

// p_c = R p + t, each row left to right
__device__ __forceinline__ void mr_to_cam(const MRCam& c, float X, float Y, float Z, float& xc, float& yc, float& zc) {
  xc = c.R[0] * X + c.R[1] * Y + c.R[2] * Z + c.t[0];
  yc = c.R[3] * X + c.R[4] * Y + c.R[5] * Z + c.t[1];
  zc = c.R[6] * X + c.R[7] * Y + c.R[8] * Z + c.t[2];
}

// pixel centre of column / row index i (already mirrored: W-1-c, H-1-r) -- pytorch3d's PixToNonSquareNdc(i, S1, S2)
__device__ __forceinline__ float mr_pix_ndc(int i, int S1, int S2) {
  float range = 2.0f;
  if (S1 > S2) range = ((float)S1 * range) / (float)S2;
  const float offset = range / 2.0f;
  return -offset + (range * (float)i + offset) / (float)S1;
}

__device__ __forceinline__ float mr_edge(float px, float py, float ax, float ay, float bx, float by) {
  return (px - ax) * (by - ay) - (py - ay) * (bx - ax);
}

struct MRBary {
  float w[3];    // screen-space barycentrics
  float b[3];    // perspective-corrected
  float area;    // E(v2, v0, v1) + eps
  float denom;   // max(sum of the corrected numerators, eps)
  float pz;
};

// the barycentrics of pytorch3d's BarycentricCoordinatesForward + BarycentricPerspectiveCorrectionForward and its pz
__device__ __forceinline__ void mr_bary(const MRFace& f, float px, float py, MRBary& o) {
  o.area = mr_edge(f.x[2], f.y[2], f.x[0], f.y[0], f.x[1], f.y[1]) + MR_EPS;
  o.w[0] = mr_edge(px, py, f.x[1], f.y[1], f.x[2], f.y[2]) / o.area;
  o.w[1] = mr_edge(px, py, f.x[2], f.y[2], f.x[0], f.y[0]) / o.area;
  o.w[2] = mr_edge(px, py, f.x[0], f.y[0], f.x[1], f.y[1]) / o.area;
  const float t0 = o.w[0] * f.z[1] * f.z[2];
  const float t1 = f.z[0] * o.w[1] * f.z[2];
  const float t2 = f.z[0] * f.z[1] * o.w[2];
  o.denom = fmaxf(t0 + t1 + t2, MR_EPS);
  o.b[0] = t0 / o.denom;
  o.b[1] = t1 / o.denom;
  o.b[2] = t2 / o.denom;
  o.pz = o.b[0] * f.z[0] + o.b[1] * f.z[1] + o.b[2] * f.z[2];
}

// the full coverage test of one pixel centre: pytorch3d's xy box, pz >= 0, all three corrected barycentrics > 0
__device__ __forceinline__ bool mr_covers(const MRFace& f, float px, float py, MRBary& o) {
  const float xmin = fminf(f.x[0], fminf(f.x[1], f.x[2])), xmax = fmaxf(f.x[0], fmaxf(f.x[1], f.x[2]));
  const float ymin = fminf(f.y[0], fminf(f.y[1], f.y[2])), ymax = fmaxf(f.y[0], fmaxf(f.y[1], f.y[2]));
  if (px > xmax || px < xmin || py > ymax || py < ymin) return false;
  mr_bary(f, px, py, o);
  if (o.pz < 0.f) return false;
  return o.b[0] > 0.f && o.b[1] > 0.f && o.b[2] > 0.f;
}

// inclusive pixel range [lo, hi] along one axis of n pixels whose centres u = i + 0.5 can lie in NDC [a, b]
// (u = n / 2 - ndc * s); one pixel of margin absorbs the rounding, the exact test decides
__device__ __forceinline__ void mr_axis_range(float a, float b, int n, float s, int& lo, int& hi) {
  const float ulo = 0.5f * (float)n - b * s - 0.5f, uhi = 0.5f * (float)n - a * s - 0.5f;
  lo = (int)fminf(fmaxf(floorf(ulo) - 1.f, 0.f), (float)n);
  hi = (int)fmaxf(fminf(ceilf(uhi) + 1.f, (float)(n - 1)), -1.f);
}

__device__ __forceinline__ uint64_t mr_key(float pz, int f) {
  const float z = pz == 0.f ? 0.f : pz;  // -0 orders with +0
  return ((uint64_t)__float_as_uint(z) << 32) | (uint32_t)f;
}

__device__ __forceinline__ void mr_raster_pixel(const MRFace& fc, int f, int W, int H, int c, int r,
                                                unsigned long long* __restrict__ keys) {
  MRBary o;
  if (mr_covers(fc, mr_pix_ndc(W - 1 - c, W, H), mr_pix_ndc(H - 1 - r, H, W), o))
    atomicMin(keys + (size_t)r * W + c, (unsigned long long)mr_key(o.pz, f));
}

__global__ void __launch_bounds__(MR_THREADS) mr_face_kernel(const B2RMeshRender m, MRFace* __restrict__ recs) {
  const int f = blockIdx.x * MR_THREADS + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const bool valid = f < m.F;
  MRFace fc;
  int area = 0;
  if (valid) {
    const MRCam cam = mr_load_cam(m);
    const float W2 = 0.5f * (float)m.width, H2 = 0.5f * (float)m.height;
    const float s = 0.5f * (float)min(m.width, m.height);
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const int v = m.faces[3 * f + k];
      if (v < 0 || v >= m.V) { ok = false; fc.x[k] = fc.y[k] = fc.z[k] = 0.f; continue; }
      float xc, yc, zc;
      mr_to_cam(cam, m.mesh[3 * v], m.mesh[3 * v + 1], m.mesh[3 * v + 2], xc, yc, zc);
      const float u = cam.fx * xc / zc + cam.cx, w = cam.fy * yc / zc + cam.cy;
      fc.x[k] = (W2 - u) / s;
      fc.y[k] = (H2 - w) / s;
      fc.z[k] = zc;
      ok = ok && isfinite(fc.x[k]) && isfinite(fc.y[k]) && isfinite(zc);
    }
    const float zmax = fmaxf(fc.z[0], fmaxf(fc.z[1], fc.z[2]));
    const float e = mr_edge(fc.x[0], fc.y[0], fc.x[1], fc.y[1], fc.x[2], fc.y[2]);
    fc.c0 = fc.r0 = 1;
    fc.c1 = fc.r1 = 0;  // empty box = skipped
    if (ok && !(zmax < 0.f) && !(e <= MR_EPS && e >= -MR_EPS)) {
      mr_axis_range(fminf(fc.x[0], fminf(fc.x[1], fc.x[2])), fmaxf(fc.x[0], fmaxf(fc.x[1], fc.x[2])), m.width, s,
                    fc.c0, fc.c1);
      mr_axis_range(fminf(fc.y[0], fminf(fc.y[1], fc.y[2])), fmaxf(fc.y[0], fmaxf(fc.y[1], fc.y[2])), m.height, s,
                    fc.r0, fc.r1);
      if (fc.c0 > fc.c1 || fc.r0 > fc.r1) { fc.c0 = fc.r0 = 1; fc.c1 = fc.r1 = 0; }
    }
    fc.pad[0] = fc.pad[1] = fc.pad[2] = 0.f;
    recs[f] = fc;
    area = (fc.c1 - fc.c0 + 1) * (fc.r1 - fc.r0 + 1);  // 0 when skipped
  }
  unsigned long long* keys = (unsigned long long*)m.keys;
  if (area > 0 && area <= MR_SMALL) {
    for (int r = fc.r0; r <= fc.r1; r++)
      for (int c = fc.c0; c <= fc.c1; c++) mr_raster_pixel(fc, f, m.width, m.height, c, r, keys);
  }
  // big boxes: the whole warp walks them one face at a time
  unsigned big = __ballot_sync(0xffffffffu, area > MR_SMALL);
  if (!big) return;
  __syncwarp();  // the records of this warp's faces are visible to every lane
  while (big) {
    const int l = __ffs(big) - 1;
    big &= big - 1;
    const int g = (f - lane) + l;
    const MRFace bf = recs[g];
    const int bw = bf.c1 - bf.c0 + 1;
    const int n = bw * (bf.r1 - bf.r0 + 1);
    for (int i = lane; i < n; i += 32) mr_raster_pixel(bf, g, m.width, m.height, bf.c0 + i % bw, bf.r0 + i / bw, keys);
  }
}

// grid_sample(bilinear, align_corners=True, padding_mode="border") source index along one axis of n texels, with the
// derivative mask of ATen's clip_coordinates_set_grad (the border itself counts as outside)
__device__ __forceinline__ float mr_src(float g, int n, float& mult) {
  float i = ((g + 1.f) / 2.f) * (float)(n - 1);
  mult = ((float)(n - 1) / 2.f);
  if (i <= 0.f) { mult = 0.f; i = 0.f; }
  else if (i >= (float)(n - 1)) { mult = 0.f; i = (float)(n - 1); }
  return i;
}

// texture value of channel ch at (row iy, column ix) of the vertically FLIPPED map, 0 outside (ATen's within_bounds)
__device__ __forceinline__ float mr_tex(const B2RMeshRender& m, int ch, int iy, int ix) {
  if (ix < 0 || ix >= m.tex_width || iy < 0 || iy >= m.tex_height) return 0.f;
  return m.texture[((size_t)ch * m.tex_height + (m.tex_height - 1 - iy)) * m.tex_width + ix];
}

// uv of the three corners of face f after MeshRenderer's flip (a, 1 - b)
__device__ __forceinline__ void mr_face_uv(const B2RMeshRender& m, int f, float ux[3], float uy[3]) {
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const int t = m.face_uv[3 * f + k];
    ux[k] = m.vertex_uv[2 * t];
    uy[k] = 1.f - m.vertex_uv[2 * t + 1];
  }
}

__global__ void __launch_bounds__(MR_THREADS) mr_resolve_kernel(const B2RMeshRender m, const MRFace* __restrict__ recs,
                                                                float* __restrict__ image, int32_t* __restrict__ p2f) {
  const int p = blockIdx.x * MR_THREADS + threadIdx.x;
  const int N = m.width * m.height;
  if (p >= N) return;
  const uint64_t key = m.keys[p];
  m.keys[p] = ~0ull;
  if (key == ~0ull) {
    p2f[p] = -1;
    for (int ch = 0; ch < m.C; ch++) image[(size_t)ch * N + p] = -1.f;
    return;
  }
  const int f = (int)(uint32_t)key;
  p2f[p] = f;
  const int c = p % m.width, r = p / m.width;
  float u, v;
  {
    const MRFace fc = recs[f];
    MRBary o;
    mr_bary(fc, mr_pix_ndc(m.width - 1 - c, m.width, m.height), mr_pix_ndc(m.height - 1 - r, m.height, m.width), o);
    float ux[3], uy[3];
    mr_face_uv(m, f, ux, uy);
    u = o.b[0] * ux[0] + o.b[1] * ux[1] + o.b[2] * ux[2];
    v = o.b[0] * uy[0] + o.b[1] * uy[1] + o.b[2] * uy[2];
  }
  float mx, my;
  const float ix = mr_src(u * 2.f - 1.f, m.tex_width, mx), iy = mr_src(v * 2.f - 1.f, m.tex_height, my);
  const int ix_nw = (int)floorf(ix), iy_nw = (int)floorf(iy);
  const float ix_se = (float)(ix_nw + 1), iy_se = (float)(iy_nw + 1);
  const float nw = (ix_se - ix) * (iy_se - iy);
  const float ne = (ix - (float)ix_nw) * (iy_se - iy);
  const float sw = (ix_se - ix) * (iy - (float)iy_nw);
  const float se = (ix - (float)ix_nw) * (iy - (float)iy_nw);
  for (int ch = 0; ch < m.C; ch++) {
    float acc = 0.f;
    acc += mr_tex(m, ch, iy_nw, ix_nw) * nw;
    acc += mr_tex(m, ch, iy_nw, ix_nw + 1) * ne;
    acc += mr_tex(m, ch, iy_nw + 1, ix_nw) * sw;
    acc += mr_tex(m, ch, iy_nw + 1, ix_nw + 1) * se;
    image[(size_t)ch * N + p] = acc;
  }
}

// dL/d(x, y, z) of the three corners from one covered pixel: grid_sample's derivative -> uv -> corrected barycentrics
// -> screen barycentrics and z -> the edge functions' corners
__device__ __forceinline__ void mr_pixel_grad(const B2RMeshRender& m, const MRFace& fc, const float ux[3],
                                              const float uy[3], const float* __restrict__ dimg, int p, int c, int r,
                                              float g[9]) {
  const int N = m.width * m.height;
  const float px = mr_pix_ndc(m.width - 1 - c, m.width, m.height), py = mr_pix_ndc(m.height - 1 - r, m.height, m.width);
  MRBary o;
  mr_bary(fc, px, py, o);
  const float u = o.b[0] * ux[0] + o.b[1] * ux[1] + o.b[2] * ux[2];
  const float v = o.b[0] * uy[0] + o.b[1] * uy[1] + o.b[2] * uy[2];
  float mx, my;
  const float ix = mr_src(u * 2.f - 1.f, m.tex_width, mx), iy = mr_src(v * 2.f - 1.f, m.tex_height, my);
  const int ix_nw = (int)floorf(ix), iy_nw = (int)floorf(iy);
  const float ix_se = (float)(ix_nw + 1), iy_se = (float)(iy_nw + 1);
  float gix = 0.f, giy = 0.f;
  for (int ch = 0; ch < m.C; ch++) {
    const float go = dimg[(size_t)ch * N + p];
    const float vnw = mr_tex(m, ch, iy_nw, ix_nw), vne = mr_tex(m, ch, iy_nw, ix_nw + 1);
    const float vsw = mr_tex(m, ch, iy_nw + 1, ix_nw), vse = mr_tex(m, ch, iy_nw + 1, ix_nw + 1);
    gix += (-vnw * (iy_se - iy) + vne * (iy_se - iy) - vsw * (iy - (float)iy_nw) + vse * (iy - (float)iy_nw)) * go;
    giy += (-vnw * (ix_se - ix) - vne * (ix - (float)ix_nw) + vsw * (ix_se - ix) + vse * (ix - (float)ix_nw)) * go;
  }
  const float du = 2.f * mx * gix, dv = 2.f * my * giy;  // grid = 2 uv - 1
  float gb[3];
#pragma unroll
  for (int k = 0; k < 3; k++) gb[k] = du * ux[k] + dv * uy[k];
  // b_k = t_k / S  (the max(S, eps) inactive)
  const float gdot = gb[0] * o.b[0] + gb[1] * o.b[1] + gb[2] * o.b[2];
  float gt[3];
#pragma unroll
  for (int k = 0; k < 3; k++) gt[k] = (gb[k] - gdot) / o.denom;
  const float z0 = fc.z[0], z1 = fc.z[1], z2 = fc.z[2];
  // t0 = w0 z1 z2, t1 = z0 w1 z2, t2 = z0 z1 w2
  const float gw0 = gt[0] * z1 * z2, gw1 = gt[1] * z0 * z2, gw2 = gt[2] * z0 * z1;
  g[2] += gt[1] * o.w[1] * z2 + gt[2] * z1 * o.w[2];
  g[5] += gt[0] * o.w[0] * z2 + gt[2] * z0 * o.w[2];
  g[8] += gt[0] * o.w[0] * z1 + gt[1] * z0 * o.w[1];
  // w_k = E_k / A
  const float gE0 = gw0 / o.area, gE1 = gw1 / o.area, gE2 = gw2 / o.area;
  const float gA = -(gw0 * o.w[0] + gw1 * o.w[1] + gw2 * o.w[2]) / o.area;
  const float x0 = fc.x[0], y0 = fc.y[0], x1 = fc.x[1], y1 = fc.y[1], x2 = fc.x[2], y2 = fc.y[2];
  // E(p, a, b): d/da = (p.y - b.y, b.x - p.x), d/db = (a.y - p.y, p.x - a.x)
  // E0 = E(p, v1, v2), E1 = E(p, v2, v0), E2 = E(p, v0, v1), A = E(v2, v0, v1) (v2 in the role of p: (b.y - a.y, a.x - b.x))
  g[0] += gE1 * (y2 - py) + gE2 * (py - y1) + gA * (y2 - y1);
  g[1] += gE1 * (px - x2) + gE2 * (x1 - px) + gA * (x1 - x2);
  g[3] += gE0 * (py - y2) + gE2 * (y0 - py) + gA * (y0 - y2);
  g[4] += gE0 * (x2 - px) + gE2 * (px - x0) + gA * (x2 - x0);
  g[6] += gE0 * (y1 - py) + gE1 * (py - y0) + gA * (y1 - y0);
  g[7] += gE0 * (px - x1) + gE1 * (x0 - px) + gA * (x0 - x1);
}

__global__ void __launch_bounds__(MR_THREADS) mr_face_bwd_kernel(const B2RMeshRender m, const MRFace* __restrict__ recs,
                                                                 const int32_t* __restrict__ p2f,
                                                                 const float* __restrict__ dimg,
                                                                 float* __restrict__ gface) {
  const int f = blockIdx.x * MR_THREADS + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const bool valid = f < m.F;
  float g[9];
#pragma unroll
  for (int i = 0; i < 9; i++) g[i] = 0.f;
  int area = 0;
  MRFace fc;
  if (valid) {
    fc = recs[f];
    area = max(fc.c1 - fc.c0 + 1, 0) * max(fc.r1 - fc.r0 + 1, 0);
  }
  if (area > 0 && area <= MR_SMALL) {
    float ux[3], uy[3];
    mr_face_uv(m, f, ux, uy);
    for (int r = fc.r0; r <= fc.r1; r++)
      for (int c = fc.c0; c <= fc.c1; c++) {
        const int p = r * m.width + c;
        if (p2f[p] == f) mr_pixel_grad(m, fc, ux, uy, dimg, p, c, r, g);
      }
  }
  unsigned big = __ballot_sync(0xffffffffu, area > MR_SMALL);
  while (big) {
    const int l = __ffs(big) - 1;
    big &= big - 1;
    const int bf_id = (f - lane) + l;
    const MRFace bf = recs[bf_id];
    float ux[3], uy[3];
    mr_face_uv(m, bf_id, ux, uy);
    const int bw = bf.c1 - bf.c0 + 1;
    const int n = bw * (bf.r1 - bf.r0 + 1);
    float h[9];
#pragma unroll
    for (int i = 0; i < 9; i++) h[i] = 0.f;
    for (int i = lane; i < n; i += 32) {  // lane l takes pixels l, l + 32, ... of the box in raster order
      const int c = bf.c0 + i % bw, r = bf.r0 + i / bw;
      const int p = r * m.width + c;
      if (p2f[p] == bf_id) mr_pixel_grad(m, bf, ux, uy, dimg, p, c, r, h);
    }
#pragma unroll
    for (int i = 0; i < 9; i++) {
      for (int d = 16; d > 0; d >>= 1) h[i] += __shfl_xor_sync(0xffffffffu, h[i], d);
      if (lane == l) g[i] = h[i];
    }
  }
  if (valid) {
#pragma unroll
    for (int i = 0; i < 9; i++) gface[(size_t)9 * f + i] = g[i];
  }
}

__global__ void __launch_bounds__(MR_THREADS) mr_vertex_bwd_kernel(const B2RMeshRender m,
                                                                   const float* __restrict__ gface,
                                                                   float* __restrict__ dmesh) {
  const int v = blockIdx.x * MR_THREADS + threadIdx.x;
  if (v >= m.V) return;
  float gx = 0.f, gy = 0.f, gz = 0.f;
  const int e0 = m.vf_offsets[v], e1 = m.vf_offsets[v + 1];
  for (int e = e0; e < e1; e++) {
    const int f = m.vf_entries[e];
    if (e > e0 && m.vf_entries[e - 1] == f) continue;  // a face that repeats v: all its corners at v were taken once
#pragma unroll
    for (int k = 0; k < 3; k++) {
      if (m.faces[3 * f + k] != v) continue;
      gx += gface[(size_t)9 * f + 3 * k];
      gy += gface[(size_t)9 * f + 3 * k + 1];
      gz += gface[(size_t)9 * f + 3 * k + 2];
    }
  }
  float out[3] = {0.f, 0.f, 0.f};
  if (gx != 0.f || gy != 0.f || gz != 0.f) {
    const MRCam cam = mr_load_cam(m);
    const float s = 0.5f * (float)min(m.width, m.height);
    float xc, yc, zc;
    mr_to_cam(cam, m.mesh[3 * v], m.mesh[3 * v + 1], m.mesh[3 * v + 2], xc, yc, zc);
    // x_ndc = (W/2 - fx xc / zc - cx) / s, y likewise, z = zc
    const float ax = gx * cam.fx / (s * zc), ay = gy * cam.fy / (s * zc);
    const float gxc = -ax, gyc = -ay, gzc = gz + (ax * xc + ay * yc) / zc;
    // world: R^T g_c
    out[0] = cam.R[0] * gxc + cam.R[3] * gyc + cam.R[6] * gzc;
    out[1] = cam.R[1] * gxc + cam.R[4] * gyc + cam.R[7] * gzc;
    out[2] = cam.R[2] * gxc + cam.R[5] * gyc + cam.R[8] * gzc;
  }
  dmesh[3 * v] = out[0];
  dmesh[3 * v + 1] = out[1];
  dmesh[3 * v + 2] = out[2];
}

// ---------------------------------------------------------------------------------------------------------------------
// Shaded render (b2r_mesh_shade_forward): the mesh panel of ExAvatar's animation scripts (utils/vis.py render_mesh:
// pytorch3d's SoftPhongShader with the default PointLights, white TexturesVertex, no specular, then the host composite).
// mr_face_kernel's coverage, then one thread per pixel.  Shading runs in the op's camera coordinates (p_c = R p + t,
// n_c = R n) with the light at (0, -1, 0): pytorch3d's light (0, 1, 0) seen from the xy-negated frame it renders in.
// Negating x and y is exact, so every dot product is the one pytorch3d forms.
// ---------------------------------------------------------------------------------------------------------------------

// n_c = R n, each row left to right
__device__ __forceinline__ void mr_rotate(const MRCam& c, float X, float Y, float Z, float& xc, float& yc, float& zc) {
  xc = c.R[0] * X + c.R[1] * Y + c.R[2] * Z;
  yc = c.R[3] * X + c.R[4] * Y + c.R[5] * Z;
  zc = c.R[6] * X + c.R[7] * Y + c.R[8] * Z;
}

__global__ void __launch_bounds__(MR_THREADS) mr_shade_kernel(const B2RMeshRender m, const MRFace* __restrict__ recs,
                                                              const float* __restrict__ normals,
                                                              const float* __restrict__ bkg, const float blend,
                                                              const float blend_c, float* __restrict__ out) {
  const int p = blockIdx.x * MR_THREADS + threadIdx.x;
  const int N = m.width * m.height;
  if (p >= N) return;
  const uint64_t key = m.keys[p];
  m.keys[p] = ~0ull;
  float c = 1.f;       // softmax_rgb_blend's white background where no face covers the pixel
  float is_bkg = 1.f;  // vis.py: zbuf <= 0, and zbuf is -1 where no face covers the pixel
  if (key != ~0ull) {
    const int f = (int)(uint32_t)key;
    if (__uint_as_float((uint32_t)(key >> 32)) > 0.f) is_bkg = 0.f;
    const int col = p % m.width, r = p / m.width;
    MRBary o;
    mr_bary(recs[f], mr_pix_ndc(m.width - 1 - col, m.width, m.height), mr_pix_ndc(m.height - 1 - r, m.height, m.width),
            o);
    const MRCam cam = mr_load_cam(m);
    // interpolate_face_attributes: position, normal and the all-ones texture, corners in order 0, 1, 2
    float P[3], Nv[3], texel = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const int v = m.faces[3 * f + k];
      float q[3], n[3];
      mr_to_cam(cam, m.mesh[3 * v], m.mesh[3 * v + 1], m.mesh[3 * v + 2], q[0], q[1], q[2]);
      mr_rotate(cam, normals[3 * v], normals[3 * v + 1], normals[3 * v + 2], n[0], n[1], n[2]);
#pragma unroll
      for (int i = 0; i < 3; i++) {
        P[i] = k ? P[i] + o.b[k] * q[i] : o.b[k] * q[i];
        Nv[i] = k ? Nv[i] + o.b[k] * n[i] : o.b[k] * n[i];
      }
      texel = k ? texel + o.b[k] : o.b[k];
    }
    // _apply_lighting: F.normalize(normal), F.normalize(light - point), relu of their dot product
    const float d[3] = {0.f - P[0], -1.f - P[1], 0.f - P[2]};
    const float nl = fmaxf(sqrtf(Nv[0] * Nv[0] + Nv[1] * Nv[1] + Nv[2] * Nv[2]), 1e-6f);
    const float dl = fmaxf(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), 1e-6f);
    float cosa = (Nv[0] / nl) * (d[0] / dl) + (Nv[1] / nl) * (d[1] / dl) + (Nv[2] / nl) * (d[2] / dl);
    if (cosa < 0.f) cosa = 0.f;  // relu; a NaN stays NaN as in torch
    // (ambient 1 * 0.5 + diffuse 1 * 0.3 * angle) * texel; the specular term is 0
    c = (0.5f + 0.3f * cosa) * texel;
  }
  // vis.py:107-108 in float32, numpy's order: fg = c * blend + bkg / 255 * (1 - blend); fg (1 - is_bkg) 255 + bkg is_bkg
  const float* bg = bkg + (size_t)3 * p;
  float* o3 = out + (size_t)3 * p;
#pragma unroll
  for (int ch = 0; ch < 3; ch++) {
    const float b = bg[ch];
    const float fg = c * blend + (b / 255.f) * blend_c;
    o3[ch] = (fg * (1.f - is_bkg)) * 255.f + b * is_bkg;
  }
}

size_t mesh_render_scratch_bytes(int F) { return mr_layout(F).total; }

int launch_mesh_render_forward(const B2RMeshRender& m, float* image, int32_t* pix_to_face, void* scratch,
                               cudaStream_t st) {
  const MRLayout L = mr_layout(m.F);
  MRFace* recs = (MRFace*)((char*)scratch + L.faces);
  if (m.F > 0) {
    ProfScope p(K_MISC, st);
    launch_k(mr_face_kernel, (m.F + MR_THREADS - 1) / MR_THREADS, MR_THREADS, 0, st, true, m, recs);
  }
  {
    const int N = m.width * m.height;
    ProfScope p(K_MISC, st);
    launch_k(mr_resolve_kernel, (N + MR_THREADS - 1) / MR_THREADS, MR_THREADS, 0, st, true, m, (const MRFace*)recs,
             image, pix_to_face);
  }
  return check_launch();
}

int launch_mesh_shade_forward(const B2RMeshRender& m, const float* normals, const float* bkg, float blend,
                              float blend_complement, float* out, void* scratch, cudaStream_t st) {
  const MRLayout L = mr_layout(m.F);
  MRFace* recs = (MRFace*)((char*)scratch + L.faces);
  if (m.F > 0) {
    ProfScope p(K_MISC, st);
    launch_k(mr_face_kernel, (m.F + MR_THREADS - 1) / MR_THREADS, MR_THREADS, 0, st, true, m, recs);
  }
  {
    const int N = m.width * m.height;
    ProfScope p(K_MISC, st);
    launch_k(mr_shade_kernel, (N + MR_THREADS - 1) / MR_THREADS, MR_THREADS, 0, st, true, m, (const MRFace*)recs,
             normals, bkg, blend, blend_complement, out);
  }
  return check_launch();
}

int launch_mesh_render_backward(const B2RMeshRender& m, const int32_t* pix_to_face, const float* dimage, float* dmesh,
                                void* scratch, cudaStream_t st) {
  const MRLayout L = mr_layout(m.F);
  const MRFace* recs = (const MRFace*)((const char*)scratch + L.faces);
  float* gface = (float*)((char*)scratch + L.grad);
  if (m.F > 0) {
    ProfScope p(K_MISC, st);
    launch_k(mr_face_bwd_kernel, (m.F + MR_THREADS - 1) / MR_THREADS, MR_THREADS, 0, st, true, m, recs, pix_to_face,
             dimage, gface);
  }
  if (m.V > 0) {
    ProfScope p(K_MISC, st);
    launch_k(mr_vertex_bwd_kernel, (m.V + MR_THREADS - 1) / MR_THREADS, MR_THREADS, 0, st, true, m,
             (const float*)gface, dmesh);
  }
  return check_launch();
}

}  // namespace b2r
