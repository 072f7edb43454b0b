// geometry.cu -- the two per-frame mesh queries in front of ExAvatar's human posing (avatar/common/nets/module.py):
//   nearest rows   knn_points(mean_3d, mesh_neutral_pose_wo_upsample, K=1) + the hand / face self-map (541-546)
//   vertex normals Meshes(xyz, face_upsampled).verts_normals_packed() + the cavity flip (501-504)
//
// Nearest rows: the neutral mesh changes every step (shape_param and joint_offset are learnt), so every call builds a
// uniform grid over the targets on the device before it answers the queries.
//   nn_build_kernel  ONE CTA: bounding box (min / max, order-free), grid size from V and the box aspect, counting sort
//                    of the targets into cells (histogram with atomics, block scan, scatter).  The order of the targets
//                    inside a cell is whatever the atomics give; the (distance, index) tie-break below makes the result
//                    independent of it.  Every buffer is sized from V alone, so the host never reads device data.
//   nn_query_kernel  one thread per query: visit cell shells k = 0, 1, 2, ... around the query's (clamped) cell and stop
//                    only when the distance to every unvisited cell, shrunk by a rounding margin, is STRICTLY greater
//                    than the best distance found -- an equal-distance, lower-index target farther out still wins.
// d(i,j) = dx*dx + dy*dy + dz*dz left to right in fp32: this unit is compiled with --fmad=false (build_ext.py), so the
// distances are the bits of the torch restatement (geometry.nearest_rows_reference) and the argmin is exact.
//
// Vertex normals: one gather kernel over a vertex -> face CSR built once by the caller (include/b200raster.h); the face
// cross products are summed in CSR order, no float atomics, so two runs are bit-identical.
#include <float.h>
#include <limits.h>

#include "common.cuh"

namespace b2r {

constexpr int NN_BUILD_THREADS = 1024;
constexpr int NN_QUERY_THREADS = 128;
constexpr int NN_MAX_DIM = 1024;  // cells per axis

// grid parameters written by the build kernel, read by the query kernel
struct NNGrid {
  float ox, oy, oz;  // grid origin (box minimum)
  float s, inv_s;    // cell edge and its reciprocal
  float span;        // largest |coordinate| the grid reaches: scales the rounding margin of the stop test
  int dx, dy, dz;    // cells per axis, dx * dy * dz <= nn_max_cells(V)
};

__host__ __device__ inline int nn_max_cells(int V) { return 2 * V + 64; }

struct NNLayout {
  size_t grid, offsets, cursor, sorted, total;
};
inline NNLayout nn_layout(int V) {
  const int v = V > 0 ? V : 1;
  const size_t C = (size_t)nn_max_cells(v);
  NNLayout L;
  size_t o = 0;
  L.grid = o; o += align_up(sizeof(NNGrid));
  L.offsets = o; o += align_up((C + 1) * sizeof(int));
  L.cursor = o; o += align_up(C * sizeof(int));
  L.sorted = o; o += align_up((size_t)v * sizeof(float4));
  L.total = o;
  return L;
}

// cell coordinate along one axis, clamped to [0, n); NaN lands in cell 0
__device__ __forceinline__ int nn_axis_cell(float x, float o, float inv_s, int n) {
  const float c = fminf(fmaxf(floorf((x - o) * inv_s), 0.f), (float)(n - 1));
  return (int)c;
}

__device__ __forceinline__ int nn_cell_of(const NNGrid& g, float x, float y, float z) {
  return (nn_axis_cell(z, g.oz, g.inv_s, g.dz) * g.dy + nn_axis_cell(y, g.oy, g.inv_s, g.dy)) * g.dx +
         nn_axis_cell(x, g.ox, g.inv_s, g.dx);
}

// cells along an axis of extent e for edge s: floor(e / s) + 1 in [1, NN_MAX_DIM] (non-finite ratios give 1)
__device__ __forceinline__ int nn_dim(double e, double s) {
  const double r = e / s;
  if (!(r >= 0.0)) return 1;
  if (r >= (double)(NN_MAX_DIM - 1)) return NN_MAX_DIM;
  return (int)floor(r) + 1;
}

__global__ void __launch_bounds__(NN_BUILD_THREADS) nn_build_kernel(const int V, const float* __restrict__ targets,
                                                                    NNGrid* __restrict__ grid_out,
                                                                    int* __restrict__ offsets, int* __restrict__ cursor,
                                                                    float4* __restrict__ sorted) {
  __shared__ float red[6][NN_BUILD_THREADS / 32];
  __shared__ NNGrid g;
  __shared__ int wsum[NN_BUILD_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = NN_BUILD_THREADS / 32;

  // 1. bounding box: min / max are exact and order-free, so the box is the same bits on every run
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int j = tid; j < V; j += NN_BUILD_THREADS) {
#pragma unroll
    for (int a = 0; a < 3; a++) {
      const float v = targets[3 * j + a];
      mn[a] = fminf(mn[a], v);
      mx[a] = fmaxf(mx[a], v);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; a++) {
    for (int d = 16; d > 0; d >>= 1) {
      mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], d));
      mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], d));
    }
    if (lane == 0) { red[a][warp] = mn[a]; red[3 + a][warp] = mx[a]; }
  }
  __syncthreads();

  // 2. grid: about one cell per target over the box volume, degenerate extents clamped to 1/1000 of the largest (a
  //    flat or single-point set still gets a grid), the edge grown until the cell count fits the buffers sized from V
  if (tid == 0) {
    double lo[3], e[3], emax = 0.0;
    for (int a = 0; a < 3; a++) {
      float l = FLT_MAX, h = -FLT_MAX;
      for (int w = 0; w < NW; w++) { l = fminf(l, red[a][w]); h = fmaxf(h, red[3 + a][w]); }
      lo[a] = l;
      e[a] = (double)h - (double)l;
      if (e[a] > emax) emax = e[a];  // NaN / negative (non-finite targets) stay out
    }
    const int cmax = nn_max_cells(V);
    double s = 1.0;
    int d[3] = {1, 1, 1};
    if (emax > 0.0 && emax < 1e300) {
      double vol = 1.0;
      for (int a = 0; a < 3; a++) vol *= fmax(e[a] > 0.0 ? e[a] : 0.0, emax * 1e-3);
      s = cbrt(vol / (double)V);
      for (int it = 0;; it++) {
        long long n = 1;
        for (int a = 0; a < 3; a++) { d[a] = nn_dim(e[a], s); n *= d[a]; }
        if (n <= cmax) break;
        if (it == 400) { d[0] = d[1] = d[2] = 1; break; }
        s *= 1.1;
      }
    }
    g.ox = (float)lo[0]; g.oy = (float)lo[1]; g.oz = (float)lo[2];
    g.s = (float)s;
    g.inv_s = 1.f / g.s;
    g.dx = d[0]; g.dy = d[1]; g.dz = d[2];
    float span = 0.f;
    const float o[3] = {g.ox, g.oy, g.oz};
    for (int a = 0; a < 3; a++) span = fmaxf(span, fabsf(o[a]) + (float)d[a] * g.s);
    g.span = span;
    *grid_out = g;
  }
  __syncthreads();
  const int ncell = g.dx * g.dy * g.dz;

  // 3. histogram
  for (int c = tid; c < ncell; c += NN_BUILD_THREADS) offsets[c] = 0;
  __syncthreads();
  for (int j = tid; j < V; j += NN_BUILD_THREADS)
    atomicAdd(offsets + nn_cell_of(g, targets[3 * j], targets[3 * j + 1], targets[3 * j + 2]), 1);
  __syncthreads();

  // 4. exclusive scan in place: each thread owns a contiguous chunk, the chunk sums are scanned across the block
  const int chunk = (ncell + NN_BUILD_THREADS - 1) / NN_BUILD_THREADS;
  const int c0 = min(tid * chunk, ncell), c1 = min(c0 + chunk, ncell);
  int local = 0;
  for (int c = c0; c < c1; c++) local += offsets[c];
  int incl = local;
  for (int d = 1; d < 32; d <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = wsum[lane];
    for (int d = 1; d < 32; d <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += v;
    }
    wsum[lane] = w;  // inclusive over warps
  }
  __syncthreads();
  int run = incl - local + (warp > 0 ? wsum[warp - 1] : 0);
  for (int c = c0; c < c1; c++) {
    const int n = offsets[c];
    offsets[c] = run;
    cursor[c] = run;
    run += n;
  }
  if (tid == 0) offsets[ncell] = V;
  __syncthreads();

  // 5. scatter: (x, y, z, index) per target, grouped by cell
  for (int j = tid; j < V; j += NN_BUILD_THREADS) {
    const float x = targets[3 * j], y = targets[3 * j + 1], z = targets[3 * j + 2];
    const int pos = atomicAdd(cursor + nn_cell_of(g, x, y, z), 1);
    sorted[pos] = make_float4(x, y, z, __int_as_float(j));
  }
}

// (distance, index) lexicographic minimum over the targets [b, e) of the sorted array
__device__ __forceinline__ void nn_scan_range(const float4* __restrict__ sorted, int b, int e, float qx, float qy,
                                              float qz, float& best, int& bj) {
  for (int p = b; p < e; p++) {
    const float4 t = __ldg(sorted + p);
    const float ddx = qx - t.x, ddy = qy - t.y, ddz = qz - t.z;
    const float d = ddx * ddx + ddy * ddy + ddz * ddz;  // no contraction in this unit: the reference's bits
    const int j = __float_as_int(t.w);
    if (d < best || (d == best && j < bj)) { best = d; bj = j; }
  }
}

__global__ void __launch_bounds__(NN_QUERY_THREADS) nn_query_kernel(const int P, const float* __restrict__ queries,
                                                                    const uint8_t* __restrict__ self_map,
                                                                    const NNGrid* __restrict__ grid,
                                                                    const int* __restrict__ offsets,
                                                                    const float4* __restrict__ sorted,
                                                                    int32_t* __restrict__ rows) {
  const int i = blockIdx.x * NN_QUERY_THREADS + threadIdx.x;
  if (i >= P) return;
  if (self_map && self_map[i]) { rows[i] = i; return; }
  const float qx = queries[3 * i], qy = queries[3 * i + 1], qz = queries[3 * i + 2];
  if (!isfinite(qx) || !isfinite(qy) || !isfinite(qz)) { rows[i] = 0; return; }  // argmin of an all-NaN row
  const NNGrid g = *grid;
  const int cx = nn_axis_cell(qx, g.ox, g.inv_s, g.dx), cy = nn_axis_cell(qy, g.oy, g.inv_s, g.dy),
            cz = nn_axis_cell(qz, g.oz, g.inv_s, g.dz);
  // Rounding margin of the stop test: a target's cell index and the cell planes below are computed in fp32 with
  // relative error ~1e-7 of the coordinates involved; 1e-5 of the largest of them covers both with a wide margin.
  const float margin = 1e-5f * (g.span + fmaxf(fabsf(qx), fmaxf(fabsf(qy), fabsf(qz))));
  float best = INFINITY;
  int bj = INT_MAX;  // all-inf distances (an overflowing query) still resolve to the lowest index
  for (int k = 0;; k++) {
    const int z0 = max(cz - k, 0), z1 = min(cz + k, g.dz - 1);
    const int y0 = max(cy - k, 0), y1 = min(cy + k, g.dy - 1);
    const int xl = cx - k, xh = cx + k;
    for (int z = z0; z <= z1; z++) {
      const bool zs = z == cz - k || z == cz + k;
      for (int y = y0; y <= y1; y++) {
        const int row = (z * g.dy + y) * g.dx;
        if (zs || y == cy - k || y == cy + k) {  // a whole row of the shell: one contiguous range of targets
          nn_scan_range(sorted, offsets[row + max(xl, 0)], offsets[row + min(xh, g.dx - 1) + 1], qx, qy, qz, best, bj);
        } else {  // the two end cells of the row
          if (xl >= 0) nn_scan_range(sorted, offsets[row + xl], offsets[row + xl + 1], qx, qy, qz, best, bj);
          if (xh < g.dx && xh != xl) nn_scan_range(sorted, offsets[row + xh], offsets[row + xh + 1], qx, qy, qz, best, bj);
        }
      }
    }
    // distance from the query to the cells outside the visited block, per side that has any
    float lb = INFINITY;
    bool more = false;
    if (xl > 0) { more = true; lb = fminf(lb, qx - (g.ox + (float)xl * g.s)); }
    if (xh < g.dx - 1) { more = true; lb = fminf(lb, (g.ox + (float)(xh + 1) * g.s) - qx); }
    if (cy - k > 0) { more = true; lb = fminf(lb, qy - (g.oy + (float)(cy - k) * g.s)); }
    if (cy + k < g.dy - 1) { more = true; lb = fminf(lb, (g.oy + (float)(cy + k + 1) * g.s) - qy); }
    if (cz - k > 0) { more = true; lb = fminf(lb, qz - (g.oz + (float)(cz - k) * g.s)); }
    if (cz + k < g.dz - 1) { more = true; lb = fminf(lb, (g.oz + (float)(cz + k + 1) * g.s) - qz); }
    if (!more) break;
    lb -= margin;
    // strictly greater: every unvisited target's fp32 distance then exceeds `best` (the factor absorbs the rounding of
    // lb * lb and of the targets' distances, both within a few ulps)
    if (lb > 0.f && lb * lb * (1.f - 1e-5f) > best) break;
  }
  rows[i] = bj;
}

size_t nearest_scratch_bytes(int V) { return nn_layout(V).total; }

int launch_nearest_rows(int P, const float* queries, int V, const float* targets, const uint8_t* self_map,
                        int32_t* rows, void* scratch, cudaStream_t st) {
  const NNLayout L = nn_layout(V);
  char* s = (char*)scratch;
  NNGrid* grid = (NNGrid*)(s + L.grid);
  int* offsets = (int*)(s + L.offsets);
  float4* sorted = (float4*)(s + L.sorted);
  {
    ProfScope p(K_MISC, st);
    launch_k(nn_build_kernel, 1, NN_BUILD_THREADS, 0, st, true, V, targets, grid, offsets, (int*)(s + L.cursor),
             sorted);
  }
  {
    ProfScope p(K_MISC, st);
    launch_k(nn_query_kernel, (P + NN_QUERY_THREADS - 1) / NN_QUERY_THREADS, NN_QUERY_THREADS, 0, st, true, P, queries,
             self_map, (const NNGrid*)grid, (const int*)offsets, (const float4*)sorted, rows);
  }
  return check_launch();
}

// ---------------------------------------------------------------------------------------------------------------------
// Vertex normals: n_v = sum over the CSR entries of v (ascending face order, one per corner) of (v1 - v0) x (v2 - v0),
// then n / max(|n|, 1e-6) (F.normalize), negated where flip is set.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int VN_THREADS = 128;

__global__ void __launch_bounds__(VN_THREADS) vertex_normals_kernel(const int P, const float* __restrict__ xyz,
                                                                    const int32_t* __restrict__ faces,
                                                                    const int32_t* __restrict__ vf_offsets,
                                                                    const int32_t* __restrict__ vf_entries,
                                                                    const uint8_t* __restrict__ flip,
                                                                    float* __restrict__ normals) {
  const int v = blockIdx.x * VN_THREADS + threadIdx.x;
  if (v >= P) return;
  float nx = 0.f, ny = 0.f, nz = 0.f;
  const int e1 = vf_offsets[v + 1];
  for (int e = vf_offsets[v]; e < e1; e++) {
    const int f = vf_entries[e];
    const int i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
    const float ax = xyz[3 * i0], ay = xyz[3 * i0 + 1], az = xyz[3 * i0 + 2];
    const float ux = xyz[3 * i1] - ax, uy = xyz[3 * i1 + 1] - ay, uz = xyz[3 * i1 + 2] - az;
    const float wx = xyz[3 * i2] - ax, wy = xyz[3 * i2 + 1] - ay, wz = xyz[3 * i2 + 2] - az;
    nx += uy * wz - uz * wy;
    ny += uz * wx - ux * wz;
    nz += ux * wy - uy * wx;
  }
  float d = fmaxf(sqrtf(nx * nx + ny * ny + nz * nz), 1e-6f);
  if (flip && flip[v]) d = -d;
  normals[3 * v] = nx / d;
  normals[3 * v + 1] = ny / d;
  normals[3 * v + 2] = nz / d;
}

int launch_vertex_normals(int P, const float* xyz, const int32_t* faces, const int32_t* vf_offsets,
                          const int32_t* vf_entries, const uint8_t* flip, float* normals, cudaStream_t st) {
  ProfScope p(K_MISC, st);
  launch_k(vertex_normals_kernel, (P + VN_THREADS - 1) / VN_THREADS, VN_THREADS, 0, st, true, P, xyz, faces,
           vf_offsets, vf_entries, flip, normals);
  return check_launch();
}

}  // namespace b2r
