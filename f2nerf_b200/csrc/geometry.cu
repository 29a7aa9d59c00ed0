// geometry.cu — a trained scene's geometry on the device: point location through the perspective-warp octree and
// isosurface extraction from a logit lattice by marching tetrahedra (DESIGN.md §3i); the opacity and median depth of rendered
// rays and the depth-consistency test of points against a view (DESIGN.md §3l).  The field query itself is the
// fused encode + MLP kernel of field.cu with a located-point source (f2b_query_logit_points / _grid).
//
// Isosurface.  The lattice is nx x ny x nz logits (x fastest); lattice points outside it read empty_logit (a virtual pad
// layer), so the surface closes where it leaves the box.  Owner points and cells both range over [-1, n) per axis: the
// "extended" lattice of (nx+1)(ny+1)(nz+1) entries, extended index e = (x+1) + (nx+1) * ((y+1) + (ny+1) * (z+1)).  Owner
// point e owns the 7 edges towards +(1,0,0), (0,1,0), (0,0,1), (1,1,0), (1,0,1), (0,1,1), (1,1,1) (direction index 0..6);
// cell e is the cube whose lowest corner is point e, cut into the six Kuhn tetrahedra around its (0,0,0)-(1,1,1)
// diagonal.  Every tetrahedron edge joins two corners a < b whose offsets are nested, so it is the edge owned by corner a
// in direction b - a, and the diagonal of every cube face runs from the face's lowest corner to its highest: neighbouring
// cells cut a shared face identically and the mesh is closed by construction.
//
// A point is inside when its logit > level.  Vertices are numbered by (extended point, direction); faces by (cell,
// tetrahedron, triangle), each triangle oriented outward (towards the lower logit).  Work goes in z-slabs of cells
// [ez0, ez1): the counts cover owner layers [ez0, min(ez1 + 1, nz + 1)) (the extra layer numbers the vertices the slab's
// top cells share with the next slab), so the per-slab scratch is 13 B per owner point and 12 B per cell of the slab.
#include "camera.cuh"
#include "common.cuh"
#include "locate.cuh"

namespace f2b {

// ---- point location -------------------------------------------------------------------------------------------------
__global__ void locate_points_kernel(const TreeNode* __restrict__ nodes, const TransInfo* __restrict__ trans,
                                     const float* __restrict__ pts, int n, float* __restrict__ warped,
                                     int* __restrict__ anchors) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = pts[3 * size_t(i)], y = pts[3 * size_t(i) + 1], z = pts[3 * size_t(i) + 2];
  int ti = -1;
  const int leaf = locate_leaf(nodes, x, y, z, ti);
  float w[3] = {0.f, 0.f, 0.f};
  if (leaf >= 0) warp_point(trans + ti, x, y, z, w);
  else ti = -1;
  warped[3 * size_t(i)] = w[0]; warped[3 * size_t(i) + 1] = w[1]; warped[3 * size_t(i) + 2] = w[2];
  anchors[2 * size_t(i)] = ti; anchors[2 * size_t(i) + 1] = leaf;
}

// QueryFrameTransformJac at located points (DESIGN §3j): J [n,3,3] row-major, d warp_r / d x_c; 0 where no valid leaf holds the point
__global__ void warp_jacobian_points_kernel(const TreeNode* __restrict__ nodes, const TransInfo* __restrict__ trans,
                                            const float* __restrict__ pts, int n, float* __restrict__ jac) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = pts[3 * size_t(i)], y = pts[3 * size_t(i) + 1], z = pts[3 * size_t(i) + 2];
  int ti = -1;
  float J[3][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
  if (locate_leaf(nodes, x, y, z, ti) >= 0) warp_jacobian(trans + ti, x, y, z, J);
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) jac[9 * size_t(i) + 3 * r + c] = J[r][c];
}

// ---- marching tetrahedra ------------------------------------------------------------------------------------------
// The six Kuhn tetrahedra of a cell, corners as offset codes (bit 0 x, bit 1 y, bit 2 z), ordered by the axis
// permutations xyz, xzy, yxz, yzx, zxy, zyx, with the last two corners swapped for the odd permutations so that every
// tetrahedron is positively oriented.
__constant__ unsigned char c_tet[6][4] = {{0, 1, 3, 7}, {0, 1, 7, 5}, {0, 2, 7, 3}, {0, 2, 6, 7}, {0, 4, 5, 7}, {0, 4, 7, 6}};
// direction code b - a (= b ^ a) -> direction index
__constant__ signed char c_dir[8] = {-1, 0, 1, 3, 2, 4, 5, 6};
// face opposite each corner of a positive tetrahedron, ordered so that its normal points away from that corner
__constant__ unsigned char c_opp[4][3] = {{1, 2, 3}, {0, 3, 2}, {0, 1, 3}, {0, 2, 1}};

struct Lattice {
  const float* logit;
  int nx, ny, nz;
  float empty;
  __device__ __forceinline__ float at(int x, int y, int z) const {   // x, y, z: real lattice coordinates
    if (x < 0 || y < 0 || z < 0 || x >= nx || y >= ny || z >= nz) return empty;
    return __ldg(logit + x + size_t(nx) * (y + size_t(ny) * z));
  }
};

__device__ __forceinline__ int n_triangles(int mask) {
  const int k = __popc(mask);
  return k == 2 ? 2 : (k & 1);
}

// Triangle j of a tetrahedron with inside mask `mask` as three edges (pairs of tetrahedron corner positions).
__device__ __forceinline__ void tet_triangle(int mask, int j, int e[3][2]) {
  const int k = __popc(mask);
  if (k == 1 || k == 3) {
    const int apex = __ffs(k == 1 ? mask : (~mask & 15)) - 1;   // the lone inside (k = 1) or outside (k = 3) corner
    const unsigned char* f = c_opp[apex];
    for (int q = 0; q < 3; q++) { e[q][0] = apex; e[q][1] = f[k == 1 ? q : 2 - q]; }
    return;
  }
  int in[2], out[2], ni = 0, no = 0;
  for (int c = 0; c < 4; c++) { if (mask >> c & 1) in[ni++] = c; else out[no++] = c; }
  if ((in[0] == 0 && in[1] == 2) || (in[0] == 1 && in[1] == 3)) { const int t = out[0]; out[0] = out[1]; out[1] = t; }
  // (in0, in1, out0, out1) is now an even permutation: the quad (in0-out0, in0-out1, in1-out1, in1-out0) faces outward
  const int a = in[0], b = in[1], c = out[0], d = out[1];
  if (j == 0) { e[0][0] = a; e[0][1] = c; e[1][0] = a; e[1][1] = d; e[2][0] = b; e[2][1] = d; }
  else        { e[0][0] = a; e[0][1] = c; e[1][0] = b; e[1][1] = d; e[2][0] = b; e[2][1] = c; }
}

// pass 1 (owner points of layers [ez0, ez0 + n_layers)) and pass 2 (cells of layers [ez0, ez0 + n_cell_layers)) in one grid
__global__ void iso_count_kernel(Lattice L, float level, int ez0, int n_pt_layers, int n_cell_layers,
                                 unsigned char* __restrict__ edge_mask, int* __restrict__ vert_counts,
                                 int* __restrict__ tri_counts) {
  const int ex_n = L.nx + 1, ey_n = L.ny + 1;
  const int64_t per_layer = int64_t(ex_n) * ey_n;
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= per_layer * n_pt_layers) return;
  const int ex = int(i % ex_n), ey = int((i / ex_n) % ey_n), ez = ez0 + int(i / per_layer);
  const int x = ex - 1, y = ey - 1, z = ez - 1;
  bool in[8];
#pragma unroll
  for (int c = 0; c < 8; c++) in[c] = L.at(x + (c & 1), y + (c >> 1 & 1), z + (c >> 2)) > level;
  int mask = 0;
#pragma unroll
  for (int code = 1; code < 8; code++) mask |= int(in[0] != in[code]) << c_dir[code];
  edge_mask[i] = (unsigned char)mask;
  vert_counts[i] = __popc(mask);
  if (i < per_layer * n_cell_layers) {
    int n = 0;
#pragma unroll
    for (int t = 0; t < 6; t++) {
      int m = 0;
#pragma unroll
      for (int q = 0; q < 4; q++) m |= int(in[c_tet[t][q]]) << q;
      n += n_triangles(m);
    }
    tri_counts[i] = n;
  }
}

__global__ void iso_emit_kernel(Lattice L, float level, float ox, float oy, float oz, float vx, float vy, float vz,
                                int ez0, int n_cell_layers, int vert_base, const unsigned char* __restrict__ edge_mask,
                                const int* __restrict__ vert_bounds, const int* __restrict__ tri_bounds,
                                float* __restrict__ verts, int* __restrict__ faces) {
  const int ex_n = L.nx + 1, ey_n = L.ny + 1;
  const int64_t per_layer = int64_t(ex_n) * ey_n;
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= per_layer * n_cell_layers) return;
  const int ex = int(i % ex_n), ey = int((i / ex_n) % ey_n), ez = ez0 + int(i / per_layer);
  const int x = ex - 1, y = ey - 1, z = ez - 1;
  // vertices of the edges this point owns: t = (level - f_a) / (f_b - f_a), position = origin + voxel * (index + t * dir)
  const int mask = edge_mask[i];
  if (mask) {
    const float fa = L.at(x, y, z);
    int v = vert_bounds[2 * i];
    for (int code = 1; code < 8; code++) {
      if (!(mask >> c_dir[code] & 1)) continue;
      const int dx = code & 1, dy = code >> 1 & 1, dz = code >> 2;
      const float fb = L.at(x + dx, y + dy, z + dz);
      const float t = fdiv(fsub(level, fa), fsub(fb, fa));
      // (vertices of one point are numbered in direction-index order: codes 1, 2, 4, 3, 5, 6, 7)
      const int slot = v + __popc(mask & ((1 << c_dir[code]) - 1));
      const float ux = dx ? fadd(float(x), t) : float(x), uy = dy ? fadd(float(y), t) : float(y),
                  uz = dz ? fadd(float(z), t) : float(z);
      verts[3 * size_t(slot)] = fadd(ox, fmul(vx, ux));
      verts[3 * size_t(slot) + 1] = fadd(oy, fmul(vy, uy));
      verts[3 * size_t(slot) + 2] = fadd(oz, fmul(vz, uz));
    }
  }
  // triangles of the cell
  int f = tri_bounds[2 * i];
  if (f == tri_bounds[2 * i + 1]) return;
  bool in[8];
#pragma unroll
  for (int c = 0; c < 8; c++) in[c] = L.at(x + (c & 1), y + (c >> 1 & 1), z + (c >> 2)) > level;
  for (int t = 0; t < 6; t++) {
    int m = 0;
    for (int q = 0; q < 4; q++) m |= int(in[c_tet[t][q]]) << q;
    const int nt = n_triangles(m);
    for (int j = 0; j < nt; j++, f++) {
      int e[3][2];
      tet_triangle(m, j, e);
      for (int q = 0; q < 3; q++) {
        int a = c_tet[t][e[q][0]], b = c_tet[t][e[q][1]];
        if (a > b) { const int s = a; a = b; b = s; }
        const int64_t owner = i + (a & 1) + int64_t(a >> 1 & 1) * ex_n + int64_t(a >> 2) * per_layer;
        const int om = edge_mask[owner], d = c_dir[a ^ b];
        faces[3 * size_t(f) + q] = vert_base + vert_bounds[2 * owner] + __popc(om & ((1 << d) - 1));
      }
    }
  }
}

// ---- depth of a view and depth consistency (DESIGN §3l) ------------------------------------------------------------
// One warp per ray.  Lanes load 32 consecutive kept weights (coalesced); the running sum is chained through the lanes in slot
// order, one fadd per sample starting from +0, so W is the serial left-to-right fp32 sum (lanes past the kept prefix add +0,
// which leaves the sum unchanged).  The running sum at the end of every 32-slot chunk goes to shared memory; the median is then
// found without a second pass over the ray: a ballot over the chunk ends picks the first chunk that reaches 0.5 W, and one
// more chain over that chunk, started from the previous chunk's end, gives the same partial sums bit for bit.
constexpr int kTermWarps = 8;

__global__ void __launch_bounds__(kTermWarps * 32)
ray_termination_kernel(const float* __restrict__ slot_t, const int* __restrict__ kept, const float* __restrict__ w_slots,
                       const float* __restrict__ rays_o, const float* __restrict__ rays_d, int n_rays, int slot_size,
                       float* __restrict__ opacity, float* __restrict__ median_t, float* __restrict__ point) {
  extern __shared__ float s_ends[];                               // [kTermWarps][chunks] running sum at each chunk's end
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ray = blockIdx.x * kTermWarps + warp;
  if (ray >= n_rays) return;
  const int chunks = (slot_size + 31) >> 5;
  float* ends = s_ends + warp * chunks;
  const int k = __ldg(kept + ray);
  const float* w = w_slots + size_t(ray) * slot_size;
  float run = 0.f;
  for (int base = 0; base < k; base += 32) {
    const float v = base + lane < k ? __ldg(w + base + lane) : 0.f;
#pragma unroll
    for (int j = 0; j < 32; j++) run = fadd(run, __shfl_sync(0xffffffffu, v, j));
    if (lane == 0) ends[base >> 5] = run;
  }
  __syncwarp();
  const float W = run;
  float tm = 0.f, px = 0.f, py = 0.f, pz = 0.f;
  if (W > 0.f) {
    const float half = fmul(.5f, W);
    const int n_chunks = (k + 31) >> 5;
    int c = -1;
    for (int g = 0; g < n_chunks && c < 0; g += 32) {
      const unsigned hit = __ballot_sync(0xffffffffu, g + lane < n_chunks && ends[g + lane] >= half);
      if (hit) c = g + __ffs(hit) - 1;
    }
    const int base = c << 5;
    const float v = base + lane < k ? __ldg(w + base + lane) : 0.f;
    float r = c > 0 ? ends[c - 1] : 0.f, mine = 0.f;
#pragma unroll
    for (int j = 0; j < 32; j++) {
      r = fadd(r, __shfl_sync(0xffffffffu, v, j));
      if (lane == j) mine = r;                                   // the running sum through my sample
    }
    const unsigned hit = __ballot_sync(0xffffffffu, base + lane < k && mine >= half);
    const int m = base + __ffs(hit) - 1;
    tm = __ldg(slot_t + size_t(ray) * slot_size + m);
    px = ffma(tm, __ldg(rays_d + ray * 3), __ldg(rays_o + ray * 3));
    py = ffma(tm, __ldg(rays_d + ray * 3 + 1), __ldg(rays_o + ray * 3 + 1));
    pz = ffma(tm, __ldg(rays_d + ray * 3 + 2), __ldg(rays_o + ray * 3 + 2));
  }
  if (lane == 0) {
    opacity[ray] = W > 0.f ? W : 0.f;
    median_t[ray] = tm;
    if (point) { point[ray * 3] = px; point[ray * 3 + 1] = py; point[ray * 3 + 2] = pz; }
  }
}

// One thread per candidate point: project into view b (pose P = [R | o] camera-to-world, the camera looking down -z), take the
// nearest cell of the out_h x out_w grid, and count the view when its depth map agrees there.
__global__ void __launch_bounds__(128)
depth_consistency_kernel(const float* __restrict__ pts, const int* __restrict__ source, int n_pts, int view,
                         const float* __restrict__ pose, const float* __restrict__ intri, const float* __restrict__ dist_params,
                         int out_h, int out_w, float step_i, float step_j, const float* __restrict__ opacity,
                         const float* __restrict__ median_t, float min_opacity, float rel_tol, int* __restrict__ count,
                         int* __restrict__ cell) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pts) return;
  if (source && __ldg(source + i) == view) {
    if (cell) cell[i] = -1;
    return;
  }
  float dx, dy, dz;
  const int idx = project_cell(LdgLoad(), pose, intri, dist_params, [&](int k) { return __ldg(pts + 3 * size_t(i) + k); }, out_h, out_w,
                               step_i, step_j, dx, dy, dz);
  if (cell) cell[i] = idx;
  if (idx < 0 || !(__ldg(opacity + idx) >= min_opacity)) return;
  const float tb = __ldg(median_t + idx);
  const float dist = fsqrt(fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz)));
  if (fabsf(fsub(dist, tb)) <= fmul(rel_tol, tb)) count[i] += 1;
}


// ---- TSDF fusion (DESIGN §3p) ----------------------------------------------------------------------------------------
// One thread per lattice point of a z-slab, over a group of views whose camera table (kTsdfCam floats per view: pose 12, rows
// 0-1 of K 6, distortion 4) is staged in shared memory.  The point's sums are read once (unless the group is the first), carried
// in registers across the group's views in order, and written once; every addition is one fp32 op in view order, so the bits do
// not depend on how the views are split into groups.
constexpr int kTsdfCam = 22;
constexpr int kTsdfMaxViews = 64;
constexpr int kTsdfThreads = 128;

__global__ void __launch_bounds__(kTsdfThreads)
tsdf_integrate_kernel(const float* __restrict__ cams, int n_views, const float* __restrict__ opacity, const float* __restrict__ median_t,
                      const float* __restrict__ colors, int out_h, int out_w, float step_i, float step_j, float ox, float oy,
                      float oz, float vox, int nx, int ny, int z0, int n_layers, float mu, float min_opacity, int first,
                      float* __restrict__ sdf_sum, float* __restrict__ weight, float* __restrict__ color_sum) {
  __shared__ float s_cam[kTsdfMaxViews * kTsdfCam];
  for (int k = threadIdx.x; k < n_views * kTsdfCam; k += blockDim.x) s_cam[k] = __ldg(cams + k);
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nx * ny * n_layers) return;
  const int ix = i % nx, iy = (i / nx) % ny, iz = z0 + i / (nx * ny);
  const float p[3] = {fadd(ox, fmul(vox, float(ix))), fadd(oy, fmul(vox, float(iy))), fadd(oz, fmul(vox, float(iz)))};
  const size_t g = size_t(iz) * nx * ny + size_t(iy) * nx + ix;
  float s = 0.f, w = 0.f, r = 0.f, gr = 0.f, b = 0.f;
  if (!first) {
    s = sdf_sum[g]; w = weight[g];
    r = color_sum[3 * g]; gr = color_sum[3 * g + 1]; b = color_sum[3 * g + 2];
  }
  const size_t n_cells = size_t(out_h) * out_w;
  const float neg_mu = -mu;
  for (int v = 0; v < n_views; v++) {
    const float* cam = s_cam + v * kTsdfCam;
    float dx, dy, dz;
    const int idx = project_cell(PlainLoad(), cam, cam + 12, cam + 18, [&](int k) { return p[k]; }, out_h, out_w, step_i, step_j, dx, dy, dz);
    if (idx < 0) continue;
    const size_t c = v * n_cells + idx;
    if (!(__ldg(opacity + c) >= min_opacity)) continue;
    const float dist = fsqrt(fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz)));
    const float sdf = fsub(__ldg(median_t + c), dist);
    if (!(sdf >= neg_mu)) continue;
    s = fadd(s, fminf(1.f, fdiv(sdf, mu)));
    w = fadd(w, 1.f);
    r = fadd(r, __ldg(colors + 3 * c)); gr = fadd(gr, __ldg(colors + 3 * c + 1)); b = fadd(b, __ldg(colors + 3 * c + 2));
  }
  sdf_sum[g] = s; weight[g] = w;
  color_sum[3 * g] = r; color_sum[3 * g + 1] = gr; color_sum[3 * g + 2] = b;
}

// One thread per vertex: trilinear interpolation of color_sum / weight over the observed corners of the vertex's cell (weight > 0
// and not on the lattice's outermost layer), their trilinear weights renormalised; 0 where no corner is observed.
__global__ void __launch_bounds__(128)
tsdf_colors_kernel(const float* __restrict__ verts, int n_verts, const float* __restrict__ weight, const float* __restrict__ color_sum,
                   int nx, int ny, int nz, float ox, float oy, float oz, float vox, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_verts) return;
  const int n[3] = {nx, ny, nz};
  const float o[3] = {ox, oy, oz};
  int i0[3];
  float f[3];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float u = fdiv(fsub(__ldg(verts + 3 * size_t(i) + k), o[k]), vox);
    const int c = min(max(int(floorf(u)), 0), n[k] - 2);
    i0[k] = c;
    f[k] = fminf(fmaxf(fsub(u, float(c)), 0.f), 1.f);
  }
  float acc[3] = {0.f, 0.f, 0.f}, tw = 0.f;
#pragma unroll
  for (int q = 0; q < 8; q++) {
    const int x = i0[0] + (q & 1), y = i0[1] + (q >> 1 & 1), z = i0[2] + (q >> 2);
    if (x == 0 || y == 0 || z == 0 || x == nx - 1 || y == ny - 1 || z == nz - 1) continue;
    const size_t g = size_t(z) * nx * ny + size_t(y) * nx + x;
    const float wg = __ldg(weight + g);
    if (!(wg > 0.f)) continue;
    const float t = fmul(fmul(q & 1 ? f[0] : fsub(1.f, f[0]), q & 2 ? f[1] : fsub(1.f, f[1])), q & 4 ? f[2] : fsub(1.f, f[2]));
#pragma unroll
    for (int k = 0; k < 3; k++) acc[k] = ffma(t, fdiv(__ldg(color_sum + 3 * g + k), wg), acc[k]);
    tw = fadd(tw, t);
  }
#pragma unroll
  for (int k = 0; k < 3; k++) out[3 * size_t(i) + k] = tw > 0.f ? fdiv(acc[k], tw) : 0.f;
}

}  // namespace f2b

using namespace f2b;

extern "C" int f2b_ray_termination_slots(const float* slot_t, const int* kept_counts, const float* w_slots, const float* rays_o,
                                         const float* rays_d, int n_rays, int slot_size, float* opacity, float* median_t,
                                         float* point, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(slot_t && kept_counts && w_slots && rays_o && rays_d && opacity && median_t, "f2b_ray_termination_slots: null pointer");
  F2B_REQUIRE(slot_size > 0 && slot_size <= 32 * 1024, "f2b_ray_termination_slots: slot_size %d outside [1, 32768]", slot_size);
  F2B_REQUIRE(int64_t(n_rays) * slot_size < (int64_t(1) << 31), "f2b_ray_termination_slots: n_rays * slot_size overflows int32");
  const size_t smem = size_t(kTermWarps) * ((slot_size + 31) / 32) * sizeof(float);
  ray_termination_kernel<<<div_up(n_rays, kTermWarps), kTermWarps * 32, smem, as_stream(stream)>>>(
      slot_t, kept_counts, w_slots, rays_o, rays_d, n_rays, slot_size, opacity, median_t, point);
  return check_launch("f2b_ray_termination_slots");
}

extern "C" int f2b_depth_consistency(const float* pts, const int* source, int n_pts, int view, const float* pose, const float* intri,
                                     const float* dist_params, int height, int width, int out_h, int out_w, const float* opacity,
                                     const float* median_t, float min_opacity, float rel_tol, int* count, int* cell, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(pts && pose && intri && dist_params && opacity && median_t && count, "f2b_depth_consistency: null pointer");
  F2B_REQUIRE(out_h >= 2 && out_h <= height && out_w >= 2 && out_w <= width, "f2b_depth_consistency: grid %dx%d outside image %dx%d",
              out_h, out_w, height, width);
  F2B_REQUIRE(int64_t(out_h) * out_w < (int64_t(1) << 31), "f2b_depth_consistency: %d x %d cells overflow int32", out_h, out_w);
  depth_consistency_kernel<<<div_up(n_pts, 128), 128, 0, as_stream(stream)>>>(
      pts, source, n_pts, view, pose, intri, dist_params, out_h, out_w, linspace_step(height, out_h), linspace_step(width, out_w),
      opacity, median_t, min_opacity, rel_tol, count, cell);
  return check_launch("f2b_depth_consistency");
}

extern "C" int f2b_locate_points(const void* tree_nodes, int n_nodes, const void* trans, const float* pts, int n_pts,
                                 float* warped, int* anchors, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(tree_nodes && n_nodes > 0 && trans && pts && warped && anchors, "f2b_locate_points: bad argument");
  locate_points_kernel<<<div_up(n_pts, 128), 128, 0, as_stream(stream)>>>((const TreeNode*)tree_nodes, (const TransInfo*)trans,
                                                                          pts, n_pts, warped, anchors);
  return check_launch("f2b_locate_points");
}

extern "C" int f2b_warp_jacobian_points(const void* tree_nodes, int n_nodes, const void* trans, const float* pts, int n_pts,
                                        float* jac, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(tree_nodes && n_nodes > 0 && trans && pts && jac, "f2b_warp_jacobian_points: bad argument");
  warp_jacobian_points_kernel<<<div_up(n_pts, 128), 128, 0, as_stream(stream)>>>((const TreeNode*)tree_nodes, (const TransInfo*)trans,
                                                                                 pts, n_pts, jac);
  return check_launch("f2b_warp_jacobian_points");
}

static bool iso_slab_ok(int nx, int ny, int nz, int ez0, int ez1) {
  return nx > 0 && ny > 0 && nz > 0 && ez0 >= 0 && ez0 < ez1 && ez1 <= nz + 1 &&
         int64_t(nx + 1) * (ny + 1) * (ez1 - ez0 + 1) < (int64_t(1) << 31);
}

extern "C" int f2b_iso_count(const float* logit, int nx, int ny, int nz, float level, float empty_logit, int ez0, int ez1,
                             uint8_t* edge_mask, int* vert_counts, int* tri_counts, void* stream) {
  F2B_REQUIRE(logit && edge_mask && vert_counts && tri_counts, "f2b_iso_count: null pointer");
  F2B_REQUIRE(iso_slab_ok(nx, ny, nz, ez0, ez1), "f2b_iso_count: bad lattice or slab");
  F2B_REQUIRE(empty_logit <= level, "f2b_iso_count: empty_logit must not be above the level (the pad must be outside)");
  const int pt_layers = min(ez1 + 1, nz + 1) - ez0;
  const int64_t n = int64_t(nx + 1) * (ny + 1) * pt_layers;
  iso_count_kernel<<<div_up(n, 256), 256, 0, as_stream(stream)>>>(Lattice{logit, nx, ny, nz, empty_logit}, level, ez0, pt_layers,
                                                                  ez1 - ez0, edge_mask, vert_counts, tri_counts);
  return check_launch("f2b_iso_count");
}

extern "C" int f2b_iso_emit(const float* logit, int nx, int ny, int nz, float level, float empty_logit, const float* origin3,
                            const float* voxel3, int ez0, int ez1, int vert_base, const uint8_t* edge_mask,
                            const int* vert_bounds, const int* tri_bounds, float* verts, int* faces, void* stream) {
  F2B_REQUIRE(logit && origin3 && voxel3 && edge_mask && vert_bounds && tri_bounds, "f2b_iso_emit: null pointer");
  F2B_REQUIRE(iso_slab_ok(nx, ny, nz, ez0, ez1), "f2b_iso_emit: bad lattice or slab");
  const int64_t n = int64_t(nx + 1) * (ny + 1) * (ez1 - ez0);
  iso_emit_kernel<<<div_up(n, 256), 256, 0, as_stream(stream)>>>(Lattice{logit, nx, ny, nz, empty_logit}, level, origin3[0], origin3[1],
                                                                 origin3[2], voxel3[0], voxel3[1], voxel3[2], ez0, ez1 - ez0, vert_base,
                                                                 edge_mask, vert_bounds, tri_bounds, verts, faces);
  return check_launch("f2b_iso_emit");
}

extern "C" int f2b_tsdf_integrate(const float* cams, int n_views, const float* opacity, const float* median_t, const float* colors,
                                  int height, int width, int out_h, int out_w, const float* origin3, float voxel, int nx, int ny,
                                  int nz, int z0, int n_layers, float mu, float min_opacity, int first, float* sdf_sum,
                                  float* weight, float* color_sum, void* stream) {
  F2B_REQUIRE(cams && opacity && median_t && colors && origin3 && sdf_sum && weight && color_sum, "f2b_tsdf_integrate: null pointer");
  F2B_REQUIRE(n_views >= 1 && n_views <= kTsdfMaxViews, "f2b_tsdf_integrate: %d views outside [1, %d] per launch", n_views, kTsdfMaxViews);
  F2B_REQUIRE(out_h >= 2 && out_h <= height && out_w >= 2 && out_w <= width, "f2b_tsdf_integrate: grid %dx%d outside image %dx%d",
              out_h, out_w, height, width);
  F2B_REQUIRE(int64_t(out_h) * out_w < (int64_t(1) << 31), "f2b_tsdf_integrate: %d x %d cells overflow int32", out_h, out_w);
  F2B_REQUIRE(nx >= 1 && ny >= 1 && nz >= 1 && z0 >= 0 && n_layers >= 1 && z0 + n_layers <= nz,
              "f2b_tsdf_integrate: bad lattice %d x %d x %d or slab [%d, %d)", nx, ny, nz, z0, z0 + n_layers);
  F2B_REQUIRE(int64_t(nx) * ny * n_layers < (int64_t(1) << 31), "f2b_tsdf_integrate: the slab's points overflow int32");
  F2B_REQUIRE(isfinite(voxel) && voxel > 0.f, "f2b_tsdf_integrate: voxel must be finite and > 0");
  F2B_REQUIRE(isfinite(mu) && mu > 0.f, "f2b_tsdf_integrate: mu must be finite and > 0");
  F2B_REQUIRE(min_opacity > 0.f && min_opacity <= 1.f, "f2b_tsdf_integrate: min_opacity must lie in (0, 1]");
  const int64_t n = int64_t(nx) * ny * n_layers;
  tsdf_integrate_kernel<<<div_up(n, kTsdfThreads), kTsdfThreads, 0, as_stream(stream)>>>(
      cams, n_views, opacity, median_t, colors, out_h, out_w, linspace_step(height, out_h), linspace_step(width, out_w), origin3[0],
      origin3[1], origin3[2], voxel, nx, ny, z0, n_layers, mu, min_opacity, first, sdf_sum, weight, color_sum);
  return check_launch("f2b_tsdf_integrate");
}

extern "C" int f2b_tsdf_colors(const float* verts, int n_verts, const float* weight, const float* color_sum, int nx, int ny, int nz,
                               const float* origin3, float voxel, float* colors, void* stream) {
  if (n_verts <= 0) return F2B_OK;
  F2B_REQUIRE(verts && weight && color_sum && origin3 && colors, "f2b_tsdf_colors: null pointer");
  F2B_REQUIRE(nx >= 2 && ny >= 2 && nz >= 2, "f2b_tsdf_colors: lattice %d x %d x %d has an axis under 2 points", nx, ny, nz);
  F2B_REQUIRE(isfinite(voxel) && voxel > 0.f, "f2b_tsdf_colors: voxel must be finite and > 0");
  tsdf_colors_kernel<<<div_up(n_verts, 128), 128, 0, as_stream(stream)>>>(verts, n_verts, weight, color_sum, nx, ny, nz, origin3[0],
                                                                        origin3[1], origin3[2], voxel, colors);
  return check_launch("f2b_tsdf_colors");
}
