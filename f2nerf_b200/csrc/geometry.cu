// geometry.cu — a trained scene's geometry on the device: point location through the perspective-warp octree and
// isosurface extraction from a logit lattice by marching tetrahedra (DESIGN.md §3i).  The field query itself is the
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

}  // namespace f2b

using namespace f2b;

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
