// locate.cuh — a world point through the perspective-warp octree: the leaf that holds it and its warped coordinates.
// Shared by sampler.cu (edge samples), geometry.cu (f2b_locate_points, vertex location) and field.cu (the fused point
// query).  See DESIGN.md §3i.
#pragma once
#include "common.cuh"

namespace f2b {

// QueryFrameTransform (PersSampler.cu:155-169) in the march's roundings (DESIGN §4): xz = (x*a0 + y*a1) + (z*a2 + a3),
// v = xz0 / xz1, then the 12-term mixing sums in Eigen's redux tree.  The march forms the same sums one lane per row.
__device__ __forceinline__ void warp_point(const TransInfo* __restrict__ T, float X, float Y, float Z,
                                           float out[3]) {
  float v[12];
#pragma unroll
  for (int i = 0; i < 12; i++) {
    const float* a = T->w2xz[i];
    const float xz0 = fadd(ffma(X, a[0], fmul(Y, a[1])), ffma(Z, a[2], a[3]));
    const float xz1 = fadd(ffma(X, a[4], fmul(Y, a[5])), ffma(Z, a[6], a[7]));
    v[i] = fdiv(xz0, xz1);
  }
#pragma unroll
  for (int r = 0; r < 3; r++) {
    const float* w = T->weight[r];
    float g[4];
#pragma unroll
    for (int s = 0; s < 4; s++)
      g[s] = ffma(w[3 * s], v[3 * s], ffma(w[3 * s + 1], v[3 * s + 1], fmul(w[3 * s + 2], v[3 * s + 2])));
    out[r] = fadd(fadd(g[0], g[1]), fadd(g[2], g[3]));
  }
}

// QueryFrameTransformJac (PersSampler.cu:171-187): J[r][c] = d warp_r / d x_c at (X, Y, Z), in the roundings of the march's
// phases A and B (sampler.cu): per projection rr = rcp(xz1), q = -xz0 / xz1^2 and the rows fma(a, rr, b * q), then each
// mixing sum in Eigen's redux tree ((g0 + g1) + (g2 + g3)).  One thread forms all nine entries (DESIGN §3j).
__device__ __forceinline__ void warp_jacobian(const TransInfo* __restrict__ T, float X, float Y, float Z, float J[3][3]) {
  float t0[12], t1[12], t2[12];
#pragma unroll
  for (int i = 0; i < 12; i++) {
    const float* a = T->w2xz[i];
    const float xz0 = fadd(ffma(X, a[0], fmul(Y, a[1])), ffma(Z, a[2], a[3]));
    const float xz1 = fadd(ffma(X, a[4], fmul(Y, a[5])), ffma(Z, a[6], a[7]));
    const float rr = frcp(xz1);
    const float q = fdiv(-xz0, fmul(xz1, xz1));
    t0[i] = ffma(a[0], rr, fmul(a[4], q));
    t1[i] = ffma(rr, a[1], fmul(q, a[5]));
    t2[i] = ffma(rr, a[2], fmul(q, a[6]));
  }
#pragma unroll
  for (int r = 0; r < 3; r++) {
    const float* w = T->weight[r];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const float* v = c == 0 ? t0 : (c == 1 ? t1 : t2);
      float g[4];
#pragma unroll
      for (int s = 0; s < 4; s++)
        g[s] = ffma(w[3 * s], v[3 * s], ffma(w[3 * s + 1], v[3 * s + 1], fmul(w[3 * s + 2], v[3 * s + 2])));
      J[r][c] = fadd(fadd(g[0], g[1]), fadd(g[2], g[3]));
    }
  }
}

// The march visits nodes down to depth 23 (its 24-entry stack, sampler.cu kMaxDepth); the walk stops at the same depth.
constexpr int kLocateMaxDepth = 24;

// Leaf of the point (x, y, z), or -1.  Walks from the root, one child per level, child slot
// st = (x >= cx) << 2 | (y >= cy) << 1 | (z >= cz) (ConstructTreeNode, PersSampler.cpp:359-421).
// Tie rule: every node is the half-open cube [c - s/2, c + s/2) on each axis, so a point on a splitting plane belongs to the
// upper child and a point on the root's upper faces to no leaf.  Each visited node's own cube is tested, because a compacted
// tree links a node straight to a deeper descendant (ProcOctree's single-child compression) that covers only part of the
// octant.  A node without live children is a leaf (as the march treats it); trans_idx < 0 there, a dead child slot, or a
// point outside the node's cube give -1.
__device__ __forceinline__ int locate_leaf(const TreeNode* __restrict__ nodes, float x, float y, float z, int& trans_idx) {
  int u = 0;
  for (int depth = 0; depth < kLocateMaxDepth; depth++) {
    const int4* np = reinterpret_cast<const int4*>(nodes + u);
    const int4 q0 = __ldg(np), q1 = __ldg(np + 1), q2 = __ldg(np + 2), q3 = __ldg(np + 3);
    const float cx = __int_as_float(q0.x), cy = __int_as_float(q0.y), cz = __int_as_float(q0.z);
    const float hf = fmul(__int_as_float(q0.w), .5f);
    const bool inside = x >= fsub(cx, hf) && x < fadd(cx, hf) && y >= fsub(cy, hf) && y < fadd(cy, hf) &&
                        z >= fsub(cz, hf) && z < fadd(cz, hf);
    if (!inside) return -1;
    const int childs[8] = {q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x};
    bool live = false;
#pragma unroll
    for (int k = 0; k < 8; k++) live |= childs[k] >= 0;
    if (!live) {
      if (q3.z < 0) return -1;
      trans_idx = q3.z;
      return u;
    }
    const int st = (int(x >= cx) << 2) | (int(y >= cy) << 1) | int(z >= cz);
    const int v = __ldg(reinterpret_cast<const int*>(np) + 5 + st);   // childs[st] (@20 B)
    if (v < 0) return -1;
    u = v;
  }
  return -1;
}

}  // namespace f2b
