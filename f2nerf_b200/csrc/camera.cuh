// camera.cuh — the dataset's lens model, shared by ray generation (rays.cu) and projection into a view (geometry.cu).
#pragma once
#include "common.cuh"

namespace f2b {

struct Dist { float k1, k2, p1, p2, two_p1, two_p2; };

// apply_camera_distortion (Dataset.cu:16-28) as compiled: radial = fma(r2,k1, r2*(r2*k2));
// du = fma(fma(u2,2,r2), p2, fma(uv, 2p1, u*radial)); dv = fma(fma(v2,2,r2), p1, fma(v, radial, uv*2p2))
__device__ __forceinline__ void distort(const Dist& d, float u, float v, float u2, float uv, float v2, float r2, float& du, float& dv) {
  const float radial = ffma(r2, d.k1, fmul(r2, fmul(r2, d.k2)));
  du = ffma(ffma(u2, 2.f, r2), d.p2, ffma(uv, d.two_p1, fmul(u, radial)));
  dv = ffma(ffma(v2, 2.f, r2), d.p1, ffma(v, radial, fmul(uv, d.two_p2)));
}

// how a camera's floats are read: through the read-only cache from global memory, or plainly (a table staged in shared memory)
struct LdgLoad { __device__ __forceinline__ float operator()(const float* p) const { return __ldg(p); } };
struct PlainLoad { __device__ __forceinline__ float operator()(const float* p) const { return *p; } };

template <class Ld = LdgLoad>
__device__ __forceinline__ Dist load_dist(const float* dp, Ld ld = Ld()) {
  Dist d;
  d.k1 = ld(dp); d.k2 = ld(dp + 1); d.p1 = ld(dp + 2); d.p2 = ld(dp + 3);
  d.two_p1 = fadd(d.p1, d.p1); d.two_p2 = fadd(d.p2, d.p2);
  return d;
}

// The nearest cell (a * out_w + b) of the out_h x out_w grid linspace(0, H-1, out_h) x linspace(0, W-1, out_w) that world point
// (pt(0), pt(1), pt(2)) projects to in a view, or -1 behind the camera or outside the grid.  pose [3,4] camera-to-world (the camera looks
// down -z), intri rows 0-1 of K (fx at 0, cx at 2, fy at 4, cy at 5), dist (k1, k2, p1, p2).  dx, dy, dz: p - o, whose length
// is the point's distance from the camera.  Shared by the depth-consistency test and TSDF fusion (DESIGN §3l, §3p).
template <class Ld, class Pt>
__device__ __forceinline__ int project_cell(Ld ld, const float* pose, const float* intri, const float* dist_params, Pt pt, int out_h,
                                            int out_w, float step_i, float step_j, float& dx, float& dy, float& dz) {
  dx = fsub(pt(0), ld(pose + 3));
  dy = fsub(pt(1), ld(pose + 7));
  dz = fsub(pt(2), ld(pose + 11));
  float xc[3];
#pragma unroll
  for (int k = 0; k < 3; k++)                                     // R^T (p - o): column k of R
    xc[k] = ffma(ld(pose + 8 + k), dz, ffma(ld(pose + 4 + k), dy, fmul(ld(pose + k), dx)));
  int idx = -1;
  if (xc[2] < 0.f) {
    const float u = fdiv(xc[0], -xc[2]), v = fdiv(xc[1], xc[2]);  // dir = (u, -v, -1) in the camera frame
    const float u2 = fmul(u, u), uv = fmul(u, v), v2 = fmul(v, v);
    float du, dv;
    distort(load_dist(dist_params, ld), u, v, u2, uv, v2, fadd(u2, v2), du, dv);
    const float x = ffma(ld(intri), fadd(u, du), ld(intri + 2));        // fx u_d + cx
    const float y = ffma(ld(intri + 4), fadd(v, dv), ld(intri + 5));    // fy v_d + cy
    const float fb = fdiv(fsub(x, .5f), step_j), fa = fdiv(fsub(y, .5f), step_i);   // the grid's pixel centres sit at +.5
    if (fb > -1.f && fb < float(out_w) && fa > -1.f && fa < float(out_h)) {
      const int b = __float2int_rn(fb), a = __float2int_rn(fa);
      if (b >= 0 && b < out_w && a >= 0 && a < out_h) idx = a * out_w + b;
    }
  }
  return idx;
}

// torch::linspace(0.f, extent - 1.f, n)'s step, in fp32 on the host exactly as ATen forms it: the pixel pitch of an n-point grid
// spread over extent pixels (f2b_camera_rays)
static inline float linspace_step(int extent, int n) { return n > 1 ? (float(extent) - 1.f - 0.f) / float(n - 1) : 0.f; }

}  // namespace f2b
