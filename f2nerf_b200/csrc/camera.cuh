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

__device__ __forceinline__ Dist load_dist(const float* dp) {
  Dist d;
  d.k1 = __ldg(dp); d.k2 = __ldg(dp + 1); d.p1 = __ldg(dp + 2); d.p2 = __ldg(dp + 3);
  d.two_p1 = fadd(d.p1, d.p1); d.two_p2 = fadd(d.p2, d.p2);
  return d;
}

// torch::linspace(0.f, extent - 1.f, n)'s step, in fp32 on the host exactly as ATen forms it: the pixel pitch of an n-point grid
// spread over extent pixels (f2b_camera_rays)
static inline float linspace_step(int extent, int n) { return n > 1 ? (float(extent) - 1.f - 0.f) / float(n - 1) : 0.f; }

}  // namespace f2b
