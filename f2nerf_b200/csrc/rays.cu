// rays.cu — SURVEY §8(f) N3: ray generation, the step immediately before the path.
//
// Replaces Dataset::Img2WorldRayFlex + Img2WorldRayKernel (src/Dataset/Dataset.cu:100-152, with the 100-iteration
// Newton undistortion of :30-74 taken from instant-ngp) and the CPU-side ground-truth gather + host->device copy of
// Dataset::RandRaysData (src/Dataset/Dataset.cpp:290): with the images resident in HBM one small kernel each.
// The fp32 operation order of the undistortion was read off the reference build's SASS (nvcc 12.9; ptxas
// fuses further mul+sub pairs that the PTX still shows separately) and is spelled out with explicit roundings, so rays are bit-identical to the reference's (tests/test_ref_parity.py).
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

__global__ void __launch_bounds__(128)
img2world_kernel(int n_rays, const float* __restrict__ poses, const float* __restrict__ intri,
                 const float* __restrict__ dist_params, const int* __restrict__ cam_indices,
                 const int* __restrict__ ij, float* __restrict__ rays_o, float* __restrict__ rays_d) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  const int cam = __ldg(cam_indices + r);
  const float pi = fadd((float)__ldg(ij + 2 * r), .5f), pj = fadd((float)__ldg(ij + 2 * r + 1), .5f);   // (ij + .5f), Dataset.cu:128
  const float* K = intri + size_t(cam) * 9;
  const float fx = __ldg(K), cx = __ldg(K + 2), fy = __ldg(K + 4), cy = __ldg(K + 5);
  const float u0 = fdiv(fsub(pj, cx), fx), v0 = fdiv(fsub(pi, cy), fy);              // OpenCV style
  const float* dp = dist_params + size_t(cam) * 4;
  Dist d;
  d.k1 = __ldg(dp); d.k2 = __ldg(dp + 1); d.p1 = __ldg(dp + 2); d.p2 = __ldg(dp + 3);
  d.two_p1 = fadd(d.p1, d.p1); d.two_p2 = fadd(d.p2, d.p2);
  float u = u0, v = v0;
  for (int it = 0; it < 100; it++) {                                                   // iterative_camera_undistortion
    const float s0 = fmaxf(fabsf(fmul(u, 1e-6f)), 1.1920929e-7f), s1 = fmaxf(fabsf(fmul(v, 1e-6f)), 1.1920929e-7f);
    const float u2 = fmul(u, u), uv = fmul(u, v), v2 = fmul(v, v);
    float du, dv, b0x, b0y, f0x, f0y, b1x, b1y, f1x, f1y;
    distort(d, u, v, u2, uv, v2, fadd(u2, v2), du, dv);
    { const float a = fsub(u, s0), a2 = fmul(a, a); distort(d, a, v, a2, fmul(v, a), v2, fadd(v2, a2), b0x, b0y); }
    { const float a = fadd(u, s0), a2 = fmul(a, a); distort(d, a, v, a2, fmul(v, a), v2, fadd(v2, a2), f0x, f0y); }
    { const float a = fsub(v, s1), a2 = fmul(a, a); distort(d, u, a, u2, fmul(u, a), a2, fadd(u2, a2), b1x, b1y); }
    { const float a = fadd(v, s1), a2 = fmul(a, a); distort(d, u, a, u2, fmul(u, a), a2, fadd(u2, a2), f1x, f1y); }
    const float two_s0 = fadd(s0, s0), two_s1 = fadd(s1, s1);
    const float j00 = fadd(fdiv(fsub(f0x, b0x), two_s0), 1.f), j01 = fdiv(fsub(f1x, b1x), two_s1);
    const float j10 = fdiv(fsub(f0y, b0y), two_s0), j11 = fadd(fdiv(fsub(f1y, b1y), two_s1), 1.f);
    const float inv = frcp(ffma(j00, j11, -fmul(j10, j01)));                           // Eigen 2x2 inverse (ptxas fuses the mul+sub)
    const float rx = fsub(fadd(u, du), u0), ry = fsub(fadd(v, dv), v0);
    const float sx = ffma(fmul(j11, inv), rx, -fmul(fmul(inv, j01), ry));
    const float sy = ffma(fmul(j00, inv), ry, -fmul(fmul(inv, j10), rx));
    u = fsub(u, sx); v = fsub(v, sy);
    if (ffma(sx, sx, fmul(sy, sy)) < 1e-10f) break;                                   // squaredNorm() < kMaxStepNorm (NaN keeps iterating)
  }
  const float nv = -v;                                                                 // dir = (u, -v, -1), OpenGL style
  const float* P = poses + size_t(cam) * 12;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    rays_d[size_t(r) * 3 + k] = ffma(u, __ldg(P + 4 * k), ffma(nv, __ldg(P + 4 * k + 1), -__ldg(P + 4 * k + 2)));
    rays_o[size_t(r) * 3 + k] = __ldg(P + 4 * k + 3);
  }
}

__global__ void __launch_bounds__(256)
gather_pixels_kernel(int n, const float* __restrict__ images, const int* __restrict__ cam_indices,
                     const int* __restrict__ ij, int height, int width, float* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const size_t px = (size_t(__ldg(cam_indices + r)) * height + __ldg(ij + 2 * r)) * width + __ldg(ij + 2 * r + 1);
  out[size_t(r) * 3] = __ldg(images + px * 3);
  out[size_t(r) * 3 + 1] = __ldg(images + px * 3 + 1);
  out[size_t(r) * 3 + 2] = __ldg(images + px * 3 + 2);
}

}  // namespace f2b

using namespace f2b;

extern "C" int f2b_img2world_rays(const float* poses, const float* intri, const float* dist_params, const int* cam_indices,
                                  const int* ij, int n_rays, float* rays_o, float* rays_d, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(poses && intri && dist_params && cam_indices && ij && rays_o && rays_d, "f2b_img2world_rays: null pointer");
  img2world_kernel<<<div_up(n_rays, 128), 128, 0, as_stream(stream)>>>(n_rays, poses, intri, dist_params, cam_indices, ij,
                                                                      rays_o, rays_d);
  return check_launch("f2b_img2world_rays");
}

extern "C" int f2b_gather_pixels(const float* images, const int* cam_indices, const int* ij, int height, int width,
                                 int n, float* out, void* stream) {
  if (n <= 0) return F2B_OK;
  F2B_REQUIRE(images && cam_indices && ij && out && height > 0 && width > 0, "f2b_gather_pixels: bad argument");
  gather_pixels_kernel<<<div_up(n, 256), 256, 0, as_stream(stream)>>>(n, images, cam_indices, ij, height, width, out);
  return check_launch("f2b_gather_pixels");
}
