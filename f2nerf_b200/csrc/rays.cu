// rays.cu — SURVEY §8(f) N3: ray generation, the step immediately before the path.
//
// Replaces Dataset::Img2WorldRayFlex + Img2WorldRayKernel (src/Dataset/Dataset.cu:100-152, with the 100-iteration
// Newton undistortion of :30-74 taken from instant-ngp) and the CPU-side ground-truth gather + host->device copy of
// Dataset::RandRaysData (src/Dataset/Dataset.cpp:290): with the images resident in HBM one small kernel each.
// The fp32 operation order of the undistortion was read off the reference build's SASS (nvcc 12.9; ptxas
// fuses further mul+sub pairs that the PTX still shows separately) and is spelled out with explicit roundings, so rays are bit-identical to the reference's (tests/test_ref_parity.py).
// f2b_camera_rays is the whole-camera path of the evaluation modes (Dataset::RaysOfCamera / RaysFromPose), an ATen sequence in the
// reference, in one kernel (tests/test_gpu_eval.py).
#include "camera.cuh"

namespace f2b {

// iterative_camera_undistortion (Dataset.cu:30-69) on the OpenCV-style point (u0, v0).  It is inlined twice in the reference
// build, into Img2WorldRayKernel and into CameraUndistortKernel (:71-76); ptxas schedules the two loops differently but makes
// the same contractions (the same 140 FP instructions per iteration, FFMA for FFMA; only two FADD subtractions list their
// operands the other way round), so one function serves both kernels.
__device__ __forceinline__ void undistort(const Dist& d, const float u0, const float v0, float& u_out, float& v_out) {
  float u = u0, v = v0;
  for (int it = 0; it < 100; it++) {
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
  u_out = u; v_out = v;
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
  float u, v;
  undistort(load_dist(dist_params + size_t(cam) * 4), u0, v0, u, v);
  const float nv = -v;                                                                 // dir = (u, -v, -1), OpenGL style
  const float* P = poses + size_t(cam) * 12;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    rays_d[size_t(r) * 3 + k] = ffma(u, __ldg(P + 4 * k), ffma(nv, __ldg(P + 4 * k + 1), -__ldg(P + 4 * k + 2)));
    rays_o[size_t(r) * 3 + k] = __ldg(P + 4 * k + 3);
  }
}

// ATen's CUDA linspace(0, end, n) (RangeFactories.cu) at index idx: two-sided, step = end / (n - 1) computed on the host in
// fp32; the lower half is start + step*idx (exact to round(step*idx) with start 0, fused or not), the upper half
// end - step*(n-1-idx), which nvcc contracts into one FFMA.
__device__ __forceinline__ float linspace_at(float end, float step, int n, int idx) {
  if (n == 1) return 0.f;
  if (idx < n / 2) return fmul(step, (float)idx);
  return ffma(-step, (float)(n - 1 - idx), end);
}

// Dataset::RaysOfCamera / RaysFromPose (Dataset.cpp:177-218) -> Img2WorldRay (:152-175): an out_h x out_w meshgrid of
// linspace(0, height-1, out_h) x linspace(0, width-1, out_w) pixel rows/columns, + .5, ATen's division by the CPU scalars
// fx / fy (a multiply by the host-rounded reciprocal, div_true_kernel_cuda), CameraUndistortKernel (Dataset.cu:71-95; its two
// sign flips cancel exactly), and torch::matmul([1,3,3], [N,3,1]), whose cuBLAS kernel sums k = 0, 1, 2 in order.
__global__ void __launch_bounds__(128)
camera_rays_kernel(int out_h, int out_w, float end_i, float step_i, float end_j, float step_j, const float* __restrict__ pose,
                   const float* __restrict__ intri, const float* __restrict__ dist_params, float* __restrict__ rays_o,
                   float* __restrict__ rays_d) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= out_h * out_w) return;
  const int a = r / out_w, b = r - a * out_w;
  const float pi = fadd(linspace_at(end_i, step_i, out_h, a), .5f), pj = fadd(linspace_at(end_j, step_j, out_w, b), .5f);
  const float fx = __ldg(intri), cx = __ldg(intri + 2), fy = __ldg(intri + 4), cy = __ldg(intri + 5);
  const float u0 = fmul(fsub(pj, cx), frcp(fx)), v0 = fmul(fsub(pi, cy), frcp(fy));
  float u, v;
  undistort(load_dist(dist_params), u0, v0, u, v);
  const float nv = -v;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    rays_d[size_t(r) * 3 + k] = fsub(ffma(__ldg(pose + 4 * k + 1), nv, fmul(__ldg(pose + 4 * k), u)), __ldg(pose + 4 * k + 2));
    rays_o[size_t(r) * 3 + k] = __ldg(pose + 4 * k + 3);
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

// Lens rays (DESIGN.md §3o).  Angles are carried in half-turns so that sincospi never rounds pi; everything up to the stores is
// float64, with the fmas written out, and each output is rounded to fp32 once.  The equirectangular directions are one function
// that the ODS model calls with the same arguments, so ODS at ipd 0 reproduces them bit for bit.
__device__ __forceinline__ void equirect_dir(int a, int b, int height, int width, double hfov, double vfov, double& x, double& y,
                                             double& z, double& sin_lam, double& cos_lam) {
  const double lam = __ddiv_rn(__dmul_rn(hfov, double(2 * b + 1 - width)), __dmul_rn(360., double(width)));    // half-turns
  const double phi = __ddiv_rn(__dmul_rn(vfov, double(height - 2 * a - 1)), __dmul_rn(360., double(height)));
  double sin_phi, cos_phi;
  sincospi(lam, &sin_lam, &cos_lam);
  sincospi(phi, &sin_phi, &cos_phi);
  x = __dmul_rn(cos_phi, sin_lam);
  y = sin_phi;
  z = -__dmul_rn(cos_phi, cos_lam);
}

template <int Model>
__global__ void __launch_bounds__(128)
lens_rays_kernel(int n, int height, int width, double p0, double p1, double p2, const float* __restrict__ pose,
                 float* __restrict__ rays_o, float* __restrict__ rays_d, uint8_t* __restrict__ valid) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const int hw = height * width;
  const int eye = Model == F2B_LENS_ODS ? r / hw : 0;                 // ODS: 0 = left (top half), 1 = right
  const int q = r - eye * hw;
  const int a = q / width, b = q - a * width;
  double x, y, z, sin_lam = 0., cos_lam = 1.;
  bool ok = true;
  if (Model == F2B_LENS_FISHEYE) {
    // twice the pixel offset, an integer: the circle test r <= min(H, W) / 2 (theta <= fov / 2) is exact
    const int64_t X = 2 * int64_t(b) + 1 - width, Y = 2 * int64_t(a) + 1 - height, m = height < width ? height : width;
    ok = uint64_t(X * X) + uint64_t(Y * Y) <= uint64_t(m * m);
    const double px = 0.5 * double(X), py = 0.5 * double(Y);
    const double rad = sqrt(__fma_rn(px, px, __dmul_rn(py, py)));
    if (rad == 0.) {
      x = 0.; y = 0.; z = -1.;
    } else {
      double s, c;
      sincospi(__ddiv_rn(__dmul_rn(rad, p0), __dmul_rn(180., double(m))), &s, &c);   // theta = r / f in half-turns
      x = __dmul_rn(s, __ddiv_rn(px, rad));
      y = -__dmul_rn(s, __ddiv_rn(py, rad));
      z = -c;
    }
  } else {
    equirect_dir(a, b, height, width, p0, p1, x, y, z, sin_lam, cos_lam);
  }
  double off[3] = {0., 0., 0.};
  if (Model == F2B_LENS_ODS) {
    const double h = eye ? 0.5 * p2 : -0.5 * p2;                      // s ipd / 2, the eye on the viewing circle
    off[0] = __dmul_rn(h, cos_lam);
    off[2] = __dmul_rn(h, sin_lam);
  }
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const double r0 = __ldg(pose + 4 * k), r1 = __ldg(pose + 4 * k + 1), r2 = __ldg(pose + 4 * k + 2);
    const double t = __ldg(pose + 4 * k + 3);
    const double d = __fma_rn(r0, x, __fma_rn(r1, y, __dmul_rn(r2, z)));
    rays_d[size_t(r) * 3 + k] = ok ? __double2float_rn(d) : 0.f;
    rays_o[size_t(r) * 3 + k] =
        Model == F2B_LENS_ODS && p2 != 0. ? __double2float_rn(__dadd_rn(t, __fma_rn(r0, off[0], __dmul_rn(r2, off[2])))) : float(t);
  }
  valid[r] = ok;
}

}  // namespace f2b

using namespace f2b;

extern "C" int f2b_lens_rays(int model, const float* pose, int height, int width, double p0, double p1, double p2,
                             float* rays_o, float* rays_d, uint8_t* valid, void* stream) {
  F2B_REQUIRE(pose && rays_o && rays_d && valid, "f2b_lens_rays: null pointer");
  F2B_REQUIRE(model == F2B_LENS_EQUIRECT || model == F2B_LENS_FISHEYE || model == F2B_LENS_ODS, "f2b_lens_rays: unknown model %d",
              model);
  F2B_REQUIRE(height >= 1 && width >= 1, "f2b_lens_rays: size %dx%d", height, width);
  const int64_t n = int64_t(model == F2B_LENS_ODS ? 2 : 1) * height * width;
  F2B_REQUIRE(n < (int64_t(1) << 31), "f2b_lens_rays: %lld rays overflow int32", (long long)n);
  if (model == F2B_LENS_FISHEYE) {
    F2B_REQUIRE(isfinite(p0) && p0 > 0. && p0 <= 360., "f2b_lens_rays: fisheye fov %g outside (0, 360]", p0);
  } else {
    F2B_REQUIRE(isfinite(p0) && p0 > 0. && p0 <= 360., "f2b_lens_rays: hfov %g outside (0, 360]", p0);
    F2B_REQUIRE(isfinite(p1) && p1 > 0. && p1 <= 180., "f2b_lens_rays: vfov %g outside (0, 180]", p1);
  }
  if (model == F2B_LENS_ODS) F2B_REQUIRE(isfinite(p2) && p2 >= 0., "f2b_lens_rays: ipd %g must be finite and >= 0", p2);
  const int grid = div_up(n, 128);
  cudaStream_t st = as_stream(stream);
  if (model == F2B_LENS_EQUIRECT)
    lens_rays_kernel<F2B_LENS_EQUIRECT><<<grid, 128, 0, st>>>(int(n), height, width, p0, p1, p2, pose, rays_o, rays_d, valid);
  else if (model == F2B_LENS_FISHEYE)
    lens_rays_kernel<F2B_LENS_FISHEYE><<<grid, 128, 0, st>>>(int(n), height, width, p0, p1, p2, pose, rays_o, rays_d, valid);
  else
    lens_rays_kernel<F2B_LENS_ODS><<<grid, 128, 0, st>>>(int(n), height, width, p0, p1, p2, pose, rays_o, rays_d, valid);
  return check_launch("f2b_lens_rays");
}

extern "C" int f2b_img2world_rays(const float* poses, const float* intri, const float* dist_params, const int* cam_indices,
                                  const int* ij, int n_rays, float* rays_o, float* rays_d, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(poses && intri && dist_params && cam_indices && ij && rays_o && rays_d, "f2b_img2world_rays: null pointer");
  img2world_kernel<<<div_up(n_rays, 128), 128, 0, as_stream(stream)>>>(n_rays, poses, intri, dist_params, cam_indices, ij,
                                                                      rays_o, rays_d);
  return check_launch("f2b_img2world_rays");
}

extern "C" int f2b_camera_rays(const float* pose, const float* intri, const float* dist_params, int height, int width,
                               int out_h, int out_w, float* rays_o, float* rays_d, void* stream) {
  F2B_REQUIRE(pose && intri && dist_params && rays_o && rays_d, "f2b_camera_rays: null pointer");
  F2B_REQUIRE(out_h >= 1 && out_h <= height && out_w >= 1 && out_w <= width, "f2b_camera_rays: grid %dx%d outside image %dx%d",
              out_h, out_w, height, width);
  F2B_REQUIRE(int64_t(out_h) * out_w < (int64_t(1) << 31), "f2b_camera_rays: %d x %d rays overflow int32", out_h, out_w);
  // torch::linspace(0.f, H - 1.f, n): end and step in fp32 on the host, exactly as ATen forms them
  const float end_i = float(height) - 1.f, end_j = float(width) - 1.f;
  const float step_i = linspace_step(height, out_h), step_j = linspace_step(width, out_w);
  const int n = out_h * out_w;
  camera_rays_kernel<<<div_up(n, 128), 128, 0, as_stream(stream)>>>(out_h, out_w, end_i, step_i, end_j, step_j, pose, intri,
                                                                    dist_params, rays_o, rays_d);
  return check_launch("f2b_camera_rays");
}

extern "C" int f2b_gather_pixels(const float* images, const int* cam_indices, const int* ij, int height, int width,
                                 int n, float* out, void* stream) {
  if (n <= 0) return F2B_OK;
  F2B_REQUIRE(images && cam_indices && ij && out && height > 0 && width > 0, "f2b_gather_pixels: bad argument");
  gather_pixels_kernel<<<div_up(n, 256), 256, 0, as_stream(stream)>>>(n, images, cam_indices, ij, height, width, out);
  return check_launch("f2b_gather_pixels");
}
