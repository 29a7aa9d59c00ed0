/* camera_rays.c — CPU restatement of the reference's whole-camera rays (TEST INFRASTRUCTURE ONLY, like f2_oracle.c):
 * Dataset::RaysOfCamera / RaysFromPose -> Dataset::Img2WorldRay (src/Dataset/Dataset.cpp:152-218), the ATen sequence as the GPU
 * runs it, every fp32 operation and fma explicit (compiled with -ffp-contract=off):
 *  - torch::linspace(0, end, n) (ATen's RangeFactories.cu, two-sided): step = end / (n - 1) in fp32 on the host; index k < n/2
 *    gives start + step*k (= step*k), the rest end - step*(n-1-k), which nvcc contracts into one fma; n == 1 gives start;
 *  - i + .5f, j + .5f (:157-158);
 *  - (j - cx) / fx and -(i - cy) / fy (:165): ATen's CUDA division by a CPU scalar multiplies by the fp32 reciprocal 1.f / fx
 *    (div_true_kernel_cuda); the negation there and the one in CameraUndistort (Dataset.cu:85) cancel exactly;
 *  - CameraUndistortKernel (Dataset.cu:71-76) -> iterative_camera_undistortion (:30-69), with the contractions ptxas makes in
 *    the reference build (the same as in Img2WorldRayKernel, which f2_oracle.c's orc_img2world_rays restates);
 *  - torch::matmul([1,3,3], [N,3,1]) (:169): cuBLAS's strided-batched gemv sums k = 0, 1, 2 in order, fma(p1, -v, p0*u) - p2.
 * Built into oracle/libcamrays_oracle.so; bound by tests/camera_rays_oracle.py. */
#include <math.h>
#include <stddef.h>

/* apply_camera_distortion (Dataset.cu:14-27) as compiled */
static void distort(const float* dp, float two_p1, float two_p2, float u, float v, float u2, float uv, float v2, float r2,
                    float* du, float* dv) {
  const float radial = fmaf(r2, dp[0], r2 * (r2 * dp[1]));
  *du = fmaf(fmaf(u2, 2.f, r2), dp[3], fmaf(uv, two_p1, u * radial));
  *dv = fmaf(fmaf(v2, 2.f, r2), dp[2], fmaf(v, radial, uv * two_p2));
}

/* iterative_camera_undistortion (Dataset.cu:30-69) of the OpenCV-style point (u0, v0) */
static void undistort(const float* dp, float u0, float v0, float* u_out, float* v_out) {
  const float two_p1 = dp[2] + dp[2], two_p2 = dp[3] + dp[3];
  float u = u0, v = v0;
  for (int it = 0; it < 100; it++) {
    const float s0 = fmaxf(fabsf(u * 1e-6f), 1.1920929e-7f), s1 = fmaxf(fabsf(v * 1e-6f), 1.1920929e-7f);
    const float u2 = u * u, uv = u * v, v2 = v * v;
    float du, dv, b0x, b0y, f0x, f0y, b1x, b1y, f1x, f1y, a, a2;
    distort(dp, two_p1, two_p2, u, v, u2, uv, v2, u2 + v2, &du, &dv);
    a = u - s0; a2 = a * a; distort(dp, two_p1, two_p2, a, v, a2, v * a, v2, v2 + a2, &b0x, &b0y);
    a = u + s0; a2 = a * a; distort(dp, two_p1, two_p2, a, v, a2, v * a, v2, v2 + a2, &f0x, &f0y);
    a = v - s1; a2 = a * a; distort(dp, two_p1, two_p2, u, a, u2, u * a, a2, u2 + a2, &b1x, &b1y);
    a = v + s1; a2 = a * a; distort(dp, two_p1, two_p2, u, a, u2, u * a, a2, u2 + a2, &f1x, &f1y);
    const float two_s0 = s0 + s0, two_s1 = s1 + s1;
    const float j00 = (f0x - b0x) / two_s0 + 1.f, j01 = (f1x - b1x) / two_s1;
    const float j10 = (f0y - b0y) / two_s0, j11 = (f1y - b1y) / two_s1 + 1.f;
    const float inv = 1.f / fmaf(j00, j11, -(j10 * j01));                 /* Eigen 2x2 inverse, mul+sub fused */
    const float rx = (u + du) - u0, ry = (v + dv) - v0;
    const float sx = fmaf(j11 * inv, rx, -((inv * j01) * ry));
    const float sy = fmaf(j00 * inv, ry, -((inv * j10) * rx));
    u = u - sx; v = v - sy;
    if (fmaf(sx, sx, sy * sy) < 1e-10f) break;                           /* squaredNorm() < kMaxStepNorm */
  }
  *u_out = u; *v_out = v;
}

static float linspace_at(float end, float step, int n, int k) {
  if (n == 1) return 0.f;
  if (k < n / 2) return step * (float)k;
  return fmaf(-step, (float)(n - 1 - k), end);
}

/* pose [12], intri [9], dist [4] of one camera.  idx: the n_idx ray indices a*out_w + b to compute, or NULL for all
 * out_h*out_w of them; rays_o / rays_d [n,3] in that order. */
void orc_camera_rays(const float* pose, const float* intri, const float* dist, int height, int width, int out_h, int out_w,
                     const int* idx, int n_idx, float* rays_o, float* rays_d) {
  const float end_i = (float)height - 1.f, end_j = (float)width - 1.f;
  const float step_i = out_h > 1 ? end_i / (float)(out_h - 1) : 0.f, step_j = out_w > 1 ? end_j / (float)(out_w - 1) : 0.f;
  const float rfx = 1.f / intri[0], rfy = 1.f / intri[4], cx = intri[2], cy = intri[5];
  const int n = idx ? n_idx : out_h * out_w;
#pragma omp parallel for schedule(static)
  for (int q = 0; q < n; q++) {
    const int r = idx ? idx[q] : q, a = r / out_w, b = r - a * out_w;
    const float pi = linspace_at(end_i, step_i, out_h, a) + .5f, pj = linspace_at(end_j, step_j, out_w, b) + .5f;
    float u, v;
    undistort(dist, (pj - cx) * rfx, (pi - cy) * rfy, &u, &v);
    const float nv = -v;
    for (int k = 0; k < 3; k++) {
      rays_d[(size_t)q * 3 + k] = fmaf(pose[4 * k + 1], nv, pose[4 * k] * u) - pose[4 * k + 2];
      rays_o[(size_t)q * 3 + k] = pose[4 * k + 3];
    }
  }
}
