// shader.cuh — device functions shared by the stand-alone operators (shader.cu, composite.cu) and the kernels that fuse
// the same work (the tensor-core MLP epilogues of mlp_tc.cu, fused_fwd.cu).  Explicit roundings: every user produces
// bit-identical values.
#pragma once
#include "common.cuh"
#include <cuda_fp16.h>

namespace f2b {

// degree-4 real spherical harmonics in tiny-cuda-nn ordering (SHShader.cu:32-50).  Explicit roundings, in the
// contraction pattern ptxas chose for the reference TU (-fmad=true; read off the SASS of the reference build):
// o6 = fma(c,z2,-k), o8 = fma(c,x2,-(c*y2)), the inner factors of o9/o11/o12/o13/o15 are single FMAs.  Both users
// (stand-alone operator, fused epilogue) spell out the same sequence => rows bit-identical to the reference kernel's.
__device__ __forceinline__ void sh4(float x, float y, float z, float o[16]) {
  const float xy = fmul(x, y), xz = fmul(x, z), yz = fmul(y, z), x2 = fmul(x, x), y2 = fmul(y, y), z2 = fmul(z, z);
  o[0] = 0.28209479177387814f;
  o[1] = fmul(-0.48860251190291987f, y);
  o[2] = fmul(0.48860251190291987f, z);
  o[3] = fmul(-0.48860251190291987f, x);
  o[4] = fmul(1.0925484305920792f, xy);
  o[5] = fmul(-1.0925484305920792f, yz);
  o[6] = __fmaf_rn(z2, 0.94617469575755997f, -0.31539156525251999f);
  o[7] = fmul(-1.0925484305920792f, xz);
  o[8] = __fmaf_rn(x2, 0.54627421529603959f, -fmul(y2, 0.54627421529603959f));
  o[9] = fmul(fmul(y, 0.59004358992664352f), __fmaf_rn(x2, -3.0f, y2));
  o[10] = fmul(z, fmul(xy, 2.8906114426405538f));
  const float f15 = __fmaf_rn(z2, -5.0f, 1.0f);
  o[11] = fmul(fmul(y, 0.45704579946446572f), f15);
  o[12] = fmul(fmul(z, 0.3731763325901154f), __fmaf_rn(z2, 5.0f, -3.0f));
  o[13] = fmul(f15, fmul(x, 0.45704579946446572f));
  o[14] = fmul(fmul(z, 1.4453057213202769f), fsub(x2, y2));
  o[15] = fmul(fmul(x, 0.59004358992664352f), __fmaf_rn(y2, 3.0f, -x2));
}

// d[16] . d sh4 / d(x, y, z): the gradient of sum_k d[k] o[k] with respect to the direction, from the polynomials of sh4 taken
// with x, y, z independent (the caller chains through the normalisation).  Pose refinement (ray_grad_kernel, DESIGN §3k).
__device__ __forceinline__ void sh4_grad(float x, float y, float z, const float d[16], float g[3]) {
  const float xy = fmul(x, y), xz = fmul(x, z), yz = fmul(y, z), x2 = fmul(x, x), y2 = fmul(y, y), z2 = fmul(z, z);
  const float c1 = 0.48860251190291987f, c4 = 1.0925484305920792f, c9 = 0.59004358992664352f, c10 = 2.8906114426405538f;
  const float c11 = 0.45704579946446572f, c12 = 0.3731763325901154f, c14 = 1.4453057213202769f;
  const float f15 = __fmaf_rn(z2, -5.0f, 1.0f);                   // 1 - 5 z^2
  const float q9 = fmul(3.f * c9, fsub(y2, x2));                   // d o9 / dy = d o15 / dx = 3 c9 (y^2 - x^2)
  float gx = fmul(-c1, d[3]);
  gx = ffma(fmul(c4, y), d[4], gx);
  gx = ffma(fmul(-c4, z), d[7], gx);
  gx = ffma(fmul(2.f * 0.54627421529603959f, x), d[8], gx);
  gx = ffma(fmul(-6.f * c9, xy), d[9], gx);
  gx = ffma(fmul(c10, yz), d[10], gx);
  gx = ffma(fmul(c11, f15), d[13], gx);
  gx = ffma(fmul(2.f * c14, xz), d[14], gx);
  gx = ffma(q9, d[15], gx);
  float gy = fmul(-c1, d[1]);
  gy = ffma(fmul(c4, x), d[4], gy);
  gy = ffma(fmul(-c4, z), d[5], gy);
  gy = ffma(fmul(-2.f * 0.54627421529603959f, y), d[8], gy);
  gy = ffma(q9, d[9], gy);
  gy = ffma(fmul(c10, xz), d[10], gy);
  gy = ffma(fmul(c11, f15), d[11], gy);
  gy = ffma(fmul(-2.f * c14, yz), d[14], gy);
  gy = ffma(fmul(6.f * c9, xy), d[15], gy);
  float gz = fmul(c1, d[2]);
  gz = ffma(fmul(-c4, y), d[5], gz);
  gz = ffma(fmul(2.f * 0.94617469575755997f, z), d[6], gz);
  gz = ffma(fmul(-c4, x), d[7], gz);
  gz = ffma(fmul(c10, xy), d[10], gz);
  gz = ffma(fmul(-10.f * c11, yz), d[11], gz);
  gz = ffma(fmul(c12, __fmaf_rn(z2, 15.f, -3.f)), d[12], gz);
  gz = ffma(fmul(-10.f * c11, xz), d[13], gz);
  gz = ffma(fmul(c14, fsub(x2, y2)), d[14], gz);
  g[0] = gx; g[1] = gy; g[2] = gz;
}

// Shader-MLP input row: fp16([1, feat[1..15]] + app_emb[cam] | SH4(dir)) (Renderer.cpp:179-187, SHShader.cpp:23-26,
// identity-encoding cast).  feat[0..15] = the field output (fp16-rounded values), feat[0] is ignored.  kSharedEmb: emb_row
// points to shared memory (the fused forward stages its one row per CTA) and is read with plain loads; same adds, same bits.
template <bool kSharedEmb>
__device__ __forceinline__ void shade_row_t(const float feat[16], const float* __restrict__ emb_row /* nullable */,
                                            float dx, float dy, float dz, uint4 row[4]) {
  float v[32];
#pragma unroll
  for (int k = 0; k < 16; k++) v[k] = feat[k];
  v[0] = 1.f;
  if (emb_row) {
    const float4* e4 = reinterpret_cast<const float4*>(emb_row);
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const float4 a = kSharedEmb ? e4[q] : __ldg(e4 + q);
      v[4 * q] = fadd(v[4 * q], a.x); v[4 * q + 1] = fadd(v[4 * q + 1], a.y);
      v[4 * q + 2] = fadd(v[4 * q + 2], a.z); v[4 * q + 3] = fadd(v[4 * q + 3], a.w);
    }
  }
  sh4(dx, dy, dz, v + 16);
#pragma unroll
  for (int q = 0; q < 4; q++) {
    __half2 h[4];
#pragma unroll
    for (int k = 0; k < 4; k++) h[k] = __floats2half2_rn(v[8 * q + 2 * k], v[8 * q + 2 * k + 1]);
    row[q] = *reinterpret_cast<uint4*>(h);
  }
}

__device__ __forceinline__ void shade_row(const float feat[16], const float* __restrict__ emb_row /* nullable */,
                                          float dx, float dy, float dz, uint4 row[4]) {
  shade_row_t<false>(feat, emb_row, dx, dy, dz, row);
}

// rgb = (1 + 2e-3) / (1 + exp(-o)) - 1e-3 on the fp16 MLP output (SHShader.cpp:27-28)
__device__ __forceinline__ float shade_act(float o) {
  const float eps = 1e-3f;
  const float c = 1.f + 2.f * eps;
  return fsub(fdiv(c, fadd(1.f, expf(-o))), eps);
}

// backward of shade_act for one channel: loss_scale * d_rgb * (1 + 2e-3) * sigmoid'(o)   (fp32, rounded to fp16 by the caller)
__device__ __forceinline__ float shade_act_bwd(float o, float d_rgb, float loss_scale) {
  const float c = 1.f + 2.f * 1e-3f;
  const float s = fdiv(1.f, fadd(1.f, expf(-o)));
  return fmul(fmul(fmul(fmul(d_rgb, c), s), fsub(1.f, s)), loss_scale);
}

}  // namespace f2b
