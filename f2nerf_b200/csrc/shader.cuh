// shader.cuh — device functions shared by shader.cu (stand-alone operators) and mlp_tc.cu (the same work fused into
// the tensor-core MLP epilogues).  Explicit roundings: both users produce bit-identical rows.
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

// Shader-MLP input row: fp16([1, feat[1..15]] + app_emb[cam] | SH4(dir)) (Renderer.cpp:179-187, SHShader.cpp:23-26,
// identity-encoding cast).  feat[0..15] = the field output (fp16-rounded values), feat[0] is ignored.
__device__ __forceinline__ void shade_row(const float feat[16], const float* __restrict__ emb_row /* nullable */,
                                          float dx, float dy, float dz, uint4 row[4]) {
  float v[32];
#pragma unroll
  for (int k = 0; k < 16; k++) v[k] = feat[k];
  v[0] = 1.f;
  if (emb_row) {
    const float4* e4 = reinterpret_cast<const float4*>(emb_row);
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const float4 a = __ldg(e4 + q);
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
