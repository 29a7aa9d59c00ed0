// hash.cuh — device functions of the anchored hash-grid encode shared by hash.cu (stand-alone encode)
// and field.cu (encode fused in front of the wgmma MLP).  See hash.cu for the design notes.
#pragma once
#include "common.cuh"

namespace f2b {

__device__ __forceinline__ float level_scale(int l) {
  // exp2f((10-3)*float(l)/15 + 3): cvt(7*l) ; div.rn 15 ; add 3 ; ex2.approx  (Hash3DAnchored.cu:29)
  return exp2f(fadd(fdiv((float)(7 * l), 15.f), 3.f));
}

struct Corner8 {
  unsigned idx[8];   // order 000,001,010,011,100,101,110,111 (z fastest)
  float w[8];
  unsigned cell[3];  // integer cell coordinates (exact run key for the backward's merging)
};

// index/weight computation shared by forward and backward (Hash3DAnchored.cu:27-66)
__device__ __forceinline__ void corners(float x0, float x1, float x2, float scale,
                                        const int* __restrict__ prim, const float* __restrict__ bias,
                                        unsigned local_size, Corner8& c) {
  const float px = ffma(x0, scale, __ldg(bias)), py = ffma(x1, scale, __ldg(bias + 1)),
              pz = ffma(x2, scale, __ldg(bias + 2));
  const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
  const unsigned ix = (unsigned)fx, iy = (unsigned)fy, iz = (unsigned)fz;   // cvt.rzi.u32.f32 (saturating)
  c.cell[0] = ix; c.cell[1] = iy; c.cell[2] = iz;
  const unsigned pa = (unsigned)__ldg(prim), pb = (unsigned)__ldg(prim + 1), pc = (unsigned)__ldg(prim + 2);
  const unsigned hx0 = ix * pa, hx1 = hx0 + pa, hy0 = iy * pb, hy1 = hy0 + pb, hz0 = iz * pc, hz1 = hz0 + pc;
  const bool pow2 = (local_size & (local_size - 1)) == 0;
  const unsigned mask = local_size - 1;
#define F2B_MOD(v) (pow2 ? ((v) & mask) : ((v) % local_size))
  c.idx[0] = F2B_MOD(hx0 ^ hy0 ^ hz0);
  c.idx[1] = F2B_MOD(hx0 ^ hy0 ^ hz1);
  c.idx[2] = F2B_MOD(hx0 ^ hy1 ^ hz0);
  c.idx[3] = F2B_MOD(hx0 ^ hy1 ^ hz1);
  c.idx[4] = F2B_MOD(hx1 ^ hy0 ^ hz0);
  c.idx[5] = F2B_MOD(hx1 ^ hy0 ^ hz1);
  c.idx[6] = F2B_MOD(hx1 ^ hy1 ^ hz0);
  c.idx[7] = F2B_MOD(hx1 ^ hy1 ^ hz1);
#undef F2B_MOD
  const float a = fsub(px, fx), b = fsub(py, fy), cc = fsub(pz, fz);
  const float na = fsub(1.f, a), nb = fsub(1.f, b), nc = fsub(1.f, cc);
  const float nanb = fmul(na, nb), nab = fmul(na, b), anb = fmul(a, nb), ab = fmul(a, b);
  c.w[0] = fmul(nanb, nc); c.w[1] = fmul(cc, nanb);
  c.w[2] = fmul(nab, nc);  c.w[3] = fmul(nab, cc);
  c.w[4] = fmul(anb, nc);  c.w[5] = fmul(cc, anb);
  c.w[6] = fmul(ab, nc);   c.w[7] = fmul(ab, cc);
}

__device__ __forceinline__ uint32_t ldg_nc_u32(const void* p) {
  uint32_t v;
  asm volatile("ld.global.nc.b32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}

// Encode one sample at one level: returns the two blended channels packed as half2 bits.
__device__ __forceinline__ uint32_t encode_level(const __half* __restrict__ table, int l, int local_size,
                                                 const Corner8& c) {
  const __half* base = table + size_t(l) * local_size;         // HALF-element offset: levels overlap (quirk)
  uint32_t raw[8];
#pragma unroll
  for (int k = 0; k < 8; k++) raw[k] = ldg_nc_u32(base + size_t(c.idx[k]) * 2);
  float2 f[8];
#pragma unroll
  for (int k = 0; k < 8; k++) f[k] = __half22float2(*reinterpret_cast<const __half2*>(&raw[k]));
  float a0 = fmul(c.w[1], f[1].x), a1 = fmul(c.w[1], f[1].y);
  a0 = ffma(c.w[0], f[0].x, a0); a1 = ffma(c.w[0], f[0].y, a1);
#pragma unroll
  for (int k = 2; k < 8; k++) { a0 = ffma(c.w[k], f[k].x, a0); a1 = ffma(c.w[k], f[k].y, a1); }
  const __half2 h = __floats2half2_rn(a0, a1);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// Encode all 16 levels of one sample into 16 half2 words (registers).  Shared with field.cu.
// `scales` = the 16 level scales computed AT RUN TIME (shared memory): a compile-time-folded exp2f
// would be correctly rounded, MUFU.EX2 (what the reference executes) is not.
__device__ __forceinline__ void encode_point(const __half* __restrict__ table,
                                             const int* __restrict__ prim_pool,
                                             const float* __restrict__ bias_pool, int n_volumes,
                                             int local_size, const float* scales, float p0, float p1,
                                             float p2, int v, uint32_t out[16]) {
  const float x0 = fmul(fadd(p0, 1.f), .5f), x1 = fmul(fadd(p1, 1.f), .5f), x2 = fmul(fadd(p2, 1.f), .5f);
#pragma unroll
  for (int l = 0; l < F2B_N_LEVELS; l++) {
    const int tv = l * n_volumes + v;
    Corner8 c;
    corners(x0, x1, x2, scales[l], prim_pool + tv * 3, bias_pool + tv * 3, (unsigned)local_size, c);
    out[l] = encode_level(table, l, local_size, c);
  }
}

}  // namespace f2b
