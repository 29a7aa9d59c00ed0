// crop.cuh — the crop box of a trained scene (DESIGN.md §3n): the one predicate every kernel that crops evaluates.
#pragma once
#include "common.cuh"

namespace f2b {

// A box in the normalised scene frame: b = M (x, y, z, 1), M = box_from_scene [3,4] row-major; a point is inside when
// |b_k| <= 1 for k = 0, 1, 2, and kept when it is inside, or, with invert, when it is not.  Passed to kernels by value.
struct CropBox {
  float m[12];
  int invert;
};

// b_k = fma(M[k][0], x, fma(M[k][1], y, fma(M[k][2], z, M[k][3]))) in this fp32 order; a NaN point is not inside.
__device__ __forceinline__ bool crop_keep(const CropBox& c, float x, float y, float z) {
  bool inside = true;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float* r = c.m + 4 * k;
    inside = inside && (fabsf(ffma(r[0], x, ffma(r[1], y, ffma(r[2], z, r[3])))) <= 1.f);
  }
  return inside != (c.invert != 0);
}

}  // namespace f2b
