// common.cuh — shared helpers for the f2nerf_b200 sm_90a kernels (no torch, no Eigen).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/f2nerf_b200.h"

namespace f2b {

// ---- error plumbing (C ABI never throws) -------------------------------------------------
void set_error(const char* fmt, ...);
int  check_launch(const char* what);   // cudaGetLastError -> F2B_ECUDA + message

#define F2B_REQUIRE(cond, ...)                                   \
  do {                                                           \
    if (!(cond)) {                                               \
      f2b::set_error(__VA_ARGS__);                               \
      return F2B_EINVAL;                                         \
    }                                                            \
  } while (0)

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }
static inline int div_up(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }
// CTAs of a persistent kernel that are resident on one SM at once (registers and shared memory decide), at least 1
template <class Kernel>
static inline int resident_per_sm(Kernel kernel, int threads, size_t smem_bytes) {
  int n = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, threads, smem_bytes) != cudaSuccess) n = 1;
  return n > 0 ? n : 1;
}
// grid of a persistent kernel over n_work tiles (or rays): one CTA per tile, at most per_sm CTAs on every SM
static inline int persistent_grid(int n_work, int per_sm) {
  int sms = 132;
  f2b_device_info(&sms, nullptr);
  return n_work < sms * per_sm ? n_work : sms * per_sm;
}

// ---- reference POD layouts (PersSampler.h:15-37), restated without Eigen -------------------
struct __align__(32) TreeNode {      // 64 B
  float center[3];
  float side_len;
  int   parent;
  int   childs[8];
  unsigned char is_leaf_node;        // bool @52 ...
  unsigned char _pad0[3];            // ... + 3 padding bytes the reference never initialises
  int   trans_idx;                   // @56  (<0 => pruned / invalid: the "occupancy bit")
  int   _pad;
};
struct __align__(32) TransInfo {     // 544 B
  float w2xz[12][8];                 // 12 row-major 2x4 projections
  float weight[3][12];               // row-major 3x12 mixing matrix
  float center[3];
  float dis_summary;
};
struct __align__(32) EdgePool {      // 64 B
  int   t_idx_a, t_idx_b;
  float center[3];
  float dir_0[3];
  float dir_1[3];
  int   _pad[5];
};
static_assert(sizeof(TreeNode) == 64, "TreeNode layout");
static_assert(sizeof(TransInfo) == 544, "TransInfo layout");
static_assert(sizeof(EdgePool) == 64, "EdgePool layout");

// ---- explicitly rounded fp32 arithmetic: the compiler may not re-contract these ------------
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float frcp(float a) { return __frcp_rn(a); }
__device__ __forceinline__ float fsqrt(float a) { return __fsqrt_rn(a); }

}  // namespace f2b
