// tc.cuh — minimal hand-written wgmma layer for sm_90a (no CUTLASS).
//
// Conventions:
//  * shared-memory matrix descriptor (64 bit): [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 |
//    [49,52) base_offset | [62,64) layout (0 none, 1 SW128, 2 SW64, 3 SW32)
//  * K-major operand tiles are stored as rows of 32/64/128 bytes with the matching 32B/64B/128B
//    swizzle: 16-byte chunk c of row r lands at chunk c ^ f(r) (f = (r>>2)&1 / (r>>1)&3 / r&7); tiles
//    are 1024-byte aligned; 8-row groups are SBO bytes apart; advancing K by 16 elements = +32 bytes
//    on the start address (the hardware swizzles on address bits).  An MN-major operand is the same
//    kind of tile read the other way: its rows run along K, each row holds the (<= one swizzle atom of)
//    M or N elements, 16 rows = one K step.
//  * a CTA of 128 threads (one warpgroup) owns a 128-row tile; D[128 x N] is two m64 wgmma halves whose
//    fp32 accumulators live in registers (Acc<N>).  Thread t of the warpgroup holds, in half h, element i
//    at row 64h + 16(t/32) + (t%32)/4 + 8((i/2)%2), column 8(i/4) + 2(t%4) + i%2 (acc_row / acc_col).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace f2b { namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

enum : uint64_t { kLayoutNone = 0, kLayoutSW128 = 1, kLayoutSW64 = 2, kLayoutSW32 = 3 };

__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint64_t layout) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) |
         (layout << 62);
}
__device__ __forceinline__ uint64_t layout_of(int row_bytes) {
  return row_bytes == 128 ? kLayoutSW128 : (row_bytes == 64 ? kLayoutSW64 : kLayoutSW32);
}
// K-major tile with `row_bytes` (32/64/128) per row and the matching swizzle
__device__ __forceinline__ uint64_t kmajor_desc(uint32_t saddr, int row_bytes) {
  return make_desc(saddr, 16, 8 * row_bytes, layout_of(row_bytes));
}
// MN-major operand: tile of [k rows][row_bytes] with matching swizzle; k-step = 16 rows
__device__ __forceinline__ uint64_t mnmajor_desc(uint32_t tile, int row_bytes, int k_step) {
  return make_desc(tile + k_step * 16 * row_bytes, 16, 8 * row_bytes, layout_of(row_bytes));
}

// byte offset of 16-byte chunk `c` of row `r` inside a swizzled K-major tile
__device__ __forceinline__ uint32_t sw128_off(int r, int c) { return r * 128 + ((c ^ (r & 7)) << 4); }
__device__ __forceinline__ uint32_t sw64_off(int r, int c) { return r * 64 + ((c ^ ((r >> 1) & 3)) << 4); }
__device__ __forceinline__ uint32_t sw32_off(int r, int c) { return r * 32 + ((c ^ ((r >> 2) & 1)) << 4); }
// byte offset of fp16 column `col` (even) of row `r` inside a [rows x 64] SW128 tile
__device__ __forceinline__ uint32_t sw128_col(int r, int col) { return sw128_off(r, col >> 3) + ((col & 7) << 1); }

// generic-proxy smem writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma ----------------------------------------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x N] (+)= A[64 x 16] . B[16 x N], both operands in shared memory; TA / TB: operand is MN-major
template <int N, int TA, int TB> struct Wgmma;

#define F2B_WGMMA_HEAD(N)                                                                                       \
  "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #N ", 0;\n\t"
template <int TA, int TB> struct Wgmma<16, TA, TB> {
  static __device__ __forceinline__ void run(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(F2B_WGMMA_HEAD(10)
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};
template <int TA, int TB> struct Wgmma<32, TA, TB> {
  static __device__ __forceinline__ void run(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(F2B_WGMMA_HEAD(18)
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15},"
                 " %16, %17, p, 1, 1, %19, %20;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};
template <int TA, int TB> struct Wgmma<64, TA, TB> {
  static __device__ __forceinline__ void run(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(F2B_WGMMA_HEAD(34)
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};
#undef F2B_WGMMA_HEAD

// accumulators of a [128 x N] tile (two m64 halves) / of a [64 x N] tile
template <int N> struct Acc { float d[2][N / 2]; };
template <int N> struct Acc64 { float d[N / 2]; };

__device__ __forceinline__ int acc_row(int t, int half, int i) { return 64 * half + 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int acc_col(int t, int i) { return 8 * (i >> 2) + 2 * (t & 3) + (i & 1); }

// D[128 x N] (+)= A[128 x 16*KS] . B: A a K-major tile (a_row_bytes per row); B a K-major tile (TB = 0, b_row_bytes per
// row, N rows) or an MN-major one (TB = 1, 16 rows per K step).  Issue only: wg_commit + wg_wait complete it.
template <int N, int TB, int KS>
__device__ __forceinline__ void mma_m128(Acc<N>& acc, uint32_t a, int a_row_bytes, uint32_t b, int b_row_bytes, bool accumulate) {
#pragma unroll
  for (int k = 0; k < KS; k++) {
    const uint64_t bd = TB ? mnmajor_desc(b, b_row_bytes, k) : kmajor_desc(b + 32 * k, b_row_bytes);
    const uint32_t on = (k > 0 || accumulate) ? 1u : 0u;
    Wgmma<N, 0, TB>::run(acc.d[0], kmajor_desc(a + 32 * k, a_row_bytes), bd, on);
    Wgmma<N, 0, TB>::run(acc.d[1], kmajor_desc(a + 64 * a_row_bytes + 32 * k, a_row_bytes), bd, on);
  }
}
// D[64 x N] += A^T . B over a 128-row batch: both operands MN-major views of [128 x M] / [128 x N] tiles (batch reduction)
template <int N>
__device__ __forceinline__ void mma_batch128(Acc64<N>& acc, uint32_t a, int a_row_bytes, uint32_t b, int b_row_bytes) {
#pragma unroll
  for (int k = 0; k < 8; k++) Wgmma<N, 1, 1>::run(acc.d, mnmajor_desc(a, a_row_bytes, k), mnmajor_desc(b, b_row_bytes, k), 1u);
}

// accumulator -> ReLU -> fp16 -> the [128 x 64] SW128 operand tile
__device__ __forceinline__ void acc_relu_to_tile(const Acc<64>& acc, unsigned char* h_tile, int t) {
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const __half2 v = __floats2half2_rn(fmaxf(acc.d[h][i], 0.f), fmaxf(acc.d[h][i + 1], 0.f));
      *reinterpret_cast<__half2*>(h_tile + sw128_col(acc_row(t, h, i), acc_col(t, i))) = v;
    }
}

// accumulator -> fp32 rows [128][ld] in shared memory (ld = 20 for N = 16: conflict-free float4 row reads)
template <int N>
__device__ __forceinline__ void acc_to_rows(const Acc<N>& acc, float* rows, int ld, int t) {
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int i = 0; i < N / 2; i += 2)
      *reinterpret_cast<float2*>(rows + acc_row(t, h, i) * ld + acc_col(t, i)) = make_float2(acc.d[h][i], acc.d[h][i + 1]);
}
// 16 fp32 of row `row` of such rows (as bits)
__device__ __forceinline__ void row_ld16(const float* rows, int ld, int row, uint32_t (&r)[16]) {
  const uint4* src = reinterpret_cast<const uint4*>(rows + row * ld);
#pragma unroll
  for (int q = 0; q < 4; q++) reinterpret_cast<uint4*>(r)[q] = src[q];
}
constexpr int kRowLd16 = 20;

}}  // namespace f2b::tc
