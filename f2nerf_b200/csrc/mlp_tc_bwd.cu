// mlp_tc_bwd.cu — MLP backward on Hopper wgmma tensor cores (impl 1).
//
// Replaces kernel_mlp_fused_backward (External/tiny-cuda-nn/src/fully_fused_mlp.cu:150-259), the CUTLASS
// dL/dinput GEMM (:832-835) and the three split-K weight-gradient GEMMs on side streams (:785,819,828)
// with ONE persistent kernel per call (one warpgroup per CTA).  Per 128-sample tile:
//   activation gradients  dH = dOut.Wout, dH0 = dH1.Wh, dIn = dH0.W0   — two m64 wgmmas, A = K-major tile of the
//       gradient rows, B = the weight matrix used as MN-major operand straight from its row-major layout
//       (no transposed weight copies);
//   weight gradients      dW = dAct^T . Act  — batch-reduction wgmmas with K = the 128 samples of the tile:
//       both operands MN-major views of the very same shared-memory tiles, M = 64 output rows, fp32
//       accumulators that stay resident in registers across all tiles of the CTA and are flushed once with
//       atomicAdd at the end (no split-K workspace, no fp16 accumulation, no reduction kernels).
#include "common.cuh"
#include "hash.cuh"
#include "tc.cuh"

namespace f2b {
using namespace tc;

constexpr int kBT = 128;   // tile rows

// Shared memory: resident weights, then TWO stages of per-tile operands (double-buffered cp.async prefetch).
// The activation gradients overwrite the activations they mask in place (dH1 over H1, dH0 over H0): every MMA
// that still needs the forward activation as an operand is issued in the step BEFORE the overwrite.
template <int NH>
struct BwdSmem {
  static constexpr int W0 = 0;                              // [64 x 32]  SW64   4 KB   (B operand, MN-major, K = out row)
  static constexpr int WH = 4096;                           // [64 x 64]  SW128  8 KB   (NH only)
  static constexpr int WO = NH ? 12288 : 4096;              // [16 x 64]  SW128  2 KB
  static constexpr int STAGE0 = WO + 2048;
  static constexpr int DO = 0;                              // stage-relative: [128 x 16] SW32   4 KB
  static constexpr int X = 4096;                            //                 [128 x 32] SW64   8 KB
  static constexpr int H0 = 12288;                          //                 [128 x 64] SW128 16 KB (becomes dH0)
  static constexpr int H1 = 28672;                          //                 [128 x 64] SW128 16 KB (becomes dH1; NH only)
  static constexpr int STAGE_BYTES = NH ? 45056 : 28672;
  static constexpr int BYTES = STAGE0 + 2 * STAGE_BYTES + 1024;
};

__device__ __forceinline__ uint32_t pk(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <int K>
__device__ __forceinline__ void stage_w(const __half* __restrict__ w, int rows, unsigned char* dst) {
  constexpr int chunks = K / 8;
  for (int i = threadIdx.x; i < rows * chunks; i += blockDim.x) {
    const int r = i / chunks, c = i % chunks;
    *reinterpret_cast<uint4*>(dst + (K == 64 ? sw128_off(r, c) : sw64_off(r, c))) = *reinterpret_cast<const uint4*>(w + r * K + c * 8);
  }
}

__device__ __forceinline__ void cp16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

// One tile's operand rows (dOut 32 B, x 64 B, h0 128 B, h1 128 B per sample; each a contiguous block in global
// memory) -> swizzled tiles of one stage, 16 B per thread and pass, linear sweep = full 128 B lines.
template <int NH>
__device__ __forceinline__ void prefetch_tile(const __half* __restrict__ dout, const __half* __restrict__ in,
                                              const __half* __restrict__ hidden, const __half* __restrict__ hid_last,
                                              int tile, int n_pts, uint32_t stage) {
  using S = BwdSmem<NH>;
  const int rows = min(kBT, n_pts - tile * kBT);
  const size_t t0 = size_t(tile) * kBT;
  const unsigned char* s_do = reinterpret_cast<const unsigned char*>(dout + t0 * 16);
  const unsigned char* s_x = reinterpret_cast<const unsigned char*>(in + t0 * 32);
  const unsigned char* s_h0 = reinterpret_cast<const unsigned char*>(hidden + t0 * 64);
  const unsigned char* s_h1 = reinterpret_cast<const unsigned char*>(hid_last + t0 * 64);
#pragma unroll
  for (int j = 0; j < 2; j++) {
    const int c = threadIdx.x + kBT * j, r = c >> 1;
    const bool ok = r < rows;
    cp16(stage + S::DO + sw32_off(r, c & 1), s_do + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
  }
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int c = threadIdx.x + kBT * j, r = c >> 2;
    const bool ok = r < rows;
    cp16(stage + S::X + sw64_off(r, c & 3), s_x + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
  }
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int c = threadIdx.x + kBT * j, r = c >> 3;
    const bool ok = r < rows;
    cp16(stage + S::H0 + sw128_off(r, c & 7), s_h0 + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
    if (NH) cp16(stage + S::H1 + sw128_off(r, c & 7), s_h1 + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
  }
}

// masked epilogue: acc * [h > 0] -> fp16 dH tile (SW128); h_tile may be dh_tile (each element is read, then written, by one thread)
__device__ __forceinline__ void relu_bwd_epilogue(const Acc<64>& acc, const unsigned char* h_tile, unsigned char* dh_tile, int t) {
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const uint32_t off = sw128_col(acc_row(t, h, i), acc_col(t, i));
      const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(h_tile + off));
      *reinterpret_cast<uint32_t*>(dh_tile + off) = pk(hf.x > 0.f ? acc.d[h][i] : 0.f, hf.y > 0.f ? acc.d[h][i + 1] : 0.f);
    }
}

// dIn rows of the tile -> global fp16 [P,32]
__device__ __forceinline__ void store_din(const Acc<32>& acc, __half* __restrict__ din, int tile, int n_pts, int t) {
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int i = 0; i < 16; i += 2) {
      const int p = tile * kBT + acc_row(t, h, i);
      if (p < n_pts) *reinterpret_cast<uint32_t*>(din + size_t(p) * 32 + acc_col(t, i)) = pk(acc.d[h][i], acc.d[h][i + 1]);
    }
}

// weight-gradient accumulators (rows = output features) -> dparams with atomicAdd; dWout is held transposed
template <int NH>
__device__ __forceinline__ void flush_weight_grads(const Acc64<32>& gw0, const Acc64<16>& gwo, const Acc64<64>& gwh,
                                                   float* __restrict__ dparams, int t) {
  float* g0 = dparams;
  float* gh = dparams + 64 * 32;
  float* go = gh + NH * 64 * 64;
#pragma unroll
  for (int i = 0; i < 16; i++) atomicAdd(g0 + acc_row(t, 0, i) * 32 + acc_col(t, i), gw0.d[i]);
#pragma unroll
  for (int i = 0; i < 8; i++) atomicAdd(go + acc_col(t, i) * 64 + acc_row(t, 0, i), gwo.d[i]);
  if (NH)
#pragma unroll
    for (int i = 0; i < 32; i++) atomicAdd(gh + acc_row(t, 0, i) * 64 + acc_col(t, i), gwh.d[i]);
}

template <int N>
__device__ __forceinline__ void zero(Acc64<N>& a) {
#pragma unroll
  for (int i = 0; i < N / 2; i++) a.d[i] = 0.f;
}

template <int NH>
__global__ void __launch_bounds__(kBT)
mlp_bwd_tc_kernel(const __half* __restrict__ dout, const __half* __restrict__ in, const __half* __restrict__ hidden,
                  const __half* __restrict__ hid_last, const __half* __restrict__ params, int n_pts,
                  __half* __restrict__ din, float* __restrict__ dparams) {
  using S = BwdSmem<NH>;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x;
  const int n_tiles = (n_pts + kBT - 1) / kBT;
  const uint32_t stage0 = smem_u32(sm + S::STAGE0);

  int tile = blockIdx.x;
  if (tile < n_tiles) prefetch_tile<NH>(dout, in, hidden, hid_last, tile, n_pts, stage0);
  asm volatile("cp.async.commit_group;" ::: "memory");
  stage_w<32>(params, 64, sm + S::W0);
  if (NH) stage_w<64>(params + 64 * 32, 64, sm + S::WH);
  stage_w<64>(params + 64 * 32 + NH * 64 * 64, 16, sm + S::WO);
  const uint32_t s_w0 = smem_u32(sm + S::W0), s_wh = smem_u32(sm + S::WH), s_wo = smem_u32(sm + S::WO);
  Acc<64> act;
  Acc<32> act_in;
  Acc64<32> gw0;
  Acc64<16> gwo;
  Acc64<64> gwh;
  zero(gw0); zero(gwo); zero(gwh);
  const bool any = tile < n_tiles;
  uint32_t buf = 0;

  for (; tile < n_tiles; tile += gridDim.x, buf ^= 1) {
    __syncthreads();                                             // every warp's MMAs are done with the stage refilled below
    const int next = tile + gridDim.x;
    if (next < n_tiles) prefetch_tile<NH>(dout, in, hidden, hid_last, next, n_pts, stage0 + (buf ^ 1) * S::STAGE_BYTES);
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 1;" ::: "memory");         // this tile's operands have landed
    fence_async_smem();
    __syncthreads();
    unsigned char* const st = sm + S::STAGE0 + buf * S::STAGE_BYTES;
    const uint32_t sb = stage0 + buf * S::STAGE_BYTES;
    const uint32_t s_do = sb + S::DO, s_x = sb + S::X, s_h0 = sb + S::H0, s_h1 = sb + S::H1;
    const uint32_t s_hl = NH ? s_h1 : s_h0;
    // ---- A: dH_last = dOut . Wout  (K = 16) ; dWout^T += H_last^T . dOut (needs H_last before it is overwritten)
    wg_fence();
    mma_m128<64, 1, 1>(act, s_do, 32, s_wo, 128, false);
    mma_batch128<16>(gwo, s_hl, 128, s_do, 32);
    wg_commit();
    wg_wait();
    __syncthreads();                                             // every warp's MMAs are done reading H_last
    relu_bwd_epilogue(act, st + (NH ? S::H1 : S::H0), st + (NH ? S::H1 : S::H0), tid);   // in place
    fence_async_smem();
    __syncthreads();
    if (NH) {
      // ---- B: dH0 = dH1 . Wh ; dWh += dH1^T . H0 (H0 still the forward activation) ---------------------
      wg_fence();
      mma_m128<64, 1, 4>(act, s_h1, 128, s_wh, 128, false);
      mma_batch128<64>(gwh, s_h1, 128, s_h0, 128);
      wg_commit();
      wg_wait();
      __syncthreads();
      relu_bwd_epilogue(act, st + S::H0, st + S::H0, tid);                                                  // in place
      fence_async_smem();
      __syncthreads();
    }
    // ---- C: dIn = dH0 . W0 ; dW0 += dH0^T . X -----------------------------------------------------------
    wg_fence();
    mma_m128<32, 1, 4>(act_in, s_h0, 128, s_w0, 64, false);
    mma_batch128<32>(gw0, s_h0, 128, s_x, 64);
    wg_commit();
    wg_wait();
    if (din) store_din(act_in, din, tile, n_pts, tid);
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  if (any) flush_weight_grads<NH>(gw0, gwo, gwh, dparams, tid);
}


// ---------------------------------------------------------------------------------------------------------------------
// Recompute variant (hidden0 == NULL in f2b_mlp_bwd2): the forward pass saves NO hidden activations — 128 B (field) /
// 256 B (shader) per sample it no longer writes and this kernel no longer reads.  The tile's activations are rebuilt on
// the tensor pipe from the 64 B input row (same MMAs, same operands, same fp16 rounding as mlp_fwd_tc_kernel => the
// very same bits the forward would have saved), then the backward proceeds as above: the saved-activation kernels are
// bound by HBM traffic with the tensor pipe mostly idle, so the recompute rides on idle MMA issue slots.
// Per sample: 32 (dOut) + 64 (x) B read, 64 B written  (was 224 / 352 B read).
//   NH = 0:  F0  H0 = relu(X.W0^T)                                  -> H0 tile
//            A   dH0 = (dOut.Wout) * [H0 > 0] ; dWout^T += H0^T.dOut -> dH0 over H0
//            C   dX = dH0.W0 ; dW0 += dH0^T.X
//   NH = 1:  F0  H0 = relu(X.W0^T)
//            F1  H1 = relu(H0.Wh^T) -> H1 tile
//            G   dH1 = (dOut.Wout) * [H1 > 0]  -> D1 tile   (the mask tests the fp16 H1 tile the forward would have saved)
//            B   dWout^T += H1^T.dOut ; dH0 = (dH1.Wh) * [H0 > 0] ; dWh += dH1^T.H0 -> dH0 over H0
//            C   dX = dH0.W0 ; dW0 += dH0^T.X
template <int NH>
struct RcSmem {
  static constexpr int W0 = 0;                              // [64 x 32]  SW64   4 KB  (K-major for the forward, MN-major view for the backward)
  static constexpr int WH = 4096;                           // [64 x 64]  SW128  8 KB  (NH only)
  static constexpr int WO = NH ? 12288 : 4096;              // [16 x 64]  SW128  2 KB
  static constexpr int H0 = WO + 2048;                      // [128 x 64] SW128 16 KB  forward H0, then dH0
  static constexpr int H1 = H0 + 16384;                     // [128 x 64] SW128 16 KB  forward H1            (NH only)
  static constexpr int D1 = H1 + 16384;                     // [128 x 64] SW128 16 KB  dH1                   (NH only)
  static constexpr int STAGE0 = NH ? D1 + 16384 : H0 + 16384;
  static constexpr int DO = 0;                              // stage-relative: [128 x 16] SW32 4 KB
  static constexpr int X = 4096;                            //                 [128 x 32] SW64 8 KB
  static constexpr int STAGE_BYTES = 12288;
  static constexpr int BYTES = STAGE0 + 2 * STAGE_BYTES + 1024;
};

template <int NH>
__device__ __forceinline__ void prefetch_tile_rc(const __half* __restrict__ dout, const __half* __restrict__ in, int tile, int n_pts,
                                                 uint32_t stage) {
  using S = RcSmem<NH>;
  const int rows = min(kBT, n_pts - tile * kBT);
  const size_t t0 = size_t(tile) * kBT;
  const unsigned char* s_do = reinterpret_cast<const unsigned char*>(dout + t0 * 16);
  const unsigned char* s_x = reinterpret_cast<const unsigned char*>(in + t0 * 32);
#pragma unroll
  for (int j = 0; j < 2; j++) {
    const int c = threadIdx.x + kBT * j, r = c >> 1;
    const bool ok = r < rows;
    cp16(stage + S::DO + sw32_off(r, c & 1), s_do + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
  }
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int c = threadIdx.x + kBT * j, r = c >> 2;
    const bool ok = r < rows;
    cp16(stage + S::X + sw64_off(r, c & 3), s_x + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
  }
}

template <int NH>
__global__ void __launch_bounds__(kBT)
mlp_bwd_rc_kernel(const __half* __restrict__ dout, const __half* __restrict__ in, const __half* __restrict__ params, int n_pts,
                  __half* __restrict__ din, float* __restrict__ dparams) {
  using S = RcSmem<NH>;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x;
  const int n_tiles = (n_pts + kBT - 1) / kBT;
  const uint32_t stage0 = smem_u32(sm + S::STAGE0);

  int tile = blockIdx.x;
  if (tile < n_tiles) prefetch_tile_rc<NH>(dout, in, tile, n_pts, stage0);
  asm volatile("cp.async.commit_group;" ::: "memory");
  stage_w<32>(params, 64, sm + S::W0);
  if (NH) stage_w<64>(params + 64 * 32, 64, sm + S::WH);
  stage_w<64>(params + 64 * 32 + NH * 64 * 64, 16, sm + S::WO);
  const uint32_t s_w0 = smem_u32(sm + S::W0), s_wh = smem_u32(sm + S::WH), s_wo = smem_u32(sm + S::WO);
  const uint32_t s_h0 = smem_u32(sm + S::H0), s_h1 = smem_u32(sm + S::H1), s_d1 = smem_u32(sm + S::D1);
  Acc<64> act;
  Acc<32> act_in;
  Acc64<32> gw0;
  Acc64<16> gwo;
  Acc64<64> gwh;
  zero(gw0); zero(gwo); zero(gwh);
  const bool any = tile < n_tiles;
  uint32_t buf = 0;

  for (; tile < n_tiles; tile += gridDim.x, buf ^= 1) {
    __syncthreads();                                             // every warp's MMAs are done with the stage refilled below
    const int next = tile + gridDim.x;
    if (next < n_tiles) prefetch_tile_rc<NH>(dout, in, next, n_pts, stage0 + (buf ^ 1) * S::STAGE_BYTES);
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 1;" ::: "memory");         // this tile's operands have landed
    fence_async_smem();
    __syncthreads();                                             // (also: the previous tile's MMAs are done with H0 / H1 / D1)
    const uint32_t sb = stage0 + buf * S::STAGE_BYTES;
    const uint32_t s_do = sb + S::DO, s_x = sb + S::X;
    // ---- F0: H0 = relu(X . W0^T) ---------------------------------------------------------------------------
    wg_fence();
    mma_m128<64, 0, 2>(act, s_x, 64, s_w0, 64, false);
    wg_commit();
    wg_wait();
    acc_relu_to_tile(act, sm + S::H0, tid);
    fence_async_smem();
    __syncthreads();
    if (NH) {
      // ---- F1: H1 = relu(H0 . Wh^T) ------------------------------------------------------------------------
      wg_fence();
      mma_m128<64, 0, 4>(act, s_h0, 128, s_wh, 128, false);
      wg_commit();
      wg_wait();
      acc_relu_to_tile(act, sm + S::H1, tid);
      fence_async_smem();
      __syncthreads();
      // ---- G: dH1 = (dOut . Wout) * [H1 > 0] -----------------------------------------------------------------
      wg_fence();
      mma_m128<64, 1, 1>(act, s_do, 32, s_wo, 128, false);
      wg_commit();
      wg_wait();
      relu_bwd_epilogue(act, sm + S::H1, sm + S::D1, tid);
      fence_async_smem();
      __syncthreads();
      // ---- B: dWout^T += H1^T . dOut ; dH0 = dH1 . Wh ; dWh += dH1^T . H0 (H0 still the forward activation) ----
      wg_fence();
      mma_batch128<16>(gwo, s_h1, 128, s_do, 32);
      mma_m128<64, 1, 4>(act, s_d1, 128, s_wh, 128, false);
      mma_batch128<64>(gwh, s_d1, 128, s_h0, 128);
      wg_commit();
    } else {
      // ---- A: dH0 = dOut . Wout ; dWout^T += H0^T . dOut -------------------------------------------------
      wg_fence();
      mma_m128<64, 1, 1>(act, s_do, 32, s_wo, 128, false);
      mma_batch128<16>(gwo, s_h0, 128, s_do, 32);
      wg_commit();
    }
    wg_wait();
    __syncthreads();                                             // every warp's MMAs are done reading H0
    relu_bwd_epilogue(act, sm + S::H0, sm + S::H0, tid);                                                    // dH0 over H0, in place
    fence_async_smem();
    __syncthreads();
    // ---- C: dIn = dH0 . W0 ; dW0 += dH0^T . X -----------------------------------------------------------
    wg_fence();
    mma_m128<32, 1, 4>(act_in, s_h0, 128, s_w0, 64, false);
    mma_batch128<32>(gw0, s_h0, 128, s_x, 64);
    wg_commit();
    wg_wait();
    if (din) store_din(act_in, din, tile, n_pts, tid);
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  if (any) flush_weight_grads<NH>(gw0, gwo, gwh, dparams, tid);
}


// ---------------------------------------------------------------------------------------------------------------------
// Field-MLP backward with the hash-grid scatter fused behind it (f2b_field_bwd_scatter): mlp_bwd_rc_kernel<0> per tile
// (F0 -> A -> C, same operands and fp16 roundings), then the tile's dL/dfeat rows go to a shared [128 x 32] fp16 tile instead
// of HBM, and warp w scatters rows [32w, 32w + 32) into the table gradient, all 16 levels, with scatter_level (hash.cuh).
// Tiles start at multiples of 128 from the segment start, so every 32-row group is the group f2b_hash_bwd forms: the same
// run merging and shuffle-scan order, hence bit-identical reductions (only their arrival order at L2 differs).  The scatter
// is bound by L2 reduction issue and the MMAs by the tensor pipe; with 3 CTAs per SM one CTA's reductions (fire-and-forget)
// drain while another CTA runs its MMAs.  The tile's points and volume ids are prefetched with the operand rows, so the
// scatter issues no dependent global loads.
constexpr int kDinLd = 40;                                  // DIN tile row pitch in halfs

struct FbsSmem {
  static constexpr int W0 = RcSmem<0>::W0;                  // [64 x 32]  SW64   4 KB
  static constexpr int WO = RcSmem<0>::WO;                  // [16 x 64]  SW128  2 KB
  static constexpr int H0 = RcSmem<0>::H0;                  // [128 x 64] SW128 16 KB  forward H0, then dH0
  static constexpr int DIN = H0 + 16384;                    // [128 x 32] fp16, rows padded to 80 B        10 KB
  static constexpr int STAGE0 = DIN + 128 * kDinLd * 2;
  static constexpr int DO = RcSmem<0>::DO;                  // stage-relative: [128 x 16] SW32 4 KB
  static constexpr int X = RcSmem<0>::X;                    //                 [128 x 32] SW64 8 KB
  static constexpr int PTS = 12288;                         //                 [128 x 3] fp32  1.5 KB
  static constexpr int VOL = PTS + 1536;                    //                 [128] int32     0.5 KB
  static constexpr int STAGE_BYTES = 14336;                 // a multiple of 1024: both stages keep the swizzle-atom alignment
  static constexpr int BYTES = STAGE0 + 2 * STAGE_BYTES + 1024;
};

__device__ __forceinline__ void cp4(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

// the tile's points (3 fp32 per row, contiguous) and volume ids (vol[i * vol_stride]); rows past n_pts are zero-filled
__device__ __forceinline__ void prefetch_pts_vol(const float* __restrict__ pts, const int* __restrict__ vol, int vol_stride, int tile,
                                                 int n_pts, uint32_t stage) {
  const int rows = min(kBT, n_pts - tile * kBT);
  const size_t t0 = size_t(tile) * kBT;
#pragma unroll
  for (int j = 0; j < 3; j++) {
    const int c = threadIdx.x + kBT * j;
    const bool ok = c < rows * 3;
    cp4(stage + FbsSmem::PTS + 4 * c, pts + t0 * 3 + (ok ? c : 0), ok ? 4u : 0u);
  }
  const bool ok = int(threadIdx.x) < rows;
  cp4(stage + FbsSmem::VOL + 4 * threadIdx.x, vol + (t0 + (ok ? threadIdx.x : 0)) * vol_stride, ok ? 4u : 0u);
}

// byte offset of fp16 column `col` of row `r` in the DIN tile.  The 80 B row pitch makes the accumulator stores conflict-free and
// keeps every offset a per-thread base plus a constant (a swizzle would hold a few more registers across the tile loop)
__device__ __forceinline__ uint32_t din_off(int r, int col) { return (r * kDinLd + col) * 2; }

__global__ void __launch_bounds__(kBT, 3)
field_bwd_scatter_kernel(const __half* __restrict__ dout, const __half* __restrict__ in, const __half* __restrict__ params, int n_pts,
                         const float* __restrict__ pts, const int* __restrict__ vol, int vol_stride, const int* __restrict__ prim_pool,
                         const float* __restrict__ bias_pool, int n_volumes, int local_size, float grad_mul,
                         float* __restrict__ dparams, float* __restrict__ grad_table, __half* __restrict__ din) {
  using S = FbsSmem;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_tiles = (n_pts + kBT - 1) / kBT;
  const uint32_t stage0 = smem_u32(sm + S::STAGE0);

  int tile = blockIdx.x;
  if (tile < n_tiles) {
    prefetch_tile_rc<0>(dout, in, tile, n_pts, stage0);
    prefetch_pts_vol(pts, vol, vol_stride, tile, n_pts, stage0);
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  stage_w<32>(params, 64, sm + S::W0);
  stage_w<64>(params + 64 * 32, 16, sm + S::WO);
  const uint32_t s_w0 = smem_u32(sm + S::W0), s_wo = smem_u32(sm + S::WO), s_h0 = smem_u32(sm + S::H0);
  unsigned char* const s_din = sm + S::DIN;
  Acc<64> act;
  Acc<32> act_in;
  Acc64<32> gw0;
  Acc64<16> gwo;
  Acc64<64> gwh;                                                 // unused: no hidden matmul (flush_weight_grads<0> skips it)
  zero(gw0); zero(gwo);
  uint32_t buf = 0;

  for (; tile < n_tiles; tile += gridDim.x, buf ^= 1) {
    __syncthreads();                                             // every warp is done with the stage refilled below
    const int next = tile + gridDim.x;
    if (next < n_tiles) {
      const uint32_t nb = stage0 + (buf ^ 1) * S::STAGE_BYTES;
      prefetch_tile_rc<0>(dout, in, next, n_pts, nb);
      prefetch_pts_vol(pts, vol, vol_stride, next, n_pts, nb);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 1;" ::: "memory");         // this tile's operands have landed
    fence_async_smem();
    __syncthreads();                                             // (also: the previous tile's MMAs and scatter are done with H0 / DIN)
    const unsigned char* const st = sm + S::STAGE0 + buf * S::STAGE_BYTES;
    const uint32_t sb = stage0 + buf * S::STAGE_BYTES;
    const uint32_t s_do = sb + S::DO, s_x = sb + S::X;
    // ---- F0: H0 = relu(X . W0^T) ---------------------------------------------------------------------------
    wg_fence();
    mma_m128<64, 0, 2>(act, s_x, 64, s_w0, 64, false);
    wg_commit();
    wg_wait();
    acc_relu_to_tile(act, sm + S::H0, tid);
    fence_async_smem();
    __syncthreads();
    // ---- A: dH0 = dOut . Wout ; dWout^T += H0^T . dOut -------------------------------------------------------
    wg_fence();
    mma_m128<64, 1, 1>(act, s_do, 32, s_wo, 128, false);
    mma_batch128<16>(gwo, s_h0, 128, s_do, 32);
    wg_commit();
    wg_wait();
    __syncthreads();                                             // every warp's MMAs are done reading H0
    relu_bwd_epilogue(act, sm + S::H0, sm + S::H0, tid);         // dH0 over H0, in place
    fence_async_smem();
    __syncthreads();
    // ---- C: dIn = dH0 . W0 ; dW0 += dH0^T . X -----------------------------------------------------------------
    wg_fence();
    mma_m128<32, 1, 4>(act_in, s_h0, 128, s_w0, 64, false);
    mma_batch128<32>(gw0, s_h0, 128, s_x, 64);
    wg_commit();
    wg_wait();
#pragma unroll
    for (int h = 0; h < 2; h++)                                  // the same fp16 packing as store_din
#pragma unroll
      for (int i = 0; i < 16; i += 2)
        *reinterpret_cast<uint32_t*>(s_din + din_off(acc_row(tid, h, i), acc_col(tid, i))) = pk(act_in.d[h][i], act_in.d[h][i + 1]);
    if (din) store_din(act_in, din, tile, n_pts, tid);
    __syncthreads();
    // ---- scatter: warp w, rows [32w, 32w + 32) of the tile = sample group 4 * tile + w -----------------------
    const int r = 32 * warp + lane;
    if (tile * kBT + 32 * warp < n_pts) {                        // warp-uniform: the group has a sample
      const bool valid = tile * kBT + r < n_pts;
      const float* p = reinterpret_cast<const float*>(st + S::PTS) + 3 * r;
      const float x0 = fmul(fadd(p[0], 1.f), .5f), x1 = fmul(fadd(p[1], 1.f), .5f), x2 = fmul(fadd(p[2], 1.f), .5f);
      const int v = reinterpret_cast<const int*>(st + S::VOL)[r];
#pragma unroll 1
      for (int l = 0; l < F2B_N_LEVELS; l++) {
        const float2 g = __half22float2(*reinterpret_cast<const __half2*>(s_din + din_off(r, 2 * l)));
        const bool live = valid && !(g.x == 0.f && g.y == 0.f);
        scatter_level(l, lane, g.x * grad_mul, g.y * grad_mul, x0, x1, x2, v, live, prim_pool, bias_pool, n_volumes, local_size,
                      grad_table);
      }
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  if (int(blockIdx.x) < n_tiles) flush_weight_grads<0>(gw0, gwo, gwh, dparams, tid);
}

}  // namespace f2b

using namespace f2b;

extern "C" int f2b_field_bwd_scatter(const void* dout_f16, const void* feat_f16, const void* params_f16, int n_pts, const float* pts,
                                     const int* vol, int vol_stride, const int* prim_pool, const float* bias_pool, int n_volumes,
                                     int local_size, float grad_mul, float* dparams_f32, float* grad_table_f32, void* din_f16,
                                     void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(dout_f16 && feat_f16 && params_f16 && pts && vol && prim_pool && bias_pool && dparams_f32 && grad_table_f32,
              "f2b_field_bwd_scatter: null pointer");
  F2B_REQUIRE(n_volumes > 0 && local_size > 0 && (local_size % 2) == 0 && vol_stride > 0,
              "f2b_field_bwd_scatter: bad n_volumes/local_size/vol_stride");
  int sms = 132;
  f2b_device_info(&sms, nullptr);
  constexpr int bytes = FbsSmem::BYTES;
  cudaFuncSetAttribute(field_bwd_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  const int n_tiles = div_up(n_pts, kBT);
  const int cap = sms * resident_per_sm(field_bwd_scatter_kernel, kBT, bytes);   // persistent: weight gradients flushed once per CTA
  field_bwd_scatter_kernel<<<n_tiles < cap ? n_tiles : cap, kBT, bytes, as_stream(stream)>>>(
      (const __half*)dout_f16, (const __half*)feat_f16, (const __half*)params_f16, n_pts, pts, vol, vol_stride, prim_pool, bias_pool,
      n_volumes, local_size, grad_mul, dparams_f32, grad_table_f32, (__half*)din_f16);
  return check_launch("f2b_field_bwd_scatter");
}

extern "C" int f2b_mlp_bwd2(const void* dout_f16, const void* in_f16, const void* hidden0_f16, const void* hidden1_f16,
                            const void* params_f16, int n_hidden_matmuls, int n_pts, void* din_f16,
                            float* dparams_f32, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(dout_f16 && in_f16 && params_f16 && dparams_f32, "f2b_mlp_bwd: null pointer");
  F2B_REQUIRE(n_hidden_matmuls == 0 || n_hidden_matmuls == 1, "f2b_mlp_bwd: n_hidden_matmuls must be 0 or 1");
  int sms = 132;
  f2b_device_info(&sms, nullptr);
  const int n_tiles = div_up(n_pts, kBT);
  // persistent grid: as many CTAs as are resident at once (each flushes its weight gradients once)
#define F2B_BWD_LAUNCH(KERNEL, BYTES, ...)                                                          \
  {                                                                                                 \
    cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, BYTES);               \
    const int cap = sms * resident_per_sm(KERNEL, kBT, BYTES);                                      \
    KERNEL<<<n_tiles < cap ? n_tiles : cap, kBT, BYTES, as_stream(stream)>>>(__VA_ARGS__);          \
  }
  if (!hidden0_f16) {                                             // no saved activations: rebuild them on the tensor pipe
    if (n_hidden_matmuls == 0)
      F2B_BWD_LAUNCH(mlp_bwd_rc_kernel<0>, RcSmem<0>::BYTES, (const __half*)dout_f16, (const __half*)in_f16,
                     (const __half*)params_f16, n_pts, (__half*)din_f16, dparams_f32)
    else
      F2B_BWD_LAUNCH(mlp_bwd_rc_kernel<1>, RcSmem<1>::BYTES, (const __half*)dout_f16, (const __half*)in_f16,
                     (const __half*)params_f16, n_pts, (__half*)din_f16, dparams_f32)
    return check_launch("f2b_mlp_bwd(wgmma, recompute)");
  }
  F2B_REQUIRE(n_hidden_matmuls == 0 || hidden1_f16, "f2b_mlp_bwd: hidden1 missing (n_hidden_matmuls == 1 with saved activations)");
  if (n_hidden_matmuls == 0)
    F2B_BWD_LAUNCH(mlp_bwd_tc_kernel<0>, BwdSmem<0>::BYTES, (const __half*)dout_f16, (const __half*)in_f16,
                   (const __half*)hidden0_f16, (const __half*)hidden0_f16, (const __half*)params_f16, n_pts, (__half*)din_f16,
                   dparams_f32)
  else
    F2B_BWD_LAUNCH(mlp_bwd_tc_kernel<1>, BwdSmem<1>::BYTES, (const __half*)dout_f16, (const __half*)in_f16,
                   (const __half*)hidden0_f16, (const __half*)hidden1_f16, (const __half*)params_f16, n_pts, (__half*)din_f16,
                   dparams_f32)
#undef F2B_BWD_LAUNCH
  return check_launch("f2b_mlp_bwd(wgmma)");
}

extern "C" int f2b_mlp_bwd(const void* dout_f16, const void* in_f16, const void* hidden_save_f16,
                           const void* params_f16, int n_hidden_matmuls, int n_pts, void* din_f16,
                           float* dparams_f32, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(hidden_save_f16, "f2b_mlp_bwd: null pointer");
  const __half* h = (const __half*)hidden_save_f16;
  return f2b_mlp_bwd2(dout_f16, in_f16, h, h + size_t(n_hidden_matmuls ? 1 : 0) * n_pts * 64, params_f16, n_hidden_matmuls, n_pts,
                      din_f16, dparams_f32, stream);
}
