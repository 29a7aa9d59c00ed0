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
    cp_async<16>(stage + S::DO + sw32_off(r, c & 1), s_do + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
  }
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int c = threadIdx.x + kBT * j, r = c >> 2;
    const bool ok = r < rows;
    cp_async<16>(stage + S::X + sw64_off(r, c & 3), s_x + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
  }
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int c = threadIdx.x + kBT * j, r = c >> 3;
    const bool ok = r < rows;
    cp_async<16>(stage + S::H0 + sw128_off(r, c & 7), s_h0 + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
    if (NH) cp_async<16>(stage + S::H1 + sw128_off(r, c & 7), s_h1 + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
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
  unsigned char* sm = smem_base();
  const int tid = threadIdx.x;
  const int n_tiles = (n_pts + kBT - 1) / kBT;
  const uint32_t stage0 = smem_u32(sm + S::STAGE0);

  int tile = blockIdx.x;
  if (tile < n_tiles) prefetch_tile<NH>(dout, in, hidden, hid_last, tile, n_pts, stage0);
  cp_async_commit();
  stage_weights<32, 0>(params, 64, sm + S::W0, threadIdx.x);
  if (NH) stage_weights<64, 0>(params + 64 * 32, 64, sm + S::WH, threadIdx.x);
  stage_weights<64, 0>(params + 64 * 32 + NH * 64 * 64, 16, sm + S::WO, threadIdx.x);
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
    cp_async_commit();
    cp_async_wait<1>();                                          // this tile's operands have landed
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
  cp_async_wait<0>();
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
    cp_async<16>(stage + S::DO + sw32_off(r, c & 1), s_do + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
  }
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int c = threadIdx.x + kBT * j, r = c >> 2;
    const bool ok = r < rows;
    cp_async<16>(stage + S::X + sw64_off(r, c & 3), s_x + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
  }
}

template <int NH>
__global__ void __launch_bounds__(kBT)
mlp_bwd_rc_kernel(const __half* __restrict__ dout, const __half* __restrict__ in, const __half* __restrict__ params, int n_pts,
                  __half* __restrict__ din, float* __restrict__ dparams) {
  using S = RcSmem<NH>;
  unsigned char* sm = smem_base();
  const int tid = threadIdx.x;
  const int n_tiles = (n_pts + kBT - 1) / kBT;
  const uint32_t stage0 = smem_u32(sm + S::STAGE0);

  int tile = blockIdx.x;
  if (tile < n_tiles) prefetch_tile_rc<NH>(dout, in, tile, n_pts, stage0);
  cp_async_commit();
  stage_weights<32, 0>(params, 64, sm + S::W0, threadIdx.x);
  if (NH) stage_weights<64, 0>(params + 64 * 32, 64, sm + S::WH, threadIdx.x);
  stage_weights<64, 0>(params + 64 * 32 + NH * 64 * 64, 16, sm + S::WO, threadIdx.x);
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
    cp_async_commit();
    cp_async_wait<1>();                                          // this tile's operands have landed
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
  cp_async_wait<0>();
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

// the tile's points (3 fp32 per row, contiguous) to s_pts and volume ids (vol[i * vol_stride]) to s_vol; rows past n_pts are zero-filled
__device__ __forceinline__ void prefetch_pts_vol(const float* __restrict__ pts, const int* __restrict__ vol, int vol_stride, int tile,
                                                 int n_pts, uint32_t s_pts, uint32_t s_vol) {
  const int rows = min(kBT, n_pts - tile * kBT);
  const size_t t0 = size_t(tile) * kBT;
#pragma unroll
  for (int j = 0; j < 3; j++) {
    const int c = threadIdx.x + kBT * j;
    const bool ok = c < rows * 3;
    cp_async<4>(s_pts + 4 * c, pts + t0 * 3 + (ok ? c : 0), ok ? 4u : 0u);
  }
  const bool ok = int(threadIdx.x) < rows;
  cp_async<4>(s_vol + 4 * threadIdx.x, vol + (t0 + (ok ? threadIdx.x : 0)) * vol_stride, ok ? 4u : 0u);
}

// byte offset of fp16 column `col` of row `r` in the DIN tile.  The 80 B row pitch makes the accumulator stores conflict-free and
// keeps every offset a per-thread base plus a constant (a swizzle would hold a few more registers across the tile loop)
__device__ __forceinline__ uint32_t din_off(int r, int col) { return (r * kDinLd + col) * 2; }

// warp-collective: row r = 32 w + lane of a tile's DIN / PTS / VOL blocks (group w of the tile) into the table gradient, all 16 levels.
// valid: the row is a sample of the segment
__device__ __forceinline__ void scatter_row(const unsigned char* s_din, const unsigned char* s_pts, const unsigned char* s_vol, int r,
                                            int lane, bool valid, const int* __restrict__ prim_pool, const float* __restrict__ bias_pool,
                                            int n_volumes, int local_size, float grad_mul, float* __restrict__ grad_table) {
  const float* p = reinterpret_cast<const float*>(s_pts) + 3 * r;
  const float x0 = fmul(fadd(p[0], 1.f), .5f), x1 = fmul(fadd(p[1], 1.f), .5f), x2 = fmul(fadd(p[2], 1.f), .5f);
  const int v = reinterpret_cast<const int*>(s_vol)[r];
#pragma unroll 1
  for (int l = 0; l < F2B_N_LEVELS; l++) {
    const float2 g = __half22float2(*reinterpret_cast<const __half2*>(s_din + din_off(r, 2 * l)));
    const bool live = valid && !(g.x == 0.f && g.y == 0.f);
    scatter_level(l, lane, g.x * grad_mul, g.y * grad_mul, x0, x1, x2, v, live, prim_pool, bias_pool, n_volumes, local_size, grad_table);
  }
}

__global__ void __launch_bounds__(kBT, 3)
field_bwd_scatter_kernel(const __half* __restrict__ dout, const __half* __restrict__ in, const __half* __restrict__ params, int n_pts,
                         const float* __restrict__ pts, const int* __restrict__ vol, int vol_stride, const int* __restrict__ prim_pool,
                         const float* __restrict__ bias_pool, int n_volumes, int local_size, float grad_mul,
                         float* __restrict__ dparams, float* __restrict__ grad_table, __half* __restrict__ din) {
  using S = FbsSmem;
  unsigned char* sm = smem_base();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_tiles = (n_pts + kBT - 1) / kBT;
  const uint32_t stage0 = smem_u32(sm + S::STAGE0);

  int tile = blockIdx.x;
  if (tile < n_tiles) {
    prefetch_tile_rc<0>(dout, in, tile, n_pts, stage0);
    prefetch_pts_vol(pts, vol, vol_stride, tile, n_pts, stage0 + S::PTS, stage0 + S::VOL);
  }
  cp_async_commit();
  stage_weights<32, 0>(params, 64, sm + S::W0, threadIdx.x);
  stage_weights<64, 0>(params + 64 * 32, 16, sm + S::WO, threadIdx.x);
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
      prefetch_pts_vol(pts, vol, vol_stride, next, n_pts, nb + S::PTS, nb + S::VOL);
    }
    cp_async_commit();
    cp_async_wait<1>();                                          // this tile's operands have landed
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
    if (tile * kBT + 32 * warp < n_pts)                          // warp-uniform: the group has a sample
      scatter_row(s_din, st + S::PTS, st + S::VOL, r, lane, tile * kBT + r < n_pts, prim_pool, bias_pool, n_volumes, local_size,
                  grad_mul, grad_table);
  }
  cp_async_wait<0>();
  if (int(blockIdx.x) < n_tiles) flush_weight_grads<0>(gw0, gwo, gwh, dparams, tid);
}


// ---------------------------------------------------------------------------------------------------------------------
// The whole per-sample backward of the ray samples behind the composite backward, in one kernel (f2b_shade_field_bwd_scatter):
// shader-MLP backward -> shading-input backward (f2b_shader_prep_bwd_f16) -> field-MLP backward -> hash scatter.  The scatter is
// bound by L2 reductions and leaves the tensor pipe idle, so the MMAs of both MLPs hide under it.  Warp-specialised, one CTA per
// SM:
//   warpgroup 0 (MMA): per 128-sample tile, mlp_bwd_rc_kernel<1>'s F0 F1 G B C on the shader operands (same MMAs, same fp16
//     roundings); the shader_prep_bwd_f16 epilogue in registers (fp16 dIn as store_din rounds it, x inv_loss_scale, channel 0
//     replaced by d_logit, x field_loss_scale, fp16) straight into the field's SW32 dL/dout tile; field_bwd_scatter_kernel's
//     F0 A C on it.  The fp16 dL/dfeat rows, the tile's points / volume ids and the fp16 shader dIn channels 0..15 go to ring
//     slot k % 2 (k = the CTA's tile count).
//   warpgroups 1, 2 (scatter): warpgroup 1 + k % 2 consumes slot k % 2; warp w takes rows [32w, 32w + 32), i.e. sample group
//     4 * tile + w as f2b_hash_bwd forms it (same run merging, bit-identical reduction values), scatters them over all 16 levels
//     and adds their d_app rows, one atomicAdd per run of equal pt_emb_idx and channel.
// Slots are handed over with named barriers (FULL: MMA warpgroup arrives, scatter warpgroup waits; EMPTY: the reverse).
// setmaxnreg moves registers to the MMA warpgroup (two MLPs' weight-gradient accumulators stay resident across its tiles).
// Tiles come from an atomic ticket, so a CTA that starts late (its SM still busy with another kernel) takes fewer of them;
// the groups depend on the tile index only.
constexpr int kSfbThreads = 384;
constexpr int kSdinLd = 24;                                 // shader dIn rows in a slot: 16 fp16 + pad (conflict-free both ways)
constexpr int kBarFull = 1, kBarEmpty = 3, kBarMma = 5;     // named barrier ids (0 is __syncthreads)

struct SfbSmem {
  static constexpr int SW0 = 0;                             // shader [64 x 32]  SW64   4 KB
  static constexpr int SWH = 4096;                          // shader [64 x 64]  SW128  8 KB
  static constexpr int SWO = 12288;                         // shader [16 x 64]  SW128  2 KB
  static constexpr int FW0 = 14336;                         // field  [64 x 32]  SW64   4 KB
  static constexpr int FWO = 18432;                         // field  [16 x 64]  SW128  2 KB
  static constexpr int H0 = 20480;                          // [128 x 64] SW128 16 KB  shader H0 / dH0, then field H0 / dH0
  static constexpr int H1 = H0 + 16384;                     // [128 x 64] SW128 16 KB  shader H1
  static constexpr int D1 = H1 + 16384;                     // [128 x 64] SW128 16 KB  shader dH1
  static constexpr int FDO = D1 + 16384;                    // [128 x 16] SW32   4 KB  field dL/dout
  static constexpr int SDIN = FDO + 4096;                   // [128 x 16] fp16 shader dIn channels 0..15, rows padded to 48 B  6 KB
  static constexpr int STAGE0 = SDIN + 128 * kSdinLd * 2;
  static constexpr int DO = 0;                              // stage-relative: shader dL/dout [128 x 16] SW32 4 KB
  static constexpr int X = 4096;                            //                 shader input   [128 x 32] SW64 8 KB
  static constexpr int FX = 12288;                          //                 field input    [128 x 32] SW64 8 KB
  static constexpr int PTS = 20480;                         //                 [128 x 3] fp32 1.5 KB
  static constexpr int VOL = PTS + 1536;                    //                 [128] int32    0.5 KB
  static constexpr int DLOG = VOL + 512;                    //                 [128] fp32 d_logit 0.5 KB
  static constexpr int STAGE_BYTES = 23552;                 // a multiple of 1024: both stages keep the swizzle-atom alignment
  static constexpr int RING0 = STAGE0 + 2 * STAGE_BYTES;
  static constexpr int R_DIN = 0;                           // slot-relative: [128 x 32] fp16, rows padded to 80 B   10 KB
  static constexpr int R_PTS = 128 * kDinLd * 2;            //                [128 x 3] fp32
  static constexpr int R_VOL = R_PTS + 1536;                //                [128] int32
  static constexpr int R_SDIN = R_VOL + 512;                //                copy of SDIN
  static constexpr int R_TILE = R_SDIN + 128 * kSdinLd * 2; //                tile index (-1: no more tiles)
  static constexpr int SLOT_BYTES = R_TILE + 128;
  static constexpr int TICKET = RING0 + 2 * SLOT_BYTES;     // [2] int: the MMA warpgroup's next tile, double-buffered
  static constexpr int BYTES = TICKET + 16 + 1024;
};
static_assert(SfbSmem::STAGE0 % 1024 == 0 && SfbSmem::DLOG + 512 <= SfbSmem::STAGE_BYTES, "SfbSmem stage layout");
static_assert(SfbSmem::R_PTS + 2048 == SfbSmem::R_SDIN, "pts + vol of a slot are one 2 KB block (one uint4 per MMA thread)");

__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// one tile's operands: shader dOut + input rows, field input rows, points, volume ids, d_logit
__device__ __forceinline__ void prefetch_tile_sfb(const __half* __restrict__ d_raw, const __half* __restrict__ mlp_in,
                                                  const __half* __restrict__ feat, const float* __restrict__ d_logit,
                                                  const float* __restrict__ pts, const int* __restrict__ vol, int vol_stride, int tile,
                                                  int n_pts, uint32_t stage) {
  using S = SfbSmem;
  prefetch_tile_rc<1>(d_raw, mlp_in, tile, n_pts, stage);     // DO, X
  const int rows = min(kBT, n_pts - tile * kBT);
  const size_t t0 = size_t(tile) * kBT;
  const unsigned char* s_fx = reinterpret_cast<const unsigned char*>(feat + t0 * 32);
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int c = threadIdx.x + kBT * j, r = c >> 2;
    const bool ok = r < rows;
    cp_async<16>(stage + S::FX + sw64_off(r, c & 3), s_fx + (ok ? size_t(c) * 16 : 0), ok ? 16u : 0u);
  }
  prefetch_pts_vol(pts, vol, vol_stride, tile, n_pts, stage + S::PTS, stage + S::VOL);
  const bool ok = int(threadIdx.x) < rows;
  cp_async<4>(stage + S::DLOG + 4 * threadIdx.x, d_logit + t0 + (ok ? threadIdx.x : 0), ok ? 4u : 0u);
}

// warp-collective: d_app[e] += sum of the warp's rows with embedding index e, per run of equal e (a camera index is constant along a
// ray, so a group holds one or two runs).  e = -1 marks a row that is not a sample.
__device__ __forceinline__ void app_grad_runs(float (&g)[16], int e, int lane, float* __restrict__ d_app) {
  const int prev_e = __shfl_up_sync(0xffffffffu, e, 1);
  const unsigned heads = __ballot_sync(0xffffffffu, lane == 0 || e != prev_e);
  const int run_start = 31 - __clz(heads & ((2u << lane) - 1u));
  const int max_run = __reduce_max_sync(0xffffffffu, lane - run_start + 1);
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    if (o >= max_run) break;
    const bool take = (lane - o) >= run_start;
#pragma unroll
    for (int k = 0; k < 16; k++) {
      const float u = __shfl_up_sync(0xffffffffu, g[k], o);
      if (take) g[k] += u;
    }
  }
  const bool tail = (lane == 31) || ((heads >> (lane + 1)) & 1u);
  if (e >= 0 && tail) {
#pragma unroll
    for (int k = 0; k < 16; k++) atomicAdd(d_app + size_t(e) * 16 + k, g[k]);
  }
}

__global__ void __launch_bounds__(kSfbThreads, 1)
shade_field_bwd_scatter_kernel(const __half* __restrict__ d_raw, const __half* __restrict__ mlp_in, const __half* __restrict__ sparams,
                               const float* __restrict__ d_logit, const int* __restrict__ pt_emb_idx, float inv_loss_scale,
                               float field_loss_scale, const __half* __restrict__ feat, const __half* __restrict__ fparams, int n_pts,
                               const float* __restrict__ pts, const int* __restrict__ vol, int vol_stride,
                               const int* __restrict__ prim_pool, const float* __restrict__ bias_pool, int n_volumes, int local_size,
                               float grad_mul, float* __restrict__ d_sparams, float* __restrict__ d_fparams,
                               float* __restrict__ grad_table, float* __restrict__ d_app, int* __restrict__ ticket,
                               __half* __restrict__ d_in16, __half* __restrict__ d_scene16, __half* __restrict__ dfeat16) {
  using S = SfbSmem;
  unsigned char* sm = smem_base();
  int* s_tk = reinterpret_cast<int*>(sm + S::TICKET);                 // read after barriers only ("memory" clobbers)
  if (threadIdx.x == 0) s_tk[0] = atomicAdd(ticket, 1);
  stage_weights<32, 0>(sparams, 64, sm + S::SW0, threadIdx.x);
  stage_weights<64, 0>(sparams + 64 * 32, 64, sm + S::SWH, threadIdx.x);
  stage_weights<64, 0>(sparams + 64 * 32 + 64 * 64, 16, sm + S::SWO, threadIdx.x);
  stage_weights<32, 0>(fparams, 64, sm + S::FW0, threadIdx.x);
  stage_weights<64, 0>(fparams + 64 * 32, 16, sm + S::FWO, threadIdx.x);
  __syncthreads();

  if (threadIdx.x >= kBT) {
    // ================================ scatter warpgroups =================================================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 128;" ::: "memory");
    const int j = (threadIdx.x >> 7) - 1, w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, r = 32 * w + lane;
    const unsigned char* slot = sm + S::RING0 + j * S::SLOT_BYTES;
    bar_arrive(kBarEmpty + j, 2 * kBT);                          // the slot starts empty
    for (;;) {
      bar_sync(kBarFull + j, 2 * kBT);
      const int tile = *reinterpret_cast<const int*>(slot + S::R_TILE);
      if (tile < 0) break;
      if (tile * kBT + 32 * w < n_pts) {                         // warp-uniform: the group has a sample
        const int p = tile * kBT + r;
        const bool valid = p < n_pts;
        if (pt_emb_idx) {
          float g[16];
          const uint4* src = reinterpret_cast<const uint4*>(slot + S::R_SDIN + r * kSdinLd * 2);
#pragma unroll
          for (int q = 0; q < 2; q++) {
            const uint4 u = src[q];
            const uint32_t h[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
            for (int k = 0; k < 4; k++) {
              const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h[k]));
              g[8 * q + 2 * k] = f.x * inv_loss_scale;
              g[8 * q + 2 * k + 1] = f.y * inv_loss_scale;
            }
          }
          app_grad_runs(g, valid ? pt_emb_idx[p] : -1, lane, d_app);
        }
        scatter_row(slot + S::R_DIN, slot + S::R_PTS, slot + S::R_VOL, r, lane, valid, prim_pool, bias_pool, n_volumes, local_size,
                    grad_mul, grad_table);
      }
      bar_arrive(kBarEmpty + j, 2 * kBT);
    }
    return;
  }

  // ================================== MMA warpgroup ======================================================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;" ::: "memory");
  const int tid = threadIdx.x;
  const int n_tiles = (n_pts + kBT - 1) / kBT;
  const uint32_t stage0 = smem_u32(sm + S::STAGE0);
  const uint32_t s_sw0 = smem_u32(sm + S::SW0), s_swh = smem_u32(sm + S::SWH), s_swo = smem_u32(sm + S::SWO);
  const uint32_t s_fw0 = smem_u32(sm + S::FW0), s_fwo = smem_u32(sm + S::FWO);
  const uint32_t s_h0 = smem_u32(sm + S::H0), s_h1 = smem_u32(sm + S::H1), s_d1 = smem_u32(sm + S::D1), s_fdo = smem_u32(sm + S::FDO);
  int tile = s_tk[0];
  if (tile < n_tiles) prefetch_tile_sfb(d_raw, mlp_in, feat, d_logit, pts, vol, vol_stride, tile, n_pts, stage0);
  cp_async_commit();
  Acc<64> act;
  Acc<32> act_in;
  Acc64<32> sgw0, fgw0;
  Acc64<16> sgwo, fgwo;
  Acc64<64> sgwh;
  zero(sgw0); zero(sgwo); zero(sgwh); zero(fgw0); zero(fgwo);
  const bool any = tile < n_tiles;
  int k = 0;
  for (; tile < n_tiles; k++) {
    const int b = k & 1;
    if (tid == 0) s_tk[b ^ 1] = atomicAdd(ticket, 1);
    bar_sync(kBarMma, kBT);                                      // every warp's MMAs are done with the stage refilled below
    const int next = s_tk[b ^ 1];
    if (next < n_tiles) prefetch_tile_sfb(d_raw, mlp_in, feat, d_logit, pts, vol, vol_stride, next, n_pts, stage0 + (b ^ 1) * S::STAGE_BYTES);
    cp_async_commit();
    cp_async_wait<1>();                                          // this tile's operands have landed
    fence_async_smem();
    bar_sync(kBarMma, kBT);
    const unsigned char* const st = sm + S::STAGE0 + b * S::STAGE_BYTES;
    const uint32_t sb = stage0 + b * S::STAGE_BYTES;
    const uint32_t s_do = sb + S::DO, s_x = sb + S::X, s_fx = sb + S::FX;
    // ---- shader F0: H0 = relu(X . W0^T) ---------------------------------------------------------------------------
    wg_fence();
    mma_m128<64, 0, 2>(act, s_x, 64, s_sw0, 64, false);
    wg_commit();
    wg_wait();
    acc_relu_to_tile(act, sm + S::H0, tid);
    fence_async_smem();
    bar_sync(kBarMma, kBT);
    // ---- shader F1: H1 = relu(H0 . Wh^T) --------------------------------------------------------------------------
    wg_fence();
    mma_m128<64, 0, 4>(act, s_h0, 128, s_swh, 128, false);
    wg_commit();
    wg_wait();
    acc_relu_to_tile(act, sm + S::H1, tid);
    fence_async_smem();
    bar_sync(kBarMma, kBT);
    // ---- shader G: dH1 = (dOut . Wout) * [H1 > 0] ----------------------------------------------------------------
    wg_fence();
    mma_m128<64, 1, 1>(act, s_do, 32, s_swo, 128, false);
    wg_commit();
    wg_wait();
    relu_bwd_epilogue(act, sm + S::H1, sm + S::D1, tid);
    fence_async_smem();
    bar_sync(kBarMma, kBT);
    // ---- shader B: dWout^T += H1^T . dOut ; dH0 = dH1 . Wh ; dWh += dH1^T . H0 -------------------------------------
    wg_fence();
    mma_batch128<16>(sgwo, s_h1, 128, s_do, 32);
    mma_m128<64, 1, 4>(act, s_d1, 128, s_swh, 128, false);
    mma_batch128<64>(sgwh, s_d1, 128, s_h0, 128);
    wg_commit();
    wg_wait();
    bar_sync(kBarMma, kBT);                                      // every warp's MMAs are done reading H0
    relu_bwd_epilogue(act, sm + S::H0, sm + S::H0, tid);         // dH0 over H0, in place
    fence_async_smem();
    bar_sync(kBarMma, kBT);
    // ---- shader C: dIn = dH0 . W0 ; dW0 += dH0^T . X ---------------------------------------------------------------
    wg_fence();
    mma_m128<32, 1, 4>(act_in, s_h0, 128, s_sw0, 64, false);
    mma_batch128<32>(sgw0, s_h0, 128, s_x, 64);
    wg_commit();
    wg_wait();
    if (d_in16) store_din(act_in, d_in16, tile, n_pts, tid);
    // ---- input-assembly backward (shader_prep_bwd_f16 on the fp16 dIn row) -> the field's dL/dout tile --------------
    const float* dlog = reinterpret_cast<const float*>(st + S::DLOG);
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int i = 0; i < 8; i += 2) {
        const int row = acc_row(tid, h, i), col = acc_col(tid, i);
        const uint32_t hin = pk(act_in.d[h][i], act_in.d[h][i + 1]);
        *reinterpret_cast<uint32_t*>(sm + S::SDIN + (row * kSdinLd + col) * 2) = hin;   // for d_app
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hin));
        const float g0 = col == 0 ? dlog[row] : f.x * inv_loss_scale, g1 = f.y * inv_loss_scale;
        const uint32_t o = pk(g0 * field_loss_scale, g1 * field_loss_scale);
        *reinterpret_cast<uint32_t*>(sm + S::FDO + sw32_off(row, col >> 3) + ((col & 7) << 1)) = o;
        const int p = tile * kBT + row;
        if (d_scene16 && p < n_pts) *reinterpret_cast<uint32_t*>(d_scene16 + size_t(p) * 16 + col) = o;
      }
    fence_async_smem();
    bar_sync(kBarMma, kBT);                                      // (also: every warp's MMAs are done reading dH0)
    // ---- field F0: H0 = relu(X . W0^T) ----------------------------------------------------------------------------
    wg_fence();
    mma_m128<64, 0, 2>(act, s_fx, 64, s_fw0, 64, false);
    wg_commit();
    wg_wait();
    acc_relu_to_tile(act, sm + S::H0, tid);
    fence_async_smem();
    bar_sync(kBarMma, kBT);
    // ---- field A: dH0 = dOut . Wout ; dWout^T += H0^T . dOut ------------------------------------------------------
    wg_fence();
    mma_m128<64, 1, 1>(act, s_fdo, 32, s_fwo, 128, false);
    mma_batch128<16>(fgwo, s_h0, 128, s_fdo, 32);
    wg_commit();
    wg_wait();
    bar_sync(kBarMma, kBT);                                      // every warp's MMAs are done reading H0
    relu_bwd_epilogue(act, sm + S::H0, sm + S::H0, tid);
    fence_async_smem();
    bar_sync(kBarMma, kBT);
    // ---- field C: dIn = dH0 . W0 ; dW0 += dH0^T . X ---------------------------------------------------------------
    wg_fence();
    mma_m128<32, 1, 4>(act_in, s_h0, 128, s_fw0, 64, false);
    mma_batch128<32>(fgw0, s_h0, 128, s_fx, 64);
    wg_commit();
    wg_wait();
    if (dfeat16) store_din(act_in, dfeat16, tile, n_pts, tid);
    // ---- hand the tile to scatter warpgroup 1 + b ---------------------------------------------------------------------
    unsigned char* slot = sm + S::RING0 + b * S::SLOT_BYTES;
    bar_sync(kBarEmpty + b, 2 * kBT);
#pragma unroll
    for (int h = 0; h < 2; h++)                                  // the same fp16 packing as store_din
#pragma unroll
      for (int i = 0; i < 16; i += 2)
        *reinterpret_cast<uint32_t*>(slot + S::R_DIN + din_off(acc_row(tid, h, i), acc_col(tid, i))) = pk(act_in.d[h][i], act_in.d[h][i + 1]);
#pragma unroll
    for (int q = 0; q < 3; q++)
      reinterpret_cast<uint4*>(slot + S::R_SDIN)[tid + kBT * q] = reinterpret_cast<const uint4*>(sm + S::SDIN)[tid + kBT * q];
    reinterpret_cast<uint4*>(slot + S::R_PTS)[tid] = reinterpret_cast<const uint4*>(st + S::PTS)[tid];   // points + volume ids
    if (tid == 0) *reinterpret_cast<int*>(slot + S::R_TILE) = tile;
    bar_arrive(kBarFull + b, 2 * kBT);
    tile = next;
  }
  for (int q = 0; q < 2; q++, k++) {                             // no more tiles: release both scatter warpgroups
    unsigned char* slot = sm + S::RING0 + (k & 1) * S::SLOT_BYTES;
    bar_sync(kBarEmpty + (k & 1), 2 * kBT);
    if (tid == 0) *reinterpret_cast<int*>(slot + S::R_TILE) = -1;
    bar_arrive(kBarFull + (k & 1), 2 * kBT);
  }
  cp_async_wait<0>();
  if (any) {
    flush_weight_grads<1>(sgw0, sgwo, sgwh, d_sparams, tid);
    flush_weight_grads<0>(fgw0, fgwo, sgwh, d_fparams, tid);
  }
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
  constexpr int bytes = FbsSmem::BYTES;
  cudaFuncSetAttribute(field_bwd_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  // persistent: weight gradients flushed once per CTA
  const int grid = persistent_grid(div_up(n_pts, kBT), resident_per_sm(field_bwd_scatter_kernel, kBT, bytes));
  field_bwd_scatter_kernel<<<grid, kBT, bytes, as_stream(stream)>>>(
      (const __half*)dout_f16, (const __half*)feat_f16, (const __half*)params_f16, n_pts, pts, vol, vol_stride, prim_pool, bias_pool,
      n_volumes, local_size, grad_mul, dparams_f32, grad_table_f32, (__half*)din_f16);
  return check_launch("f2b_field_bwd_scatter");
}

extern "C" int f2b_shade_field_bwd_scatter(const void* d_raw_f16, const void* mlp_in_f16, const void* sparams_f16, const float* d_logit,
                                           const int* pt_emb_idx, float inv_loss_scale, float field_loss_scale, const void* feat_f16,
                                           const void* fparams_f16, int n_pts, const float* pts, const int* vol, int vol_stride,
                                           const int* prim_pool, const float* bias_pool, int n_volumes, int local_size, float grad_mul,
                                           float* d_sparams_f32, float* d_fparams_f32, float* grad_table_f32, float* d_app_emb,
                                           int* ticket, void* d_in16, void* d_scene16, void* dfeat16, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(d_raw_f16 && mlp_in_f16 && sparams_f16 && d_logit && feat_f16 && fparams_f16 && pts && vol && prim_pool && bias_pool &&
                  d_sparams_f32 && d_fparams_f32 && grad_table_f32 && ticket,
              "f2b_shade_field_bwd_scatter: null pointer");
  F2B_REQUIRE(!pt_emb_idx == !d_app_emb, "f2b_shade_field_bwd_scatter: pt_emb_idx and d_app_emb go together");
  F2B_REQUIRE(n_volumes > 0 && local_size > 0 && (local_size % 2) == 0 && vol_stride > 0,
              "f2b_shade_field_bwd_scatter: bad n_volumes/local_size/vol_stride");
  if (cudaMemsetAsync(ticket, 0, sizeof(int), as_stream(stream)) != cudaSuccess) {
    set_error("f2b_shade_field_bwd_scatter: memset failed");
    return F2B_ECUDA;
  }
  constexpr int bytes = SfbSmem::BYTES;
  cudaFuncSetAttribute(shade_field_bwd_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  shade_field_bwd_scatter_kernel<<<persistent_grid(div_up(n_pts, kBT), 1), kSfbThreads, bytes, as_stream(stream)>>>(
      (const __half*)d_raw_f16, (const __half*)mlp_in_f16, (const __half*)sparams_f16, d_logit, pt_emb_idx, inv_loss_scale,
      field_loss_scale, (const __half*)feat_f16, (const __half*)fparams_f16, n_pts, pts, vol, vol_stride, prim_pool, bias_pool, n_volumes,
      local_size, grad_mul, d_sparams_f32, d_fparams_f32, grad_table_f32, d_app_emb, ticket, (__half*)d_in16, (__half*)d_scene16,
      (__half*)dfeat16);
  return check_launch("f2b_shade_field_bwd_scatter");
}

extern "C" int f2b_mlp_bwd2(const void* dout_f16, const void* in_f16, const void* hidden0_f16, const void* hidden1_f16,
                            const void* params_f16, int n_hidden_matmuls, int n_pts, void* din_f16,
                            float* dparams_f32, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(dout_f16 && in_f16 && params_f16 && dparams_f32, "f2b_mlp_bwd: null pointer");
  F2B_REQUIRE(n_hidden_matmuls == 0 || n_hidden_matmuls == 1, "f2b_mlp_bwd: n_hidden_matmuls must be 0 or 1");
  const int n_tiles = div_up(n_pts, kBT);
  // persistent grid: as many CTAs as are resident at once (each flushes its weight gradients once)
#define F2B_BWD_LAUNCH(KERNEL, BYTES, ...)                                                        \
  {                                                                                               \
    cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, BYTES);             \
    const int grid = persistent_grid(n_tiles, resident_per_sm(KERNEL, kBT, BYTES));               \
    KERNEL<<<grid, kBT, BYTES, as_stream(stream)>>>(__VA_ARGS__);                                 \
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
