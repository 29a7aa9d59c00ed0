// mlp_tc.cu — the fully-fused MLP on Hopper's warpgroup tensor-core instructions (impl 1).
//
// Replaces tiny-cuda-nn's wmma 16x16x16 fp16-accumulate kernels (kernel_mlp_fused /
// kernel_mlp_fused_backward, External/tiny-cuda-nn/src/fully_fused_mlp.cu:150-259,499-557) with
// wgmma.mma_async (two m64 x N{64,16} x k16 per K step, fp16 operands from shared memory, fp32 accumulators
// in registers):
//   * one CTA (4 warps = one warpgroup) owns a 128-sample tile;
//   * the layer input is written to shared memory in the canonical K-major swizzled layout
//     (64 B rows / SWIZZLE_64B for K=32, 128 B rows / SWIZZLE_128B for K=64), the weights sit
//     resident in shared memory in the same layouts for the CTA's lifetime (persistent tiles);
//   * the warpgroup issues 2*K/16 wgmmas per layer, waits for them, applies ReLU to its accumulator
//     fragments, rounds to fp16 and writes them straight back to shared memory as the next layer's operand
//     tile — activations never visit HBM except for the optional hidden_save the backward pass needs;
//   * the 16 outputs of a sample are gathered into one thread (thread i == sample i) through an fp32 row
//     buffer in shared memory, so the epilogues below work on whole rows;
//   * global traffic is decoupled from the per-thread row ownership: the next tile's input is fetched with
//     cp.async (16 B per thread, linear sweep of the contiguous 8 KB tile) into the second half of a double
//     buffer while the current tile computes, and each finished activation tile is copied out to hidden_save
//     by all threads as whole 128 B lines WHILE the tensor core is consuming the same tile for the next layer
//     (r01 profile: per-row 16 B stores at 128 B stride + exposed load latency were ~50 % of the stall samples);
//   * several CTAs share an SM (as many as registers and shared memory allow) and overlap each other's MMA
//     round trips.
#include "common.cuh"
#include "tc.cuh"
#include "shader.cuh"

namespace f2b {
using namespace tc;

constexpr int kTcTile = 128;

template <int NH>
struct TcSmem {                         // offsets from a 1024-byte aligned base
  static constexpr int A0 = 0;          // 2 x [128 x 32] f16, SW64   (double-buffered input tile, 2 x 8 KB)
  static constexpr int H0 = 16384;      // [128 x 64] f16, SW128  (16 KB)  layer-0 activations
  static constexpr int H1 = 32768;      // [128 x 64] f16, SW128  (16 KB)  hidden-layer activations (NH only)
  static constexpr int W0 = NH ? 49152 : 32768;   // [64 x 32]  f16, SW64   (4 KB)
  static constexpr int WH = W0 + 4096;            // [64 x 64]  f16, SW128  (8 KB, NH only)
  static constexpr int WO = WH + (NH ? 8192 : 0); // [16 x 64]  f16, SW128  (2 KB)
  static constexpr int BYTES = WO + 2048 + 1024;  // + alignment slack
};

// Input tile (128 rows x 64 B, contiguous in global memory) -> swizzled K-major tile, fully coalesced:
// the CTA's 128 threads sweep the 8 KB linearly, 16 B per thread and pass.
__device__ __forceinline__ void prefetch_input(const __half* __restrict__ in, int tile, int n_pts, uint32_t a0_tile) {
  const int rows = min(kTcTile, n_pts - tile * kTcTile);
  const unsigned char* src = reinterpret_cast<const unsigned char*>(in) + size_t(tile) * kTcTile * 64;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int c = threadIdx.x + kTcTile * j, r = c >> 2;
    cp_async<16>(a0_tile + sw64_off(r, c & 3), src + (r < rows ? size_t(c) * 16 : 0), r < rows ? 16u : 0u);
  }
}

// Activation tile (swizzled, 128 rows x 128 B) -> its contiguous 16 KB slot in the hidden_save array.  Runs
// while the tensor core consumes the same tile: both only read it.
__device__ __forceinline__ void copy_out_hidden(const unsigned char* h_tile, __half* __restrict__ dst_base, int tile, int n_pts) {
  const int rows = min(kTcTile, n_pts - tile * kTcTile);
  uint4* dst = reinterpret_cast<uint4*>(dst_base + size_t(tile) * kTcTile * 64);
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int c = threadIdx.x + kTcTile * j, r = c >> 3;
    if (r < rows) dst[c] = *reinterpret_cast<const uint4*>(h_tile + sw128_off(r, c & 7));
  }
}

// Work that follows (or precedes) the MLP in Renderer::Render, done in its output epilogue while the row is in registers:
//   EPI_SHADE (field MLP, NH = 0): the shading-feature assembly of Renderer.cpp:179-187 + SHShader.cpp:23-26 — the thread
//     turns its 16 outputs into the shader MLP's fp16 input row ([1, feat 1..15] + appearance embedding | SH4(dir)) and
//     the density logit; the fp32 [P,16] scene_feat tensor and the separate assembly kernel disappear;
//   EPI_RGB (shader MLP, NH = 1): the scaled sigmoid of SHShader.cpp:27-28 -> rgb [P,3] next to the raw fp16 output.
enum { EPI_NONE = 0, EPI_SHADE = 1, EPI_RGB = 2 };
struct EpiArgs {
  const float* dirs;          // [P,3]                     (SHADE)
  const float* app_emb;       // [n_emb,16] or NULL         (SHADE)
  const int* pt_emb_idx;      // [P] or NULL                (SHADE)
  float* logit;               // [P]                        (SHADE)
  __half* mlp_in;             // [P,32]                     (SHADE)
  float* rgb;                 // [P,3]                      (RGB)
};

template <int NH, int EPI>
__global__ void __launch_bounds__(kTcTile)
mlp_fwd_tc_kernel(const __half* __restrict__ in, const __half* __restrict__ params, int n_pts,
                  __half* __restrict__ out, float* __restrict__ out_f32, __half* __restrict__ hidden_save, EpiArgs epi) {
  using S = TcSmem<NH>;
  unsigned char* sm = smem_base();
  float* s_rows = reinterpret_cast<float*>(sm + S::H0);             // output rows [128][20] fp32 (H0 is dead by then)
  const int tid = threadIdx.x;
  const int n_tiles = (n_pts + kTcTile - 1) / kTcTile;
  const uint32_t a0 = smem_u32(sm + S::A0);

  int tile = blockIdx.x;
  if (tile < n_tiles) prefetch_input(in, tile, n_pts, a0);       // overlaps the weight staging
  cp_async_commit();
  stage_weights<32, 0>(params, 64, sm + S::W0, tid);
  if (NH) stage_weights<64, 0>(params + 64 * 32, 64, sm + S::WH, tid);
  stage_weights<64, 0>(params + 64 * 32 + NH * 64 * 64, 16, sm + S::WO, tid);

  const uint32_t h0 = smem_u32(sm + S::H0), h1 = smem_u32(sm + S::H1);
  const uint32_t w0 = smem_u32(sm + S::W0), wh = smem_u32(sm + S::WH), wo = smem_u32(sm + S::WO);
  uint32_t buf = 0;
  Acc<64> acc;
  Acc<16> acc_out;

  for (; tile < n_tiles; tile += gridDim.x, buf ^= 1) {
    const int p = tile * kTcTile + tid;
    const bool valid = p < n_pts;
    // ---- input: tile i has been in flight since the previous iteration; start tile i+1 now ---------
    const int next = tile + gridDim.x;
    if (next < n_tiles) prefetch_input(in, next, n_pts, a0 + (buf ^ 1) * 8192);
    cp_async_commit();
    cp_async_wait<1>();                                          // everything but the newest group has landed
    fence_async_smem();
    __syncthreads();                                             // (also: the previous tile's output rows have been read)
    // ---- layer 0: D[128x64] = A0[128x32] . W0^T ------------------------------------------------
    wg_fence();
    mma_m128<64, 0, 2>(acc, a0 + buf * 8192, 64, w0, 64, false);
    wg_commit();
    wg_wait();
    acc_relu_to_tile(acc, sm + S::H0, tid);
    fence_async_smem();
    __syncthreads();
    if (NH) {
      // ---- hidden layer: D[128x64] = H0[128x64] . Wh^T ---------------------------------------------
      wg_fence();
      mma_m128<64, 0, 4>(acc, h0, 128, wh, 128, false);
      wg_commit();
      if (hidden_save) copy_out_hidden(sm + S::H0, hidden_save, tile, n_pts);        // while the MMA runs
      wg_wait();
      acc_relu_to_tile(acc, sm + S::H1, tid);
      fence_async_smem();
      __syncthreads();
    }
    // ---- output layer: D[128x16] = H_last[128x64] . Wout^T (linear) ----------------------------------
    wg_fence();
    mma_m128<16, 0, 4>(acc_out, NH ? h1 : h0, 128, wo, 128, false);
    wg_commit();
    if (hidden_save) copy_out_hidden(sm + (NH ? S::H1 : S::H0), hidden_save + size_t(NH) * n_pts * 64, tile, n_pts);
    wg_wait();
    __syncthreads();                                             // every warp is done with H0 (operand / copy-out)
    acc_to_rows(acc_out, s_rows, kRowLd16, tid);
    __syncthreads();
    {
      uint32_t r[16];
      row_ld16(s_rows, kRowLd16, tid, r);
      if (valid) {
        uint4 v0, v1;
        v0.x = pk(__uint_as_float(r[0]), __uint_as_float(r[1]));   v0.y = pk(__uint_as_float(r[2]), __uint_as_float(r[3]));
        v0.z = pk(__uint_as_float(r[4]), __uint_as_float(r[5]));   v0.w = pk(__uint_as_float(r[6]), __uint_as_float(r[7]));
        v1.x = pk(__uint_as_float(r[8]), __uint_as_float(r[9]));   v1.y = pk(__uint_as_float(r[10]), __uint_as_float(r[11]));
        v1.z = pk(__uint_as_float(r[12]), __uint_as_float(r[13])); v1.w = pk(__uint_as_float(r[14]), __uint_as_float(r[15]));
        if (out) {
          uint4* dst = reinterpret_cast<uint4*>(out + size_t(p) * 16);
          dst[0] = v0; dst[1] = v1;
        }
        if (out_f32) {                                           // the fp16-rounded values, widened (TCNNWP.cpp:112)
          const __half2* h = reinterpret_cast<const __half2*>(&v0);
          const __half2* g = reinterpret_cast<const __half2*>(&v1);
          float4* dst = reinterpret_cast<float4*>(out_f32 + size_t(p) * 16);
          const float2 a = __half22float2(h[0]), b = __half22float2(h[1]), c = __half22float2(h[2]), d = __half22float2(h[3]);
          const float2 e = __half22float2(g[0]), f = __half22float2(g[1]), u = __half22float2(g[2]), w = __half22float2(g[3]);
          dst[0] = make_float4(a.x, a.y, b.x, b.y); dst[1] = make_float4(c.x, c.y, d.x, d.y);
          dst[2] = make_float4(e.x, e.y, f.x, f.y); dst[3] = make_float4(u.x, u.y, w.x, w.y);
        }
        if (EPI == EPI_RGB) {
          const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v0.x));
          const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&v0.y));
          float* dst = epi.rgb + size_t(p) * 3;
          dst[0] = shade_act(a.x); dst[1] = shade_act(a.y); dst[2] = shade_act(b.x);
        }
      }
      if (EPI == EPI_SHADE) {
        // my row of the shader MLP's input, staged in the (now dead) input tile of this iteration and copied out as whole
        // lines by all threads; the density logit goes out directly (4 B per thread, contiguous per warp)
        unsigned char* stage = sm + S::A0 + buf * 8192;
        uint4 row[4] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
        if (valid) {
          uint4 v0, v1;
          v0.x = pk(__uint_as_float(r[0]), __uint_as_float(r[1]));   v0.y = pk(__uint_as_float(r[2]), __uint_as_float(r[3]));
          v0.z = pk(__uint_as_float(r[4]), __uint_as_float(r[5]));   v0.w = pk(__uint_as_float(r[6]), __uint_as_float(r[7]));
          v1.x = pk(__uint_as_float(r[8]), __uint_as_float(r[9]));   v1.y = pk(__uint_as_float(r[10]), __uint_as_float(r[11]));
          v1.z = pk(__uint_as_float(r[12]), __uint_as_float(r[13])); v1.w = pk(__uint_as_float(r[14]), __uint_as_float(r[15]));
          float feat[16];
          const __half2* h = reinterpret_cast<const __half2*>(&v0);
          const __half2* g = reinterpret_cast<const __half2*>(&v1);
#pragma unroll
          for (int k = 0; k < 4; k++) {
            const float2 a = __half22float2(h[k]), b = __half22float2(g[k]);
            feat[2 * k] = a.x; feat[2 * k + 1] = a.y; feat[8 + 2 * k] = b.x; feat[8 + 2 * k + 1] = b.y;
          }
          epi.logit[p] = feat[0];
          const float* emb_row = epi.app_emb ? epi.app_emb + size_t(__ldg(epi.pt_emb_idx + p)) * 16 : nullptr;
          shade_row(feat, emb_row, __ldg(epi.dirs + size_t(p) * 3), __ldg(epi.dirs + size_t(p) * 3 + 1),
                    __ldg(epi.dirs + size_t(p) * 3 + 2), row);
        }
#pragma unroll
        for (int c = 0; c < 4; c++) *reinterpret_cast<uint4*>(stage + sw64_off(tid, c)) = row[c];
        __syncthreads();
        const int rows = min(kTcTile, n_pts - tile * kTcTile);
        uint4* dst = reinterpret_cast<uint4*>(epi.mlp_in + size_t(tile) * kTcTile * 32);
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const int c = tid + kTcTile * j, rr = c >> 2;
          if (rr < rows) dst[c] = *reinterpret_cast<const uint4*>(stage + sw64_off(rr, c & 3));
        }
        __syncthreads();                                         // the stage is the next-but-one tile's prefetch target
      }
    }
  }
  cp_async_wait<0>();
}

}  // namespace f2b

using namespace f2b;

template <int NH, int EPI>
static void launch_fwd(const void* in_f16, const void* params_f16, int n_pts, void* out_f16, float* out_f32,
                       void* hidden_save_f16, const EpiArgs& epi, void* stream) {
  cudaFuncSetAttribute(mlp_fwd_tc_kernel<NH, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcSmem<NH>::BYTES);
  const int grid = persistent_grid(div_up(n_pts, kTcTile), resident_per_sm(mlp_fwd_tc_kernel<NH, EPI>, kTcTile, TcSmem<NH>::BYTES));
  mlp_fwd_tc_kernel<NH, EPI><<<grid, kTcTile, TcSmem<NH>::BYTES, as_stream(stream)>>>(
      (const __half*)in_f16, (const __half*)params_f16, n_pts, (__half*)out_f16, out_f32, (__half*)hidden_save_f16, epi);
}

extern "C" int f2b_mlp_fwd(const void* in_f16, const void* params_f16, int n_hidden_matmuls, int n_pts,
                           void* out_f16, void* hidden_save_f16, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(in_f16 && params_f16 && out_f16, "f2b_mlp_fwd: null pointer");
  F2B_REQUIRE(n_hidden_matmuls == 0 || n_hidden_matmuls == 1, "f2b_mlp_fwd: n_hidden_matmuls must be 0 or 1");
  const EpiArgs none = {};
  if (n_hidden_matmuls == 0) launch_fwd<0, EPI_NONE>(in_f16, params_f16, n_pts, out_f16, nullptr, hidden_save_f16, none, stream);
  else launch_fwd<1, EPI_NONE>(in_f16, params_f16, n_pts, out_f16, nullptr, hidden_save_f16, none, stream);
  return check_launch("f2b_mlp_fwd(wgmma)");
}

// Same network, output widened to fp32 in the epilogue (what TCNNWP::Query hands back, TCNNWP.cpp:112):
// out_f32 [P,16] and/or out_f16 [P,16] (either may be NULL, not both).
extern "C" int f2b_mlp_fwd_f32(const void* in_f16, const void* params_f16, int n_hidden_matmuls, int n_pts,
                               float* out_f32, void* out_f16, void* hidden_save_f16, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(in_f16 && params_f16 && (out_f32 || out_f16), "f2b_mlp_fwd_f32: null pointer");
  F2B_REQUIRE(n_hidden_matmuls == 0 || n_hidden_matmuls == 1, "f2b_mlp_fwd_f32: n_hidden_matmuls must be 0 or 1");
  const EpiArgs none = {};
  if (n_hidden_matmuls == 0) launch_fwd<0, EPI_NONE>(in_f16, params_f16, n_pts, out_f16, out_f32, hidden_save_f16, none, stream);
  else launch_fwd<1, EPI_NONE>(in_f16, params_f16, n_pts, out_f16, out_f32, hidden_save_f16, none, stream);
  return check_launch("f2b_mlp_fwd_f32(wgmma)");
}

// The MLP entry points always run the wgmma kernels (1).
extern "C" int f2b_get_mlp_impl(void) { return 1; }

// Field MLP (32 -> 64 -> 16) on encoded features + the shading-feature assembly in its epilogue:
// logit[p] = out[p,0]; mlp_in[p] = fp16([1, out[p,1:16]] + app_emb[pt_emb_idx[p]] | SH4(dirs[p])).

extern "C" int f2b_field_shade_fwd(const void* feat_f16, const void* field_params_f16, const float* dirs, const float* app_emb,
                                   const int* pt_emb_idx, int n_pts, float* logit, void* mlp_in_f16, void* hidden_save_f16,
                                   void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(feat_f16 && field_params_f16 && dirs && logit && mlp_in_f16, "f2b_field_shade_fwd: null pointer");
  F2B_REQUIRE(!app_emb || pt_emb_idx, "f2b_field_shade_fwd: app_emb without pt_emb_idx");
  EpiArgs e = {};
  e.dirs = dirs; e.app_emb = app_emb; e.pt_emb_idx = pt_emb_idx; e.logit = logit; e.mlp_in = (__half*)mlp_in_f16;
  launch_fwd<0, EPI_SHADE>(feat_f16, field_params_f16, n_pts, nullptr, nullptr, hidden_save_f16, e, stream);
  return check_launch("f2b_field_shade_fwd");
}

// Shader MLP (32 -> 64 -> 64 -> 16) + the colour activation in its epilogue: raw [P,16] fp16 (the backward needs it)
// and rgb [P,3] = (1 + 2e-3) * sigmoid(raw[:, :3]) - 1e-3.
extern "C" int f2b_shader_mlp_rgb_fwd(const void* mlp_in_f16, const void* shader_params_f16, int n_pts, void* raw_f16,
                                      float* rgb, void* hidden_save_f16, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(mlp_in_f16 && shader_params_f16 && raw_f16 && rgb, "f2b_shader_mlp_rgb_fwd: null pointer");
  EpiArgs e = {};
  e.rgb = rgb;
  launch_fwd<1, EPI_RGB>(mlp_in_f16, shader_params_f16, n_pts, raw_f16, nullptr, hidden_save_f16, e, stream);
  return check_launch("f2b_shader_mlp_rgb_fwd");
}
