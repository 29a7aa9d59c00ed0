// fused_fwd.cu — the forward-only (VALIDATE) half of Renderer::Render as ONE kernel behind the ray march:
//   hash encode -> field MLP -> early stop -> shading-feature assembly + SH -> shader MLP -> colour activation -> composite.
//
// Replaces, for a no-grad batch (ExpRunner::RenderWholeImage -> Renderer::Render, src/ExpRunner.cpp:257-293,
// src/Renderer/Renderer.cpp:107-208): the early-stop AnchoredQuery over ALL samples, the where / index compaction, the second
// AnchoredQuery on the survivors, SHShader::Query, and the ~25 ATen passes of the composite — i.e. every per-sample tensor
// between the march's output and the per-ray result.  Nothing per-sample goes to HBM: a sample costs 28 B read from the march's
// slots + its 128 table gathers (SURVEY.md §8d "fused forward pipeline": 512 B/pt of gathers is the whole traffic).
//
// Shape: a "walker" (128 threads = one warpgroup, thread i == sample i) walks ONE RAY front to back, a 128-sample tile at a
// time, and carries the ray's optical depth across tiles; a CTA is one walker.  Because the reference's early-stop mask `T_i > 1e-4`
// (Renderer.cpp:125) is a prefix of the ray (tau >= 0 => T non-increasing), the walk simply ENDS at the first tile whose
// leading sample is already opaque: the samples behind it are never encoded (the unfused path encodes every marched sample,
// then drops them).  No occupancy votes are taken in VALIDATE mode, so nothing downstream needs those samples.
// Rays are handed out through an atomic ticket (ray lengths differ by 10x).
//
// Arithmetic is the unfused path's, operation for operation: encode_point (hash.cuh), the two wgmma MLPs with the same
// operand tiles (row results do not depend on which other rows share the tile), shade_row / shade_act (shader.cuh), and the
// composite's SERIAL left-to-right sums (FlexOps.cu:5-73 order, as composite.cu) — colours / depth / disparity / weights come
// out bit-identical to f2b_render_phase1 + _phase2_fwd (tests/test_gpu_render.py::test_fused_forward_matches_unfused).
// f2b_render_fwd_fused_app is the same kernel with one appearance row added to every ray's shader input (DESIGN.md §3m), bit-identical
// to the launch sequences with that row as a [1,16] table (tests/test_gpu_appearance.py).
// f2b_render_fwd_fused_crop renders only what a crop box keeps (DESIGN.md §3n): a sample whose world point fma(t, d, o) the box
// removes has density 0 (tau = alpha = weight = +0) and is never encoded, and a tile the box removes whole skips both MLPs.  The result is
// bit-identical to the same kernel over a slot layout with the removed samples deleted (tests/test_gpu_crop.py).
#include "common.cuh"
#include "crop.cuh"
#include "hash.cuh"
#include "shader.cuh"
#include "tc.cuh"

namespace f2b {
using namespace tc;

constexpr int kRT = 128;

// Shared memory of a CTA (one ray walker, 128 threads):
//   [0, 20 KB) the two MLPs' weights | A0 8 KB + H0 16 KB | ray ticket + level scales (+ the appearance row, kApp only).  The
//   composite's scratch (tau, optical depth, the five addend rows) lives inside the walker's H0 tile, which is dead whenever the
//   scratch is live (between an MLP's last MMA and the next MLP's first epilogue).
struct FusedSmem {
  static constexpr int SWH = 0;           // shader Wh   [64 x 64] SW128  8 KB
  static constexpr int FWO = 8192;        // field  Wout [16 x 64] SW128  2 KB
  static constexpr int SWO = 10240;       // shader Wout [16 x 64] SW128  2 KB
  static constexpr int FW0 = 12288;       // field  W0   [64 x 32] SW64   4 KB
  static constexpr int SW0 = 16384;       // shader W0   [64 x 32] SW64   4 KB
  static constexpr int WALK0 = 20480;     // the walker's A0, H0 behind it
  static constexpr int WALK = 8192 + 16384;
  static constexpr int A0 = 0;            // [128 x 32] f16 SW64   8 KB   encoded features, then the shader MLP's input rows
  static constexpr int H0 = 8192;         // [128 x 64] f16 SW128 16 KB   hidden activations (both MLPs, rewritten in place)
  static constexpr int TAU = H0;          // float tau[128]          (inside H0)
  static constexpr int ACC = H0 + 512;    // float acc[129]
  static constexpr int ADD = H0 + 2048;   // float add[5][128]
  static constexpr int ROWS = H0 + 4608;  // float rows[128][20]     (inside H0) an MLP's 16 outputs per sample
  static constexpr int BAR = WALK0 + WALK;        // 16 B: ray ticket (4); then 16 B | 16 level scales
  static constexpr int BYTES = BAR + 16 + 16 + 64 + 1024;   // + alignment slack (the tiles need 1024-byte alignment)
  static constexpr int EMB = BAR + 16 + 16 + 64;  // float emb[16]: the appearance row of every ray of the launch (kApp only)
  static constexpr int BYTES_APP = BYTES + 64;
};

__device__ __forceinline__ float h16(uint32_t acc_bits) { return __half2float(__float2half_rn(__uint_as_float(acc_bits))); }

// barrier over the walker's 128 threads (named barrier 1; barrier 0 stays the CTA-wide one)
__device__ __forceinline__ void walker_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
__device__ __forceinline__ int walker_sync_count(bool pred) {
  int n;
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %1, 0;\n\tbar.red.popc.u32 %0, 1, 128, p;\n\t}\n" : "=r"(n) : "r"((int)pred) : "memory");
  return n;
}

// 3 CTAs per SM, <= 168 registers: the wgmma accumulators live in registers.  kApp: every ray is shaded with the one appearance
// row app_emb [16], staged in shared memory once per CTA (read there by the shading-input assembly, not held in registers).
// kCrop: samples whose world point fma(t, d, o) `crop` does not keep have density 0 (crop.cuh); the box stays in the parameter
// bank.  (slot_pts are the warped coordinates the encode reads, so the point is formed from the slot's t and the ray, rays_o [R,3].)
template <bool kApp, bool kCrop>
__global__ void __launch_bounds__(kRT, 3)
render_fwd_fused_kernel(const __half* __restrict__ table, const int* __restrict__ prim_pool, const float* __restrict__ bias_pool,
                        int n_volumes, int local_size, const __half* __restrict__ fparams, const __half* __restrict__ sparams,
                        const float* __restrict__ s_pts, const float* __restrict__ s_dt, const float* __restrict__ s_t,
                        const int* __restrict__ s_anchors, const int* __restrict__ counts, const float* __restrict__ rays_d,
                        const float* __restrict__ bg, int n_rays, int slot, const int* __restrict__ total_all,
                        int* __restrict__ ticket, float* __restrict__ colors, float* __restrict__ disparity,
                        float* __restrict__ depth, int* __restrict__ kept_counts, float* __restrict__ weights_slots,
                        const float* __restrict__ app_emb, const CropBox crop, const float* __restrict__ rays_o) {
  using S = FusedSmem;
  unsigned char* sm = smem_base();
  const int tid = threadIdx.x;                                   // thread == sample
  unsigned char* wsm = sm + S::WALK0;
  int* s_ray = reinterpret_cast<int*>(sm + S::BAR);
  float* s_scale = reinterpret_cast<float*>(sm + S::BAR + 16 + 16);
  float* s_emb = reinterpret_cast<float*>(sm + S::EMB);
  float* s_tau = reinterpret_cast<float*>(wsm + S::TAU);
  float* s_acc = reinterpret_cast<float*>(wsm + S::ACC);         // exclusive optical depth per sample, [128] = inclusive end
  float* s_add = reinterpret_cast<float*>(wsm + S::ADD);         // [5][128] addends of the five per-ray sums
  float* s_rows = reinterpret_cast<float*>(wsm + S::ROWS);

  stage_weights<32, 0>(fparams, 64, sm + S::FW0, tid);
  stage_weights<64, 0>(fparams + 64 * 32, 16, sm + S::FWO, tid);
  stage_weights<32, 0>(sparams, 64, sm + S::SW0, tid);
  stage_weights<64, 0>(sparams + 64 * 32, 64, sm + S::SWH, tid);
  stage_weights<64, 0>(sparams + 64 * 32 + 64 * 64, 16, sm + S::SWO, tid);
  if (threadIdx.x < F2B_N_LEVELS) s_scale[threadIdx.x] = level_scale(threadIdx.x);
  if (kApp && threadIdx.x < 16) s_emb[threadIdx.x] = __ldg(app_emb + threadIdx.x);
  fence_async_smem();
  __syncthreads();
  const uint32_t a0 = smem_u32(wsm + S::A0), h0 = smem_u32(wsm + S::H0);
  const uint32_t fw0 = smem_u32(sm + S::FW0), fwo = smem_u32(sm + S::FWO);
  const uint32_t sw0 = smem_u32(sm + S::SW0), swh = smem_u32(sm + S::SWH), swo = smem_u32(sm + S::SWO);
  Acc<64> acc;
  Acc<16> acc_out;
  const bool empty_batch = total_all && (__ldg(total_all) <= 0);   // Renderer.cpp:83-97: no sample in the WHOLE batch

  // one MMA group issued by the CTA's warpgroup, which waits for it
#define F2B_MMA_STAGE(...) \
  do {                     \
    wg_fence();            \
    __VA_ARGS__;           \
    wg_commit();           \
    wg_wait();             \
  } while (0)
  // the walker's 16 outputs per sample -> my row (the rows sit in H0, the operand of the MMA just completed)
#define F2B_OUT_ROW(r)                               \
  do {                                               \
    walker_sync();                                   \
    acc_to_rows(acc_out, s_rows, kRowLd16, tid);     \
    walker_sync();                                   \
    row_ld16(s_rows, kRowLd16, tid, r);              \
  } while (0)

  for (;;) {
    if (tid == 0) *s_ray = atomicAdd(ticket, 1);
    walker_sync();
    const int ray = *s_ray;
    if (ray >= n_rays) break;
    const int cnt = __ldg(counts + ray);
    const size_t base = size_t(ray) * slot;
    const float dx = __ldg(rays_d + ray * 3), dy = __ldg(rays_d + ray * 3 + 1), dz = __ldg(rays_d + ray * 3 + 2);
    float run = 0.f;                                             // thread 0: optical depth in front of the current tile
    float acc5 = 0.f;                                            // threads 0..4: the five per-ray sums (r, g, b, w/t, w*t)
    float run_end = 0.f;                                         // thread 0: optical depth behind the last KEPT sample
    int n_kept = 0;
    for (int t0 = 0; t0 < cnt; t0 += kRT) {
      const int nv = min(kRT, cnt - t0);
      const bool valid = tid < nv;
      const size_t p = base + t0 + tid;
      // ---- crop: a removed sample is a padding lane with density 0 -----------------------------------------------
      bool in_crop = true;                                       // (kCrop) my sample is kept by the box
      if (kCrop) {
        if (valid) {
          const float t = __ldg(s_t + p);
          in_crop = crop_keep(crop, ffma(t, dx, __ldg(rays_o + ray * 3)), ffma(t, dy, __ldg(rays_o + ray * 3 + 1)),
                              ffma(t, dz, __ldg(rays_o + ray * 3 + 2)));
        }
        if (walker_sync_count(valid && in_crop) == 0) {          // the box removes the whole tile: every sample has T = exp(-run),
          if (walker_sync_count(tid == 0 && expf(-run) > 1e-4f) == 0) break;   // so all of them are kept (weight 0), or none
          if (valid && weights_slots) weights_slots[p] = 0.f;
          n_kept += nv;                                          // run and run_end stay: the tile adds no optical depth
          continue;
        }
      }
      // ---- encode my sample -> operand row ------------------------------------------------------------------------
      uint32_t enc[16];
      float dt_i = 0.f;
      if (valid && in_crop) {
        encode_point(table, prim_pool, bias_pool, n_volumes, local_size, s_scale, __ldg(s_pts + p * 3), __ldg(s_pts + p * 3 + 1),
                     __ldg(s_pts + p * 3 + 2), __ldg(s_anchors + p * 2), enc);
        dt_i = __ldg(s_dt + p);
      } else {
#pragma unroll
        for (int l = 0; l < 16; l++) enc[l] = 0u;
      }
#pragma unroll
      for (int c = 0; c < 4; c++)
        *reinterpret_cast<uint4*>(wsm + S::A0 + sw64_off(tid, c)) = make_uint4(enc[4 * c], enc[4 * c + 1], enc[4 * c + 2], enc[4 * c + 3]);
      fence_async_smem();
      walker_sync();                                             // (also: the previous tile's sums have been read out of H0)
      // ---- field MLP: 32 -> 64 (ReLU) -> 16 -------------------------------------------------------------------------
      F2B_MMA_STAGE(mma_m128<64, 0, 2>(acc, a0, 64, fw0, 64, false));
      acc_relu_to_tile(acc, wsm + S::H0, tid);
      fence_async_smem();
      walker_sync();
      F2B_MMA_STAGE(mma_m128<16, 0, 4>(acc_out, h0, 128, fwo, 128, false));
      float feat[16];
      {
        uint32_t r[16];
        F2B_OUT_ROW(r);
#pragma unroll
        for (int k = 0; k < 16; k++) feat[k] = h16(r[k]);        // the fp16-rounded outputs TCNNWP::Query returns
      }
      // ---- early stop: optical depth in serial order, transmittance, keep = T > 1e-4 (Renderer.cpp:115-126) ----------
      // (H0 is dead from here to the shader MLP's first epilogue: tau / acc live in it)
      float tau = 0.f, alpha = 0.f;                              // +0 for padding lanes and removed samples
      if (valid && in_crop) {
        const float dens = expf(fsub(feat[0], 3.f));             // TruncExp(x - 3)
        tau = fmul(dens, dt_i);
        alpha = fsub(1.f, expf(-tau));
      }
      s_tau[tid] = tau;
      walker_sync();
      if (tid == 0) {                                            // fixed trip count (lanes past nv hold tau = +0: x + 0 == x), so the
        float a = run;                                           // loads pipeline ahead of the 128-long dependent add chain
#pragma unroll 16
        for (int j = 0; j < kRT; j++) { s_acc[j] = a; a = fadd(a, s_tau[j]); }
        s_acc[kRT] = a;
        run = a;
      }
      walker_sync();
      const float trans = expf(-s_acc[tid < nv ? tid : 0]);
      const bool keep = valid && (trans > 1e-4f);
      const int nk = walker_sync_count(keep);                    // kept samples are a prefix of the ray: the first nk of the tile
      if (tid == 0) run_end = s_acc[nk];
      if (nk == 0) break;                                        // the ray is opaque in front of this tile: done (walker-uniform)
      // ---- shader MLP input: [1, feat 1..15 | SH4(dir)] -> 64 -> 64 -> 16, colour activation --------------------------
      {
        uint4 row[4] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
        if (valid && in_crop) shade_row_t<true>(feat, kApp ? s_emb : nullptr, dx, dy, dz, row);
#pragma unroll
        for (int c = 0; c < 4; c++) *reinterpret_cast<uint4*>(wsm + S::A0 + sw64_off(tid, c)) = row[c];
      }
      fence_async_smem();
      walker_sync();                                             // (thread 0 has read acc[nk]: H0 may be overwritten again)
      F2B_MMA_STAGE(mma_m128<64, 0, 2>(acc, a0, 64, sw0, 64, false));
      acc_relu_to_tile(acc, wsm + S::H0, tid);
      fence_async_smem();
      walker_sync();
      F2B_MMA_STAGE(mma_m128<64, 0, 4>(acc, h0, 128, swh, 128, false));
      walker_sync();                                             // in place: every warp's part of the hidden layer's MMA has completed
      acc_relu_to_tile(acc, wsm + S::H0, tid);
      fence_async_smem();
      walker_sync();
      F2B_MMA_STAGE(mma_m128<16, 0, 4>(acc_out, h0, 128, swo, 128, false));
      {                                                          // (H0 is dead again: the five addend rows live in it)
        uint32_t r[16];
        F2B_OUT_ROW(r);
        float w = 0.f, cr = 0.f, cg = 0.f, cb = 0.f, ts = 1.f;
        if (keep) {
          cr = shade_act(h16(r[0])); cg = shade_act(h16(r[1])); cb = shade_act(h16(r[2]));
          w = fmul(trans, alpha);
          ts = fadd(__ldg(s_t + p), 1e-2f);
          if (weights_slots) weights_slots[p] = w;
        }
        s_add[0 * 128 + tid] = fmul(w, cr); s_add[1 * 128 + tid] = fmul(w, cg); s_add[2 * 128 + tid] = fmul(w, cb);
        s_add[3 * 128 + tid] = fdiv(w, ts); s_add[4 * 128 + tid] = fmul(w, ts);
      }
      walker_sync();
      if (tid < 5) {                                             // FlexOps::Sum order: serial, left to right; samples that are not
        const float* mine = s_add + tid * 128;                   // kept add +0 (w = 0), which leaves the running sum bit-identical
#pragma unroll 16
        for (int j = 0; j < kRT; j++) acc5 = fadd(acc5, mine[j]);
      }
      n_kept += nk;
      if (nk < nv) break;                                        // terminated inside this tile
    }
    // ---- per-ray results (Renderer.cpp:196-208; empty batch :83-97) -------------------------------------------------
    walker_sync();                                               // the sums above have been read out of the addend rows
    if (tid < 5) s_add[tid] = acc5;
    walker_sync();
    if (tid == 0) {
      const float lt = expf(-run_end);                           // last_trans = exp(-Sum(sec_density)) over the kept samples
      colors[ray * 3 + 0] = fadd(s_add[0], fmul(lt, bg[ray * 3 + 0]));
      colors[ray * 3 + 1] = fadd(s_add[1], fmul(lt, bg[ray * 3 + 1]));
      colors[ray * 3 + 2] = fadd(s_add[2], fmul(lt, bg[ray * 3 + 2]));
      disparity[ray] = s_add[3];
      depth[ray] = empty_batch ? 512.f : fdiv(s_add[4], fadd(fsub(1.f, lt), 1e-4f));
      kept_counts[ray] = n_kept;
    }
  }
#undef F2B_MMA_STAGE
#undef F2B_OUT_ROW
}

// kept[i] = crop_keep(pts[i]) for n points (f2b_crop_mask)
__global__ void __launch_bounds__(256)
crop_mask_kernel(const float* __restrict__ pts, int n, const CropBox crop, uint8_t* __restrict__ kept) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) kept[i] = crop_keep(crop, __ldg(pts + size_t(i) * 3), __ldg(pts + size_t(i) * 3 + 1), __ldg(pts + size_t(i) * 3 + 2));
}

// weights of the kept samples out of the slot layout into the reference's packed layout (RenderResult.weights, Renderer.h:24)
__global__ void __launch_bounds__(256)
gather_kept_weights_kernel(const float* __restrict__ w_slots, const int* __restrict__ new_bounds, int n_rays, int slot,
                           float* __restrict__ weights) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_rays) return;
  const int beg = new_bounds[2 * ray], n = new_bounds[2 * ray + 1] - beg;
  const float* src = w_slots + size_t(ray) * slot;
  for (int i = lane; i < n; i += 32) weights[beg + i] = src[i];
}

}  // namespace f2b

using namespace f2b;

namespace {
template <bool kApp, bool kCrop>
int launch_render_fwd_fused(const char* name, const void* table_f16, const int* prim_pool, const float* bias_pool, int n_volumes,
                            int local_size, const void* field_params_f16, const void* shader_params_f16, const float* slot_pts,
                            const float* slot_dt, const float* slot_t, const int* slot_anchors, const int* ray_counts,
                            const float* rays_d, const float* bg, int n_rays, int slot_size, const int* total_all, int* ticket,
                            float* colors, float* disparity, float* depth, int* kept_counts, float* weights_slots,
                            const float* app_emb, const CropBox& crop, const float* rays_o, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(table_f16 && prim_pool && bias_pool && field_params_f16 && shader_params_f16 && slot_pts && slot_dt && slot_t &&
                  slot_anchors && ray_counts && rays_d && bg && ticket && colors && disparity && depth && kept_counts &&
                  (!kApp || app_emb) && (!kCrop || rays_o),
              "%s: null pointer", name);
  F2B_REQUIRE(n_volumes > 0 && local_size > 0 && (local_size % 2) == 0, "%s: bad n_volumes/local_size", name);
  F2B_REQUIRE(slot_size > 0 && int64_t(n_rays) * slot_size < (int64_t(1) << 31), "%s: n_rays * slot_size overflows int32", name);
  if (cudaMemsetAsync(ticket, 0, sizeof(int), as_stream(stream)) != cudaSuccess) { set_error("%s: memset failed", name); return F2B_ECUDA; }
  const int smem = kApp ? FusedSmem::BYTES_APP : FusedSmem::BYTES;
  cudaFuncSetAttribute(render_fwd_fused_kernel<kApp, kCrop>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  const int grid = persistent_grid(n_rays, resident_per_sm(render_fwd_fused_kernel<kApp, kCrop>, kRT, smem));
  render_fwd_fused_kernel<kApp, kCrop><<<grid, kRT, smem, as_stream(stream)>>>(
      (const __half*)table_f16, prim_pool, bias_pool, n_volumes, local_size, (const __half*)field_params_f16,
      (const __half*)shader_params_f16, slot_pts, slot_dt, slot_t, slot_anchors, ray_counts, rays_d, bg, n_rays, slot_size,
      total_all, ticket, colors, disparity, depth, kept_counts, weights_slots, app_emb, crop, rays_o);
  return check_launch(name);
}
}  // namespace

extern "C" int f2b_render_fwd_fused(const void* table_f16, const int* prim_pool, const float* bias_pool, int n_volumes, int local_size,
                                    const void* field_params_f16, const void* shader_params_f16, const float* slot_pts,
                                    const float* slot_dt, const float* slot_t, const int* slot_anchors, const int* ray_counts,
                                    const float* rays_d, const float* bg, int n_rays, int slot_size, const int* total_all,
                                    int* ticket, float* colors, float* disparity, float* depth, int* kept_counts,
                                    float* weights_slots, void* stream) {
  return launch_render_fwd_fused<false, false>("f2b_render_fwd_fused", table_f16, prim_pool, bias_pool, n_volumes, local_size,
                                        field_params_f16, shader_params_f16, slot_pts, slot_dt, slot_t, slot_anchors, ray_counts,
                                        rays_d, bg, n_rays, slot_size, total_all, ticket, colors, disparity, depth, kept_counts,
                                        weights_slots, nullptr, CropBox{}, nullptr, stream);
}

extern "C" int f2b_render_fwd_fused_app(const void* table_f16, const int* prim_pool, const float* bias_pool, int n_volumes,
                                        int local_size, const void* field_params_f16, const void* shader_params_f16,
                                        const float* slot_pts, const float* slot_dt, const float* slot_t, const int* slot_anchors,
                                        const int* ray_counts, const float* rays_d, const float* bg, int n_rays, int slot_size,
                                        const int* total_all, int* ticket, float* colors, float* disparity, float* depth,
                                        int* kept_counts, float* weights_slots, const float* app_emb, void* stream) {
  return launch_render_fwd_fused<true, false>("f2b_render_fwd_fused_app", table_f16, prim_pool, bias_pool, n_volumes, local_size,
                                       field_params_f16, shader_params_f16, slot_pts, slot_dt, slot_t, slot_anchors, ray_counts,
                                       rays_d, bg, n_rays, slot_size, total_all, ticket, colors, disparity, depth, kept_counts,
                                       weights_slots, app_emb, CropBox{}, nullptr, stream);
}

extern "C" int f2b_render_fwd_fused_crop(const void* table_f16, const int* prim_pool, const float* bias_pool, int n_volumes,
                                         int local_size, const void* field_params_f16, const void* shader_params_f16,
                                         const float* slot_pts, const float* slot_dt, const float* slot_t, const int* slot_anchors,
                                         const int* ray_counts, const float* rays_d, const float* bg, int n_rays, int slot_size,
                                         const int* total_all, int* ticket, float* colors, float* disparity, float* depth,
                                         int* kept_counts, float* weights_slots, const float* app_emb, const float* rays_o,
                                         const float* box12, int invert, void* stream) {
  F2B_REQUIRE(box12, "f2b_render_fwd_fused_crop: null box");
  CropBox crop;
  for (int k = 0; k < 12; k++) crop.m[k] = box12[k];
  crop.invert = invert != 0;
  const auto launch = app_emb ? launch_render_fwd_fused<true, true> : launch_render_fwd_fused<false, true>;
  return launch("f2b_render_fwd_fused_crop", table_f16, prim_pool, bias_pool, n_volumes, local_size, field_params_f16,
                shader_params_f16, slot_pts, slot_dt, slot_t, slot_anchors, ray_counts, rays_d, bg, n_rays, slot_size, total_all, ticket,
                colors, disparity, depth, kept_counts, weights_slots, app_emb, crop, rays_o, stream);
}

extern "C" int f2b_crop_mask(const float* pts, int n, const float* box12, int invert, uint8_t* kept, void* stream) {
  if (n <= 0) return F2B_OK;
  F2B_REQUIRE(pts && box12 && kept, "f2b_crop_mask: null pointer");
  CropBox crop;
  for (int k = 0; k < 12; k++) crop.m[k] = box12[k];
  crop.invert = invert != 0;
  crop_mask_kernel<<<div_up(n, 256), 256, 0, as_stream(stream)>>>(pts, n, crop, kept);
  return check_launch("f2b_crop_mask");
}

extern "C" int f2b_gather_kept_weights(const float* weights_slots, const int* new_bounds, int n_rays, int slot_size, float* weights,
                                       void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(weights_slots && new_bounds && weights, "f2b_gather_kept_weights: null pointer");
  gather_kept_weights_kernel<<<div_up(int64_t(n_rays) * 32, 256), 256, 0, as_stream(stream)>>>(weights_slots, new_bounds, n_rays,
                                                                                                slot_size, weights);
  return check_launch("f2b_gather_kept_weights");
}
