// field.cu — Hash3DAnchored::AnchoredQuery as ONE kernel: 16-level hash encode fused in front of the
// wgmma field MLP (32 -> 64 -> 16).
//
// Replaces, per call, the reference's chain  (pts+1)/2 [ATen]  ->  Hash3DAnchoredForwardKernel x16 grid.y
// passes  ->  fp16->fp32 cast  ->  pad  ->  fp32->fp16 identity encoding  ->  kernel_mlp_fused  ->  slice +
// fp16->fp32 cast (src/Field/Hash3DAnchored.cpp:84-99, Hash3DAnchored.cu:160-197, TCNNWP.cpp:102-113).
// The 32 encoded halfs of a sample go from registers straight into the wgmma operand tile in shared
// memory (SWIZZLE_64B K-major row of thread i == sample i); they reach HBM only when the backward pass
// needs them (feat_save).  Modes:
//   logit_only  — the no-grad early-stop pass (Renderer.cpp:107-126) needs only channel 0: 4 B/sample out
//                 (+ optionally the encoded features, which the gradient pass re-uses for the surviving
//                 samples instead of gathering the table a second time);
//   full        — out [P,16] fp32 (fp16-rounded values, as TCNNWP::Query returns) + optional saves.
// Per sample the kernel moves 16 B in + 512 B of L2 gathers; the MLP rides along on the tensor pipe.
#include "common.cuh"
#include "hash.cuh"
#include "locate.cuh"
#include "tc.cuh"

namespace f2b {
using namespace tc;

constexpr int kFT = 128;
constexpr int kFieldDefaultMinB = 4;   // resident CTAs per SM the kernel is compiled for; see DESIGN.md

struct FieldSmem {
  static constexpr int A0 = 0;          // [128 x 32] f16 SW64   8 KB
  static constexpr int A1 = 8192;       // [128 x 64] f16 SW128 16 KB
  static constexpr int W0 = 24576;      // [64 x 32]  SW64       4 KB
  static constexpr int WO = 28672;      // [16 x 64]  SW128      2 KB
  static constexpr int SCALE = 30720;   // 16 level scales
  static constexpr int BYTES = 30720 + 64 + 1024;
};

// Where a tile's rows come from.  rows(tile, n_pts): the tile's output rows are its first rows(...) rows (0: skip the tile,
// CTA-uniform); point(p, ...): row p's warped point and volume, false when it has none (the row still takes part in the
// tile's MMAs with zero features and is written as `empty`).
struct SampleSource {      // the march's warped samples: a compact [P] layout, or the one-pass march's scratch slots
  const float* pts;
  const int* vol;
  int vol_stride;
  const int* slot_counts;  // slot layout: ray r owns slots [r*slot_size, r*slot_size + count[r]); NULL: compact
  int slot_size;
  static constexpr float empty = 0.f;   // unused: every output row has a point
  // slot_size is a multiple of the tile, so a tile lies inside one ray
  __device__ __forceinline__ int rows(int tile, int n_pts) const {
    const int t0 = tile * kFT;
    if (!slot_counts) return n_pts - t0;
    const int ray = t0 / slot_size;
    return min(n_pts, ray * slot_size + __ldg(slot_counts + ray)) - t0;
  }
  __device__ __forceinline__ bool point(int p, float& x, float& y, float& z, int& v) const {
    x = __ldg(pts + size_t(p) * 3); y = __ldg(pts + size_t(p) * 3 + 1); z = __ldg(pts + size_t(p) * 3 + 2);
    v = __ldg(vol + size_t(p) * vol_stride);
    return true;
  }
};

// World points located in the octree and warped (locate.cuh) in front of the encode: an array of points, or (GRID) the
// lattice origin + voxel * (x, y, z0 + z) of an nx x ny x nz slab, generated here (row p = x + nx * (y + ny * z)).
template <bool GRID>
struct LocateSource {
  const TreeNode* nodes;
  const TransInfo* trans;
  const float* pts;        // !GRID: [n,3] world points
  float ox, oy, oz, vx, vy, vz;
  int nx, ny, z0;
  float empty;
  __device__ __forceinline__ int rows(int tile, int n_pts) const { return n_pts - tile * kFT; }
  __device__ __forceinline__ bool point(int p, float& x, float& y, float& z, int& v) const {
    float wx, wy, wz;
    if (GRID) {
      const int ix = p % nx, iy = (p / nx) % ny, iz = z0 + p / (nx * ny);
      wx = fadd(ox, fmul(vx, float(ix))); wy = fadd(oy, fmul(vy, float(iy))); wz = fadd(oz, fmul(vz, float(iz)));
    } else {
      wx = __ldg(pts + size_t(p) * 3); wy = __ldg(pts + size_t(p) * 3 + 1); wz = __ldg(pts + size_t(p) * 3 + 2);
    }
    int ti = -1;
    if (locate_leaf(nodes, wx, wy, wz, ti) < 0) return false;
    float w[3];
    warp_point(trans + ti, wx, wy, wz, w);
    x = w[0]; y = w[1]; z = w[2]; v = ti;
    return true;
  }
};

template <bool LOGIT_ONLY, int MINB, class Src>
__global__ void __launch_bounds__(kFT, MINB)
field_fwd_kernel(const __half* __restrict__ table, const int* __restrict__ prim_pool,
                 const float* __restrict__ bias_pool, int n_volumes, int local_size,
                 const __half* __restrict__ params, const Src src, int n_pts,
                 float* __restrict__ out, __half* __restrict__ feat_save, __half* __restrict__ hidden_save) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* s_scale = reinterpret_cast<float*>(sm + FieldSmem::SCALE);
  float* s_rows = reinterpret_cast<float*>(sm + FieldSmem::A1);     // output rows [128][20] fp32 (A1 is dead by then)
  const int tid = threadIdx.x;

  for (int i = tid; i < 64 * 4; i += kFT) {                       // W0 [64 x 32] -> SW64
    const int r = i >> 2, c = i & 3;
    *reinterpret_cast<uint4*>(sm + FieldSmem::W0 + sw64_off(r, c)) = *reinterpret_cast<const uint4*>(params + r * 32 + c * 8);
  }
  for (int i = tid; i < 16 * 8; i += kFT) {                       // Wout [16 x 64] -> SW128
    const int r = i >> 3, c = i & 7;
    *reinterpret_cast<uint4*>(sm + FieldSmem::WO + sw128_off(r, c)) = *reinterpret_cast<const uint4*>(params + 64 * 32 + r * 64 + c * 8);
  }
  if (tid < F2B_N_LEVELS) s_scale[tid] = level_scale(tid);        // run-time MUFU.EX2, like the reference
  __syncthreads();
  const uint32_t a0 = smem_u32(sm + FieldSmem::A0), a1 = smem_u32(sm + FieldSmem::A1);
  const uint32_t w0 = smem_u32(sm + FieldSmem::W0), wo = smem_u32(sm + FieldSmem::WO);
  Acc<64> acc;
  Acc<16> acc_out;

  const int n_tiles = (n_pts + kFT - 1) / kFT;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int rows = src.rows(tile, n_pts);
    if (rows <= 0) continue;                                        // CTA-uniform
    const int p = tile * kFT + tid;
    const bool valid = tid < rows;
    // ---- encode my sample: 16 levels x 8 corner gathers -> 32 halfs in registers ------------------
    uint32_t enc[16];
    float x, y, z;
    int v;
    const bool hit = valid && src.point(p, x, y, z, v);
    if (hit) {
      encode_point(table, prim_pool, bias_pool, n_volumes, local_size, s_scale, x, y, z, v, enc);
    } else {
#pragma unroll
      for (int l = 0; l < 16; l++) enc[l] = 0u;
    }
#pragma unroll
    for (int c = 0; c < 4; c++)
      *reinterpret_cast<uint4*>(sm + FieldSmem::A0 + sw64_off(tid, c)) = make_uint4(enc[4 * c], enc[4 * c + 1], enc[4 * c + 2], enc[4 * c + 3]);
    fence_async_smem();
    __syncthreads();                                              // (also: the previous tile's output rows have been read)
    // ---- layer 0 on the tensor pipe -------------------------------------------------------------------
    wg_fence();
    mma_m128<64, 0, 2>(acc, a0, 64, w0, 64, false);
    wg_commit();
    if (feat_save) {                                              // whole-line copy-out of the tile while the MMA reads it
      const int rows = min(kFT, n_pts - tile * kFT);
      uint4* dst = reinterpret_cast<uint4*>(feat_save + size_t(tile) * kFT * 32);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int c = tid + kFT * j, r = c >> 2;
        if (r < rows) dst[c] = *reinterpret_cast<const uint4*>(sm + FieldSmem::A0 + sw64_off(r, c & 3));
      }
    }
    wg_wait();
    acc_relu_to_tile(acc, sm + FieldSmem::A1, tid);
    fence_async_smem();
    __syncthreads();
    // ---- output layer -------------------------------------------------------------------------------
    wg_fence();
    mma_m128<16, 0, 4>(acc_out, a1, 128, wo, 128, false);
    wg_commit();
    if (!LOGIT_ONLY && hidden_save) {
      const int rows = min(kFT, n_pts - tile * kFT);
      uint4* dst = reinterpret_cast<uint4*>(hidden_save + size_t(tile) * kFT * 64);
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int c = tid + kFT * j, r = c >> 3;
        if (r < rows) dst[c] = *reinterpret_cast<const uint4*>(sm + FieldSmem::A1 + sw128_off(r, c & 7));
      }
    }
    wg_wait();
    __syncthreads();                                              // every warp is done with A1 (operand / copy-out)
    acc_to_rows(acc_out, s_rows, kRowLd16, tid);
    __syncthreads();
    {
      uint32_t r[16];
      row_ld16(s_rows, kRowLd16, tid, r);
      if (valid) {
        if (LOGIT_ONLY) {
          out[p] = hit ? __half2float(__float2half_rn(__uint_as_float(r[0]))) : src.empty;
        } else {
          float4* dst = reinterpret_cast<float4*>(out + size_t(p) * 16);
#pragma unroll
          for (int q = 0; q < 4; q++)
            dst[q] = make_float4(__half2float(__float2half_rn(__uint_as_float(r[4 * q]))), __half2float(__float2half_rn(__uint_as_float(r[4 * q + 1]))),
                                 __half2float(__float2half_rn(__uint_as_float(r[4 * q + 2]))), __half2float(__float2half_rn(__uint_as_float(r[4 * q + 3]))));
        }
      }
    }
  }
}

}  // namespace f2b

using namespace f2b;

static int field_fwd_launch(const void* table_f16, const int* prim_pool, const float* bias_pool, int n_volumes,
                            int local_size, const void* mlp_params_f16, const float* pts, const int* vol,
                            int vol_stride, int n_pts, const int* slot_counts, int slot_size, int logit_only,
                            float* out_f32, void* feat_save_f16, void* hidden_save_f16, void* stream);

extern "C" int f2b_field_fwd(const void* table_f16, const int* prim_pool, const float* bias_pool, int n_volumes,
                             int local_size, const void* mlp_params_f16, const float* pts, const int* vol,
                             int vol_stride, int n_pts, int logit_only, float* out_f32, void* feat_save_f16,
                             void* hidden_save_f16, void* stream) {
  return field_fwd_launch(table_f16, prim_pool, bias_pool, n_volumes, local_size, mlp_params_f16, pts, vol, vol_stride,
                          n_pts, nullptr, 0, logit_only, out_f32, feat_save_f16, hidden_save_f16, stream);
}

extern "C" int f2b_field_fwd_slots(const void* table_f16, const int* prim_pool, const float* bias_pool, int n_volumes,
                                   int local_size, const void* mlp_params_f16, const float* slot_pts, const int* slot_vol,
                                   int vol_stride, const int* ray_counts, int n_rays, int slot_size, int logit_only,
                                   float* out_f32, void* feat_save_f16, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(ray_counts && slot_size > 0 && (slot_size % kFT) == 0, "f2b_field_fwd_slots: slot_size must be a positive multiple of 128");
  F2B_REQUIRE(int64_t(n_rays) * slot_size < (int64_t(1) << 31), "f2b_field_fwd_slots: n_rays * slot_size overflows int32");
  return field_fwd_launch(table_f16, prim_pool, bias_pool, n_volumes, local_size, mlp_params_f16, slot_pts, slot_vol,
                          vol_stride, n_rays * slot_size, ray_counts, slot_size, logit_only, out_f32, feat_save_f16, nullptr,
                          stream);
}

template <bool LO, class Src>
static void field_launch(const void* table_f16, const int* prim_pool, const float* bias_pool, int n_volumes, int local_size,
                         const void* mlp_params_f16, const Src& src, int n_pts, float* out_f32, void* feat_save_f16,
                         void* hidden_save_f16, void* stream) {
  constexpr int MB = kFieldDefaultMinB;
  int sms = 132;
  f2b_device_info(&sms, nullptr);
  const int n_tiles = div_up(n_pts, kFT);
  const int grid = n_tiles < sms * MB ? n_tiles : sms * MB;
  cudaFuncSetAttribute(field_fwd_kernel<LO, MB, Src>, cudaFuncAttributeMaxDynamicSharedMemorySize, FieldSmem::BYTES);
  field_fwd_kernel<LO, MB, Src><<<grid, kFT, FieldSmem::BYTES, as_stream(stream)>>>(
      (const __half*)table_f16, prim_pool, bias_pool, n_volumes, local_size, (const __half*)mlp_params_f16, src, n_pts, out_f32,
      (__half*)feat_save_f16, LO ? nullptr : (__half*)hidden_save_f16);
}

static int field_fwd_launch(const void* table_f16, const int* prim_pool, const float* bias_pool, int n_volumes,
                            int local_size, const void* mlp_params_f16, const float* pts, const int* vol,
                            int vol_stride, int n_pts, const int* slot_counts, int slot_size, int logit_only,
                            float* out_f32, void* feat_save_f16, void* hidden_save_f16, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(table_f16 && prim_pool && bias_pool && mlp_params_f16 && pts && vol && out_f32, "f2b_field_fwd: null pointer");
  F2B_REQUIRE(n_volumes > 0 && local_size > 0 && (local_size % 2) == 0, "f2b_field_fwd: bad n_volumes/local_size");
  const SampleSource src{pts, vol, vol_stride, slot_counts, slot_size};
  if (logit_only)
    field_launch<true>(table_f16, prim_pool, bias_pool, n_volumes, local_size, mlp_params_f16, src, n_pts, out_f32, feat_save_f16,
                       hidden_save_f16, stream);
  else
    field_launch<false>(table_f16, prim_pool, bias_pool, n_volumes, local_size, mlp_params_f16, src, n_pts, out_f32, feat_save_f16,
                        hidden_save_f16, stream);
  return check_launch("f2b_field_fwd");
}

// ---- point query (DESIGN §3i): the same kernel behind f2b_locate_points' walk and warp ------------------------------------
template <bool GRID>
static int query_logit_launch(const char* what, const void* tree_nodes, int n_nodes, const void* trans, const void* table_f16,
                              const int* prim_pool, const float* bias_pool, int n_volumes, int local_size,
                              const void* mlp_params_f16, const LocateSource<GRID>& src, int n, float* logit, void* stream) {
  if (n <= 0) return F2B_OK;
  F2B_REQUIRE(tree_nodes && n_nodes > 0 && trans && table_f16 && prim_pool && bias_pool && mlp_params_f16 && logit, "%s: null pointer",
              what);
  F2B_REQUIRE(n_volumes > 0 && local_size > 0 && (local_size % 2) == 0, "%s: bad n_volumes/local_size", what);
  field_launch<true>(table_f16, prim_pool, bias_pool, n_volumes, local_size, mlp_params_f16, src, n, logit, nullptr, nullptr, stream);
  return check_launch(what);
}

extern "C" int f2b_query_logit_points(const void* tree_nodes, int n_nodes, const void* trans, const void* table_f16,
                                      const int* prim_pool, const float* bias_pool, int n_volumes, int local_size,
                                      const void* mlp_params_f16, const float* pts, int n_pts, float empty_logit, float* logit,
                                      void* stream) {
  F2B_REQUIRE(pts || n_pts <= 0, "f2b_query_logit_points: null pointer");
  LocateSource<false> src{(const TreeNode*)tree_nodes, (const TransInfo*)trans, pts, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0, 0, 0, empty_logit};
  return query_logit_launch("f2b_query_logit_points", tree_nodes, n_nodes, trans, table_f16, prim_pool, bias_pool, n_volumes,
                            local_size, mlp_params_f16, src, n_pts, logit, stream);
}

extern "C" int f2b_query_logit_grid(const void* tree_nodes, int n_nodes, const void* trans, const void* table_f16,
                                    const int* prim_pool, const float* bias_pool, int n_volumes, int local_size,
                                    const void* mlp_params_f16, const float* origin3, const float* voxel3, int nx, int ny, int z0,
                                    int nz, float empty_logit, float* logit, void* stream) {
  F2B_REQUIRE(origin3 && voxel3 && nx >= 0 && ny >= 0 && nz >= 0 && z0 >= 0, "f2b_query_logit_grid: bad lattice");
  F2B_REQUIRE(int64_t(nx) * ny * nz < (int64_t(1) << 31), "f2b_query_logit_grid: slab of 2^31 points or more");
  LocateSource<true> src{(const TreeNode*)tree_nodes, (const TransInfo*)trans, nullptr, origin3[0], origin3[1], origin3[2],
                         voxel3[0], voxel3[1], voxel3[2], nx, ny, z0, empty_logit};
  return query_logit_launch("f2b_query_logit_grid", tree_nodes, n_nodes, trans, table_f16, prim_pool, bias_pool, n_volumes,
                            local_size, mlp_params_f16, src, nx * ny * nz, logit, stream);
}
