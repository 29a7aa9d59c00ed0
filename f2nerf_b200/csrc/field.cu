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
#include "shader.cuh"
#include "tc.cuh"

namespace f2b {
using namespace tc;

constexpr int kFT = 128;
constexpr int kFieldDefaultMinB = 4;   // resident CTAs per SM the kernel is compiled for; see DESIGN.md

// Shared memory of the field MLP's 128-row tile, the common prefix of the field kernels' layouts
struct FieldTileSmem {
  static constexpr int A0 = 0;          // [128 x 32] f16 SW64   8 KB  the encoded features
  static constexpr int A1 = 8192;       // [128 x 64] f16 SW128 16 KB  H (the gradient kernels: then dH in place)
  static constexpr int W0 = 24576;      // [64 x 32]  SW64       4 KB
  static constexpr int WO = 28672;      // [16 x 64]  SW128      2 KB
  static constexpr int END = 30720;
};
struct FieldSmem : FieldTileSmem {
  static constexpr int SCALE = END;     // 16 level scales
  static constexpr int BYTES = SCALE + 64 + 1024;
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
  __device__ __forceinline__ int rows(int tile, int n_pts) const {
    return slot_counts ? slot_rows(tile, n_pts, slot_counts, slot_size) : n_pts - tile * kFT;
  }
  // slot layout: slot_size is a multiple of the tile, so a tile lies inside one ray
  static __device__ __forceinline__ int slot_rows(int tile, int n_pts, const int* counts, int slot_size) {
    const int t0 = tile * kFT;
    const int ray = t0 / slot_size;
    return min(n_pts, ray * slot_size + __ldg(counts + ray)) - t0;
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
  // the world point of row p (the gradient kernel's Jacobian; !GRID only)
  __device__ __forceinline__ void world(int p, float& X, float& Y, float& Z) const {
    X = __ldg(pts + size_t(p) * 3); Y = __ldg(pts + size_t(p) * 3 + 1); Z = __ldg(pts + size_t(p) * 3 + 2);
  }
};

// The kept samples of a VALIDATE render in the march's slot layout (DESIGN §3j): ray r's rows are [r*slot_size, r*slot_size +
// kept[r]); the warped point and volume are the march's s_pts / s_anchors, the world point fma(t, d, o) as the march formed it.
struct KeptSlotSource {
  const float* s_pts;
  const float* s_t;
  const int* s_anchors;    // [.,2] (trans_idx, node)
  const int* kept;
  const float* rays_o;
  const float* rays_d;
  int slot_size;
  static constexpr float empty = 0.f;   // unused: every output row has a point
  __device__ __forceinline__ int rows(int tile, int n_pts) const { return SampleSource::slot_rows(tile, n_pts, kept, slot_size); }
  __device__ __forceinline__ bool point(int p, float& x, float& y, float& z, int& v) const {
    x = __ldg(s_pts + size_t(p) * 3); y = __ldg(s_pts + size_t(p) * 3 + 1); z = __ldg(s_pts + size_t(p) * 3 + 2);
    v = __ldg(s_anchors + size_t(p) * 2);
    return true;
  }
  __device__ __forceinline__ void world(int p, float& X, float& Y, float& Z) const {
    const int ray = p / slot_size;
    const float t = __ldg(s_t + p);
    X = ffma(t, __ldg(rays_d + ray * 3), __ldg(rays_o + ray * 3));
    Y = ffma(t, __ldg(rays_d + ray * 3 + 1), __ldg(rays_o + ray * 3 + 1));
    Z = ffma(t, __ldg(rays_d + ray * 3 + 2), __ldg(rays_o + ray * 3 + 2));
  }
};

// ---- steps of the field MLP on a 128-row tile, shared by the field kernels ------------------------------------------------------
// W0 / Wout into the tile's weight slots, Wout row 0 also to wo0 (may be NULL; fp16 [64]), and the 16 level scales into s_scale
// (run-time MUFU.EX2, like the reference).  The weights are staged by shifts and masks rather than by tc::stage_weights, whose
// signed division compiles to different code in these kernels.
__device__ __forceinline__ void stage_field(const __half* __restrict__ params, unsigned char* sm, float* s_scale, unsigned char* wo0,
                                            int t) {
  for (int i = t; i < 64 * 4; i += kFT) {                         // W0 [64 x 32] -> SW64
    const int r = i >> 2, c = i & 3;
    *reinterpret_cast<uint4*>(sm + FieldTileSmem::W0 + sw64_off(r, c)) = *reinterpret_cast<const uint4*>(params + r * 32 + c * 8);
  }
  for (int i = t; i < 16 * 8; i += kFT) {                         // Wout [16 x 64] -> SW128
    const int r = i >> 3, c = i & 7;
    *reinterpret_cast<uint4*>(sm + FieldTileSmem::WO + sw128_off(r, c)) =
        *reinterpret_cast<const uint4*>(params + 64 * 32 + r * 64 + c * 8);
  }
  if (wo0 && t < 8) reinterpret_cast<uint4*>(wo0)[t] = reinterpret_cast<const uint4*>(params + 64 * 32)[t];
  if (t < F2B_N_LEVELS) s_scale[t] = level_scale(t);
}

// layer 0: H = relu(A0 . W0^T) -> fp16 into A1.  `during()` runs while the MMA is in flight.
template <class During>
__device__ __forceinline__ void field_layer0(Acc<64>& acc, uint32_t a0, uint32_t w0, unsigned char* a1_tile, int t, During&& during) {
  wg_fence();
  mma_m128<64, 0, 2>(acc, a0, 64, w0, 64, false);
  wg_commit();
  during();
  wg_wait();
  acc_relu_to_tile(acc, a1_tile, t);
}

// output layer: acc_out = A1 . Wout^T.  `during()` runs while the MMA is in flight.
template <class During>
__device__ __forceinline__ void field_out_layer(Acc<16>& acc_out, uint32_t a1, uint32_t wo, During&& during) {
  wg_fence();
  mma_m128<16, 0, 4>(acc_out, a1, 128, wo, 128, false);
  wg_commit();
  during();
  wg_wait();
}

template <bool LOGIT_ONLY, int MINB, class Src>
__global__ void __launch_bounds__(kFT, MINB)
field_fwd_kernel(const __half* __restrict__ table, const int* __restrict__ prim_pool,
                 const float* __restrict__ bias_pool, int n_volumes, int local_size,
                 const __half* __restrict__ params, const Src src, int n_pts,
                 float* __restrict__ out, __half* __restrict__ feat_save, __half* __restrict__ hidden_save) {
  unsigned char* sm = smem_base();
  float* s_scale = reinterpret_cast<float*>(sm + FieldSmem::SCALE);
  float* s_rows = reinterpret_cast<float*>(sm + FieldSmem::A1);     // output rows [128][20] fp32 (A1 is dead by then)
  const int tid = threadIdx.x;

  stage_field(params, sm, s_scale, nullptr, tid);
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
    field_layer0(acc, a0, w0, sm + FieldSmem::A1, tid, [&] {
      if (feat_save) {                                            // whole-line copy-out of the tile while the MMA reads it
        const int rows = min(kFT, n_pts - tile * kFT);
        uint4* dst = reinterpret_cast<uint4*>(feat_save + size_t(tile) * kFT * 32);
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const int c = tid + kFT * j, r = c >> 2;
          if (r < rows) dst[c] = *reinterpret_cast<const uint4*>(sm + FieldSmem::A0 + sw64_off(r, c & 3));
        }
      }
    });
    fence_async_smem();
    __syncthreads();
    // ---- output layer -------------------------------------------------------------------------------
    field_out_layer(acc_out, a1, wo, [&] {
      if (!LOGIT_ONLY && hidden_save) {
        const int rows = min(kFT, n_pts - tile * kFT);
        uint4* dst = reinterpret_cast<uint4*>(hidden_save + size_t(tile) * kFT * 64);
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const int c = tid + kFT * j, r = c >> 3;
          if (r < rows) dst[c] = *reinterpret_cast<const uint4*>(sm + FieldSmem::A1 + sw128_off(r, c & 7));
        }
      }
    });
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

// ---- density gradient (DESIGN §3j) -------------------------------------------------------------------------------------------
// g = J^T . sum_l 0.5 scale_l . sum_c (dfeat_l . f_c) dw_c/dp, dfeat = W0^T (Wout[0,:] * [H > 0]) per 128-row tile: the field
// kernel's forward (same operand tiles, so the logit keeps its bits), dH over the fp16 hidden tile in place, dfeat = dH . W0 on
// the tensor pipe (W0 as the MN-major operand, as mlp_tc_bwd.cu), rounded to fp16 as the training backward rounds it, then per
// thread the 16 level gradients and the leaf's Jacobian.  Points: logit and g per row.  Kept slots: sum_i w_i n_i over the tile's
// rows, serial in row order, one partial per tile (normals_finish_kernel sums a ray's partials in tile order).
struct GradSmem : FieldTileSmem {
  static constexpr int ROWS = 0;        // [128][kGradLd] fp32 dfeat rows (over A0 / A1, both dead by then)
  static constexpr int SCALE = END;     // 16 level scales
  static constexpr int LOGIT = 30784;   // [128] fp32 output channel 0
  static constexpr int WO0 = 31296;     // [64] f16 Wout row 0
  static constexpr int ADD = 31424;     // [3][128] fp32 w_i n_i (slot source)
  static constexpr int BYTES = ADD + 1536 + 1024;
};
constexpr int kGradLd = 36;             // fp32 row pitch: conflict-free float4 row reads

// sum_l 0.5 scale_l . grad_level(dfeat_l): the gradient with respect to the warped point (x, y, z) of volume v, given the row's 16
// level pairs of dL/dfeat (fp32 values of the fp16 rows)
__device__ __forceinline__ void warped_grad(const __half* __restrict__ table, const int* __restrict__ prim_pool,
                                            const float* __restrict__ bias_pool, int n_volumes, int local_size, const float* s_scale,
                                            float x, float y, float z, int v, const float* row, float gw[3]) {
  const float x0 = fmul(fadd(x, 1.f), .5f), x1 = fmul(fadd(y, 1.f), .5f), x2 = fmul(fadd(z, 1.f), .5f);
  gw[0] = gw[1] = gw[2] = 0.f;
#pragma unroll 1
  for (int l = 0; l < F2B_N_LEVELS; l++) {
    const int tv = l * n_volumes + v;
    const float* bias = bias_pool + tv * 3;
    const float scale = s_scale[l];
    Corner8 c;
    corners(x0, x1, x2, scale, prim_pool + tv * 3, bias, (unsigned)local_size, c);
    const float px = ffma(x0, scale, __ldg(bias)), py = ffma(x1, scale, __ldg(bias + 1)), pz = ffma(x2, scale, __ldg(bias + 2));
    const float2 d = *reinterpret_cast<const float2*>(row + 2 * l);
    float gl[3];
    grad_level(table, l, local_size, c, fsub(px, floorf(px)), fsub(py, floorf(py)), fsub(pz, floorf(pz)), d.x, d.y, gl);
    const float dpdw = fmul(.5f, scale);                          // p = ((w + 1) / 2) * scale + bias
#pragma unroll
    for (int k = 0; k < 3; k++) gw[k] = ffma(dpdw, gl[k], gw[k]);
  }
}

template <bool SLOTS, class Src>
__global__ void __launch_bounds__(kFT, kFieldDefaultMinB)
field_grad_kernel(const __half* __restrict__ table, const int* __restrict__ prim_pool, const float* __restrict__ bias_pool,
                  int n_volumes, int local_size, const __half* __restrict__ params, const TransInfo* __restrict__ trans, const Src src,
                  int n_pts, float empty, float* __restrict__ logit_out, float* __restrict__ grad_out, const float* __restrict__ w_slots,
                  float* __restrict__ tile_partials) {
  using S = GradSmem;
  unsigned char* sm = smem_base();
  float* s_scale = reinterpret_cast<float*>(sm + S::SCALE);
  float* s_logit = reinterpret_cast<float*>(sm + S::LOGIT);
  const __half* s_wo0 = reinterpret_cast<const __half*>(sm + S::WO0);
  float* s_rows = reinterpret_cast<float*>(sm + S::ROWS);
  float* s_add = reinterpret_cast<float*>(sm + S::ADD);
  const int tid = threadIdx.x;

  stage_field(params, sm, s_scale, sm + S::WO0, tid);
  __syncthreads();
  const uint32_t a0 = smem_u32(sm + S::A0), a1 = smem_u32(sm + S::A1);
  const uint32_t w0 = smem_u32(sm + S::W0), wo = smem_u32(sm + S::WO);

  const int n_tiles = (n_pts + kFT - 1) / kFT;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int rows = src.rows(tile, n_pts);
    if (rows <= 0) continue;                                        // CTA-uniform
    const int p = tile * kFT + tid;
    const bool valid = tid < rows;
    float x = 0.f, y = 0.f, z = 0.f;
    int v = 0;
    const bool hit = valid && src.point(p, x, y, z, v);
    {
      uint32_t enc[16];
      if (hit) {
        encode_point(table, prim_pool, bias_pool, n_volumes, local_size, s_scale, x, y, z, v, enc);
      } else {
#pragma unroll
        for (int l = 0; l < 16; l++) enc[l] = 0u;
      }
#pragma unroll
      for (int c = 0; c < 4; c++)
        *reinterpret_cast<uint4*>(sm + S::A0 + sw64_off(tid, c)) = make_uint4(enc[4 * c], enc[4 * c + 1], enc[4 * c + 2], enc[4 * c + 3]);
    }
    fence_async_smem();
    __syncthreads();
    // ---- forward: layer 0, output layer (field_fwd_kernel's MMAs) ---------------------------------------------------------
    {
      Acc<64> acc;
      field_layer0(acc, a0, w0, sm + S::A1, tid, [] {});
    }
    fence_async_smem();
    __syncthreads();
    {
      Acc<16> acc_out;
      field_out_layer(acc_out, a1, wo, [] {});
      if ((tid & 3) == 0) {                                         // column 0 of the accumulator: elements 0 and 2 of each half
#pragma unroll
        for (int h = 0; h < 2; h++) { s_logit[acc_row(tid, h, 0)] = acc_out.d[h][0]; s_logit[acc_row(tid, h, 2)] = acc_out.d[h][2]; }
      }
    }
    __syncthreads();                                                // every warp is done with A1 as an operand
    // ---- dH = Wout[0,:] * [H > 0] over my row of the fp16 hidden tile (dL/dout = e_0: exact in fp16) ------------------------
#pragma unroll
    for (int c = 0; c < 8; c++) {
      uint4* q = reinterpret_cast<uint4*>(sm + S::A1 + sw128_off(tid, c));
      uint4 hv = *q;
      uint32_t* hw = reinterpret_cast<uint32_t*>(&hv);
      const uint32_t* ww = reinterpret_cast<const uint32_t*>(s_wo0 + 8 * c);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const __half2 h2 = *reinterpret_cast<const __half2*>(&hw[j]);
        const uint32_t wj = ww[j];
        const uint32_t lo = __low2float(h2) > 0.f ? (wj & 0xFFFFu) : 0u, hi = __high2float(h2) > 0.f ? (wj & 0xFFFF0000u) : 0u;
        hw[j] = lo | hi;
      }
      *q = hv;
    }
    fence_async_smem();
    __syncthreads();
    // ---- dfeat = dH . W0 -> fp16 -> fp32 rows ----------------------------------------------------------------------------------
    {
      Acc<32> acc_in;
      wg_fence();
      mma_m128<32, 1, 4>(acc_in, a1, 128, w0, 64, false);
      wg_commit();
      wg_wait();
      __syncthreads();                                              // every warp's MMA is done reading A1 (the rows overwrite it)
#pragma unroll
      for (int h = 0; h < 2; h++)
#pragma unroll
        for (int i = 0; i < 16; i += 2) {
          const float2 d = __half22float2(__floats2half2_rn(acc_in.d[h][i], acc_in.d[h][i + 1]));
          *reinterpret_cast<float2*>(s_rows + acc_row(tid, h, i) * kGradLd + acc_col(tid, i)) = d;
        }
    }
    __syncthreads();
    // ---- my row: 16 level gradients, then J^T ----------------------------------------------------------------------------------
    float g[3] = {0.f, 0.f, 0.f};
    if (hit) {
      float gw[3];
      warped_grad(table, prim_pool, bias_pool, n_volumes, local_size, s_scale, x, y, z, v, s_rows + tid * kGradLd, gw);
      float X, Y, Z, J[3][3];
      src.world(p, X, Y, Z);
      warp_jacobian(trans + v, X, Y, Z, J);
#pragma unroll
      for (int k = 0; k < 3; k++) g[k] = ffma(J[0][k], gw[0], ffma(J[1][k], gw[1], fmul(J[2][k], gw[2])));
    }
    if (!SLOTS) {
      if (valid) {
        logit_out[p] = hit ? __half2float(__float2half_rn(s_logit[tid])) : empty;
        grad_out[size_t(p) * 3] = g[0]; grad_out[size_t(p) * 3 + 1] = g[1]; grad_out[size_t(p) * 3 + 2] = g[2];
      }
      __syncthreads();                                              // the rows have been read before the next tile's A0 stores
    } else {
      float wn[3] = {0.f, 0.f, 0.f};
      if (valid) {                                                  // n = -g / |g| (0 where g = 0), weighted by the render's w_i
        const float len = fsqrt(fadd(fadd(fmul(g[0], g[0]), fmul(g[1], g[1])), fmul(g[2], g[2])));
        const float w = __ldg(w_slots + p);
        if (len > 0.f) {
#pragma unroll
          for (int k = 0; k < 3; k++) wn[k] = fmul(w, fdiv(-g[k], len));
        }
      }
#pragma unroll
      for (int k = 0; k < 3; k++) s_add[k * kFT + tid] = wn[k];
      __syncthreads();
      if (tid < 3) {                                                // serial, row order; rows past the kept prefix add +0
        const float* mine = s_add + tid * kFT;
        float a = 0.f;
#pragma unroll 16
        for (int j = 0; j < kFT; j++) a = fadd(a, mine[j]);
        tile_partials[size_t(tile) * 3 + tid] = a;
      }
      __syncthreads();
    }
  }
}

// A ray's unit normal from its tile partials: N = the partials of its first ceil(kept / 128) tiles summed in tile order, N / |N|
// (0 where N = 0 or nothing was kept).
__global__ void __launch_bounds__(128)
normals_finish_kernel(const float* __restrict__ tile_partials, const int* __restrict__ kept, int n_rays, int slot_size,
                      float* __restrict__ normals) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  const int tiles = slot_size / kFT, nt = (kept[r] + kFT - 1) / kFT;
  const float* src = tile_partials + size_t(r) * tiles * 3;
  float N[3] = {0.f, 0.f, 0.f};
  for (int k = 0; k < nt; k++)
#pragma unroll
    for (int c = 0; c < 3; c++) N[c] = fadd(N[c], src[3 * k + c]);
  const float len = fsqrt(fadd(fadd(fmul(N[0], N[0]), fmul(N[1], N[1])), fmul(N[2], N[2])));
#pragma unroll
  for (int c = 0; c < 3; c++) normals[size_t(r) * 3 + c] = len > 0.f ? fdiv(N[c], len) : 0.f;
}


// ---- gradient of the rendered colour with respect to the rays (DESIGN §3k) -----------------------------------------------------
// Per 128-row tile of a VALIDATE batch's compacted survivors: the field-MLP backward of f2b_mlp_bwd2 (hidden0 == NULL,
// n_hidden_matmuls 0) on the row's fp16 dL/dout — the same MMAs on the same operand tiles, so dfeat has its bits — then per thread
// grad_w = sum_l 0.5 scale_l grad_level(dfeat_l), dL/dx = J^T grad_w at the world point fma(t, d, o) the march formed, and the SH4
// term dL/ddir = sum_k dL/dmlp_in[16 + k] dsh4_k/ddir.  Each row leaves (dL/dx, t dL/dx + dL/ddir) in row_work; ray_grad_finish_kernel
// sums a ray's rows serially in row order.  t, dt, the kept set and the leaf are data, not differentiated.
struct RayGradSmem : FieldTileSmem {
  static constexpr int ROWS = 0;        // [128][kGradLd] fp32 dfeat rows (over A0 / A1, both dead by then)
  static constexpr int DO = END;        // [128 x 16] f16 SW32   4 KB  dL/dout rows
  static constexpr int SCALE = DO + 4096;   // 16 level scales
  static constexpr int BYTES = SCALE + 64 + 1024;
};

// the ray whose rows [bounds[r,0], bounds[r,1]) hold row p: the last ray starting at or before p (rays without rows start where the
// next non-empty one does, so they are never last)
__device__ __forceinline__ int ray_of_row(const int* __restrict__ bounds, int n_rays, int p) {
  int lo = 0, hi = n_rays - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(bounds + 2 * mid) <= p) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

constexpr int kRayGradMinB = 3;          // 4 CTAs per SM would cap the kernel at 128 registers and spill

__global__ void __launch_bounds__(kFT, kRayGradMinB)
ray_grad_kernel(const __half* __restrict__ table, const int* __restrict__ prim_pool, const float* __restrict__ bias_pool, int n_volumes,
                int local_size, const __half* __restrict__ params, const TransInfo* __restrict__ trans, const __half* __restrict__ feat,
                const __half* __restrict__ d_out, const __half* __restrict__ d_in, const float* __restrict__ pts,
                const float* __restrict__ t, const float* __restrict__ dirs, const int* __restrict__ anchors,
                const float* __restrict__ rays_o, const int* __restrict__ bounds, int n_rays, int n_pts, float inv_field_scale,
                float inv_shader_scale, float* __restrict__ row_work, float* __restrict__ d_pts, float* __restrict__ d_dirs,
                __half* __restrict__ dfeat16) {
  using S = RayGradSmem;
  unsigned char* sm = smem_base();
  float* s_scale = reinterpret_cast<float*>(sm + S::SCALE);
  float* s_rows = reinterpret_cast<float*>(sm + S::ROWS);
  const int tid = threadIdx.x;

  stage_field(params, sm, s_scale, nullptr, tid);
  __syncthreads();
  const uint32_t a0 = smem_u32(sm + S::A0), a1 = smem_u32(sm + S::A1), s_do = smem_u32(sm + S::DO);
  const uint32_t w0 = smem_u32(sm + S::W0), wo = smem_u32(sm + S::WO);

  const int n_tiles = (n_pts + kFT - 1) / kFT;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int p = tile * kFT + tid;
    const bool valid = p < n_pts;
    {                                                               // my operand rows; rows past n_pts are zero, as f2b_mlp_bwd2 fills them
      const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
      const uint4* xs = reinterpret_cast<const uint4*>(feat + size_t(p) * 32);
      const uint4* ds = reinterpret_cast<const uint4*>(d_out + size_t(p) * 16);
#pragma unroll
      for (int c = 0; c < 4; c++) *reinterpret_cast<uint4*>(sm + S::A0 + sw64_off(tid, c)) = valid ? __ldg(xs + c) : z4;
#pragma unroll
      for (int c = 0; c < 2; c++) *reinterpret_cast<uint4*>(sm + S::DO + sw32_off(tid, c)) = valid ? __ldg(ds + c) : z4;
    }
    fence_async_smem();
    __syncthreads();
    // ---- F0: H = relu(X . W0^T) ---------------------------------------------------------------------------------------------
    {
      Acc<64> acc;
      field_layer0(acc, a0, w0, sm + S::A1, tid, [] {});
      fence_async_smem();
      __syncthreads();
      // ---- A: dH = dOut . Wout, masked by the fp16 hidden tile, over it in place ----------------------------------------------
      wg_fence();
      mma_m128<64, 1, 1>(acc, s_do, 32, wo, 128, false);
      wg_commit();
      wg_wait();
      __syncthreads();                                              // every warp is done with H as an operand
      relu_bwd_epilogue(acc, sm + S::A1, sm + S::A1, tid);
    }
    fence_async_smem();
    __syncthreads();
    // ---- C: dfeat = dH . W0 -> fp16 (as store_din packs it) -> fp32 rows -------------------------------------------------------
    {
      Acc<32> acc_in;
      wg_fence();
      mma_m128<32, 1, 4>(acc_in, a1, 128, w0, 64, false);
      wg_commit();
      wg_wait();
      __syncthreads();                                              // every warp's MMA is done reading A1 (the rows overwrite it)
#pragma unroll
      for (int h = 0; h < 2; h++)
#pragma unroll
        for (int i = 0; i < 16; i += 2) {
          const uint32_t bits = pk(acc_in.d[h][i], acc_in.d[h][i + 1]);
          const int r = acc_row(tid, h, i), col = acc_col(tid, i);
          if (dfeat16 && tile * kFT + r < n_pts) *reinterpret_cast<uint32_t*>(dfeat16 + size_t(tile * kFT + r) * 32 + col) = bits;
          *reinterpret_cast<float2*>(s_rows + r * kGradLd + col) = __half22float2(*reinterpret_cast<const __half2*>(&bits));
        }
    }
    __syncthreads();
    // ---- my row: grad_w, J^T, the SH4 term ---------------------------------------------------------------------------------------
    if (valid) {
      const float x = __ldg(pts + size_t(p) * 3), y = __ldg(pts + size_t(p) * 3 + 1), z = __ldg(pts + size_t(p) * 3 + 2);
      const int v = __ldg(anchors + size_t(p) * 3);
      float gw[3];
      warped_grad(table, prim_pool, bias_pool, n_volumes, local_size, s_scale, x, y, z, v, s_rows + tid * kGradLd, gw);
      const int ray = ray_of_row(bounds, n_rays, p);
      const float tp = __ldg(t + p);
      const float dx = __ldg(dirs + size_t(p) * 3), dy = __ldg(dirs + size_t(p) * 3 + 1), dz = __ldg(dirs + size_t(p) * 3 + 2);
      const float X = ffma(tp, dx, __ldg(rays_o + ray * 3)), Y = ffma(tp, dy, __ldg(rays_o + ray * 3 + 1)),
                  Z = ffma(tp, dz, __ldg(rays_o + ray * 3 + 2));
      float J[3][3];
      warp_jacobian(trans + v, X, Y, Z, J);
      float g[3];
#pragma unroll
      for (int k = 0; k < 3; k++) g[k] = fmul(ffma(J[0][k], gw[0], ffma(J[1][k], gw[1], fmul(J[2][k], gw[2]))), inv_field_scale);
      float dsh[16];
      {
        const uint4* src = reinterpret_cast<const uint4*>(d_in + size_t(p) * 32 + 16);
#pragma unroll
        for (int q = 0; q < 2; q++) {
          const uint4 u = __ldg(src + q);
          const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
          for (int j = 0; j < 4; j++) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[j]));
            dsh[8 * q + 2 * j] = fmul(f.x, inv_shader_scale);
            dsh[8 * q + 2 * j + 1] = fmul(f.y, inv_shader_scale);
          }
        }
      }
      float gd[3];
      sh4_grad(dx, dy, dz, dsh, gd);
      float* w = row_work + size_t(p) * 6;
#pragma unroll
      for (int k = 0; k < 3; k++) { w[k] = g[k]; w[3 + k] = ffma(tp, g[k], gd[k]); }
      if (d_pts) {
#pragma unroll
        for (int k = 0; k < 3; k++) d_pts[size_t(p) * 3 + k] = g[k];
      }
      if (d_dirs) {
#pragma unroll
        for (int k = 0; k < 3; k++) d_dirs[size_t(p) * 3 + k] = gd[k];
      }
    }
    __syncthreads();                                                // the rows have been read before the next tile's A0 stores
  }
}

// d_o[r] = sum of the ray's rows' dL/dx, d_d[r] = sum of their t dL/dx + dL/ddir, serially in row order
__global__ void __launch_bounds__(128)
ray_grad_finish_kernel(const float* __restrict__ row_work, const int* __restrict__ bounds, int n_rays, float* __restrict__ d_o,
                       float* __restrict__ d_d) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  float s[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int p = bounds[2 * r]; p < bounds[2 * r + 1]; p++)
#pragma unroll
    for (int k = 0; k < 6; k++) s[k] = fadd(s[k], row_work[size_t(p) * 6 + k]);
#pragma unroll
  for (int k = 0; k < 3; k++) { d_o[size_t(r) * 3 + k] = s[k]; d_d[size_t(r) * 3 + k] = s[3 + k]; }
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
  const int grid = persistent_grid(div_up(n_pts, kFT), MB);
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

// ---- density gradient (DESIGN §3j) --------------------------------------------------------------------------------------------
template <bool SLOTS, class Src>
static void grad_launch(const void* trans, const void* table_f16, const int* prim_pool, const float* bias_pool, int n_volumes,
                        int local_size, const void* mlp_params_f16, const Src& src, int n, float empty, float* logit, float* grad,
                        const float* w_slots, float* tile_partials, void* stream) {
  const int grid = persistent_grid(div_up(n, kFT), kFieldDefaultMinB);
  cudaFuncSetAttribute(field_grad_kernel<SLOTS, Src>, cudaFuncAttributeMaxDynamicSharedMemorySize, GradSmem::BYTES);
  field_grad_kernel<SLOTS, Src><<<grid, kFT, GradSmem::BYTES, as_stream(stream)>>>(
      (const __half*)table_f16, prim_pool, bias_pool, n_volumes, local_size, (const __half*)mlp_params_f16, (const TransInfo*)trans,
      src, n, empty, logit, grad, w_slots, tile_partials);
}

extern "C" int f2b_query_grad_points(const void* tree_nodes, int n_nodes, const void* trans, const void* table_f16,
                                     const int* prim_pool, const float* bias_pool, int n_volumes, int local_size,
                                     const void* mlp_params_f16, const float* pts, int n_pts, float empty_logit, float* logit,
                                     float* grad, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(tree_nodes && n_nodes > 0 && trans && table_f16 && prim_pool && bias_pool && mlp_params_f16 && pts && logit && grad,
              "f2b_query_grad_points: null pointer");
  F2B_REQUIRE(n_volumes > 0 && local_size > 0 && (local_size % 2) == 0, "f2b_query_grad_points: bad n_volumes/local_size");
  LocateSource<false> src{(const TreeNode*)tree_nodes, (const TransInfo*)trans, pts, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0, 0, 0, empty_logit};
  grad_launch<false>(trans, table_f16, prim_pool, bias_pool, n_volumes, local_size, mlp_params_f16, src, n_pts, empty_logit, logit, grad,
                     nullptr, nullptr, stream);
  return check_launch("f2b_query_grad_points");
}

extern "C" int f2b_render_normals_slots(const void* trans, const void* table_f16, const int* prim_pool, const float* bias_pool,
                                        int n_volumes, int local_size, const void* mlp_params_f16, const float* slot_pts,
                                        const float* slot_t, const int* slot_anchors, const int* kept_counts, const float* w_slots,
                                        const float* rays_o, const float* rays_d, int n_rays, int slot_size, float* tile_partials,
                                        float* normals, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(trans && table_f16 && prim_pool && bias_pool && mlp_params_f16 && slot_pts && slot_t && slot_anchors && kept_counts &&
                  w_slots && rays_o && rays_d && tile_partials && normals,
              "f2b_render_normals_slots: null pointer");
  F2B_REQUIRE(n_volumes > 0 && local_size > 0 && (local_size % 2) == 0, "f2b_render_normals_slots: bad n_volumes/local_size");
  F2B_REQUIRE(slot_size > 0 && (slot_size % kFT) == 0, "f2b_render_normals_slots: slot_size must be a positive multiple of 128");
  F2B_REQUIRE(int64_t(n_rays) * slot_size < (int64_t(1) << 31), "f2b_render_normals_slots: n_rays * slot_size overflows int32");
  const KeptSlotSource src{slot_pts, slot_t, slot_anchors, kept_counts, rays_o, rays_d, slot_size};
  grad_launch<true>(trans, table_f16, prim_pool, bias_pool, n_volumes, local_size, mlp_params_f16, src, n_rays * slot_size, 0.f, nullptr,
                    nullptr, w_slots, tile_partials, stream);
  normals_finish_kernel<<<div_up(n_rays, 128), 128, 0, as_stream(stream)>>>(tile_partials, kept_counts, n_rays, slot_size, normals);
  return check_launch("f2b_render_normals_slots");
}

extern "C" int f2b_ray_grad(const void* trans, const void* table_f16, const int* prim_pool, const float* bias_pool, int n_volumes,
                            int local_size, const void* field_params_f16, const void* feat_f16, const void* d_field_out_f16,
                            const void* d_mlp_in_f16, const float* pts, const float* t, const float* dirs, const int* anchors,
                            const float* rays_o, const int* pts_idx_bounds, int n_rays, int n_pts, float inv_field_loss_scale,
                            float inv_shader_loss_scale, float* row_work, float* d_rays_o, float* d_rays_d, float* d_pts, float* d_dirs,
                            void* dfeat16, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(pts_idx_bounds && rays_o && d_rays_o && d_rays_d && n_pts >= 0, "f2b_ray_grad: null pointer");
  if (n_pts > 0) {
    F2B_REQUIRE(trans && table_f16 && prim_pool && bias_pool && field_params_f16 && feat_f16 && d_field_out_f16 && d_mlp_in_f16 && pts &&
                    t && dirs && anchors && row_work,
                "f2b_ray_grad: null pointer");
    F2B_REQUIRE(n_volumes > 0 && local_size > 0 && (local_size % 2) == 0, "f2b_ray_grad: bad n_volumes/local_size");
    const int grid = persistent_grid(div_up(n_pts, kFT), kRayGradMinB);
    cudaFuncSetAttribute(ray_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RayGradSmem::BYTES);
    ray_grad_kernel<<<grid, kFT, RayGradSmem::BYTES, as_stream(stream)>>>(
        (const __half*)table_f16, prim_pool, bias_pool, n_volumes, local_size, (const __half*)field_params_f16, (const TransInfo*)trans,
        (const __half*)feat_f16, (const __half*)d_field_out_f16, (const __half*)d_mlp_in_f16, pts, t, dirs, anchors, rays_o,
        pts_idx_bounds, n_rays, n_pts, inv_field_loss_scale, inv_shader_loss_scale, row_work, d_pts, d_dirs, (__half*)dfeat16);
  }
  ray_grad_finish_kernel<<<div_up(n_rays, 128), 128, 0, as_stream(stream)>>>(row_work, pts_idx_bounds, n_rays, d_rays_o, d_rays_d);
  return check_launch("f2b_ray_grad");
}
