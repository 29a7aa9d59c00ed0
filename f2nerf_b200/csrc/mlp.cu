// mlp.cu — tiny bias-free ReLU MLPs (32 -> 64 [-> 64] -> 16) of the field and the shader.
//
// Replaces TCNNWP::Query / TCNNWPFunction::{forward,backward} (src/Field/TCNNWP.cpp:102-243) and
// the tiny-cuda-nn kernels they reach: kernel_mlp_fused / kernel_mlp_fused_backward
// (External/tiny-cuda-nn/src/fully_fused_mlp.cu:150-259,499-557) and the three split-K CUTLASS
// weight-gradient GEMMs (fully_fused_mlp.cu:785,819,828).
//
// This file is the CUDA-core implementation (impl 0): fp16 operands, fp32 accumulation, hidden
// activations and outputs rounded to fp16 exactly where tiny-cuda-nn stores them.  It is the
// validation twin of the wgmma tensor-core kernels in mlp_tc.cu (impl 1) and shares their C ABI.
// Parameter layout (fully_fused_mlp.cu:654-677): [W0 64x32 | Wh 64x64 (x n_hidden_matmuls) | Wout 16x64],
// row-major [out][in], fp16.
#include "common.cuh"

namespace f2b {

constexpr int kTile = 128;          // samples per tile == threads per block
constexpr int kW = F2B_MLP_WIDTH;   // 64
constexpr int kIn = F2B_MLP_IN;     // 32
constexpr int kOut = F2B_MLP_OUT_PAD;  // 16
constexpr int kHPitch = kW + 8;     // halfs; +16 B skew keeps 128-bit row reads conflict free

__device__ __forceinline__ float h2f(__half h) { return __half2float(h); }

// y[o] = sum_k x[k] * W[o][k], W fp32 in shared memory (broadcast reads), 8 outputs at a time
template <int K>
__device__ __forceinline__ void dense8(const float* __restrict__ Wrow0, const float (&x)[K], float (&acc)[8]) {
#pragma unroll
  for (int o = 0; o < 8; o++) {
    float a = 0.f;
#pragma unroll
    for (int k = 0; k < K; k += 4) {
      const float4 w = *reinterpret_cast<const float4*>(Wrow0 + o * K + k);
      a = fmaf(x[k], w.x, a); a = fmaf(x[k + 1], w.y, a); a = fmaf(x[k + 2], w.z, a); a = fmaf(x[k + 3], w.w, a);
    }
    acc[o] = a;
  }
}

template <int K>
__device__ __forceinline__ void load_row_half(const __half* row, float (&x)[K]) {
#pragma unroll
  for (int k = 0; k < K; k += 8) {
    const uint4 r = *reinterpret_cast<const uint4*>(row + k);
    const __half2* h = reinterpret_cast<const __half2*>(&r);
#pragma unroll
    for (int q = 0; q < 4; q++) { const float2 f = __half22float2(h[q]); x[k + 2 * q] = f.x; x[k + 2 * q + 1] = f.y; }
  }
}

// ---------------------------------------------------------------- forward ------------------
template <int NH>
__global__ void __launch_bounds__(kTile)
mlp_fwd_v0_kernel(const __half* __restrict__ in, const __half* __restrict__ params, int n_pts,
                  __half* __restrict__ out, __half* __restrict__ hidden_save) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* W0 = reinterpret_cast<float*>(smem_raw);           // [64][32]
  float* Wh = W0 + kW * kIn;                                // [NH][64][64]
  float* Wo = Wh + NH * kW * kW;                            // [16][64]
  __half* hbuf = reinterpret_cast<__half*>(Wo + kOut * kW); // [128][kHPitch]
  const int n_params = kW * kIn + NH * kW * kW + kOut * kW;
  for (int i = threadIdx.x; i < n_params; i += kTile) W0[i] = h2f(params[i]);
  __syncthreads();

  const int n_tiles = (n_pts + kTile - 1) / kTile;
  __half* hrow = hbuf + threadIdx.x * kHPitch;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int p = tile * kTile + threadIdx.x;
    const bool valid = p < n_pts;
    float x[kIn];
    if (valid) load_row_half<kIn>(in + size_t(p) * kIn, x);
    else {
#pragma unroll
      for (int k = 0; k < kIn; k++) x[k] = 0.f;
    }
    // layer 0: 32 -> 64, ReLU, round to fp16
    for (int oc = 0; oc < kW; oc += 8) {
      float acc[8];
      dense8<kIn>(W0 + oc * kIn, x, acc);
      __half2 h[4];
#pragma unroll
      for (int q = 0; q < 4; q++) h[q] = __floats2half2_rn(fmaxf(acc[2 * q], 0.f), fmaxf(acc[2 * q + 1], 0.f));
      *reinterpret_cast<uint4*>(hrow + oc) = *reinterpret_cast<uint4*>(h);
    }
    if (hidden_save && valid) {
      uint4* dst = reinterpret_cast<uint4*>(hidden_save + size_t(p) * kW);
#pragma unroll
      for (int q = 0; q < 8; q++) dst[q] = *reinterpret_cast<const uint4*>(hrow + 8 * q);
    }
    float hcur[kW];
    load_row_half<kW>(hrow, hcur);
    if (NH) {
      for (int oc = 0; oc < kW; oc += 8) {
        float acc[8];
        dense8<kW>(Wh + oc * kW, hcur, acc);
        __half2 h[4];
#pragma unroll
        for (int q = 0; q < 4; q++) h[q] = __floats2half2_rn(fmaxf(acc[2 * q], 0.f), fmaxf(acc[2 * q + 1], 0.f));
        *reinterpret_cast<uint4*>(hrow + oc) = *reinterpret_cast<uint4*>(h);
      }
      if (hidden_save && valid) {
        uint4* dst = reinterpret_cast<uint4*>(hidden_save + size_t(n_pts) * kW + size_t(p) * kW);
#pragma unroll
        for (int q = 0; q < 8; q++) dst[q] = *reinterpret_cast<const uint4*>(hrow + 8 * q);
      }
      load_row_half<kW>(hrow, hcur);
    }
    // output layer: 64 -> 16, linear, round to fp16
    if (valid) {
      uint4* dst = reinterpret_cast<uint4*>(out + size_t(p) * kOut);
#pragma unroll
      for (int oc = 0; oc < kOut; oc += 8) {
        float acc[8];
        dense8<kW>(Wo + oc * kW, hcur, acc);
        __half2 h[4];
#pragma unroll
        for (int q = 0; q < 4; q++) h[q] = __floats2half2_rn(acc[2 * q], acc[2 * q + 1]);
        dst[oc / 8] = *reinterpret_cast<uint4*>(h);
      }
    }
  }
}

// ---------------------------------------------------------------- backward -----------------
// Persistent blocks; per 128-sample tile:
//   dH_last = (dOut . Wout)   * [h_last > 0]         (fp16, as tiny-cuda-nn's backward activations)
//   dH_0    = (dH_last . Wh)  * [h_0 > 0]            (NH == 1)
//   dIn     =  dH_0 . W0                              (optional)
//   dWout  += dOut^T h_last ; dWh += dH_last^T h_0 ; dW0 += dH_0^T in   (fp32 registers across tiles,
//   one atomicAdd flush per block — replaces three split-K fp16 GEMMs and their reductions).
template <int NH>
__global__ void __launch_bounds__(kTile)
mlp_bwd_v0_kernel(const __half* __restrict__ dout, const __half* __restrict__ in,
                  const __half* __restrict__ hidden, const __half* __restrict__ hid_last,
                  const __half* __restrict__ params, int n_pts, __half* __restrict__ din, float* __restrict__ dparams) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  // transposed fp32 weights so the backward products read rows:  WoT [64][16], WhT [64][64], W0T [32][64]
  float* WoT = reinterpret_cast<float*>(smem_raw);
  float* WhT = WoT + kW * kOut;
  float* W0T = WhT + NH * kW * kW;
  __half* t_dout = reinterpret_cast<__half*>(W0T + kIn * kW);  // [128][16+8]
  __half* t_in = t_dout + kTile * (kOut + 8);                  // [128][32+8]
  __half* t_h0 = t_in + kTile * (kIn + 8);                     // [128][kHPitch]
  __half* t_dh0 = t_h0 + kTile * kHPitch;                      // [128][kHPitch]
  __half* t_h1 = t_dh0 + kTile * kHPitch;                      // NH only
  __half* t_dh1 = t_h1 + NH * kTile * kHPitch;                 // NH only
  const __half* pW0 = params;
  const __half* pWh = params + kW * kIn;
  const __half* pWo = pWh + NH * kW * kW;
  for (int i = threadIdx.x; i < kOut * kW; i += kTile) { const int o = i / kW, j = i % kW; WoT[j * kOut + o] = h2f(pWo[i]); }
  if (NH) for (int i = threadIdx.x; i < kW * kW; i += kTile) { const int o = i / kW, j = i % kW; WhT[j * kW + o] = h2f(pWh[i]); }
  for (int i = threadIdx.x; i < kW * kIn; i += kTile) { const int o = i / kIn, k = i % kIn; W0T[k * kW + o] = h2f(pW0[i]); }

  // weight-gradient register tiles
  const int t = threadIdx.x;
  float gW0[16];   // rows o0..o0+3 (o0 = (t/8)*4), cols k0..k0+3 (k0 = (t%8)*4)
  float gWh[32];   // rows o0..o0+3 (o0 = (t/8)*4), cols j0..j0+7 (j0 = (t%8)*8)
  float gWo[8];    // rows o0..o0+7 (o0 = (t/64)*8), col j = t%64
#pragma unroll
  for (int i = 0; i < 16; i++) gW0[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 32; i++) gWh[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; i++) gWo[i] = 0.f;
  __syncthreads();

  const int n_tiles = (n_pts + kTile - 1) / kTile;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int p = tile * kTile + t;
    const bool valid = p < n_pts;
    // stage this thread's row of every operand
    {
      uint4 z = make_uint4(0, 0, 0, 0);
      const uint4* s;
      s = reinterpret_cast<const uint4*>(dout + size_t(p) * kOut);
#pragma unroll
      for (int q = 0; q < 2; q++) *reinterpret_cast<uint4*>(t_dout + t * (kOut + 8) + 8 * q) = valid ? s[q] : z;
      s = reinterpret_cast<const uint4*>(in + size_t(p) * kIn);
#pragma unroll
      for (int q = 0; q < 4; q++) *reinterpret_cast<uint4*>(t_in + t * (kIn + 8) + 8 * q) = valid ? s[q] : z;
      s = reinterpret_cast<const uint4*>(hidden + size_t(p) * kW);
#pragma unroll
      for (int q = 0; q < 8; q++) *reinterpret_cast<uint4*>(t_h0 + t * kHPitch + 8 * q) = valid ? s[q] : z;
      if (NH) {
        s = reinterpret_cast<const uint4*>(hid_last + size_t(p) * kW);
#pragma unroll
        for (int q = 0; q < 8; q++) *reinterpret_cast<uint4*>(t_h1 + t * kHPitch + 8 * q) = valid ? s[q] : z;
      }
    }
    // dH_last = dOut . Wout, masked by the last hidden activation
    {
      float g[kOut];
      load_row_half<kOut>(t_dout + t * (kOut + 8), g);
      const __half* hl = (NH ? t_h1 : t_h0) + t * kHPitch;
      __half* dst = (NH ? t_dh1 : t_dh0) + t * kHPitch;
      for (int jc = 0; jc < kW; jc += 8) {
        float acc[8];
        dense8<kOut>(WoT + jc * kOut, g, acc);
        const uint4 hr = *reinterpret_cast<const uint4*>(hl + jc);
        const __half2* hh = reinterpret_cast<const __half2*>(&hr);
        __half2 o[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const float2 hv = __half22float2(hh[q]);
          o[q] = __floats2half2_rn(hv.x > 0.f ? acc[2 * q] : 0.f, hv.y > 0.f ? acc[2 * q + 1] : 0.f);
        }
        *reinterpret_cast<uint4*>(dst + jc) = *reinterpret_cast<uint4*>(o);
      }
    }
    if (NH) {   // dH_0 = dH_last . Wh, masked by h_0
      float g[kW];
      load_row_half<kW>(t_dh1 + t * kHPitch, g);
      for (int jc = 0; jc < kW; jc += 8) {
        float acc[8];
        dense8<kW>(WhT + jc * kW, g, acc);
        const uint4 hr = *reinterpret_cast<const uint4*>(t_h0 + t * kHPitch + jc);
        const __half2* hh = reinterpret_cast<const __half2*>(&hr);
        __half2 o[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const float2 hv = __half22float2(hh[q]);
          o[q] = __floats2half2_rn(hv.x > 0.f ? acc[2 * q] : 0.f, hv.y > 0.f ? acc[2 * q + 1] : 0.f);
        }
        *reinterpret_cast<uint4*>(t_dh0 + t * kHPitch + jc) = *reinterpret_cast<uint4*>(o);
      }
    }
    if (din) {  // dIn = dH_0 . W0
      float g[kW];
      load_row_half<kW>(t_dh0 + t * kHPitch, g);
      uint4* dst = reinterpret_cast<uint4*>(din + size_t(p) * kIn);
#pragma unroll
      for (int kc = 0; kc < kIn; kc += 8) {
        float acc[8];
        dense8<kW>(W0T + kc * kW, g, acc);
        __half2 o[4];
#pragma unroll
        for (int q = 0; q < 4; q++) o[q] = __floats2half2_rn(acc[2 * q], acc[2 * q + 1]);
        if (valid) dst[kc / 8] = *reinterpret_cast<uint4*>(o);
      }
    }
    __syncthreads();
    // weight gradients over the tile's 128 samples
    {
      const int o0 = (t / 8) * 4, k0 = (t % 8) * 4, j0 = (t % 8) * 8;
      const int oo = (t / 64) * 8, jj = t % 64;
      for (int q = 0; q < kTile; q++) {
        const __half* rdh0 = t_dh0 + q * kHPitch;
        float a[4];
        { const uint2 r = *reinterpret_cast<const uint2*>(rdh0 + o0); const __half2* h = reinterpret_cast<const __half2*>(&r);
          const float2 f0 = __half22float2(h[0]), f1 = __half22float2(h[1]); a[0] = f0.x; a[1] = f0.y; a[2] = f1.x; a[3] = f1.y; }
        float b[4];
        { const uint2 r = *reinterpret_cast<const uint2*>(t_in + q * (kIn + 8) + k0); const __half2* h = reinterpret_cast<const __half2*>(&r);
          const float2 f0 = __half22float2(h[0]), f1 = __half22float2(h[1]); b[0] = f0.x; b[1] = f0.y; b[2] = f1.x; b[3] = f1.y; }
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) gW0[i * 4 + j] = fmaf(a[i], b[j], gW0[i * 4 + j]);
        if (NH) {
          float c[4], d[8];
          { const uint2 r = *reinterpret_cast<const uint2*>(t_dh1 + q * kHPitch + o0); const __half2* h = reinterpret_cast<const __half2*>(&r);
            const float2 f0 = __half22float2(h[0]), f1 = __half22float2(h[1]); c[0] = f0.x; c[1] = f0.y; c[2] = f1.x; c[3] = f1.y; }
          load_row_half<8>(t_h0 + q * kHPitch + j0, d);
#pragma unroll
          for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = 0; j < 8; j++) gWh[i * 8 + j] = fmaf(c[i], d[j], gWh[i * 8 + j]);
        }
        float e[8];
        load_row_half<8>(t_dout + q * (kOut + 8) + oo, e);
        const float hv = h2f(((NH ? t_h1 : t_h0) + q * kHPitch)[jj]);
#pragma unroll
        for (int i = 0; i < 8; i++) gWo[i] = fmaf(e[i], hv, gWo[i]);
      }
    }
    __syncthreads();
  }
  // flush
  {
    const int o0 = (t / 8) * 4, k0 = (t % 8) * 4, j0 = (t % 8) * 8;
    const int oo = (t / 64) * 8, jj = t % 64;
    float* gp0 = dparams;
    float* gph = dparams + kW * kIn;
    float* gpo = gph + NH * kW * kW;
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = 0; j < 4; j++) atomicAdd(gp0 + (o0 + i) * kIn + k0 + j, gW0[i * 4 + j]);
    if (NH) {
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) atomicAdd(gph + (o0 + i) * kW + j0 + j, gWh[i * 8 + j]);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) atomicAdd(gpo + (oo + i) * kW + jj, gWo[i]);
  }
}

static size_t fwd_smem(int nh) { return sizeof(float) * (kW * kIn + nh * kW * kW + kOut * kW) + sizeof(__half) * kTile * kHPitch; }
static size_t bwd_smem(int nh) {
  return sizeof(float) * (kW * kOut + nh * kW * kW + kIn * kW) +
         sizeof(__half) * (kTile * (kOut + 8) + kTile * (kIn + 8) + (2 + 2 * nh) * kTile * kHPitch);
}

}  // namespace f2b

using namespace f2b;

extern "C" int f2b_mlp_fwd_v0(const void* in_f16, const void* params_f16, int n_hidden_matmuls, int n_pts,
                              void* out_f16, void* hidden_save_f16, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(in_f16 && params_f16 && out_f16, "f2b_mlp_fwd: null pointer");
  F2B_REQUIRE(n_hidden_matmuls == 0 || n_hidden_matmuls == 1, "f2b_mlp_fwd: n_hidden_matmuls must be 0 or 1");
  int sms = 132;
  f2b_device_info(&sms, nullptr);
  const int n_tiles = div_up(n_pts, kTile);
  const int grid = n_tiles < sms * 8 ? n_tiles : sms * 8;
  const size_t smem = fwd_smem(n_hidden_matmuls);
  if (n_hidden_matmuls == 0) {
    cudaFuncSetAttribute(mlp_fwd_v0_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    mlp_fwd_v0_kernel<0><<<grid, kTile, smem, as_stream(stream)>>>((const __half*)in_f16, (const __half*)params_f16, n_pts,
                                                                 (__half*)out_f16, (__half*)hidden_save_f16);
  } else {
    cudaFuncSetAttribute(mlp_fwd_v0_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    mlp_fwd_v0_kernel<1><<<grid, kTile, smem, as_stream(stream)>>>((const __half*)in_f16, (const __half*)params_f16, n_pts,
                                                                 (__half*)out_f16, (__half*)hidden_save_f16);
  }
  return check_launch("f2b_mlp_fwd");
}

extern "C" int f2b_mlp_bwd2_v0(const void* dout_f16, const void* in_f16, const void* hidden0_f16, const void* hidden1_f16,
                               const void* params_f16, int n_hidden_matmuls, int n_pts, void* din_f16,
                               float* dparams_f32, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(dout_f16 && in_f16 && hidden0_f16 && params_f16 && dparams_f32, "f2b_mlp_bwd: null pointer");
  F2B_REQUIRE(n_hidden_matmuls == 0 || (n_hidden_matmuls == 1 && hidden1_f16), "f2b_mlp_bwd: n_hidden_matmuls must be 0 or 1 (with hidden1)");
  int sms = 132;
  f2b_device_info(&sms, nullptr);
  const int n_tiles = div_up(n_pts, kTile);
  const int grid = n_tiles < sms * 2 ? n_tiles : sms * 2;
  const size_t smem = bwd_smem(n_hidden_matmuls);
  if (n_hidden_matmuls == 0) {
    cudaFuncSetAttribute(mlp_bwd_v0_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    mlp_bwd_v0_kernel<0><<<grid, kTile, smem, as_stream(stream)>>>((const __half*)dout_f16, (const __half*)in_f16,
                                                                 (const __half*)hidden0_f16, (const __half*)hidden0_f16,
                                                                 (const __half*)params_f16, n_pts, (__half*)din_f16, dparams_f32);
  } else {
    cudaFuncSetAttribute(mlp_bwd_v0_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    mlp_bwd_v0_kernel<1><<<grid, kTile, smem, as_stream(stream)>>>((const __half*)dout_f16, (const __half*)in_f16,
                                                                 (const __half*)hidden0_f16, (const __half*)hidden1_f16,
                                                                 (const __half*)params_f16, n_pts, (__half*)din_f16, dparams_f32);
  }
  return check_launch("f2b_mlp_bwd");
}

extern "C" int f2b_mlp_bwd_v0(const void* dout_f16, const void* in_f16, const void* hidden_save_f16,
                              const void* params_f16, int n_hidden_matmuls, int n_pts, void* din_f16,
                              float* dparams_f32, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  F2B_REQUIRE(hidden_save_f16, "f2b_mlp_bwd: null pointer");
  const __half* h = (const __half*)hidden_save_f16;
  return f2b_mlp_bwd2_v0(dout_f16, in_f16, h, h + size_t(n_hidden_matmuls ? 1 : 0) * n_pts * kW, params_f16, n_hidden_matmuls, n_pts,
                         din_f16, dparams_f32, stream);
}
