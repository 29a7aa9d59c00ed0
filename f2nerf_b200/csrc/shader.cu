// shader.cu — SH view-direction encode, the scaled-sigmoid colour activation and the backward of the
// shader-MLP input assembly (constant-1 channel, appearance embedding).  The forward assembly runs in the
// field MLP's epilogue (shade_row in shader.cuh, called from mlp_tc.cu and fused_fwd.cu).
//
// Replaces SHKenerl (src/Shader/SHShader.cu:10-106, degree <= 4 used by every shipped config),
// the torch::cat / ones_like / ScatterIdx / ScatterAdd chain of Renderer::Render
// (src/Renderer/Renderer.cpp:179-187, src/Utils/CustomOps/Scatter.cu:10-40,110-120),
// tiny-cuda-nn's identity encoding cast (encodings/identity.h:45-85) and the sigmoid of
// SHShader::Query (src/Shader/SHShader.cpp:27-28).
#include "common.cuh"
#include "shader.cuh"

namespace f2b {

__global__ void sh_encode_kernel(const float* __restrict__ dirs, int n, int degree, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float o[16];
  sh4(dirs[size_t(i) * 3], dirs[size_t(i) * 3 + 1], dirs[size_t(i) * 3 + 2], o);
  const int m = degree * degree;
  for (int k = 0; k < m; k++) out[size_t(i) * m + k] = o[k];
}

// ScatterIdxKernal (Scatter.cu:110-120): ray -> sample broadcast of the camera index, warp per ray.
__global__ void scatter_idx_kernel(int n_rays, const int* __restrict__ bounds, const int* __restrict__ emb_idx,
                                   int* __restrict__ out) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_rays) return;
  const int v = emb_idx[ray];
  for (int i = bounds[2 * ray] + lane; i < bounds[2 * ray + 1]; i += 32) out[i] = v;
}

// rgb = (1 + 2e-3) / (1 + exp(-o)) - 1e-3 on the fp16 MLP output (SHShader.cpp:27-28)
__global__ void shader_act_kernel(const __half* __restrict__ raw, int n, float* __restrict__ rgb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
#pragma unroll
  for (int k = 0; k < 3; k++) rgb[size_t(i) * 3 + k] = shade_act(__half2float(raw[size_t(i) * 16 + k]));
}

// dL/d raw_out (fp16, times loss_scale) from dL/d rgb; channels 3..15 get zero.
__global__ void shader_act_bwd_kernel(const __half* __restrict__ raw, const float* __restrict__ d_rgb, int n,
                                      float loss_scale, __half* __restrict__ d_raw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  __half2 h[8];
#pragma unroll
  for (int k = 0; k < 8; k++) h[k] = __floats2half2_rn(0.f, 0.f);
  float g[3];
#pragma unroll
  for (int k = 0; k < 3; k++) g[k] = shade_act_bwd(__half2float(raw[size_t(i) * 16 + k]), d_rgb[size_t(i) * 3 + k], loss_scale);
  h[0] = __floats2half2_rn(g[0], g[1]);
  h[1] = __floats2half2_rn(g[2], 0.f);
  uint4* dst = reinterpret_cast<uint4*>(d_raw + size_t(i) * 16);
  dst[0] = *reinterpret_cast<uint4*>(h);
  dst[1] = *reinterpret_cast<uint4*>(h + 4);
}

// Backward of the input assembly, one warp per ray: d scene_feat[:,1:16] = d mlp_in[:,1:16] / loss_scale
// (channel 0 of scene_feat is the density logit, taken from the composite backward's d logit) and the appearance-
// embedding gradient d app_emb[cam(ray)] += sum over the ray's samples of d mlp_in[:,0:16]
// (ScatterAddFuncBackwardBlock, Scatter.cu:23-40 — there a dense [n_emb x n_blocks] compare-and-sum).  The
// camera index is constant along a ray, so the sum is a register accumulation + one warp reduction + 16
// atomicAdds per ray instead of one atomic per sample and channel.
// Lane mapping: 4 lanes per sample (4 channels each), 8 samples per warp pass — every load is a full 32 B
// sector of the row and every store instruction covers whole rows.
// The output is not d scene_feat in fp32 but what TCNNWPFunction::backward (TCNNWP.cpp:213-216) makes of it
// one call later, half((d/loss_scale_shader) * loss_scale_field): the field MLP's dL/dout row, with no fp32
// [P,16] round trip through HBM and no zero-fill.
__global__ void __launch_bounds__(256)
shader_prep_bwd_kernel(const __half* __restrict__ d_mlp_in, const float* __restrict__ d_logit,
                       const int* __restrict__ bounds, const int* __restrict__ emb_idx, int n_rays,
                       float inv_loss_scale, float out_scale, __half* __restrict__ d_out16,
                       float* __restrict__ d_app_emb) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_rays) return;
  const int beg = bounds[2 * ray], end = bounds[2 * ray + 1];
  const int sub = lane & 3;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = beg + (lane >> 2); i < end; i += 8) {
    const uint2 r = __ldg(reinterpret_cast<const uint2*>(d_mlp_in + size_t(i) * 32) + sub);
    const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&r.x));
    const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
    float g[4] = {f0.x * inv_loss_scale, f0.y * inv_loss_scale, f1.x * inv_loss_scale, f1.y * inv_loss_scale};
#pragma unroll
    for (int k = 0; k < 4; k++) acc[k] += g[k];
    if (sub == 0) g[0] = __ldg(d_logit + i);
    const __half2 h0 = __floats2half2_rn(g[0] * out_scale, g[1] * out_scale);
    const __half2 h1 = __floats2half2_rn(g[2] * out_scale, g[3] * out_scale);
    uint2 o;
    o.x = *reinterpret_cast<const uint32_t*>(&h0);
    o.y = *reinterpret_cast<const uint32_t*>(&h1);
    reinterpret_cast<uint2*>(d_out16 + size_t(i) * 16)[sub] = o;
  }
  if (d_app_emb) {
#pragma unroll
    for (int k = 0; k < 4; k++) {
      float v = acc[k];
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      acc[k] = v;
    }
    if (lane < 4 && end > beg) {
      float* dst = d_app_emb + size_t(emb_idx[ray]) * 16 + 4 * sub;
#pragma unroll
      for (int k = 0; k < 4; k++) atomicAdd(dst + k, acc[k]);
    }
  }
}

}  // namespace f2b

using namespace f2b;

extern "C" int f2b_sh_encode(const float* dirs, int n_pts, int degree, float* out, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  if (degree < 1 || degree > 4) { set_error("f2b_sh_encode: degree %d unsupported (1..4)", degree); return F2B_EUNSUPPORTED; }
  sh_encode_kernel<<<div_up(n_pts, 256), 256, 0, as_stream(stream)>>>(dirs, n_pts, degree, out);
  return check_launch("f2b_sh_encode");
}

extern "C" int f2b_scatter_idx(const int* pts_idx_bounds, const int* emb_idx, int n_rays, int* out, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  scatter_idx_kernel<<<div_up(int64_t(n_rays) * 32, 256), 256, 0, as_stream(stream)>>>(n_rays, pts_idx_bounds, emb_idx, out);
  return check_launch("f2b_scatter_idx");
}

extern "C" int f2b_shader_act(const void* raw_out_f16, int n_pts, float* rgb, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  shader_act_kernel<<<div_up(n_pts, 256), 256, 0, as_stream(stream)>>>((const __half*)raw_out_f16, n_pts, rgb);
  return check_launch("f2b_shader_act");
}

extern "C" int f2b_shader_act_bwd(const void* raw_out_f16, const float* d_rgb, int n_pts, float loss_scale,
                                  void* d_raw_f16, void* stream) {
  if (n_pts <= 0) return F2B_OK;
  shader_act_bwd_kernel<<<div_up(n_pts, 256), 256, 0, as_stream(stream)>>>((const __half*)raw_out_f16, d_rgb, n_pts,
                                                                          loss_scale, (__half*)d_raw_f16);
  return check_launch("f2b_shader_act_bwd");
}

extern "C" int f2b_shader_prep_bwd_f16(const void* d_mlp_in_f16, const float* d_logit, const int* pts_idx_bounds,
                                       const int* emb_idx, int n_rays, float inv_loss_scale, float field_loss_scale,
                                       void* d_field_out_f16, float* d_app_emb, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(d_mlp_in_f16 && d_logit && pts_idx_bounds && d_field_out_f16, "f2b_shader_prep_bwd_f16: null pointer");
  F2B_REQUIRE(!d_app_emb || emb_idx, "f2b_shader_prep_bwd_f16: d_app_emb without emb_idx");
  shader_prep_bwd_kernel<<<div_up(int64_t(n_rays) * 32, 256), 256, 0, as_stream(stream)>>>(
      (const __half*)d_mlp_in_f16, d_logit, pts_idx_bounds, emb_idx, n_rays, inv_loss_scale, field_loss_scale,
      (__half*)d_field_out_f16, d_app_emb);
  return check_launch("f2b_shader_prep_bwd_f16");
}
