// composite.cu — front-to-back alpha compositing, early-stop compaction and the per-ray
// segmented ops, one warp per ray, for sm_90a.
//
// Replaces the tail of Renderer::Render (src/Renderer/Renderer.cpp:107-150 early-stop pass,
// :196-208 composite), TruncExp (src/Utils/CustomOps/CustomOps.cpp:9-18), FlexOps::Sum /
// AccumulateSum (src/Utils/CustomOps/FlexOps.cu:5-93), FilterIdxBounds + CountValidPts
// (src/Renderer/Renderer.cu:8-50), the where/index gather-compaction (Renderer.cpp:126-132),
// GradientScaling backward (CustomOps.cu:68-80) and WeightVarLoss (CustomOps.cu:12-66).
//
// The reference spends ~25 ATen launches (each a full pass over all samples) plus thread-per-ray
// serial kernels here.  This is pure HBM streaming: one kernel reads 24 B/sample once and
// writes 4 B/sample.  Lanes load 32 consecutive samples (coalesced); the per-ray prefix/sums are
// then chained IN THE REFERENCE'S serial left-to-right order through warp shuffles, so forward
// values (and the early-stop mask / compacted indices that depend on them) round exactly like
// FlexAccumulateSumForwardKernel / FlexSumForwardKernel do.  Backward uses ordinary warp scans.
#include "common.cuh"
#include "scan.cuh"
#include "shader.cuh"

namespace f2b {

constexpr unsigned kFull = 0xffffffffu;

// serial-order exclusive prefix over the warp's 32 values; `run` carries across chunks.
// returns this lane's exclusive prefix; n_valid = number of valid lanes in the chunk.
__device__ __forceinline__ float chain_excl(float v, float& run, int n_valid, int lane) {
  float mine = 0.f;
  for (int j = 0; j < n_valid; j++) {
    const float vj = __shfl_sync(kFull, v, j);
    if (lane == j) mine = run;
    run = fadd(run, vj);
  }
  return mine;
}
// serial-order sum
__device__ __forceinline__ void chain_sum(float v, float& run, int n_valid) {
  for (int j = 0; j < n_valid; j++) run = fadd(run, __shfl_sync(kFull, v, j));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

// ---- early stop (no-grad pass): weights, alphas, keep mask, per-ray survivor counts ------------
__global__ void __launch_bounds__(256)
early_stop_kernel(const float* __restrict__ logit, int logit_stride, const float* __restrict__ dt,
                  const int* __restrict__ bounds, int n_rays, float* __restrict__ weights,
                  float* __restrict__ alphas, uint8_t* __restrict__ keep, int* __restrict__ counts) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_rays) return;
  const int beg = bounds[2 * ray], end = bounds[2 * ray + 1];
  float run = 0.f;
  int cnt = 0;
  for (int base = beg; base < end; base += 32) {
    const int i = base + lane;
    const bool valid = i < end;
    float tau = 0.f, alpha = 0.f;
    if (valid) {
      const float dens = expf(fsub(__ldg(logit + size_t(i) * logit_stride), 3.f));   // TruncExp(x - 3)
      tau = fmul(dens, __ldg(dt + i));
      alpha = fsub(1.f, expf(-tau));
    }
    const float acc = chain_excl(tau, run, min(32, end - base), lane);
    const float trans = expf(-acc);
    const bool k = valid && (trans > 1e-4f);
    if (valid) {
      weights[i] = fmul(trans, alpha);
      alphas[i] = alpha;
      keep[i] = k ? 1 : 0;
    }
    cnt += __popc(__ballot_sync(kFull, k));
  }
  if (lane == 0) counts[ray] = cnt;
}

// ---- gather-compaction of the surviving samples ------------------------------------------------
__global__ void __launch_bounds__(256)
compact_kernel(const uint8_t* __restrict__ keep, const int* __restrict__ old_bounds,
               const int* __restrict__ new_bounds, int n_rays, const float* __restrict__ pts,
               const float* __restrict__ dirs, const float* __restrict__ dt, const float* __restrict__ t,
               const int* __restrict__ anchors, const uint4* __restrict__ feat, float* __restrict__ pts_o,
               float* __restrict__ dirs_o, float* __restrict__ dt_o, float* __restrict__ t_o,
               int* __restrict__ anchors_o, uint4* __restrict__ feat_o) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_rays) return;
  const int beg = old_bounds[2 * ray], end = old_bounds[2 * ray + 1];
  int out = new_bounds[2 * ray];
  for (int base = beg; base < end; base += 32) {
    const int i = base + lane;
    const bool k = (i < end) && keep[i];
    const unsigned m = __ballot_sync(kFull, k);
    if (k) {
      const size_t o = size_t(out) + __popc(m & ((1u << lane) - 1u));
      const size_t s = size_t(i);
#pragma unroll
      for (int c = 0; c < 3; c++) {
        pts_o[o * 3 + c] = pts[s * 3 + c];
        dirs_o[o * 3 + c] = dirs[s * 3 + c];
        anchors_o[o * 3 + c] = anchors[s * 3 + c];
      }
      dt_o[o] = dt[s];
      t_o[o] = t[s];
      if (feat) {                                  // the sample's 32 encoded halfs (64 B) from the early-stop pass
#pragma unroll
        for (int c = 0; c < 4; c++) feat_o[o * 4 + c] = feat[s * 4 + c];
      }
    }
    out += __popc(m);
  }
}

// Same compaction straight out of the one-pass march's scratch slots (ray r owns slots
// [r*slot, r*slot + count[r]); 28 B/sample there): directions are the ray's, anchors[:,2] is 0 — the
// all-sample SampleResultFlex the reference materialises between march and early stop is never built.
__global__ void __launch_bounds__(256)
compact_slots_kernel(const uint8_t* __restrict__ keep, const int* __restrict__ slot_bounds,
                     const int* __restrict__ new_bounds, int n_rays, const float* __restrict__ rays_d,
                     const float* __restrict__ s_pts, const float* __restrict__ s_dt, const float* __restrict__ s_t,
                     const int* __restrict__ s_anchors, const uint4* __restrict__ feat, float* __restrict__ pts_o,
                     float* __restrict__ dirs_o, float* __restrict__ dt_o, float* __restrict__ t_o,
                     int* __restrict__ anchors_o, uint4* __restrict__ feat_o) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_rays) return;
  const int beg = slot_bounds[2 * ray], end = slot_bounds[2 * ray + 1];
  const float d0 = __ldg(rays_d + ray * 3), d1 = __ldg(rays_d + ray * 3 + 1), d2 = __ldg(rays_d + ray * 3 + 2);
  int out = new_bounds[2 * ray];
  for (int base = beg; base < end; base += 32) {
    const int i = base + lane;
    const bool k = (i < end) && keep[i];
    const unsigned m = __ballot_sync(kFull, k);
    if (k) {
      const size_t o = size_t(out) + __popc(m & ((1u << lane) - 1u));
      const size_t s = size_t(i);
      pts_o[o * 3] = s_pts[s * 3]; pts_o[o * 3 + 1] = s_pts[s * 3 + 1]; pts_o[o * 3 + 2] = s_pts[s * 3 + 2];
      dirs_o[o * 3] = d0; dirs_o[o * 3 + 1] = d1; dirs_o[o * 3 + 2] = d2;
      anchors_o[o * 3] = s_anchors[s * 2]; anchors_o[o * 3 + 1] = s_anchors[s * 2 + 1]; anchors_o[o * 3 + 2] = 0;
      dt_o[o] = s_dt[s];
      t_o[o] = s_t[s];
      if (feat) {
#pragma unroll
        for (int c = 0; c < 4; c++) feat_o[o * 4 + c] = feat[s * 4 + c];
      }
    }
    out += __popc(m);
  }
}

__global__ void slot_bounds_kernel(const int* __restrict__ counts, int n_rays, int slot, int first_ray, int* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  const int b = (first_ray + r) * slot;
  out[2 * r] = b;
  out[2 * r + 1] = b + counts[r];
}

// ---- forward composite ------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
composite_fwd_kernel(const float* __restrict__ logit, int logit_stride, const float* __restrict__ rgb,
                     const float* __restrict__ dt, const float* __restrict__ t,
                     const int* __restrict__ bounds, const float* __restrict__ bg, int n_rays,
                     float* __restrict__ colors, float* __restrict__ disparity, float* __restrict__ depth,
                     float* __restrict__ weights) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_rays) return;
  const int beg = bounds[2 * ray], end = bounds[2 * ray + 1];
  // The five per-ray sums (FlexOps::Sum: serial left-to-right per ray, FlexOps.cu:5-30) are independent serial chains:
  // lanes 0..4 each own one and walk the chunk's 32 addends out of shared memory (32 LDS + 32 FADD for all five
  // together) instead of five 32-step shuffle chains executed by every lane — same additions in the same order.
  __shared__ float s_add[8][5][32];
  float (*sa)[32] = s_add[threadIdx.x >> 5];
  float run = 0.f, acc5 = 0.f;                                  // acc5: lane c < 5 holds sum c (r, g, b, w/t, w*t)
  for (int base = beg; base < end; base += 32) {
    const int i = base + lane;
    const bool valid = i < end;
    const int nv = min(32, end - base);
    float tau = 0.f, alpha = 0.f, ts = 1.f, r = 0.f, g = 0.f, b = 0.f;
    if (valid) {
      const float dens = expf(fsub(__ldg(logit + size_t(i) * logit_stride), 3.f));
      tau = fmul(dens, __ldg(dt + i));
      alpha = fsub(1.f, expf(-tau));
      ts = fadd(__ldg(t + i), 1e-2f);
      r = __ldg(rgb + size_t(i) * 3); g = __ldg(rgb + size_t(i) * 3 + 1); b = __ldg(rgb + size_t(i) * 3 + 2);
    }
    const float acc = chain_excl(tau, run, nv, lane);
    const float w = fmul(expf(-acc), alpha);
    if (valid) weights[i] = w;
    sa[0][lane] = fmul(w, r); sa[1][lane] = fmul(w, g); sa[2][lane] = fmul(w, b);
    sa[3][lane] = fdiv(w, ts); sa[4][lane] = fmul(w, ts);
    __syncwarp();
    if (lane < 5) {
      const float* mine = sa[lane];
      for (int j = 0; j < nv; j++) acc5 = fadd(acc5, mine[j]);
    }
    __syncwarp();
  }
  const float cr = __shfl_sync(kFull, acc5, 0), cg = __shfl_sync(kFull, acc5, 1), cb = __shfl_sync(kFull, acc5, 2);
  const float sd = __shfl_sync(kFull, acc5, 3), sz = __shfl_sync(kFull, acc5, 4);
  if (lane == 0) {
    const float lt = expf(-run);                              // last_trans = exp(-Sum(sec_density))
    colors[ray * 3 + 0] = fadd(cr, fmul(lt, bg[ray * 3 + 0]));
    colors[ray * 3 + 1] = fadd(cg, fmul(lt, bg[ray * 3 + 1]));
    colors[ray * 3 + 2] = fadd(cb, fmul(lt, bg[ray * 3 + 2]));
    disparity[ray] = sd;
    depth[ray] = fdiv(sz, fadd(fsub(1.f, lt), 1e-4f));
  }
}

// ---- backward composite -----------------------------------------------------------------------
// sweep 1 (front to back): exclusive optical depth A_i (serial order, parked in d_logit), S, Zs.
// sweep 2 (back to front): per-sample gradients with a reverse warp scan for sum_{k>i} dA_k.
template <bool FUSE_ACT>
__global__ void __launch_bounds__(256)
composite_bwd_kernel(const float* __restrict__ logit, int logit_stride, const float* __restrict__ rgb,
                     const float* __restrict__ dt, const float* __restrict__ t,
                     const int* __restrict__ bounds, const float* __restrict__ bg, int n_rays,
                     const float* __restrict__ d_colors, const float* __restrict__ d_disp,
                     const float* __restrict__ d_depth, const float* __restrict__ d_weights,
                     float gs_progress, float* __restrict__ d_logit, int dlogit_stride,
                     float* __restrict__ d_rgb, const __half* __restrict__ raw, __half* __restrict__ d_raw,
                     float act_loss_scale) {
  // FUSE_ACT: the colour gradient goes straight through the scaled sigmoid's backward (SHShader.cpp:27-28) into the
  // shader MLP's fp16 dL/dout row [g_r, g_g, g_b, 0 x 13] * loss_scale instead of being written as fp32 d_rgb.
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_rays) return;
  const int beg = bounds[2 * ray], end = bounds[2 * ray + 1];
  const int n = end - beg;
  if (n <= 0) return;
  float run = 0.f, zs = 0.f;
  for (int base = beg; base < end; base += 32) {
    const int i = base + lane;
    const bool valid = i < end;
    float tau = 0.f, alpha = 0.f, ts = 0.f;
    if (valid) {
      const float dens = expf(fsub(__ldg(logit + size_t(i) * logit_stride), 3.f));
      tau = fmul(dens, __ldg(dt + i));
      alpha = fsub(1.f, expf(-tau));
      ts = fadd(__ldg(t + i), 1e-2f);
    }
    const float acc = chain_excl(tau, run, min(32, end - base), lane);
    if (valid) {
      d_logit[size_t(i) * dlogit_stride] = acc;
      zs += expf(-acc) * alpha * ts;
    }
  }
  zs = warp_sum(zs);
  const float lt = expf(-run);
  const float dcr = d_colors[ray * 3], dcg = d_colors[ray * 3 + 1], dcb = d_colors[ray * 3 + 2];
  const float ddisp = d_disp ? d_disp[ray] : 0.f;
  const float den = (1.f - lt) + 1e-4f;
  const float ddep = d_depth ? d_depth[ray] / den : 0.f;           // d depth / d Zs
  // d loss / d last_trans, then / d S (S = sum tau, last_trans = exp(-S))
  const float dlt = dcr * bg[ray * 3] + dcg * bg[ray * 3 + 1] + dcb * bg[ray * 3 + 2] +
                    (d_depth ? d_depth[ray] * zs / (den * den) : 0.f);
  const float dS = -lt * dlt;
  const bool scaling = gs_progress < 1.f;
  float carry = 0.f;                                                // sum of dA over later chunks
  const int n_chunks = (n + 31) / 32;
  for (int c = n_chunks - 1; c >= 0; c--) {
    const int i = beg + c * 32 + lane;
    const bool valid = i < end;
    float dA = 0.f, direct = 0.f, dens = 0.f, dtv = 0.f, x = 0.f, w = 0.f, r = 0.f, g = 0.f, b = 0.f;
    if (valid) {
      x = fsub(__ldg(logit + size_t(i) * logit_stride), 3.f);
      dens = expf(x);
      dtv = __ldg(dt + i);
      const float tau = fmul(dens, dtv);
      const float e = expf(-tau);
      const float alpha = fsub(1.f, e);
      const float ts = fadd(__ldg(t + i), 1e-2f);
      const float T = expf(-d_logit[size_t(i) * dlogit_stride]);
      w = T * alpha;
      r = __ldg(rgb + size_t(i) * 3); g = __ldg(rgb + size_t(i) * 3 + 1); b = __ldg(rgb + size_t(i) * 3 + 2);
      const float gw = (d_weights ? d_weights[i] : 0.f) + dcr * r + dcg * g + dcb * b + ddisp / ts + ddep * ts;
      dA = -gw * w;                // through T_i = exp(-A_i)
      direct = gw * T * e;         // through alpha_i = 1 - exp(-tau_i)
    }
    // reverse inclusive scan of dA within the chunk, then make it exclusive (k > i only)
    float s = dA;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float v = __shfl_down_sync(kFull, s, o);
      if (lane + o < 32) s += v;
    }
    const float suffix = (s - dA) + carry;
    carry += __shfl_sync(kFull, s, 0);
    if (valid) {
      float scale = 1.f;
      if (scaling) {
        const float a = (float(i - beg) + .5f) / float(n);
        scale = gs_progress + (1.f - gs_progress) * a * a;
      }
      const float dtau = direct + suffix + dS;
      const float ddens = dtau * dtv * scale;
      // TruncExp backward: g * exp(clamp(x, -100, 5))   (CustomOps.cpp:16-18)
      d_logit[size_t(i) * dlogit_stride] = ddens * expf(fminf(fmaxf(x, -100.f), 5.f));
      const float gr = w * dcr * scale, gg = w * dcg * scale, gb = w * dcb * scale;
      if (FUSE_ACT) {
        const uint2 rw = __ldg(reinterpret_cast<const uint2*>(raw + size_t(i) * 16));
        const float2 o01 = __half22float2(*reinterpret_cast<const __half2*>(&rw.x));
        const float2 o2x = __half22float2(*reinterpret_cast<const __half2*>(&rw.y));
        const __half2 h0 = __floats2half2_rn(shade_act_bwd(o01.x, gr, act_loss_scale), shade_act_bwd(o01.y, gg, act_loss_scale));
        const __half2 h1 = __floats2half2_rn(shade_act_bwd(o2x.x, gb, act_loss_scale), 0.f);
        uint4 v0 = make_uint4(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1), 0u, 0u);
        uint4* dst = reinterpret_cast<uint4*>(d_raw + size_t(i) * 16);
        dst[0] = v0;
        dst[1] = make_uint4(0u, 0u, 0u, 0u);
      } else {
        d_rgb[size_t(i) * 3 + 0] = gr;
        d_rgb[size_t(i) * 3 + 1] = gg;
        d_rgb[size_t(i) * 3 + 2] = gb;
      }
    }
  }
}

// ---- stand-alone FlexOps (serial order, FlexOps.cu:5-73) ------------------------------------------
__global__ void __launch_bounds__(256)
flex_sum_kernel(const float* __restrict__ val, int vec, const int* __restrict__ bounds, int n_outs,
                float* __restrict__ sum) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_outs) return;
  const int beg = bounds[2 * ray], end = bounds[2 * ray + 1];
  for (int j = 0; j < vec; j++) {
    float run = 0.f;
    for (int base = beg; base < end; base += 32) {
      const int i = base + lane;
      const float v = i < end ? __ldg(val + size_t(i) * vec + j) : 0.f;
      chain_sum(v, run, min(32, end - base));
    }
    if (lane == 0) sum[size_t(ray) * vec + j] = run;
  }
}

__global__ void __launch_bounds__(256)
flex_accumulate_kernel(const float* __restrict__ val, const int* __restrict__ bounds, int n_outs,
                       int include_this, float* __restrict__ out) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_outs) return;
  const int beg = bounds[2 * ray], end = bounds[2 * ray + 1];
  float run = 0.f;
  for (int base = beg; base < end; base += 32) {
    const int i = base + lane;
    const float v = i < end ? __ldg(val + i) : 0.f;
    const float ex = chain_excl(v, run, min(32, end - base), lane);
    if (i < end) out[i] = include_this ? fadd(ex, v) : ex;
  }
}

// ---- WeightVar loss (CustomOps.cu:12-66): variance of the sample index/16 under the weights ------
__global__ void __launch_bounds__(256)
weight_var_fwd_kernel(const float* __restrict__ w, const int* __restrict__ bounds, int n_outs,
                      float* __restrict__ out_vars) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_outs) return;
  const int beg = bounds[2 * ray], end = bounds[2 * ray + 1];
  if (beg >= end) { if (lane == 0) out_vars[ray] = 0.f; return; }
  float m = 0.f, ws = 0.f;
  for (int i = beg + lane; i < end; i += 32) { const float wi = w[i]; m += wi * (float(i - beg) / 16.f); ws += wi; }
  m = warp_sum(m); ws = warp_sum(ws) + 1e-6f;
  const float mean = m / ws;
  float var = 0.f;
  for (int i = beg + lane; i < end; i += 32) { const float bias = float(i - beg) / 16.f - mean; var += w[i] * bias * bias; }
  var = warp_sum(var);
  if (lane == 0) out_vars[ray] = var;
}

__global__ void __launch_bounds__(256)
weight_var_bwd_kernel(const float* __restrict__ w, const int* __restrict__ bounds, int n_outs,
                      const float* __restrict__ dl_dvars, float* __restrict__ dl_dw) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_outs) return;
  const int beg = bounds[2 * ray], end = bounds[2 * ray + 1];
  if (beg >= end) return;
  float m = 0.f, ws = 0.f;
  for (int i = beg + lane; i < end; i += 32) { const float wi = w[i]; m += wi * (float(i - beg) / 16.f); ws += wi; }
  m = warp_sum(m); ws = warp_sum(ws) + 1e-6f;
  const float mean = m / ws;
  float tmp = 0.f;
  for (int i = beg + lane; i < end; i += 32) { const float bias = float(i - beg) / 16.f - mean; tmp += w[i] * 2.f * bias; }
  tmp = warp_sum(tmp);
  const float g = dl_dvars[ray];
  for (int i = beg + lane; i < end; i += 32) {
    const float x = float(i - beg) / 16.f;
    const float bias = x - mean;
    dl_dw[i] = g * (bias * bias + tmp * -x / ws);
  }
}

}  // namespace f2b

using namespace f2b;

static inline int warp_grid(int n_rays) { return div_up(int64_t(n_rays) * 32, 256); }

extern "C" int f2b_early_stop(const float* logit, int logit_stride, const float* dt, const int* pts_idx_bounds,
                              int n_rays, float* weights, float* alphas, uint8_t* keep, int* ray_counts,
                              int* new_bounds, int* total_kept, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(logit && dt && pts_idx_bounds && weights && alphas && keep && ray_counts && new_bounds && total_kept,
              "f2b_early_stop: null pointer");
  cudaStream_t st = as_stream(stream);
  early_stop_kernel<<<warp_grid(n_rays), 256, 0, st>>>(logit, logit_stride, dt, pts_idx_bounds, n_rays, weights,
                                                      alphas, keep, ray_counts);
  scan_counts_kernel<<<1, 1024, 0, st>>>(ray_counts, n_rays, new_bounds, total_kept);
  return check_launch("f2b_early_stop");
}

extern "C" int f2b_early_stop_rays(const float* logit, int logit_stride, const float* dt, const int* pts_idx_bounds,
                                   int n_rays, float* weights, float* alphas, uint8_t* keep, int* ray_counts, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(logit && dt && pts_idx_bounds && weights && alphas && keep && ray_counts, "f2b_early_stop_rays: null pointer");
  early_stop_kernel<<<warp_grid(n_rays), 256, 0, as_stream(stream)>>>(logit, logit_stride, dt, pts_idx_bounds, n_rays,
                                                                     weights, alphas, keep, ray_counts);
  return check_launch("f2b_early_stop_rays");
}

extern "C" int f2b_count_scan(const int* counts, int n, int* bounds, int* total, void* stream) {
  F2B_REQUIRE(bounds && total && (counts || n <= 0), "f2b_count_scan: null pointer");
  scan_counts_kernel<<<1, 1024, 0, as_stream(stream)>>>(counts, n > 0 ? n : 0, bounds, total);
  return check_launch("f2b_count_scan");
}

extern "C" int f2b_slot_bounds(const int* ray_counts, int n_rays, int slot_size, int first_ray, int* slot_bounds, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(ray_counts && slot_bounds && slot_size > 0, "f2b_slot_bounds: bad argument");
  slot_bounds_kernel<<<div_up(n_rays, 256), 256, 0, as_stream(stream)>>>(ray_counts, n_rays, slot_size, first_ray, slot_bounds);
  return check_launch("f2b_slot_bounds");
}

extern "C" int f2b_compact_slots(const uint8_t* keep, const int* slot_bounds, const int* new_bounds, int n_rays,
                                 const float* rays_d, const float* s_pts, const float* s_dt, const float* s_t,
                                 const int* s_anchors, const void* feat_slots_f16, float* pts_o, float* dirs_o,
                                 float* dt_o, float* t_o, int* anchors_o, void* feat_o_f16, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(keep && slot_bounds && new_bounds && rays_d && s_pts && s_dt && s_t && s_anchors && pts_o && dirs_o && dt_o &&
                  t_o && anchors_o, "f2b_compact_slots: null pointer");
  F2B_REQUIRE(!feat_slots_f16 || feat_o_f16, "f2b_compact_slots: feat_slots_f16 without feat_o_f16");
  compact_slots_kernel<<<warp_grid(n_rays), 256, 0, as_stream(stream)>>>(
      keep, slot_bounds, new_bounds, n_rays, rays_d, s_pts, s_dt, s_t, s_anchors, (const uint4*)feat_slots_f16, pts_o, dirs_o,
      dt_o, t_o, anchors_o, (uint4*)feat_o_f16);
  return check_launch("f2b_compact_slots");
}

extern "C" int f2b_compact_samples(const uint8_t* keep, const int* old_bounds, const int* new_bounds, int n_rays,
                                   const float* pts, const float* dirs, const float* dt, const float* t,
                                   const int* anchors, const void* feat_f16, float* pts_o, float* dirs_o,
                                   float* dt_o, float* t_o, int* anchors_o, void* feat_o_f16, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(!feat_f16 || feat_o_f16, "f2b_compact_samples: feat_f16 without feat_o_f16");
  compact_kernel<<<warp_grid(n_rays), 256, 0, as_stream(stream)>>>(keep, old_bounds, new_bounds, n_rays, pts, dirs, dt, t,
                                                                  anchors, (const uint4*)feat_f16, pts_o, dirs_o, dt_o,
                                                                  t_o, anchors_o, (uint4*)feat_o_f16);
  return check_launch("f2b_compact_samples");
}

extern "C" int f2b_composite_fwd(const float* logit, int logit_stride, const float* rgb, const float* dt,
                                 const float* t, const int* pts_idx_bounds, const float* bg_color, int n_rays,
                                 float* colors, float* disparity, float* depth, float* weights, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(logit && rgb && dt && t && pts_idx_bounds && bg_color && colors && disparity && depth && weights,
              "f2b_composite_fwd: null pointer");
  composite_fwd_kernel<<<warp_grid(n_rays), 256, 0, as_stream(stream)>>>(logit, logit_stride, rgb, dt, t, pts_idx_bounds,
                                                                        bg_color, n_rays, colors, disparity, depth, weights);
  return check_launch("f2b_composite_fwd");
}

extern "C" int f2b_composite_bwd(const float* logit, int logit_stride, const float* rgb, const float* dt,
                                 const float* t, const int* pts_idx_bounds, const float* bg_color, int n_rays,
                                 const float* d_colors, const float* d_disparity, const float* d_depth,
                                 const float* d_weights, float grad_scaling_progress, float* d_logit,
                                 int dlogit_stride, float* d_rgb, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(logit && rgb && dt && t && pts_idx_bounds && bg_color && d_colors && d_logit && d_rgb,
              "f2b_composite_bwd: null pointer");
  composite_bwd_kernel<false><<<warp_grid(n_rays), 256, 0, as_stream(stream)>>>(
      logit, logit_stride, rgb, dt, t, pts_idx_bounds, bg_color, n_rays, d_colors, d_disparity, d_depth, d_weights,
      grad_scaling_progress, d_logit, dlogit_stride, d_rgb, nullptr, nullptr, 0.f);
  return check_launch("f2b_composite_bwd");
}

extern "C" int f2b_composite_act_bwd(const float* logit, int logit_stride, const float* rgb, const float* dt,
                                     const float* t, const int* pts_idx_bounds, const float* bg_color, int n_rays,
                                     const float* d_colors, const float* d_disparity, const float* d_depth,
                                     const float* d_weights, float grad_scaling_progress, const void* raw_f16,
                                     float loss_scale, float* d_logit, int dlogit_stride, void* d_raw_f16, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(logit && rgb && dt && t && pts_idx_bounds && bg_color && d_colors && d_logit && raw_f16 && d_raw_f16,
              "f2b_composite_act_bwd: null pointer");
  composite_bwd_kernel<true><<<warp_grid(n_rays), 256, 0, as_stream(stream)>>>(
      logit, logit_stride, rgb, dt, t, pts_idx_bounds, bg_color, n_rays, d_colors, d_disparity, d_depth, d_weights,
      grad_scaling_progress, d_logit, dlogit_stride, nullptr, (const __half*)raw_f16, (__half*)d_raw_f16, loss_scale);
  return check_launch("f2b_composite_act_bwd");
}

extern "C" int f2b_flex_sum(const float* val, int vec, const int* idx_start_end, int n_outs, float* sum, void* stream) {
  if (n_outs <= 0) return F2B_OK;
  flex_sum_kernel<<<warp_grid(n_outs), 256, 0, as_stream(stream)>>>(val, vec, idx_start_end, n_outs, sum);
  return check_launch("f2b_flex_sum");
}
extern "C" int f2b_flex_accumulate_sum(const float* val, const int* idx_start_end, int n_outs, int include_this,
                                       float* out, void* stream) {
  if (n_outs <= 0) return F2B_OK;
  flex_accumulate_kernel<<<warp_grid(n_outs), 256, 0, as_stream(stream)>>>(val, idx_start_end, n_outs, include_this, out);
  return check_launch("f2b_flex_accumulate_sum");
}
extern "C" int f2b_weight_var_fwd(const float* weights, const int* idx_start_end, int n_outs, float* out_vars, void* stream) {
  if (n_outs <= 0) return F2B_OK;
  weight_var_fwd_kernel<<<warp_grid(n_outs), 256, 0, as_stream(stream)>>>(weights, idx_start_end, n_outs, out_vars);
  return check_launch("f2b_weight_var_fwd");
}
extern "C" int f2b_weight_var_bwd(const float* weights, const int* idx_start_end, int n_outs, const float* dl_dvars,
                                  float* dl_dw, void* stream) {
  if (n_outs <= 0) return F2B_OK;
  weight_var_bwd_kernel<<<warp_grid(n_outs), 256, 0, as_stream(stream)>>>(weights, idx_start_end, n_outs, dl_dvars, dl_dw);
  return check_launch("f2b_weight_var_bwd");
}
