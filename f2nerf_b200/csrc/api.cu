// api.cu — implementation selection for the MLP entry points of the C ABI.
// impl 0 = CUDA-core twin (mlp.cu), impl 1 = wgmma tensor-core kernels (mlp_tc.cu).  The default is the
// tensor-core path; F2B_MLP_IMPL=0 in the environment (or f2b_set_mlp_impl) selects the twin.
#include "common.cuh"
#include <stdlib.h>

#ifndef F2B_TC_BWD_DEFAULT
#define F2B_TC_BWD_DEFAULT 1   // mlp_tc_bwd.cu validated on H100 (tests/test_gpu_parity.py::test_mlp_fwd_bwd[tc-*])
#endif

extern "C" int f2b_mlp_fwd_v0(const void*, const void*, int, int, void*, void*, void*);
extern "C" int f2b_mlp_bwd_v0(const void*, const void*, const void*, const void*, int, int, void*, float*, void*);
extern "C" int f2b_mlp_bwd2_v0(const void*, const void*, const void*, const void*, const void*, int, int, void*, float*, void*);
#ifdef F2B_HAVE_TC
extern "C" int f2b_mlp_fwd_tc(const void*, const void*, int, int, void*, void*, void*);
extern "C" int f2b_mlp_bwd_tc(const void*, const void*, const void*, const void*, int, int, void*, float*, void*);
extern "C" int f2b_mlp_bwd2_tc(const void*, const void*, const void*, const void*, const void*, int, int, void*, float*, void*);
extern "C" int f2b_mlp_fwd_tc_f32(const void*, const void*, int, int, float*, void*, void*, void*);
#endif
extern "C" int f2b_cast_f16_to_f32(const void* src, float* dst, int64_t n, float scale, void* stream);

static int g_mlp_bwd_impl = -1;
static int mlp_bwd_impl() {          // backward implementation follows F2B_MLP_BWD_IMPL, else the forward choice
  if (g_mlp_bwd_impl < 0) {
    const char* e = getenv("F2B_MLP_BWD_IMPL");
#ifdef F2B_HAVE_TC
    g_mlp_bwd_impl = e ? atoi(e) : F2B_TC_BWD_DEFAULT;
#else
    g_mlp_bwd_impl = 0;
    (void)e;
#endif
  }
  return g_mlp_bwd_impl;
}

static int g_mlp_impl = -1;
static int mlp_impl() {
  if (g_mlp_impl < 0) {
    const char* e = getenv("F2B_MLP_IMPL");
#ifdef F2B_HAVE_TC
    g_mlp_impl = e ? atoi(e) : 1;
#else
    g_mlp_impl = 0;
    (void)e;
#endif
  }
  return g_mlp_impl;
}

extern "C" int f2b_set_mlp_impl(int impl) {
#ifndef F2B_HAVE_TC
  if (impl != 0) { f2b::set_error("f2b_set_mlp_impl: tensor-core path not built"); return F2B_EUNSUPPORTED; }
#endif
  g_mlp_impl = impl;
  g_mlp_bwd_impl = impl ? F2B_TC_BWD_DEFAULT : 0;
  return F2B_OK;
}
extern "C" int f2b_get_mlp_impl(void) { return mlp_impl(); }

extern "C" int f2b_mlp_fwd(const void* in_f16, const void* params_f16, int n_hidden_matmuls, int n_pts,
                           void* out_f16, void* hidden_save_f16, void* stream) {
#ifdef F2B_HAVE_TC
  if (mlp_impl() == 1) return f2b_mlp_fwd_tc(in_f16, params_f16, n_hidden_matmuls, n_pts, out_f16, hidden_save_f16, stream);
#endif
  return f2b_mlp_fwd_v0(in_f16, params_f16, n_hidden_matmuls, n_pts, out_f16, hidden_save_f16, stream);
}
extern "C" int f2b_mlp_fwd_f32(const void* in_f16, const void* params_f16, int n_hidden_matmuls, int n_pts,
                               float* out_f32, void* out_f16, void* hidden_save_f16, void* stream) {
#ifdef F2B_HAVE_TC
  if (mlp_impl() == 1) return f2b_mlp_fwd_tc_f32(in_f16, params_f16, n_hidden_matmuls, n_pts, out_f32, out_f16, hidden_save_f16, stream);
#endif
  if (!out_f16) { f2b::set_error("f2b_mlp_fwd_f32: the CUDA-core twin needs the fp16 output buffer as well"); return F2B_EINVAL; }
  const int rc = f2b_mlp_fwd_v0(in_f16, params_f16, n_hidden_matmuls, n_pts, out_f16, hidden_save_f16, stream);
  if (rc != F2B_OK || !out_f32) return rc;
  return f2b_cast_f16_to_f32(out_f16, out_f32, int64_t(n_pts) * 16, 1.f, stream);
}
extern "C" int f2b_mlp_bwd(const void* dout_f16, const void* in_f16, const void* hidden_save_f16,
                           const void* params_f16, int n_hidden_matmuls, int n_pts, void* din_f16,
                           float* dparams_f32, void* stream) {
#ifdef F2B_HAVE_TC
  if (mlp_bwd_impl() == 1) return f2b_mlp_bwd_tc(dout_f16, in_f16, hidden_save_f16, params_f16, n_hidden_matmuls, n_pts, din_f16, dparams_f32, stream);
#endif
  return f2b_mlp_bwd_v0(dout_f16, in_f16, hidden_save_f16, params_f16, n_hidden_matmuls, n_pts, din_f16, dparams_f32, stream);
}

// Backward with the per-layer activation blocks passed separately (row ranges of a larger saved batch:
// ray-chunked backward passes on separate streams).  dparams is ACCUMULATED into (caller zeroes once).
extern "C" int f2b_mlp_bwd2(const void* dout_f16, const void* in_f16, const void* hidden0_f16, const void* hidden1_f16,
                            const void* params_f16, int n_hidden_matmuls, int n_pts, void* din_f16,
                            float* dparams_f32, void* stream) {
#ifdef F2B_HAVE_TC
  if (mlp_bwd_impl() == 1) return f2b_mlp_bwd2_tc(dout_f16, in_f16, hidden0_f16, hidden1_f16, params_f16, n_hidden_matmuls, n_pts, din_f16, dparams_f32, stream);
#endif
  if (!hidden0_f16 && n_pts > 0) { f2b::set_error("f2b_mlp_bwd2: recompute (hidden0 == NULL) needs the tensor-core implementation"); return F2B_EUNSUPPORTED; }
  return f2b_mlp_bwd2_v0(dout_f16, in_f16, hidden0_f16, hidden1_f16, params_f16, n_hidden_matmuls, n_pts, din_f16, dparams_f32, stream);
}
