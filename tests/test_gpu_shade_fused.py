"""f2b_shade_field_bwd_scatter: the ray samples' shader-MLP backward, input-assembly backward, field-MLP backward and hash scatter
in one kernel, against the three kernels it replaces (f2b_mlp_bwd2 with rebuilt activations, f2b_shader_prep_bwd_f16,
f2b_field_bwd_scatter) and against the CPU oracle's scatter."""
import numpy as np
import pytest
import torch

from test_gpu_bwd_fused import segment
from test_gpu_parity import N, T, assert_close

pytestmark = pytest.mark.gpu


def rays_of(n, rng):
    """[R,2] sample bounds of rays of 1..60 samples covering [0, n)."""
    ends = np.minimum(np.cumsum(rng.integers(1, 61, n)), n)
    ends = ends[: int(np.searchsorted(ends, n)) + 1]
    return np.ascontiguousarray(np.stack([np.concatenate([[0], ends[:-1]]), ends], 1).astype(np.int32))


@pytest.mark.parametrize("emb", [False, True])
@pytest.mark.parametrize("n", [1, 31, 32, 127, 128, 129, 5000, 2 * 132 * 128 + 51])   # the last: CTAs with two and three tiles
def test_shade_field_bwd_scatter_matches_unfused(scene, oracle, hash_params, n, emb):
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    hp = hash_params
    pts, vol, stride = segment(scene, oracle, hp, "rays", n)
    rng = np.random.default_rng(2000 + n)
    sparams = T((oracle.mlp_init(32, 1) * 2).astype(np.float16))
    fparams = T((oracle.mlp_init(32, 0) * 2).astype(np.float16))
    mlp_in = T((rng.standard_normal((n, 32)) * 0.5).astype(np.float16))
    feat = T((rng.standard_normal((n, 32)) * 0.5).astype(np.float16))
    d_raw = (rng.standard_normal((n, 16)) * 0.1).astype(np.float16)
    d_raw[1::5] = 0                                                 # all-zero shader dL/dout rows
    d_logit = (rng.standard_normal(n) * 0.05).astype(np.float32)
    d_logit[1::10] = 0                                              # ... some with a zero d_logit too: all-zero field rows
    d_raw, d_logit = T(d_raw), T(d_logit)
    s_scale, f_scale, grad_mul = 128.0, 64.0, 1.0 / 64.0
    bounds = T(rays_of(n, rng))
    n_rays, n_emb = bounds.shape[0], 7
    ray_emb = T(rng.integers(0, n_emb, n_rays).astype(np.int32)) if emb else None
    pt_emb = ops.scatter_idx(n, bounds, ray_emb) if emb else None
    prim, bias, S = T(hp["prim"]), T(hp["bias"]), hp["local_size"]
    hash_args = (prim, bias, hp["V"], S)
    zf = lambda *s: torch.zeros(s, dtype=torch.float32, device="cuda")
    nan16 = lambda *s: torch.full(s, float("nan"), dtype=torch.float16, device="cuda")

    # the three kernels the fused one replaces
    din_ref, scene_ref, dfeat_ref = nan16(n, 32), nan16(n, 16), nan16(n, 32)
    dsp_ref, dfp_ref, table_ref = zf(sparams.numel()), zf(fparams.numel()), zf(hp["pool"], 2)
    app_ref = zf(n_emb, 16) if emb else None
    call("f2b_mlp_bwd2", d_raw, mlp_in, None, None, sparams, 1, n, din_ref, dsp_ref, stream())
    ops.shader_prep_bwd_f16(din_ref, d_logit, bounds, ray_emb, 1.0 / s_scale, f_scale, scene_ref, app_ref)
    call("f2b_field_bwd_scatter", scene_ref, feat, fparams, n, T(pts), T(vol), stride, *hash_args, grad_mul, dfp_ref, table_ref,
         dfeat_ref, stream())
    scales = ops.hash_level_scales().numpy()
    exact = oracle.hash_bwd(hp["prim"], hp["bias"], hp["V"], S, scales, pts, vol, stride, N(dfeat_ref).astype(np.float32), grad_mul,
                            hp["pool"])
    ticket = torch.empty((1,), dtype=torch.int32, device="cuda")
    for debug_rows in (True, False):
        din, scene16, dfeat = (nan16(n, 32), nan16(n, 16), nan16(n, 32)) if debug_rows else (None, None, None)
        dsp, dfp, table = zf(sparams.numel()), zf(fparams.numel()), zf(hp["pool"], 2)
        app = zf(n_emb, 16) if emb else None
        call("f2b_shade_field_bwd_scatter", d_raw, mlp_in, sparams, d_logit, pt_emb, 1.0 / s_scale, f_scale, feat, fparams, n, T(pts),
             T(vol), stride, *hash_args, grad_mul, dsp, dfp, table, app, ticket, din, scene16, dfeat, stream())
        tag = f"n={n} emb={emb}"
        if debug_rows:
            for got, ref in ((din, din_ref), (scene16, scene_ref), (dfeat, dfeat_ref)):
                np.testing.assert_array_equal(N(got).view(np.uint16), N(ref).view(np.uint16))
        assert_close(N(dsp), N(dsp_ref), rtol=1e-5, atol_frac=1e-6, name=f"shader dparams {tag}")
        assert_close(N(dfp), N(dfp_ref), rtol=1e-5, atol_frac=1e-6, name=f"field dparams {tag}")
        assert_close(N(table), exact, rtol=1e-4, atol_frac=1e-5, name=f"table vs oracle {tag}")
        np.testing.assert_allclose(N(table), N(table_ref), rtol=1e-5, atol=1e-6 * max(float(table_ref.abs().max()), 1e-30))
        assert float(table[(17 * S) // 2 + 1:].abs().max()) == 0.0
        if emb:
            assert float(app_ref.abs().max()) > 0
            assert_close(N(app), N(app_ref), rtol=1e-5, atol_frac=1e-6, name=f"d_app {tag}")
