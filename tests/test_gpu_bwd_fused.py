"""f2b_field_bwd_scatter: the field-MLP backward with the hash-grid scatter fused behind it, against the two kernels it replaces
(f2b_mlp_bwd2 with rebuilt activations, then f2b_hash_bwd on its fp16 dL/dfeat rows) and against the CPU oracle's scatter."""
import numpy as np
import pytest
import torch

from test_gpu_bwd_reference import ray_layout
from test_gpu_parity import N, T, assert_close, sample_points

pytestmark = pytest.mark.gpu


def segment(scene, oracle, hp, kind, n):
    """(pts [n,3], volume ids, stride): ray samples (consecutive samples share coarse cells: merged runs) with anchors [n,3]
    (stride 3), or edge-like point pairs with a flat volume id (stride 1).  Beyond the oracle-sampled rays' samples, synthetic rays."""
    if kind == "rays":
        s = sample_points(scene, oracle)
        if s["pts"].shape[0] < n:
            pts, anchors, _ = ray_layout(n, hp["V"], np.random.default_rng(n))
            return pts, anchors, 3
        return np.ascontiguousarray(s["pts"][:n]), np.ascontiguousarray(s["anchors"][:n]), 3
    rng = np.random.default_rng(n)
    a = rng.random((n // 2 + 1, 3), dtype=np.float32) * 2 - 1
    b = np.clip(a + rng.standard_normal(a.shape).astype(np.float32) * 1e-3, -1, 1).astype(np.float32)
    pts = np.stack([a, b], 1).reshape(-1, 3)[:n]
    vol = np.repeat(rng.integers(0, hp["V"], n // 2 + 1).astype(np.int32), 2)[:n]
    return np.ascontiguousarray(pts), np.ascontiguousarray(vol), 1


@pytest.mark.parametrize("kind,n", [("rays", 1), ("rays", 31), ("rays", 32), ("rays", 127), ("rays", 128), ("rays", 129),
                                    ("rays", 5000), ("rays", 12 * 132 * 128 + 51), ("edges", 4099)])   # 12*132*128+51: 4-5 tiles per CTA
def test_field_bwd_scatter_matches_unfused(scene, oracle, hash_params, kind, n):
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    hp = hash_params
    pts, vol, stride = segment(scene, oracle, hp, kind, n)
    rng = np.random.default_rng(1000 + n)
    params = T((oracle.mlp_init(32, 0) * 2).astype(np.float16))
    x = T((rng.standard_normal((n, 32)) * 0.5).astype(np.float16))
    dout = (rng.standard_normal((n, 16)) * 0.1).astype(np.float16)
    dout[::5] = 0                                                   # all-zero gradient rows: no reductions
    dout[3::11] = 0
    dout = T(dout)
    prim, bias, S, grad_mul = T(hp["prim"]), T(hp["bias"]), hp["local_size"], 0.5
    # the two kernels the fused one replaces
    din_ref = torch.empty((n, 32), dtype=torch.float16, device="cuda")
    dp_ref = torch.zeros(params.numel(), dtype=torch.float32, device="cuda")
    call("f2b_mlp_bwd2", dout, x, None, None, params, 0, n, din_ref, dp_ref, stream())
    table_ref = torch.zeros((hp["pool"], 2), dtype=torch.float32, device="cuda")
    ops.hash_bwd(prim, bias, hp["V"], S, T(pts), T(vol), stride, din_ref, grad_mul, table_ref)
    scales = ops.hash_level_scales().numpy()
    exact = oracle.hash_bwd(hp["prim"], hp["bias"], hp["V"], S, scales, pts, vol, stride, N(din_ref).astype(np.float32), grad_mul,
                            hp["pool"])
    for with_din in (True, False):
        din = torch.full((n, 32), float("nan"), dtype=torch.float16, device="cuda") if with_din else None
        dp = torch.zeros(params.numel(), dtype=torch.float32, device="cuda")
        table = torch.zeros((hp["pool"], 2), dtype=torch.float32, device="cuda")
        call("f2b_field_bwd_scatter", dout, x, params, n, T(pts), T(vol), stride, prim, bias, hp["V"], S, grad_mul, dp, table, din,
             stream())
        if with_din:
            np.testing.assert_array_equal(N(din).view(np.uint16), N(din_ref).view(np.uint16))
        assert_close(N(dp), N(dp_ref), rtol=1e-5, atol_frac=1e-6, name=f"dparams {kind} n={n}")
        assert_close(N(table), exact, rtol=1e-4, atol_frac=1e-5, name=f"table vs oracle {kind} n={n}")
        # the same reductions as f2b_hash_bwd: they differ only in the order they reach L2
        np.testing.assert_allclose(N(table), N(table_ref), rtol=1e-5, atol=1e-6 * max(float(table_ref.abs().max()), 1e-30))
        assert float(table[(17 * S) // 2 + 1:].abs().max()) == 0.0

