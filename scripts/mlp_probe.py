"""Probe: how much of the tensor-core MLP kernels' time is HBM traffic for the saved activations?  Times f2b_mlp_fwd with and
without hidden_save, f2b_field_shade_fwd / f2b_shader_mlp_rgb_fwd, and f2b_mlp_bwd2, on N samples (default 3.1 M = the headline's
kept samples).  If the no-save forward is several times faster, recomputing the hidden layers in the backward (instead of
saving 384 B/sample) pays.  Output: one JSON line."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from f2nerf_b200 import ops  # noqa: E402
from f2nerf_b200._lib import call, stream  # noqa: E402


def timed(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 3_100_000
    dev = "cuda"
    g = torch.Generator(dev).manual_seed(0)
    x = (torch.randn((n, 32), device=dev, generator=g) * .5).half()
    out = {"n": n}
    for nh in (0, 1):
        p = (torch.randn((64 * 32 + nh * 64 * 64 + 16 * 64,), device=dev, generator=g) * .2).half()
        o16 = torch.empty((n, 16), dtype=torch.float16, device=dev)
        hid = torch.empty((nh + 1, n, 64), dtype=torch.float16, device=dev)
        out[f"fwd_nh{nh}_save_ms"] = timed(lambda: call("f2b_mlp_fwd", x, p, nh, n, o16, hid, stream()))
        out[f"fwd_nh{nh}_nosave_ms"] = timed(lambda: call("f2b_mlp_fwd", x, p, nh, n, o16, None, stream()))
        dout = (torch.randn((n, 16), device=dev, generator=g) * .1).half()
        din = torch.empty((n, 32), dtype=torch.float16, device=dev)
        dp = torch.zeros(p.numel(), device=dev)
        out[f"bwd_nh{nh}_ms"] = timed(lambda: call("f2b_mlp_bwd2", dout, x, hid[0], hid[nh] if nh else None, p, nh, n, din, dp, stream()))
        out[f"bwd_nh{nh}_recompute_ms"] = timed(lambda: call("f2b_mlp_bwd2", dout, x, None, None, p, nh, n, din, dp, stream()))
        out[f"bwd_nh{nh}_recompute_GBs"] = n * (32 + 64 + 64) / out[f"bwd_nh{nh}_recompute_ms"] / 1e6
        bytes_fwd_save = n * (64 + 32 + 128 * (nh + 1))
        out[f"fwd_nh{nh}_save_GBs"] = bytes_fwd_save / out[f"fwd_nh{nh}_save_ms"] / 1e6
        out[f"fwd_nh{nh}_nosave_GBs"] = n * 96 / out[f"fwd_nh{nh}_nosave_ms"] / 1e6
        out[f"bwd_nh{nh}_GBs"] = n * (32 + 64 + 128 * (nh + 1) + 64) / out[f"bwd_nh{nh}_ms"] / 1e6
    # plain HBM copy of the same size as the shader MLP's saved activations, for scale
    a = torch.empty((n, 128), dtype=torch.float16, device=dev); b = torch.empty_like(a)
    out["copy_256B_per_sample_ms"] = timed(lambda: b.copy_(a))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
