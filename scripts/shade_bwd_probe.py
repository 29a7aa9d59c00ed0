#!/usr/bin/env python
"""shade_bwd_probe.py — the ray samples' per-sample backward on the headline batch (wanjinyou, 4096 rays): the three kernels in
sequence against f2b_shade_field_bwd_scatter, which runs them as one warp-specialised kernel under the hash scatter.

  python scripts/shade_bwd_probe.py [--out profiles/h100_shade_bwd_probe.json] [--red-rate profiles/h100_red_rate.json] [--iters 60]

Runs the forward of one TRAIN step through Renderer.Render (bwd_probe.capture_step) and keeps the inputs of
f2b_shade_field_bwd_scatter (shader dL/dout, shader input rows, d_logit, field input rows, both MLPs' fp16 parameters, points /
anchors, camera indices) and of the step's f2b_sampler_march (the batch marched once more through PersSampler.march_rays).
Then times, with CUDA events (median of --iters launches after warm-up, gradients zeroed before each):
  sequence  f2b_mlp_bwd2 (shader, recompute) -> f2b_shader_prep_bwd_f16 -> f2b_field_bwd_scatter, as the parent issued them;
  fused     f2b_shade_field_bwd_scatter alone;
  +march    the fused kernel with the march of a ray batch launched just before it on a second stream (as in training, where
            the next batch's march is pipelined behind the backward); the events bracket the fused kernel on its own stream.
The lane reductions of the scatter are counted on the host (bwd_probe.count_reductions) and set against the microbenchmark's
v2f32 `spread` peak.  The field's dL/dout rows of the fused kernel are also compared bit for bit with the sequence's."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_shade_bwd_probe.json"))
    ap.add_argument("--red-rate", default=os.path.join(ROOT, "profiles", "h100_red_rate.json"))
    ap.add_argument("--iters", type=int, default=60)
    args = ap.parse_args()
    import torch
    import bench
    from bwd_probe import capture_step, count_reductions, gpu_info
    from f2nerf_b200 import ops, sampler as SM
    from f2nerf_b200._lib import call, stream

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bargs = argparse.Namespace(config="wanjinyou", rays=0)
    prob = bench.build_problem(0, 1, bargs, dev)
    o, d, cam, gt = prob["host"]
    rays_o, rays_d, emb, gt = (torch.from_numpy(a).to(dev) for a in (o, d, cam, gt))
    c = capture_step(prob, rays_o, rays_d, emb, gt)
    d_raw, mlp_in, sp16, d_logit, pt_emb, inv_s, f_scale, feat, fp16_, n, pts, anc, grad_mul, d_sp, d_fp, d_table, d_app, bounds = (
        c[k] for k in ("d_raw", "mlp_in", "sp16", "d_logit", "pt_emb", "inv_s", "f_scale", "feat", "fp16", "n", "pts", "anc",
                       "grad_mul", "d_sp", "d_fp", "d_table", "d_app", "bounds"))
    stride = 3
    ticket = torch.empty((1,), dtype=torch.int32, device=dev)
    n_rays = bounds.shape[0]
    kept = {}
    real_s = SM.call

    def spy(name, *a):
        if name == "f2b_sampler_march":
            kept[name] = [t.clone() if isinstance(t, torch.Tensor) else t for t in a]
        return real_s(name, *a)

    SM.call = spy
    try:
        prob["renderer"].pts_sampler_.march_rays(c["slots"])
    finally:
        SM.call = real_s
    ray_emb = emb.to(torch.int32).contiguous() if pt_emb is not None else None
    f16 = lambda *s: torch.empty(s, dtype=torch.float16, device=dev)
    d_in16, d_scene16, dfeat16 = f16(n, 32), f16(n, 16), f16(n, 32)
    sp, fp, table = torch.zeros_like(d_sp), torch.zeros_like(d_fp), torch.zeros_like(d_table)
    app = torch.zeros_like(d_app) if d_app is not None else None
    hash_args = c["hash_args"]
    prim, bias, n_vol, S = hash_args

    def seq():
        call("f2b_mlp_bwd2", d_raw, mlp_in, None, None, sp16, 1, n, d_in16, sp, stream())
        call("f2b_shader_prep_bwd_f16", d_in16, d_logit, bounds, ray_emb, n_rays, float(inv_s), float(f_scale), d_scene16, app, stream())
        call("f2b_field_bwd_scatter", d_scene16, feat, fp16_, n, pts, anc, stride, *hash_args, grad_mul, fp, table, None, stream())

    def fused(d_scene_out=None, dfeat_out=None):
        call("f2b_shade_field_bwd_scatter", d_raw, mlp_in, sp16, d_logit, pt_emb, inv_s, f_scale, feat, fp16_, n, pts, anc, stride,
             *hash_args, grad_mul, sp, fp, table, app, ticket, None, d_scene_out, dfeat_out, stream())

    march_args = kept["f2b_sampler_march"]
    side = torch.cuda.Stream(dev)

    def fused_after_march():
        side.wait_stream(torch.cuda.current_stream(dev))
        call("f2b_sampler_march", *march_args[:-1], side.cuda_stream)
        fused()

    def zero():
        table.zero_(); sp.zero_(); fp.zero_()
        if app is not None:
            app.zero_()

    def timed(fn):
        for _ in range(5):
            zero()
            fn()
        ms = []
        for _ in range(args.iters):
            zero()
            torch.cuda.current_stream(dev).wait_stream(side)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        torch.cuda.synchronize()
        return {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms)), "launches": len(ms)}

    def timed_march():                       # the march alone on the side stream, for reference
        for _ in range(3):
            call("f2b_sampler_march", *march_args[:-1], side.cuda_stream)
        ms = []
        for _ in range(args.iters // 2):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(side)
            call("f2b_sampler_march", *march_args[:-1], side.cuda_stream)
            e1.record(side)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms)), "launches": len(ms)}

    # bit-identity of the fused kernel's intermediate rows on this batch, and the dL/dfeat rows the scatter consumes
    zero()
    seq()
    ref_scene = d_scene16.clone()
    zero()
    fused(d_scene16, dfeat16)
    torch.cuda.synchronize()
    same = bool(torch.equal(ref_scene.view(torch.int16), d_scene16.view(torch.int16)))
    scales = ops.hash_level_scales().numpy()
    vol = anc.view(-1, stride)[:, 0].cpu().numpy() if stride > 1 else anc.cpu().numpy()
    reds = count_reductions(pts.cpu().numpy().reshape(-1, 3), vol.astype(np.int64), dfeat16.cpu().numpy(), scales, bias.cpu().numpy(),
                            int(n_vol))
    out = dict(gpu_info(), workload="wanjinyou, 4096 rays: shader-MLP bwd + input-assembly bwd + field-MLP bwd + hash scatter "
                                    "of the ray samples", ray_samples=int(n), iters=args.iters, app_embedding=pt_emb is not None,
               field_dout_rows_bit_identical=same)
    out["kernels"] = {
        "f2b_mlp_bwd2 (shader) + f2b_shader_prep_bwd_f16 + f2b_field_bwd_scatter (rays, in sequence)": timed(seq),
        "f2b_shade_field_bwd_scatter (rays)": timed(fused),
        "f2b_shade_field_bwd_scatter (rays, a march launched just before on a second stream)": timed(fused_after_march),
        "f2b_sampler_march (one batch, alone, for reference)": timed_march(),
    }
    peak = None
    if os.path.exists(args.red_rate):
        mb = json.load(open(args.red_rate))
        peak = max(r["g_lane_red_per_s"] for r in mb["rows"] if r["kind"] == "v2f32" and r["pattern"] == "spread")
    out["reductions"] = {"v2_lane_reductions": reds, "per_sample": reds / n, "v2f32_spread_peak_g_per_s": peak,
                         "note": "host count (bwd_probe.count_reductions); rate = count / kernel time, sequence: over its 3 kernels"}
    for name, k in out["kernels"].items():
        if "march" in name and "alone" in name:
            continue
        rate = reds / (k["median_ms"] * 1e-3) / 1e9
        out["reductions"][name] = {"g_lane_red_per_s": rate, "frac_of_v2f32_spread_peak": None if peak is None else rate / peak}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
