#!/usr/bin/env python
"""bwd_probe.py — what bounds the tail of the backward on the headline batch (wanjinyou, 4096 rays), kernel by kernel.

  python scripts/bwd_probe.py [--out profiles/h100_bwd_probe.json] [--red-rate profiles/h100_red_rate.json] [--iters 60]

Runs the forward of one TRAIN step through Renderer.Render (capture_step) and keeps the inputs of the field-MLP backward + hash
scatter of the ray samples (encoded features, fp16 field parameters, compacted points / anchors; the TV-loss edge segment is
reported by size).  The step's backward runs the rays' shader backward fused into the same kernel (f2b_shade_field_bwd_scatter),
so their field dL/dout rows are rebuilt here with the unfused kernels, f2b_mlp_bwd2 (shader) and f2b_shader_prep_bwd_f16.  Then times, with CUDA events (median of --iters launches after warm-up, table gradient zeroed before each):
  f2b_mlp_bwd2 (field, rays) | f2b_hash_bwd (rays) | the two in sequence | f2b_field_bwd_scatter (rays, the fused kernel).
The reductions the scatter issues are counted on the host (numpy restatement of the cell key of corners() and of the run rule
of scatter_level, hash.cuh), so the achieved lane-reduction rate can be set against the microbenchmark's v2f32 `spread` peak
(scripts/microbench_red.cu)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KDIRECT_HEADS = 24          # scatter_level: more run heads than this in a warp -> one reduction per live lane


def count_reductions(pts, vol, din, scales, bias, n_volumes):
    """v2 lane-reductions (8 per merged run, or 8 per live lane on the direct path) of the scatter over consecutive groups of 32."""
    n = pts.shape[0]
    pad = (-n) % 32
    x = ((pts.astype(np.float32) + np.float32(1)) * np.float32(.5)).astype(np.float32)
    g = din.astype(np.float32).reshape(n, 16, 2)
    total = 0
    for l in range(16):
        b = bias.reshape(-1, 3)[l * n_volumes + vol]                       # [n,3]
        p = (x.astype(np.float64) * np.float64(scales[l]) + b.astype(np.float64)).astype(np.float32)   # ~ fmaf
        cell = np.floor(p).astype(np.int64)
        live = (g[:, l, 0] != 0) | (g[:, l, 1] != 0)
        key = np.concatenate([cell, vol[:, None].astype(np.int64)], 1)
        key = np.concatenate([key, np.full((pad, 4), -1, np.int64)]).reshape(-1, 32, 4)
        live = np.concatenate([live, np.zeros(pad, bool)]).reshape(-1, 32)
        same = np.zeros_like(live)
        same[:, 1:] = (key[:, 1:] == key[:, :-1]).all(-1) & live[:, 1:] & live[:, :-1]
        head = ~same                                                        # lane 0, dead lanes and key changes start runs
        n_heads = head.sum(1)
        direct = n_heads > KDIRECT_HEADS
        live_runs = (head & live).sum(1)
        total += int(8 * np.where(direct, live.sum(1), live_runs).sum())
    return total


def capture_step(prob, rays_o, rays_d, emb, gt):
    """The forward of one TRAIN step through Render with the argument block ``ra`` of the launch sequences and the tensors it points
    to (``keepalive``) kept; dL/dcolors of the probes' loss from autograd, and from it dL/draw + dL/dlogit by one f2b_composite_act_bwd
    call: the inputs of the backward behind the composite as f2b_render_bwd sees them.  -> dict with the tensors the probes read."""
    import torch
    from f2nerf_b200 import renderer as R
    from f2nerf_b200._lib import call, stream
    renderer, field, shader = prob["renderer"], prob["field"], prob["shader"]
    seen = {}
    real = R._FusedRenderFunction.forward

    def keep(ctx, feat_pool, field_params, shader_params, app_emb, rnd, ra, keepalive, grad_on):
        seen.update(ra=ra, keepalive=keepalive)
        return real(ctx, feat_pool, field_params, shader_params, app_emb, rnd, ra, keepalive, grad_on)

    R._FusedRenderFunction.forward = staticmethod(keep)
    try:
        res = renderer.Render(rays_o, rays_d, None, emb)
    finally:
        R._FusedRenderFunction.forward = staticmethod(real)
    loss = torch.sqrt((res.colors - gt) ** 2 + 1e-4).mean() + ((res.edge_feats[:, 0] - res.edge_feats[:, 1]) ** 2).mean() * 1e-1
    (d_colors,) = torch.autograd.grad(loss, res.colors)
    ra, keepalive = seen["ra"], seen["keepalive"]
    T, n = keepalive[-1], ra.n_kept
    bounds, bg = keepalive[4], keepalive[6]
    d_logit = torch.empty((n,), dtype=torch.float32, device=rays_o.device)
    d_raw = torch.empty((n, 16), dtype=torch.float16, device=rays_o.device)
    call("f2b_composite_act_bwd", T["logit"], 1, T["rgb"], T["dt"], T["t"], bounds, bg, ra.n_rays, d_colors.contiguous(), None, None,
         None, float(renderer.global_data_pool_.gradient_scaling_progress_), T["raw"], float(shader.mlp_.loss_scale_), d_logit, 1,
         d_raw, stream())
    torch.cuda.synchronize()
    f_scale = float(field.mlp_.loss_scale_)
    pt_emb = T.get("pt_emb_idx")
    return dict(slots=keepalive[0], bounds=bounds, d_raw=d_raw, d_logit=d_logit, mlp_in=T["mlp_in"][:n], sp16=keepalive[3],
                fp16=keepalive[2], feat=T["feat_q"], pts=T["pts"][:n], anc=T["anchors"][:n], pt_emb=pt_emb, n=n, edge_rows=2 * ra.n_edge_pairs,
                inv_s=1.0 / float(shader.mlp_.loss_scale_), f_scale=f_scale, grad_mul=1.0 / f_scale,
                hash_args=(field.prim_pool_, field.bias_pool_, int(field.n_volumes_), int(field.local_size_)),
                d_sp=torch.zeros(ra.n_shader_params, dtype=torch.float32, device=rays_o.device),
                d_fp=torch.zeros(ra.n_field_params, dtype=torch.float32, device=rays_o.device),
                d_table=torch.zeros_like(field.feat_pool_),
                d_app=torch.zeros_like(renderer.app_emb_) if pt_emb is not None else None)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clk = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": power, "sm_clock_max": clk}
    except Exception as e:  # noqa: BLE001
        return {"gpu_info_error": str(e)[:120]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bwd_probe.json"))
    ap.add_argument("--red-rate", default=os.path.join(ROOT, "profiles", "h100_red_rate.json"))
    ap.add_argument("--iters", type=int, default=60)
    args = ap.parse_args()
    import torch
    import bench
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bargs = argparse.Namespace(config="wanjinyou", rays=0)
    prob = bench.build_problem(0, 1, bargs, dev)
    o, d, cam, gt = prob["host"]
    rays_o, rays_d, emb, gt = (torch.from_numpy(a).to(dev) for a in (o, d, cam, gt))
    c = capture_step(prob, rays_o, rays_d, emb, gt)
    bounds, d_raw, mlp_in, sp16, d_logit, pt_emb, inv_s, f_scale, feat, fparams16, n, pts, anc, grad_mul, d_sp, d_fp, d_table, d_app = (
        c[k] for k in ("bounds", "d_raw", "mlp_in", "sp16", "d_logit", "pt_emb", "inv_s", "f_scale", "feat", "fp16", "n", "pts", "anc",
                       "grad_mul", "d_sp", "d_fp", "d_table", "d_app"))
    prim, bias, n_vol, S = c["hash_args"]
    stride, edge_rows = 3, c["edge_rows"]
    d_in16 = torch.empty((n, 32), dtype=torch.float16, device=dev)
    dout = torch.empty((n, 16), dtype=torch.float16, device=dev)
    call("f2b_mlp_bwd2", d_raw, mlp_in, None, None, sp16, 1, n, d_in16, torch.zeros_like(d_sp), stream())
    ray_emb = emb.to(torch.int32).contiguous() if pt_emb is not None else None
    call("f2b_shader_prep_bwd_f16", d_in16, d_logit, bounds, ray_emb, bounds.shape[0], float(inv_s), float(f_scale), dout,
         None if d_app is None else torch.zeros_like(d_app), stream())
    din = torch.empty((n, 32), dtype=torch.float16, device=dev)
    dp = torch.zeros_like(d_fp)
    table = torch.zeros_like(d_table)

    def mlp():
        call("f2b_mlp_bwd2", dout, feat, None, None, fparams16, 0, n, din, dp, stream())

    def scat():
        ops.hash_bwd(prim, bias, n_vol, S, pts, anc, stride, din, grad_mul, table)

    def seq():
        mlp()
        scat()

    def fused():
        call("f2b_field_bwd_scatter", dout, feat, fparams16, n, pts, anc, stride, prim, bias, n_vol, S, grad_mul, dp, table, None,
             stream())

    def timed(fn):
        for _ in range(5):
            table.zero_(); dp.zero_()
            fn()
        ms = []
        for _ in range(args.iters):
            table.zero_(); dp.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms)), "launches": len(ms)}

    mlp()
    torch.cuda.synchronize()
    scales = ops.hash_level_scales().numpy()
    vol = anc.view(-1, stride)[:, 0].cpu().numpy() if stride > 1 else anc.cpu().numpy()
    reds = count_reductions(pts.cpu().numpy().reshape(-1, 3), vol.astype(np.int64), din.cpu().numpy(), scales, bias.cpu().numpy(),
                            int(n_vol))
    out = dict(gpu_info(), workload="wanjinyou, 4096 rays: field-MLP backward + hash scatter of the ray samples",
               ray_samples=int(n), edge_points=edge_rows, iters=args.iters)
    out["kernels"] = {"f2b_mlp_bwd2 (field, rays)": timed(mlp), "f2b_hash_bwd (rays)": timed(scat),
                      "f2b_mlp_bwd2 + f2b_hash_bwd (rays, in sequence)": timed(seq),
                      "f2b_field_bwd_scatter (rays, fused)": timed(fused)}
    peak = None
    if os.path.exists(args.red_rate):
        mb = json.load(open(args.red_rate))
        peak = max(r["g_lane_red_per_s"] for r in mb["rows"] if r["kind"] == "v2f32" and r["pattern"] == "spread")
    k = out["kernels"]
    out["reductions"] = {"v2_lane_reductions": reds, "per_sample": reds / n,
                         "note": "host count: numpy restatement of corners()' cell key and scatter_level's run rule (hash.cuh)"}
    for name in ("f2b_hash_bwd (rays)", "f2b_field_bwd_scatter (rays, fused)"):
        rate = reds / (k[name]["median_ms"] * 1e-3) / 1e9
        out["reductions"][name] = {"g_lane_red_per_s": rate, "frac_of_v2f32_spread_peak": None if peak is None else rate / peak}
    out["reductions"]["v2f32_spread_peak_g_per_s"] = peak
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
