#!/usr/bin/env python
"""march_probe.py — what the ray march costs the training step it is pipelined under (headline batch: wanjinyou, 4096 rays on
the reference's ngp_fox blobs).

  python scripts/march_probe.py [--out profiles/h100_march_probe.json] [--iters 60] [--bench-pairs 5] [--bench-steps 50]

Runs the forward of one TRAIN step through Renderer.Render (bwd_probe.capture_step) and keeps the inputs of the step's
f2b_shade_field_bwd_scatter (the ray samples' backward) and of its f2b_sampler_march (the batch marched once more through
PersSampler.march_rays).  Then records, with CUDA events (median of --iters launches after warm-up):
  march alone          f2b_sampler_march on its stream (the march kernel in its one-pass mode + the count scan);
  backward alone       f2b_shade_field_bwd_scatter, gradients zeroed before each launch;
  backward + march     the march launched on a second stream just before the backward (as in training, where the next batch's
                       march is pipelined behind the backward): each kernel's own time and the pair's, first start to last end;
and a digest of the march's outputs (counts, pts, dt, t, anchors, first_oct_dis), so two builds can be compared bit for bit.
With --bench-pairs N > 0 it also runs `bench.py --steps S --warmup 10 --no-cpu-baseline` against the same command with
--no-pipeline-march, alternating, N pairs: what the pipelined march costs the step end to end."""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def stats(ms):
    return {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms)), "launches": len(ms)}


def bench_line(steps, extra):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", "10",
           "--no-cpu-baseline"] + extra
    p = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT, timeout=900)
    lines = [s for s in p.stdout.splitlines() if s.startswith("{")]
    if p.returncode or not lines:
        return {"error": (p.stderr or p.stdout)[-600:]}
    r = json.loads(lines[-1])
    fo = r.get("forward_only") or {}
    return {"ms_per_step": r["ms_per_step"], "clocks": r.get("clocks"), "forward_only_ms": fo.get("ms_per_step"),
            "samples_per_ray": r["workload_measured"]["samples_per_ray"],
            "march_ms_per_step": (r["kernels"].get("f2b_sampler_march") or {}).get("ms_per_step")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_march_probe.json"))
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--bench-pairs", type=int, default=5)
    ap.add_argument("--bench-steps", type=int, default=50)
    args = ap.parse_args()
    import torch
    import bench
    from bwd_probe import capture_step, gpu_info
    from f2nerf_b200 import sampler as SM
    from f2nerf_b200._lib import call, stream

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bargs = argparse.Namespace(config="wanjinyou", rays=0)
    prob = bench.build_problem(0, 1, bargs, dev)
    o, d, cam, gt = prob["host"]
    rays_o, rays_d, emb, gt = (torch.from_numpy(a).to(dev) for a in (o, d, cam, gt))
    c = capture_step(prob, rays_o, rays_d, emb, gt)
    d_raw, mlp_in, sp16, d_logit, pt_emb, inv_s, f_scale, feat, fp16_, n, pts, anc, grad_mul, d_sp, d_fp, d_table, d_app = (
        c[k] for k in ("d_raw", "mlp_in", "sp16", "d_logit", "pt_emb", "inv_s", "f_scale", "feat", "fp16", "n", "pts", "anc",
                       "grad_mul", "d_sp", "d_fp", "d_table", "d_app"))
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
    march_args = kept["f2b_sampler_march"][:-1]
    ticket = torch.empty((1,), dtype=torch.int32, device=dev)
    sp, fp, table = torch.zeros_like(d_sp), torch.zeros_like(d_fp), torch.zeros_like(d_table)
    app = torch.zeros_like(d_app) if d_app is not None else None
    hash_args = c["hash_args"]
    main_s, side = torch.cuda.current_stream(dev), torch.cuda.Stream(dev)

    def march(st):
        call("f2b_sampler_march", *march_args, st.cuda_stream)

    def bwd():
        call("f2b_shade_field_bwd_scatter", d_raw, mlp_in, sp16, d_logit, pt_emb, inv_s, f_scale, feat, fp16_, n, pts, anc, 3,
             *hash_args, grad_mul, sp, fp, table, app, ticket, None, None, None, stream())

    def zero():
        table.zero_(); sp.zero_(); fp.zero_()
        if app is not None:
            app.zero_()

    ev = lambda: torch.cuda.Event(enable_timing=True)

    def time_march():
        for _ in range(5):
            march(side)
        ms = []
        for _ in range(args.iters):
            e0, e1 = ev(), ev()
            e0.record(side)
            march(side)
            e1.record(side)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return stats(ms)

    def time_bwd():
        for _ in range(5):
            zero()
            bwd()
        ms = []
        for _ in range(args.iters):
            zero()
            e0, e1 = ev(), ev()
            e0.record(main_s)
            bwd()
            e1.record(main_s)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return stats(ms)

    def time_pair():
        m_ms, b_ms, p_ms = [], [], []
        for i in range(args.iters + 5):
            zero()
            torch.cuda.synchronize()
            e0, s0, s1, b0, b1, e1 = ev(), ev(), ev(), ev(), ev(), ev()
            e0.record(main_s)
            side.wait_stream(main_s)
            s0.record(side)
            march(side)
            s1.record(side)
            b0.record(main_s)
            bwd()
            b1.record(main_s)
            main_s.wait_stream(side)
            e1.record(main_s)
            e1.synchronize()
            if i >= 5:
                m_ms.append(s0.elapsed_time(s1)); b_ms.append(b0.elapsed_time(b1)); p_ms.append(e0.elapsed_time(e1))
        return {"march": stats(m_ms), "backward": stats(b_ms), "pair": stats(p_ms)}

    # the march's outputs on this batch, as one digest
    march(main_s)
    torch.cuda.synchronize()
    s_pts, s_dt, s_t, s_anc, counts, bounds, totals, fod = (march_args[i] for i in range(14, 22))
    n_rays = int(march_args[7])
    h = hashlib.sha256()
    for tsr in (counts[:n_rays], totals, fod[:n_rays]):
        h.update(tsr.cpu().numpy().tobytes())
    cnt = counts[:n_rays].cpu().numpy()
    for tsr, w in ((s_pts, 3), (s_dt, 1), (s_t, 1), (s_anc, 2)):
        a = tsr.reshape(-1)[:n_rays * 1024 * w].view(n_rays, 1024, w).cpu().numpy()
        for r in range(n_rays):
            h.update(a[r, :cnt[r]].tobytes())

    out = dict(gpu_info(), workload="wanjinyou, 4096 rays: f2b_sampler_march (one-pass march + count scan) and "
                                    "f2b_shade_field_bwd_scatter (the ray samples' backward)", iters=args.iters,
               march_samples=int(cnt.sum()), march_rays=int(cnt.shape[0]), march_output_sha256=h.hexdigest())
    out["march_alone"] = time_march()
    out["backward_alone"] = time_bwd()
    out["backward_with_march_on_second_stream"] = time_pair()
    pair = out["backward_with_march_on_second_stream"]
    out["march_cost_to_backward_ms"] = pair["pair"]["median_ms"] - out["backward_alone"]["median_ms"]
    if args.bench_pairs > 0:
        rows = []
        for i in range(args.bench_pairs):
            rows.append({"pair": i + 1, "pipelined": bench_line(args.bench_steps, []),
                         "unpipelined": bench_line(args.bench_steps, ["--no-pipeline-march"])})
        out["bench"] = {"command": f"python bench.py --gpus 1 --steps {args.bench_steps} --warmup 10 --no-cpu-baseline "
                                   "[--no-pipeline-march], pipelined first in each pair", "pairs": rows}
        ok = [r for r in rows if "ms_per_step" in r["pipelined"] and "ms_per_step" in r["unpipelined"]]
        if ok:
            out["bench"]["median_ms_per_step_pipelined"] = float(np.median([r["pipelined"]["ms_per_step"] for r in ok]))
            out["bench"]["median_ms_per_step_unpipelined"] = float(np.median([r["unpipelined"]["ms_per_step"] for r in ok]))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({k: v for k, v in out.items() if k != "bench"}))


if __name__ == "__main__":
    main()
