"""Timing and loss-scale check of pose refinement (DESIGN.md §3k) on the ngp_fox scene (the reference's octree and warps from
tests/golden, the test suite's deterministic field parameters), one 4096-ray batch of the wanjinyou workload:
- one refinement iteration split into its parts: march + early stop (f2b_render_phase1), forward (f2b_render_phase2_fwd), the
  backward chain (f2b_composite_act_bwd, f2b_mlp_bwd2, f2b_shader_prep_bwd_f16) and f2b_ray_grad;
- f2b_ray_grad per survivor against geometry.QueryGradient per point at 2^20 points;
- the fraction of the non-zero fp16 rows of the chain that are subnormal, at the chosen loss scales and at the trainer's 128, for
  the gradient of a mean squared colour error against random targets.
CUDA events; medians over --reps after one warm-up.  The card's name and power limit are read in the same run.

    python scripts/pose_probe.py [--reps 20] [--out profiles/h100_pose_probe.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def subnormal_fraction(x):
    import torch
    a = x.float().abs()
    nz = a > 0
    return float(((a < 2. ** -14) & nz).sum()) / max(int(nz.sum()), 1)


def main():
    import numpy as np
    import torch
    import workloads
    from f2nerf_b200 import geometry as G, ops, pose as P
    from f2nerf_b200._lib import call
    from normals_probe import power_limit
    from test_gpu_normals import make_renderer
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_pose_probe.json"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    renderer, sb = make_renderer()
    n_rays = 4096
    o, d, _ = workloads.host_rays("wanjinyou", n_rays, seed=7)
    o, d = torch.from_numpy(np.asarray(o, np.float32)).cuda(), torch.from_numpy(np.asarray(d, np.float32)).cuda()
    dh = P._unit(d)
    g = torch.Generator(device="cpu").manual_seed(8)
    gt = torch.rand((n_rays, 3), generator=g).cuda()
    ev = lambda: torch.cuda.Event(enable_timing=True)

    # per-part times of one iteration: the entry points of the library bracketed by events (the Python binding's TRACE)
    import f2nerf_b200._lib as L
    parts = {}
    b = P._render(renderer, o, dh)
    d_colors = (2. * (b.colors - gt) / gt.numel()).contiguous()
    for rep in range(args.reps + 1):
        L.TRACE = []
        torch.cuda.synchronize()
        e0 = ev()
        e0.record()
        b = P._render(renderer, o, dh)
        P._vjp(b, d_colors, d)
        e1 = ev()
        e1.record()
        torch.cuda.synchronize()
        tr, L.TRACE = L.TRACE, None
        if rep == 0:
            continue
        acc = dict(iteration_ms=e0.elapsed_time(e1))
        for name, a, z, _ in tr:
            key = {"f2b_sampler_march": "march", "f2b_slot_bounds": "march", "f2b_field_fwd_slots": "early_stop",
                   "f2b_early_stop_rays": "early_stop", "f2b_count_scan": "early_stop", "f2b_ray_grad": "ray_grad",
                   "f2b_composite_act_bwd": "backward_chain", "f2b_mlp_bwd2": "backward_chain",
                   "f2b_shader_prep_bwd_f16": "backward_chain"}.get(name, "forward" if name not in ("f2b_cast_f32_to_f16",) else "casts")
            acc[key] = acc.get(key, 0.) + a.elapsed_time(z)
        for k, v in acc.items():
            parts.setdefault(k, []).append(v)
    iteration = {k: float(np.median(v)) for k, v in parts.items()}
    iteration["n_rays"], iteration["n_kept"] = n_rays, int(b.n_kept)

    # ray_grad per survivor against QueryGradient per point
    rows = P._backprop(b, d_colors, P.SHADER_LOSS_SCALE, P.FIELD_LOSS_SCALE, rows=True)
    per_survivor_ns = iteration["ray_grad"] * 1e6 / max(b.n_kept, 1)
    from f2nerf_b200.octree_build import TREE_NODE
    nd = sb["nodes"].view(TREE_NODE)
    leaf = np.nonzero((nd["trans_idx"] >= 0) & (nd["childs"] < 0).all(1))[0]
    n = 1 << 20
    gg = torch.Generator(device="cuda").manual_seed(20)
    pick = torch.as_tensor(leaf, device="cuda")[torch.randint(0, len(leaf), (n,), generator=gg, device="cuda")]
    pts = (torch.as_tensor(nd["center"], device="cuda")[pick] +
           (torch.rand((n, 3), generator=gg, device="cuda") - .5) * .98 * torch.as_tensor(nd["side_len"], device="cuda")[pick, None]).contiguous()
    G.QueryGradient(renderer, pts)
    ms = []
    for _ in range(args.reps):
        e0, e1 = ev(), ev()
        e0.record()
        G.QueryGradient(renderer, pts)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    qg = float(np.median(ms))
    compare = dict(ray_grad_ns_per_survivor=per_survivor_ns, query_gradient_ns_per_point=qg * 1e6 / n, query_gradient_points=n)

    # subnormal fractions of the chain's fp16 rows
    sub = {}
    for name, (ss, fs) in (("chosen", (P.SHADER_LOSS_SCALE, P.FIELD_LOSS_SCALE)), ("trainer_128", (128., 128.))):
        r = P._backprop(b, d_colors, ss, fs, rows=True)
        sub[name] = dict(shader_loss_scale=ss, field_loss_scale=fs,
                         **{k: subnormal_fraction(r[k]) for k in ("d_raw", "d_in16", "d_field_out", "dfeat16")},
                         finite=bool(torch.isfinite(r["d_o"]).all() & torch.isfinite(r["d_d"]).all()))
    del rows
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit(), reps=args.reps, iteration=iteration,
               ray_grad_vs_query_gradient=compare, subnormal_fraction=sub,
               d_colors="2 (colour - target) / (3 n_rays), targets uniform in [0, 1)")
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
