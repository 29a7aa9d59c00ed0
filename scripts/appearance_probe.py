"""Timing of appearance rendering and fitting (DESIGN.md §3m) on the ngp_fox scene (the reference's octree and warps and the cameras
from tests/golden, the test suite's deterministic field parameters):
- per 960 x 540 view (the 7 test cameras): render_forward without a row (f2b_render_fwd_fused) and with one
  (f2b_render_fwd_fused_app), each summed over the view's 8192-ray chunks; the two run alternately, view by view;
- one FitAppearance iteration at 4096 rays of the wanjinyou workload, split into its parts: march (f2b_sampler_march,
  f2b_slot_bounds), early stop (f2b_field_fwd_slots, f2b_early_stop_rays, f2b_count_scan), forward (f2b_render_phase2_fwd's
  entry points), the backward chain (f2b_composite_act_bwd, f2b_mlp_bwd2) and the reduction of dL/drow; and the wall time per
  iteration of a whole FitAppearance call (host syncs and the Adam step included).
CUDA events; medians over --reps after one warm-up.  The card's name and power limit are read in the same run.

    python scripts/appearance_probe.py [--reps 5] [--out profiles/h100_appearance_probe.json]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import numpy as np
    import torch
    import workloads
    import f2nerf_b200._lib as L
    from f2nerf_b200 import FitAppearance, RayGenerator, pose as P
    from f2nerf_b200.eval import _Validate
    from normals_probe import power_limit
    from test_gpu_normals import make_renderer
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_appearance_probe.json"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    renderer, _ = make_renderer()
    ev = lambda: torch.cuda.Event(enable_timing=True)
    g = torch.Generator(device="cpu").manual_seed(9)
    row = (torch.randn(16, generator=g) * .1).cuda()
    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_camrays.npz")))
    test = [int(c) for c in d["cam_test_set"]]
    H, W = (int(v) for v in d["ds_hw"])
    n_cams = d["ds_poses"].shape[0]
    ds = RayGenerator(d["ds_poses"].reshape(-1, 3, 4), d["ds_intri"].reshape(-1, 3, 3), d["ds_dist_params"], d["ds_bounds"],
                      height=H, width=W, train_set=[i for i in range(n_cams) if i not in test], test_set=test)
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit(), reps=args.reps, height=H, width=W)

    def view_ms(b, app):
        o, dd, _ = ds.RaysOfCamera(b)
        n, tot = o.shape[0], 0.
        with torch.no_grad(), _Validate(renderer):
            for i in range(0, n, 8192):
                j = min(i + 8192, n)
                e0, e1 = ev(), ev()
                e0.record()
                renderer.render_forward(o[i:j], dd[i:j], app=app)
                e1.record()
                torch.cuda.synchronize()
                tot += e0.elapsed_time(e1)
        return tot

    view_ms(test[0], None)
    view_ms(test[0], row)
    t = {"none": [], "row": []}
    for _ in range(args.reps):
        for b in test:
            t["none"].append(view_ms(b, None))
            t["row"].append(view_ms(b, row))
    none, app = np.array(t["none"]), np.array(t["row"])
    out["view"] = dict(n_views=len(test), none_ms=float(np.median(none)), row_ms=float(np.median(app)),
                       row_over_none=float(np.median(app / none)))

    n_rays = 4096
    o, dd, _ = workloads.host_rays("wanjinyou", n_rays, seed=7)
    o, dh = torch.from_numpy(np.asarray(o, np.float32)).cuda(), P._unit(torch.from_numpy(np.asarray(dd, np.float32)).cuda())
    gt = torch.rand((n_rays, 3), generator=g).cuda()
    names = {"f2b_sampler_march": "march", "f2b_slot_bounds": "march", "f2b_field_fwd_slots": "early_stop",
             "f2b_early_stop_rays": "early_stop", "f2b_count_scan": "early_stop", "f2b_composite_act_bwd": "backward_chain",
             "f2b_mlp_bwd2": "backward_chain"}
    parts = {}
    for rep in range(args.reps * 4 + 1):
        L.TRACE = []
        torch.cuda.synchronize()
        e0 = ev()
        e0.record()
        b = P._render(renderer, o, dh, app=row)
        d_colors = (2. * (b.colors - gt) / gt.numel()).contiguous()
        _, _, d_in16 = P._shader_input_bwd(b, d_colors, P.SHADER_LOSS_SCALE)
        r0, r1 = ev(), ev()
        r0.record()
        (d_in16[:, :16].double().sum(0) / P.SHADER_LOSS_SCALE).float()       # appearance._row_grad's reduction
        r1.record()
        e1 = ev()
        e1.record()
        torch.cuda.synchronize()
        tr, L.TRACE = L.TRACE, None
        if rep == 0:
            continue
        acc = dict(iteration_ms=e0.elapsed_time(e1), reduction=r0.elapsed_time(r1))
        for name, a, z, _ in tr:
            key = names.get(name, "casts" if name == "f2b_cast_f32_to_f16" else "forward")
            acc[key] = acc.get(key, 0.) + a.elapsed_time(z)
        for k, v in acc.items():
            parts.setdefault(k, []).append(v)
    it = {k: float(np.median(v)) for k, v in parts.items()}
    it["n_rays"], it["n_kept"] = n_rays, int(b.n_kept)
    iters = 50
    img = torch.rand((H, W, 3), generator=g)
    cam, pose = (ds.intri_[test[0]].cpu(), ds.dist_params_[test[0]].cpu()), ds.poses_[test[0]]
    FitAppearance(renderer, img, cam, pose, iters=3, n_rays=n_rays)
    wall = []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        FitAppearance(renderer, img, cam, pose, iters=iters, n_rays=n_rays)
        torch.cuda.synchronize()
        wall.append((time.perf_counter() - t0) * 1e3 / iters)
    it["fit_wall_ms_per_iteration"] = float(np.median(wall))
    out["fit_iteration"] = it
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
