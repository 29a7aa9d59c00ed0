"""Timing of the depth and point-cloud kernels (DESIGN.md §3l) on the ngp_fox scene (the reference's octree and warps and the
cameras from tests/golden, the test suite's deterministic field parameters):
- per 960 x 540 view (the 7 test cameras): render_forward, f2b_ray_termination_slots and f2b_render_normals_slots, each summed
  over the view's 8192-ray chunks, run one after another on one stream;
- one f2b_depth_consistency launch over the candidate points (opacity >= 0.9) of all 50 views;
- geometry.ExtractPointCloud over the 43 training views at reso_level 1 and 4, with and without normals.
CUDA events; medians over --reps after one warm-up.  The card's name and power limit are read in the same run.

    python scripts/points_probe.py [--reps 5] [--out profiles/h100_points_probe.json]
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
    from f2nerf_b200 import RayGenerator, ops
    from f2nerf_b200 import geometry as G
    from f2nerf_b200.eval import _Validate
    from normals_probe import power_limit
    from test_gpu_normals import make_renderer
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_points_probe.json"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    renderer, _ = make_renderer()
    f = renderer.scene_field_
    trans = renderer.pts_sampler_.pers_trans_gpu_
    ev = lambda: torch.cuda.Event(enable_timing=True)
    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_camrays.npz")))
    test = [int(c) for c in d["cam_test_set"]]
    H, W = (int(v) for v in d["ds_hw"])
    n_cams = d["ds_poses"].shape[0]
    ds = RayGenerator(d["ds_poses"].reshape(-1, 3, 4), d["ds_intri"].reshape(-1, 3, 3), d["ds_dist_params"], d["ds_bounds"],
                      height=H, width=W, train_set=[i for i in range(n_cams) if i not in test], test_set=test)
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit(), reps=args.reps, height=H, width=W)

    def view_split(b):
        """[render, termination, normals] ms of one view, each summed over its chunks."""
        o, dd, _ = ds.RaysOfCamera(b)
        n = o.shape[0]
        opa, med, pt, nm = (torch.empty(s, dtype=torch.float32, device="cuda") for s in ((n,), (n,), (n, 3), (n, 3)))
        tot = np.zeros(3)
        with torch.no_grad(), _Validate(renderer):
            for i in range(0, n, 8192):
                j = min(i + 8192, n)
                e = [ev() for _ in range(4)]
                e[0].record()
                r = renderer.render_forward(o[i:j], dd[i:j])
                e[1].record()
                ops.ray_termination_slots(r._keep[0], r.kept_counts, r._w_slots, opa[i:j], med[i:j], pt[i:j])
                e[2].record()
                ops.render_normals_slots(trans, f.table_f16(), f.prim_pool_, f.bias_pool_, f.n_volumes_, f.local_size_, f.mlp_.params_f16(),
                                         r._keep[0], r.kept_counts, r._w_slots, out=nm[i:j])
                e[3].record()
                torch.cuda.synchronize()
                tot += [e[k].elapsed_time(e[k + 1]) for k in range(3)]
        return tot

    view_split(test[0])
    per = np.median(np.stack([np.stack([view_split(b) for b in test]) for _ in range(args.reps)]), axis=0)   # [views, 3]
    out["per_view"] = dict(n_views=len(test), render_ms=float(np.median(per[:, 0])), termination_ms=float(np.median(per[:, 1])),
                           normals_ms=float(np.median(per[:, 2])), termination_over_render=float(np.median(per[:, 1] / per[:, 0])))

    allv = list(range(n_cams))
    cand = G.ExtractPointCloud(renderer, ds, views=allv, reso_level=1, min_views=0)
    P = cand.points.shape[0]
    b = test[0]
    o, dd = ds._camera_rays(ds.poses_[b], ds.intri_[b], ds.dist_params_[b], H, W)
    from f2nerf_b200 import RenderDepth
    opa, med, _ = (x.cuda() for x in RenderDepth(renderer, o, dd))
    count = torch.zeros((P,), dtype=torch.int32, device="cuda")
    src = cand.source[:, 0].contiguous()
    run = lambda: ops.depth_consistency(cand.points, src, b, ds.poses_[b], ds.intri_[b], ds.dist_params_[b], H, W, H, W, opa, med, .9, .01,
                                        count)
    run()
    ms = []
    for _ in range(args.reps):
        e0, e1 = ev(), ev()
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    out["consistency"] = dict(views_of_candidates=n_cams, candidates=P, launch_ms=float(np.median(ms)),
                              points_per_s=P / (float(np.median(ms)) * 1e-3))
    del cand, count, src

    out["extract"] = {}
    for reso in (1, 4):
        for nrm in (False, True):
            G.ExtractPointCloud(renderer, ds, reso_level=reso, normals=nrm)
            ts, n_pts = [], 0
            for _ in range(args.reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                pc = G.ExtractPointCloud(renderer, ds, reso_level=reso, normals=nrm)
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
                n_pts = int(pc.points.shape[0])
            out["extract"][f"reso{reso}{'_normals' if nrm else ''}"] = dict(views=len(ds.train_set_), ms=float(np.median(ts)), points=n_pts)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
