"""Timing of TSDF fusion (DESIGN.md §3p) on the ngp_fox scene (the reference's octree and warps and the cameras from tests/golden,
the test suite's deterministic field parameters):
- one f2b_tsdf_integrate launch per group of views (the 43 training views' maps at reso_level 4, groups of 43) over 256^3 and 512^3
  lattices, with the bytes of sums a launch must move per lattice point: 20 B written, and 20 B read on every group but the first;
- geometry.ExtractTSDFMesh over the 43 training views at reso_level 1 and 4 (512^3), split into rendering (pass 1 and the default
  box), fusion (FuseTSDF), surface (TSDFSurface without its colours) and colours (f2b_tsdf_colors).
CUDA events and host clocks around synchronised work; medians over --reps after one warm-up.  The card's name and power limit are
read in the same run.

    python scripts/tsdf_probe.py [--reps 5] [--out profiles/h100_tsdf_probe.json]
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
    from normals_probe import power_limit
    from test_gpu_normals import make_renderer
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_tsdf_probe.json"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    renderer, _ = make_renderer()
    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_camrays.npz")))
    test = [int(c) for c in d["cam_test_set"]]
    H, W = (int(v) for v in d["ds_hw"])
    n_cams = d["ds_poses"].shape[0]
    ds = RayGenerator(d["ds_poses"].reshape(-1, 3, 4), d["ds_intri"].reshape(-1, 3, 3), d["ds_dist_params"], d["ds_bounds"],
                      height=H, width=W, train_set=[i for i in range(n_cams) if i not in test], test_set=test)
    views = list(ds.train_set_)
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit(), reps=args.reps, height=H, width=W, views=len(views))
    ev = lambda: torch.cuda.Event(enable_timing=True)
    med = lambda x: float(np.median(x))

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return r, (time.perf_counter() - t0) * 1e3

    # ---- the integrate kernel alone, on the maps of reso_level 4
    apps = [None] * len(views)
    opa, mt, col, lo, hi = G._tsdf_maps(renderer, ds, views, 4, None, None, .9, apps, None)
    idx = torch.as_tensor(views, device="cuda")
    cams = torch.cat([ds.poses_[idx].reshape(-1, 12), ds.intri_[idx].reshape(-1, 9)[:, :6], ds.dist_params_[idx]], 1).contiguous()
    out["box"] = dict(bbox_min=list(lo), bbox_max=list(hi))
    out["integrate"] = {}
    for reso in (256, 512):
        origin, voxel, (nx, ny, nz) = G._lattice(lo, hi, reso, "probe")
        s = torch.empty((nz, ny, nx), device="cuda")
        w, c = torch.empty_like(s), torch.empty((nz, ny, nx, 3), device="cuda")
        mu = float(np.float32(4 * voxel))
        res = {}
        for first in (True, False):
            run = lambda: ops.tsdf_integrate(cams, opa, mt, col, H, W, origin, voxel, 0, nz, mu, .9, first, s, w, c)
            run()
            ms = []
            for _ in range(args.reps):
                e0, e1 = ev(), ev()
                e0.record()
                run()
                e1.record()
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1))
            n = nx * ny * nz
            moved = n * (20 if first else 40)
            res["first_group" if first else "later_group"] = dict(ms=med(ms), sum_bytes=moved, sum_bytes_per_s=moved / (med(ms) * 1e-3),
                                                                  point_views_per_s=n * len(views) / (med(ms) * 1e-3))
        out["integrate"][f"{reso}^3"] = dict(lattice=[nx, ny, nz], group=len(views), **res)
        del s, w, c
    del opa, mt, col

    # ---- ExtractTSDFMesh end to end, split into its phases
    out["extract"] = {}
    for rl in (1, 4):
        G.ExtractTSDFMesh(renderer, ds, reso_level=rl)                                     # warm-up
        phases = {k: [] for k in ("render", "fusion", "surface", "colors", "total")}
        for _ in range(args.reps):
            (o_, m_, c_, lo_, hi_), t_r = timed(lambda: G._tsdf_maps(renderer, ds, views, rl, None, None, .9, apps, None))
            grid, t_f = timed(lambda: G.FuseTSDF(ds.poses_[idx], ds.intri_[idx], ds.dist_params_[idx], H, W, o_, m_, c_, lo_, hi_))
            del o_, m_, c_
            mesh, t_s = timed(lambda: G.TSDFSurface(grid))
            _, t_c = timed(lambda: ops.tsdf_colors(mesh.verts, grid.weight, grid.color_sum, grid.origin, grid.voxel))
            del grid
            _, t_all = timed(lambda: G.ExtractTSDFMesh(renderer, ds, reso_level=rl))
            for k, v in zip(phases, (t_r, t_f, t_s - t_c, t_c, t_all)):
                phases[k].append(v)
        ph = {k: med(v) for k, v in phases.items()}
        out["extract"][f"reso_level{rl}"] = dict(reso=512, render_ms=ph["render"], fusion_ms=ph["fusion"], surface_ms=ph["surface"],
                                                 colors_ms=ph["colors"], total_ms=ph["total"],
                                                 fusion_share=ph["fusion"] / (ph["render"] + ph["fusion"] + ph["surface"] + ph["colors"]),
                                                 verts=int(mesh.verts.shape[0]), faces=int(mesh.faces.shape[0]))
        del mesh
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
