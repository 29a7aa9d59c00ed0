"""Timing of lens rendering (DESIGN.md §3o) on the H100:
- f2b_lens_rays for a 4096 x 2048 equirectangular panorama, a 4096 x 2048-per-eye ODS pair and a 2048^2 fisheye, with the rate
  of the 25 B it writes per ray (rays_o, rays_d, valid);
- RenderLens of a 2048 x 1024 equirectangular panorama against a 960 x 540 pinhole view (60 degrees vertical) from the same level
  pose at test view 0's position, on the ngp_fox scene (the reference's octree and warps and the cameras from tests/golden, the
  test suite's deterministic field parameters), with the samples marched and walked per ray and the rays per second.
CUDA events; medians over --reps with the cases alternating within every repetition, after one warm-up of each.  The card's name
and power limit are read in the same run.

    python scripts/lens_probe.py [--reps 7] [--out profiles/h100_lens_probe.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

BYTES_PER_RAY = 25
LAUNCHES = 20          # f2b_lens_rays launches per timed window


def main():
    import numpy as np
    import torch
    from f2nerf_b200 import Lens, RayGenerator, RenderLens, level_pose
    from f2nerf_b200.eval import _Validate
    from normals_probe import power_limit
    from test_gpu_normals import make_renderer
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_lens_probe.json"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit(), reps=args.reps)

    # ---- ray generation
    pose = torch.eye(3, 4, dtype=torch.float64)
    gens = {"equirect_4096x2048": Lens.equirect(2048, 4096), "ods_4096x2048_per_eye": Lens.ods(2048, 4096, ipd=0.01),
            "fisheye_2048x2048": Lens.fisheye(2048, fov=180.)}

    def time_rays(lens):
        lens.rays(pose)
        e0, e1 = ev(), ev()
        e0.record()
        for _ in range(LAUNCHES):
            lens.rays(pose)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / LAUNCHES

    for lens in gens.values():
        time_rays(lens)
    t = {k: [] for k in gens}
    for _ in range(args.reps):
        for k, lens in gens.items():
            t[k].append(time_rays(lens))
    out["lens_rays"] = {}
    for k, v in t.items():
        n = gens[k].n_rays
        ms = float(np.median(v))
        out["lens_rays"][k] = dict(rays=n, median_ms=ms, runs_ms=v, gb_per_s=n * BYTES_PER_RAY / ms / 1e6)
    out["lens_rays_note"] = "each timed call also allocates its outputs and copies the pose (Lens.rays)"

    # ---- rendering
    renderer, _ = make_renderer()
    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_camrays.npz")))
    test = [int(c) for c in d["cam_test_set"]]
    H, W = (int(v) for v in d["ds_hw"])
    n_cams = d["ds_poses"].shape[0]
    ds = RayGenerator(d["ds_poses"].reshape(-1, 3, 4), d["ds_intri"].reshape(-1, 3, 3), d["ds_dist_params"], d["ds_bounds"],
                      height=H, width=W, train_set=[i for i in range(n_cams) if i not in test], test_set=test)
    lp = level_pose(ds, test[0])
    views = {"equirect_2048x1024": Lens.equirect(1024, 2048), "pinhole_960x540": Lens.pinhole(540, 960, 60.)}
    out["render_pose"] = lp.tolist()

    def samples(lens):
        o, dd, _ = lens.rays(lp)
        marched = walked = 0
        with torch.no_grad(), _Validate(renderer):
            for i in range(0, o.shape[0], 8192):
                r = renderer.render_forward(o[i:i + 8192], dd[i:i + 8192])
                marched += int(r._keep[0].counts.sum())
                walked += int(r.kept_counts.sum())
        return marched, walked

    def time_view(lens):
        torch.cuda.synchronize()
        e0, e1 = ev(), ev()
        e0.record()
        RenderLens(renderer, lens, lp)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    counts = {k: samples(v) for k, v in views.items()}
    for v in views.values():
        time_view(v)
    t = {k: [] for k in views}
    for _ in range(args.reps):
        for k, v in views.items():
            t[k].append(time_view(v))
    out["render_lens"] = {}
    for k, v in t.items():
        n = views[k].n_rays
        ms = float(np.median(v))
        out["render_lens"][k] = dict(rays=n, median_ms=ms, runs_ms=v, rays_per_s=n / ms * 1e3,
                                     marched_per_ray=counts[k][0] / n, walked_per_ray=counts[k][1] / n)
    out["render_lens_note"] = "RenderLens end to end: rays, the tiled render and the one device->host copy of the colours"
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
