"""Timing of cropped rendering (DESIGN.md §3n) on the ngp_fox scene (the reference's octree and warps and the cameras from
tests/golden, the test suite's deterministic field parameters), one 960 x 540 test view (the first test camera):
- render_forward (march + fused kernel) summed over the view's 8192-ray chunks, four ways, alternating within every repetition:
  no crop (f2b_render_fwd_fused), a box covering everything (f2b_render_fwd_fused_crop: the variant's overhead), a small box
  around the middle of what the view sees, and that box inverted;
- for each, the samples the march produced, the samples walked (inside the kept prefix, ``kept_counts``) and the samples encoded
  (walked and kept by the box), which explain a speed-up or a slow-down.
CUDA events; medians over --reps after one warm-up of every variant.  The card's name and power limit are read in the same run.

    python scripts/crop_probe.py [--reps 7] [--out profiles/h100_crop_probe.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

CHUNK = 8192


def main():
    import numpy as np
    import torch
    from f2nerf_b200 import Crop, RayGenerator
    from f2nerf_b200.eval import _Validate
    from normals_probe import power_limit
    from test_gpu_normals import make_renderer
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_crop_probe.json"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    renderer, _ = make_renderer()
    ev = lambda: torch.cuda.Event(enable_timing=True)
    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_camrays.npz")))
    test = [int(c) for c in d["cam_test_set"]]
    H, W = (int(v) for v in d["ds_hw"])
    n_cams = d["ds_poses"].shape[0]
    ds = RayGenerator(d["ds_poses"].reshape(-1, 3, 4), d["ds_intri"].reshape(-1, 3, 3), d["ds_dist_params"], d["ds_bounds"],
                      height=H, width=W, train_set=[i for i in range(n_cams) if i not in test], test_set=test)
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit(), reps=args.reps, height=H, width=W, view=test[0])
    o, dd, _ = ds.RaysOfCamera(test[0])
    o, dd = o.cuda(), dd.cuda()
    n = o.shape[0]

    # the small box: a cube around the median world point o + t d of the uncropped view's kept samples, half side the 15th
    # percentile of their L-inf distance from it (the box of tests/test_gpu_crop.py)
    pts = []
    with torch.no_grad(), _Validate(renderer):
        for i in range(0, n, CHUNK):
            r = renderer.render_forward(o[i:i + CHUNK], dd[i:i + CHUNK])
            s = r._keep[0]
            valid = torch.arange(s.slot, device="cuda")[None, :] < r.kept_counts[:, None]
            t = s.s_t.reshape(s.n_rays, s.slot, 1).double()
            pts.append((s.rays_o[:, None].double() + t * s.rays_d[:, None].double())[valid][::16])
    p = torch.cat(pts)
    c = p.median(0).values.cpu().numpy()
    dist = (p - torch.from_numpy(c).cuda()).abs().max(1).values
    h = float(dist.kthvalue(max(1, int(0.15 * dist.numel()))).values)
    small = Crop.box(c - h, c + h)
    variants = {"none": None, "cover": Crop.box([-1e6] * 3, [1e6] * 3), "small": small, "small_inverted": small.inverted()}
    out["small_box"] = dict(center=c.tolist(), half_side=h)

    def view(crop, count=False):
        tot, cnt = 0., dict(marched=0, walked=0, encoded=0)
        with torch.no_grad(), _Validate(renderer):
            for i in range(0, n, CHUNK):
                j = min(i + CHUNK, n)
                e0, e1 = ev(), ev()
                e0.record()
                r = renderer.render_forward(o[i:j], dd[i:j], crop=crop)
                e1.record()
                torch.cuda.synchronize()
                tot += e0.elapsed_time(e1)
                if count:
                    s = r._keep[0]
                    walked = torch.arange(s.slot, device="cuda")[None, :] < r.kept_counts[:, None]
                    w = torch.addcmul(s.rays_o[:, None], s.s_t.reshape(s.n_rays, s.slot, 1), s.rays_d[:, None])   # o + t d
                    kept = crop.mask(w).reshape(s.n_rays, s.slot) if crop is not None else torch.ones_like(walked)
                    cnt["marched"] += int(s.counts.sum())
                    cnt["walked"] += int(walked.sum())
                    cnt["encoded"] += int((walked & kept).sum())
        return tot, cnt

    counts = {k: view(v, count=True)[1] for k, v in variants.items()}      # (also the warm-up of every variant)
    t = {k: [] for k in variants}
    for _ in range(args.reps):
        for k, v in variants.items():
            t[k].append(view(v)[0])
    base = np.array(t["none"])
    out["view_ms"] = {k: dict(median_ms=float(np.median(v)), over_none=float(np.median(np.array(v) / base)), runs_ms=v, **counts[k])
                      for k, v in t.items()}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
