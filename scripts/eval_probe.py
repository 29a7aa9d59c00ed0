"""Where eval.TestImages spends its time on ngp_fox-sized images (540 wide, 960 high): ray generation (f2b_camera_rays), the tiled fused
render, and the metrics (quantise + float64 MSE + PSNR), per image, over the 7 test cameras of the ngp_fox scene
(tests/golden/ref_ngp_fox_camrays.npz; seeded synthetic ground truth, the images themselves are not in the repository).
CUDA events on the current stream; medians over --reps passes after one warm-up pass.

    python scripts/eval_probe.py [--reps 5] > eval_probe.json
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                                            # noqa: BLE001  (no nvidia-smi: say so in the record)
        return None


def main():
    import numpy as np
    import torch
    from f2nerf_b200 import RayGenerator, TestImages
    from f2nerf_b200.eval import RAY_BATCH_SIZE, _render_rays, _Validate, quantify
    from test_ref_parity import build_from_ref
    from workloads import load_golden
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    gdp, sampler, field, shader, renderer = build_from_ref(load_golden())
    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_ngp_fox_camrays.npz")))
    H, W = (int(v) for v in d["ds_hw"])
    cams = [int(c) for c in d["cam_test_set"]]
    g = torch.Generator(device=dev).manual_seed(0)
    images = torch.rand((len(cams), H, W, 3), generator=g, device=dev)
    gen = RayGenerator(d["ds_poses"].reshape(-1, 3, 4)[cams], d["ds_intri"].reshape(-1, 3, 3)[cams], d["ds_dist_params"][cams],
                       d["ds_bounds"][cams], images=images, test_set=range(len(cams)))
    n_img = len(cams)
    TestImages(renderer, gen)                                    # warm-up: scratch buffers, fp16 tables
    torch.cuda.synchronize()
    ev = lambda: torch.cuda.Event(enable_timing=True)
    total, rays, render, metrics = [], [], [], []
    for _ in range(args.reps):
        e0, e1 = ev(), ev()
        e0.record()
        res = TestImages(renderer, gen)
        e1.record()
        torch.cuda.synchronize()
        total.append(e0.elapsed_time(e1) / n_img)
        # the same work phase by phase (events between the phases; one sync at the end of the pass)
        marks = []
        with torch.no_grad(), _Validate(renderer):
            for idx in gen.test_set_:
                e = [ev() for _ in range(4)]
                e[0].record()
                o, dd, _ = gen.RaysOfCamera(idx)
                e[1].record()
                colors, first, disp = _render_rays(renderer, o, dd, RAY_BATCH_SIZE, dev)
                e[2].record()
                q = quantify(colors.reshape(H, W, 3))
                mse = (q.double() - gen.image_tensors_[idx].double()).square().mean()
                20. * torch.log10(1. / torch.sqrt(mse))
                e[3].record()
                marks.append(e)
        torch.cuda.synchronize()
        rays.append(sum(e[0].elapsed_time(e[1]) for e in marks) / n_img)
        render.append(sum(e[1].elapsed_time(e[2]) for e in marks) / n_img)
        metrics.append(sum(e[2].elapsed_time(e[3]) for e in marks) / n_img)
    med = lambda a: float(np.median(a))
    out = {"probe": "eval_probe", "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(),
           "image_hw": [H, W], "ground_truth": "synthetic (seeded uniform)",
           "scene": "ngp_fox octree and parameters of the golden reference run (seeded, untrained field)",
           "n_test_images": n_img, "reps": args.reps, "mean_psnr_synthetic_gt": res["mean_psnr"],
           "ms_per_image": {"test_images_total": med(total), "ray_generation": med(rays), "render": med(render),
                            "metrics": med(metrics)},
           "ms_per_image_all_reps": {"test_images_total": total, "ray_generation": rays, "render": render, "metrics": metrics}}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
