"""Where eval.TestImages spends its time on ngp_fox-sized images (540 wide, 960 high): ray generation (f2b_camera_rays), the tiled fused
render, the metrics (quantise + float64 MSE + PSNR) and the evaluation script's 8-bit PSNR + SSIM (f2b_image_metrics), per image,
over the 7 test cameras of the ngp_fox scene (tests/golden/ref_ngp_fox_camrays.npz; seeded synthetic ground truth, the images
themselves are not in the repository).  CUDA events on the current stream; medians over --reps passes after one warm-up pass.
Besides: f2b_image_metrics alone, back to back on one view, and the same PSNR + SSIM computed on the host by the float64
numpy / scipy restatement of the script (tests/image_metrics_oracle.py) from the view's 8-bit images, timed on the CPU.

    python scripts/eval_probe.py [--reps 5] > eval_probe.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

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
    import image_metrics_oracle as IM
    from f2nerf_b200.eval import RAY_BATCH_SIZE, _image_metrics, _render_rays, _Validate, quantify
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
    total, rays, render, metrics, image_metrics = [], [], [], [], []
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
                e = [ev() for _ in range(5)]
                e[0].record()
                o, dd, _ = gen.RaysOfCamera(idx)
                e[1].record()
                colors, first, disp = _render_rays(renderer, o, dd, RAY_BATCH_SIZE, dev)
                e[2].record()
                q = quantify(colors.reshape(H, W, 3))
                mse = (q.double() - gen.image_tensors_[idx].double()).square().mean()
                20. * torch.log10(1. / torch.sqrt(mse))
                e[3].record()
                _image_metrics(q, gen.image_tensors_[idx])
                e[4].record()
                marks.append(e)
        torch.cuda.synchronize()
        rays.append(sum(e[0].elapsed_time(e[1]) for e in marks) / n_img)
        render.append(sum(e[1].elapsed_time(e[2]) for e in marks) / n_img)
        metrics.append(sum(e[2].elapsed_time(e[3]) for e in marks) / n_img)
        image_metrics.append(sum(e[3].elapsed_time(e[4]) for e in marks) / n_img)
    # f2b_image_metrics alone: CALLS launches back to back on the last view's quantised colours and ground truth
    calls = 200
    gt = gen.image_tensors_[gen.test_set_[-1]]
    kernel = []
    for _ in range(args.reps):
        e0, e1 = ev(), ev()
        e0.record()
        for _ in range(calls):
            _image_metrics(q, gt)
        e1.record()
        torch.cuda.synchronize()
        kernel.append(e0.elapsed_time(e1) / calls)
    # the evaluation script's arithmetic on the host (float64 numpy / scipy) for the same view, from its 8-bit images
    p8, g8 = IM.pred_to_u8(q.cpu().numpy()), IM.gt_to_u8(gt.cpu().numpy())
    host = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        IM.psnr(p8, g8), IM.ssim(p8, g8)
        host.append((time.perf_counter() - t0) * 1e3)
    med = lambda a: float(np.median(a))
    out = {"probe": "eval_probe", "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(),
           "image_hw": [H, W], "ground_truth": "synthetic (seeded uniform)",
           "scene": "ngp_fox octree and parameters of the golden reference run (seeded, untrained field)",
           "n_test_images": n_img, "reps": args.reps, "mean_psnr_synthetic_gt": res["mean_psnr"],
           "mean_psnr_8bit_synthetic_gt": res["mean_psnr_8bit"], "mean_ssim_synthetic_gt": res["mean_ssim"],
           "ms_per_image": {"test_images_total": med(total), "ray_generation": med(rays), "render": med(render),
                            "metrics": med(metrics), "image_metrics": med(image_metrics)},
           "ms_per_image_all_reps": {"test_images_total": total, "ray_generation": rays, "render": render, "metrics": metrics,
                                     "image_metrics": image_metrics},
           "image_metrics_alone": {"ms_per_call": med(kernel), "calls_per_rep": calls, "ms_per_call_all_reps": kernel,
                                   "bytes_read": 2 * H * W * 3 * 4},
           "host_psnr_ssim": {"ms_per_image": med(host), "ms_all_reps": host, "cpu": cpu_name(), "threads": os.cpu_count(),
                              "what": "image_metrics_oracle.psnr + ssim (float64 numpy / scipy) on the view's 8-bit images"}}
    print(json.dumps(out, indent=1))


def cpu_name():
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return None


if __name__ == "__main__":
    main()
