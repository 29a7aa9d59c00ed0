"""Evaluate trained reference checkpoints on the device: for each experiment directory (a ``base_exp_dir`` the reference program
trained into: checkpoints/latest/{renderer,scalars}.pt, test_images/), ``checkpoint.load_scene`` + ``eval.TestImages`` on its test
views.  Per view: the render time (CUDA events around a one-view TestImages: rays, tiled fused render, metrics; medians over
--reps after a warm-up pass over all views), PSNR, 8-bit PSNR and SSIM, the PSNR the program wrote to test_images/info.yaml,
and how far this path's colour PNG bytes are from the program's own PNG of that view.  Records the GPU and its power limit.
``--appearance`` adds ``appearance.TestAppearance``'s numbers (DESIGN.md §3m): the right half of each test view scored with no
appearance row, the training views' mean row and a row fitted on the left half.

    python scripts/eval_trained.py /tmp/f2b_train_ref /tmp/f2b_train_b200 [--config oracle/ref_config_ngp_fox.yaml] [--reps 3]
        [--appearance]

Run from the directory the program trained in: the config's dataset.data_path is relative to it.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                                            # noqa: BLE001  (no nvidia-smi: say so in the record)
        return None


def evaluate(exp, config, reps, appearance=False):
    import numpy as np
    import torch
    import yaml
    from PIL import Image
    from f2nerf_b200 import TestImages, load_scene
    scene = load_scene(config, checkpoint_dir=os.path.join(exp, "checkpoints", "latest"))
    renderer, ds = scene.renderer, scene.dataset
    info_path = os.path.join(exp, "test_images", "info.yaml")
    info = {}
    if os.path.isfile(info_path):
        with open(info_path) as f:
            info = {str(k): float(v) for k, v in yaml.safe_load(f).items()}
    out = TestImages(renderer, ds)                               # warm-up pass; its scores are the record
    torch.cuda.synchronize()
    test_set = list(ds.test_set_)
    times = {idx: [] for idx in test_set}
    try:
        for _ in range(reps):
            for idx in test_set:
                ds.test_set_ = [idx]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                TestImages(renderer, ds)
                e1.record()
                torch.cuda.synchronize()
                times[idx].append(e0.elapsed_time(e1))
    finally:
        ds.test_set_ = test_set
    views = []
    for k, idx in enumerate(test_set):
        v = dict(view=idx, ms=float(np.median(times[idx])), psnr=out["psnr"][idx], psnr_8bit=out["psnr_8bit"][idx],
                 ssim=out["ssim"][idx], program_psnr=info.get(str(idx)))
        png = os.path.join(exp, "test_images", f"color_{scene.iter_step}_{idx:03d}.png")
        if os.path.isfile(png):
            ref = np.asarray(Image.open(png)).astype(np.int16)
            ours = (out["colors"][k].cpu() * 255.).clip(0., 255.).to(torch.uint8).numpy().astype(np.int16)
            d = np.abs(ours - ref)
            v["png_vs_program"] = dict(values_differing=int((d != 0).sum()), of=int(d.size), max_levels=int(d.max()),
                                       mean_abs_levels=float(d.mean()))
        views.append(v)
    mean = lambda key: float(np.mean([v[key] for v in views]))
    rec = dict(experiment=exp, iter_step=scene.iter_step, ray_march_fineness=scene.global_data_pool.ray_march_fineness_,
               image_hw=[ds.height_, ds.width_], n_test_views=len(views), ms_per_view=mean("ms"), mean_psnr=out["mean_psnr"],
               mean_psnr_8bit=out["mean_psnr_8bit"], mean_ssim=out["mean_ssim"], program_mean_psnr=info.get("mean_psnr"),
               views=views)
    if appearance:
        from f2nerf_b200 import TestAppearance
        res = TestAppearance(renderer, ds)
        rec["appearance"] = {k: {m: res[k][m] for m in ("psnr", "psnr_8bit", "ssim", "mean_psnr", "mean_psnr_8bit", "mean_ssim")}
                             for k in ("none", "mean", "fit")}
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("experiments", nargs="+")
    ap.add_argument("--config", default=os.path.join(ROOT, "oracle", "ref_config_ngp_fox.yaml"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--appearance", action="store_true", help="also run TestAppearance (fit on the left half, score the right)")
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    rec = dict(probe="eval_trained", gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit(), config=args.config,
               reps=args.reps, experiments=[evaluate(e, args.config, args.reps, args.appearance) for e in args.experiments])
    text = json.dumps(rec, indent=1)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
