#!/usr/bin/env python
"""Generate the committed fixture tests/golden/ref_eval_metrics.npz with the reference's OWN evaluation code: ``rgb_ssim`` of
scripts/eval.py, run on the CPU, and skimage's peak_signal_noise_ratio beside it.

    python oracle/make_golden_metrics.py REFERENCE_DIR OUT_DIR     # writes OUT_DIR/ref_eval_metrics.npz
    mv OUT_DIR/ref_eval_metrics.npz tests/golden/

scripts/eval.py imports lpips (and skimage) at module level, so the module cannot be imported without them: ``rgb_ssim`` is taken
out of the file with ``ast`` and executed on its own, with numpy and scipy.signal, which is all it uses.  skimage's PSNR for two
uint8 images is one formula, restated here: data range 255, MSE = np.mean of the float64 squared differences,
10 log10(255^2 / MSE), inf when the MSE is 0.

For each pair NAME in ``names``: NAME_gt, NAME_pred (uint8 [H,W,3], as the script reads the PNGs), NAME_psnr and NAME_ssim
(float64, rgb_ssim(gt / 255., pred / 255., max_val=1)).  The pairs cover the 11 x 11 minimum (one valid SSIM pixel), odd sizes,
a constant ground truth, two constant images, identical images (PSNR inf) and a structured image with noise.  Under 100 KB.
"""
import ast
import os
import sys

import numpy as np
import scipy
import scipy.signal


def load_rgb_ssim(reference_dir):
    path = os.path.join(reference_dir, "scripts", "eval.py")
    tree = ast.parse(open(path).read(), path)
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "rgb_ssim"]
    assert len(fn) == 1, "rgb_ssim not found in " + path
    ns = {"np": np, "scipy": scipy}
    exec(compile(ast.Module(body=fn, type_ignores=[]), path, "exec"), ns)
    return ns["rgb_ssim"]


def skimage_psnr_u8(gt, pred):
    mse = np.mean((gt.astype(np.float64) - pred.astype(np.float64)) ** 2, dtype=np.float64)
    with np.errstate(divide="ignore"):
        return np.float64(10 * np.log10((255 ** 2) / mse))


def pairs(rng):
    u8 = lambda a: np.clip(np.rint(a), 0, 255).astype(np.uint8)
    noisy = lambda gt, s: u8(gt.astype(np.float64) + rng.normal(0., s, gt.shape))
    out = {}
    gt = rng.integers(0, 256, (11, 11, 3), dtype=np.uint8)
    out["min11"] = (gt, noisy(gt, 20.))
    gt = rng.integers(0, 256, (37, 53, 3), dtype=np.uint8)
    out["odd37x53"] = (gt, noisy(gt, 12.))
    gt = rng.integers(0, 256, (61, 17, 3), dtype=np.uint8)
    out["tall61x17"] = (gt, rng.integers(0, 256, gt.shape, dtype=np.uint8))
    gt = np.full((23, 29, 3), 118, np.uint8)
    out["constant_gt"] = (gt, noisy(gt, 3.))
    out["both_constant"] = (np.full((19, 31, 3), 40, np.uint8), np.full((19, 31, 3), 203, np.uint8))
    gt = rng.integers(0, 256, (31, 47, 3), dtype=np.uint8)
    out["identical"] = (gt, gt.copy())
    yy, xx = np.mgrid[0:64, 0:80].astype(np.float64)
    base = np.stack([120 + 90 * np.sin(xx / 7.) * np.cos(yy / 11.), 2.5 * xx + yy, 60 + 140 * ((xx > 30) & (yy < 40))], -1)
    gt = u8(base)
    out["structured"] = (gt, noisy(np.roll(gt, 1, axis=1), 6.))
    return out


def main():
    reference_dir, dst_dir = sys.argv[1], sys.argv[2]
    rgb_ssim = load_rgb_ssim(reference_dir)
    data = {}
    ps = pairs(np.random.default_rng(20261016))
    for name, (gt, pred) in ps.items():
        data[f"{name}_gt"], data[f"{name}_pred"] = gt, pred
        data[f"{name}_psnr"] = skimage_psnr_u8(gt, pred)
        data[f"{name}_ssim"] = np.float64(rgb_ssim(gt / 255., pred / 255., max_val=1))
        print(f"{name:14s} {gt.shape}  psnr {data[f'{name}_psnr']:.6f}  ssim {data[f'{name}_ssim']:.12f}")
    data["names"] = np.array(list(ps))
    os.makedirs(dst_dir, exist_ok=True)
    dst = os.path.join(dst_dir, "ref_eval_metrics.npz")
    np.savez_compressed(dst, **data)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
