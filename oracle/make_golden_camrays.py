#!/usr/bin/env python
"""Generate the committed fixture tests/golden/ref_ngp_fox_camrays.npz by running the UNMODIFIED reference's Dataset
(oracle/_ref/ref_camrays, built by oracle/Makefile.camrays) on an H100:

    python oracle/make_golden_camrays.py OUT_DIR      # writes OUT_DIR/ref_ngp_fox_camrays.npz
    mv OUT_DIR/ref_ngp_fox_camrays.npz tests/golden/

It holds the reference's whole-camera rays (Dataset::RaysOfCamera(test_set_[0]), Dataset::RaysFromPose(render_poses_[0], 2) and
(render_poses_[5], 3)) with the camera tables, render poses and test set they come from.  Per image ``cam_<tag>_idx`` (int32 ray
indices: the first and last 64 and CAM_RAYS_SUB seeded ones), the rays and bounds at those indices, and ``cam_<tag>_n``, the
image's ray count.  Under 1 MB.
"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAM_RAYS_SUB = 4096               # seeded rays kept per image, besides its first and last 64
CAM_RAYS = ("test0", "path0_reso2", "path5_reso3")


def main():
    dst_dir = sys.argv[1]
    drv = os.path.join(ROOT, "oracle", "_ref", "ref_camrays")
    out = "/tmp/f2b_golden_camrays"
    r = subprocess.run([drv, os.path.join(ROOT, "oracle", "ref_config_ngp_fox.yaml"), out], cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    if r.returncode != 0:
        print(r.stdout[-2000:], r.stderr[-4000:])
        sys.exit(1)
    ld = lambda k: np.load(os.path.join(out, k + ".npy"))
    data = {k: ld(k) for k in ("ds_poses", "ds_intri", "ds_dist_params", "ds_bounds", "ds_hw", "cam_render_poses", "cam_test_set")}
    rng = np.random.default_rng(5)
    for tag in CAM_RAYS:
        o, d, b = ld(f"cam_{tag}_rays_o"), ld(f"cam_{tag}_rays_d"), ld(f"cam_{tag}_bounds")
        n = o.shape[0]
        idx = np.unique(np.concatenate([np.arange(64), np.arange(n - 64, n), rng.choice(n, CAM_RAYS_SUB, replace=False)]))
        data[f"cam_{tag}_idx"] = idx.astype(np.int32)
        data[f"cam_{tag}_n"] = np.array([n], np.int32)
        data[f"cam_{tag}_rays_o"], data[f"cam_{tag}_rays_d"], data[f"cam_{tag}_bounds"] = o[idx], d[idx], b[idx]
    os.makedirs(dst_dir, exist_ok=True)
    dst = os.path.join(dst_dir, "ref_ngp_fox_camrays.npz")
    np.savez_compressed(dst, **data)
    print("wrote", dst, os.path.getsize(dst) / 1e6, "MB")


if __name__ == "__main__":
    main()
