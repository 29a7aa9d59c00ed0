"""Refine the camera pose of a photo of a trained scene on the device.

    python scripts/register_pose.py <runtime_config.yaml> <checkpoint_dir> --view I [--perturb-deg 3 --perturb-frac 0.03 --seed 0]
                                    [--image photo.png --pose pose0.npy] [--iters 300 --rays 4096 --lr 2e-3] --out pose.npy

load_scene -> pose.RefinePose (DESIGN.md §3k).  The photo and the camera are dataset view I's unless --image is given (then view I
only supplies the intrinsics and distortion); the initial pose is --pose (a [3,4] camera-to-world .npy in the data's own frame) or
view I's pose perturbed by a seeded rotation of --perturb-deg about a random axis and a move of --perturb-frac of the camera's
distance to the scene centre.  The refined pose is written in the data's own frame.  Prints one JSON line: the losses, and against
view I's dataset pose the rotation and translation errors before and after.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("config")
    ap.add_argument("checkpoint_dir")
    ap.add_argument("--view", type=int, required=True)
    ap.add_argument("--image", default=None)
    ap.add_argument("--pose", default=None)
    ap.add_argument("--perturb-deg", type=float, default=3.0)
    ap.add_argument("--perturb-frac", type=float, default=0.03)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--lr", type=float, default=2e-3)
    ap.add_argument("--out", required=True)
    a = ap.parse_args(argv)

    import numpy as np
    import torch
    from f2nerf_b200 import load_scene, pose as P
    from f2nerf_b200.dataset import read_image_u8

    scene = load_scene(a.config, a.checkpoint_dir, device="cuda")
    ds, i = scene.dataset, a.view
    if not 0 <= i < ds.n_images_:
        raise SystemExit(f"--view {i} outside [0, {ds.n_images_})")
    image = ds.image_tensors_[i] if a.image is None else torch.from_numpy(read_image_u8(a.image)).float() / 255.
    gt = ds.poses_[i].double().cpu()
    if a.pose is not None:
        p0 = P.data_to_scene(np.load(a.pose).reshape(3, 4), ds)
    else:
        p0 = P.perturb(gt, a.perturb_deg, a.perturb_frac * float(torch.linalg.norm(gt[:, 3])), a.seed)
    t0 = time.perf_counter()
    pose, losses = P.RefinePose(scene.renderer, image, i, p0, iters=a.iters, n_rays=a.rays, lr=a.lr, seed=a.seed, dataset=ds)
    secs = time.perf_counter() - t0
    np.save(a.out, P.scene_to_data(pose, ds).numpy())
    print(json.dumps(dict(view=i, iters=a.iters, rays=a.rays, seconds=secs, loss_first=losses[0] if losses else None,
                          loss_last=losses[-1] if losses else None,
                          rot_err_deg=[P.rotation_error_deg(p0, gt), P.rotation_error_deg(pose, gt)],
                          trans_err_scene=[P.translation_error(p0, gt), P.translation_error(pose, gt)],
                          gpu=torch.cuda.get_device_name(0))))


if __name__ == "__main__":
    main()
