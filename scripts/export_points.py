"""Export a trained scene's surface as a coloured PLY point cloud, fused from the training views on the device.

    python scripts/export_points.py <runtime_config.yaml> <checkpoint_dir> --out cloud.ply [--reso-level 1]
                                    [--min-opacity 0.9] [--min-views 2] [--normals] [--crop x0 y0 z0 x1 y1 z1 [--crop-invert]]

load_scene -> ExtractPointCloud (f2nerf_b200/geometry.py, DESIGN.md §3l); the cloud is written in the data's own world frame
(PointCloud.to_data_frame).  --crop renders only what an axis-aligned box of the normalised scene frame holds (DESIGN.md §3n).
Prints one JSON line: views, grid, point count, time and the GPU.
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
    ap.add_argument("--out", required=True)
    ap.add_argument("--reso-level", type=int, default=1, help="render each view on a (height // r) x (width // r) grid")
    ap.add_argument("--min-opacity", type=float, default=0.9, help="pixels below this opacity give no point")
    ap.add_argument("--min-views", type=int, default=2, help="other views that must confirm a point's depth (0: keep all)")
    ap.add_argument("--normals", action="store_true", help="the pixels' field normals (written as nx ny nz)")
    ap.add_argument("--crop", type=float, nargs=6, default=None, metavar=("X0", "Y0", "Z0", "X1", "Y1", "Z1"),
                    help="keep only the axis-aligned box [x0, x1] x [y0, y1] x [z0, z1] of the normalised scene frame")
    ap.add_argument("--crop-invert", action="store_true", help="keep everything but the --crop box")
    a = ap.parse_args(argv)

    import torch
    from f2nerf_b200 import Crop, geometry as G, load_scene

    scene = load_scene(a.config, a.checkpoint_dir, device="cuda")
    ds = scene.dataset
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pc = G.ExtractPointCloud(scene.renderer, ds, reso_level=a.reso_level, min_opacity=a.min_opacity, min_views=a.min_views,
                             normals=a.normals, crop=Crop.box(a.crop[:3], a.crop[3:], invert=a.crop_invert) if a.crop else None)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    G.write_ply(a.out, pc.to_data_frame(ds))
    print(json.dumps(dict(views=len(ds.train_set_), grid=[ds.height_ // a.reso_level, ds.width_ // a.reso_level],
                          min_opacity=a.min_opacity, min_views=a.min_views, crop=a.crop, crop_invert=a.crop_invert, points=int(pc.points.shape[0]), extract_s=dt,
                          gpu=torch.cuda.get_device_properties(0).name, out=a.out)))


if __name__ == "__main__":
    main()
