"""Render a trained scene through a lens: an equirectangular panorama, an omnidirectional-stereo pair, a fisheye or a pinhole view.

    python scripts/render_panorama.py <runtime_config.yaml> <checkpoint_dir> --out pano.png
        [--lens {equirect,ods,fisheye,pinhole}] [--height 1024] [--width W] [--hfov 360] [--vfov 180] [--fov 180] [--ipd 0.064]
        [--camera i | --position x y z] [--level] [--yaw 0] [--pitch 0]
        [--depth] [--normals] [--appearance i] [--crop x0 y0 z0 x1 y1 z1 [--crop-invert]] [--path]

load_scene -> Lens (f2nerf_b200/lens.py) -> RenderLens (DESIGN.md §3o).  The pose is training camera i's (--camera, the default 0)
or a level pose at a point of the normalised scene frame (--position); --level turns a camera's pose into the level pose at its
position (``level_pose``: up = the training cameras' mean up), and --yaw / --pitch turn a level pose.  --ipd is in the data's own
units.  Colours are written as 8-bit PNGs quantised as TestImages writes them (trunc(clip(x, 0, 1) * 255)); --depth writes
<out>_opacity.npy and <out>_median_depth.npy (data units, radial distance along each pixel's ray), --normals <out>_normals.npy
(normalised scene frame), and <out>_valid.npy for a fisheye.  --path renders every frame of the dataset's render path through
the lens instead (<out>_0000.png, ...).  Prints one JSON line.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def write_png(path, colors):
    import numpy as np
    from PIL import Image
    img = (np.clip(colors.cpu().numpy(), 0., 1.) * 255.).astype(np.uint8)      # truncation, as TestImages' writer
    Image.fromarray(img).save(path)


def make_lens(a):
    from f2nerf_b200 import Lens
    if a.lens == "equirect":
        return Lens.equirect(a.height, a.width, hfov=a.hfov, vfov=a.vfov)
    if a.lens == "ods":
        return Lens.ods(a.height, a.width, hfov=a.hfov, vfov=a.vfov, ipd=a.ipd)
    if a.lens == "fisheye":
        return Lens.fisheye(a.height, a.width, fov=a.fov)
    return Lens.pinhole(a.height, a.width if a.width else a.height, a.vfov)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("config")
    ap.add_argument("checkpoint_dir")
    ap.add_argument("--out", required=True, help="PNG path (ODS: the left eye on top of the right)")
    ap.add_argument("--lens", choices=["equirect", "ods", "fisheye", "pinhole"], default="equirect")
    ap.add_argument("--height", type=int, default=1024, help="image height (ODS: per eye)")
    ap.add_argument("--width", type=int, default=None, help="default: 2 x height (equirect, ODS), height (fisheye, pinhole)")
    ap.add_argument("--hfov", type=float, default=360.)
    ap.add_argument("--vfov", type=float, default=None, help="default: 180 (equirect, ODS), 60 (pinhole)")
    ap.add_argument("--fov", type=float, default=180., help="fisheye field of view in degrees, up to 360")
    ap.add_argument("--ipd", type=float, default=0.064, help="ODS eye separation in the data's own units")
    pos = ap.add_mutually_exclusive_group()
    pos.add_argument("--camera", type=int, default=None, help="the pose of this camera (default 0)")
    pos.add_argument("--position", type=float, nargs=3, default=None, metavar=("X", "Y", "Z"),
                     help="a level pose at this point of the normalised scene frame")
    ap.add_argument("--level", action="store_true", help="with --camera: the level pose at the camera's position")
    ap.add_argument("--yaw", type=float, default=0., help="level pose: degrees to the right")
    ap.add_argument("--pitch", type=float, default=0., help="level pose: degrees up")
    ap.add_argument("--depth", action="store_true")
    ap.add_argument("--normals", action="store_true")
    ap.add_argument("--appearance", type=int, default=None, help="render with this training image's appearance row")
    ap.add_argument("--crop", type=float, nargs=6, default=None, metavar=("X0", "Y0", "Z0", "X1", "Y1", "Z1"),
                    help="keep only the axis-aligned box [x0, x1] x [y0, y1] x [z0, z1] of the normalised scene frame")
    ap.add_argument("--crop-invert", action="store_true", help="keep everything but the --crop box")
    ap.add_argument("--path", action="store_true", help="render the dataset's render path through the lens")
    a = ap.parse_args(argv)
    if a.vfov is None:
        a.vfov = 60. if a.lens == "pinhole" else 180.

    import numpy as np
    import torch
    from f2nerf_b200 import Crop, RenderLens, RenderPath, level_pose, load_scene

    lens = make_lens(a)
    scene = load_scene(a.config, a.checkpoint_dir, device="cuda")
    r, ds = scene.renderer, scene.dataset
    crop = Crop.box(a.crop[:3], a.crop[3:], invert=a.crop_invert) if a.crop else None
    stem = os.path.splitext(a.out)[0]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    info = dict(lens=repr(lens), shape=list(lens.shape))
    if a.path:
        if a.lens == "ods":
            from f2nerf_b200.lens import Lens
            lens = Lens.ods(lens.height, lens.width, lens.p0, lens.p1, ipd=a.ipd / float(ds.radius_))   # the path is in scene units
        frames = RenderPath(r, ds, lens=lens, appearance=a.appearance, crop=crop)
        for k, (c, _, _) in enumerate(frames):
            write_png(f"{stem}_{k:04d}.png", c)
        info["frames"] = len(frames)
    else:
        if a.position is not None:
            pose = level_pose(ds, a.position, a.yaw, a.pitch)
        elif a.level:
            pose = level_pose(ds, 0 if a.camera is None else a.camera, a.yaw, a.pitch)
        else:
            pose = ds.poses_[0 if a.camera is None else a.camera].double().cpu()
        if lens.model == "ods":
            from f2nerf_b200.lens import Lens
            lens = Lens.ods(lens.height, lens.width, lens.p0, lens.p1, ipd=a.ipd / float(ds.radius_))
        out = RenderLens(r, lens, pose, depth=a.depth, normals=a.normals, appearance=a.appearance, crop=crop)
        write_png(a.out, out["colors"])
        if a.depth:
            np.save(f"{stem}_opacity.npy", out["opacity"].numpy())
            np.save(f"{stem}_median_depth.npy", out["median_depth"].numpy() * float(ds.radius_))
        if a.normals:
            np.save(f"{stem}_normals.npy", out["normals"].numpy())
        if lens.may_be_invalid:
            np.save(f"{stem}_valid.npy", out["valid"].numpy())
        info["pose"] = pose.tolist()
    torch.cuda.synchronize()
    info.update(render_s=time.perf_counter() - t0, gpu=torch.cuda.get_device_properties(0).name, out=a.out)
    print(json.dumps(info))


if __name__ == "__main__":
    main()
