"""Extract a trained scene's surface as a coloured PLY mesh on the device.

    python scripts/extract_mesh.py <runtime_config.yaml> <checkpoint_dir> [--reso 512] [--alpha 0.5]
                                   [--bbox x0 y0 z0 x1 y1 z1] [--crop x0 y0 z0 x1 y1 z1 [--crop-invert]]
                                   [--tsdf [--reso-level N] [--trunc T]] --out scene.ply

load_scene -> DensityGrid -> Isosurface -> VertexColors (f2nerf_b200/geometry.py); the mesh is written in the data's own world
frame (Mesh.to_data_frame).  --bbox is in the normalised scene frame (default: the valid leaves' bounding box, or with --crop
the crop box within it).  --crop keeps only what an axis-aligned box of the scene frame holds (DESIGN.md §3n).  Prints one
JSON line: lattice size, grid-query time and rate, extraction time, colour time, vertex and face counts, and the GPU.
--tsdf meshes the surface fused from the training views' depth maps instead (ExtractTSDFMesh, DESIGN.md §3p), rendered at
--reso-level with a truncation of --trunc voxels (default box: the opaque pixels' median points, or the crop box); its JSON line
gives the lattice size, the total time, vertex and face counts, and the GPU.
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
    ap.add_argument("--reso", type=int, default=512)
    ap.add_argument("--alpha", type=float, default=0.5)
    ap.add_argument("--bbox", type=float, nargs=6, default=None)
    ap.add_argument("--out", required=True)
    ap.add_argument("--crop", type=float, nargs=6, default=None, metavar=("X0", "Y0", "Z0", "X1", "Y1", "Z1"),
                    help="keep only the axis-aligned box [x0, x1] x [y0, y1] x [z0, z1] of the normalised scene frame")
    ap.add_argument("--crop-invert", action="store_true", help="keep everything but the --crop box")
    ap.add_argument("--normals", action="store_true", help="field normals on the vertices (written as nx ny nz; colours seen along them)")
    ap.add_argument("--repeat", type=int, default=1, help="time the grid query and the extraction this many times (median)")
    ap.add_argument("--tsdf", action="store_true", help="fuse the training views' depth maps into a TSDF and mesh its zero level set")
    ap.add_argument("--reso-level", dest="reso_level", type=int, default=1, help="--tsdf: render the views at height and width / N")
    ap.add_argument("--trunc", type=float, default=4., help="--tsdf: truncation distance in voxels")
    a = ap.parse_args(argv)

    import torch
    from f2nerf_b200 import Crop, geometry as G, load_scene

    scene = load_scene(a.config, a.checkpoint_dir, device="cuda")
    r = scene.renderer
    lo, hi = (a.bbox[:3], a.bbox[3:]) if a.bbox else (None, None)
    crop = Crop.box(a.crop[:3], a.crop[3:], invert=a.crop_invert) if a.crop else None

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0

    props = torch.cuda.get_device_properties(0)
    if a.tsdf:
        mesh, t = timed(lambda: G.ExtractTSDFMesh(r, scene.dataset, reso_level=a.reso_level, reso=a.reso, bbox_min=lo, bbox_max=hi,
                                                  trunc=a.trunc, crop=crop))
        G.write_ply(a.out, mesh.to_data_frame(scene.dataset))
        print(json.dumps(dict(tsdf=True, reso=a.reso, reso_level=a.reso_level, trunc=a.trunc, crop=a.crop, crop_invert=a.crop_invert,
                              total_s=t, verts=int(mesh.verts.shape[0]), faces=int(mesh.faces.shape[0]), gpu=props.name, out=a.out)))
        return
    level = G.level_from_alpha(r, a.alpha)

    G.DensityGrid(r, lo, hi, reso=16, crop=crop)                                # warm-up: module load, shadow table, allocator
    grids, t_grid = zip(*(timed(lambda: G.DensityGrid(r, lo, hi, reso=a.reso, crop=crop)) for _ in range(a.repeat)))
    g = grids[-1]
    del grids
    meshes, t_iso = zip(*(timed(lambda: G.Isosurface(g.logit, level, g.origin, g.voxel)) for _ in range(a.repeat)))
    verts, faces = meshes[-1]
    del meshes
    n_pts = g.logit.numel()
    del g
    normals, t_nrm = timed(lambda: G.QueryNormal(r, verts)) if a.normals else (None, 0.)
    colors, t_col = timed(lambda: G.VertexColors(r, verts, faces, normals))
    mesh = G.Mesh(verts, faces, colors, normals).to_data_frame(scene.dataset)
    G.write_ply(a.out, mesh)
    med = lambda x: sorted(x)[len(x) // 2]
    print(json.dumps(dict(reso=a.reso, alpha=a.alpha, crop=a.crop, crop_invert=a.crop_invert, level=level, lattice_points=n_pts, grid_query_s=med(t_grid),
                          grid_points_per_s=n_pts / med(t_grid), extract_s=med(t_iso), colors_s=t_col, normals_s=t_nrm, verts=int(verts.shape[0]),
                          faces=int(faces.shape[0]), gpu=props.name, out=a.out)))


if __name__ == "__main__":
    main()
