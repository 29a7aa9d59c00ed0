"""Extract a trained scene's surface as a coloured PLY mesh on the device.

    python scripts/extract_mesh.py <runtime_config.yaml> <checkpoint_dir> [--reso 512] [--alpha 0.5]
                                   [--bbox x0 y0 z0 x1 y1 z1] --out scene.ply

load_scene -> DensityGrid -> Isosurface -> VertexColors (f2nerf_b200/geometry.py); the mesh is written in the data's own world
frame (Mesh.to_data_frame).  --bbox is in the normalised scene frame (default: the valid leaves' bounding box).  Prints one
JSON line: lattice size, grid-query time and rate, extraction time, colour time, vertex and face counts, and the GPU.
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
    ap.add_argument("--normals", action="store_true", help="field normals on the vertices (written as nx ny nz; colours seen along them)")
    ap.add_argument("--repeat", type=int, default=1, help="time the grid query and the extraction this many times (median)")
    a = ap.parse_args(argv)

    import torch
    from f2nerf_b200 import geometry as G, load_scene

    scene = load_scene(a.config, a.checkpoint_dir, device="cuda")
    r = scene.renderer
    lo, hi = (a.bbox[:3], a.bbox[3:]) if a.bbox else (None, None)
    level = G.level_from_alpha(r, a.alpha)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0

    G.DensityGrid(r, lo, hi, reso=16)                                # warm-up: module load, shadow table, allocator
    grids, t_grid = zip(*(timed(lambda: G.DensityGrid(r, lo, hi, reso=a.reso)) for _ in range(a.repeat)))
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
    props = torch.cuda.get_device_properties(0)
    print(json.dumps(dict(reso=a.reso, alpha=a.alpha, level=level, lattice_points=n_pts, grid_query_s=med(t_grid),
                          grid_points_per_s=n_pts / med(t_grid), extract_s=med(t_iso), colors_s=t_col, normals_s=t_nrm, verts=int(verts.shape[0]),
                          faces=int(faces.shape[0]), gpu=props.name, out=a.out)))


if __name__ == "__main__":
    main()
