"""A trained scene's geometry on the device: its density at world points and its surface as a coloured triangle mesh.

Everything works in the renderer's normalised scene frame (``NormalizeScene``: world = x * radius_ + center_) and reads the
renderer's objects without changing them.  A point is taken through the same pieces the ray march uses: the
perspective-warp octree (the leaf that holds it, ``f2b_locate_points``), its leaf's warp, the anchored hash grid and the
field MLP (``f2b_query_logit_points`` / ``f2b_query_logit_grid``: one fused kernel).  Points that no valid leaf holds get
the logit ``EMPTY_LOGIT``, so their density ``exp(logit - 3)`` is exactly 0.

The surface is a level set of the density logit on a lattice, extracted by marching tetrahedra (``Isosurface``): closed and
consistently oriented by construction, outward towards lower density.  DESIGN.md §3i has the details and the parity anchors.

Surface normals (DESIGN.md §3j) come from the density itself: ``QueryGradient`` returns g = d logit / d x at world points (one
kernel: the field query's forward, the field MLP's backward on the tensor pipe, the hash-grid blend's derivative and the leaf
warp's Jacobian), ``QueryNormal`` the outward normal -g / |g|.
"""
import math
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import ops
from ._lib import call, stream
from .octree_build import TREE_NODE

EMPTY_LOGIT = -1e4          # logit of a point outside every valid leaf: finite, and exp(EMPTY_LOGIT - 3) == 0 in fp32
SLAB_POINTS = 1 << 23       # Isosurface: owner points per z-slab; scratch <= 25 B x (SLAB_POINTS + one layer), ~210 MB
GRID_SLAB_POINTS = 1 << 30  # DensityGrid: lattice points per kernel launch (the kernel indexes a slab with int32)


class Grid(NamedTuple):
    """A logit lattice: ``logit`` [nz, ny, nx] fp32 on the device, lattice point (i, j, k) at origin + voxel * (i, j, k)."""
    logit: torch.Tensor
    origin: tuple
    voxel: tuple


class Mesh(NamedTuple):
    """``verts`` [V,3] fp32, ``faces`` [F,3] int32 (outward = towards lower density), ``colors`` [V,3] fp32 in [0, 1] or
    None; on the device, in the frame the mesh was made in."""
    verts: torch.Tensor
    faces: torch.Tensor
    colors: Optional[torch.Tensor] = None
    normals: Optional[torch.Tensor] = None

    def to_data_frame(self, dataset):
        """The mesh in the data's own world frame: x * radius_ + center_ (undoes ``load_dataset``'s normalisation).  The frames
        differ by a uniform scale and a translation, so the normals carry over unchanged."""
        center = torch.as_tensor(dataset.center_, dtype=torch.float32, device=self.verts.device)
        return Mesh(self.verts * float(dataset.radius_) + center, self.faces, self.colors, self.normals)


def _octree(renderer):
    s = renderer.pts_sampler_
    return s.tree_nodes_gpu_, s.pers_trans_gpu_


def _field_args(renderer):
    f = renderer.scene_field_
    return f.table_f16(), f.prim_pool_, f.bias_pool_, f.n_volumes_, f.local_size_, f.mlp_.params_f16()


def _points(pts, renderer):
    dev = renderer.pts_sampler_.tree_nodes_gpu_.device
    pts = torch.as_tensor(pts, dtype=torch.float32, device=dev).reshape(-1, 3).contiguous()
    return pts


def LocatePoints(renderer, pts):
    """World points [n,3] -> (warped [n,3], anchors [n,2] int32 = (trans_idx, leaf node)), both as the march would give them
    for a sample at that point; (-1, -1) and warped 0 where no valid leaf holds the point."""
    nodes, trans = _octree(renderer)
    return ops.locate_points(nodes, trans, _points(pts, renderer))


def QueryLogit(renderer, pts):
    """Density logit (field output channel 0) at world points [n,3]; ``EMPTY_LOGIT`` where no valid leaf holds the point."""
    nodes, trans = _octree(renderer)
    return ops.query_logit_points(nodes, trans, *_field_args(renderer), _points(pts, renderer), EMPTY_LOGIT)


def QueryDensity(renderer, pts):
    """Density at world points [n,3]: the renderer's density activation exp(logit - 3) (Renderer.cpp:100-103); 0 where no valid
    leaf holds the point.  The density is per unit of warped length, the quantity the renderer integrates along a ray."""
    return torch.exp(QueryLogit(renderer, pts) - 3.)


def QueryGradient(renderer, pts):
    """(logit [n], grad [n,3]) at world points [n,3]: the logit of ``QueryLogit`` (same bits) and its gradient d logit / d x in
    the normalised scene frame (DESIGN.md §3j); ``EMPTY_LOGIT`` and a zero gradient where no valid leaf holds the point."""
    nodes, trans = _octree(renderer)
    return ops.query_grad_points(nodes, trans, *_field_args(renderer), _points(pts, renderer), EMPTY_LOGIT)


def unit_normals(grad):
    """-g / |g| per row of [n,3] (the outward normal, towards lower density); 0 where g = 0."""
    n = torch.linalg.norm(grad, dim=1, keepdim=True)
    return torch.where(n > 0, -grad / n.clamp_min(1e-38), torch.zeros_like(grad))


def QueryNormal(renderer, pts):
    """Outward unit normals [n,3] of the density at world points [n,3]: -g / |g| of ``QueryGradient``; 0 where the gradient is
    0 or no valid leaf holds the point."""
    return unit_normals(QueryGradient(renderer, pts)[1])


def QueryColor(renderer, pts, dirs):
    """Colour [n,3] of world points [n,3] seen along unit directions ``dirs`` [n,3] (the way a ray travels), without the
    appearance embedding, as the renderer's VALIDATE mode shades; 0 where no valid leaf holds the point."""
    pts = _points(pts, renderer)
    dirs = torch.as_tensor(dirs, dtype=torch.float32, device=pts.device).reshape(-1, 3).contiguous()
    warped, anchors = LocatePoints(renderer, pts)
    rows = torch.nonzero(anchors[:, 0] >= 0).squeeze(1)
    rgb = torch.zeros_like(pts)
    n = int(rows.numel())
    if n == 0:
        return rgb
    table16, prim, bias, n_volumes, local_size, fparams = _field_args(renderer)
    _, feat, _ = ops.field_fwd(table16, prim, bias, n_volumes, local_size, fparams, warped[rows].contiguous(),
                               anchors[rows, 0].contiguous(), 1, logit_only=True, save_feat=True)
    d = dirs[rows].contiguous()
    logit = torch.empty((n,), dtype=torch.float32, device=pts.device)
    mlp_in = torch.empty((n, 32), dtype=torch.float16, device=pts.device)
    call("f2b_field_shade_fwd", feat, fparams, d, None, None, n, logit, mlp_in, None, stream())
    raw = torch.empty((n, 16), dtype=torch.float16, device=pts.device)
    out = torch.empty((n, 3), dtype=torch.float32, device=pts.device)
    call("f2b_shader_mlp_rgb_fwd", mlp_in, renderer.shader_.mlp_.params_f16(), n, raw, out, None, stream())
    rgb[rows] = out
    return rgb


def leaf_bounds(renderer):
    """(min, max) corners of the bounding box of the octree's valid leaves (trans_idx >= 0, no live child)."""
    nodes = renderer.pts_sampler_.tree_nodes_gpu_.cpu().numpy().view(TREE_NODE)
    leaf = (nodes["trans_idx"] >= 0) & (nodes["childs"] < 0).all(1)
    if not leaf.any():
        raise ValueError("leaf_bounds: the octree has no valid leaf")
    c, h = nodes["center"][leaf], (nodes["side_len"][leaf] * np.float32(.5))[:, None]
    return tuple(float(x) for x in (c - h).min(0)), tuple(float(x) for x in (c + h).max(0))


def DensityGrid(renderer, bbox_min=None, bbox_max=None, reso=256):
    """The density logit on a lattice over the box [bbox_min, bbox_max] (default: ``leaf_bounds``) with cubic voxels, ``reso``
    points along the box's longest axis -> ``Grid``.  The lattice points are generated in the kernel, in z-slabs."""
    if bbox_min is None or bbox_max is None:
        lo, hi = leaf_bounds(renderer)
        bbox_min = lo if bbox_min is None else bbox_min
        bbox_max = hi if bbox_max is None else bbox_max
    lo, hi = np.asarray(bbox_min, np.float64).reshape(3), np.asarray(bbox_max, np.float64).reshape(3)
    ext = hi - lo
    if int(reso) < 2 or not (ext > 0).all():
        raise ValueError("DensityGrid: reso must be >= 2 and the box must have a positive extent on every axis")
    voxel = float(np.float32(ext.max() / (int(reso) - 1)))
    nx, ny, nz = (min(int(reso), int(math.ceil(e / voxel - 1e-6)) + 1) for e in ext)
    origin = tuple(float(np.float32(v)) for v in lo)
    nodes, trans = _octree(renderer)
    fargs = _field_args(renderer)
    logit = torch.empty((nz, ny, nx), dtype=torch.float32, device=nodes.device)
    step = max(1, GRID_SLAB_POINTS // (nx * ny))
    for z0 in range(0, nz, step):
        n = min(step, nz - z0)
        ops.query_logit_grid(nodes, trans, *fargs, origin, (voxel,) * 3, nx, ny, z0, n, EMPTY_LOGIT, logit[z0:z0 + n])
    return Grid(logit, origin, (voxel,) * 3)


def level_from_alpha(renderer, alpha):
    """The logit level whose density gives opacity ``alpha`` over one VALIDATE march step, sample_l * fineness in warp units
    (alpha = 1 - exp(-sigma * dt)): sigma = -ln(1 - alpha) / (sample_l * fineness), logit = ln(sigma) + 3."""
    if not 0. < float(alpha) < 1.:
        raise ValueError("level_from_alpha: alpha must lie in (0, 1)")
    dt = renderer.pts_sampler_.sample_l_ * renderer.global_data_pool_.ray_march_fineness_
    return math.log(-math.log1p(-float(alpha)) / dt) + 3.


def Isosurface(logit, level, origin=(0., 0., 0.), voxel=(1., 1., 1.), empty_logit=EMPTY_LOGIT, slab_points=SLAB_POINTS):
    """The surface {logit = level} of a lattice ``logit`` [nz, ny, nx] (fp32, device) by marching tetrahedra -> (verts [V,3] fp32,
    faces [F,3] int32), outward towards lower logits; lattice points outside the lattice read ``empty_logit`` (<= level), so
    the surface is closed.  Vertices are ordered by (lattice point, edge direction), faces by (cell, tetrahedron, triangle);
    the result does not depend on ``slab_points``, which bounds the scratch (25 B per owner point of a slab)."""
    if logit.dim() != 3 or logit.dtype != torch.float32 or not logit.is_cuda:
        raise ValueError("Isosurface: logit must be a [nz, ny, nx] float32 CUDA tensor")
    if not float(empty_logit) <= float(np.float32(level)):
        raise ValueError("Isosurface: empty_logit must not be above the level")
    logit = logit.contiguous()
    nz, ny, nx = logit.shape
    per_layer = (nx + 1) * (ny + 1)
    layers = max(1, int(slab_points) // per_layer - 1)
    dev = logit.device
    mask = torch.empty(((layers + 1) * per_layer,), dtype=torch.uint8, device=dev)
    vcnt = torch.empty(((layers + 1) * per_layer,), dtype=torch.int32, device=dev)
    tcnt = torch.empty((layers * per_layer,), dtype=torch.int32, device=dev)
    verts, faces, vbase = [], [], 0
    for ez0 in range(0, nz + 1, layers):
        ez1 = min(ez0 + layers, nz + 1)
        n_pt, n_cell = (min(ez1 + 1, nz + 1) - ez0) * per_layer, (ez1 - ez0) * per_layer
        ops.iso_count(logit, level, empty_logit, ez0, ez1, mask, vcnt, tcnt)
        vb, _ = ops.count_scan(vcnt, n_pt)
        tb, tt = ops.count_scan(tcnt, n_cell)
        nv, nf = (int(x) for x in torch.stack([vb[n_cell - 1, 1], tt[0]]).tolist())
        v = torch.empty((nv, 3), dtype=torch.float32, device=dev)
        f = torch.empty((nf, 3), dtype=torch.int32, device=dev)
        ops.iso_emit(logit, level, empty_logit, origin, voxel, ez0, ez1, vbase, mask, vb, tb, v, f)
        verts.append(v)
        faces.append(f)
        vbase += nv
    return torch.cat(verts), torch.cat(faces)


def vertex_normals(verts, faces):
    """Area-weighted vertex normals (unnormalised sums of the incident faces' cross products)."""
    f = faces.long()
    v0, v1, v2 = verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]]
    fn = torch.linalg.cross(v1 - v0, v2 - v0)
    n = torch.zeros_like(verts)
    for k in range(3):
        n.index_add_(0, f[:, k], fn)
    return n


def VertexColors(renderer, verts, faces, normals=None):
    """Colour of each vertex seen from outside along its normal: ``QueryColor`` with view direction -n / |n|.  By default n is
    the area-weighted face normal (``vertex_normals``: sums of float atomics, so a colour can differ by an ulp from run to run);
    ``normals`` [V,3] (unit or 0, e.g. ``QueryNormal``) replaces it wherever it is non-zero."""
    n = vertex_normals(verts, faces)
    if normals is not None:
        n = torch.where((normals != 0).any(1, keepdim=True), normals, n)
    d = -n / torch.linalg.norm(n, dim=1, keepdim=True).clamp_min(1e-30)
    return QueryColor(renderer, verts, d)


def ExtractMesh(renderer, bbox_min=None, bbox_max=None, reso=512, alpha=0.5, density=None, colors=True, normals=False):
    """The scene's surface as a ``Mesh`` on the device, in the normalised frame (``Mesh.to_data_frame`` maps it back).
    The level is the density that reaches opacity ``alpha`` over one VALIDATE march step (``level_from_alpha``), or
    ``density`` (per warp unit) when given; the lattice is ``DensityGrid(renderer, bbox_min, bbox_max, reso)``.
    ``normals``: the vertices get the field's normals (``QueryNormal``), and the colours are seen along them (the face normal
    where the field normal is 0)."""
    level = math.log(float(density)) + 3. if density is not None else level_from_alpha(renderer, alpha)
    g = DensityGrid(renderer, bbox_min, bbox_max, reso)
    verts, faces = Isosurface(g.logit, level, g.origin, g.voxel)
    del g
    nrm = QueryNormal(renderer, verts) if normals else None
    rgb = VertexColors(renderer, verts, faces, nrm) if colors and verts.shape[0] else None
    return Mesh(verts, faces, rgb, nrm)


def write_ply(path, mesh):
    """Binary little-endian PLY: float x, y, z (+ float nx, ny, nz when the mesh has normals, + uchar red, green, blue when it
    has colours) and uchar-counted int triangle lists."""
    v = mesh.verts.detach().cpu().numpy().astype("<f4")
    f = mesh.faces.detach().cpu().numpy().astype("<i4")
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if mesh.normals is not None:
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
    if mesh.colors is not None:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    vr = np.empty(len(v), fields)
    vr["x"], vr["y"], vr["z"] = v[:, 0], v[:, 1], v[:, 2]
    if mesh.normals is not None:
        nm = mesh.normals.detach().cpu().numpy().astype("<f4")
        vr["nx"], vr["ny"], vr["nz"] = nm[:, 0], nm[:, 1], nm[:, 2]
    if mesh.colors is not None:
        c = np.clip(np.rint(mesh.colors.detach().cpu().numpy() * 255.), 0, 255).astype(np.uint8)
        vr["red"], vr["green"], vr["blue"] = c[:, 0], c[:, 1], c[:, 2]
    fr = np.empty(len(f), [("n", "u1"), ("v", "<i4", (3,))])
    fr["n"], fr["v"] = 3, f
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}", "property float x", "property float y",
            "property float z"]
    if mesh.normals is not None:
        head += ["property float nx", "property float ny", "property float nz"]
    if mesh.colors is not None:
        head += ["property uchar red", "property uchar green", "property uchar blue"]
    head += [f"element face {len(f)}", "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as out:
        out.write(("\n".join(head) + "\n").encode("ascii"))
        out.write(vr.tobytes())
        out.write(fr.tobytes())
