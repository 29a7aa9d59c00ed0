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

A point cloud (DESIGN.md §3l) samples the surface where the views see it rather than on a lattice, so it keeps the detail of an
unbounded scene near and far: ``ExtractPointCloud`` renders every view on a grid, puts a point at each opaque pixel's median
sample (``eval.RenderDepth``'s termination kernel), coloured by the pixel's foreground colour, and keeps the points whose depth
the other views confirm (``f2b_depth_consistency``).

A crop box (``crop.Crop``, DESIGN.md §3n) restricts the lattice, the mesh and the point cloud to what the box keeps: lattice points
it does not keep read ``EMPTY_LOGIT``, so the mesh stays closed and caps the cut, and the point cloud's renders are cropped.
"""
import math
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import ops
from ._lib import call, stream
from .crop import resolve_crop
from .eval import resolve_appearance
from .octree_build import TREE_NODE

EMPTY_LOGIT = -1e4          # logit of a point outside every valid leaf: finite, and exp(EMPTY_LOGIT - 3) == 0 in fp32
SLAB_POINTS = 1 << 23       # Isosurface: owner points per z-slab; scratch <= 25 B x (SLAB_POINTS + one layer), ~210 MB
GRID_SLAB_POINTS = 1 << 30  # DensityGrid: lattice points per kernel launch (the kernel indexes a slab with int32)
CROP_MASK_POINTS = 1 << 24  # DensityGrid(crop=): lattice points masked per f2b_crop_mask launch (12 B of points each)


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


class PointCloud(NamedTuple):
    """``points`` [P,3] fp32, ``colors`` [P,3] fp32 in [0, 1], ``normals`` [P,3] fp32 (unit or 0) or None, ``source`` [P,2] int32
    (dataset view, grid cell a * w + b of the view's h x w grid); on the device, in the frame the cloud was made in."""
    points: torch.Tensor
    colors: torch.Tensor
    normals: Optional[torch.Tensor]
    source: torch.Tensor

    def to_data_frame(self, dataset):
        """The cloud in the data's own world frame: x * radius_ + center_, as ``Mesh.to_data_frame``; normals carry over."""
        center = torch.as_tensor(dataset.center_, dtype=torch.float32, device=self.points.device)
        return PointCloud(self.points * float(dataset.radius_) + center, self.colors, self.normals, self.source)


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


def QueryColor(renderer, pts, dirs, appearance=None):
    """Colour [n,3] of world points [n,3] seen along unit directions ``dirs`` [n,3] (the way a ray travels); 0 where no valid
    leaf holds the point.  ``appearance`` (``Renderer.appearance_row``): None shades without the appearance embedding, as the
    renderer's VALIDATE mode does; a training image's index or a [16] row is added to the shader input (DESIGN.md §3m)."""
    app = resolve_appearance(renderer, appearance)
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
    emb = (app[None], torch.zeros((n,), dtype=torch.int32, device=pts.device)) if app is not None else (None, None)
    call("f2b_field_shade_fwd", feat, fparams, d, *emb, n, logit, mlp_in, None, stream())
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


def _crop_lattice(crop, logit, origin, voxel, z0):
    """Lattice layers [z0, z0 + nz) of ``logit`` [nz, ny, nx] read ``EMPTY_LOGIT`` where ``crop`` does not keep the lattice point
    origin + voxel * (i, j, k), formed as the grid kernel forms it: fadd(origin, fmul(voxel, i)) per axis (one fp32 op each)."""
    nz, ny, nx = logit.shape
    dev = logit.device
    o = [torch.tensor(float(x), dtype=torch.float32, device=dev) for x in origin]
    v = [torch.tensor(float(x), dtype=torch.float32, device=dev) for x in voxel]
    axis = lambda a, n, i0: o[a] + v[a] * torch.arange(i0, i0 + n, dtype=torch.float32, device=dev)
    xs, ys = axis(0, nx, 0), axis(1, ny, 0)
    layers = max(1, CROP_MASK_POINTS // (nx * ny))
    for k0 in range(0, nz, layers):
        n = min(layers, nz - k0)
        zs = axis(2, n, z0 + k0)
        pts = torch.stack([xs.expand(n, ny, nx), ys[:, None].expand(n, ny, nx), zs[:, None, None].expand(n, ny, nx)], -1)
        logit[k0:k0 + n].masked_fill_(~crop.mask(pts).view(n, ny, nx), EMPTY_LOGIT)


def DensityGrid(renderer, bbox_min=None, bbox_max=None, reso=256, crop=None):
    """The density logit on a lattice over the box [bbox_min, bbox_max] (default: ``leaf_bounds``) with cubic voxels, ``reso``
    points along the box's longest axis -> ``Grid``.  The lattice points are generated in the kernel, in z-slabs.
    ``crop``: a ``Crop``; lattice points it does not keep read ``EMPTY_LOGIT`` (its predicate, ``f2b_crop_mask``, over each slab's
    points), and when the box is not given and the crop is not inverted it defaults to ``crop.aabb()`` within ``leaf_bounds``."""
    crop = resolve_crop(crop)
    if bbox_min is None or bbox_max is None:
        lo, hi = leaf_bounds(renderer)
        if crop is not None and not crop.invert:
            clo, chi = crop.aabb()
            lo, hi = tuple(max(a, b) for a, b in zip(lo, clo)), tuple(min(a, b) for a, b in zip(hi, chi))
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
        if crop is not None:
            _crop_lattice(crop, logit[z0:z0 + n], origin, (voxel,) * 3, z0)
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


def VertexColors(renderer, verts, faces, normals=None, appearance=None):
    """Colour of each vertex seen from outside along its normal: ``QueryColor`` with view direction -n / |n|.  By default n is
    the area-weighted face normal (``vertex_normals``: sums of float atomics, so a colour can differ by an ulp from run to run);
    ``normals`` [V,3] (unit or 0, e.g. ``QueryNormal``) replaces it wherever it is non-zero.  ``appearance``: as ``QueryColor``."""
    n = vertex_normals(verts, faces)
    if normals is not None:
        n = torch.where((normals != 0).any(1, keepdim=True), normals, n)
    d = -n / torch.linalg.norm(n, dim=1, keepdim=True).clamp_min(1e-30)
    return QueryColor(renderer, verts, d, appearance)


def ExtractMesh(renderer, bbox_min=None, bbox_max=None, reso=512, alpha=0.5, density=None, colors=True, normals=False,
                appearance=None, crop=None):
    """The scene's surface as a ``Mesh`` on the device, in the normalised frame (``Mesh.to_data_frame`` maps it back).
    The level is the density that reaches opacity ``alpha`` over one VALIDATE march step (``level_from_alpha``), or
    ``density`` (per warp unit) when given; the lattice is ``DensityGrid(renderer, bbox_min, bbox_max, reso)``.
    ``normals``: the vertices get the field's normals (``QueryNormal``), and the colours are seen along them (the face normal
    where the field normal is 0).  ``appearance``: the colours' appearance row, as ``QueryColor``.  ``crop``: a ``Crop``
    (``DensityGrid``): the surface of what the box keeps, closed where the box cuts it."""
    app = resolve_appearance(renderer, appearance)               # argument errors before the lattice is built
    level = math.log(float(density)) + 3. if density is not None else level_from_alpha(renderer, alpha)
    g = DensityGrid(renderer, bbox_min, bbox_max, reso, crop)
    verts, faces = Isosurface(g.logit, level, g.origin, g.voxel)
    del g
    nrm = QueryNormal(renderer, verts) if normals else None
    rgb = VertexColors(renderer, verts, faces, nrm, app) if colors and verts.shape[0] else None
    return Mesh(verts, faces, rgb, nrm)


def ExtractPointCloud(renderer, dataset, views=None, reso_level=1, min_opacity=0.9, min_views=2, rel_tol=0.01, normals=False,
                      appearance=None, crop=None):
    """The scene's surface as a coloured ``PointCloud`` on the device, in the normalised frame (``to_data_frame`` maps it back).
    Pass 1, per view of ``views`` (default ``dataset.train_set_``): the VALIDATE render of the view's own camera on the
    (height // reso_level) x (width // reso_level) grid, with a black background, and the termination kernel on its slots (as
    ``eval.RenderDepth``).  Every pixel with opacity W >= ``min_opacity`` gives a candidate: the world point of its median sample,
    the colour C / W (the composite without background over the opacity, clipped to [0, 1]), with ``normals`` the pixel's normal
    (as ``eval.RenderNormals``).  Pass 2, when ``min_views`` > 0: every candidate is projected into every other view of ``views``
    (``f2b_depth_consistency``) and kept when at least ``min_views`` of them see an opaque pixel (opacity >= ``min_opacity``)
    whose median depth is within ``rel_tol`` of the point's distance.  Points are ordered by (position of the view in ``views``,
    cell); a run gives the same bits every time.  One host sync per view.  ``appearance`` colours the points
    (``Renderer.appearance_row``): None, a training image's index, a [16] row, or ``"own"``: each view's own row.  The points
    themselves do not depend on it (weights and density do not).  ``crop``: a ``Crop``; every render is cropped (DESIGN.md §3n), so
    the candidates and the consistency pass see only what the box keeps."""
    from .eval import RAY_BATCH_SIZE, _slot_chunks, _Validate
    crop = resolve_crop(crop)
    views = [int(v) for v in (dataset.train_set_ if views is None else views)]
    reso_level, min_views = int(reso_level), int(min_views)
    if not views:
        raise ValueError("ExtractPointCloud: no views")
    if reso_level < 1:
        raise ValueError("ExtractPointCloud: reso_level must be >= 1")
    if not 0. < float(min_opacity) <= 1.:
        raise ValueError("ExtractPointCloud: min_opacity must lie in (0, 1]")
    if not 0 <= min_views <= len(views) - 1:
        raise ValueError(f"ExtractPointCloud: min_views {min_views} outside [0, {len(views) - 1}] (the other views of {len(views)})")
    if not float(rel_tol) >= 0.:
        raise ValueError("ExtractPointCloud: rel_tol must be >= 0")
    apps = [resolve_appearance(renderer, appearance, view=b) for b in views]
    H, W = dataset.height_, dataset.width_
    h, w = H // reso_level, W // reso_level
    if h < 2 or w < 2:
        raise ValueError(f"ExtractPointCloud: reso_level {reso_level} leaves a {h} x {w} grid of a {H} x {W} image")
    n = h * w
    dev = dataset.poses_.device
    f = renderer.scene_field_
    trans = renderer.pts_sampler_.pers_trans_gpu_
    black = torch.zeros((3,), dtype=torch.float32, device=dev)
    f32 = lambda *sh: torch.empty(sh, dtype=torch.float32, device=dev)
    maps, pts, cols, nrms, srcs = [], [], [], [], []
    with torch.no_grad(), _Validate(renderer):
        for b, app in zip(views, apps):
            o, d = dataset._camera_rays(dataset.poses_[b], dataset.intri_[b], dataset.dist_params_[b], h, w)
            opa, med, point, rgb = f32(n), f32(n), f32(n, 3), f32(n, 3)
            nm = f32(n, 3) if normals else None

            def each(r, i, j):
                ops.ray_termination_slots(r._keep[0], r.kept_counts, r._w_slots, opacity=opa[i:j], median_t=med[i:j], point=point[i:j])
                if normals:
                    ops.render_normals_slots(trans, f.table_f16(), f.prim_pool_, f.bias_pool_, f.n_volumes_, f.local_size_,
                                             f.mlp_.params_f16(), r._keep[0], r.kept_counts, r._w_slots, out=nm[i:j])

            _slot_chunks(renderer, o, d, RAY_BATCH_SIZE, dev, each, out=(rgb, f32(n), f32(n)), bg=black, app=app, crop=crop)
            cell = torch.nonzero(opa >= float(min_opacity)).squeeze(1)            # the host sync of the view; cells ascending
            maps.append((opa, med))
            pts.append(point[cell])
            cols.append((rgb[cell] / opa[cell, None]).clamp_(0., 1.))
            nrms.append(nm[cell] if normals else None)
            srcs.append(torch.stack([torch.full_like(cell, b), cell], 1).to(torch.int32))
        points, colors, source = torch.cat(pts), torch.cat(cols), torch.cat(srcs)
        nrm = torch.cat(nrms) if normals else None
        if min_views > 0 and points.shape[0] > 0:
            count = torch.zeros((points.shape[0],), dtype=torch.int32, device=dev)
            src_view = source[:, 0].contiguous()
            for b, (opa, med) in zip(views, maps):
                ops.depth_consistency(points, src_view, b, dataset.poses_[b], dataset.intri_[b], dataset.dist_params_[b], H, W, h, w,
                                      opa, med, min_opacity, rel_tol, count)
            keep = count >= min_views
            points, colors, source = points[keep], colors[keep], source[keep]
            nrm = nrm[keep] if normals else None
    return PointCloud(points, colors, nrm, source)


def write_ply(path, mesh):
    """Binary little-endian PLY of a ``Mesh`` or a ``PointCloud``: float x, y, z (+ float nx, ny, nz when it has normals, + uchar
    red, green, blue when it has colours) and, for a mesh, uchar-counted int triangle lists (a point cloud has no face element)."""
    cloud = isinstance(mesh, PointCloud)
    v = (mesh.points if cloud else mesh.verts).detach().cpu().numpy().astype("<f4")
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
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}", "property float x", "property float y",
            "property float z"]
    if mesh.normals is not None:
        head += ["property float nx", "property float ny", "property float nz"]
    if mesh.colors is not None:
        head += ["property uchar red", "property uchar green", "property uchar blue"]
    if not cloud:
        f = mesh.faces.detach().cpu().numpy().astype("<i4")
        fr = np.empty(len(f), [("n", "u1"), ("v", "<i4", (3,))])
        fr["n"], fr["v"] = 3, f
        head += [f"element face {len(f)}", "property list uchar int vertex_indices"]
    head += ["end_header"]
    with open(path, "wb") as out:
        out.write(("\n".join(head) + "\n").encode("ascii"))
        out.write(vr.tobytes())
        if not cloud:
            out.write(fr.tobytes())
