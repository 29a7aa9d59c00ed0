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

A TSDF mesh (DESIGN.md §3p) meshes the surface the views' median depths agree on rather than a density level: ``FuseTSDF``
averages, per lattice point, the truncated signed distances to the depth maps of the views that see it (``f2b_tsdf_integrate``),
``TSDFSurface`` extracts their zero level set over the observed lattice points and colours it (``f2b_tsdf_colors``), and
``ExtractTSDFMesh`` renders the maps of the training views (``ExtractPointCloud``'s pass 1) and does both.

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
TSDF_SLAB_POINTS = 1 << 30  # FuseTSDF: lattice points per kernel launch (the kernel indexes a slab with int32)


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


class TSDFGrid(NamedTuple):
    """The sums of a TSDF fusion (DESIGN.md §3p), fp32 on the device: ``sdf_sum`` and ``weight`` [nz, ny, nx], ``color_sum``
    [nz, ny, nx, 3]; lattice point (i, j, k) at origin + voxel * (i, j, k), ``voxel`` one float (cubic voxels)."""
    sdf_sum: torch.Tensor
    weight: torch.Tensor
    color_sum: torch.Tensor
    origin: tuple
    voxel: float


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


def _lattice(bbox_min, bbox_max, reso, who):
    """(origin, voxel, (nx, ny, nz)) of the lattice over [bbox_min, bbox_max] with cubic voxels, ``reso`` points along the box's
    longest axis; origin and voxel rounded to fp32."""
    lo, hi = np.asarray(bbox_min, np.float64).reshape(3), np.asarray(bbox_max, np.float64).reshape(3)
    ext = hi - lo
    if int(reso) < 2 or not (ext > 0).all():
        raise ValueError(f"{who}: reso must be >= 2 and the box must have a positive extent on every axis")
    voxel = float(np.float32(ext.max() / (int(reso) - 1)))
    shape = tuple(min(int(reso), int(math.ceil(e / voxel - 1e-6)) + 1) for e in ext)
    return tuple(float(np.float32(v)) for v in lo), voxel, shape


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
    origin, voxel, (nx, ny, nz) = _lattice(bbox_min, bbox_max, reso, "DensityGrid")
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


def _view_maps(renderer, dataset, views, h, w, apps, crop, normals=False):
    """Pass 1 of ``ExtractPointCloud`` and ``ExtractTSDFMesh``: per view of ``views`` (with its appearance row of ``apps``), the
    VALIDATE render of the view's own camera on the h x w grid with a black background, cropped by ``crop``, and the termination
    kernel (with ``normals`` the normals kernel) on its slots -> yields (opacity [n], median_t [n], point [n,3], rgb [n,3],
    normals [n,3] or None), n = h * w.  The caller holds ``torch.no_grad()`` and ``eval._Validate(renderer)``."""
    from .eval import RAY_BATCH_SIZE, _slot_chunks
    n = h * w
    dev = dataset.poses_.device
    f = renderer.scene_field_
    trans = renderer.pts_sampler_.pers_trans_gpu_
    black = torch.zeros((3,), dtype=torch.float32, device=dev)
    f32 = lambda *sh: torch.empty(sh, dtype=torch.float32, device=dev)
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
        yield opa, med, point, rgb, nm


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
    from .eval import _Validate
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
    dev = dataset.poses_.device
    maps, pts, cols, nrms, srcs = [], [], [], [], []
    with torch.no_grad(), _Validate(renderer):
        for b, (opa, med, point, rgb, nm) in zip(views, _view_maps(renderer, dataset, views, h, w, apps, crop, normals)):
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


def _tsdf_args(trunc, min_opacity, who):
    if not (math.isfinite(float(trunc)) and float(trunc) > 0.):
        raise ValueError(f"{who}: trunc must be finite and > 0")
    if not 0. < float(min_opacity) <= 1.:
        raise ValueError(f"{who}: min_opacity must lie in (0, 1]")


def FuseTSDF(poses, intri, dist_params, height, width, opacity, median_t, colors, bbox_min, bbox_max, reso=512, trunc=4., min_opacity=0.9):
    """TSDF fusion of V views' depth maps into a lattice over [bbox_min, bbox_max] (cubic voxels, ``reso`` points along the
    longest axis, as ``DensityGrid``) -> ``TSDFGrid`` (DESIGN.md §3p).  View v: camera ``poses[v]`` [3,4] camera-to-world,
    ``intri[v]`` [3,3], ``dist_params[v]`` (k1, k2, p1, p2) of a ``height`` x ``width`` image, and its maps on the h x w grid
    ``f2b_camera_rays`` renders: ``opacity`` and ``median_t`` (along the unit ray) [V,h,w], ``colors`` [V,h,w,3] (fp32 CUDA tensors).
    Per lattice point and view, in view order: where the point projects into the grid (``f2b_depth_consistency``'s projection) on
    a pixel with opacity >= ``min_opacity`` and sdf = median_t - |p - o| >= -mu, mu = fp32(trunc * voxel): sdf_sum += min(1, sdf
    / mu), weight += 1, color_sum += the pixel's colour.  The views go through ``f2b_tsdf_integrate`` in groups of
    ``ops.TSDF_MAX_VIEWS``; the bits do not depend on the grouping."""
    if not (isinstance(opacity, torch.Tensor) and opacity.dim() == 3):
        raise ValueError("FuseTSDF: opacity must be a [V, h, w] tensor")
    V, h, w = opacity.shape
    shapes = ((poses, (V, 3, 4), "poses"), (intri, (V, 3, 3), "intri"), (dist_params, (V, 4), "dist_params"),
              (median_t, (V, h, w), "median_t"), (colors, (V, h, w, 3), "colors"))
    for t, shape, name in shapes:
        if tuple(torch.as_tensor(t).shape) != shape:
            raise ValueError(f"FuseTSDF: {name} has shape {tuple(torch.as_tensor(t).shape)}, expected {shape}")
    if V < 1 or not (2 <= h <= int(height) and 2 <= w <= int(width)):
        raise ValueError(f"FuseTSDF: {V} views of a {h} x {w} grid of a {height} x {width} image")
    _tsdf_args(trunc, min_opacity, "FuseTSDF")
    if not (np.isfinite(np.asarray(bbox_min, np.float64)).all() and np.isfinite(np.asarray(bbox_max, np.float64)).all()):
        raise ValueError("FuseTSDF: the box must be finite")
    origin, voxel, (nx, ny, nz) = _lattice(bbox_min, bbox_max, reso, "FuseTSDF")
    for t, name in ((opacity, "opacity"), (median_t, "median_t"), (colors, "colors")):
        ops._chk(t, torch.float32, f"FuseTSDF: {name}")
    dev = opacity.device
    cam = lambda t, k: torch.as_tensor(t, dtype=torch.float32, device=dev).reshape(V, -1)[:, :k]
    cams = torch.cat([cam(poses, 12), cam(intri, 6), cam(dist_params, 4)], 1).contiguous()      # pose, rows 0-1 of K, distortion
    mu = float(np.float32(float(trunc) * voxel))
    sdf_sum = torch.empty((nz, ny, nx), dtype=torch.float32, device=dev)
    weight, color_sum = torch.empty_like(sdf_sum), torch.empty((nz, ny, nx, 3), dtype=torch.float32, device=dev)
    step = max(1, TSDF_SLAB_POINTS // (nx * ny))
    for z0 in range(0, nz, step):
        n = min(step, nz - z0)
        for g0 in range(0, V, ops.TSDF_MAX_VIEWS):
            g = slice(g0, min(g0 + ops.TSDF_MAX_VIEWS, V))
            ops.tsdf_integrate(cams[g], opacity[g], median_t[g], colors[g], height, width, origin, voxel, z0, n, mu, min_opacity, g0 == 0,
                               sdf_sum, weight, color_sum)
    return TSDFGrid(sdf_sum, weight, color_sum, origin, voxel)


def TSDFSurface(grid):
    """The zero level set of a ``TSDFGrid`` as a coloured ``Mesh`` (no normals), in the grid's frame (DESIGN.md §3p).  A lattice point
    is observed when its weight is > 0 and it is not on the lattice's outermost layer; the surface is the marching-tetrahedra
    surface of -sdf_sum / weight at 0 over the tetrahedra whose corners are all observed, outward towards free space.  It is
    ``Isosurface`` of a lattice holding NaN where a point is not observed: every face of a tetrahedron with a NaN corner has a
    vertex on an edge to it, whose position is NaN, so dropping the faces with a non-finite vertex and then the unreferenced
    vertices (renumbered in order) leaves the fully observed tetrahedra.  Vertex colours: ``f2b_tsdf_colors``."""
    wt = grid.weight
    obs = wt > 0
    for a in range(3):
        obs.narrow(a, 0, 1).fill_(False)
        obs.narrow(a, obs.shape[a] - 1, 1).fill_(False)
    value = torch.where(obs, -grid.sdf_sum / wt, torch.full_like(wt, float("nan")))
    verts, faces = Isosurface(value, 0., grid.origin, (grid.voxel,) * 3, empty_logit=-1.)
    del value, obs
    f = faces.long()
    f = f[torch.isfinite(verts).all(1)[f].all(1)]
    used = torch.zeros((verts.shape[0],), dtype=torch.bool, device=verts.device)
    used[f.reshape(-1)] = True
    renum = torch.cumsum(used, 0, dtype=torch.int32) - 1
    verts, faces = verts[used], renum[f]
    return Mesh(verts, faces, ops.tsdf_colors(verts, wt, grid.color_sum, grid.origin, grid.voxel), None)


def _tsdf_maps(renderer, dataset, views, reso_level, bbox_min, bbox_max, min_opacity, apps, crop):
    """Pass 1 of ``ExtractTSDFMesh`` -> (opacity, median_t [V,h,w], colors [V,h,w,3], h, w, bbox_min, bbox_max), the box completed
    by its default where not given."""
    from .eval import _Validate
    h, w = dataset.height_ // reso_level, dataset.width_ // reso_level
    need_box = bbox_min is None or bbox_max is None
    pct = need_box and (crop is None or crop.invert)
    opas, meds, cols, pts = [], [], [], []
    with torch.no_grad(), _Validate(renderer):
        for opa, med, point, rgb, _ in _view_maps(renderer, dataset, views, h, w, apps, crop):
            opas.append(opa.view(h, w))
            meds.append(med.view(h, w))
            cols.append((rgb / opa[:, None]).clamp_(0., 1.).view(h, w, 3))     # only read where opa >= min_opacity > 0
            if pct:
                pts.append(point[opa >= float(min_opacity)])
    opacity, median_t, colors = torch.stack(opas), torch.stack(meds), torch.stack(cols)
    del opas, meds, cols
    if need_box:
        lo, hi = leaf_bounds(renderer)
        if pct:
            p = torch.cat(pts)
            if p.shape[0] == 0:
                raise ValueError("ExtractTSDFMesh: no pixel reaches min_opacity, so there is no default box; pass bbox_min and bbox_max")
            s = torch.sort(p, dim=0).values                       # per axis (torch.quantile refuses more than 2^24 elements)
            n = s.shape[0]
            p1, p99 = s[int(math.floor(.01 * (n - 1)))].double(), s[int(math.ceil(.99 * (n - 1)))].double()
            pad = (p99 - p1) * .05
            clo, chi = (p1 - pad).tolist(), (p99 + pad).tolist()
            del p, s
        else:
            clo, chi = crop.aabb()
        lo, hi = tuple(max(a, b) for a, b in zip(lo, clo)), tuple(min(a, b) for a, b in zip(hi, chi))
        bbox_min = lo if bbox_min is None else bbox_min
        bbox_max = hi if bbox_max is None else bbox_max
    return opacity, median_t, colors, bbox_min, bbox_max


def ExtractTSDFMesh(renderer, dataset, views=None, reso_level=1, reso=512, bbox_min=None, bbox_max=None, trunc=4., min_opacity=0.9,
                    appearance=None, crop=None):
    """The scene's surface as a coloured ``Mesh`` on the device fused from the views' depth maps, in the normalised frame
    (``Mesh.to_data_frame`` maps it back; DESIGN.md §3p).  Pass 1 is ``ExtractPointCloud``'s: every view of ``views`` (default
    ``dataset.train_set_``) rendered on the (height // reso_level) x (width // reso_level) grid, its opacity, median depth and
    foreground colour C / W.  Then ``FuseTSDF`` over the box [bbox_min, bbox_max] at ``reso`` with ``trunc`` and ``min_opacity``,
    and ``TSDFSurface``.  The default box: with a crop that is not inverted, ``crop.aabb()``; otherwise, per axis, the 1st to 99th
    percentile of the median points of the pixels with opacity >= ``min_opacity``, widened by 5 % of its extent; both within
    ``leaf_bounds``.  ``appearance`` (including ``"own"``) colours the mesh only; ``crop`` crops every render (DESIGN.md §3n).
    The result has the same bits every run."""
    crop = resolve_crop(crop)
    views = [int(v) for v in (dataset.train_set_ if views is None else views)]
    reso_level = int(reso_level)
    if not views:
        raise ValueError("ExtractTSDFMesh: no views")
    if reso_level < 1:
        raise ValueError("ExtractTSDFMesh: reso_level must be >= 1")
    _tsdf_args(trunc, min_opacity, "ExtractTSDFMesh")
    if int(reso) < 2:
        raise ValueError("ExtractTSDFMesh: reso must be >= 2")
    if bbox_min is not None and bbox_max is not None:
        _lattice(bbox_min, bbox_max, reso, "ExtractTSDFMesh")
    H, W = dataset.height_, dataset.width_
    if H // reso_level < 2 or W // reso_level < 2:
        raise ValueError(f"ExtractTSDFMesh: reso_level {reso_level} leaves a {H // reso_level} x {W // reso_level} grid of a {H} x {W} image")
    apps = [resolve_appearance(renderer, appearance, view=b) for b in views]
    opacity, median_t, colors, lo, hi = _tsdf_maps(renderer, dataset, views, reso_level, bbox_min, bbox_max, min_opacity, apps, crop)
    idx = torch.as_tensor(views, device=dataset.poses_.device)
    grid = FuseTSDF(dataset.poses_[idx], dataset.intri_[idx], dataset.dist_params_[idx], H, W, opacity, median_t, colors, lo, hi, reso,
                    trunc, min_opacity)
    del opacity, median_t, colors
    return TSDFSurface(grid)


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
