"""Twins of the TSDF fusion of csrc/geometry.cu and geometry.py (DESIGN.md §3p) for the tests.  Test infrastructure: never imported
by the f2nerf_b200 package.

- ``lattice_points``: the lattice points as the kernel forms them, fadd(origin, fmul(voxel, i)) per axis in float32.
- ``integrate64``: f2b_tsdf_integrate in float64 on those points, the projection by ``points_oracle.project64``, with the
  margins that say where fp32 may decide differently (a projection near a cell boundary, an sdf near the -mu cut) and a bound on
  the fp32 error of the sums.  ``mode`` selects a deliberately broken twin ("sign", "nocut", "axis") that the tests must reject.
- ``surface``: ``TSDFSurface``'s lattice (NaN where not observed) through ``isosurface_oracle.extract`` and the face filter.
- ``observed_tets``: the faces of the fully observed tetrahedra enumerated directly, cell by cell.
- ``look_at`` / ``pinhole_rays`` / ``sphere_maps``: cameras around a point and exact depth maps of a sphere, without distortion.
"""
import numpy as np

import isosurface_oracle as ISO
import points_oracle as PO

f32 = np.float32
EPS32 = 2. ** -23


def lattice_points(origin, voxel, shape):
    """[nz*ny*nx, 3] float32 lattice points, x fastest, formed as f2b_tsdf_integrate forms them."""
    nz, ny, nx = shape
    zz, yy, xx = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    return np.stack([f32(o) + f32(voxel) * i.astype(f32) for o, i in zip(origin, (xx, yy, zz))], -1).reshape(-1, 3)


def integrate64(pts, poses, intri, dist, height, width, opacity, median_t, colors, mu, min_opacity, mode=None):
    """-> dict(sdf_sum, weight, color_sum [n,3], bound_sdf, bound_col (fp32 error bounds of the sums), margin_px (smallest distance
    in pixels of a projection from a cell boundary, over the views), margin_cut (smallest |sdf + mu| / |p - o| over the views
    whose cell counts))."""
    pts = np.asarray(pts, np.float64)
    V, h, w = opacity.shape
    n = len(pts)
    out = dict(sdf_sum=np.zeros(n), weight=np.zeros(n), color_sum=np.zeros((n, 3)), bound_sdf=np.zeros(n), bound_col=np.zeros(n),
               margin_px=np.full(n, np.inf), margin_cut=np.full(n, np.inf))
    mu = float(mu)
    sj, si = PO.grid_step(width, w), PO.grid_step(height, h)
    for v in range(V):
        pr = PO.project64(pts, poses[v], intri[v], dist[v], height, width, h, w)
        with np.errstate(invalid="ignore"):
            mb = np.abs(np.abs(pr["fb"] - pr["b"]) - .5) * sj
            ma = np.abs(np.abs(pr["fa"] - pr["a"]) - .5) * si
            out["margin_px"] = np.minimum(out["margin_px"], np.where(pr["front"], np.minimum(ma, mb), np.inf))
        cell = pr["cell"]
        ok = cell >= 0
        c = np.where(ok, cell, 0)
        op = np.asarray(opacity[v], np.float64).reshape(-1)[c]
        t = np.asarray(median_t[v], np.float64).reshape(-1)[c]
        dist_ = pr["dist"]
        if mode == "axis":                                      # distance along the optical axis instead of along the ray
            dist_ = np.abs((pts - np.asarray(poses[v], np.float64)[:, 3]) @ np.asarray(poses[v], np.float64)[:, 2])
        sdf = t - dist_ if mode != "sign" else dist_ - t
        counts = ok & (op >= min_opacity)
        take = counts & ((sdf >= -mu) | (mode == "nocut"))
        out["margin_cut"] = np.minimum(out["margin_cut"], np.where(counts, np.abs(sdf + mu) / pr["dist"], np.inf))
        term = np.minimum(1., sdf / mu)
        out["sdf_sum"] += np.where(take, term, 0.)
        out["weight"] += take
        out["color_sum"] += np.where(take[:, None], np.asarray(colors[v], np.float64).reshape(-1, 3)[c], 0.)
        # per term: |p - o| and t carry a few fp32 ulps of their size, divided by mu; the division and min add one more
        out["bound_sdf"] += np.where(take, 8. * EPS32 * (dist_ + np.abs(t)) / mu + 2. * EPS32, 0.)
    # the serial fp32 sums round once per addition, each by at most half an ulp of the running sum
    out["bound_sdf"] += out["weight"] * EPS32 * np.maximum(out["weight"], 1.)
    out["bound_col"] = out["weight"] * EPS32 * np.maximum(out["weight"], 1.)
    return out


def observed(weight):
    """weight [nz,ny,nx] -> the observed mask: weight > 0 and not on the outermost layer."""
    obs = np.asarray(weight) > 0
    obs[[0, -1]] = False
    obs[:, [0, -1]] = False
    obs[:, :, [0, -1]] = False
    return obs


def tsdf_lattice(sdf_sum, weight):
    """-sdf_sum / weight in float32 where observed, NaN elsewhere (TSDFSurface's lattice)."""
    obs = observed(weight)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(obs, -np.asarray(sdf_sum, f32) / np.asarray(weight, f32), f32(np.nan)).astype(f32)


def filter_faces(verts, faces):
    """Drop the faces with a non-finite vertex, then the unreferenced vertices, renumbering in order."""
    f = np.asarray(faces, np.int64)
    f = f[np.isfinite(verts).all(1)[f].all(1)]
    used = np.zeros(len(verts), bool)
    used[f.reshape(-1)] = True
    renum = np.cumsum(used) - 1
    return verts[used], renum[f].astype(np.int32)


def surface(lattice, origin=(0., 0., 0.), voxel=(1., 1., 1.)):
    """TSDFSurface's mesh of a NaN lattice (without colours): extract at 0 with the pad at -1, then the face filter."""
    with np.errstate(invalid="ignore"):
        v, f = ISO.extract(lattice, 0., origin, voxel, empty=-1.)
    return filter_faces(v, f)


def observed_tets(lattice):
    """The triangles [F,3,3] (vertex positions, origin 0, unit voxels) of the tetrahedra whose four corners are in the lattice and
    finite, enumerated cell by cell in (cell, tetrahedron, triangle) order, vertices formed as the kernel forms them."""
    L = np.asarray(lattice, f32)
    nz, ny, nx = L.shape
    tris = []
    for z in range(nz - 1):
        for y in range(ny - 1):
            for x in range(nx - 1):
                corner = lambda c: (x + (c & 1), y + (c >> 1 & 1), z + (c >> 2))
                vals = [L[corner(c)[::-1]] for c in range(8)]
                for tet in ISO.TETS:
                    if not all(np.isfinite(vals[c]) for c in tet):
                        continue
                    m = sum(int(vals[tet[q]] > 0) << q for q in range(4))
                    for tri in ISO.CASES[m]:
                        pos = []
                        for p0, p1 in tri:
                            a, b = sorted((tet[p0], tet[p1]))
                            fa, fb = vals[a], vals[b]
                            t = (f32(0) - fa) / (fb - fa)
                            ca, d = corner(a), (a ^ b)
                            pos.append([f32(ca[k]) + t if d >> k & 1 else f32(ca[k]) for k in range(3)])
                        tris.append(pos)
    return np.asarray(tris, f32).reshape(-1, 3, 3)


def look_at(eye, target, up=(0., 0., 1.)):
    """[3,4] camera-to-world pose at ``eye`` looking at ``target`` (the camera looks down its -z axis)."""
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    back = eye - target
    back /= np.linalg.norm(back)
    right = np.cross(np.asarray(up, np.float64), back)
    if np.linalg.norm(right) < 1e-6:
        right = np.cross((1., 0., 0.), back)
    right /= np.linalg.norm(right)
    yy = np.cross(back, right)
    return np.concatenate([np.stack([right, yy, back], 1), eye[:, None]], 1)


def pinhole_rays(pose, K, height, width, h, w):
    """Unit rays [h*w,3] (float64) through the cells of the h x w grid of an undistorted camera (x = fb * step + .5, as
    ``project64`` inverts it); origins are the pose's translation."""
    P, K = np.asarray(pose, np.float64), np.asarray(K, np.float64)
    a, b = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    x, y = b.reshape(-1) * PO.grid_step(width, w) + .5, a.reshape(-1) * PO.grid_step(height, h) + .5
    u, v = (x - K[0, 2]) / K[0, 0], (y - K[1, 2]) / K[1, 1]
    d = np.stack([u, -v, -np.ones_like(u)], 1) @ P[:, :3].T
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def sphere_maps(pose, K, height, width, h, w, center, radius, colour):
    """Exact maps of a sphere seen by an undistorted camera: opacity 1 where the ray hits (0 elsewhere), median_t the distance
    to the first hit, colours ``colour(hit points [n,3]) -> [n,3]`` -> float32 (opacity [h,w], median_t [h,w], colors [h,w,3])."""
    d = pinhole_rays(pose, K, height, width, h, w)
    oc = np.asarray(pose, np.float64)[:, 3] - np.asarray(center, np.float64)
    bq = d @ oc
    disc = bq * bq - (oc @ oc - radius * radius)
    hit = disc > 0
    t = np.where(hit, -bq - np.sqrt(np.maximum(disc, 0.)), 0.)
    hit &= t > 0
    t = np.where(hit, t, 0.)
    p = np.asarray(pose, np.float64)[:, 3] + t[:, None] * d
    col = np.where(hit[:, None], colour(p), 0.)
    return hit.astype(f32).reshape(h, w), t.astype(f32).reshape(h, w), col.astype(f32).reshape(h, w, 3)


def sphere_cameras(n, center, dist, seed=0):
    """``n`` poses at distance ``dist`` from ``center`` (a Fibonacci sphere, slightly jittered), looking at it."""
    rng = np.random.default_rng(seed)
    k = np.arange(n) + .5
    z = 1. - 2. * k / n
    phi = np.pi * (1. + 5. ** .5) * k
    r = np.sqrt(1. - z * z)
    dirs = np.stack([r * np.cos(phi), r * np.sin(phi), z], 1) + rng.normal(size=(n, 3)) * .02
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    c = np.asarray(center, np.float64)
    return np.stack([look_at(c + dist * e, c) for e in dirs])
