"""Twins of the depth kernels of csrc/geometry.cu (DESIGN.md §3l) for the tests.  Test infrastructure: never imported by the
f2nerf_b200 package.

- ``termination``: f2b_ray_termination_slots restated in numpy float32: each ray's kept weights summed serially in slot order
  (``np.cumsum`` over float32 rows accumulates one element at a time), the first sample whose running sum reaches 0.5 W, and
  its world point fmaf(t, d, o).
- ``fma32``: C's fmaf on float32 arrays, exact: the float64 product of two floats is exact, their sum with c is rounded to odd
  (TwoSum gives the error, a non-zero error on an even result moves it one float64 ulp towards the exact value), and a value
  rounded to odd with 29 spare bits rounds to float32 as the exact value would.
- ``project64``: f2b_depth_consistency's projection in float64: camera frame, forward distortion, pixel and the continuous grid
  coordinates whose nearest integers are the cell.
"""
import numpy as np

f32 = np.float32


def fma32(a, b, c):
    """Correctly rounded float32 a * b + c, elementwise."""
    a, b, c = np.broadcast_arrays(np.asarray(a, f32), np.asarray(b, f32), np.asarray(c, f32))
    p = a.astype(np.float64) * b.astype(np.float64)                 # exact: 24 + 24 bits
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)                               # TwoSum: s + err == p + c exactly
    even = (s.view(np.uint64) & np.uint64(1)) == 0
    bump = (err != 0) & even & np.isfinite(s)
    s = np.where(bump, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(f32)


def termination(w_slots, kept, slot_t, rays_o, rays_d):
    """w_slots, slot_t [R,S] float32 (entries past kept[r] are ignored), kept [R], rays_o / rays_d [R,3] (unit directions) ->
    (opacity [R], median_t [R], point [R,3]) float32, as f2b_ray_termination_slots."""
    w_slots, slot_t = np.asarray(w_slots, f32), np.asarray(slot_t, f32)
    R, S = w_slots.shape
    kept = np.asarray(kept, np.int64)
    valid = np.arange(S)[None, :] < kept[:, None]
    cum = np.cumsum(np.where(valid, w_slots, f32(0)), axis=1, dtype=f32)
    W = cum[:, -1] if S else np.zeros(R, f32)
    half = f32(.5) * W
    hit = valid & (cum >= half[:, None])
    m = np.argmax(hit, axis=1)
    ok = W > 0
    opacity = np.where(ok, W, f32(0)).astype(f32)
    tm = np.where(ok, slot_t[np.arange(R), m], f32(0)).astype(f32)
    point = fma32(tm[:, None], np.asarray(rays_d, f32), np.asarray(rays_o, f32))
    point[~ok] = 0
    return opacity, tm, point


def termination_serial(w, k, t):
    """One ray in plain float32 scalars, one addition at a time: (W, median t, m)."""
    run = f32(0)
    for i in range(k):
        run = f32(run + f32(w[i]))
    if not run > 0:
        return f32(0), f32(0), -1
    half = f32(f32(.5) * run)
    acc = f32(0)
    for i in range(k):
        acc = f32(acc + f32(w[i]))
        if acc >= half:
            return run, f32(t[i]), i
    raise AssertionError("the running sum never reached half of its own total")


def grid_step(extent, n):
    """linspace(0, extent - 1, n)'s pitch in pixels."""
    return (extent - 1.) / (n - 1.)


def project64(pts, pose, intri, dist_params, height, width, out_h, out_w):
    """World points [n,3] into a view (pose [3,4] camera-to-world, intri [3,3], dist (k1, k2, p1, p2)) in float64 ->
    dict(front [n] bool, fa, fb [n] the continuous grid row / column, a, b [n] their nearest integers, cell [n] (a * out_w + b,
    -1 behind the camera or outside the grid), dist [n] = |p - o|)."""
    pts = np.asarray(pts, np.float64).reshape(-1, 3)
    P = np.asarray(pose, np.float64).reshape(3, 4)
    K = np.asarray(intri, np.float64).reshape(3, 3)
    k1, k2, p1, p2 = np.asarray(dist_params, np.float64).reshape(4)
    d = pts - P[:, 3][None]
    xc = d @ P[:, :3]                                                # R^T (p - o)
    front = xc[:, 2] < 0
    with np.errstate(divide="ignore", invalid="ignore"):
        u, v = xc[:, 0] / -xc[:, 2], xc[:, 1] / xc[:, 2]
    r2 = u * u + v * v
    radial = r2 * k1 + r2 * r2 * k2
    ud = u + (u * radial + 2 * p1 * u * v + p2 * (r2 + 2 * u * u))
    vd = v + (v * radial + 2 * p2 * u * v + p1 * (r2 + 2 * v * v))
    x, y = K[0, 0] * ud + K[0, 2], K[1, 1] * vd + K[1, 2]
    fb, fa = (x - .5) / grid_step(width, out_w), (y - .5) / grid_step(height, out_h)
    with np.errstate(invalid="ignore"):
        a, b = np.rint(np.nan_to_num(fa, nan=-9)), np.rint(np.nan_to_num(fb, nan=-9))
        inside = front & (a >= 0) & (a < out_h) & (b >= 0) & (b < out_w)
    cell = np.where(inside, a * out_w + b, -1).astype(np.int64)
    return dict(front=front, fa=fa, fb=fb, a=a, b=b, cell=cell, dist=np.linalg.norm(d, axis=1))


def consistency64(pts, source, view, pose, intri, dist_params, height, width, out_h, out_w, opacity, median_t, min_opacity,
                  rel_tol):
    """f2b_depth_consistency's test in float64 -> (consistent [n] bool, cell [n], margin_px [n], margin_tol [n]): margin_px the
    distance of the projection from the nearest cell boundary (in pixels), margin_tol | |p - o| - t | - rel_tol t | / t where
    the cell is opaque (inf elsewhere)."""
    pr = project64(pts, pose, intri, dist_params, height, width, out_h, out_w)
    cell = pr["cell"].copy()
    skip = np.asarray(source) == view
    cell[skip] = -1
    sj, si = grid_step(width, out_w), grid_step(height, out_h)
    with np.errstate(invalid="ignore"):
        mb = np.abs(np.abs(pr["fb"] - pr["b"]) - .5) * sj
        ma = np.abs(np.abs(pr["fa"] - pr["a"]) - .5) * si
        # the grid's outer edges are boundaries too
        margin_px = np.where(pr["front"], np.minimum(ma, mb), np.inf)
    margin_px[skip] = np.inf
    ok = cell >= 0
    op = np.zeros(len(cell))
    tb = np.zeros(len(cell))
    op[ok] = np.asarray(opacity, np.float64)[cell[ok]]
    tb[ok] = np.asarray(median_t, np.float64)[cell[ok]]
    opaque = ok & (op >= min_opacity)
    with np.errstate(divide="ignore", invalid="ignore"):
        dev = np.abs(pr["dist"] - tb) - rel_tol * tb
        margin_tol = np.where(opaque, np.abs(dev) / tb, np.inf)
    consistent = opaque & (dev <= 0)
    return consistent, cell, margin_px, margin_tol
