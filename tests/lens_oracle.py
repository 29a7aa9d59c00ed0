"""float64 twin of f2b_lens_rays (DESIGN.md §3o) in numpy, and the inverse maps the tests check it with.

The twin follows the documented maps, not the kernel's operation order: angles in half-turns through an exact quadrant
reduction (so cos(pi / 2) is 0, as sincospi gives it), then numpy's sin / cos.  ``broken`` selects a deliberately wrong twin
("lam_sign": longitude flipped, "corner": the pixel centre at b instead of b + 1/2, "eyes": the ODS eyes swapped) so a test can
show that its bar rejects it.
"""
import numpy as np

EQUIRECT, FISHEYE, ODS = 0, 1, 2


def sincospi(x):
    """(sin(pi x), cos(pi x)) in float64 with x reduced exactly to [-1/4, 1/4] plus a quarter-turn count."""
    x = np.asarray(x, dtype=np.float64)
    q = np.rint(2. * x)                              # x = q / 2 + r, exact
    r = x - q / 2.
    s, c = np.sin(np.pi * r), np.cos(np.pi * r)
    k = np.mod(q, 4.).astype(np.int64)
    sin = np.choose(k, [s, c, -s, -c])
    cos = np.choose(k, [c, -s, -c, s])
    return sin, cos


def equirect_dirs(H, W, hfov, vfov, broken=None):
    """Camera-frame directions [H*W,3] and (sin lam, cos lam) of an equirectangular image, ray a*W + b."""
    a, b = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    a, b = a.reshape(-1), b.reshape(-1)
    bc = b if broken == "corner" else b + .5
    lam = hfov * (bc / W - .5) / 180.                                     # half-turns
    if broken == "lam_sign":
        lam = -lam
    phi = vfov * (.5 - (a + .5) / H) / 180.
    sl, cl = sincospi(lam)
    sp, cp = sincospi(phi)
    return np.stack([cp * sl, sp, -cp * cl], 1), sl, cl


def fisheye_dirs(H, W, fov, broken=None):
    """Camera-frame directions [H*W,3] (0 where not valid) and valid [H*W] of an equidistant fisheye."""
    a, b = np.meshgrid(np.arange(H, dtype=np.int64), np.arange(W, dtype=np.int64), indexing="ij")
    X, Y = (2 * b + 1 - W).reshape(-1), (2 * a + 1 - H).reshape(-1)
    if broken == "corner":
        X = X - 1
    m = min(H, W)
    valid = X * X + Y * Y <= m * m                                        # r <= min(H, W) / 2, exactly
    x, y = X / 2., Y / 2.
    r = np.hypot(x, y)
    st, ct = sincospi(r * fov / (180. * m))                               # theta = r / f, f = (m / 2) / (fov / 2), in half-turns
    safe = np.where(r > 0, r, 1.)
    d = np.stack([np.where(r > 0, st * x / safe, 0.), np.where(r > 0, -st * y / safe, 0.), np.where(r > 0, -ct, -1.)], 1)
    return np.where(valid[:, None], d, 0.), valid


def lens_rays(model, pose, H, W, p0, p1=0., p2=0., broken=None):
    """-> (rays_o [N,3], rays_d [N,3], valid [N]) float64, N = H*W (2*H*W for ODS, left eye on top)."""
    P = np.asarray(pose, dtype=np.float64).reshape(3, 4)
    R, t = P[:, :3], P[:, 3]
    if model == FISHEYE:
        dc, valid = fisheye_dirs(H, W, p0, broken)
        d = dc @ R.T
        return np.broadcast_to(t, d.shape).copy(), np.where(valid[:, None], d, 0.), valid
    dc, sl, cl = equirect_dirs(H, W, p0, p1, broken)
    d = dc @ R.T
    if model == EQUIRECT:
        return np.broadcast_to(t, d.shape).copy(), d, np.ones(len(d), bool)
    os_, ds = [], []
    for s in (-1., 1.):
        if broken == "eyes":
            s = -s
        off = np.stack([s * p2 / 2. * cl, np.zeros_like(cl), s * p2 / 2. * sl], 1)
        os_.append(t + off @ R.T)
        ds.append(d)
    o, d = np.concatenate(os_), np.concatenate(ds)
    return o, d, np.ones(len(d), bool)


def equirect_pixel(d, H, W, hfov, vfov):
    """The inverse map: camera-frame directions [n,3] -> continuous pixel coordinates (row, col) of their centres' grid."""
    d = np.asarray(d, dtype=np.float64)
    lam = np.degrees(np.arctan2(d[:, 0], -d[:, 2]))
    phi = np.degrees(np.arctan2(d[:, 1], np.hypot(d[:, 0], d[:, 2])))
    return H * (.5 - phi / vfov) - .5, W * (lam / hfov + .5) - .5


def pinhole_dirs(K, H, W):
    """Camera-frame directions [H*W,3] of an undistorted pinhole K, ray a*W + b through (a + .5, b + .5) (OpenGL frame)."""
    a, b = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    u = (b.reshape(-1) + .5 - K[0, 2]) / K[0, 0]
    v = (a.reshape(-1) + .5 - K[1, 2]) / K[1, 1]
    return np.stack([u, -v, -np.ones_like(u)], 1)


def ulp_diff(got, want):
    """|ordered-int distance| between float32 ``got`` and float64 ``want`` rounded to float32 (+0 and -0 are the same)."""
    g = np.ascontiguousarray(got, dtype=np.float32).view(np.int32).astype(np.int64)
    w = np.ascontiguousarray(np.asarray(want, dtype=np.float64).astype(np.float32)).view(np.int32).astype(np.int64)
    key = lambda i: np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(g) - key(w))
