"""float32 numpy restatement of the marching-tetrahedra extraction of f2b_iso_count / f2b_iso_emit (f2nerf_b200/csrc/geometry.cu,
DESIGN.md §3i), and the mesh checks the geometry tests apply.  Test infrastructure: never imported by the f2nerf_b200 package.

Every arithmetic step is a float32 numpy operation in the kernel's order, so the vertices come out with the same bits:
t = (level - f_a) / (f_b - f_a), position = origin + voxel * (index + t * dir)."""
import numpy as np

f32 = np.float32
# the six Kuhn tetrahedra of a cell, corners as offset codes (bit 0 x, bit 1 y, bit 2 z), each positively oriented
TETS = ((0, 1, 3, 7), (0, 1, 7, 5), (0, 2, 7, 3), (0, 2, 6, 7), (0, 4, 5, 7), (0, 4, 7, 6))
DIR_CODES = (1, 2, 4, 3, 5, 6, 7)        # edge direction index -> offset code: (1,0,0) (0,1,0) (0,0,1) (1,1,0) (1,0,1) (0,1,1) (1,1,1)
DIR_INDEX = {c: i for i, c in enumerate(DIR_CODES)}
OPP = ((1, 2, 3), (0, 3, 2), (0, 1, 3), (0, 2, 1))   # face opposite each corner, normal pointing away from it


def tet_triangles(mask):
    """Triangles of a positive tetrahedron whose corners in ``mask`` (bit q: corner q) are inside, each as three edges
    (pairs of corner positions), oriented outward (towards the outside corners)."""
    inside = [q for q in range(4) if mask >> q & 1]
    outside = [q for q in range(4) if not mask >> q & 1]
    if len(inside) in (1, 3):
        apex = inside[0] if len(inside) == 1 else outside[0]
        ring = OPP[apex] if len(inside) == 1 else OPP[apex][::-1]
        return [[(apex, r) for r in ring]]
    if len(inside) == 2:
        a, b = inside
        c, d = outside
        if (a, b) in ((0, 2), (1, 3)):     # make (a, b, c, d) an even permutation of (0, 1, 2, 3)
            c, d = d, c
        return [[(a, c), (a, d), (b, d)], [(a, c), (b, d), (b, c)]]
    return []


CASES = [tet_triangles(m) for m in range(16)]


def extract(logit, level, origin=(0., 0., 0.), voxel=(1., 1., 1.), empty=-1e4):
    """logit [nz, ny, nx] -> (verts [V,3] f32, faces [F,3] i32) in the kernel's order."""
    L = np.ascontiguousarray(logit, f32)
    nz, ny, nx = L.shape
    level, empty = f32(level), f32(empty)
    P = np.full((nz + 2, ny + 2, nx + 2), empty, f32)       # padded index e holds lattice coordinate e - 1
    P[1:-1, 1:-1, 1:-1] = L
    inside = P > level
    EZ, EY, EX = nz + 1, ny + 1, nx + 1

    def corner(a, code):
        dx, dy, dz = code & 1, code >> 1 & 1, code >> 2
        return a[dz:dz + EZ, dy:dy + EY, dx:dx + EX]

    cross = np.stack([corner(inside, 0) != corner(inside, c) for c in DIR_CODES], -1)      # [EZ, EY, EX, 7]
    vid = np.full((EZ + 1, EY + 1, EX + 1, 7), -1, np.int64)
    vid[:EZ, :EY, :EX] = np.where(cross, np.cumsum(cross.reshape(-1)).reshape(cross.shape) - 1, -1)
    pt, d = np.nonzero(cross.reshape(-1, 7))
    ez, ey, ex = np.unravel_index(pt, (EZ, EY, EX))
    code = np.asarray(DIR_CODES)[d]
    dx, dy, dz = code & 1, code >> 1 & 1, code >> 2
    fa, fb = P[ez, ey, ex], P[ez + dz, ey + dy, ex + dx]
    t = (level - fa) / (fb - fa)
    verts = np.empty((len(pt), 3), f32)
    for k, (idx, dk) in enumerate(((ex, dx), (ey, dy), (ez, dz))):
        u = (idx - 1).astype(f32)
        u = np.where(dk == 1, u + t, u)
        verts[:, k] = f32(origin[k]) + f32(voxel[k]) * u
    # faces: only cells whose corners disagree have any, in (cell, tetrahedron, triangle) order
    corners = np.stack([corner(inside, c) for c in range(8)], -1).reshape(-1, 8)
    cells = np.nonzero(corners.any(1) & ~corners.all(1))[0]
    cz, cy, cx = np.unravel_index(cells, (EZ, EY, EX))
    out = np.full((len(cells), 6, 2, 3), -1, np.int64)
    for ti, tet in enumerate(TETS):
        m = sum(corners[cells, tet[q]].astype(np.int64) << q for q in range(4))
        for case in range(16):
            sel = np.nonzero(m == case)[0]
            for j, tri in enumerate(CASES[case]):
                for q, (p0, p1) in enumerate(tri):
                    a, b = sorted((tet[p0], tet[p1]))
                    out[sel, ti, j, q] = vid[cz[sel] + (a >> 2), cy[sel] + (a >> 1 & 1), cx[sel] + (a & 1), DIR_INDEX[a ^ b]]
    faces = out[out[..., 0] >= 0]
    assert (faces >= 0).all()
    return verts, faces.astype(np.int32)


def mesh_stats(verts, faces):
    """Checks that faces form a closed, consistently oriented 2-manifold: every directed edge once and its reverse once (so
    every edge lies in exactly two faces), and the faces around every vertex one cycle.  -> dict(V, E, F, euler, volume)
    with the signed volume (positive for outward orientation)."""
    f = np.asarray(faces, np.int64)
    V = int(np.asarray(verts).shape[0])
    assert len(f) > 0 and f.min() >= 0 and f.max() < V
    assert (f[:, 0] != f[:, 1]).all() and (f[:, 1] != f[:, 2]).all() and (f[:, 0] != f[:, 2]).all()
    a, b = f.reshape(-1), f[:, [1, 2, 0]].reshape(-1)
    key, rev = a * V + b, b * V + a
    assert len(np.unique(key)) == len(key), "a directed edge is used twice: not an oriented manifold"
    assert np.isin(rev, key).all(), "an edge lies in only one face: not closed"
    used = np.unique(f)
    assert len(used) == V, "unreferenced vertices"
    # vertex links: face (v0, v1, v2) gives v0 the link edge v1 -> v2, v1 the edge v2 -> v0, v2 the edge v0 -> v1
    lv = f.reshape(-1)
    lf, lt = f[:, [1, 2, 0]].reshape(-1), f[:, [2, 0, 1]].reshape(-1)
    lkey = lv * V + lf
    order = np.argsort(lkey)
    skey, sto = lkey[order], lt[order]
    deg = np.bincount(lv, minlength=V)
    first = np.searchsorted(skey, np.arange(V, dtype=np.int64) * V)      # each vertex's first link edge (sorted by from)
    start = lf[order][first]
    cur, back = start.copy(), np.zeros(V, np.int64)
    vv = np.arange(V, dtype=np.int64)
    for step in range(1, int(deg.max()) + 1):
        pos = np.searchsorted(skey, vv * V + cur)
        assert (skey[np.minimum(pos, len(skey) - 1)] == vv * V + cur).all(), "a vertex link is not closed"
        cur = sto[pos]
        back = np.where((back == 0) & (cur == start), step, back)
    assert (back == deg).all(), "the faces around a vertex form more than one cycle"
    E = len(key) // 2
    p = np.asarray(verts, np.float64)
    vol = float(np.einsum("ij,ij->i", p[f[:, 0]], np.cross(p[f[:, 1]], p[f[:, 2]])).sum() / 6.)
    return dict(V=V, E=E, F=len(f), euler=V - E + len(f), volume=vol)


def sphere(n, r, center=None):
    """Signed distance (positive inside) of a sphere on an n^3 lattice of unit voxels, float32."""
    c = (n - 1) / 2. if center is None else center
    z, y, x = np.meshgrid(*(np.arange(n, dtype=np.float64),) * 3, indexing="ij")
    return (r - np.sqrt((x - c) ** 2 + (y - c) ** 2 + (z - c) ** 2)).astype(f32)


def torus(n, R, r):
    c = (n - 1) / 2.
    z, y, x = np.meshgrid(*(np.arange(n, dtype=np.float64) - c,) * 3, indexing="ij")
    return (r - np.sqrt((np.sqrt(x * x + y * y) - R) ** 2 + z * z)).astype(f32)
