"""CPU checks of the surface-normal pieces (DESIGN.md §3j): the float64 twin the GPU tests compare the gradient kernel against,
and ``write_ply``'s normals.

1. The twin's warp Jacobian (normals_oracle.jacobian64) == central differences of the float64 warp, at located points of
   ngp_fox's octree and warps (tests/golden), relative 1e-7.
2. The twin's hash-blend derivative (normals_oracle.blend_grad) == central differences inside a cell (relative 1e-9), and on
   both sides of a cell face it is the derivative of the cell floor() picks (the piecewise derivative).
3. write_ply writes nx ny nz when the mesh has normals and they read back; a mesh without normals gives the bytes of the
   format without them.
"""
import numpy as np
import torch

import locate_oracle as LO
import normals_oracle as N
import workloads

F64 = torch.float64


def located_fox_points(n, seed):
    sb = workloads.scene_blobs("wanjinyou")
    from f2nerf_b200.octree_build import TREE_NODE
    nd = sb["nodes"].view(TREE_NODE)
    rng = np.random.default_rng(seed)
    leaf = np.nonzero((nd["trans_idx"] >= 0) & (nd["childs"] < 0).all(1))[0]
    pick = leaf[rng.integers(0, len(leaf), 2 * n)]
    pts = (nd["center"][pick] + (rng.random((2 * n, 3)) - .5) * .98 * nd["side_len"][pick, None]).astype(np.float32)
    _, a = LO.locate_points(sb["nodes"], sb["trans"], pts)
    keep = a[:, 0] >= 0
    return sb, pts[keep][:n], a[keep][:n]


def test_twin_jacobian_equals_central_differences():
    sb, pts, a = located_fox_points(4000, seed=1)
    assert len(pts) >= 1000 and len(np.unique(a[:, 0])) > 50
    w2xz, weight = N.trans_arrays(sb["trans"])
    w2xz, weight = w2xz[a[:, 0]], weight[a[:, 0]]
    x = pts.astype(np.float64)
    J = N.jacobian64(w2xz, weight, x)
    h = 1e-7 * np.abs(x).max()                                 # truncation ~h^2, rounding ~1e-16 / h: both far below 1e-7
    for c in range(3):
        e = np.zeros(3)
        e[c] = h
        cd = (N.warp64(w2xz, weight, x + e) - N.warp64(w2xz, weight, x - e)) / (2 * h)
        err = np.abs(cd - J[:, :, c]).max(1) / np.abs(J).reshape(len(x), -1).max(1)
        assert err.max() < 1e-7, (c, err.max())


def rand_cells(n, seed, S=1 << 12):
    g = torch.Generator().manual_seed(seed)
    table = torch.randn((S, 2), dtype=F64, generator=g).half().to(F64)
    rows = torch.randint(0, S, (n, 8), generator=g)
    dfeat = torch.randn((n, 2), dtype=F64, generator=g)
    return table, rows, dfeat, g


def blend(table, rows, frac, dfeat):
    return (N.corner_weights(frac) * (table[rows] * dfeat[:, None, :]).sum(-1)).sum(1)


def test_twin_blend_derivative_inside_a_cell():
    table, rows, dfeat, g = rand_cells(5000, seed=2)
    frac = torch.rand((5000, 3), dtype=F64, generator=g) * 0.98 + 0.01
    got = N.blend_grad(table, rows, frac, dfeat)
    h = 1e-5
    for a in range(3):
        e = torch.zeros(3, dtype=F64)
        e[a] = h
        cd = (blend(table, rows, frac + e, dfeat) - blend(table, rows, frac - e, dfeat)) / (2 * h)
        scale = got.abs().max(1).values.clamp_min(1e-12)
        assert float(((cd - got[:, a]).abs() / scale).max()) < 1e-9


def test_twin_blend_derivative_at_a_cell_face():
    """At p = k (frac 0 in the upper cell) and one fp32 ulp below it (frac ~ 1 in the lower cell, other rows), the derivative
    is each cell's own multilinear slope: its exact difference form sum_{y,z} w_y w_z (s_{1yz} - s_{0yz})."""
    table, rows_hi, dfeat, g = rand_cells(2000, seed=3)
    rows_lo = torch.randint(0, table.shape[0], rows_hi.shape, generator=g)
    k = torch.randint(1, 4096, (2000,), generator=g).to(torch.float32)
    p_hi = k
    p_lo = torch.nextafter(k, torch.zeros_like(k))
    yz = torch.rand((2000, 2), dtype=F64, generator=g)
    for p, rows in ((p_hi, rows_hi), (p_lo, rows_lo)):
        assert ((torch.floor(p) == k) == (p is p_hi)).all()
        fx = (p - torch.floor(p)).to(F64)
        frac = torch.cat([fx[:, None], yz], 1)
        got = N.blend_grad(table, rows, frac, dfeat)[:, 0]
        s = (table[rows] * dfeat[:, None, :]).sum(-1)
        wy, wz = frac[:, 1], frac[:, 2]
        want = ((1 - wy) * (1 - wz) * (s[:, 4] - s[:, 0]) + (1 - wy) * wz * (s[:, 5] - s[:, 1]) +
                wy * (1 - wz) * (s[:, 6] - s[:, 2]) + wy * wz * (s[:, 7] - s[:, 3]))
        assert float(((got - want).abs() / want.abs().clamp_min(1e-12)).max()) < 1e-12


def tiny_mesh(normals):
    from f2nerf_b200.geometry import Mesh
    v = torch.tensor([[0., 0., 0.], [1., 0., 0.], [0., 1., 0.], [0., 0., 1.]])
    f = torch.tensor([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], dtype=torch.int32)
    c = torch.tensor([[1., 0., 0.], [0., 1., 0.], [0., 0., 1.], [.5, .5, .5]])
    n = -v + 0.25 if normals else None
    return Mesh(v, f, c, n)


def read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").splitlines()
    nv = int([h for h in head if h.startswith("element vertex")][0].split()[-1])
    props = [h.split() for h in head if h.startswith("property ") and "list" not in h]
    dt = np.dtype([(p[2], {"float": "<f4", "uchar": "u1"}[p[1]]) for p in props])
    return head, np.frombuffer(data[end:end + nv * dt.itemsize], dt), data


def test_write_ply_normals_round_trip(tmp_path):
    from f2nerf_b200.geometry import write_ply
    m = tiny_mesh(True)
    write_ply(tmp_path / "n.ply", m)
    head, v, _ = read_ply(tmp_path / "n.ply")
    assert "property float nx" in head and head.index("property float nz") < head.index("property uchar red")
    assert np.array_equal(np.stack([v["nx"], v["ny"], v["nz"]], 1), m.normals.numpy())
    assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], 1), m.verts.numpy())


def test_write_ply_without_normals_is_unchanged(tmp_path):
    from f2nerf_b200.geometry import write_ply
    m = tiny_mesh(False)
    write_ply(tmp_path / "p.ply", m)
    head = ["ply", "format binary_little_endian 1.0", "element vertex 4", "property float x", "property float y", "property float z",
            "property uchar red", "property uchar green", "property uchar blue", "element face 4",
            "property list uchar int vertex_indices", "end_header"]
    vr = np.empty(4, [("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    v = m.verts.numpy()
    vr["x"], vr["y"], vr["z"] = v[:, 0], v[:, 1], v[:, 2]
    c = np.clip(np.rint(m.colors.numpy() * 255.), 0, 255).astype(np.uint8)
    vr["red"], vr["green"], vr["blue"] = c[:, 0], c[:, 1], c[:, 2]
    fr = np.empty(4, [("n", "u1"), ("v", "<i4", (3,))])
    fr["n"], fr["v"] = 3, m.faces.numpy()
    want = ("\n".join(head) + "\n").encode("ascii") + vr.tobytes() + fr.tobytes()
    assert open(tmp_path / "p.ply", "rb").read() == want
