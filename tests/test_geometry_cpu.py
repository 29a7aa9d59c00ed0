"""Geometry without a GPU: point location (orc_locate_points, tests/locate_oracle.c) against the oracle march's own samples on the reference's ngp_fox
octree, the marching-tetrahedra restatement (tests/isosurface_oracle.py) on analytic and random fields, and the PLY writer."""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import isosurface_oracle as ISO  # noqa: E402
import locate_oracle as LO  # noqa: E402
import oracle_lib as O  # noqa: E402
import workloads  # noqa: E402
from f2nerf_b200.octree_build import TREE_NODE  # noqa: E402

f32 = np.float32


def march_world_points(nodes, trans, n_rays, seed, scale_by_dis=True, sample_l=1. / 256):
    """The oracle march on the ngp_fox rays -> (world points in the march's rounding fmaf(t, d, o), march output)."""
    o, d, _ = workloads.host_rays("wanjinyou", n_rays, seed)
    dn = (d / np.linalg.norm(d.astype(np.float64), axis=1, keepdims=True)).astype(f32)
    noise = np.ones(1024 + n_rays + 10, f32)
    s = O.sampler(nodes, trans, o, dn, noise, 0.01, 1e8, sample_l, scale_by_dis, 1024)
    ray = np.repeat(np.arange(n_rays), np.diff(s["bounds"], axis=1)[:, 0])
    return fmaf(s["t"][:, None], dn[ray], o[ray]), s


def fmaf(a, b, c):
    """C's fmaf elementwise (libm), float32."""
    import ctypes
    libm = ctypes.CDLL("libm.so.6")
    libm.fmaf.restype = ctypes.c_float
    libm.fmaf.argtypes = [ctypes.c_float] * 3
    a, b, c = np.broadcast_arrays(np.asarray(a, f32), np.asarray(b, f32), np.asarray(c, f32))
    return np.array([libm.fmaf(x, y, z) for x, y, z in zip(a.ravel().tolist(), b.ravel().tolist(), c.ravel().tolist())],
                    f32).reshape(a.shape)


def face_straddle(nodes_u8, w, anchors_got, anchors_want):
    """Rows located in another leaf than the march's: each must lie within a few ulp of a face of the march's leaf."""
    nodes = nodes_u8.view(TREE_NODE)
    bad = np.nonzero((anchors_got != anchors_want).any(1))[0]
    for i in bad:
        nd = nodes[anchors_want[i, 1]]
        lo, hi = nd["center"] - nd["side_len"] * f32(.5), nd["center"] + nd["side_len"] * f32(.5)
        gap = np.minimum(np.abs(w[i] - lo), np.abs(w[i] - hi)).min()
        assert gap <= 8 * np.spacing(np.abs(w[i]).max()), (i, w[i], anchors_got[i], anchors_want[i], gap)
    return len(bad)


@pytest.mark.parametrize("scale_by_dis", [True, False])
def test_locate_points_recovers_the_march_samples(scale_by_dis):
    """Every sample of the oracle march on the golden ngp_fox octree (897 nodes, 372 warps), located from its world point,
    lands in the march's leaf with the march's warped point, bit for bit; the exceptions are samples on a face the two leaves
    share (counted and reported)."""
    sb = workloads.scene_blobs("wanjinyou")
    w, s = march_world_points(sb["nodes"], sb["trans"], 512, seed=5, scale_by_dis=scale_by_dis)
    assert len(w) > 50000
    warped, anchors = LO.locate_points(sb["nodes"], sb["trans"], w)
    want = s["anchors"][:, :2]
    n_straddle = face_straddle(sb["nodes"], w, anchors, want)
    same = (anchors == want).all(1)
    assert np.array_equal(warped[same].view(np.uint32), s["pts"][same].view(np.uint32))
    assert n_straddle <= len(w) // 1000
    with open(workloads.diag_path(f"locate_straddle_cpu_{int(scale_by_dis)}.json"), "w") as f:
        json.dump(dict(samples=len(w), face_straddle=n_straddle), f)
    print(f"\n{len(w)} samples, {n_straddle} on a face shared by two leaves")


def test_locate_points_tie_rule_and_outside():
    """Points on a splitting plane go to the upper child; the root's upper faces, points outside it and NaN locate nowhere."""
    sb = workloads.scene_blobs("wanjinyou")
    nodes = sb["nodes"].view(TREE_NODE)
    root = nodes[0]
    h = root["side_len"] * f32(.5)
    c = root["center"]
    pts = np.array([c + h, c - h, c + f32(2) * h, [np.nan, 0, 0]], f32)
    _, a = LO.locate_points(sb["nodes"], sb["trans"], pts)
    assert (a[[0, 2, 3]] == -1).all()
    # every leaf's own centre and its lowest corner locate to that leaf when it is valid
    leaf = np.nonzero((nodes["childs"] < 0).all(1))[0]
    ctr = nodes["center"][leaf]
    low = ctr - (nodes["side_len"][leaf] * f32(.5))[:, None]
    for q in (ctr, low):
        _, a = LO.locate_points(sb["nodes"], sb["trans"], np.ascontiguousarray(q, f32))
        valid = nodes["trans_idx"][leaf] >= 0
        assert np.array_equal(a[valid, 1], leaf[valid]) and np.array_equal(a[valid, 0], nodes["trans_idx"][leaf][valid])
        assert (a[~valid] == -1).all()


def test_case_table_is_exhaustively_outward():
    """All 16 inside patterns of a tetrahedron: 0 / 1 / 2 triangles as the count of inside corners says, each with its normal
    pointing from the inside corners' centroid towards the outside corners' (linear field, midpoint vertices)."""
    corners = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float64)
    for m in range(16):
        tris = ISO.CASES[m]
        k = bin(m).count("1")
        assert len(tris) == {0: 0, 1: 1, 2: 2, 3: 1, 4: 0}[k]
        if not tris:
            continue
        ins = corners[[q for q in range(4) if m >> q & 1]].mean(0)
        out = corners[[q for q in range(4) if not m >> q & 1]].mean(0)
        for tri in tris:
            p = np.array([(corners[a] + corners[b]) / 2 for a, b in tri])
            for a, b in tri:
                assert (m >> a & 1) != (m >> b & 1)
            n = np.cross(p[1] - p[0], p[2] - p[0])
            assert np.dot(n, out - ins) > 0, (m, tri)
    for tet in ISO.TETS:
        p = np.array([[c & 1, c >> 1 & 1, c >> 2] for c in tet], np.float64)
        assert np.linalg.det(p[1:] - p[0]) > 0
        for i in range(4):
            for j in range(i + 1, 4):
                lo, hi = min(tet[i], tet[j]), max(tet[i], tet[j])
                assert lo & hi == lo                    # nested offsets: the edge is owned by its lower corner


def test_sphere_is_a_closed_sphere():
    n, r = 96, 30.
    v, f = ISO.extract(ISO.sphere(n, r), 0.)
    st = ISO.mesh_stats(v, f)
    assert st["euler"] == 2 and st["volume"] > 0
    assert abs(st["volume"] / (4. / 3. * np.pi * r ** 3) - 1) < 0.01, st


def test_torus_is_a_closed_torus():
    v, f = ISO.extract(ISO.torus(96, 25., 10.), 0.)
    st = ISO.mesh_stats(v, f)
    assert st["euler"] == 0 and st["volume"] > 0, st


@pytest.mark.parametrize("shape,seed", [((17, 23, 29), 0), ((29, 17, 23), 1), ((5, 4, 3), 2), ((1, 1, 1), 3), ((2, 7, 1), 4)])
def test_random_fields_are_closed_manifolds(shape, seed):
    """Uniform random fields (many components, many boundary contacts): the virtual pad closes every component."""
    L = np.random.default_rng(seed).random(shape, dtype=f32)
    v, f = ISO.extract(L, 0.5, origin=(-1., 2., .5), voxel=(.25, .5, .125))
    if len(f):
        ISO.mesh_stats(v, f)
    assert len(f) > 0 or (L <= .5).all()


def test_surface_touching_the_box_closes_on_the_pad():
    """A field inside everywhere: the pad closes the surface around the box."""
    L = np.full((4, 5, 6), 1., f32)
    v, f = ISO.extract(L, 0.)
    st = ISO.mesh_stats(v, f)
    assert st["euler"] == 2 and st["volume"] > 0


def test_ply_round_trip(tmp_path):
    import torch
    from f2nerf_b200.geometry import Mesh, write_ply
    v, f = ISO.extract(ISO.sphere(12, 4.), 0.)
    rgb = np.random.default_rng(0).random((len(v), 3), dtype=f32)
    for colors in (None, torch.from_numpy(rgb)):
        p = str(tmp_path / "m.ply")
        write_ply(p, Mesh(torch.from_numpy(v), torch.from_numpy(f), colors))
        gv, gf, gc = read_ply(p)
        assert np.array_equal(gv.view(np.uint32), v.view(np.uint32)) and np.array_equal(gf, f)
        if colors is None:
            assert gc is None
        else:
            assert np.array_equal(gc, np.clip(np.rint(rgb * 255.), 0, 255).astype(np.uint8))


def read_ply(path):
    """A minimal binary little-endian PLY reader for the writer's layout."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").split("\n")
    assert head[0] == "ply" and head[1] == "format binary_little_endian 1.0"
    nv = int(next(x for x in head if x.startswith("element vertex")).split()[-1])
    nf = int(next(x for x in head if x.startswith("element face")).split()[-1])
    colored = "property uchar red" in head
    vfields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")] + ([("r", "u1"), ("g", "u1"), ("b", "u1")] if colored else [])
    vr = np.frombuffer(data, vfields, nv, end)
    fr = np.frombuffer(data, [("n", "u1"), ("v", "<i4", (3,))], nf, end + vr.nbytes)
    assert (fr["n"] == 3).all() and end + vr.nbytes + fr.nbytes == len(data)
    v = np.stack([vr["x"], vr["y"], vr["z"]], 1)
    c = np.stack([vr["r"], vr["g"], vr["b"]], 1) if colored else None
    return v, fr["v"].copy(), c
