"""The ray march (march16_kernel behind f2b_sampler_count / f2b_sampler_fill / f2b_sampler_march) on the rays where one fp32
predicate decides the result, against the CPU oracle (oracle/f2_oracle.c) bit for bit in all three modes, and against the
reference's own PersSampler::GetSamples (oracle/_ref/ref_driver --march) where that binary was built.

The cases, on the golden ngp_fox tree unless named otherwise:
  axis_parallel   hand-set directions with components +-0, +-1e-6 and one ulp either side, +-1e-7; origins outside the root,
                  inside leaves, at the root centre, and a few ulps from a leaf face plane whose direction component is below 1e-6
                  (the parallel guard of slab() decides whether that leaf is hit)
  on_geometry     origins exactly on leaf faces, edges and corners, at leaf centres and at the root centre
  grazing         rays inside a face plane (that component exactly 0) and rays aimed exactly through an edge or corner
                  (a node interval with near == far)
  near_*          near at a leaf's entry distance, inside a leaf, past every hit, near == far, and the hosts' 0.05 / 0.01
  noise_*         noise 0 at the first step, at the step that would hop, in a run up to the 1024-sample cap; torch.rand's range
                  ends 2^-24 and 1 - 2^-24 and the TRAIN noise's 0.5 and 1.5; a step so small that the leaf hop's step count passes
                  2^31 and the int conversion saturates.  Each with scale_by_dis 0 and 1
  step_*          a sample_l that fills the cap inside the first leaf, one where every step is a leaf hop
  deep tree       one corner chain of the golden tree subdivided down to depth 21..25 with invalid leaves and childless internal
                  nodes: the leaf at depth <= 23 is sampled, a push to depth 24 ends the traversal (kMaxDepth)
  lens / camera   f2b_lens_rays (equirectangular, ODS, fisheye 180/220/360) and f2b_camera_rays at the identity pose and at a
                  pose on a leaf face; RenderLens marches exactly these rays, with the same sample counts, first_oct_dis and
                  kept counts
Each case but the lens rays first checks, with the oracle's branch counters (orc_sampler_cover), that its batch takes the branch
it is named for (the lenses march whatever directions their pixels give).
The noise of a TRAIN step is (torch.rand - 0.5) + 1 (PersSampler.cu:377), in [0.5, 1.5): noise 0 and 2^-24 never reach the march
from the hosts; they are here because the kernel must still agree with the oracle on them.  Without NaN in the inputs the leaf hop
never divides by a zero step: t never passes the current leaf's far, so t + 0 cannot."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import yaml

import oracle_lib as O
import workloads
from test_gpu_march_lanes import CAP, check_all_modes

f32 = np.float32
ROOT = workloads.ROOT
REF_DRIVER = os.path.join(ROOT, "oracle", "_ref", "ref_driver")
MAX_WALK_DEPTH = 23          # kMaxDepth 24 stack entries: the root at 0, a push to depth 24 ends the traversal
NODE = np.dtype([("c", "<f4", 3), ("side", "<f4"), ("parent", "<i4"), ("childs", "<i4", 8), ("is_leaf", "u1"), ("pad0", "u1", 3),
                 ("trans", "<i4"), ("pad", "<i4")])
assert NODE.itemsize == 64


# ------------------------------------------------------------------------------------------------------------ trees
def golden():
    g = workloads.load_ngp_fox()
    return dict(nodes=g["tree_nodes"].copy(), trans=g["pers_trans"].copy())


def nodes_of(blob):
    return blob.view(NODE)


def depths(a):
    d = np.zeros(len(a), np.int64)
    for u in range(1, len(a)):                 # parents precede their children in every tree here
        d[u] = d[a["parent"][u]] + 1
    return d


def live_leaves(a):
    return np.nonzero((a["childs"] < 0).all(1) & (a["trans"] >= 0))[0]


def pick_leaves(a, k, seed=0):
    """k valid leaves of side <= 1 (the scene's detailed part), seeded."""
    leaves = live_leaves(a)
    leaves = leaves[a["side"][leaves] <= 1.]
    return np.random.default_rng(seed).choice(leaves, size=min(k, leaves.size), replace=False)


def ulps(x, k):
    """x moved k ulps (k may be negative), in float32."""
    x = f32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, f32(np.inf) if k > 0 else f32(-np.inf), dtype=f32)
    return x


def noise_of(n, value=1.):
    return np.full(CAP + n + 10, value, f32)


def case(nodes, trans, o, d, noise=None, near=0.05, far=1e8, sample_l=1 / 256, sbd=False, max_hits=CAP, covers=(), check=None):
    o, d = np.ascontiguousarray(o, f32), np.ascontiguousarray(d, f32)
    return dict(nodes=nodes, trans=trans, o=o, d=d, noise=noise_of(len(o)) if noise is None else noise, near=near, far=far,
                sample_l=sample_l, sbd=sbd, max_hits=max_hits, covers=covers, check=check)


# ------------------------------------------------------------------------------------------------- 1. axis-parallel
SMALL = [f32(0.), f32(-0.), f32(1e-6), ulps(1e-6, -1), ulps(1e-6, 1), f32(1e-7)]
SMALL = SMALL + [f32(-v) for v in SMALL[2:]]


def axis_parallel():
    g = golden()
    a = nodes_of(g["nodes"])
    rng = np.random.default_rng(1)
    o, d = [], []
    leaves = pick_leaves(a, 24, seed=1)
    for ax in range(3):
        b, c = (ax + 1) % 3, (ax + 2) % 3
        for u in leaves:                                    # a few ulps from a face plane of axis ax, moving along b
            cen, hf = a["c"][u], a["side"][u] / 2
            for sgn in (-1, 1):
                plane = f32(cen[ax] + sgn * hf)
                for k in (-3, -1, 1, 3):
                    p = cen.copy()
                    p[ax] = ulps(plane, k)
                    p[c] = f32(cen[c] + f32(0.3) * hf)
                    for s in SMALL[2:]:
                        v = np.zeros(3, f32)
                        v[b] = f32(rng.choice([-1., 1.]))
                        v[ax] = s
                        v[c] = rng.choice(SMALL)
                        o.append(p); d.append(v)
        # one, two or three components near zero, from the root centre, from leaf centres and from outside the root
        for s1 in SMALL:
            for s2 in SMALL[::2]:
                for start in ("centre", "leaf", "outside"):
                    v = np.zeros(3, f32)
                    v[ax], v[b], v[c] = f32(rng.choice([-1., 1.])), s1, s2
                    if start == "centre":
                        p = np.zeros(3, f32)
                    elif start == "leaf":
                        p = a["c"][rng.choice(leaves)].copy()
                    else:
                        p = a["c"][rng.choice(leaves)].copy()
                        p[ax] = f32(-300. * v[ax])
                    o.append(p); d.append(v)
    for s1 in SMALL:                                        # three components near zero
        for s2 in SMALL[::3]:
            o.append(a["c"][leaves[0]]); d.append(np.array([s1, s2, f32(1e-6)], f32))
    return case(g["nodes"], g["trans"], o, d, covers=("guard", "guard_zero", "guard_decides"))


# ----------------------------------------------------------------------------------------------- 2. origins on geometry
def on_geometry():
    g = golden()
    a = nodes_of(g["nodes"])
    rng = np.random.default_rng(2)
    leaves = pick_leaves(a, 40, seed=2)
    pts = [np.zeros(3, f32)]
    for u in leaves:
        cen, hf = a["c"][u], a["side"][u] / 2
        corner = np.array([rng.choice([-1, 1]) for _ in range(3)], f32)
        pts.append(cen.copy())
        for m in ([1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [0, 1, 1], [1, 1, 1]):   # faces, edges, a corner
            pts.append((cen + corner * hf * np.array(m, f32)).astype(f32))
    axes = [np.array(v, f32) for v in ([1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1])]
    o, d = [], []
    for p in pts:
        for v in axes + [x / np.linalg.norm(x) for x in rng.normal(size=(4, 3)).astype(f32)]:
            o.append(p); d.append(v)
    return case(g["nodes"], g["trans"], o, d, covers=("guard_zero", "guard_plane"))


# ----------------------------------------------------------------------------------------------------------- 3. grazing
def grazing():
    g = golden()
    a = nodes_of(g["nodes"])
    rng = np.random.default_rng(3)
    leaves = pick_leaves(a, 40, seed=3)
    o, d = [], []
    s2, s3 = f32(np.sqrt(.5)), f32(np.sqrt(1. / 3))
    for u in leaves:
        cen, hf = a["c"][u], a["side"][u] / 2
        for ax in range(3):                                 # in a face plane: that component exactly 0
            p = cen.copy()
            p[ax] = f32(cen[ax] + rng.choice([-1, 1]) * hf)
            v = rng.normal(size=3).astype(f32)
            v[ax] = 0.
            v = (v / np.linalg.norm(v)).astype(f32)
            o.append(p - 2 * v); d.append(v)
        corner = (cen + hf).astype(f32)                     # exactly through an edge (2 axes) and a corner (3 axes)
        off = f32(hf / 2)
        for ax in range(3):
            v = np.full(3, s2, f32)
            v[ax] = 0.
            p = corner - np.where(v > 0, off, 0).astype(f32)
            p[ax] = f32(cen[ax] + f32(.25) * hf)
            o.append(p); d.append(v)
            o.append(p); d.append(-v)
        o.append(corner - off); d.append(np.full(3, s3, f32))
        o.append(corner - off); d.append(np.full(3, -s3, f32))
    return case(g["nodes"], g["trans"], o, d, covers=("empty_eq", "guard_zero"))


# ------------------------------------------------------------------------------------------------------ 4. near and far
def dataset_rays(n, seed):
    """Rays from the ngp_fox training cameras' centres through random directions, unit length in fp32."""
    g = workloads.load_ngp_fox()
    P = g["ds_poses"].reshape(-1, 3, 4)
    rng = np.random.default_rng(seed)
    o = P[rng.integers(0, len(P), n), :, 3].astype(f32)
    v = rng.normal(size=(n, 3)).astype(f32) - o * f32(0.8)
    d = (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(f32)
    return o, d


def near_case(which):
    g = golden()
    o, d = dataset_rays(200, seed=4)
    if which in ("near_host_free", "near_host_wanjinyou"):
        return case(g["nodes"], g["trans"], o, d, near={"near_host_free": .05, "near_host_wanjinyou": .01}[which])
    first = O.sampler(g["nodes"], g["trans"], o, d, noise_of(len(o)), 0., 1e8, 1 / 256, False, CAP)
    hit = np.nonzero((first["first_oct_dis"][:, 0] > 0.) & (first["first_oct_dis"][:, 0] < 1e9))[0]   # origin outside the leaf
    r = hit[0]
    b = first["bounds"][r]
    entry = f32(first["first_oct_dis"][r, 0])
    node = first["anchors"][b[0], 1]
    ts = first["t"][b[0]:b[1]][first["anchors"][b[0]:b[1], 1] == node]
    if which == "near_entry":
        return case(g["nodes"], g["trans"], o, d, near=entry, covers=("near_entry",))
    if which == "near_inside":
        return case(g["nodes"], g["trans"], o, d, near=f32((ts[0] + ts[-1]) / 2), covers=("near_past",))
    if which == "near_past_all":
        return case(g["nodes"], g["trans"], o, d, near=2000., covers=("near_past",))
    if which == "near_eq_far":
        return case(g["nodes"], g["trans"], o, d, near=1., far=1., covers=("empty_eq",))
    raise KeyError(which)


NEAR_CASES = ["near_host_free", "near_host_wanjinyou", "near_entry", "near_inside", "near_past_all", "near_eq_far"]


# ------------------------------------------------------------------------------------------------------------ 5. noise
def hop_steps(ref, n):
    """Per ray the sample index k whose step leaves its leaf (the next sample is in another node), or -1."""
    k = np.full(n, -1)
    for r, (b, e) in enumerate(ref["bounds"]):
        if e - b < 2:
            continue
        ch = np.nonzero(ref["anchors"][b + 1:e, 1] != ref["anchors"][b:e - 1, 1])[0]
        if ch.size:
            k[r] = ch[0]
    return k


def hop_sat_tree():
    """The golden tree with a gap: a ray along +x leaves valid leaf A 2^-10 past its origin and meets no valid leaf for 4 units,
    so with a step of a few ulps of 2^-10 the leaf hop's step count is past 2^31."""
    g = golden()
    a = nodes_of(g["nodes"])
    A = pick_leaves(a, 1, seed=5)[0]
    cen, hf = a["c"][A], a["side"][A] / 2
    o = np.array([cen[0] + hf - f32(2. ** -10), cen[1] + f32(.3) * hf, cen[2] - f32(.2) * hf], f32)
    leaves = np.nonzero((a["childs"] < 0).all(1))[0]
    lo, hi = a["c"][leaves] - a["side"][leaves, None] / 2, a["c"][leaves] + a["side"][leaves, None] / 2
    on_line = (lo[:, 1] <= o[1]) & (o[1] <= hi[:, 1]) & (lo[:, 2] <= o[2]) & (o[2] <= hi[:, 2])
    in_gap = on_line & (hi[:, 0] > o[0]) & (lo[:, 0] < o[0] + 4.) & (leaves != A)
    a["trans"][leaves[in_gap]] = -1
    return g, o


def noise_case(which, sbd):
    g = golden()
    o, d = dataset_rays(160, seed=6)
    n = len(o)
    base = dict(sbd=sbd)
    if which == "noise_zero_first":
        nz = noise_of(n)
        nz[:n] = 0.
        return case(g["nodes"], g["trans"], o, d, nz, covers=("step0",), **base)
    if which == "noise_zero_at_hop":
        # With noise 1, the step from sample k of ray r (noise[r + k]) leaves the leaf.  Zero exactly that entry, for rays whose
        # noise window [r, r + k] holds no other zeroed entry: their samples 0..k stay as they were, and sample k + 1 then sits
        # at sample k's t in sample k's leaf instead of in the next leaf.
        sl = 1 / 16                                         # a few samples per leaf: short windows, many rays qualify
        ones = O.sampler(g["nodes"], g["trans"], o, d, noise_of(n), .05, 1e8, sl, sbd, CAP)
        k = hop_steps(ones, n)
        chosen, zeros = [], set()
        for r in np.nonzero(k >= 1)[0]:
            z = r + k[r]
            if z in zeros or any(q <= z <= q + k[q] for q in chosen) or any(r <= y < z for y in zeros):
                continue
            chosen.append(r)
            zeros.add(z)
        nz = noise_of(n)
        nz[sorted(zeros)] = 0.

        def stays_at_hop(ref):
            assert len(chosen) >= 8
            for r in chosen:
                b, kr = ref["bounds"][r, 0], k[r]
                b1 = ones["bounds"][r, 0]
                assert ref["bounds"][r, 1] - b > kr + 1
                np.testing.assert_array_equal(ref["t"][b:b + kr + 1].view(np.uint32), ones["t"][b1:b1 + kr + 1].view(np.uint32))
                assert ones["anchors"][b1 + kr + 1, 1] != ones["anchors"][b1 + kr, 1]       # noise 1 hops here ...
                assert ref["t"][b + kr + 1] == ref["t"][b + kr]                             # ... noise 0 stays put
                assert ref["anchors"][b + kr + 1, 1] == ref["anchors"][b + kr, 1]
        return case(g["nodes"], g["trans"], o, d, nz, sample_l=sl, covers=("step0", "hop"), check=stays_at_hop, **base)
    if which == "noise_zero_run":
        nz = noise_of(n)
        nz[n // 2:n // 2 + CAP + 2] = 0.                    # the rays from n/2 on march with step 0 to the cap
        return case(g["nodes"], g["trans"], o, d, nz, covers=("step0",), check=lambda ref: cap_reached(ref, n // 2), **base)
    if which == "noise_rand_lo":                             # t + step rounds to t: every ray that hits stays at its entry
        return case(g["nodes"], g["trans"], o, d, noise_of(n, 2. ** -24), check=lambda ref: cap_reached(ref, 0), **base)
    if which in ("noise_rand_hi", "noise_train_lo", "noise_train_hi"):
        v = {"noise_rand_hi": 1. - 2. ** -24, "noise_train_lo": .5, "noise_train_hi": 1.5}[which]
        return case(g["nodes"], g["trans"], o, d, noise_of(n, v), covers=("hop",), **base)
    if which == "noise_hop_sat":
        g, p = hop_sat_tree()
        m = 64
        nz = noise_of(m)
        nz[:m] = (2. ** (-40 + np.arange(m) / 3.)).astype(f32)   # the first step's noise sweeps past the window
        near = ulps(2. ** -10, -1)
        return case(g["nodes"], g["trans"], np.tile(p, (m, 1)), np.tile(np.array([1, 0, 0], f32), (m, 1)), nz, near=near,
                    covers=("hop_sat",), **base)
    raise KeyError(which)


def cap_reached(ref, first_ray):
    cnt = np.diff(ref["bounds"], axis=1)[:, 0]
    assert (cnt[first_ray:] == CAP).sum() >= 8, "no ray of the zero-noise run reaches the cap"


NOISE_CASES = ["noise_zero_first", "noise_zero_at_hop", "noise_zero_run", "noise_rand_lo", "noise_rand_hi", "noise_train_lo",
               "noise_train_hi", "noise_hop_sat"]


# ----------------------------------------------------------------------------------------------------------- 6. step size
def step_case(which):
    g = golden()
    o, d = dataset_rays(160, seed=7)
    if which == "step_tiny":
        def one_leaf(ref):
            cnt = np.diff(ref["bounds"], axis=1)[:, 0]
            full = np.nonzero(cnt == CAP)[0]
            assert full.size >= 16
            for r in full:
                b, e = ref["bounds"][r]
                assert (ref["anchors"][b:e, 1] == ref["anchors"][b, 1]).all(), "the cap was not reached inside the first leaf"
        return case(g["nodes"], g["trans"], o, d, sample_l=1e-6, check=one_leaf)

    def all_hops(ref):
        b, e = ref["bounds"][:, 0], ref["bounds"][:, 1]
        node = ref["anchors"][:, 1]
        inner = np.ones(len(node), bool)
        inner[b[e > b]] = False                                     # first sample of a ray
        assert (e - b).max() >= 4
        assert (node[1:][inner[1:]] != node[:-1][inner[1:]]).all(), "a step stayed inside its leaf"
    return case(g["nodes"], g["trans"], o, d, sample_l=4., covers=("hop",), check=all_hops)


STEP_CASES = ["step_tiny", "step_hop_every"]


# ---------------------------------------------------------------------------------------------------------- 7. deep trees
def deep_tree(depth):
    """The golden tree with one corner chain subdivided from its deepest leaf down to a live leaf at `depth`.  Every new level
    gets the continuing internal node (child 0), an invalid leaf (child 2, trans_idx -1), a childless internal node (child 3,
    trans_idx -1) and live leaves; the last level is eight live leaves.  -> (blob, index of the deepest leaf, index of the chain's node at depth MAX_WALK_DEPTH or -1)."""
    g = golden()
    a = nodes_of(g["nodes"]).copy()
    dep = depths(a)
    live = live_leaves(a)
    u = live[np.argmax(dep[live])]
    tr = int(a["trans"][u])
    cur, d, at23 = u, int(dep[u]), -1

    def node(c, side, parent, is_leaf, trans):
        r = np.zeros(1, NODE)[0]
        r["c"], r["side"], r["parent"], r["childs"], r["is_leaf"], r["trans"] = c, side, parent, -1, is_leaf, trans
        return r

    rows_list = list(a)
    while d < depth:
        me = rows_list[cur]
        side = f32(me["side"] / 2)
        kids = []
        for k in range(8):
            off = np.array([(k >> 2) & 1, (k >> 1) & 1, k & 1], f32) * 2 - 1
            c = (me["c"] + off * f32(side / 2)).astype(f32)
            role = k if d + 1 < depth else (0 if k == 0 else 1)
            is_leaf, trans = {0: (1, tr), 1: (1, tr), 2: (1, -1), 3: (0, -1)}.get(role, (1, tr))
            rows_list.append(node(c, side, cur, is_leaf, trans))
            kids.append(len(rows_list) - 1)
        me = rows_list[cur]
        me["childs"] = kids
        me["is_leaf"], me["trans"] = 0, -1
        rows_list[cur] = me
        cur = kids[0]                                        # the chain continues in child 0 (the -x -y -z corner)
        d += 1
        if d == MAX_WALK_DEPTH:
            at23 = cur
        if d < depth:
            rows_list[cur]["is_leaf"], rows_list[cur]["trans"] = 0, -1
    out = np.array(rows_list, NODE)
    return dict(nodes=out.view(np.uint8).reshape(-1).copy(), trans=g["trans"]), cur, at23


def deep_case(depth):
    blob, leaf, at23 = deep_tree(depth)
    a = nodes_of(blob["nodes"])
    rng = np.random.default_rng(8 + depth)
    tgt = a["c"][leaf]
    v = rng.normal(size=(96, 3))
    v[:, 0] = np.abs(v[:, 0]) + .5
    p = (tgt[None] - 2. * v / np.linalg.norm(v, axis=1, keepdims=True)).astype(f32)
    dd = (tgt[None] - p).astype(f32)
    dd = (dd / np.linalg.norm(dd, axis=1, keepdims=True)).astype(f32)
    # rays through the chain's other nodes and past it
    jit = (tgt[None] + rng.normal(size=(32, 3)).astype(f32) * f32(a["side"][leaf] * 4)).astype(f32)
    o = np.concatenate([p, p[:32]])
    d = np.concatenate([dd, ((jit - p[:32]) / np.linalg.norm(jit - p[:32], axis=1, keepdims=True)).astype(f32)])
    return blob, leaf, at23, o, d


def slab_np(o, d, c, side):
    """slab() of oracle/f2_oracle.c in numpy float32, for the node interval of each ray -> (near, far) over [0, 1e8]."""
    hf = f32(side * f32(.5))
    lo = np.where(d > 0, (c - hf - o) / d, (c + hf - o) / d).astype(f32)
    hi = np.where(d > 0, (c + hf - o) / d, (c - hf - o) / d).astype(f32)
    par = np.abs(d) < f32(1e-6)
    ins = (o > c - hf) & (o < c + hf)
    lo = np.where(par, np.where(ins, f32(-1e6), f32(1e6)), lo)
    hi = np.where(par, np.where(ins, f32(1e6), f32(-1e6)), hi)
    return np.maximum(f32(0.), lo.max(1)), np.minimum(f32(1e8), hi.min(1))


DEPTHS = [21, 22, 23, 24, 25]


def check_deep(ref, cov, blob, leaf, at23, depth, o, d):
    a = nodes_of(blob["nodes"])
    assert depths(a)[leaf] == depth
    sampled = set(np.unique(ref["anchors"][:, 1]).tolist())
    if depth <= MAX_WALK_DEPTH:
        assert cov["stack_stop"] == 0
        assert leaf in sampled, f"the live leaf at depth {depth} is never sampled"
    else:
        assert cov["stack_stop"] > 0 and leaf not in sampled
        # truncation: a ray that reaches the depth-23 node of the chain has no sample past its entry
        with np.errstate(divide="ignore", invalid="ignore"):
            near, far = slab_np(o, d, a["c"][at23], a["side"][at23])
        reach = np.nonzero(near < far)[0]
        assert reach.size >= 8
        for r in reach:
            b, e = ref["bounds"][r]
            if e > b:
                assert ref["t"][e - 1] <= near[r]


# ----------------------------------------------------------------------------------------------------------- 8. lenses
def leaf_face_pose():
    a = nodes_of(golden()["nodes"])
    u = pick_leaves(a, 1, seed=9)[0]
    P = np.eye(3, 4, dtype=f32)
    P[:, 3] = a["c"][u]
    P[0, 3] = f32(a["c"][u][0] + a["side"][u] / 2)
    return P


LENSES = [("equirect", dict(height=16)), ("ods", dict(height=12, ipd=0.)), ("ods", dict(height=12, ipd=0.064)),
          ("ods", dict(height=12, ipd=0.5)), ("fisheye", dict(height=20, fov=180.)), ("fisheye", dict(height=20, fov=220.)),
          ("fisheye", dict(height=20, fov=360.)), ("pinhole", dict(height=18, width=24, vfov=60.))]


def lens_rays(kind, kw, pose):
    import torch
    from f2nerf_b200.lens import Lens
    lens = getattr(Lens, kind)(**kw)
    o, dr, valid = lens.rays(pose)
    o, dr = o[valid], dr[valid]
    d = dr / torch.linalg.norm(dr, 2, -1, True)              # what the samplers march (PersSampler.begin_march)
    return o.cpu().numpy(), d.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------- the checks
CASES = {"axis_parallel": axis_parallel, "on_geometry": on_geometry, "grazing": grazing}
CASES.update({k: (lambda k=k: near_case(k)) for k in NEAR_CASES})
CASES.update({k: (lambda k=k: step_case(k)) for k in STEP_CASES})
NOISE = [(k, s) for k in NOISE_CASES for s in (False, True)]
_built = {}


def build(name, sbd=None):
    key = (name, sbd)
    if key not in _built:
        _built[key] = noise_case(name, sbd) if sbd is not None else CASES[name]()
    return _built[key]


def cover(c):
    cov = O.sampler_cover(c["nodes"], c["trans"], c["o"], c["d"], c["noise"], c["near"], c["far"], c["sample_l"], c["sbd"],
                          c["max_hits"])
    for k in c["covers"]:
        assert cov[k] > 0, f"the batch never takes the {k} branch: {cov}"
    assert cov["hop_inf"] == 0 and cov["hop_nan"] == 0
    return cov


def oracle_run(c):
    return O.sampler(c["nodes"], c["trans"], c["o"], c["d"], c["noise"], c["near"], c["far"], c["sample_l"], c["sbd"], c["max_hits"])


def check_case(c, oracle):
    cover(c)
    ref = check_all_modes(dict(nodes=c["nodes"], trans=c["trans"]), oracle, c["o"], c["d"], c["noise"], c["sample_l"], c["sbd"],
                          c["max_hits"], near=c["near"], far=c["far"])
    if c["check"]:
        c["check"](ref)
    return ref


# CPU: the batches cover their branches (the oracle alone)
@pytest.mark.parametrize("name", list(CASES))
def test_case_covers_branch(oracle, name):
    c = build(name)
    cover(c)
    if c["check"]:
        c["check"](oracle_run(c))


@pytest.mark.parametrize("name,sbd", NOISE)
def test_noise_case_covers_branch(oracle, name, sbd):
    c = build(name, sbd)
    cover(c)
    if c["check"]:
        c["check"](oracle_run(c))


@pytest.mark.parametrize("depth", DEPTHS)
def test_deep_tree_depth(oracle, depth):
    blob, leaf, at23, o, d = deep_case(depth)
    a = nodes_of(blob["nodes"])
    dep = depths(a)
    live = live_leaves(a)
    assert dep[live].max() == depth and dep[leaf] == depth
    assert ((a["childs"] < 0).all(1) & (a["is_leaf"] == 0)).any(), "no childless internal node"
    assert ((a["childs"] < 0).all(1) & (a["trans"] < 0)).sum() > 0
    c = case(blob["nodes"], blob["trans"], o, d)
    check_deep(oracle_run(c), cover(c), blob, leaf, at23, depth, o, d)


# GPU: every mode of the device march equals the oracle
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_march_case(oracle, name):
    check_case(build(name), oracle)


@pytest.mark.gpu
@pytest.mark.parametrize("name,sbd", NOISE)
def test_march_noise(oracle, name, sbd):
    check_case(build(name, sbd), oracle)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", DEPTHS)
def test_march_deep_tree(oracle, depth):
    blob, leaf, at23, o, d = deep_case(depth)
    c = case(blob["nodes"], blob["trans"], o, d)
    ref = check_case(c, oracle)
    check_deep(ref, cover(c), blob, leaf, at23, depth, o, d)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,kw", LENSES, ids=[f"{k}-{'-'.join(f'{a}{b}' for a, b in kw.items())}" for k, kw in LENSES])
@pytest.mark.parametrize("pose", ["identity", "leaf_face"])
def test_march_lens_rays(oracle, kind, kw, pose):
    P = np.eye(3, 4, dtype=f32) if pose == "identity" else leaf_face_pose()
    o, d = lens_rays(kind, kw, P)
    g = golden()
    check_case(case(g["nodes"], g["trans"], o, d), oracle)


@pytest.fixture(scope="module")
def lens_renderer():
    """A renderer on the golden tree with the march settings of the cases above (near 0.05, sample_l 1/256, no scale_by_dis)
    and a seeded random field."""
    import torch
    from f2nerf_b200 import GlobalDataPool, Hash3DAnchored, PersSampler, Renderer, SHShader
    g = workloads.load_ngp_fox()
    torch.manual_seed(0)
    gdp = GlobalDataPool()
    sampler = PersSampler(gdp, g["tree_nodes"], g["pers_trans"], g["edge_pool"], near=0.05, sample_l=1 / 256, scale_by_dis=False)
    field = Hash3DAnchored(gdp, log2_table_size=15)
    field.Reset()
    return Renderer(gdp, sampler, field, SHShader(gdp), n_images=1)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,kw", LENSES, ids=[f"{k}-{'-'.join(f'{a}{b}' for a, b in kw.items())}" for k, kw in LENSES])
@pytest.mark.parametrize("pose", ["identity", "leaf_face"])
def test_render_lens_marches_checked_rays(oracle, lens_renderer, kind, kw, pose):
    """RenderLens marches the rays test_march_lens_rays checks: every chunk its tiled loop renders is recorded, and the rays it
    marched (after its own normalisation), its sample counts and first_oct_dis equal the lens rays above and the oracle's march
    of them; its kept counts (after early stop) equal render_forward's on the same rays in one chunk."""
    import torch
    from f2nerf_b200 import VALIDATE
    from f2nerf_b200.eval import RenderLens
    from f2nerf_b200.lens import Lens
    R = lens_renderer
    P = np.eye(3, 4, dtype=f32) if pose == "identity" else leaf_face_pose()
    o, d = lens_rays(kind, kw, P)
    seen, render_forward = [], R.render_forward

    def spy(rays_o, rays_d, **kwargs):
        r = render_forward(rays_o, rays_d, **kwargs)
        s = r._keep[0]
        seen.append((s.rays_o, s.rays_d, s.counts[:s.n_rays], r.first_oct_dis, r.kept_counts))
        return r
    R.render_forward = spy
    try:
        RenderLens(R, getattr(Lens, kind)(**kw), P, ray_batch_size=160)
    finally:
        del R.render_forward
    assert len(seen) >= 2                                        # several chunks, on both lanes
    ro, rd, cnt, first, kept = (torch.cat([s[i].reshape(s[i].shape[0], -1) for s in seen]).cpu().numpy() for i in range(5))
    np.testing.assert_array_equal(ro.view(np.uint32), o.view(np.uint32))
    np.testing.assert_array_equal(rd.view(np.uint32), d.view(np.uint32))
    g = golden()
    ref = O.sampler(g["nodes"], g["trans"], o, d, noise_of(len(o)), 0.05, 1e8, 1 / 256, False, CAP)
    np.testing.assert_array_equal(cnt[:, 0], np.diff(ref["bounds"], axis=1)[:, 0])
    np.testing.assert_array_equal(first.view(np.uint32), ref["first_oct_dis"].view(np.uint32))
    gdp = R.global_data_pool_
    mode, gdp.mode_ = gdp.mode_, VALIDATE
    try:
        with torch.no_grad():
            direct = R.render_forward(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()).kept_counts.cpu().numpy()
    finally:
        gdp.mode_ = mode
    np.testing.assert_array_equal(kept[:, 0], direct)
    assert (kept[:, 0] <= cnt[:, 0]).all() and kept.max() > 0


def milestone_schedules():
    out = {}
    for f in sorted(os.listdir(os.path.join(ROOT, "oracle"))):
        if f.startswith("ref_config_") and f.endswith(".yaml"):
            with open(os.path.join(ROOT, "oracle", f)) as fh:
                cfg = yaml.safe_load(fh)
            out[f] = list(cfg["pts_sampler"]["sub_div_milestones"])
    for name, cfg in workloads.CONFIGS.items():
        assert cfg["ref_yaml"] is None or os.path.basename(cfg["ref_yaml"]) in out, name
    return out


def test_milestone_schedules_listed():
    s = milestone_schedules()
    assert s and max(len(m) for m in s.values()) >= 5


def test_shipped_schedules_stay_walkable():
    """The bound behind test_subdivision_depth_stays_walkable for any scene: the initial octree stops splitting below depth
    max_level (a node at depth max_level still splits, its children are leaves: octree_build.build_tree_nodes, PersSampler.cpp
    ConstructTreeNode), so its leaves lie at depth <= max_level + 1; each milestone splits a leaf once, one level; so a config
    reaches at most max_level + 1 + len(sub_div_milestones), which must be within the levels the march walks."""
    for f in sorted(os.listdir(os.path.join(ROOT, "oracle"))):
        if f.startswith("ref_config_") and f.endswith(".yaml"):
            with open(os.path.join(ROOT, "oracle", f)) as fh:
                cfg = yaml.safe_load(fh)["pts_sampler"]
            assert int(cfg["max_level"]) + 1 + len(cfg["sub_div_milestones"]) <= MAX_WALK_DEPTH, f


@pytest.mark.gpu
@pytest.mark.parametrize("config", sorted(milestone_schedules()))
def test_subdivision_depth_stays_walkable(config):
    """Every milestone of the config's schedule splits the deepest live leaves (and only those): the deepest chain grows one
    level per milestone, the fastest the octree can deepen, and must stay within the levels the march walks."""
    import torch
    from f2nerf_b200 import GlobalDataPool, PersSampler
    g = golden()
    s = PersSampler(GlobalDataPool(), g["nodes"], g["trans"])
    deepest = []
    for _ in milestone_schedules()[config]:
        a = nodes_of(s.tree_nodes_gpu_.cpu().numpy())
        dep, live = depths(a), live_leaves(a)
        top = live[dep[live] == dep[live].max()]
        visit = np.zeros(len(a), np.int32)
        visit[top] = 5
        s.tree_visit_cnt_ = torch.from_numpy(visit).cuda()
        s.ProcOctree(True, True, False)
        a = nodes_of(s.tree_nodes_gpu_.cpu().numpy())
        dep, live = depths(a), live_leaves(a)
        deepest.append(int(dep[live].max()))
    print(f"\n{config}: deepest live leaf per milestone {deepest}")
    assert all(y == x + 1 for x, y in zip(deepest, deepest[1:]))
    assert deepest[-1] <= MAX_WALK_DEPTH


# -------------------------------------------------------------------------------------------- the reference's GetSamples
# near_eq_far stays out: the reference's GetSamples always marches to far 1e8 (PersSampler.cu:322-323).  Trees deeper than
# MAX_WALK_DEPTH stay out too: the reference's 48-int DFS stack has no bounds check (PersSampler.cu:70).
REF_CASES = ["axis_parallel", "on_geometry", "grazing", "near_host_free", "near_host_wanjinyou", "near_entry", "near_inside",
             "near_past_all"]


def ref_batches():
    out = {n: build(n) for n in REF_CASES}
    for depth in DEPTHS:
        if depth <= MAX_WALK_DEPTH:
            blob, _, _, o, d = deep_case(depth)
            out[f"deep{depth}"] = case(blob["nodes"], blob["trans"], o, d)
    return out


@pytest.fixture(scope="module")
def ref_march():
    """Runs every reference case through one oracle/_ref/ref_driver --march call -> {case: (batch, dumps)}."""
    if not os.access(REF_DRIVER, os.X_OK):
        pytest.skip("oracle/_ref/ref_driver not built (the reference's sources were absent at build time)")
    import torch
    batches = ref_batches()
    for pose in ("identity", "leaf_face"):
        P = np.eye(3, 4, dtype=f32) if pose == "identity" else leaf_face_pose()
        for kind, kw in LENSES:
            o, d = lens_rays(kind, kw, P)
            g = golden()
            batches[f"lens_{pose}_{kind}_{len(batches)}"] = case(g["nodes"], g["trans"], o, d)
    batches["train_axis_parallel"] = dict(build("axis_parallel"), train=True)
    work = tempfile.mkdtemp(prefix="f2b_march_ref_")
    try:
        for name, c in batches.items():
            p = os.path.join(work, name)
            os.makedirs(p)
            np.save(os.path.join(p, "tree_nodes.npy"), c["nodes"].reshape(-1))
            np.save(os.path.join(p, "pers_trans.npy"), c["trans"].reshape(-1))
            np.save(os.path.join(p, "rays_o.npy"), c["o"])
            np.save(os.path.join(p, "rays_d.npy"), c["d"])
            np.save(os.path.join(p, "params.npy"), np.array([c.get("train", False), c["near"], c["sample_l"], c["sbd"],
                                                            c["max_hits"], 4242], f32))
        torch.cuda.synchronize()
        r = subprocess.run([REF_DRIVER, "--march", os.path.join(ROOT, "oracle", "ref_config_ngp_fox.yaml"), work], cwd=ROOT,
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        out = {}
        for name, c in batches.items():
            p = os.path.join(work, name)
            out[name] = (c, {f[:-4]: np.load(os.path.join(p, f)) for f in os.listdir(p) if f.endswith(".npy")})
        return out
    finally:
        shutil.rmtree(work, ignore_errors=True)


@pytest.mark.gpu
def test_march_vs_reference(ref_march, oracle):
    """The reference's GetSamples, the oracle and the device march agree bit for bit on every reference case.  The reference
    normalises the directions itself, so the others march what it marched (rays_d_used); TRAIN takes the noise it drew."""
    for name, (c, ref) in ref_march.items():
        d = ref["rays_d_used"].astype(f32)
        c = dict(c, d=d, noise=ref["noise"].astype(f32) if c.get("train") else c["noise"])
        orc = check_case(dict(c, covers=()), oracle)
        np.testing.assert_array_equal(ref["bounds"], orc["bounds"], err_msg=name)
        for k in ("first_oct_dis", "t", "dt", "pts", "dirs"):
            np.testing.assert_array_equal(ref[k].astype(f32).reshape(orc[k].shape).view(np.uint32), orc[k].view(np.uint32),
                                          err_msg=f"{name} {k}")
        np.testing.assert_array_equal(ref["anchors"].reshape(-1, 2), orc["anchors"][:, :2], err_msg=name)
