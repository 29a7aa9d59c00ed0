"""CPU-only checks of the oracle restatement and the host-side logic (run with -m "not gpu").

The oracle is checked against independent statements of the same maths (numpy / plain PyTorch fp32-fp64)
and against known answers recorded from the reference (SURVEY.md §8a probes); the golden-vector pin
against outputs of the reference itself lives in test_golden_ref.py.
"""
import numpy as np
import pytest
import torch

from conftest import make_rays


def test_struct_layouts_match_reference_bytes():
    import synth_scene as S
    assert S.TREE_NODE.itemsize == 64 and S.TRANS_INFO.itemsize == 544 and S.EDGE_POOL.itemsize == 64
    assert S.TREE_NODE.fields["childs"][1] == 20 and S.TREE_NODE.fields["trans_idx"][1] == 56
    assert S.TRANS_INFO.fields["weight"][1] == 384 and S.TRANS_INFO.fields["dis_summary"][1] == 540


def test_search_order_table_known_answer(oracle):
    """Rows recorded from the reference's own std::sort (SURVEY.md §8a a3)."""
    import ctypes
    want = ["7 3 5 1 6 2 4 0", "6 2 4 0 7 3 5 1", "5 1 7 3 4 0 6 2", "4 0 6 2 5 1 7 3",
            "3 7 1 5 2 6 0 4", "2 6 0 4 3 7 1 5", "1 5 3 7 0 4 2 6", "0 4 2 6 1 5 3 7"]
    # the oracle keeps its table internal; re-derive through the closed form the CUDA kernel uses and
    # through a python transcription of the comparator, and check both against the recorded rows.
    import functools
    for st in range(8):
        def cmp(a, b):
            bt = (a ^ b) & -(a ^ b)
            return -1 if ((a & bt) ^ (st & bt)) else 1
        row = sorted(range(8), key=functools.cmp_to_key(cmp))
        closed = [((~st) & 7) ^ (((k & 1) << 2) | (k & 2) | ((k >> 2) & 1)) for k in range(8)]
        assert " ".join(map(str, row)) == want[st]
        assert closed == row


def test_sampler_structure(scene, oracle):
    o, d, dn, _ = make_rays(scene, 64)
    noise = (np.random.default_rng(0).random(1024 + 64 + 10, dtype=np.float32) + .5).astype(np.float32)
    s = oracle.sampler(scene["nodes"], scene["trans"], o, dn, noise, 0.05, 1e8, 1 / 256, False, 1024)
    b = s["bounds"]
    assert (b[:, 0] <= b[:, 1]).all() and b[0, 0] == 0 and (b[1:, 0] == b[:-1, 1]).all()
    assert b[-1, 1] == s["pts"].shape[0] and ((b[:, 1] - b[:, 0]) <= 1024).all()
    from synth_scene import view_nodes
    nodes = view_nodes(scene["nodes"])
    for r in range(64):
        sl = slice(b[r, 0], b[r, 1])
        t = s["t"][sl]
        assert (np.diff(t) > 0).all()                                    # front to back
        assert (t > s["first_oct_dis"][r, 0]).all()                      # first point of a ray is skipped
        # dt == sample_l * noise[ray + k] up to the (step*den)/den round trip
        k = np.arange(t.size)
        np.testing.assert_allclose(s["dt"][sl], noise[r + k] / 256, rtol=3e-7)
        np.testing.assert_array_equal(nodes["trans_idx"][s["anchors"][sl, 1]], s["anchors"][sl, 0])
        np.testing.assert_array_equal(s["dirs"][sl], np.broadcast_to(dn[r], (t.size, 3)))


def test_warp_matches_plain_numpy(scene, oracle):
    """QueryFrameTransform in float64 numpy vs the oracle's fp32 tree-ordered evaluation."""
    from synth_scene import view_trans
    o, d, dn, _ = make_rays(scene, 16)
    noise = np.ones(1024 + 16 + 10, np.float32)
    s = oracle.sampler(scene["nodes"], scene["trans"], o, dn, noise, 0.05, 1e8, 1 / 256, False, 1024)
    trans = view_trans(scene["trans"])
    ray_of = np.repeat(np.arange(16), s["bounds"][:, 1] - s["bounds"][:, 0])
    sel = np.random.default_rng(0).choice(s["pts"].shape[0], 200, replace=False)
    for i in sel:
        T = trans[s["anchors"][i, 0]]
        x = o[ray_of[i]].astype(np.float64) + dn[ray_of[i]].astype(np.float64) * float(s["t"][i])
        xz = np.einsum("nrk,k->nr", T["w2xz"].astype(np.float64), np.append(x, 1.0))
        ref = T["weight"].astype(np.float64) @ (xz[:, 0] / xz[:, 1])
        np.testing.assert_allclose(s["pts"][i], ref, rtol=2e-4, atol=2e-5)


def test_hash_fwd_matches_numpy(oracle, hash_params):
    hp = hash_params
    rng = np.random.default_rng(1)
    pts = (rng.random((50, 3), dtype=np.float32) * 2 - 1)
    vol = rng.integers(0, hp["V"], 50).astype(np.int32)
    scales = oracle.level_scales()
    np.testing.assert_allclose(scales, 2.0 ** (3 + 7 * np.arange(16) / 15), rtol=1e-6)   # fp32 exponent rounding
    got = oracle.hash_fwd(hp["table"], hp["prim"], hp["bias"], hp["V"], hp["local_size"], scales, pts, vol).astype(np.float64)
    flat = hp["table"].reshape(-1).astype(np.float64)
    L = hp["local_size"]
    for i in range(50):
        x = (pts[i].astype(np.float64) + 1) / 2
        for l in range(16):
            p = x * float(scales[l]) + hp["bias"][l * hp["V"] + vol[i]].astype(np.float64)
            c = np.floor(p); f = p - c
            pr = hp["prim"][l, vol[i]].astype(np.uint32).astype(np.uint64)
            acc = np.zeros(2)
            for dx in (0, 1):
                for dy in (0, 1):
                    for dz in (0, 1):
                        h = ((np.uint64(c[0] + dx) * pr[0]) & 0xffffffff) ^ ((np.uint64(c[1] + dy) * pr[1]) & 0xffffffff) ^ \
                            ((np.uint64(c[2] + dz) * pr[2]) & 0xffffffff)
                        idx = int(h % L)
                        w = (f[0] if dx else 1 - f[0]) * (f[1] if dy else 1 - f[1]) * (f[2] if dz else 1 - f[2])
                        acc += w * flat[l * L + idx * 2: l * L + idx * 2 + 2]       # half-element level offset (quirk)
            np.testing.assert_allclose(got[i, 2 * l: 2 * l + 2], acc, rtol=3e-3, atol=2e-3)


def test_mlp_matches_plain_torch(oracle):
    """fp32 PyTorch reference of the same op on the same fp16-rounded operands."""
    rng = np.random.default_rng(2)
    for nh in (0, 1):
        x = (rng.standard_normal((300, 32)) * .5).astype(np.float16)
        p = (oracle.mlp_init(32, nh) * 2).astype(np.float16)
        out, hid = oracle.mlp_fwd(x, p, nh, save_hidden=True)
        pt = torch.from_numpy(p.astype(np.float32))
        W0 = pt[:2048].reshape(64, 32); Wh = pt[2048:2048 + nh * 4096].reshape(nh, 64, 64); Wo = pt[2048 + nh * 4096:].reshape(16, 64)
        h = torch.relu(torch.from_numpy(x.astype(np.float32)) @ W0.T).half().float()
        np.testing.assert_allclose(hid[0].astype(np.float32), h.numpy(), rtol=2e-3, atol=1e-3)
        for k in range(nh):
            h = torch.relu(h @ Wh[k].T).half().float()
        o = (h @ Wo.T).half().float()
        np.testing.assert_allclose(out.astype(np.float32), o.numpy(), rtol=4e-3, atol=2e-3)
        # backward vs autograd (fp64) of the un-rounded network: loose, the oracle rounds activations to fp16
        xt = torch.from_numpy(x.astype(np.float64)).requires_grad_(True)
        Ws = [W0.double().requires_grad_(True)] + [Wh[k].double().requires_grad_(True) for k in range(nh)] + [Wo.double().requires_grad_(True)]
        a = xt
        for W in Ws[:-1]:
            a = torch.relu(a @ W.T)
        y = a @ Ws[-1].T
        g = (rng.standard_normal((300, 16)) * .1).astype(np.float16)
        y.backward(torch.from_numpy(g.astype(np.float64)))
        din, dp = oracle.mlp_bwd(g, x, hid, p, nh)
        ref_dp = np.concatenate([W.grad.numpy().reshape(-1) for W in Ws])
        assert np.abs(dp - ref_dp).max() <= 0.03 * np.abs(ref_dp).max()
        assert np.abs(din.astype(np.float64) - xt.grad.numpy()).max() <= 0.03 * np.abs(xt.grad.numpy()).max()


def test_mlp_init_stream(oracle):
    from f2nerf_b200.field import tcnn_xavier_params
    p = oracle.mlp_init(32, 0)
    assert p.shape == (3072,) and np.abs(p[:2048]).max() <= np.sqrt(6 / 96) and np.abs(p[2048:]).max() <= np.sqrt(6 / 80)
    np.testing.assert_array_equal(tcnn_xavier_params(32, 1).numpy(), p)
    np.testing.assert_array_equal(tcnn_xavier_params(32, 2).numpy(), oracle.mlp_init(32, 1))


def test_composite_matches_plain_torch(oracle):
    rng = np.random.default_rng(3)
    lens = np.array([0, 5, 37, 1, 64, 0, 130], np.int32)
    b = np.stack([np.cumsum(lens) - lens, np.cumsum(lens)], -1).astype(np.int32)
    P = int(lens.sum())
    logit = (rng.standard_normal(P) * 2 + 3).astype(np.float32)
    dt = (rng.random(P, dtype=np.float32) * .01 + .002)
    t = np.sort(rng.random(P, dtype=np.float32) * 5)
    rgb = rng.random((P, 3), dtype=np.float32); bg = rng.random((7, 3), dtype=np.float32)
    colors, disp, depth, w = oracle.composite_fwd(logit, 1, rgb, dt, t, b, bg)
    for r in range(7):
        sl = slice(b[r, 0], b[r, 1])
        tau = torch.exp(torch.tensor(logit[sl]) - 3) * torch.tensor(dt[sl])
        A = torch.cumsum(tau, 0) - tau
        wr = torch.exp(-A) * (1 - torch.exp(-tau))
        lt = torch.exp(-tau.sum())
        np.testing.assert_allclose(w[sl], wr.numpy(), rtol=2e-5, atol=1e-7)
        np.testing.assert_allclose(colors[r], ((wr[:, None] * torch.tensor(rgb[sl])).sum(0) + lt * torch.tensor(bg[r])).numpy(), rtol=2e-5, atol=1e-6)
        ts = torch.tensor(t[sl]) + 1e-2
        np.testing.assert_allclose(disp[r], float((wr / ts).sum()), rtol=2e-5, atol=1e-6)
        np.testing.assert_allclose(depth[r], float((wr * ts).sum() / (1 - lt + 1e-4)), rtol=2e-5, atol=1e-6)
    # empty rays return the background / zeros (Renderer.cpp:83-97 semantics for empty segments)
    np.testing.assert_array_equal(colors[0], bg[0]); assert disp[0] == 0 and depth[0] == 0
    # early stop: mask == (T > 1e-4), bounds == cumsum of kept
    wq, a, keep, nb, tot = oracle.early_stop(logit + 6, 1, dt, b)
    assert tot == keep.sum() and (nb[:, 1] - nb[:, 0]).sum() == tot and tot < P
    nb2, tot2 = oracle.filter_bounds(keep, b)
    np.testing.assert_array_equal(nb, nb2)


def test_octree_votes_small(oracle):
    """Hand-checked case of MarkVistNodeKernel + stat update."""
    b = np.array([[0, 5]], np.int32)
    oct_idx = np.array([2, 2, 3, 3, 3], np.int32)
    w = np.array([0.5, 0.0, 0.0001, 0.0002, 0.0], np.float32)       # node 2 occupied (0.5 > min(.05,.01)), node 3 not
    a = np.array([0.001, 0.0, 0.5, 0.0, 0.0], np.float32)            # alpha: node 3 occupied, node 2 not
    vc = np.zeros(5, np.int32)
    vw, va, mk = oracle.mark_visit(b, oct_idx, 1, w, a, 5, vc)
    assert vw.tolist() == [-1, -1, 512, -1, -1] and va.tolist() == [-1, -1, -1, 32, -1]
    assert mk.tolist() == [0, 0, 1, 1, 0] and vc.tolist() == [0, 0, 2, 3, 0]
    from synth_scene import TREE_NODE, to_bytes, view_nodes
    nodes = np.zeros(5, TREE_NODE); nodes["trans_idx"] = np.arange(5)
    blob = to_bytes(nodes)
    sw, sa = np.array([1000, 0, 0, 0, 5], np.int32), np.array([1000, 0, 0, 0, 5], np.int32)
    oracle.update_stats(vw, va, mk, sw, sa, blob)
    assert sw.tolist() == [1000, 0, 512, -1, 5] and sa.tolist() == [1000, 0, -1, 32, 5]
    assert view_nodes(blob)["trans_idx"].tolist() == [0, 1, -1, -1, 4]


def test_scene_builder_is_consistent(scene):
    from synth_scene import view_edges, view_nodes, view_trans
    nodes, trans, edges = view_nodes(scene["nodes"]), view_trans(scene["trans"]), view_edges(scene["edges"])
    valid = nodes[nodes["trans_idx"] >= 0]
    assert len(trans) == len(valid) > 10 and len(edges) > 0
    assert sorted(valid["trans_idx"].tolist()) == list(range(len(trans)))
    for n in nodes:
        for c in n["childs"]:
            if c >= 0:
                assert nodes[c]["parent"] >= 0 and abs(nodes[c]["side_len"] * 2 - n["side_len"]) < 1e-6
    assert (edges["t_idx_a"] < len(trans)).all() and (edges["t_idx_b"] < len(trans)).all()


def _tree(blob):
    t = np.ascontiguousarray(blob).view(np.uint8).reshape(-1, 64)
    i = t.view(np.int32)
    return dict(center=t.view(np.float32)[:, :3], side=t.view(np.float32)[:, 3], parent=i[:, 4], childs=i[:, 5:13],
                leaf=t[:, 52] != 0, trans=i[:, 14])


def test_octree_proc_invariants(scene, oracle):
    """ProcOctree restatement (SURVEY 8f N2) on the synthetic octree with random dead leaves: structural invariants of the
    result (links consistent, no dead leaf / single-child chain left, pre-order numbering, children geometry, stats)."""
    rng = np.random.default_rng(3)
    nodes = scene["nodes"].copy()
    t = _tree(nodes)
    live = np.nonzero(t["leaf"] & (t["trans"] >= 0))[0]
    kill = rng.choice(live, len(live) // 3, replace=False)
    nodes.view(np.int32).reshape(-1, 16)[kill, 14] = -1
    n = nodes.size // 64
    w, a = rng.integers(-50, 3000, n).astype(np.int32), rng.integers(-50, 3000, n).astype(np.int32)
    visit = rng.integers(0, 10, n).astype(np.int32)
    for subdivide in (False, True):
        on, ow, oa = oracle.octree_proc(nodes, w, a, visit, subdivide)
        o = _tree(on)
        m = o["parent"].shape[0]
        assert o["parent"][0] == -1 and (o["parent"][1:] >= 0).all() and (o["parent"][1:] < np.arange(1, m)).all()
        for u in range(m):
            ch = o["childs"][u][o["childs"][u] >= 0]
            assert (o["parent"][ch] == u).all()
            if o["leaf"][u]:
                assert len(ch) == 0 and o["trans"][u] >= 0                      # only live leaves survive
            else:
                assert o["trans"][u] < 0 and len(ch) >= (1 if u == 0 else 2)     # no single-child chains below the root
        # pre-order: a node's first child follows it directly
        if subdivide:
            for u in range(m):
                ch = o["childs"][u][o["childs"][u] >= 0]
                if len(ch):
                    assert ch[0] == u + 1 and (np.diff(ch) > 0).all()
        t2 = _tree(nodes)                                                          # the damaged input tree
        live_before = int((t2["leaf"] & (t2["trans"] >= 0)).sum())
        n_live_after = int((o["leaf"]).sum())
        if not subdivide:
            assert n_live_after == live_before
        else:                                                                      # each visited (> 4) live leaf -> 8 children
            lv = np.nonzero(t2["leaf"] & (t2["trans"] >= 0))[0]
            split = int((visit[lv] > 4).sum())
            assert n_live_after == live_before + 7 * split
            # children are the octants of their parent: centre +- side/4, half the side, parent's old trans_idx
            for u in range(m):
                ch = o["childs"][u]
                if (ch >= 0).all() and o["leaf"][ch].all() and np.allclose(o["side"][ch], o["side"][u] / 2) and \
                        len(set(o["trans"][ch])) == 1:
                    off = (o["center"][ch] - o["center"][u]) / (o["side"][u] / 4)
                    if np.allclose(np.abs(off), 1):
                        want = np.array([[(st >> 2) & 1, (st >> 1) & 1, st & 1] for st in range(8)]) * 2 - 1
                        np.testing.assert_array_equal(off, want)
        assert ow.shape[0] == m and oa.shape[0] == m


@pytest.mark.parametrize("schedule", ["compact", "milestone", "brute", "milestone+compact", "two-due"])
def test_train_loop_octree_invariants(scene, oracle, schedule):
    """The multi-step octree driver (tests/oracle_train_loop.py: votes, subdivision milestones, MarkInvisibleNodes, periodic
    compaction) over eight iterations on synthetic weights — leaves inside a ball around the origin are occupied, the others
    empty, statistics start at the pruning threshold.  After every step: links consistent, no dead leaf left by a compaction,
    split leaves have their 8 octants, visit counts zero after ProcOctree, milestones consumed from the back; every schedule
    prunes and renumbers, the milestone schedules subdivide."""
    import oracle_train_loop as TL
    ms, compact_freq = TL.SCHEDULES[schedule]
    n = scene["nodes"].size // 64
    rng = np.random.default_rng(2)
    st = TL.OctreeState(scene["nodes"], rng.integers(0, 3, n), rng.integers(0, 3, n), ms)
    cams = TL.scene_cameras(scene["scene"], 6)
    t0 = TL.tree_view(scene["nodes"])
    radius = np.median(np.linalg.norm(t0["center"][t0["leaf"] & (t0["trans"] >= 0)], axis=1))
    counts, kinds, splits = [n], [], 0
    for it in range(1, TL.N_ITERS + 1):
        n_rays = (150, 97)[it % 2]
        o, d, dn, _ = make_rays(scene, n_rays, seed=40 + it)
        noise = (np.random.default_rng(it).random(1024 + n_rays + 10, dtype=np.float32) + .5).astype(np.float32)
        s = oracle.sampler(st.nodes, scene["trans"], o, dn, noise, 0.05, 1e8, 1 / 64, True, 1024)
        assert s["pts"].shape[0] > 0 and s["anchors"][:, 1].max() < st.n_nodes
        t = TL.tree_view(st.nodes)
        assert t["leaf"][s["anchors"][:, 1]].all() and (t["trans"][s["anchors"][:, 1]] == s["anchors"][:, 0]).all()
        occupied = np.linalg.norm(t["center"][s["anchors"][:, 1]], axis=1) < radius
        w = np.where(occupied, np.float32(.5), np.float32(0))
        before = list(st.milestones)
        log = TL.train_step(st, it, s["bounds"], s["anchors"], w, w, cams, compact_freq)
        TL.check_maintain_log(log, st, before, it, compact_freq)
        counts.append(st.n_nodes)
        kinds += [k for k, *_ in log]
        splits += sum(int(TL.tree_view(a)["leaf"].sum()) > int((TL.tree_view(b)["leaf"] & (TL.tree_view(b)["trans"] >= 0)).sum())
                      for k, _, b, _, a in log if k == "subdivide")
    assert st.milestones == [] and len(set(counts)) > 1
    assert kinds.count("subdivide") == len(ms) and (not ms or splits >= 1)
    assert min(counts) < n or schedule == "milestone"                # dead leaves were dropped (the milestone schedule grows)


def test_img2world_rays_undistorted_closed_form(oracle):
    """Ray generation restatement (SURVEY 8f N3): with zero lens distortion the Newton iteration is a no-op and the ray is
    R [ (j+.5-cx)/fx, -(i+.5-cy)/fy, -1 ]; with distortion, re-distorting the undistorted point returns the pixel."""
    rng = np.random.default_rng(4)
    n_cam, n = 3, 500
    poses = rng.standard_normal((n_cam, 3, 4)).astype(np.float32)
    intri = np.tile(np.array([[600., 0, 320.], [0, 610., 240.], [0, 0, 1]], np.float32), (n_cam, 1, 1))
    cam = rng.integers(0, n_cam, n).astype(np.int32)
    ij = np.stack([rng.integers(0, 480, n), rng.integers(0, 640, n)], -1).astype(np.int32)
    ro, rd = oracle.img2world_rays(poses, intri, np.zeros((n_cam, 4), np.float32), cam, ij)
    u = (ij[:, 1] + .5 - 320.) / 600.
    v = (ij[:, 0] + .5 - 240.) / 610.
    want = np.einsum("nij,nj->ni", poses[cam][:, :, :3].astype(np.float64), np.stack([u, -v, -np.ones(n)], -1))
    np.testing.assert_allclose(rd, want, rtol=2e-6, atol=2e-6)
    np.testing.assert_array_equal(ro, poses[cam][:, :, 3])
    dist = np.tile(np.array([0.06, -0.08, -0.002, -0.0025], np.float32), (n_cam, 1))
    ro2, rd2 = oracle.img2world_rays(poses, intri, dist, cam, ij)
    # back to camera space, re-apply the distortion model (Dataset.cu:16-28): must land on the pixel's normalised coords
    dcam = np.einsum("nji,nj->ni", poses[cam][:, :, :3].astype(np.float64), rd2.astype(np.float64))     # R^T d
    if not np.allclose(np.abs(np.linalg.det(poses[cam][:, :, :3].astype(np.float64))), 1, atol=1e-3):
        dcam = np.linalg.solve(poses[cam][:, :, :3].astype(np.float64), rd2.astype(np.float64)[..., None])[..., 0]
    uu, vv = dcam[:, 0] / -dcam[:, 2], -dcam[:, 1] / -dcam[:, 2]
    k1, k2, p1, p2 = (float(x) for x in dist[0])
    r2 = uu * uu + vv * vv
    radial = k1 * r2 + k2 * r2 * r2
    du = uu * radial + 2 * p1 * uu * vv + p2 * (r2 + 2 * uu * uu)
    dv = vv * radial + 2 * p2 * uu * vv + p1 * (r2 + 2 * vv * vv)
    np.testing.assert_allclose(uu + du, u, atol=5e-5)
    np.testing.assert_allclose(vv + dv, v, atol=5e-5)


# ---- edge cases the reference's own flow produces: rays that hit nothing, zero rays, ragged / empty segments ---------------
def test_sampler_rays_that_miss_the_scene(scene, oracle):
    """A ray starting far outside and pointing away crosses no leaf: empty [s,s) bounds, first_oct_dis stays at its
    1e9 sentinel (PersSampler.cu:374), neighbours are unaffected (mixed with hitting rays, as in a training batch)."""
    o, d, dn, _ = make_rays(scene, 8)
    o2, dn2 = o.copy(), dn.copy()
    o2[[2, 5]] = np.float32([1e4, 1e4, 1e4]); dn2[[2, 5]] = np.float32([0.57735026, 0.57735026, 0.57735026])
    noise = np.ones(1024 + 8 + 10, np.float32)
    full = oracle.sampler(scene["nodes"], scene["trans"], o, dn, noise, 0.05, 1e8, 1 / 256, False, 1024)
    s = oracle.sampler(scene["nodes"], scene["trans"], o2, dn2, noise, 0.05, 1e8, 1 / 256, False, 1024)
    b, bf = s["bounds"], full["bounds"]
    for r in (2, 5):
        assert b[r, 0] == b[r, 1]
        assert s["first_oct_dis"][r, 0] >= 1e8
    for r in (0, 1, 3, 4, 6, 7):                                          # same samples as in the all-hitting batch
        assert b[r, 1] - b[r, 0] == bf[r, 1] - bf[r, 0]
        np.testing.assert_array_equal(s["pts"][b[r, 0]:b[r, 1]], full["pts"][bf[r, 0]:bf[r, 1]])
        np.testing.assert_array_equal(s["anchors"][b[r, 0]:b[r, 1]], full["anchors"][bf[r, 0]:bf[r, 1]])
    assert b[-1, 1] == s["pts"].shape[0]


def test_sampler_zero_rays(scene, oracle):
    z3 = np.zeros((0, 3), np.float32)
    s = oracle.sampler(scene["nodes"], scene["trans"], z3, z3, np.ones(1034, np.float32), 0.05, 1e8, 1 / 256, False, 1024)
    assert s["bounds"].shape == (0, 2) and s["pts"].shape[0] == 0 and s["t"].shape[0] == 0


def test_composite_and_flex_ops_on_ragged_and_empty_segments(oracle):
    """Segments of length 0, 1 and many in one batch: an empty ray renders the background with zero disparity / depth
    (Renderer.cpp:205-218 with nothing accumulated), FlexOps sums over [s,s) are 0 (FlexOps.cu:24-47)."""
    rng = np.random.default_rng(3)
    lens = np.array([0, 1, 7, 0, 130, 1, 0], np.int32)
    ends = np.cumsum(lens).astype(np.int32)
    bounds = np.stack([ends - lens, ends], 1).astype(np.int32)
    P, R = int(ends[-1]), len(lens)
    logit = rng.normal(size=P).astype(np.float32) * 2
    rgb = rng.random((P, 3), dtype=np.float32)
    dt = (rng.random(P, dtype=np.float32) * .01 + .001).astype(np.float32)
    t = np.concatenate([np.cumsum(dt[s:e]) + .1 for s, e in bounds]).astype(np.float32) if P else np.zeros(0, np.float32)
    bg = rng.random((R, 3), dtype=np.float32)
    colors, disp, depth, w = oracle.composite_fwd(logit, 1, rgb, dt, t, bounds, bg)
    for r in np.flatnonzero(lens == 0):
        np.testing.assert_array_equal(colors[r], bg[r])
        assert disp[r] == 0 and depth[r] == 0
    # independent float64 statement per ray
    for r, (s, e) in enumerate(bounds):
        sig = np.exp(logit[s:e].astype(np.float64) - 3.)                  # TruncExp(x - 3): the oracle's density activation
        a = 1 - np.exp(-sig * dt[s:e])
        T = np.concatenate([[1.], np.cumprod(1 - a)[:-1]]) if e > s else np.zeros(0)
        ww = a * T
        np.testing.assert_allclose(w[s:e], ww, rtol=2e-5, atol=1e-7)
        np.testing.assert_allclose(colors[r], (ww[:, None] * rgb[s:e]).sum(0) + (1 - ww.sum()) * bg[r], rtol=2e-5, atol=2e-6)
    fs = oracle.flex_sum(w, bounds)
    assert (fs[lens == 0] == 0).all()
    np.testing.assert_allclose(fs, [w[s:e].astype(np.float64).sum() for s, e in bounds], rtol=1e-5, atol=1e-7)
    acc = oracle.flex_accumulate(w, bounds, False)                      # exclusive prefix inside each segment
    for s, e in bounds:
        if e > s:
            assert acc[s] == 0
            np.testing.assert_allclose(acc[s:e], np.concatenate([[0.], np.cumsum(w[s:e].astype(np.float64))[:-1]]), rtol=1e-5, atol=1e-7)
    # early stop and the bound filter keep segment order and emptiness
    ww, aa, keep, nb, tot = oracle.early_stop(logit, 1, dt, bounds)
    nb2, tot2 = oracle.filter_bounds(keep, bounds)
    np.testing.assert_array_equal(nb, nb2)
    assert tot == tot2 == int(keep.sum()) and nb[-1, 1] == tot
    assert ((nb[:, 1] - nb[:, 0]) == [int(keep[s:e].sum()) for s, e in bounds]).all()
