"""The octree through consecutive TRAIN iterations, on the CPU: PersSampler::UpdateOctNodes (PersSampler.cu:536-614) chained
from the oracle pieces — the occupancy votes of a step (MarkVistNodeKernel, the statistics update, MarkInvalidNodes), then the
tail that changes the tree: at each due subdivision milestone ProcOctree(subdivide) -> MarkInvisibleNodes -> ProcOctree(compact),
and the periodic compaction every ``compact_freq`` iterations.

Test infrastructure (see oracle/f2_oracle.c): tests/test_gpu_train_maintenance.py follows PersSampler.maintain with it step by
step; tests/test_oracle_cpu.py runs it on synthetic weights and checks the structural invariants below.
"""
import numpy as np

import oracle_lib as O


# (subdivision milestones, consumed from the back; compact_freq) over iterations 1..8
SCHEDULES = {
    "compact": ([], 3),                   # compaction alone, at 3 and 6
    "milestone": ([6, 3], 1000),          # subdivisions at 3 and 6, no periodic compaction
    "brute": ([0], 4),                    # a milestone <= 0 splits every leaf on the first call; compactions at 4 and 8
    "milestone+compact": ([4], 4),        # both on iteration 4: the tree is compacted twice
    "two-due": ([4, 5], 1000),            # 5 is at the back: nothing at 4, both at 5 (the loop runs twice)
}
N_ITERS = 8


class OctreeState:
    """What PersOctree / PersSampler keep across iterations: the TreeNode blob, the two per-node statistics, the visit counts
    since the last ProcOctree and the subdivision milestones still to come (consumed from the back)."""

    def __init__(self, nodes, weight_stats, alpha_stats, milestones=()):
        self.nodes = np.ascontiguousarray(nodes, np.uint8).reshape(-1).copy()
        self.weight_stats = np.ascontiguousarray(weight_stats, np.int32).copy()
        self.alpha_stats = np.ascontiguousarray(alpha_stats, np.int32).copy()
        self.visit_cnt = np.zeros(self.n_nodes, np.int32)
        self.milestones = [int(m) for m in milestones]

    @property
    def n_nodes(self):
        return self.nodes.size // 64


def scene_cameras(scene, n_cams=None, bound=(0.05, 6.0)):
    """(intri [n,3,3], w2c [n,3,4], bounds [n,2]) of the synthetic scene's first ``n_cams`` cameras, as MarkInvisibleNodes
    takes them"""
    c2w = np.asarray(scene.c2w, np.float32)[:n_cams, :3, :4]
    R, t = c2w[:, :, :3], c2w[:, :, 3]
    w2c = np.concatenate([R.transpose(0, 2, 1), -(R.transpose(0, 2, 1) @ t[:, :, None])], 2).astype(np.float32)
    n = w2c.shape[0]
    intri = np.tile(np.array([[255., 0, 100.], [0, 255., 56.], [0, 0, 1]], np.float32), (n, 1, 1))
    return intri, np.ascontiguousarray(w2c), np.tile(np.array(bound, np.float32), (n, 1))


def tree_view(nodes):
    t = np.ascontiguousarray(nodes).view(np.uint8).reshape(-1, 64)
    i = t.view(np.int32)
    return dict(center=t.view(np.float32)[:, :3], side=t.view(np.float32)[:, 3], parent=i[:, 4], childs=i[:, 5:13],
                leaf=t[:, 52] != 0, trans=i[:, 14])


def cast_votes(state, bounds, anchors, weights, alphas):
    """PersSampler.cu:536-603: ``bounds`` [R,2] / ``anchors`` [P,3] of the step's samples, the early-stop pass's weights and
    alphas [P].  Statistics, visit counts and the pruned leaves (trans_idx = -1) change in place."""
    oct_idx = np.ascontiguousarray(anchors, np.int32).reshape(-1)[1:].copy()
    vw, va, mk = O.mark_visit(bounds, oct_idx, 3, weights, alphas, state.n_nodes, state.visit_cnt)
    O.update_stats(vw, va, mk, state.weight_stats, state.alpha_stats, state.nodes)
    return vw, va, mk


def proc_octree(state, subdivide, brute_force=False):
    state.nodes, state.weight_stats, state.alpha_stats = O.octree_proc(state.nodes, state.weight_stats, state.alpha_stats,
                                                                       state.visit_cnt, subdivide, brute_force)
    state.visit_cnt = np.zeros(state.n_nodes, np.int32)


def maintain(state, iter_step, cameras, compact_freq):
    """PersSampler.cu:604-614.  Returns one record per ProcOctree call: (kind, brute_force, tree before, visit counts before,
    tree after) with kind "subdivide" / "compact"."""
    log = []

    def proc(kind, brute=False):
        before, visit = state.nodes.copy(), state.visit_cnt.copy()
        proc_octree(state, kind == "subdivide", brute)
        log.append((kind, brute, before, visit, state.nodes.copy()))

    while state.milestones and state.milestones[-1] <= iter_step:
        proc("subdivide", state.milestones[-1] <= 0)
        state.nodes = O.mark_invisible(state.nodes, *cameras).reshape(-1)
        proc("compact")
        state.milestones.pop()
    if iter_step % compact_freq == 0:
        proc("compact")
    return log


def train_step(state, iter_step, bounds, anchors, weights, alphas, cameras, compact_freq):
    """One iteration of UpdateOctNodes on the CPU copy; -> maintain's log"""
    cast_votes(state, bounds, anchors, weights, alphas)
    return maintain(state, iter_step, cameras, compact_freq)


def check_links(nodes):
    """parent / child links of a ProcOctree result: a root, parents before children, every child points back, leaves carry
    a warp and have no child, inner nodes carry none and (below the root) at least two children"""
    t = tree_view(nodes)
    m = t["parent"].shape[0]
    assert m > 0 and t["parent"][0] == -1
    assert (t["parent"][1:] >= 0).all() and (t["parent"][1:] < np.arange(1, m)).all()
    has = t["childs"] >= 0
    assert (t["childs"][has] < m).all()
    owner = np.repeat(np.arange(m), has.sum(1))
    assert (t["parent"][t["childs"][has]] == owner).all()
    assert np.array_equal(np.sort(t["childs"][has]), np.arange(1, m))            # every node but the root is somebody's child, once
    n_ch = has.sum(1)
    assert (n_ch[t["leaf"]] == 0).all() and (t["trans"][t["leaf"]] >= 0).all()    # no dead leaf survives
    inner = ~t["leaf"]
    inner[0] = False
    assert (t["trans"][inner] < 0).all() and (n_ch[inner] >= 2).all()           # no single-child chain below the root


def check_maintain_log(log, state, milestones_before, iter_step, compact_freq):
    """Structural invariants of one ``maintain`` call (the tree it leaves is ``state``'s)"""
    due = []
    ms = list(milestones_before)
    while ms and ms[-1] <= iter_step:
        due.append(ms.pop())
    assert state.milestones == ms                                                # consumed from the back, in order
    kinds = [k for k, *_ in log]
    assert kinds == ["subdivide", "compact"] * len(due) + (["compact"] if iter_step % compact_freq == 0 else [])
    assert [b for k, b, *_ in log if k == "subdivide"] == [m <= 0 for m in due]
    for kind, brute, before, visit, after in log:
        b, a = tree_view(before), tree_view(after)
        live = b["leaf"] & (b["trans"] >= 0)
        check_links(after)
        if kind == "compact":
            assert int(a["leaf"].sum()) == int(live.sum())
            continue
        # subdivision: each live leaf visited more than 4 times (every one, brute force) became an inner node with 8 leaf
        # children: the octants, half the side length, the parent's warp
        split = live if brute else live & (visit > 4)
        assert int(a["leaf"].sum()) == int(live.sum()) + 7 * int(split.sum())
        full = np.nonzero((a["childs"] >= 0).all(1))[0]
        octants = np.array([[(st >> 2) & 1, (st >> 1) & 1, st & 1] for st in range(8)], np.float32) * 2 - 1
        n_split = 0
        for u in full:
            ch = a["childs"][u]
            if a["leaf"][ch].all() and (a["side"][ch] == a["side"][u] * .5).all() and len(set(a["trans"][ch].tolist())) == 1 \
                    and np.array_equal(a["center"][ch], a["center"][u] + (a["side"][u] * .5) * (octants * .5)):
                n_split += 1
        assert n_split >= int(split.sum())
    if log:
        assert not state.visit_cnt.any() and state.visit_cnt.shape[0] == state.n_nodes
        check_links(state.nodes)
    assert state.weight_stats.shape[0] == state.alpha_stats.shape[0] == state.n_nodes
