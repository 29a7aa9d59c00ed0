"""Octree maintenance inside training: PersSampler.maintain (the tail of PersSampler::UpdateOctNodes, PersSampler.cu:604-614)
between consecutive TRAIN steps, FusedAdam stepping in between, with and without the pipelined march.

a. Exact tree evolution.  The CPU driver (tests/oracle_train_loop.py) casts each step's votes from the DEVICE's own early-stop
   weights and alphas — first shown to be the oracle's numbers at the usual tolerance — so the threshold decisions are the same
   on both sides, and then tree bytes, statistics, visit counts, node count, remaining milestones and the next step's samples
   are equal bit for bit at every step.
b. Numerical step.  On the maintained tree every step's outputs and gradients against oracle_pipeline.render_train, at the bars
   of tests/test_gpu_render.py::test_render_train_step_matches_oracle.
c. The pipelined march (Renderer.set_next_rays / prefetch_next) gives the unpipelined run bit for bit, and the Render after a
   step whose maintenance replaced the tree marches again instead of consuming the march of the old tree.
d. The prefetch guard by itself: a tree written into the same storage, a tree from ProcOctree, a tree from LoadStates.
e. Two ranks with all-reduced votes keep byte-identical trees through the milestones, rank 1's shard empty on those steps.
"""
import os
import time
import traceback
from datetime import timedelta

import numpy as np
import pytest
import torch

import oracle_train_loop as TL
from conftest import make_rays
from test_gpu_data_parallel import _free_port, make_shards, train_loss
from test_gpu_parity import N, T
from test_gpu_render import assert_close_but, build, check_step_against_oracle

pytestmark = pytest.mark.gpu

N_CAMS = 6                       # MarkInvisibleNodes with the first six cameras: part of the scene is seen by none of them
RAYS = (150, 97)                 # alternating batch sizes (the second one leaves the last march warp half filled)
FLIPPED = 1e-3                   # share of a step's per-sample weights allowed past the bar (test_gpu_render.assert_close_but)
CASES = [(s, 1.0) for s in TL.SCHEDULES] + [("milestone", 0.3)]
CASE_IDS = [f"{s}-{g}" for s, g in CASES]
EXACT = ("nodes", "w_stats", "a_stats", "visits", "milestones", "bounds", "pts", "anchors", "first_oct_dis", "colors", "disparity",
         "depth", "weights", "edge_feats", "idx_start_end")


def start_near_threshold(sampler):
    """statistics in [0, 3): a leaf that is visited and found empty is pruned within three steps"""
    rng = np.random.default_rng(2)
    n = sampler.n_nodes
    sw, sa = rng.integers(0, 3, n).astype(np.int32), rng.integers(0, 3, n).astype(np.int32)
    sampler.tree_weight_stats_.copy_(T(sw))
    sampler.tree_alpha_stats_.copy_(T(sa))
    return sw, sa


def early_stop_weights(renderer):
    """the early-stop pass's weights and alphas of the last Render, out of the renderer's slot buffers, in sample order.  Only
    valid once Render has returned and the device is synchronised."""
    slots = renderer.sample_result_._slots
    sb = N(slots.slot_bounds).astype(np.int64)
    idx = np.concatenate([np.arange(b, e) for b, e in sb] + [np.zeros(0, np.int64)])
    return N(renderer._bufs_["w0"])[idx], N(renderer._bufs_["a0"])[idx]


def traced_render(renderer, ro, rd, cam):
    """-> (RenderResult, whether this Render ran the ray march itself rather than taking a prefetched one)"""
    from f2nerf_b200 import _lib
    _lib.TRACE = []
    try:
        res = renderer.Render(ro, rd, None, cam)
    finally:
        trace, _lib.TRACE = _lib.TRACE, None
    names = [t[0] for t in trace]
    return res, "f2b_sampler_march" in names[:names.index("f2b_early_stop_rays")]


def replay_draws(sampler, rng0, n_rays, n_all):
    """Render's internal draws from the generator state ``rng0`` it started at, in its order: ray noise, background, the
    early-stop query's output draw, the TV-loss edge points"""
    from f2nerf_b200.rng import burn_mlp_output
    now = torch.cuda.get_rng_state()
    torch.cuda.set_rng_state(rng0)
    noise = sampler.make_noise(n_rays, "cuda").clone()
    bg = torch.rand((n_rays, 3), device="cuda")
    burn_mlp_output(n_all, torch.device("cuda"))
    e_idx = torch.randint(0, sampler.n_edges, (8192,), dtype=torch.int32, device="cuda")
    e_coord = torch.rand((8192, 2), device="cuda") * 2. - 1.
    torch.cuda.set_rng_state(now)
    return N(noise), N(bg), N(e_idx), N(e_coord)


def oracle_scene(scene, nodes):
    return dict(nodes=nodes, trans=scene["trans"], edges=scene["edges"], near=0.05, sample_l=1 / 64, scale_by_dis=True, max_hits=1024)


def train_run(scene, schedule, gs_progress, mode, with_oracle=False, grads_from=None):
    """N_ITERS TRAIN steps on the synthetic scene: Render, loss, backward, maintain, FusedAdam.  ``mode``: "off" (every Render
    marches), "early" (set_next_rays before each Render), "late" (prefetch_next after each Render).  ``with_oracle``: follow
    every step with the CPU driver and the CPU pipeline (a. and b. of the module text).  ``grads_from``: per step the four
    gradients of another run, handed to the optimizer instead of this run's own once those are shown to agree to summation
    order — the table gradient is accumulated atomically, and Adam's first steps turn a last-bit difference of a near-zero
    entry into a full step, so only then are two runs' parameters, and with them everything else, comparable bit for bit."""
    import oracle_pipeline as OP
    from f2nerf_b200 import TRAIN, FusedAdam, check_backward_nan, ops
    ms, compact_freq = TL.SCHEDULES[schedule]
    gdp, sampler, field, shader, renderer = build(scene)
    gdp.mode_, gdp.gradient_scaling_progress_, gdp.learning_rate_ = TRAIN, gs_progress, 1e-2
    sw, sa = start_near_threshold(sampler)
    sampler.sub_div_milestones_ = list(ms)
    opt = FusedAdam(renderer.OptimParamGroups(), table_field=field)
    params = (field.mlp_.params_, shader.mlp_.params_, renderer.app_emb_, field.feat_pool_)
    cams = TL.scene_cameras(scene["scene"], N_CAMS)
    state = TL.OctreeState(scene["nodes"], sw, sa, ms) if with_oracle else None
    host = [make_rays(scene, RAYS[i % 2], seed=40 + i) for i in range(TL.N_ITERS)]
    dev = [(T(o), T(d), T(cam)) for o, d, dn, cam in host]
    scales = ops.hash_level_scales().numpy()
    torch.manual_seed(2024)
    recs, first_params = [], [p.detach().clone() for p in params]
    for i, (ro, rd, cam) in enumerate(dev):
        it = gdp.iter_step_ = i + 1
        n_rays = ro.shape[0]
        opt.zero_grad()
        nxt = dev[(i + 1) % len(dev)]
        if mode == "early":
            renderer.set_next_rays(nxt[0], nxt[1])
        rng0 = torch.cuda.get_rng_state()
        res, marched = traced_render(renderer, ro, rd, cam)
        if mode == "late":
            renderer.prefetch_next(nxt[0], nxt[1])
        if mode != "off":
            assert sampler._prefetched is not None
        loss = train_loss(res, n_rays)
        loss.backward()
        assert not check_backward_nan(renderer)
        torch.cuda.synchronize()
        sr = renderer.sample_result_
        rec = dict(marched=marched, bounds=N(sr.pts_idx_bounds), pts=N(sr.pts), anchors=N(sr.anchors), first_oct_dis=N(sr.first_oct_dis),
                   colors=N(res.colors), disparity=N(res.disparity), depth=N(res.depth), weights=N(res.weights),
                   edge_feats=N(res.edge_feats), idx_start_end=N(res.idx_start_end), grads=[N(p.grad) for p in params])
        assert int(rec["anchors"][:, 1].max()) < sampler.n_nodes
        if state is not None:
            w0, a0 = early_stop_weights(renderer)
            noise, bg, e_idx, e_coord = replay_draws(sampler, rng0, n_rays, sr.pts.shape[0])
            gt = torch.rand((n_rays, 3), device="cuda", generator=torch.Generator("cuda").manual_seed(9))
            fld = dict(table16=N(field.table_f16()), prim=N(field.prim_pool_), bias=N(field.bias_pool_), V=field.n_volumes_,
                       local_size=field.local_size_, mlp_params=N(field.mlp_.params_))
            ref = OP.render_train(oracle_scene(scene, state.nodes), host[i][0], N(rd / torch.linalg.norm(rd, 2, -1, True)), noise, bg,
                                  fld, N(shader.mlp_.params_), N(renderer.app_emb_), host[i][3], (e_idx, e_coord), N(gt),
                                  scales=scales, gs_progress=gs_progress)
            np.testing.assert_array_equal(rec["first_oct_dis"].view(np.uint32), ref["sample"]["first_oct_dis"].view(np.uint32))
            assert i > 0 or ref["n_kept"] < sr.pts.shape[0], "early stop must be exercised"
            check_step_against_oracle(res, sr, float(loss.detach()), ref, *(p.grad for p in params), flipped_share=FLIPPED)
            # the votes: the device's early weights are the oracle's numbers; cast from the device's, the decisions are the device's
            assert_close_but(w0, ref["early_weights"], 2e-3, 1e-4, f"early weights, step {it}", FLIPPED)
            assert_close_but(a0, ref["early_alphas"], 2e-3, 1e-4, f"early alphas, step {it}", FLIPPED)
            before = list(state.milestones)
            log = TL.train_step(state, it, ref["sample"]["bounds"], ref["sample"]["anchors"], w0, a0, cams, compact_freq)
            TL.check_maintain_log(log, state, before, it, compact_freq)
            rec["log"] = [(kind, TL.tree_view(b), visit, TL.tree_view(a)) for kind, _, b, visit, a in log]
        tree, voted = sampler.tree_nodes_gpu_, N(sampler.tree_nodes_gpu_)
        sampler.maintain(cams, compact_freq)
        rec.update(replaced=sampler.tree_nodes_gpu_ is not tree, nodes=N(sampler.tree_nodes_gpu_),
                   w_stats=N(sampler.tree_weight_stats_), a_stats=N(sampler.tree_alpha_stats_), visits=N(sampler.tree_visit_cnt_),
                   milestones=np.array(sampler.sub_div_milestones_, np.int64))
        rec["changed"] = not np.array_equal(voted, rec["nodes"])                  # by the maintenance, not by the votes' pruning
        if state is not None:
            for k, want in (("nodes", state.nodes), ("w_stats", state.weight_stats), ("a_stats", state.alpha_stats),
                            ("visits", state.visit_cnt), ("milestones", np.array(state.milestones, np.int64))):
                np.testing.assert_array_equal(rec[k], want, err_msg=f"octree {k} after iteration {it} ({schedule})")
        if grads_from is not None:
            for p, mine, theirs in zip(params, rec["grads"], grads_from[i]):      # fp32 atomics in another order, cancelling sums
                np.testing.assert_allclose(mine, theirs, rtol=1e-5, atol=1e-5 * np.abs(theirs).max(), err_msg=f"gradient, step {it}")
                assert np.linalg.norm(mine.astype(np.float64) - theirs) <= 1e-5 * np.linalg.norm(theirs), f"gradient, step {it}"
                p.grad.copy_(T(theirs))
        opt.step()
        recs.append(rec)
    torch.cuda.synchronize()
    assert not any(torch.equal(a, p) for a, p in zip(first_params, params)), "the optimizer must move every parameter"
    return recs


_unpipelined = {}


def unpipelined_run(scene, schedule, gs_progress):
    """the "off" run of a case, followed by the oracle; kept for the pipelined runs of the same case (one case at a time)"""
    key = (schedule, gs_progress)
    if key not in _unpipelined:
        _unpipelined.clear()
        _unpipelined[key] = train_run(scene, schedule, gs_progress, "off", with_oracle=True)
    return _unpipelined[key]


@pytest.mark.parametrize("schedule,gs_progress", CASES, ids=CASE_IDS)
def test_maintained_tree_matches_oracle(scene, oracle, schedule, gs_progress):
    """a. and b. of the module text (asserted step by step inside the run), and that the schedule did maintain: dead leaves were
    dropped and the nodes renumbered, the node count moved, every milestone subdivision split leaves"""
    recs = unpipelined_run(scene, schedule, gs_progress)
    ms, compact_freq = TL.SCHEDULES[schedule]
    assert all(r["marched"] for r in recs)
    assert len({r["nodes"].size for r in recs} | {scene["nodes"].size}) > 1
    events = [e for r in recs for e in r["log"]]
    assert len(events) == 2 * len(ms) + TL.N_ITERS // compact_freq
    dropped = [int((b["leaf"] & (b["trans"] < 0)).sum()) for _, b, _, _ in events]
    assert max(dropped) > 0, "no ProcOctree call found a dead leaf to drop"
    split = [int(a["leaf"].sum()) - int((b["leaf"] & (b["trans"] >= 0)).sum()) for kind, b, _, a in events if kind == "subdivide"]
    if schedule == "two-due":                               # the second pass of the loop finds zeroed visit counts: no split
        assert split[0] > 0 and split[1] == 0
    else:
        assert all(s > 0 for s in split) and len(split) == len(ms)
    assert [r["replaced"] for r in recs] == [bool(r["log"]) for r in recs] and any(r["changed"] for r in recs)


@pytest.mark.parametrize("mode", ["early", "late"])
@pytest.mark.parametrize("schedule,gs_progress", CASES, ids=CASE_IDS)
def test_pipelined_march_survives_maintenance(scene, oracle, schedule, gs_progress, mode):
    """c. of the module text.  The Render that follows a step whose maintenance replaced the tree runs f2b_sampler_march itself
    (the launch trace shows it ahead of the early-stop pass) and so draws its noise itself — the same numbers as the unpipelined
    run, also behind the GradientScaling draws of gs_progress < 1; every other Render but the first consumes its prefetch."""
    base = unpipelined_run(scene, schedule, gs_progress)
    recs = train_run(scene, schedule, gs_progress, mode, grads_from=[r["grads"] for r in base])
    for i, (a, b) in enumerate(zip(base, recs)):
        for k in EXACT:
            np.testing.assert_array_equal(a[k].view(np.uint32) if a[k].dtype == np.float32 else a[k],
                                          b[k].view(np.uint32) if b[k].dtype == np.float32 else b[k],
                                          err_msg=f"{k}, iteration {i + 1}, {mode} vs unpipelined")
        assert a["replaced"] == b["replaced"]
        assert b["marched"] == (i == 0 or base[i - 1]["replaced"]), f"iteration {i + 1}: marched {b['marched']}"
    assert sum(r["marched"] for r in recs[1:]) >= 1 and not all(r["marched"] for r in recs[1:])
    after_change = [i for i in range(1, len(recs)) if recs[i - 1]["changed"]]
    assert after_change and all(recs[i]["marched"] for i in after_change)


# ------------------------------------------------------------------------------------------- d. the prefetch guard ----
def _damaged(nodes, frac=0.3):
    """the tree with a share of its live leaves dead: same size, different samples"""
    t = nodes.copy().view(np.int32).reshape(-1, 16)
    live = np.nonzero((nodes.reshape(-1, 64)[:, 52] != 0) & (t[:, 14] >= 0))[0]
    t[np.random.default_rng(4).choice(live, int(len(live) * frac), replace=False), 14] = -1
    return t.reshape(-1).view(np.uint8)


@pytest.mark.parametrize("how", ["untouched", "same-storage", "proc-octree", "load-states"])
def test_prefetched_march_is_tied_to_its_tree(scene, oracle, how):
    """A prefetched march is consumed only by a Render on the very tree it marched.  ``same-storage``: another tree written
    into the tree tensor in place (same address, same size); ``proc-octree`` / ``load-states``: the tensor replaced.  The next
    Render then marches itself and its samples are the oracle's on the current tree.  ``untouched``: the votes' own in-place
    pruning, which precedes the prefetched march on its stream, does not cost the prefetch."""
    from f2nerf_b200 import TRAIN
    gdp, sampler, field, shader, renderer = build(scene)
    gdp.mode_ = TRAIN
    (o0, d0, _, c0), (o1, d1, dn1, c1) = (make_rays(scene, n, seed=70 + i) for i, n in enumerate(RAYS))
    b0, b1 = (T(o0), T(d0), T(c0)), (T(o1), T(d1), T(c1))
    torch.manual_seed(7)
    res = renderer.Render(b0[0], b0[1], None, b0[2])
    renderer.prefetch_next(b1[0], b1[1])
    train_loss(res, RAYS[0]).backward()
    torch.cuda.synchronize()
    assert sampler._prefetched is not None
    if how == "same-storage":
        ptr = sampler.tree_nodes_gpu_.data_ptr()
        sampler.tree_nodes_gpu_.copy_(T(_damaged(scene["nodes"])))
        assert sampler.tree_nodes_gpu_.data_ptr() == ptr
    elif how == "proc-octree":
        assert sampler.ProcOctree(True, True, False) != scene["nodes"].size // 64
    elif how == "load-states":
        sampler.LoadStates([T(_damaged(scene["nodes"])), sampler.pers_trans_gpu_, torch.zeros_like(sampler.tree_visit_cnt_),
                            torch.zeros(0, dtype=torch.int32)], 0)
    torch.cuda.synchronize()
    tree = N(sampler.tree_nodes_gpu_)
    rng0 = torch.cuda.get_rng_state()
    res, marched = traced_render(renderer, b1[0], b1[1], b1[2])
    assert marched == (how != "untouched")
    sr = renderer.sample_result_
    noise = replay_draws(sampler, rng0, RAYS[1], sr.pts.shape[0])[0]
    ref = oracle.sampler(tree, scene["trans"], o1, N(b1[1] / torch.linalg.norm(b1[1], 2, -1, True)), noise, 0.05, 1e8, 1 / 64, True, 1024)
    np.testing.assert_array_equal(N(sr.pts_idx_bounds), ref["bounds"])
    np.testing.assert_array_equal(N(sr.pts).view(np.uint32), ref["pts"].view(np.uint32))
    np.testing.assert_array_equal(N(sr.anchors), ref["anchors"])
    np.testing.assert_array_equal(N(res.first_oct_dis).view(np.uint32), ref["first_oct_dis"].view(np.uint32))
    assert ref["pts"].shape[0] > 0


# ------------------------------------------------------------------------------------------------- e. two ranks ----
WORLD = 2
JOIN_S = 240
DP_MILESTONES = [6, 3]


def dp_shards(scene):
    """[iteration - 1][rank] -> (rays_o, rays_d, camera index); rank 1 has no ray on the two milestone iterations"""
    full, empty = make_shards(scene, "rays"), make_shards(scene, "empty")
    return [(empty if i + 1 in DP_MILESTONES else full)[i % len(full)] for i in range(TL.N_ITERS)]


def _rank_main(rank, port, scene, shards, cams, out_dir):
    """one rank: TL.N_ITERS training steps with maintenance on its own shards, votes all-reduced; the octree after each
    iteration to out_dir/rank{r}_it{i}.npz, a traceback to out_dir/rank{r}.err on failure"""
    try:
        import torch.distributed as dist
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        torch.cuda.set_device(rank % torch.cuda.device_count())
        dist.init_process_group("gloo", rank=rank, world_size=WORLD, timeout=timedelta(seconds=60))
        from f2nerf_b200 import TRAIN, FusedAdam, check_backward_nan
        from f2nerf_b200.dist import allreduce_grads, install_vote_sync, sync_emas
        gdp, sampler, field, shader, renderer = build(scene)
        gdp.mode_, gdp.learning_rate_ = TRAIN, 1e-2
        start_near_threshold(sampler)
        sampler.sub_div_milestones_ = list(DP_MILESTONES)
        opt = FusedAdam(renderer.OptimParamGroups(), table_field=field)
        install_vote_sync(sampler)
        for i, shard in enumerate(shards):
            gdp.iter_step_ = i + 1
            o, d, cam = shard[rank]
            opt.zero_grad()
            torch.manual_seed(1000 * i + 17 * rank + 3)
            res = renderer.Render(T(o), T(d), None, T(cam))
            if res.colors.requires_grad:                        # an empty shard has no graph
                train_loss(res, o.shape[0]).backward()
            assert not check_backward_nan(renderer)
            sampler.maintain(cams, 1000)
            allreduce_grads(renderer)
            opt.step()
            sync_emas(gdp)
            torch.cuda.synchronize()
            np.savez(os.path.join(out_dir, f"rank{rank}_it{i + 1}.npz"), nodes=N(sampler.tree_nodes_gpu_),
                     w_stats=N(sampler.tree_weight_stats_), a_stats=N(sampler.tree_alpha_stats_), visits=N(sampler.tree_visit_cnt_),
                     milestones=np.array(sampler.sub_div_milestones_, np.int64), table=N(field.feat_pool_), n_rays=o.shape[0])
        dist.destroy_process_group()
    except BaseException:
        with open(os.path.join(out_dir, f"rank{rank}.err"), "w") as f:
            f.write(traceback.format_exc())
        os._exit(1)                                             # no teardown of a process group that may be stuck


def test_two_ranks_keep_one_tree_through_milestones(scene, tmp_path):
    """e. of the module text: after every iteration both ranks hold the same tree bytes, statistics, visit counts and milestones;
    both subdivisions happened, on iterations where rank 1 cast only neutral votes (Renderer._neutral_votes)"""
    import torch.multiprocessing as mp
    shards = dp_shards(scene)
    assert all(shards[it - 1][1][0].shape[0] == 0 for it in DP_MILESTONES)
    ctx = mp.get_context("spawn")
    port = _free_port()
    blobs = dict(nodes=scene["nodes"], trans=scene["trans"], edges=scene["edges"])
    cams = TL.scene_cameras(scene["scene"], N_CAMS)
    procs = [ctx.Process(target=_rank_main, args=(r, port, blobs, shards, cams, str(tmp_path)), daemon=True) for r in range(WORLD)]
    try:
        for p in procs:
            p.start()
        deadline = time.monotonic() + JOIN_S
        for p in procs:
            p.join(timeout=max(0.1, deadline - time.monotonic()))
        hung = [r for r, p in enumerate(procs) if p.is_alive()]
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)
            if p.is_alive():
                p.kill()
                p.join(timeout=10)
    assert not hung, f"rank processes {hung} still running after {JOIN_S} s"
    errs = {r: open(tmp_path / f"rank{r}.err").read() for r in range(WORLD) if (tmp_path / f"rank{r}.err").exists()}
    assert not errs and [p.exitcode for p in procs] == [0] * WORLD, errs
    counts = [scene["nodes"].size // 64]
    for it in range(1, TL.N_ITERS + 1):
        r0, r1 = (dict(np.load(tmp_path / f"rank{r}_it{it}.npz")) for r in range(WORLD))
        assert r0["n_rays"] > 0 and (r1["n_rays"] == 0) == (it in DP_MILESTONES)
        for k in r0:
            if k != "n_rays":
                np.testing.assert_array_equal(r0[k], r1[k], err_msg=f"rank 0 vs rank 1: {k} after iteration {it}")
        assert r0["w_stats"].shape[0] == r0["a_stats"].shape[0] == r0["visits"].shape[0] == r0["nodes"].size // 64
        assert r0["milestones"].tolist() == [m for m in DP_MILESTONES if m > it]
        counts.append(r0["nodes"].size // 64)
    for it in DP_MILESTONES:
        assert counts[it] != counts[it - 1], counts
    assert counts[-1] > counts[0], counts                    # the subdivisions split leaves
