"""Data-parallel training on the device (f2nerf_b200/dist.py).

a. The slab backward: with a slab hook installed (dist.install_grad_overlap), Renderer's backward runs the unfused MLP backward
   chain into HBM rows and scatters the table gradient level group by level group (f2b_hash_bwd_levels), calling the hook
   after each group.  Checked against the default fused backward of the same step (same forward, octree and RNG state bit for
   bit; gradients at the fused-vs-unfused bars of tests/test_gpu_shade_fused.py) and against the CPU oracle's double-precision
   scatter of the rows the renderer actually handed to f2b_hash_bwd_levels.
b. Two ranks exchanging gradients: two processes on gloo with CUDA tensors (host-side collectives that honour the process-group
   timeout, so a mismatched collective sequence fails the test instead of hanging), each running whole training steps
   (Render, loss, backward, allreduce_grads, FusedAdam, sync_emas) on its own shard, rank 1's shard possibly empty or all-miss.
"""
import os
import socket
import time
import traceback
from datetime import timedelta

import numpy as np
import pytest
import torch

from conftest import make_rays
from test_gpu_bwd_reference import TABLE_TOL
from test_gpu_parity import N, T, assert_close
from test_gpu_render import build

pytestmark = pytest.mark.gpu

BARS = dict(rtol=1e-5, atol_frac=1e-6)          # fused vs unfused backward chains (tests/test_gpu_shade_fused.py)
SEED = 321
N_EDGE = 2 * 8192                               # TV-loss edge points of a TRAIN step (renderer.N_EDGE_PTS pairs)


def train_loss(res, n_rays, gt_seed=9):
    """the loss of tests/test_gpu_render.py::test_render_train_step_matches_oracle"""
    from f2nerf_b200 import CustomOps
    dev = res.colors.device
    gt = torch.rand((n_rays, 3), device=dev, generator=torch.Generator(dev).manual_seed(gt_seed))
    color_loss = torch.sqrt((res.colors - gt) ** 2 + 1e-4).mean()
    var_loss = torch.sqrt(CustomOps.WeightVar(res.weights, res.idx_start_end) + 1e-2).mean()
    tv = ((res.edge_feats[:, 0] - res.edge_feats[:, 1]) ** 2).mean()
    return color_loss + 0.01 * var_loss + 0.01 * (res.disparity ** 2).mean() + 0.1 * tv


def params_of(renderer):
    return (renderer.scene_field_.feat_pool_, renderer.scene_field_.mlp_.params_, renderer.shader_.mlp_.params_, renderer.app_emb_)


# ------------------------------------------------------------------------------------------------------ a. slab backward ----
def one_step(scene, rays, gs_progress, emb, log2, slab=None):
    """one seeded TRAIN step from a freshly built renderer; ``slab`` = grad_premul_ of a recording slab hook (None: the default
    fused backward)"""
    from f2nerf_b200 import TRAIN, check_backward_nan
    gdp, sampler, field, shader, renderer = build(scene, log2=log2, use_app_emb=emb)
    gdp.mode_, gdp.gradient_scaling_progress_ = TRAIN, gs_progress
    hooks, finish = [], []
    if slab is not None:
        renderer.grad_slab_hook_ = lambda d_table, lo, local_size: hooks.append((id(d_table), lo, local_size))
        renderer.grad_slab_finish_ = lambda: finish.append(len(hooks))
        renderer.grad_premul_ = slab
    o, d, cam = rays
    torch.manual_seed(SEED)
    res = renderer.Render(T(o), T(d), None, T(cam))
    train_loss(res, o.shape[0]).backward()
    assert not check_backward_nan(renderer)
    torch.cuda.synchronize()
    sr = renderer.sample_result_
    out = dict(colors=res.colors, disparity=res.disparity, depth=res.depth, weights=res.weights, edge_feats=res.edge_feats,
               idx_start_end=res.idx_start_end, first_oct_dis=res.first_oct_dis, pts=sr.pts, anchors=sr.anchors,
               pts_idx_bounds=sr.pts_idx_bounds, nodes=sampler.tree_nodes_gpu_, w_stats=sampler.tree_weight_stats_,
               a_stats=sampler.tree_alpha_stats_, visits=sampler.tree_visit_cnt_, rng=torch.cuda.get_rng_state())
    out = {k: N(v) if isinstance(v, torch.Tensor) and v.is_cuda else v.numpy() for k, v in out.items()}
    grads = {k: None if p.grad is None else N(p.grad) for k, p in zip(("table", "field", "shader", "app"), params_of(renderer))}
    return dict(out=out, grads=grads, hooks=hooks, finish=finish, field=field, renderer=renderer)


@pytest.fixture
def spy(monkeypatch):
    """records every f2b_hash_bwd_levels call of the renderer: its scalars, and clones (on the calling stream) of the points,
    anchors and fp16 dL/dfeat rows of the first level group's calls"""
    from f2nerf_b200 import renderer as R
    calls = []
    real = R.call

    def call(name, *args):
        if name == "f2b_hash_bwd_levels":
            prim, bias, V, S, pts, anc, stride, n, rows, half, mul, table, lo, nl, _ = args
            c = dict(stride=stride, n=n, half=half, mul=mul, table=id(table), lo=lo, nl=nl)
            if not calls or calls[0]["lo"] == lo:
                c.update(pts=pts[:n].clone(), anc=anc[:n].clone(), rows=rows[:n].clone())
            calls.append(c)
        return real(name, *args)

    monkeypatch.setattr(R, "call", call)
    return calls


def check_slab_table(oracle, field, got, jobs, tag):
    """table gradient of the slab scatter vs the oracle's float64 scatter of both jobs' captured rows, per entry at the bar of
    test_gpu_bwd_reference.check_table; untouched entries and the dead tail above 17 S / 2 rows exactly 0"""
    from f2nerf_b200 import ops
    scales = ops.hash_level_scales().numpy()
    pool, S = field.feat_pool_.shape[0], int(field.local_size_)
    prim, bias = N(field.prim_pool_), N(field.bias_pool_)
    exact = np.zeros((pool, 2))
    abssum = np.zeros((pool, 2))
    for j in jobs:
        args = (prim, bias, int(field.n_volumes_), S, scales, N(j["pts"]), N(j["anc"]), j["stride"])
        g = N(j["rows"]).astype(np.float32)
        exact += oracle.hash_bwd(*args, g, j["mul"], pool)
        abssum += oracle.hash_bwd(*args, np.abs(g), j["mul"], pool)
    got = np.asarray(got, np.float64)
    err = np.abs(got - exact)
    bad = ~(err <= TABLE_TOL * abssum)
    assert (abssum > 0).any()
    assert not bad.any(), (f"slab table {tag}: {int(bad.sum())} entries off, worst at {int(np.argmax(np.where(bad, err, 0)))}: "
                           f"err {err[bad].max():.3e}; untouched entries nonzero: {int((bad & (abssum == 0)).sum())}")
    assert not got[(17 * S) // 2:].any(), f"slab table {tag}: dead tail written"


@pytest.mark.parametrize("emb", [True, False], ids=["emb", "noemb"])
@pytest.mark.parametrize("gs_progress", [1.0, 0.3])
@pytest.mark.parametrize("n_rays", [64, 129, 4096])
def test_slab_backward_matches_fused_and_oracle(scene, oracle, spy, n_rays, gs_progress, emb):
    """129: every 7th ray misses the octree (no sample); 4096 on a 2^19 table: the kept samples fill many 128-row tiles and end
    in a partial one"""
    log2 = 19 if n_rays == 4096 else 15
    o, d, _, cam = make_rays(scene, n_rays, seed=77 + n_rays)
    if n_rays == 129:
        o[::7] = 600.
        d[::7] = 1.
    rays = (o, d, cam)
    tag = f"n_rays={n_rays} gs={gs_progress} emb={emb}"
    fused = one_step(scene, rays, gs_progress, emb, log2)
    assert not spy and not fused["hooks"]
    slab = one_step(scene, rays, gs_progress, emb, log2, slab=1.0)
    # the forward, the octree votes and the RNG stream do not depend on which backward runs
    for k, a in fused["out"].items():
        np.testing.assert_array_equal(slab["out"][k], a, err_msg=f"{k} {tag}")
    field, renderer = slab["field"], slab["renderer"]
    S, n_kept = int(field.local_size_), renderer.n_kept_pts_
    assert n_kept > 0
    if n_rays == 4096:
        assert n_kept > 16 * 128 and n_kept % 128, n_kept
    # the hook: four level groups top-down, one gradient buffer, the field's local size; finish once, after the last group
    assert [lo for _, lo, _ in slab["hooks"]] == [12, 8, 4, 0], tag
    assert len({t for t, _, _ in slab["hooks"]}) == 1 and all(s == S for _, _, s in slab["hooks"])
    assert slab["finish"] == [4]
    # the scatter calls: per group the ray samples (stride-3 anchors) then the edge points (stride 1), fp16 rows
    mul = 1.0 / field.mlp_.loss_scale_
    assert [(c["lo"], c["nl"], c["stride"], c["n"]) for c in spy] == \
        [(lo, 4, st, n) for lo in (12, 8, 4, 0) for st, n in ((3, n_kept), (1, N_EDGE))], tag
    assert all(c["half"] == 1 and c["mul"] == mul and c["table"] == slab["hooks"][0][0] for c in spy)
    check_slab_table(oracle, field, slab["grads"]["table"], spy[:2], tag)
    # against the fused backward
    for k in ("field", "shader", "app", "table"):
        if k == "app" and not emb:
            assert slab["grads"][k] is None and fused["grads"][k] is None
            continue
        assert np.abs(fused["grads"][k]).max() > 0, k
        assert_close(slab["grads"][k], fused["grads"][k], **BARS, name=f"grad {k} slab vs fused {tag}")
    # the 1/world pre-scale reaches the table gradient only
    spy.clear()
    half = one_step(scene, rays, gs_progress, emb, log2, slab=0.5)
    assert len(spy) == 8 and all(c["mul"] == mul * 0.5 for c in spy)
    assert_close(half["grads"]["table"], 0.5 * slab["grads"]["table"], **BARS, name=f"grad table premul 0.5 {tag}")
    for k in ("field", "shader", "app"):
        if slab["grads"][k] is not None:
            assert_close(half["grads"][k], slab["grads"][k], **BARS, name=f"grad {k} premul 0.5 {tag}")


# ---------------------------------------------------------------------------------------------------- b. two ranks ----
WORLD = 2
STEPS = 2
JOIN_S = 240                     # > process start-up + the 60 s process-group timeout a mismatched collective runs into


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def shard_seed(step, rank):
    return 1000 * step + 17 * rank + 3


SCENARIOS = [(False, "rays"), (True, "rays"), (False, "empty"), (True, "empty"), (True, "missed")]   # (overlap, rank 1's shard)


def tag_of(overlap, shard1):
    return f"{'overlap' if overlap else 'plain'}-{shard1}"


def make_shards(scene, shard1):
    """[step][rank] -> (rays_o, rays_d, camera index); rank 1's shards hold rays, no ray at all, or only rays that miss"""
    shards = []
    for step in range(STEPS):
        o0, d0, _, c0 = make_rays(scene, 96, seed=500 + step)
        o1, d1, _, c1 = make_rays(scene, 80, seed=600 + step)
        if shard1 == "empty":
            o1, d1, c1 = o1[:0], d1[:0], c1[:0]
        elif shard1 == "missed":
            o1[:] = 600.
            d1[:] = 1.
        shards.append([(o0, d0, c0), (o1, d1, c1)])
    return shards


def _rank_main(rank, port, scene, shards, out_dir):
    """one rank: per scenario, in order, build, install the exchange hooks and run STEPS training steps on its own shards; state
    after each step to out_dir/{tag}_rank{r}_step{s}.npz; the scenario and a traceback to out_dir/rank{r}.err on failure"""
    tag = None
    try:
        import torch.distributed as dist
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        torch.cuda.set_device(rank % torch.cuda.device_count())
        dist.init_process_group("gloo", rank=rank, world_size=WORLD, timeout=timedelta(seconds=60))
        from f2nerf_b200 import TRAIN, FusedAdam, check_backward_nan
        from f2nerf_b200.dist import allreduce_grads, install_grad_overlap, install_vote_sync, sync_emas
        for overlap, shard1 in SCENARIOS:
            tag = tag_of(overlap, shard1)
            gdp, sampler, field, shader, renderer = build(scene)
            gdp.mode_ = TRAIN
            opt = FusedAdam(renderer.OptimParamGroups(), table_field=field)
            install_vote_sync(sampler)
            if overlap:
                install_grad_overlap(renderer)
            params = params_of(renderer)
            for step in range(STEPS):
                o, d, cam = shards[tag][step][rank]
                opt.zero_grad()
                torch.manual_seed(shard_seed(step, rank))
                res = renderer.Render(T(o), T(d), None, T(cam))
                if res.colors.requires_grad:                    # an empty or all-miss shard has no graph
                    train_loss(res, o.shape[0]).backward()
                assert not check_backward_nan(renderer)
                allreduce_grads(renderer)
                grads = [N(p.grad) for p in params]
                opt.step()
                sync_emas(gdp)
                torch.cuda.synchronize()
                st = [opt.state[id(p)] for p in params]
                np.savez(os.path.join(out_dir, f"{tag}_rank{rank}_step{step}.npz"),
                         **{f"param{i}": N(p) for i, p in enumerate(params)}, **{f"grad{i}": g for i, g in enumerate(grads)},
                         **{f"exp_avg{i}": N(s["exp_avg"]) for i, s in enumerate(st)},
                         **{f"exp_avg_sq{i}": N(s["exp_avg_sq"]) for i, s in enumerate(st)},
                         adam_steps=np.array([s["step"] for s in st]), shadow=N(field.table_f16()),
                         nodes=N(sampler.tree_nodes_gpu_), w_stats=N(sampler.tree_weight_stats_),
                         a_stats=N(sampler.tree_alpha_stats_), visits=N(sampler.tree_visit_cnt_),
                         emas=np.array([gdp.sampled_oct_per_ray_, gdp.sampled_pts_per_ray_, gdp.meaningful_sampled_pts_per_ray_]))
        dist.destroy_process_group()
    except BaseException:
        with open(os.path.join(out_dir, f"rank{rank}.err"), "w") as f:
            f.write(f"scenario {tag}\n{traceback.format_exc()}")
        os._exit(1)                                             # no teardown of a process group that may be stuck


@pytest.fixture(scope="module")
def two_ranks(scene, tmp_path_factory):
    """ONE pair of rank processes runs every scenario in turn (process start-up dominates a scenario's time).  A scenario whose
    collective sequences differ makes both ranks fail at the process-group timeout; the scenarios after it then have no result"""
    import torch.multiprocessing as mp
    out_dir = tmp_path_factory.mktemp("ranks")
    shards = {tag_of(*sc): make_shards(scene, sc[1]) for sc in SCENARIOS}
    ctx = mp.get_context("spawn")
    port = _free_port()
    blobs = dict(nodes=scene["nodes"], trans=scene["trans"], edges=scene["edges"])
    procs = [ctx.Process(target=_rank_main, args=(r, port, blobs, shards, str(out_dir)), daemon=True) for r in range(WORLD)]
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
    errs = {r: open(os.path.join(out_dir, f"rank{r}.err")).read() for r in range(WORLD)
            if os.path.exists(os.path.join(out_dir, f"rank{r}.err"))}
    return dict(shards=shards, out_dir=out_dir, hung=hung, exitcodes=[p.exitcode for p in procs], errs=errs)


def replay_shard(scene, rays, seed):
    """a shard's first step on a fresh renderer with no process group: its own gradients, votes and visit counts"""
    from f2nerf_b200 import TRAIN, check_backward_nan
    gdp, sampler, field, shader, renderer = build(scene)
    gdp.mode_ = TRAIN
    o, d, cam = rays
    torch.manual_seed(seed)
    res = renderer.Render(T(o), T(d), None, T(cam))
    if res.colors.requires_grad:
        train_loss(res, o.shape[0]).backward()
    assert not check_backward_nan(renderer)
    torch.cuda.synchronize()
    n = sampler.n_nodes
    votes = getattr(sampler, "last_votes_", None)
    if votes is None:                                           # no sample, no vote
        votes = (torch.full((n,), -1, dtype=torch.int32), torch.full((n,), -1, dtype=torch.int32), torch.zeros(n, dtype=torch.int32))
    grads = [N(p.grad) if p.grad is not None else np.zeros(tuple(p.shape), np.float32) for p in params_of(renderer)]
    return grads, [v.cpu().numpy() for v in votes], N(sampler.tree_visit_cnt_)


@pytest.mark.parametrize("overlap,shard1", SCENARIOS, ids=[tag_of(*sc) for sc in SCENARIOS])
def test_two_ranks_exchange(scene, two_ranks, overlap, shard1):
    """``shard1``: rank 1's shards hold rays, no rays at all, or only rays that miss the octree.  Both ranks must end every step
    with the same state bit for bit; after step 1 the exchanged gradient is the mean of the two shards' own gradients, and the
    octree is the single-process replay of the MAX of both shards' votes"""
    from f2nerf_b200 import TRAIN
    tag = tag_of(overlap, shard1)
    shards, out_dir = two_ranks["shards"][tag], two_ranks["out_dir"]
    assert not two_ranks["hung"], f"rank processes {two_ranks['hung']} still running after {JOIN_S} s"
    files = [[os.path.join(out_dir, f"{tag}_rank{r}_step{s}.npz") for r in range(WORLD)] for s in range(STEPS)]
    assert all(os.path.exists(f) for fs in files for f in fs), \
        f"scenario {tag} did not complete; exit codes {two_ranks['exitcodes']}: {two_ranks['errs']}"
    mine = [e for e in two_ranks["errs"].values() if e.startswith(f"scenario {tag}\n")]
    assert not mine, mine
    recs = [[dict(np.load(f)) for f in fs] for fs in files]
    for step, (r0, r1) in enumerate(recs):
        assert r0.keys() == r1.keys()
        for k in r0:
            np.testing.assert_array_equal(r0[k], r1[k], err_msg=f"rank 0 vs rank 1: {k} after step {step + 1}")
        assert (r0["adam_steps"] == step + 1).all()
    # step 1 against single-process replays of the two shards
    reps = [replay_shard(scene, shards[0][r], shard_seed(0, r)) for r in range(WORLD)]
    got = recs[0][0]
    for i, name in enumerate(("table", "field mlp", "shader mlp", "app emb")):
        mean = (reps[0][0][i].astype(np.float64) + reps[1][0][i]) / 2
        assert np.abs(mean).max() > 0, name
        assert_close(got[f"grad{i}"], mean, **BARS, name=f"averaged grad {name}")
    gdp, sampler, *_ = build(scene)
    gdp.mode_ = TRAIN
    w0 = N(sampler.tree_weight_stats_)
    vw, va, mk = (torch.from_numpy(np.maximum(reps[0][1][j], reps[1][1][j])).cuda() for j in range(3))
    sampler.tree_visit_cnt_ = torch.from_numpy(np.maximum(reps[0][2], reps[1][2])).cuda()
    sampler.apply_votes(vw, va, mk)
    for k, t in (("nodes", sampler.tree_nodes_gpu_), ("w_stats", sampler.tree_weight_stats_), ("a_stats", sampler.tree_alpha_stats_),
                 ("visits", sampler.tree_visit_cnt_)):
        np.testing.assert_array_equal(got[k], N(t), err_msg=f"octree {k} vs replay of the MAX of both shards' votes")
    assert (got["w_stats"] != w0).any()
