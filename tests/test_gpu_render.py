"""End to end: Renderer.Render (TRAIN mode: noise, early stop, octree votes, edge samples, appearance
embedding) + the trainer's loss + backward through the C ABI, against the oracle-composed pipeline."""
import numpy as np
import pytest
import torch

from conftest import make_rays
from test_gpu_parity import N, T, assert_close

pytestmark = pytest.mark.gpu


def build(scene, log2=15, use_app_emb=True, sample_l=1 / 64):
    from f2nerf_b200 import GlobalDataPool, Hash3DAnchored, PersSampler, Renderer, SHShader
    gdp = GlobalDataPool()
    sampler = PersSampler(gdp, scene["nodes"], scene["trans"], scene["edges"], near=0.05, sample_l=sample_l, scale_by_dis=True)
    torch.manual_seed(5)
    field = Hash3DAnchored(gdp, log2_table_size=log2)
    field.feat_pool_.data.uniform_(-1, 1)
    field.mlp_.params_.data.mul_(4.0)                 # wide density range -> early stop triggers
    shader = SHShader(gdp)
    renderer = Renderer(gdp, sampler, field, shader, n_images=24, use_app_emb=use_app_emb)
    return gdp, sampler, field, shader, renderer


@pytest.mark.parametrize("n_rays,gs_progress,seed,miss", [(192, 1.0, 77, 0), (64, 0.3, 77, 0), (129, 1.0, 11, 7)],
                         ids=["192-1.0", "64-0.3", "129-1.0-missed"])
def test_render_train_step_matches_oracle(scene, oracle, n_rays, gs_progress, seed, miss):
    """``miss``: every miss-th ray starts far outside the octree and points away (no sample at all); an odd ray count: the 16-lane
    march packs two rays per warp, so the last warp is half filled."""
    import oracle_pipeline as OP
    from f2nerf_b200 import TRAIN, check_backward_nan, ops, CustomOps
    gdp, sampler, field, shader, renderer = build(scene)
    gdp.mode_, gdp.gradient_scaling_progress_ = TRAIN, gs_progress
    o, d, dn, cam = make_rays(scene, n_rays, seed=seed)
    if miss:
        o[::miss] = 600.
        d[::miss] = 1.
    rays_o, rays_d, emb_idx = T(o), T(d), T(cam)
    seed = 321
    stats0 = N(sampler.tree_weight_stats_).copy()
    torch.manual_seed(seed)
    res = renderer.Render(rays_o, rays_d, None, emb_idx)
    state = torch.cuda.get_rng_state()
    torch.manual_seed(seed)                            # replay the internal draws, same order as Render ...
    noise = sampler.make_noise(n_rays, rays_o.device).clone()
    bg = torch.rand((n_rays, 3), device="cuda")
    from f2nerf_b200.rng import burn_mlp_output        # ... incl. the reference's torch::rand MLP output (TCNNWP.cpp:143)
    burn_mlp_output(renderer.sample_result_.pts.shape[0], rays_o.device)
    e_idx = torch.randint(0, sampler.n_edges, (8192,), dtype=torch.int32, device="cuda")
    e_coord = torch.rand((8192, 2), device="cuda") * 2. - 1.
    torch.cuda.set_rng_state(state)
    gt = torch.rand((n_rays, 3), device="cuda", generator=torch.Generator("cuda").manual_seed(9))
    color_loss = torch.sqrt((res.colors - gt) ** 2 + 1e-4).mean()
    var_loss = torch.sqrt(CustomOps.WeightVar(res.weights, res.idx_start_end) + 1e-2).mean()
    tv = ((res.edge_feats[:, 0] - res.edge_feats[:, 1]) ** 2).mean()
    loss = color_loss + 0.01 * var_loss + 0.01 * (res.disparity ** 2).mean() + 0.1 * tv
    loss.backward()
    assert not check_backward_nan(renderer)
    cnt = N(res.idx_start_end[:, 1] - res.idx_start_end[:, 0])
    assert cnt.sum() == res.weights.shape[0] and (cnt > 0).any()
    if miss:
        assert (cnt[::miss] == 0).all()
    assert torch.isfinite(field.feat_pool_.grad).all() and torch.isfinite(shader.mlp_.params_.grad).all()
    assert renderer.sample_result_.pts.shape[0] == int(renderer.sample_result_.pts_idx_bounds[-1, 1]) == renderer.n_sampled_pts_

    sc = dict(nodes=scene["nodes"], trans=scene["trans"], edges=scene["edges"], near=0.05, sample_l=1 / 64,
              scale_by_dis=True, max_hits=1024)
    fld = dict(table16=N(field.table_f16()), prim=N(field.prim_pool_), bias=N(field.bias_pool_), V=field.n_volumes_,
               local_size=field.local_size_, mlp_params=N(field.mlp_.params_))
    ref = OP.render_train(sc, o, N((rays_d / torch.linalg.norm(rays_d, 2, -1, True))), N(noise), N(bg), fld,
                          N(shader.mlp_.params_), N(renderer.app_emb_), cam, (N(e_idx), N(e_coord)), N(gt),
                          scales=ops.hash_level_scales().numpy(), gs_progress=gs_progress)
    # integer / index outputs: bit-exact
    sr = renderer.sample_result_
    np.testing.assert_array_equal(N(sr.pts_idx_bounds), ref["sample"]["bounds"])
    np.testing.assert_array_equal(N(sr.pts).view(np.uint32), ref["sample"]["pts"].view(np.uint32))
    np.testing.assert_array_equal(N(sr.anchors), ref["sample"]["anchors"])
    assert 0 < ref["n_kept"] < sr.pts.shape[0], "early stop must be exercised"
    if np.array_equal(N(res.idx_start_end), ref["bounds"]):         # identical keep mask (the usual case)
        assert_close(N(res.weights), ref["weights"], rtol=2e-3, atol_frac=1e-4, name="weights")
        assert_close(N(res.edge_feats), ref["edge_feats"], rtol=4e-3, atol_frac=2e-3, name="edge_feats")
    else:                                                           # a threshold-straddling sample: sizes differ by a few
        assert abs(int(res.idx_start_end[-1, 1]) - ref["n_kept"]) <= 3
    assert_close(N(res.colors), ref["colors"], rtol=2e-3, atol_frac=2e-3, name="colors")
    assert_close(N(res.disparity), ref["disparity"], rtol=2e-3, atol_frac=2e-3, name="disparity")
    assert_close(N(res.depth), ref["depth"], rtol=2e-3, atol_frac=2e-3, name="depth")
    assert abs(float(loss) - ref["loss"]) <= 2e-5 * abs(ref["loss"])
    # gradients.  Globally (relative L2 against the oracle's fp32-accumulate chain with the same fp16 rounding points) they
    # agree to ~1e-5 (cf. tests/test_gpu_headline.py); element-wise a single flipped fp16 rounding shows,
    # hence the looser per-element bars below
    rel = lambda a, b: float(np.linalg.norm(np.asarray(a, np.float64) - b) / (np.linalg.norm(b) + 1e-300))
    for name, mine in (("grad_field_mlp", field.mlp_.params_.grad), ("grad_shader_mlp", shader.mlp_.params_.grad),
                       ("grad_app_emb", renderer.app_emb_.grad), ("grad_feat_pool", field.feat_pool_.grad)):
        assert rel(N(mine), np.asarray(ref[name], np.float64)) <= 1e-3, (name, rel(N(mine), np.asarray(ref[name], np.float64)))
    assert_close(N(field.mlp_.params_.grad), ref["grad_field_mlp"], rtol=2e-2, atol_frac=1e-2, name="grad field mlp")
    assert_close(N(shader.mlp_.params_.grad), ref["grad_shader_mlp"], rtol=2e-2, atol_frac=1e-2, name="grad shader mlp")
    assert_close(N(renderer.app_emb_.grad), ref["grad_app_emb"], rtol=2e-2, atol_frac=1e-2, name="grad app_emb")
    g, gr = N(field.feat_pool_.grad), ref["grad_feat_pool"]
    assert_close(g, gr, rtol=3e-2, atol_frac=1e-2, name="grad feat_pool")
    assert np.abs(gr).max() > 0
    # octree statistics moved and match an oracle replay of the votes
    assert (N(sampler.tree_weight_stats_) != stats0).any()


def test_render_validate_mode_and_empty(scene):
    from f2nerf_b200 import VALIDATE
    gdp, sampler, field, shader, renderer = build(scene, use_app_emb=False)
    gdp.mode_ = VALIDATE
    o, d, dn, cam = make_rays(scene, 128, seed=5)
    with torch.no_grad():
        r1 = renderer.Render(T(o), T(d), None, None)
        r2 = renderer.Render(T(o), T(d), None, None)
    np.testing.assert_array_equal(N(r1.colors), N(r2.colors))       # VALIDATE mode is deterministic (noise == 1, bg .5)
    assert r1.edge_feats is None and torch.isfinite(r1.colors).all() and torch.isfinite(r1.depth).all()
    # rays that hit nothing: background colour, depth 512 (Renderer.cpp:83-97)
    o2 = np.full((4, 3), 600., np.float32); d2 = np.ones((4, 3), np.float32)
    with torch.no_grad():
        r = renderer.Render(T(o2), T(d2), None, None)
    assert r.weights is None and (N(r.colors) == 0.5).all() and (N(r.depth) == 512.).all()


def test_render_whole_image_matches_chunked_render(scene):
    """N4: RenderWholeImage == the reference's loop (ExpRunner.cpp:257-293) over our Render: same chunking (forced
    small here), same normalisations, CPU outputs; ragged last chunk; rays that miss everything."""
    from f2nerf_b200 import VALIDATE, RenderWholeImage
    gdp, sampler, field, shader, renderer = build(scene, use_app_emb=False)
    o, d, dn, cam = make_rays(scene, 700, seed=21)
    o[5] = 600.; d[5] = 1.
    pc, fo, pd = RenderWholeImage(renderer, torch.from_numpy(o), torch.from_numpy(d), None, ray_batch_size=256)
    assert not pc.is_cuda and pc.shape == (700, 3) and fo.shape == (700, 1) and pd.shape == (700, 1)
    gdp.mode_ = VALIDATE
    cols, disp, first = [], [], []
    with torch.no_grad():
        for i in range(0, 700, 256):
            r = renderer.Render(T(o[i:i + 256]), T(d[i:i + 256]), None, None)
            cols.append(r.colors); disp.append(r.disparity.reshape(-1, 1)); first.append(r.first_oct_dis.reshape(-1, 1))
    cols, disp, first = torch.cat(cols), torch.cat(disp), torch.cat(first)
    np.testing.assert_array_equal(N(pc), N(cols))
    np.testing.assert_array_equal(N(pd), N(disp / disp.max()))
    np.testing.assert_array_equal(N(fo), N(first.min() / first))
    assert (N(pc)[5] == 0.5).all()                                  # a ray that hits nothing shows the VALIDATE background


def test_operator_level_autograd(scene, oracle):
    """Hash3DAnchored.AnchoredQuery / SHShader.Query as stand-alone differentiable operators."""
    gdp, sampler, field, shader, renderer = build(scene)
    rng = np.random.default_rng(0)
    pts = T((rng.random((3000, 3), dtype=np.float32) * 2 - 1))
    vol = T(rng.integers(0, field.n_volumes_, 3000).astype(np.int32))
    out = field.AnchoredQuery(pts, vol)
    assert out.shape == (3000, 16) and out.requires_grad
    feats = torch.cat([torch.ones_like(out[:, :1]), out[:, 1:]], 1)
    dirs = torch.nn.functional.normalize(T(rng.standard_normal((3000, 3)).astype(np.float32)), dim=-1)
    rgb = shader.Query(feats, dirs)
    assert rgb.shape == (3000, 3)
    (rgb.sum() + out[:, 0].sum()).backward()
    for p in (field.feat_pool_, field.mlp_.params_, shader.mlp_.params_):
        assert p.grad is not None and torch.isfinite(p.grad).all() and float(p.grad.abs().sum()) > 0


@pytest.mark.parametrize("gs_progress", [1.0, 0.3])
def test_prefetched_march_equals_unpipelined(scene, gs_progress):
    """Renderer.prefetch_next (the next batch's march queued behind this batch's backward, on the octree-vote stream) must not
    change a single bit: same noise numbers (drawn ahead from the right Philox position, incl. the GradientScaling burns of
    the pending backward), same pruned octree, same outputs and gradients over three consecutive TRAIN steps; a prefetch for
    rays that are not the ones rendered next is ignored."""
    from f2nerf_b200 import TRAIN
    batches = [make_rays(scene, n, seed=40 + i) for i, n in enumerate((150, 97, 150))]
    outs = []
    for pipelined in (False, True, "early"):               # "early": Render launches the next march itself (set_next_rays),
        gdp, sampler, field, shader, renderer = build(scene)   # behind its occupancy votes, into the other scratch set
        gdp.mode_, gdp.gradient_scaling_progress_ = TRAIN, gs_progress
        torch.manual_seed(2024)
        dev_batches = [(T(o), T(d), T(cam)) for o, d, dn, cam in batches]
        rec = []
        for i, (ro, rd, cam) in enumerate(dev_batches):
            for p in (field.feat_pool_, field.mlp_.params_, shader.mlp_.params_, renderer.app_emb_):
                p.grad = None
            if pipelined == "early":
                nxt = dev_batches[(i + 1) % len(dev_batches)]
                renderer.set_next_rays(nxt[0], nxt[1])
            r = renderer.Render(ro, rd, None, cam)
            if pipelined == "early":
                assert sampler._prefetched is not None             # launched inside Render
            elif pipelined and i + 1 < len(dev_batches):
                renderer.prefetch_next(dev_batches[i + 1][0], dev_batches[i + 1][1])
            elif pipelined and i + 1 == len(dev_batches):
                renderer.prefetch_next(dev_batches[0][0], dev_batches[0][1])          # never consumed by a matching Render
            loss = (r.colors ** 2).mean() + r.disparity.mean() + 0.1 * ((r.edge_feats[:, 0] - r.edge_feats[:, 1]) ** 2).mean()
            loss.backward()
            rec += [N(r.colors), N(r.weights), N(r.idx_start_end), N(r.first_oct_dis), N(sampler.tree_weight_stats_),
                    N(shader.mlp_.params_.grad), N(renderer.app_emb_.grad)]
        # one more Render with rays the pending prefetch was NOT made for
        r = renderer.Render(dev_batches[1][0], dev_batches[1][1], None, dev_batches[1][2])
        rec += [N(r.colors), N(r.idx_start_end)]
        outs.append(rec)
    for other in outs[1:]:
        for k, (a, b) in enumerate(zip(outs[0], other)):
            if a.dtype == np.float32 and k % 7 in (5, 6) and k < 21:      # atomically accumulated gradients: summation order only
                np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-7 * np.abs(a).max())
            else:
                np.testing.assert_array_equal(a, b, err_msg=str(k))


# entry points the launch sequences of csrc/render.cu call in a TRAIN step with app embedding and TV-loss edge points
MARCH = ["f2b_sampler_march", "f2b_slot_bounds"]
PHASE1 = ["f2b_cast_f32_to_f16", "f2b_field_fwd_slots", "f2b_early_stop_rays", "f2b_count_scan"]
PHASE2 = ["f2b_compact_slots", "f2b_edge_samples", "f2b_hash_fwd", "f2b_scatter_idx", "f2b_cast_f32_to_f16", "f2b_cast_f32_to_f16",
          "f2b_field_shade_fwd", "f2b_mlp_fwd_f32", "f2b_shader_mlp_rgb_fwd", "f2b_composite_fwd"]
BWD = ["f2b_cast_f32_to_f16", "f2b_composite_act_bwd", "f2b_shade_field_bwd_scatter", "f2b_field_bwd_scatter"]
VOTES = ["f2b_oct_mark_visit", "f2b_oct_update_stats"]


@pytest.mark.parametrize("prefetch", [False, True])
def test_trace_only_observes(scene, prefetch):
    """The per-kernel trace (_lib.TRACE) of two TRAIN steps changes nothing: outputs and octree statistics bit for bit, gradients up
    to the order of the fp32 reductions, the same launch count.  It lists every entry point inside the launch sequences once per
    launch and no sequence as a whole; with ``prefetch`` the second step's march ran ahead (skip_march)."""
    from f2nerf_b200 import TRAIN, _lib
    batches = [make_rays(scene, n, seed=60 + i) for i, n in enumerate((150, 97))]
    outs, launches, trace = [], [], None
    for traced in (False, True):
        gdp, sampler, field, shader, renderer = build(scene)
        gdp.mode_ = TRAIN
        torch.manual_seed(31)
        dev_batches = [(T(o), T(d), T(cam)) for o, d, dn, cam in batches]
        rec = []
        l0 = _lib.LAUNCHES
        _lib.TRACE = [] if traced else None
        mark = torch.cuda.Event(enable_timing=True)
        mark.record()
        torch.cuda._sleep(50_000_000)                   # >= 25 ms of GPU time ahead of the step on the current stream
        try:
            for i, (ro, rd, cam) in enumerate(dev_batches):
                for p in (field.feat_pool_, field.mlp_.params_, shader.mlp_.params_, renderer.app_emb_):
                    p.grad = None
                r = renderer.Render(ro, rd, None, cam)
                if prefetch and i == 0:
                    renderer.prefetch_next(*dev_batches[1][:2])
                loss = (r.colors ** 2).mean() + r.disparity.mean() + 0.1 * ((r.edge_feats[:, 0] - r.edge_feats[:, 1]) ** 2).mean()
                loss.backward()
                rec.append(dict(colors=N(r.colors), disparity=N(r.disparity), depth=N(r.depth), weights=N(r.weights),
                                edge_feats=N(r.edge_feats), idx_start_end=N(r.idx_start_end), w_stats=N(sampler.tree_weight_stats_),
                                a_stats=N(sampler.tree_alpha_stats_), visits=N(sampler.tree_visit_cnt_),
                                g_table=N(field.feat_pool_.grad), g_field=N(field.mlp_.params_.grad),
                                g_shader=N(shader.mlp_.params_.grad), g_emb=N(renderer.app_emb_.grad)))
            torch.cuda.synchronize()
        finally:
            trace, _lib.TRACE = _lib.TRACE, None
        launches.append(_lib.LAUNCHES - l0)
        outs.append(rec)
    for a, b in zip(*outs):
        for k in a:
            if k.startswith("g_"):
                np.testing.assert_allclose(a[k], b[k], rtol=1e-5, atol=1e-7 * np.abs(a[k]).max(), err_msg=k)
            else:
                np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    assert launches[0] == launches[1]
    step = lambda march, prefetched: (["f2b_table_to_half"] + (MARCH if march else []) + PHASE1 + VOTES + PHASE2
                                      + (MARCH if prefetched else []) + BWD + ["f2b_render_grad_finalize"])
    names = [t[0] for t in trace]
    assert names == step(True, prefetch) + step(not prefetch, False), names
    assert all(a.elapsed_time(b) >= 0 for _, a, b, _ in trace)
    # the events bracket the kernels on the library's stream: the first sequence entry starts only behind the sleep (phase 1 is
    # enqueued well within 10 ms of host time, before the step's one host sync)
    assert mark.elapsed_time(trace[1][1]) > 10.0, (trace[1][0], mark.elapsed_time(trace[1][1]))


def test_render_empty_batch(scene):
    """A 0-ray batch returns the reference's empty RenderResult (Renderer.cpp:83-97) in TRAIN and VALIDATE mode.  The CUDA
    generator advances by the TRAIN noise draw only (1024 + 0 + 10 floats; the empty background takes no Philox offset), nothing
    in VALIDATE, and a pending prefetch of the next batch stays in place."""
    import contextlib
    from f2nerf_b200 import TRAIN, VALIDATE
    from f2nerf_b200.rng import rand_philox_offset
    gdp, sampler, field, shader, renderer = build(scene)
    o, d, dn, cam = make_rays(scene, 64, seed=3)
    nxt = (T(o), T(d))
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    empty = torch.zeros((0, 3), dtype=torch.float32, device="cuda")
    for mode, inc in ((TRAIN, rand_philox_offset(1034, "cuda")), (VALIDATE, 0)):
        gdp.mode_ = mode
        renderer.prefetch_next(*nxt)
        pf = sampler._prefetched
        off0 = gen.get_offset()
        with torch.no_grad() if mode == VALIDATE else contextlib.nullcontext():
            r = renderer.Render(empty, empty, None, torch.zeros((0,), dtype=torch.int32, device="cuda"))
        assert gen.get_offset() - off0 == inc
        assert sampler._prefetched is pf
        assert r.colors.shape == (0, 3) and r.first_oct_dis.shape == (0, 1) and r.disparity.shape == (0,) and r.depth.shape == (0,)
        assert r.edge_feats is None and r.weights is None and r.idx_start_end is None
        assert renderer.sample_result_._slots.n_rays == 0
        sampler.take_prefetched(*nxt)


@pytest.mark.parametrize("config", ["wanjinyou", "free"])
def test_fused_forward_matches_operator_pipeline(config, monkeypatch):
    """VALIDATE-mode Render through the ONE fused kernel behind the march (f2b_render_fwd_fused: encode -> field MLP -> early stop
    -> SH + shader MLP -> composite per ray, stopping at the first opaque sample) against the operator pipeline
    (f2b_render_phase1 + _phase2_fwd: every sample encoded, compaction, two MLP kernels, composite kernel) on the reference's
    ngp_fox scene: every RenderResult field bit for bit — colours, depth, disparity, the packed weights and their bounds."""
    import bench
    from types import SimpleNamespace
    from f2nerf_b200 import VALIDATE
    prob = bench.build_problem(0, 1, SimpleNamespace(config=config, rays=1500), torch.device("cuda", 0))
    renderer, gdp = prob["renderer"], prob["gdp"]
    o, d, cam, _ = prob["host"]
    o, d = o.copy(), d.copy()
    o[7] = 600.; d[7] = 1.                                           # a ray that hits nothing
    gdp.mode_ = VALIDATE
    with torch.no_grad():
        fused = renderer.Render(T(o), T(d), None, None)
        assert type(fused).__name__ == "ForwardRenderResult"
        f = {k: N(getattr(fused, k)) for k in ("colors", "disparity", "depth", "first_oct_dis", "weights", "idx_start_end")}
        monkeypatch.setenv("F2B_FUSED_FORWARD", "0")
        ref = renderer.Render(T(o), T(d), None, None)
        assert type(ref).__name__ == "RenderResult"
    kept = f["idx_start_end"][:, 1] - f["idx_start_end"][:, 0]
    marched = N(renderer.sample_result_.pts_idx_bounds)
    marched = marched[:, 1] - marched[:, 0]
    assert (kept < marched).sum() > 100 and kept[7] == 0             # early termination is exercised
    for k in f:
        np.testing.assert_array_equal(f[k].view(np.uint32) if f[k].dtype == np.float32 else f[k],
                                      N(getattr(ref, k)).view(np.uint32) if f[k].dtype == np.float32 else N(getattr(ref, k)), err_msg=k)
    assert (f["colors"][7] == 0.5).all()


def test_render_whole_image_matches_oracle(oracle):
    """N4: RenderWholeImage on rays of a reference ngp_fox camera (the committed fixture's blobs / cameras, the reference's
    parameter state) against the ORACLE's VALIDATE-mode forward of the same rays (noise == 1, background 0.5): sampler integers
    bit-exact upstream, colours / disparity within 1e-4 of scale given the same keep mask, the reference's normalisations
    (ExpRunner.cpp:289-290) applied on top."""
    import bench
    import oracle_pipeline as OP
    import workloads as W
    from types import SimpleNamespace
    from f2nerf_b200 import RenderWholeImage, ops
    n_rays = 3000                                                    # ragged against the 1024-ray chunks used below
    prob = bench.build_problem(0, 1, SimpleNamespace(config="wanjinyou", rays=n_rays), torch.device("cuda", 0))
    cfg, field, shader, renderer = prob["cfg"], prob["field"], prob["shader"], prob["renderer"]
    o, d, cam, _ = prob["host"]
    pc, fo, pd = RenderWholeImage(renderer, torch.from_numpy(o), torch.from_numpy(d), None, ray_batch_size=1024)
    dn = (d / np.linalg.norm(d, axis=-1, keepdims=True)).astype(np.float32)
    dn = N(T(d) / torch.linalg.norm(T(d), 2, -1, True))            # the device's normalisation (what the sampler sees)
    sc = dict(nodes=prob["blobs"][0], trans=prob["blobs"][1], edges=prob["blobs"][2], near=cfg["near"], sample_l=cfg["sample_l"],
              scale_by_dis=cfg["scale_by_dis"], max_hits=1024)
    fld = dict(table16=N(field.table_f16()), prim=N(field.prim_pool_), bias=N(field.bias_pool_), V=field.n_volumes_,
               local_size=field.local_size_, mlp_params=N(field.mlp_.params_))
    ref = OP.render_train(sc, o, dn, np.ones(1024 + n_rays + 10, np.float32), np.full((n_rays, 3), .5, np.float32), fld,
                          N(shader.mlp_.params_), None, None, None, None, scales=ops.hash_level_scales().numpy())
    colors, disp, first = ref["colors"], ref["disparity"].reshape(-1, 1), ref["sample"]["first_oct_dis"].reshape(-1, 1)
    assert np.abs(N(pc) - colors).max() <= 2e-3 and np.median(np.abs(N(pc) - colors)) <= 1e-5
    np.testing.assert_allclose(N(pd), disp / disp.max(), rtol=0, atol=5e-4)
    np.testing.assert_array_equal(N(fo), (first.min() / first).astype(np.float32))
