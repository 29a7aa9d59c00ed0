"""Resuming training from a reference checkpoint on the device (checkpoint.load_scene(trainable=True), octree_build).

- From the ngp_fox data directory, on CUDA, the rebuilt initial octree and its edge pool equal the reference program's
  (tests/golden/ref_ngp_fox.npz: ``tree_nodes`` / ``edge_pool``).
- The reference program with this library's renderer linked in (oracle/_ref/ref_driver_b200) trains ngp_fox for 300
  iterations; ``load_scene(trainable=True)`` on its checkpoint carries the reference's resumed edge pool and the saved
  iteration's gradient-scaling progress, and continues training: 20 steps of ``Render`` + the bench's loss + ``FusedAdam``
  end with finite gradients and no ``backward_nan_``.
- Against the reference program's own resume of that checkpoint (oracle/ref_resume.cpp: ExpRunner with is_continue: true,
  then one seeded TRAIN step): the same edge pool, octree, warps, fineness and gradient-scaling progress, the same edge
  draws, and the same first step — bit for bit against the program with this library's fused host, within DESIGN §5's
  fp16 bars against the unmodified program.
- Load times (plain and trainable, against the reference constructor's ``PersOctree::PersOctree`` time in the same run) are
  printed; BASELINE.md §3 records them.
"""
import os
import re
import subprocess
import time

import numpy as np
import pytest
import torch
import yaml

from test_checkpoint_cpu import FOX, FOX_CONFIG, GOLDEN, assert_same_states, need_fox
from test_octree_build_cpu import fields_mask

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRV_B200 = os.path.join(ROOT, "oracle", "_ref", "ref_driver_b200")
END_ITER = 300                       # before gradient_scaling_start (1000): the resumed progress is 0, not the default 1


def golden():
    return np.load(os.path.join(GOLDEN, "ref_ngp_fox.npz"))


def fox_config():
    with open(FOX_CONFIG) as f:
        return yaml.safe_load(f)


@need_fox
def test_initial_octree_on_device_matches_reference():
    from f2nerf_b200 import initial_octree, load_dataset
    ds = load_dataset(FOX, 2, [0.5, 4.0], "cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    nodes, pool = initial_octree(ds, fox_config()["pts_sampler"])
    print(f"initial_octree on ngp_fox: {time.perf_counter() - t0:.3f} s ({len(nodes)} nodes, {len(pool)} edges)")
    z = golden()
    got, want = nodes.view(np.uint8).reshape(-1, 64), z["tree_nodes"].reshape(-1, 64)
    assert got.shape == want.shape
    m = fields_mask()
    assert np.array_equal(got[:, m], want[:, m])
    assert np.array_equal(pool.view(np.uint8).reshape(-1), z["edge_pool"])


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


@pytest.fixture(scope="module")
def resumed(tmp_path_factory):
    if not (os.path.isfile(DRV_B200) and os.path.isfile(os.path.join(FOX, "image_list.txt"))):
        pytest.skip("oracle/_ref/ref_driver_b200 or its ngp_fox data not built (oracle/Makefile.ref)")
    from f2nerf_b200 import load_scene
    tmp = tmp_path_factory.mktemp("resume")
    cfg = fox_config()
    cfg["base_exp_dir"] = str(tmp / "exp")
    cfg["train"].update(end_iter=END_ITER, save_freq=END_ITER)
    conf = tmp / "runtime_config.yaml"
    conf.write_text(yaml.safe_dump(cfg))
    r = subprocess.run([DRV_B200, "--train", str(conf)], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    ref_octree_s = float(re.search(r"\[PersOctree::PersOctree\] end in ([0-9.e+-]+) seconds", r.stdout).group(1))
    cwd = os.getcwd()
    os.chdir(ROOT)                                               # data_path is relative to the program's directory
    try:
        _, plain_s = timed(lambda: load_scene(str(conf), device="cuda"))
        scene, trainable_s = timed(lambda: load_scene(str(conf), device="cuda", trainable=True))
        wrong = tmp / "wrong_split.yaml"
        cfg["pts_sampler"]["split_dist_thres"] = 1.25
        wrong.write_text(yaml.safe_dump(cfg))
        with pytest.raises(ValueError, match="split_dist_thres = 1.25"):
            load_scene(str(wrong), checkpoint_dir=str(tmp / "exp" / "checkpoints" / "latest"), device="cuda", trainable=True)
    finally:
        os.chdir(cwd)
    print(f"ngp_fox load times (s): load_scene {plain_s:.3f}, load_scene(trainable=True) {trainable_s:.3f}, "
          f"reference PersOctree::PersOctree {ref_octree_s:.3f}")
    cfg["pts_sampler"]["split_dist_thres"] = fox_config()["pts_sampler"]["split_dist_thres"]
    cfg["is_continue"] = True
    resume_conf = tmp / "continue.yaml"
    resume_conf.write_text(yaml.safe_dump(cfg))
    return dict(scene=scene, exp=tmp / "exp", conf=str(conf), resume_conf=str(resume_conf), tmp=tmp)


def test_resumed_scene_state(resumed):
    from f2nerf_b200 import VALIDATE, load_states
    scene = resumed["scene"]
    gdp, sampler = scene.global_data_pool, scene.renderer.pts_sampler_
    assert scene.iter_step == END_ITER and gdp.mode_ == VALIDATE
    assert gdp.gradient_scaling_progress_ == 0.0                 # UpdateAdaParams at iteration 300 of a 1000..5000 ramp
    assert sampler.n_edges == 1131
    assert np.array_equal(sampler.edge_pool_gpu_.cpu().numpy(), golden()["edge_pool"])
    archive = load_states(str(resumed["exp"] / "checkpoints" / "latest" / "renderer.pt"), "cuda")
    assert_same_states(scene.renderer.States(), archive)         # the checkpoint's octree and warps, not the rebuilt tree


def test_resumed_scene_continues_training(resumed):
    """20 optimizer steps as ExpRunner::Train takes them (ExpRunner.cpp:127-137): a step whose backward raised
    ``backward_nan_`` is not applied and the iteration is repeated.  The MLPs' loss scales are not part of the checkpoint,
    so a resumed run starts again from 128 and halves them on fp16 overflow, as the reference's TCNNWP does; that bounds
    the skipped steps by the halvings down to 1 (7 per MLP)."""
    from f2nerf_b200 import TRAIN, VALIDATE, CustomOps, FusedAdam, check_backward_nan
    scene = resumed["scene"]
    gdp, renderer, ds = scene.global_data_pool, scene.renderer, scene.dataset
    field, shader = renderer.scene_field_, renderer.shader_
    gdp.mode_, gdp.learning_rate_ = TRAIN, 1e-2                 # before OptimParamGroups, which reads it
    opt = FusedAdam(renderer.OptimParamGroups(), table_field=field)
    torch.manual_seed(2024)
    steps, skipped = 0, 0
    try:
        while steps < 20:
            assert skipped <= 14, "more non-finite backward passes than loss-scale halvings"
            gdp.iter_step_ = END_ITER + steps
            gdp.backward_nan_ = False
            opt.zero_grad()
            (rays_o, rays_d, _), gt, emb_idx = ds.RandRaysData(8192)
            res = renderer.Render(rays_o, rays_d, None, emb_idx)
            color_loss = torch.sqrt((res.colors - gt) ** 2 + 1e-4).mean()
            var_loss = torch.sqrt(CustomOps.WeightVar(res.weights, res.idx_start_end) + 1e-2).mean()
            tv_loss = ((res.edge_feats[:, 0] - res.edge_feats[:, 1]) ** 2).mean()
            loss = color_loss + var_loss * 1e-2 + tv_loss * 1e-1
            loss.backward()
            assert bool(torch.isfinite(loss)), steps
            if check_backward_nan(renderer):
                skipped += 1
                continue
            for p in (field.feat_pool_, field.mlp_.params_, shader.mlp_.params_, renderer.app_emb_):
                assert p.grad is not None and bool(torch.isfinite(p.grad).all()), (steps, tuple(p.shape))
            assert float(field.feat_pool_.grad.abs().sum()) > 0
            opt.step()
            steps += 1
        assert not gdp.backward_nan_
    finally:
        torch.cuda.synchronize()
        gdp.mode_ = VALIDATE
    print(f"resumed 20 steps: {skipped} skipped on non-finite gradients; loss scales field {field.mlp_.loss_scale_}, "
          f"shader {shader.mlp_.loss_scale_}; last loss {float(loss):.5f}")


# ---- the first resumed TRAIN step against the reference program's own resume (oracle/ref_resume.cpp) --------------------

RESUME_DRV = {"fused": os.path.join(ROOT, "oracle", "_ref", "ref_resume_b200"),
              "ref": os.path.join(ROOT, "oracle", "_ref", "ref_resume")}
N_RAYS = 4096


@pytest.fixture(scope="module")
def program_resumes(resumed):
    """ExpRunner with is_continue: true on the 300-iteration checkpoint, then one seeded TRAIN step: with this library's fused
    host as Renderer::Render (ref_resume_b200) and unmodified (ref_resume)."""
    out = {}
    for kind, binary in RESUME_DRV.items():
        if not os.path.isfile(binary):
            pytest.skip(f"{binary} not built (oracle/Makefile.resume)")
        d = resumed["tmp"] / f"resume_{kind}"
        env = {k: v for k, v in os.environ.items() if k not in ("F2B_SHIM", "F2B_RENDER")}
        r = subprocess.run([binary, resumed["resume_conf"], str(d), str(N_RAYS)], cwd=ROOT, capture_output=True, text=True,
                           timeout=900, env=env)
        assert r.returncode == 0, (kind, r.stdout[-3000:], r.stderr[-3000:])
        assert ("replaced by the fused B200 host" in r.stdout) == (kind == "fused")
        out[kind] = {f[:-4]: np.load(d / f) for f in os.listdir(d) if f.endswith(".npy")}
    return out


def fresh_resume(resumed):
    from f2nerf_b200 import load_scene
    cwd = os.getcwd()
    os.chdir(ROOT)
    try:
        return load_scene(resumed["conf"], device="cuda", trainable=True)
    finally:
        os.chdir(cwd)


def node_fields(blob):
    return np.ascontiguousarray(blob).view(np.uint8).reshape(-1, 64)[:, fields_mask()]


def test_resumed_state_matches_program(resumed, program_resumes):
    """Edge pool, octree, warps, iteration, fineness and gradient-scaling progress as the program resumes them, and the
    edge-sample draws over them bit for bit."""
    scene = fresh_resume(resumed)
    gdp, sampler = scene.global_data_pool, scene.renderer.pts_sampler_
    torch.manual_seed(4242)
    pts, anchors = sampler.GetEdgeSamples(8192)
    torch.manual_seed(4242)
    idx = torch.randint(0, sampler.n_edges, (8192,), dtype=torch.int32, device="cuda")
    coord = torch.rand((8192, 2), dtype=torch.float32, device="cuda") * 2. - 1.
    for kind, c in program_resumes.items():
        assert np.array_equal(sampler.edge_pool_gpu_.cpu().numpy(), c["edge_pool"]), kind
        assert np.array_equal(sampler.pers_trans_gpu_.cpu().numpy(), c["pers_trans"]), kind
        assert np.array_equal(node_fields(sampler.tree_nodes_gpu_.cpu().numpy()), node_fields(c["tree_nodes"])), kind
        it, fineness, progress = c["resume_scalars"].tolist()
        assert it == scene.iter_step == END_ITER, kind
        assert np.float32(gdp.ray_march_fineness_) == np.float32(fineness), kind
        assert np.float32(gdp.gradient_scaling_progress_) == np.float32(progress), kind
        for k, v in (("edge_idx", idx), ("edge_coord", coord), ("edge_pts", pts), ("edge_anchors", anchors)):
            assert np.array_equal(v.cpu().numpy().view(np.uint32), c[k].view(np.uint32)), (kind, k)


def test_resumed_train_step_matches_program(resumed, program_resumes):
    """load_scene(trainable=True) + the program's seeded TRAIN step.  Against the program with this library's fused host:
    every deterministic output bit for bit, the atomically accumulated gradients to fp32 summation order (as
    tests/test_shim_dropin.py requires of the two hosts).  Against the unmodified program: DESIGN §5's fp16 bars, as
    tests/test_shim_dropin.py applies them."""
    from f2nerf_b200 import TRAIN, CustomOps, check_backward_nan
    scene = fresh_resume(resumed)
    gdp, renderer = scene.global_data_pool, scene.renderer
    field, shader = renderer.scene_field_, renderer.shader_
    c, ref = program_resumes["fused"], program_resumes["ref"]
    for k in ("rays_o", "rays_d", "gt_colors", "emb_idx"):
        assert np.array_equal(c[k], ref[k]), k
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    rays_o, rays_d, gt, emb_idx = cuda(c["rays_o"]), cuda(c["rays_d"]), cuda(c["gt_colors"]), cuda(c["emb_idx"])
    gdp.mode_, gdp.iter_step_ = TRAIN, END_ITER
    torch.manual_seed(777)
    r = renderer.Render(rays_o, rays_d, None, emb_idx)
    loss = (torch.sqrt((r.colors - gt) ** 2 + 1e-4).mean() + torch.sqrt(CustomOps.WeightVar(r.weights, r.idx_start_end) + 1e-2).mean() * 1e-2
            + (r.disparity ** 2).mean() * 1e-2 + ((r.edge_feats[:, 0] - r.edge_feats[:, 1]) ** 2).mean() * 1e-1)
    loss.backward()
    assert not check_backward_nan(renderer)
    assert c["backward_nan"][0] == 0 and ref["backward_nan"][0] == 0
    got = {k: v.detach().cpu().numpy() for k, v in (("train_colors", r.colors), ("train_disparity", r.disparity),
           ("train_depth", r.depth), ("train_weights", r.weights), ("train_edge_feats", r.edge_feats),
           ("train_first_oct_dis", r.first_oct_dis))}
    grads = {k: g.detach().cpu().numpy().reshape(-1) for k, g in (("grad_field_mlp", field.mlp_.params_.grad),
             ("grad_shader_mlp", shader.mlp_.params_.grad), ("grad_app_emb", renderer.app_emb_.grad),
             ("grad_feat_pool", field.feat_pool_.grad))}
    # the fused host inside the resumed program
    assert np.array_equal(r.idx_start_end.cpu().numpy(), c["train_idx_start_end"])
    for k, v in got.items():
        assert np.array_equal(v.view(np.uint32), c[k].view(np.uint32)), k
    assert abs(float(loss) - float(c["train_loss"][0])) <= 1e-6 * abs(float(loss))
    for k, g in grads.items():
        a, b = g.astype(np.float64), c[k].astype(np.float64).reshape(-1)
        assert np.linalg.norm(a - b) <= 1e-5 * np.linalg.norm(b), (k, np.linalg.norm(a - b) / np.linalg.norm(b))
    # the unmodified resumed program (tiny-cuda-nn fp16 MLPs)
    ca, cb = ref["train_idx_start_end"], r.idx_start_end.cpu().numpy()
    na, nb = ca[:, 1] - ca[:, 0], cb[:, 1] - cb[:, 0]
    assert (na == nb).mean() >= 0.9 and abs(int(na.sum()) - int(nb.sum())) <= 2e-3 * na.sum(), (na == nb).mean()
    np.testing.assert_allclose(got["train_colors"], ref["train_colors"], atol=0.03)
    assert np.median(np.abs(got["train_colors"] - ref["train_colors"])) <= 3e-3
    for k in ("depth", "disparity"):
        rel = np.abs(got[f"train_{k}"] - ref[f"train_{k}"]) / (np.abs(ref[f"train_{k}"]) + 1e-3)
        assert np.median(rel) <= 1e-2, (k, np.median(rel))
    assert abs(float(loss) - float(ref["train_loss"][0])) <= 5e-3 * abs(float(ref["train_loss"][0]))
    cos = lambda a, b: float((a * b).sum() / (np.linalg.norm(a) * np.linalg.norm(b) + 1e-300))
    assert cos(got["train_edge_feats"].astype(np.float64).reshape(-1), ref["train_edge_feats"].astype(np.float64).reshape(-1)) >= 0.999
    for k, bar in (("grad_field_mlp", .98), ("grad_shader_mlp", .98), ("grad_app_emb", .98), ("grad_feat_pool", .97)):
        v = cos(grads[k].astype(np.float64), ref[k].astype(np.float64).reshape(-1))
        assert v >= bar, (k, v)
