"""The C++ drop-in host over consecutive training iterations, inside the reference's own program: ``ref_driver --steps``
(oracle/ref_driver.cpp) runs ten iterations of the body of ExpRunner::Train on ngp_fox with the schedule of
oracle/ref_config_ngp_fox_steps.yaml — compaction every 3 iterations from iteration 0, subdivision milestones at 4 and 6,
gradient-scaling progress ramping through 1, a ramping var-loss weight, the batch size from the meaningful-samples EMA —
and dumps every iteration's starting state, outputs, loss, gradients, octree afterwards and a probe of both generators.

a. The fused C++ host (f2nerf_b200/shim/B200Renderer.cpp) against the Python host, iteration by iteration.  Each iteration
   is replayed from the C++ run's dumped state (so atomic-order gradient differences do not accumulate) through Render,
   the same loss, backward and PersSampler.maintain.  Bit-identical: the probes, the batch size, every deterministic output,
   and after the step the tree, its statistics and visit counts and the remaining milestones; the loss to 1e-6, the
   gradients to fp32 summation order, the EMAs to fp32 rounding (the Python host keeps them in double).  On the
   maintenance iterations this also holds the reference's own host ProcOctree / MarkInvisibleNodes, which the C++ host runs
   inside Render, to f2b_octree_proc / f2b_octree_mark_invisible on real training states.
b. The fused host and the operator shim (F2B_SHIM=ops) against the unmodified program, with a fixed batch size.  Exact: the
   probes and the remaining milestones at every iteration, the sampler outputs at iteration 0.  Measured bars: the loss,
   and the node count after each maintenance (the arms' votes differ by tiny-cuda-nn's fp16 noise, Adam carries it on).
c. Each case asserts that it covered what it is for: compaction at iteration 0 and renumbering later, leaves split on each
   milestone (one of them a compaction iteration too), the batch size falling at least once, gradient-scaling progress
   crossing 1, and the C++ host's table-gradient storage reused across steps.
d. The non-finite back-off, on a copy of the config with an infinite TV-loss weight (three iterations, fixed batch): the TV
   term makes the edge points' dL/dout non-finite, which reaches the field MLP only.  So under TCNNWP.cpp:231-240 every
   iteration sets backward_nan_ (no Adam step, iter_step_ stays 0) and halves the field loss scale, 128 -> 64 -> 32, while
   the shader's stays 128 — in the unmodified program, on the C++ host (the flags of its gradient-finalize kernels) and on
   the Python host (check_backward_nan) replaying iteration 0 from the C++ run's state.
"""
import json
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from test_gpu_parity import N, T
from workloads import diag_path

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "ref_driver")
B200 = os.path.join(ROOT, "oracle", "_ref", "ref_driver_b200")
CONFIG = os.path.join(ROOT, "oracle", "ref_config_ngp_fox_steps.yaml")
N_ITERS = 10
FIXED_BATCH = 256
# b.: bars a few times above what an H100 SXM run measures (written to cpp_host_steps_margins_<arm>.json under
# workloads.diag_path): loss relative difference at most 1.5e-4 over the ten iterations, node counts after maintenance equal
LOSS_REL_BAR = 1e-3
NODES_REL_BAR = 2e-3
_runs = {}


def _load_dir(d):
    return {f[:-4]: np.load(os.path.join(d, f)) for f in os.listdir(d) if f.endswith(".npy")}


def _run(kind, fixed_batch, config=CONFIG, n_iters=N_ITERS):
    """``ref_driver --steps`` of one arm: "ref" (unmodified), "fused" (the C++ host) or "ops" (the operator shim), on ``config``
    (its paths are relative to the repository root, where the program runs)"""
    key = (kind, fixed_batch, config, n_iters)
    if key in _runs:
        return _runs[key]
    binary = REF if kind == "ref" else B200
    if not os.path.exists(binary):
        pytest.skip(f"{binary} not built (oracle/Makefile.ref)")
    tag = f"{kind}_{fixed_batch}" + ("" if config == CONFIG else "_" + os.path.splitext(os.path.basename(config))[0])
    out = os.path.join(tempfile.gettempdir(), f"f2b_cpp_host_steps_{tag}")
    shutil.rmtree(out, ignore_errors=True)
    env = {k: v for k, v in os.environ.items() if k not in ("F2B_SHIM", "F2B_RENDER")}
    if kind == "ops":
        env["F2B_SHIM"] = "ops"
    r = subprocess.run([binary, "--steps", config, out, str(n_iters), str(fixed_batch)], cwd=ROOT, capture_output=True, text=True,
                       timeout=900, env=env)
    open(diag_path(f"cpp_host_steps_{tag}.log"), "w").write(r.stdout[-20000:] + "\n--- stderr ---\n" + r.stderr[-20000:])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    if kind != "ref":
        assert ("replaced by the B200 subclasses" if kind == "ops" else "replaced by the fused B200 host") in r.stdout
    run = dict(root=_load_dir(out), its=[_load_dir(os.path.join(out, f"it{k}")) for k in range(n_iters)])
    shutil.rmtree(out, ignore_errors=True)
    _runs[key] = run
    return run


def node_fields(blob):
    """TreeNode blob -> the meaningful fields only (the reference never initialises the struct padding)."""
    t = np.ascontiguousarray(blob).view(np.uint8).reshape(-1, 64)
    return np.concatenate([t[:, :53], t[:, 56:60]], 1)


def valid_leaves(blob):
    t = np.ascontiguousarray(blob).view(np.uint8).reshape(-1, 64)
    return int(((t[:, 52] != 0) & (t.view(np.int32)[:, 14] >= 0)).sum())


def milestones(a):
    """the dumped [count, milestones...] -> the list as the sampler holds it (reversed, next one last)"""
    return a[1:1 + int(a[0])].tolist()


def bits(a):
    return a.view(np.uint32) if a.dtype == np.float32 else a


def ray_generator(root):
    from f2nerf_b200 import RayGenerator
    h, w = int(root["ds_hw"][0]), int(root["ds_hw"][1])
    return RayGenerator(root["ds_poses"].reshape(-1, 3, 4), root["ds_intri"].reshape(-1, 3, 3), root["ds_dist_params"], root["ds_bounds"],
                        images=None, height=h, width=w, train_set=root["ds_train_set"].tolist())


def python_step(root, it, k, gen):
    """Render + loss + backward of iteration k on the Python host, from the C++ run's dumped starting state (the caller then
    reads the non-finite flags: check_nonfinite)"""
    from test_ref_parity import build_from_ref
    from f2nerf_b200 import TRAIN, CustomOps
    st = it["state"]
    gdp, sampler, field, shader, renderer = build_from_ref(root)
    field.feat_pool_.data.copy_(T(it["feat_pool"]))
    field.mlp_.params_.data.copy_(T(it["field_mlp_params"]))
    shader.mlp_.params_.data.copy_(T(it["shader_mlp_params"]))
    renderer.app_emb_.data.copy_(T(it["app_emb"]))
    sampler.tree_nodes_gpu_ = T(it["tree_nodes"])
    sampler.tree_weight_stats_, sampler.tree_alpha_stats_ = T(it["weight_stats"]), T(it["alpha_stats"])
    sampler.tree_visit_cnt_ = T(it["visit_cnt"])
    sampler.sub_div_milestones_ = milestones(it["milestones"])          # as dumped: the reference consumes from the back
    gdp.mode_, gdp.iter_step_ = TRAIN, int(st[0])
    gdp.ray_march_fineness_, gdp.gradient_scaling_progress_ = float(st[2]), float(st[3])
    field.mlp_.loss_scale_, shader.mlp_.loss_scale_ = float(st[4]), float(st[5])
    gdp.sampled_oct_per_ray_, gdp.sampled_pts_per_ray_, gdp.meaningful_sampled_pts_per_ray_ = (float(x) for x in st[6:9])
    n_rays = int(st[1])
    pts_batch = np.float32(root["run"][1])
    assert n_rays == int(pts_batch / np.float32(st[8])) >> 4 << 4, f"iteration {k}: batch size"     # ExpRunner.cpp:86 in fp32
    torch.manual_seed(int(root["run"][2]) + k)
    (ro, rd, _), _, cam = gen.RandRaysData(n_rays)
    np.testing.assert_array_equal(N(ro).view(np.uint32), it["rays_o"].view(np.uint32), err_msg=f"rays_o, iteration {k}")
    np.testing.assert_array_equal(N(rd).view(np.uint32), it["rays_d"].view(np.uint32), err_msg=f"rays_d, iteration {k}")
    np.testing.assert_array_equal(N(cam), it["emb_idx"], err_msg=f"camera indices, iteration {k}")
    gt = T(it["gt_colors"])
    r = renderer.Render(ro, rd, None, cam)
    w_var, w_disp, w_tv = (float(x) for x in st[9:12])
    loss = (torch.sqrt((r.colors - gt) ** 2 + 1e-4).mean() + torch.sqrt(CustomOps.WeightVar(r.weights, r.idx_start_end) + 1e-2).mean() * w_var
            + (r.disparity ** 2).mean() * w_disp + ((r.edge_feats[:, 0] - r.edge_feats[:, 1]) ** 2).mean() * w_tv)
    loss.backward()
    return (gdp, sampler, field, shader, renderer), r, loss.detach()


def check_nonfinite(renderer, it, nonfinite):
    """The Python host's non-finite back-off (check_backward_nan) fired iff ``nonfinite``, as the C++ run's backward_nan_ did"""
    from f2nerf_b200 import check_backward_nan
    assert check_backward_nan(renderer) == nonfinite and it["after"][4] == int(nonfinite)


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64).reshape(-1), np.asarray(b, np.float64).reshape(-1)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def replay(root, it, k, gen):
    """Iteration k through the Python host, checked against the C++ host's dumps -> summary of the iteration"""
    compact_freq = int(root["run"][0])
    st = it["state"]
    (gdp, sampler, field, shader, renderer), r, loss = python_step(root, it, k, gen)
    check_nonfinite(renderer, it, False)
    n_rays = int(st[1])
    voted_visits = N(sampler.tree_visit_cnt_)
    sampler.maintain((root["oct_intri"].reshape(-1, 3, 3), root["oct_w2c"].reshape(-1, 3, 4), root["oct_bound"]), compact_freq)
    probe_cpu, probe_cuda = N(torch.rand(4)), N(torch.rand(4, device="cuda"))
    np.testing.assert_array_equal(probe_cpu, it["probe_cpu"], err_msg=f"CPU generator probe, iteration {k}")
    np.testing.assert_array_equal(probe_cuda, it["probe_cuda"], err_msg=f"CUDA generator probe, iteration {k}")
    for name, v in (("colors", r.colors), ("disparity", r.disparity), ("depth", r.depth), ("weights", r.weights),
                    ("idx_start_end", r.idx_start_end), ("edge_feats", r.edge_feats), ("first_oct_dis", r.first_oct_dis)):
        np.testing.assert_array_equal(bits(N(v)), bits(it[name]), err_msg=f"{name}, iteration {k}")
    assert abs(float(loss) - float(it["loss"][0])) <= 1e-6 * abs(float(it["loss"][0])), (k, float(loss), float(it["loss"][0]))
    g_table = np.zeros(it["feat_pool"].size, np.float32)
    g_table[it["grad_feat_pool_nz_idx"]] = it["grad_feat_pool_nz_val"]
    rel = {name: rel_l2(N(g), want) for name, g, want in (
        ("field_mlp", field.mlp_.params_.grad, it["grad_field_mlp"]), ("shader_mlp", shader.mlp_.params_.grad, it["grad_shader_mlp"]),
        ("app_emb", renderer.app_emb_.grad, it["grad_app_emb"]), ("feat_pool", field.feat_pool_.grad, g_table))}
    noise = None
    if rel["feat_pool"] > 1e-5:
        # The table gradient is summed with fp32 atomics in no fixed order, so two runs of the same host differ too: the same
        # iteration once more on the Python host measures that noise, and the C++ host may differ by no more than a few times it
        # (a stale or wrongly zeroed gradient storage differs by O(1)).
        objs2, _, _ = python_step(root, it, k, gen)
        check_nonfinite(objs2[4], it, False)
        noise = rel_l2(N(objs2[2].feat_pool_.grad), N(field.feat_pool_.grad))
    for name, v in rel.items():
        bar = max(1e-5, 4 * noise) if (name == "feat_pool" and noise is not None) else 1e-5
        assert v <= bar, f"gradient {name}, iteration {k}: relative L2 {v:.3g} (Python host against itself {noise})"
    np.testing.assert_array_equal(node_fields(N(sampler.tree_nodes_gpu_)), node_fields(it["after_tree_nodes"]), err_msg=f"tree, iteration {k}")
    for name, v in (("weight_stats", sampler.tree_weight_stats_), ("alpha_stats", sampler.tree_alpha_stats_), ("visit_cnt", sampler.tree_visit_cnt_)):
        np.testing.assert_array_equal(N(v), it["after_" + name], err_msg=f"{name} after iteration {k}")
    assert sampler.sub_div_milestones_ == milestones(it["after_milestones"]), k
    np.testing.assert_allclose([gdp.sampled_oct_per_ray_, gdp.sampled_pts_per_ray_, gdp.meaningful_sampled_pts_per_ray_], it["after"][1:4],
                               rtol=1e-6, err_msg=f"EMAs after iteration {k}")
    return dict(iter_step=int(st[0]), n_rays=n_rays, gs_progress=float(st[3]), fineness=float(st[2]), loss=float(loss),
                compaction=int(st[0]) % compact_freq == 0, milestones_before=milestones(it["milestones"]),
                milestones_after=milestones(it["after_milestones"]), nodes_before=it["tree_nodes"].size // 64,
                nodes_after=it["after_tree_nodes"].size // 64, leaves_before=valid_leaves(it["tree_nodes"]),
                leaves_after=valid_leaves(it["after_tree_nodes"]), voted_visits=int(voted_visits.sum()),
                visits_after=int(it["after_visit_cnt"].sum()), grad_reused=int(it["after"][5]), grad_fresh=int(it["after"][6]),
                grad_rel_l2=rel, table_grad_self_noise=noise)


def test_fused_cpp_host_equals_python_host_each_iteration():
    """a. and c. of the module text"""
    run = _run("fused", 0)
    root = run["root"]
    gen = ray_generator(root)
    recs = []
    try:
        for k, it in enumerate(run["its"]):
            recs.append(replay(root, it, k, gen))
    finally:
        json.dump(recs, open(diag_path("cpp_host_steps_fused_vs_python.json"), "w"), indent=1)
    # c. what the run covered
    assert [r["iter_step"] for r in recs] == list(range(N_ITERS))
    r0 = recs[0]
    assert r0["compaction"] and r0["voted_visits"] > 0 and r0["visits_after"] == 0, r0            # ProcOctree ran at step 0
    assert any(r["compaction"] and r["nodes_after"] != r["nodes_before"] for r in recs[1:]), "no later maintenance renumbered nodes"
    split = [r for r in recs if r["milestones_after"] != r["milestones_before"]]
    assert [r["iter_step"] for r in split] == [4, 6], [r["iter_step"] for r in split]
    assert all(r["leaves_after"] > r["leaves_before"] for r in split), [(r["leaves_before"], r["leaves_after"]) for r in split]
    assert any(r["compaction"] for r in split), "no milestone on a compaction iteration"
    n = [r["n_rays"] for r in recs]
    assert any(b < a for a, b in zip(n, n[1:])) and len(set(n)) > 2, n
    gs = [r["gs_progress"] for r in recs]
    assert gs[0] < 1 and gs[-1] >= 1 and any(0 < g < 1 for g in gs), gs
    assert recs[0]["grad_fresh"] == 1 and recs[-1]["grad_reused"] >= 1, (recs[0], recs[-1])


@pytest.mark.parametrize("kind", ["fused", "ops"])
def test_hosts_against_unmodified_program(kind):
    """b. of the module text"""
    ref, mine = _run("ref", FIXED_BATCH), _run(kind, FIXED_BATCH)
    a0, b0 = ref["its"][0], mine["its"][0]
    for name in ("rays_o", "rays_d", "emb_idx", "sample_bounds", "sample_anchors", "sample_pts", "sample_dt", "sample_t", "first_oct_dis"):
        np.testing.assert_array_equal(bits(b0[name]), bits(a0[name]), err_msg=f"{name}, iteration 0")
    margins = []
    for k, (a, b) in enumerate(zip(ref["its"], mine["its"])):
        for name in ("probe_cpu", "probe_cuda"):
            np.testing.assert_array_equal(b[name], a[name], err_msg=f"{name}, iteration {k}")
        assert milestones(b["after_milestones"]) == milestones(a["after_milestones"]), k
        assert a["after"][4] == 0 and b["after"][4] == 0
        la, lb = float(a["loss"][0]), float(b["loss"][0])
        na, nb = a["after_tree_nodes"].size // 64, b["after_tree_nodes"].size // 64
        maint = (int(a["state"][0]) % int(ref["root"]["run"][0]) == 0
                 or milestones(a["after_milestones"]) != milestones(a["milestones"]))
        margins.append(dict(iteration=k, loss_ref=la, loss=lb, loss_rel=abs(lb - la) / abs(la), maintenance=bool(maint),
                            nodes_ref=int(na), nodes=int(nb), nodes_rel=abs(nb - na) / na))
    json.dump(margins, open(diag_path(f"cpp_host_steps_margins_{kind}.json"), "w"), indent=1)
    assert max(m["loss_rel"] for m in margins) <= LOSS_REL_BAR, margins
    assert sum(m["maintenance"] for m in margins) >= 4, margins
    assert max(m["nodes_rel"] for m in margins if m["maintenance"]) <= NODES_REL_BAR, margins


def test_nonfinite_backward_backs_off_the_field_loss_scale(tmp_path):
    """d. of the module text"""
    text = open(CONFIG).read()
    assert "  tv_loss_weight: 0.1\n" in text
    config = str(tmp_path / "ref_config_ngp_fox_steps_tv_inf.yaml")
    open(config, "w").write(text.replace("  tv_loss_weight: 0.1\n", "  tv_loss_weight: .inf\n"))
    seqs = {}
    for kind in ("ref", "fused"):
        its = _run(kind, FIXED_BATCH, config, 3)["its"]
        assert all(np.isinf(it["state"][11]) for it in its), kind                  # the case covered what it is for
        # per iteration: iter_step before / after, backward_nan_ skip, Adam step taken, field / shader loss scale
        seqs[kind] = [(int(it["state"][0]), int(it["after"][0]), int(it["after"][4]), int(it["after"][7]), float(it["state"][4]),
                       float(it["state"][5])) for it in its]
        assert seqs[kind] == [(0, 0, 1, 0, 128., 128.), (0, 0, 1, 0, 64., 128.), (0, 0, 1, 0, 32., 128.)], (kind, seqs[kind])
    assert seqs["fused"] == seqs["ref"]
    # the Python host from the C++ run's state at iteration 0: the same flags, the same two loss scales afterwards
    run = _run("fused", FIXED_BATCH, config, 3)
    (gdp, _, field, shader, renderer), _, _ = python_step(run["root"], run["its"][0], 0, ray_generator(run["root"]))
    check_nonfinite(renderer, run["its"][0], True)
    assert gdp.backward_nan_
    assert (field.mlp_.loss_scale_, shader.mlp_.loss_scale_) == tuple(run["its"][1]["state"][4:6].tolist()), (
        field.mlp_.loss_scale_, shader.mlp_.loss_scale_)
