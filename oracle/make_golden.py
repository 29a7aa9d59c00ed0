#!/usr/bin/env python
"""Generate the committed golden fixtures tests/golden/ref_ngp_fox{,_512}_{run,rays,adam}.npz by running the UNMODIFIED
reference (oracle/_ref/ref_driver, built by oracle/Makefile.ref) on an H100:

    python oracle/make_golden.py OUT_DIR              # writes OUT_DIR/ref_ngp_fox{,_512}_{run,rays,adam}.npz
    python oracle/make_golden.py OUT_DIR --config free  # writes OUT_DIR/ref_free_512_{run,rays}.npz
    mv OUT_DIR/ref_*.npz tests/golden/

ref_ngp_fox_*: an 8-ray batch with every per-sample tensor.  ref_ngp_fox_512_*: the 512-ray batch tests/test_ref_parity.py's
``live`` cases run the reference on, stored for when its binary is not built: every per-ray tensor, and the per-sample tensors
of SAMPLE_RAYS seeded rays (``sample_rays``; their segments concatenated in ray order).  ``--config free``: the same 512-ray
batch under oracle/ref_config_free.yaml at the fineness and gradient-scaling progress of its iteration 0 (FREE_RUN), for
tests/test_gpu_ref_configs.py; no optimizer sample (the optimizer step does not depend on the config).

The fixture (tests/workloads.py:load_golden merges the two files, each kept under 1 MB: the scene and parameters in the first,
the ray batch's dumps in the second) holds the reference's own ngp_fox octree / warp blobs, a small seeded ray batch and every
boundary tensor of PersSampler::GetSamples, Hash3DAnchored::AnchoredQuery, SHShader::Query and
Renderer::Render for it (VALIDATE mode, plus the seeded TRAIN-mode sampler outputs and octree statistics).
tests/test_golden_ref.py pins oracle/f2_oracle.c against it on the CPU.  tests/golden/ref_ngp_fox.npz, the scene bench.py runs on,
is the scene part of an earlier run of this script, kept so that the benchmark's inputs stay fixed.  The 64 MB hash table is not stored:
both sides regenerate it from the CPU generator seed 1234 (see ref_driver.cpp).
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SAMPLE_RAYS = 6                   # rays of the 512-ray batch whose per-sample tensors are stored
N_EDGE = 1024                     # edge-point draws kept (of the 8192 the TV loss uses)
SH_STRIDE = 8                     # val_sh keeps the SH encoding of every 8th sample
SCENE = ("tree_nodes", "pers_trans", "edge_pool", "search_order", "prim_pool", "bias_pool", "field_mlp_params", "shader_mlp_params",
         "app_emb", "scalars", "ds_", "oct_", "level_scales")


# per-sample tensors -> the per-ray bounds that segment them
PER_SAMPLE = {"val_bounds": ("val_pts", "val_dirs", "val_dt", "val_t", "val_anchors", "val_scene_feat", "val_rgb", "val_sh"),
              "val_idx_start_end": ("val_weights",), "train_bounds": ("train_pts", "train_dt", "train_t", "train_anchors"),
              "train_idx_start_end": ("train_weights",)}


def segments(a, bounds, rays):
    """The rows of per-sample tensor ``a`` that belong to ``rays`` ([begin, end) row ranges per ray in ``bounds``), in ray order."""
    return np.concatenate([a[b:e] for b, e in bounds[rays]]) if len(rays) else a[:0]


# ref_driver's trailing [fineness, gs_progress] per config: what ExpRunner::UpdateAdaParams gives ref_config_free.yaml at
# iteration 0 (ray_march_init_fineness 4, no gradient scaling)
FREE_RUN = ("4", "1")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("dst_dir")
    ap.add_argument("--config", choices=("ngp_fox", "free"), default="ngp_fox")
    a = ap.parse_args()
    if a.config == "ngp_fox":
        dump(a.dst_dir, "ref_ngp_fox", 8, None)
        dump(a.dst_dir, "ref_ngp_fox_512", 512, SAMPLE_RAYS)
    else:
        dump(a.dst_dir, "ref_free_512", 512, SAMPLE_RAYS, "ref_config_free.yaml", FREE_RUN, with_adam=False)


def dump(dst_dir, prefix, n_rays, sample_rays, config="ref_config_ngp_fox.yaml", run_args=(), with_adam=True):
    drv = os.path.join(ROOT, "oracle", "_ref", "ref_driver")
    out = "/tmp/f2b_golden_dump"
    r = subprocess.run([drv, os.path.join(ROOT, "oracle", config), out, str(n_rays), "0", "1", *run_args], cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    if r.returncode != 0:
        print(r.stdout[-2000:], r.stderr[-4000:])
        sys.exit(1)
    keep = ["tree_nodes", "pers_trans", "edge_pool", "search_order", "prim_pool", "bias_pool", "field_mlp_params",
            "shader_mlp_params", "app_emb", "scalars", "rays_o", "rays_d", "rays_d_normed", "gt_colors", "emb_idx",
            "val_pts", "val_dirs", "val_dt", "val_t", "val_anchors", "val_bounds", "val_first_oct_dis", "val_scene_feat",
            "val_rgb", "val_sh", "val_colors", "val_disparity", "val_depth", "val_weights", "val_idx_start_end",
            "train_noise", "train_bg", "train_edge_idx", "train_edge_coord", "train_pts", "train_dt", "train_t", "train_anchors",
            "train_bounds", "train_colors", "train_disparity", "train_depth", "train_weights", "train_idx_start_end",
            "train_first_oct_dis", "train_tree_nodes_after", "train_weight_stats_after", "train_alpha_stats_after",
            "train_visit_cnt_after", "train_loss", "grad_field_mlp", "grad_shader_mlp",
            "edge_idx", "edge_coord", "edge_pts", "edge_anchors", "train_edge_feats",
            "ds_poses", "ds_intri", "ds_dist_params", "ray_ij", "ds_hw", "ds_bounds", "ds_train_set", "ray_bounds",
            "oct_intri", "oct_w2c", "oct_bound", "backward_nan",
            "oct_nodes_in", "oct_w_in", "oct_a_in", "oct_visit_in", "oct_nodes_sub", "oct_w_sub", "oct_a_sub",
            "oct_nodes_invis", "oct_nodes_final", "oct_w_final", "oct_a_final"]
    if os.path.exists(os.path.join(out, "grad_app_emb.npy")):          # not dumped when the config has no embedding
        keep.append("grad_app_emb")
    data = {k: np.load(os.path.join(out, k + ".npy")) for k in keep}
    if sample_rays:
        rays = np.sort(np.random.default_rng(2).choice(n_rays, sample_rays, replace=False))
        for bk, keys in PER_SAMPLE.items():
            for k in keys:
                data[k] = np.ascontiguousarray(segments(data[k], data[bk], rays))
        data["sample_rays"] = rays.astype(np.int32)
    for k in ("edge_idx", "edge_coord", "edge_pts", "edge_anchors"):         # N_EDGE of the 8192 draws are plenty
        data[k] = np.ascontiguousarray(data[k][:N_EDGE])
    data["val_sh"] = np.ascontiguousarray(data["val_sh"][::SH_STRIDE])     # SH of every SH_STRIDE-th sample direction
    data["val_sh_stride"] = np.array([SH_STRIDE], np.int32)
    # the reference's hash-table gradient (64 MB dense) as a seeded 2^15-element subsample of its live prefix + per-slab norms
    g = np.load(os.path.join(out, "grad_feat_pool.npy")).reshape(-1)
    local = ((int(data["scalars"][5]) // 16) >> 4) << 4
    sub = np.sort(np.random.default_rng(0).choice(17 * local, 1 << 15, replace=False)).astype(np.int32)
    data["grad_feat_pool_sub_idx"], data["grad_feat_pool_sub_val"] = sub, g[sub].astype(np.float32)
    data["grad_feat_pool_slab_norm"] = np.array([np.linalg.norm(g[l * local:(l + 1) * local].astype(np.float64)) for l in range(17)], np.float32)
    assert not g[17 * local:].any()
    data["train_edge_feats"] = np.ascontiguousarray(data["train_edge_feats"][:N_EDGE]).astype(np.float16)   # fp16 values
    # the level scales as the device computes them (MUFU.EX2): the oracle takes them as an input
    sys.path.insert(0, ROOT)
    from f2nerf_b200 import ops
    data["level_scales"] = ops.hash_level_scales().numpy()
    # the reference's two torch::optim::Adam steps on its own field parameters and gradients: the MLP vector whole, the table as a
    # seeded sample (Adam is elementwise) of its live prefix followed by a few elements of the dead rest, where Adam is the identity
    ld = lambda k: np.load(os.path.join(out, k + ".npy")).reshape(-1)
    live = 17 * local
    rng = np.random.default_rng(1)
    idx = np.concatenate([np.sort(rng.choice(live, 1 << 13, replace=False)), np.sort(rng.choice(np.arange(live, g.size), 256, replace=False))])
    adam = {"adam_lr": ld("adam_lr").astype(np.float32), "adam_feat_pool_n_live": np.array([1 << 13], np.int32),
            "adam_feat_pool_idx": idx.astype(np.int32), "adam_feat_pool_grad": g[idx].astype(np.float32),
            "adam_feat_pool_before": ld("feat_pool_before_adam")[idx], "adam_feat_pool_after": ld("feat_pool_after_adam")[idx],
            "adam_field_mlp_grad": ld("grad_field_mlp"), "adam_field_mlp_before": ld("field_mlp_before_adam"),
            "adam_field_mlp_after": ld("field_mlp_after_adam")}
    data["val_scene_feat"] = data["val_scene_feat"].astype(np.float16)       # tcnn outputs are fp16 values
    data["train_edge_coord"] = data["train_edge_coord"].astype(np.float32)
    os.makedirs(dst_dir, exist_ok=True)
    scene = {k: v for k, v in data.items() if k.startswith(SCENE)}
    parts = [(prefix + "_run.npz", scene), (prefix + "_rays.npz", {k: v for k, v in data.items() if k not in scene})]
    for name, part in parts + ([(prefix + "_adam.npz", adam)] if with_adam else []):
        dst = os.path.join(dst_dir, name)
        np.savez_compressed(dst, **part)
        print("wrote", dst, os.path.getsize(dst) / 1e6, "MB")


if __name__ == "__main__":
    main()
