#!/usr/bin/env python
"""Why the reference's hash-table gradient disagrees with the exact one (CPU study, test infrastructure).

The reference back-propagates the field MLP with fp16 accumulators (tiny-cuda-nn wmma fragments / CUTLASS
half accumulators) at loss scale 128, then rounds every (trilinear weight x grad) product to fp16 and adds it
with fp16 atomics (Hash3DAnchored.cu:145-151,220).  With a mean over 4096 rays the per-sample gradients x128
sit in fp16's subnormal range (step 6e-8), so every stage quantises at the 1-50 % level.  This script replays
the golden 12-ray ngp_fox step through the CPU oracle, scales the upstream gradient to the 4096-ray magnitude,
and compares  exact  vs  fp16-accumulate emulation  per level slab.  Output: one JSON on stdout.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_lib as O          # noqa: E402
import oracle_pipeline as OP    # noqa: E402

f16 = OP.f16


def mlp_bwd_half_accum(dout16, hidden16, params16):
    """field MLP (32 -> 64 -> 16, no bias) input gradient with an fp16 accumulator rounded after every
    16-wide k-step, as wmma<half accumulator> does."""
    W0 = params16[:64 * 32].reshape(64, 32).astype(np.float32)
    Wo = params16[64 * 32:64 * 32 + 16 * 64].reshape(16, 64).astype(np.float32)
    dh = f16(dout16.astype(np.float32) @ Wo)                     # K = 16: one k-step
    dh = np.where(hidden16 > 0, dh, np.float16(0))
    acc = np.zeros((dout16.shape[0], 32), np.float16)
    for c in range(4):                                           # K = 64: four k-steps
        acc = f16(acc.astype(np.float32) + dh[:, 16 * c:16 * c + 16].astype(np.float32) @ W0[16 * c:16 * c + 16])
    return acc


def cos(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(a @ b / (np.linalg.norm(a) * np.linalg.norm(b) + 1e-300))


def main():
    from workloads import load_golden
    g = load_golden()
    sc = g["scalars"]
    V, pool, R = int(sc[4]), int(sc[5]), int(sc[7])
    gen = torch.Generator().manual_seed(1234)
    table = (torch.rand((pool, 2), generator=gen) * 2. - 1.).numpy().astype(np.float16)
    local = ((pool // 16) >> 4) << 4
    scene = dict(nodes=g["tree_nodes"], trans=g["pers_trans"], edges=g["edge_pool"], near=float(sc[0]), sample_l=float(sc[1]),
                 scale_by_dis=bool(sc[2]), max_hits=int(sc[3]))
    fld = dict(table16=table, prim=g["prim_pool"], bias=g["bias_pool"], V=V, local_size=local, mlp_params=g["field_mlp_params"])
    rng = np.random.default_rng(5)
    gt = rng.random((R, 3), dtype=np.float32)
    out = OP.render_train(scene, g["rays_o"], g["rays_d_normed"], g["train_noise"], g["train_bg"], fld, g["shader_mlp_params"],
                          edge=(g["train_edge_idx"], g["train_edge_coord"]), gt_colors=gt, scales=g["level_scales"], gs_progress=0.25)
    d_scene, n_kept = out["d_scene"], out["n_kept"]
    m = out["keep"].astype(bool)
    s = out["sample"]
    e_pts, e_idx = O.edge_samples(scene["edges"], scene["trans"], g["train_edge_idx"], g["train_edge_coord"])
    q_pts = np.ascontiguousarray(np.concatenate([s["pts"][m], e_pts.reshape(-1, 3)], 0))
    q_vol = np.concatenate([s["anchors"][m][:, 0], e_idx.reshape(-1)]).astype(np.int32)
    p16 = f16(fld["mlp_params"])
    feat = O.hash_fwd(table, fld["prim"], fld["bias"], V, local, g["level_scales"], q_pts, q_vol, 1)
    _, hid = O.mlp_fwd(feat, p16, 0, save_hidden=True)
    report = {}
    for label, mul in (("12_rays", 1.0), ("as_4096_rays", R / 4096.0)):
        ds = d_scene.copy()
        ds[:n_kept] *= mul                                       # colour / variance / disparity terms are means over rays
        dout16 = f16(ds * OP.LOSS_SCALE)
        din_exact, _ = O.mlp_bwd(dout16, feat, hid, p16, 0)
        din_half = mlp_bwd_half_accum(dout16, hid.reshape(-1, 64), p16)
        args = (fld["prim"], fld["bias"], V, local, g["level_scales"], q_pts, q_vol, 1)
        exact = O.hash_bwd(*args, din_exact.astype(np.float32), 1.0 / OP.LOSS_SCALE, pool)
        emul = O.hash_bwd(*args, din_half.astype(np.float32), 1.0 / OP.LOSS_SCALE, pool, half_products=2)
        emul_mlp_only = O.hash_bwd(*args, din_half.astype(np.float32), 1.0 / OP.LOSS_SCALE, pool)
        emul_scatter_only = O.hash_bwd(*args, din_exact.astype(np.float32), 1.0 / OP.LOSS_SCALE, pool, half_products=2)
        ex, em = np.asarray(exact).ravel(), np.asarray(emul).ravel()
        slabs = [dict(slab=l, cos=cos(ex[l * local:(l + 1) * local], em[l * local:(l + 1) * local]),
                      norm_exact=float(np.linalg.norm(ex[l * local:(l + 1) * local])),
                      norm_emul=float(np.linalg.norm(em[l * local:(l + 1) * local]))) for l in range(17)]
        report[label] = dict(cos_exact_vs_full_emulation=cos(ex, em), cos_exact_vs_half_mlp_only=cos(ex, emul_mlp_only),
                             cos_exact_vs_half_scatter_only=cos(ex, emul_scatter_only),
                             din16_abs_median=float(np.median(np.abs(din_exact.astype(np.float32)))),
                             din16_frac_subnormal=float((np.abs(din_exact.astype(np.float32)) < 6.1e-5).mean()), slabs=slabs)
    print(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
