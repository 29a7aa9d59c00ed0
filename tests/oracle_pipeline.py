"""Renderer::Render (+ the trainer's loss and the full backward) composed from the CPU oracle pieces.

Test infrastructure (see oracle/f2_oracle.c): used by tests/test_gpu_render.py as the end-to-end checker,
by __graft_entry__.smoke() and by bench.py's cpu_baseline / --impl reference legs as the timed CPU port.
Follows src/Renderer/Renderer.cpp:52-213 and src/ExpRunner.cpp:94-118 step by step.
"""
import numpy as np

import oracle_lib as O

LOSS_SCALE = 128.0


def f16(x):
    return np.asarray(x, np.float32).astype(np.float16)


def render_train(sc, rays_o, rays_dn, noise, bg, field, shader_params, app_emb=None, emb_idx=None, edge=None,
                 gt_colors=None, scales=None, gs_progress=1.0, backward=True, loss_w=(1.0, 0.01, 0.01, 0.1),
                 diagnostics=False):
    """sc: dict(nodes, trans, edges, near, sample_l, scale_by_dis, max_hits)
    field: dict(table16 [pool,2] f16, prim, bias, V, local_size, mlp_params f32)
    edge: (edge_idx [n], edge_coord [n,2]) or None.  Returns dict of forward outputs (+ grads).
    loss_w: weights of the colour, variance, disparity and TV terms (ExpRunner.cpp:116-118), optionally a fifth one of a
    squared-depth term (mean depth^2) that takes the d_depth path of the composite backward."""
    out = {}
    s = O.sampler(sc["nodes"], sc["trans"], rays_o, rays_dn, noise, sc["near"], 1e8, sc["sample_l"], sc["scale_by_dis"],
                  sc["max_hits"])
    out["sample"] = s
    R, P = rays_o.shape[0], s["pts"].shape[0]
    scales = O.level_scales() if scales is None else scales
    fp16 = f16(field["mlp_params"])
    sp16 = f16(shader_params)

    def field_fwd(pts, vol, stride, save):
        feat = O.hash_fwd(field["table16"], field["prim"], field["bias"], field["V"], field["local_size"], scales, pts, vol, stride)
        o, hid = O.mlp_fwd(feat, fp16, 0, save_hidden=save)
        return o.astype(np.float32), feat, hid

    # early stop (no grad)
    feat_all, _, _ = field_fwd(s["pts"], s["anchors"], 3, False)
    w0, a0, keep, nb, n_kept = O.early_stop(feat_all, 16, s["dt"], s["bounds"])
    out.update(early_weights=w0, early_alphas=a0, keep=keep, bounds=nb, n_kept=n_kept)
    m = keep.astype(bool)
    pts, dirs, dt, t, anchors = s["pts"][m], s["dirs"][m], s["dt"][m], s["t"][m], s["anchors"][m]
    q_pts, q_vol = pts, np.ascontiguousarray(anchors[:, 0])
    n_edge = 0
    if edge is not None:
        e_pts, e_idx = O.edge_samples(sc["edges"], sc["trans"], edge[0], edge[1])
        n_edge = e_pts.shape[0] * 2
        q_pts = np.concatenate([pts, e_pts.reshape(-1, 3)], 0)
        q_vol = np.concatenate([q_vol, e_idx.reshape(-1)], 0).astype(np.int32)
    scene_feat, feat16, f_hid = field_fwd(np.ascontiguousarray(q_pts), q_vol, 1, True)
    pt_emb = None
    if app_emb is not None:
        pt_emb = np.repeat(emb_idx.astype(np.int32), nb[:, 1] - nb[:, 0])
    mlp_in = O.shader_prep(scene_feat[:n_kept], dirs, app_emb, pt_emb)
    raw, s_hid = O.mlp_fwd(mlp_in, sp16, 1, save_hidden=True)
    rgb = O.shader_act(raw)
    colors, disp, depth, weights = O.composite_fwd(scene_feat[:n_kept], 16, rgb, dt, t, nb, bg)
    edge_feats = scene_feat[n_kept:].reshape(-1, 2, 16)
    out.update(colors=colors, disparity=disp, depth=depth, weights=weights, edge_feats=edge_feats, scene_feat=scene_feat,
               rgb=rgb, pts=pts, feat16=feat16, mlp_in=mlp_in, raw=raw, q_pts=q_pts, q_vol=q_vol, dt=dt, t=t, dirs=dirs)
    if gt_colors is None:
        return out
    # losses (ExpRunner.cpp:94-118)
    wc, wv, wd, wt = loss_w[:4]
    wz = loss_w[4] if len(loss_w) > 4 else 0.0
    diff = colors - gt_colors
    color_loss = np.sqrt(diff * diff + 1e-4).mean()
    var, _ = O.weight_var(weights, nb)
    var_loss = np.sqrt(var + 1e-2).mean()
    disp_loss = (disp * disp).mean()
    tv = ((edge_feats[:, 0] - edge_feats[:, 1]) ** 2).mean() if n_edge else 0.0
    out["loss"] = wc * color_loss + wv * var_loss + wd * disp_loss + wt * tv + wz * (depth * depth).mean()
    if not backward:
        return out
    d_colors = (wc * diff / np.sqrt(diff * diff + 1e-4) / diff.size).astype(np.float32)
    d_var = (wv * 0.5 / np.sqrt(var + 1e-2) / R).astype(np.float32)
    _, d_weights = O.weight_var(weights, nb, d_var)
    d_disp = (wd * 2 * disp / R).astype(np.float32)
    d_depth = (wz * 2 * depth / R).astype(np.float32) if wz else None
    d_scene = np.zeros((scene_feat.shape[0], 16), np.float32)
    if n_edge:
        de = (wt * 2 * (edge_feats[:, 0] - edge_feats[:, 1]) / (edge_feats.shape[0] * 16)).astype(np.float32)
        d_scene[n_kept:] = np.stack([de, -de], 1).reshape(-1, 16)
    d_logit, d_rgb = O.composite_bwd(scene_feat[:n_kept], 16, rgb, dt, t, nb, bg, d_colors, d_disp, d_depth, d_weights, gs_progress)
    d_scene[:n_kept, 0] = d_logit
    # shader backward
    o3 = raw[:, :3].astype(np.float32)
    sg = 1.0 / (1.0 + np.exp(-o3))
    d_raw = np.zeros((n_kept, 16), np.float32)
    d_raw[:, :3] = d_rgb * (1.0 + 2e-3) * sg * (1 - sg) * LOSS_SCALE
    d_in16, d_sp = O.mlp_bwd(f16(d_raw), mlp_in, s_hid, sp16, 1)
    d_in = d_in16.astype(np.float32) / LOSS_SCALE
    d_scene[:n_kept, 1:] = d_in[:, 1:16]
    out["grad_shader_mlp"] = d_sp / LOSS_SCALE
    if app_emb is not None:
        g = np.zeros_like(app_emb, dtype=np.float64)
        np.add.at(g, pt_emb, d_in[:, :16].astype(np.float64))
        out["grad_app_emb"] = g
    # field backward
    d_feat16, d_fp = O.mlp_bwd(f16(d_scene * LOSS_SCALE), feat16, f_hid, fp16, 0)
    out["grad_field_mlp"] = d_fp / LOSS_SCALE
    out["grad_feat_pool"] = O.hash_bwd(field["prim"], field["bias"], field["V"], field["local_size"], scales,
                                       np.ascontiguousarray(q_pts), q_vol, 1, d_feat16.astype(np.float32), 1.0 / LOSS_SCALE,
                                       field["table16"].shape[0])
    out["d_scene"] = d_scene
    if not diagnostics:
        return out
    # ---- diagnostics only (tests/test_ref_parity.py): emulations of the reference's fp16 arithmetic ------------------
    # the same scatter with the reference's per-product fp16 rounding (Hash3DAnchored.cu:145-151) emulated
    out["grad_feat_pool_half_products"] = O.hash_bwd(field["prim"], field["bias"], field["V"], field["local_size"], scales,
                                                     np.ascontiguousarray(q_pts), q_vol, 1, d_feat16.astype(np.float32),
                                                     1.0 / LOSS_SCALE, field["table16"].shape[0], half_products=True)
    out["grad_feat_pool_half_accum"] = O.hash_bwd(field["prim"], field["bias"], field["V"], field["local_size"], scales,
                                                  np.ascontiguousarray(q_pts), q_vol, 1, d_feat16.astype(np.float32),
                                                  1.0 / LOSS_SCALE, field["table16"].shape[0], half_products=2)
    out["d_scene"] = d_scene
    # --- tiny-cuda-nn style emulation: fp16 accumulators in the field MLP's input gradient (wmma half fragments),
    # then fp16 products + fp16 accumulation in the scatter.  Statistical stand-in for the reference's own noise.
    dout16 = f16(d_scene * LOSS_SCALE)
    din_half = mlp_bwd_half_accum(dout16, np.asarray(f_hid).reshape(-1, 64), fp16)
    out["grad_feat_pool_tcnn_emulation"] = O.hash_bwd(field["prim"], field["bias"], field["V"], field["local_size"], scales,
                                                      np.ascontiguousarray(q_pts), q_vol, 1, din_half.astype(np.float32),
                                                      1.0 / LOSS_SCALE, field["table16"].shape[0], half_products=2)
    a_out, a_in = np.abs(dout16.astype(np.float32)), np.abs(d_feat16.astype(np.float32))
    out["grad_magnitudes"] = dict(dout16_median=float(np.median(a_out[a_out > 0])) if (a_out > 0).any() else 0.0,
                                  dout16_frac_zero=float((a_out == 0).mean()), dout16_frac_subnormal=float((a_out < 6.1e-5).mean()),
                                  din16_median=float(np.median(a_in[a_in > 0])) if (a_in > 0).any() else 0.0,
                                  din16_frac_zero=float((a_in == 0).mean()), din16_frac_subnormal=float((a_in < 6.1e-5).mean()))
    return out


def mlp_bwd_half_accum(dout16, hidden16, params16):
    """Field MLP (32 -> 64 -> 16, no bias) input gradient with an fp16 accumulator rounded after every 16-wide
    k-step, as tiny-cuda-nn's wmma<half accumulator> fragments do (fully_fused_mlp.cu:150-259)."""
    W0 = params16[:64 * 32].reshape(64, 32).astype(np.float32)
    Wo = params16[64 * 32:64 * 32 + 16 * 64].reshape(16, 64).astype(np.float32)
    dh = f16(dout16.astype(np.float32) @ Wo)                     # K = 16: one k-step
    dh = np.where(hidden16 > 0, dh, np.float16(0))
    acc = np.zeros((dout16.shape[0], 32), np.float16)
    for c in range(4):                                           # K = 64: four k-steps
        acc = f16(acc.astype(np.float32) + dh[:, 16 * c:16 * c + 16].astype(np.float32) @ W0[16 * c:16 * c + 16])
    return acc
