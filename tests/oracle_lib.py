"""ctypes binding of oracle/libf2oracle.so (the CPU restatement) for tests, smoke() and bench.py's
cpu_baseline leg.  Test infrastructure: never imported by the f2nerf_b200 package."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "oracle", "libf2oracle.so")


def build():
    """The oracle library build() made; (re)compiled when missing or older than its source — into a temporary directory
    when the tree is read-only."""
    src = os.path.join(ROOT, "oracle", "f2_oracle.c")
    if os.path.exists(SO) and os.path.getmtime(SO) >= os.path.getmtime(src):
        return SO
    out = SO if os.access(os.path.dirname(SO), os.W_OK) else os.path.join(tempfile.mkdtemp(prefix="f2b_oracle_"), "libf2oracle.so")
    subprocess.check_call(["gcc", "-O2", "-march=x86-64-v3", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
                           "-shared", "-fPIC", src, "-o", out, "-lm"])
    return out


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
    return _lib


def _p(a):
    if a is None:
        return None
    assert isinstance(a, np.ndarray) and a.flags["C_CONTIGUOUS"], "oracle args must be C-contiguous numpy arrays"
    return a.ctypes.data_as(ctypes.c_void_p)


F = ctypes.c_float
I = ctypes.c_int


def c(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


def sampler(tree_nodes, trans, rays_o, rays_d, noise, near, far, sample_l, scale_by_dis, max_hits):
    """-> dict(pts, dirs, dt, t, anchors, bounds, first_oct_dis, n_hits)"""
    L = lib()
    R = rays_o.shape[0]
    tree_nodes, trans = c(tree_nodes, np.uint8), c(trans, np.uint8)
    rays_o, rays_d, noise = c(rays_o, np.float32), c(rays_d, np.float32), c(noise, np.float32)
    bounds = np.zeros((R, 2), np.int32)
    totals = np.zeros(2, np.int32)
    args = [_p(tree_nodes), _p(trans), _p(rays_o), _p(rays_d), _p(noise), I(R), F(near), F(far), F(sample_l),
            I(int(scale_by_dis)), I(max_hits)]
    L.orc_sampler(*args, I(0), _p(bounds), _p(totals), None, None, None, None, None, None)
    P = int(totals[0])
    out = dict(pts=np.zeros((P, 3), np.float32), dirs=np.zeros((P, 3), np.float32), dt=np.zeros(P, np.float32),
               t=np.zeros(P, np.float32), anchors=np.zeros((P, 3), np.int32), bounds=bounds,
               first_oct_dis=np.zeros((R, 1), np.float32), n_hits=int(totals[1]))
    L.orc_sampler(*args, I(1), _p(bounds), _p(totals), _p(out["pts"]), _p(out["dirs"]), _p(out["dt"]), _p(out["t"]),
                  _p(out["anchors"]), _p(out["first_oct_dis"]))
    return out


SAMPLER_COVER = ("guard", "guard_zero", "guard_plane", "guard_decides", "empty_eq", "near_past", "step0", "hop", "hop_inf",
                 "hop_nan", "hop_sat", "stack_stop", "near_entry")


def sampler_cover(tree_nodes, trans, rays_o, rays_d, noise, near, far, sample_l, scale_by_dis, max_hits):
    """How often the march of this batch takes each branch of SAMPLER_COVER (orc_sampler_cover in oracle/f2_oracle.c)
    -> dict name -> count."""
    R = rays_o.shape[0]
    bounds, totals = np.zeros((R, 2), np.int32), np.zeros(2, np.int32)
    cov = np.zeros(len(SAMPLER_COVER), np.int64)
    lib().orc_sampler_cover(_p(c(tree_nodes, np.uint8)), _p(c(trans, np.uint8)), _p(c(rays_o, np.float32)),
                            _p(c(rays_d, np.float32)), _p(c(noise, np.float32)), I(R), F(near), F(far), F(sample_l),
                            I(int(scale_by_dis)), I(max_hits), _p(bounds), _p(totals), _p(cov))
    return dict(zip(SAMPLER_COVER, cov.tolist()))


def edge_samples(edge_pool, trans, edge_idx, coord):
    n = edge_idx.shape[0]
    out_pts, out_idx = np.zeros((n, 2, 3), np.float32), np.zeros((n, 2), np.int32)
    lib().orc_edge_samples(_p(c(edge_pool, np.uint8)), _p(c(trans, np.uint8)), _p(c(edge_idx, np.int32)),
                           _p(c(coord, np.float32)), I(n), _p(out_pts), _p(out_idx))
    return out_pts, out_idx


def mark_visit(bounds, oct_idx, stride, w, a, n_nodes, visit_cnt):
    vw, va, mk = np.full(n_nodes, -1, np.int32), np.full(n_nodes, -1, np.int32), np.zeros(n_nodes, np.int32)
    lib().orc_mark_visit(_p(c(bounds, np.int32)), I(bounds.shape[0]), _p(c(oct_idx, np.int32)), I(stride),
                         _p(c(w, np.float32)), _p(c(a, np.float32)), _p(vw), _p(va), _p(mk), _p(visit_cnt))
    return vw, va, mk


def update_stats(vw, va, mk, sw, sa, tree_nodes):
    lib().orc_update_stats(_p(vw), _p(va), _p(mk), _p(sw), _p(sa), _p(tree_nodes), I(vw.shape[0]))


def level_scales():
    s = np.zeros(16, np.float32)
    lib().orc_level_scales(_p(s))
    return s


def hash_fwd(table_h, prim, bias, n_volumes, local_size, scales, pts, vol, vol_stride=1):
    n = pts.shape[0]
    out = np.zeros((n, 32), np.uint16)
    lib().orc_hash_fwd(_p(c(table_h.view(np.uint16), np.uint16)), _p(c(prim, np.int32)), _p(c(bias, np.float32)),
                       I(n_volumes), I(local_size), _p(c(scales, np.float32)), _p(c(pts, np.float32)),
                       _p(c(vol, np.int32)), I(vol_stride), I(n), _p(out))
    return out.view(np.float16)


def hash_bwd(prim, bias, n_volumes, local_size, scales, pts, vol, vol_stride, grad_feat, grad_mul, pool_size, half_products=False):
    g = np.zeros(pool_size * 2, np.float64)
    lib().orc_hash_bwd(_p(c(prim, np.int32)), _p(c(bias, np.float32)), I(n_volumes), I(local_size),
                       _p(c(scales, np.float32)), _p(c(pts, np.float32)), _p(c(vol, np.int32)), I(vol_stride),
                       I(pts.shape[0]), _p(c(grad_feat, np.float32)), F(grad_mul), I(int(half_products)), _p(g))   # half_products: 0 exact, 1 fp16 products, 2 fp16 products + fp16 accumulation
    return g.reshape(pool_size, 2)


def mlp_fwd(x_h, params_h, nh, save_hidden=False):
    n = x_h.shape[0]
    out = np.zeros((n, 16), np.uint16)
    hid = np.zeros((nh + 1, n, 64), np.uint16) if save_hidden else None
    lib().orc_mlp_fwd(_p(c(x_h.view(np.uint16), np.uint16)), _p(c(params_h.view(np.uint16), np.uint16)), I(nh), I(n),
                      _p(out), _p(hid))
    return out.view(np.float16), (hid.view(np.float16) if hid is not None else None)


def mlp_bwd(dout_h, x_h, hidden_h, params_h, nh, need_din=True):
    n = x_h.shape[0]
    din = np.zeros((n, 32), np.uint16) if need_din else None
    dparams = np.zeros(params_h.size, np.float64)
    lib().orc_mlp_bwd(_p(c(dout_h.view(np.uint16), np.uint16)), _p(c(x_h.view(np.uint16), np.uint16)),
                      _p(c(hidden_h.view(np.uint16), np.uint16)), _p(c(params_h.view(np.uint16), np.uint16)), I(nh), I(n),
                      _p(din), _p(dparams))
    return (din.view(np.float16) if din is not None else None), dparams


def mlp_init(d_in, nh, seed=19970826):
    n = 64 * d_in + nh * 64 * 64 + 16 * 64
    p = np.zeros(n, np.float32)
    lib().orc_mlp_init(ctypes.c_uint64(seed), I(d_in), I(nh), _p(p))
    return p


def sh4(dirs):
    out = np.zeros((dirs.shape[0], 16), np.float32)
    lib().orc_sh4(_p(c(dirs, np.float32)), I(dirs.shape[0]), _p(out))
    return out


def shader_prep(scene_feat, dirs, app_emb=None, pt_emb_idx=None):
    n = scene_feat.shape[0]
    out = np.zeros((n, 32), np.uint16)
    lib().orc_shader_prep(_p(c(scene_feat, np.float32)), _p(c(dirs, np.float32)),
                          _p(c(app_emb, np.float32)) if app_emb is not None else None,
                          _p(c(pt_emb_idx, np.int32)) if pt_emb_idx is not None else None, I(n), _p(out))
    return out.view(np.float16)


def shader_act(raw_h):
    n = raw_h.shape[0]
    rgb = np.zeros((n, 3), np.float32)
    lib().orc_shader_act(_p(c(raw_h.view(np.uint16), np.uint16)), I(n), _p(rgb))
    return rgb


def early_stop(logit, stride, dt, bounds):
    P, R = dt.shape[0], bounds.shape[0]
    w, a, keep = np.zeros(P, np.float32), np.zeros(P, np.float32), np.zeros(P, np.uint8)
    nb, tot = np.zeros((R, 2), np.int32), np.zeros(1, np.int32)
    lib().orc_early_stop(_p(c(logit, np.float32)), I(stride), _p(c(dt, np.float32)), _p(c(bounds, np.int32)), I(R),
                         _p(w), _p(a), _p(keep), _p(nb), _p(tot))
    return w, a, keep, nb, int(tot[0])


def filter_bounds(keep, bounds):
    R = bounds.shape[0]
    nb, tot = np.zeros((R, 2), np.int32), np.zeros(1, np.int32)
    lib().orc_filter_bounds(_p(c(keep, np.uint8)), _p(c(bounds, np.int32)), I(R), _p(nb), _p(tot))
    return nb, int(tot[0])


def composite_fwd(logit, stride, rgb, dt, t, bounds, bg):
    P, R = dt.shape[0], bounds.shape[0]
    colors, disp, depth, w = np.zeros((R, 3), np.float32), np.zeros(R, np.float32), np.zeros(R, np.float32), np.zeros(P, np.float32)
    lib().orc_composite_fwd(_p(c(logit, np.float32)), I(stride), _p(c(rgb, np.float32)), _p(c(dt, np.float32)),
                            _p(c(t, np.float32)), _p(c(bounds, np.int32)), _p(c(bg, np.float32)), I(R), _p(colors),
                            _p(disp), _p(depth), _p(w))
    return colors, disp, depth, w


def composite_bwd(logit, stride, rgb, dt, t, bounds, bg, d_colors, d_disp, d_depth, d_weights, gs_progress):
    P, R = dt.shape[0], bounds.shape[0]
    d_logit, d_rgb = np.zeros(P, np.float64), np.zeros((P, 3), np.float64)
    opt = lambda a: _p(c(a, np.float32)) if a is not None else None
    lib().orc_composite_bwd(_p(c(logit, np.float32)), I(stride), _p(c(rgb, np.float32)), _p(c(dt, np.float32)),
                            _p(c(t, np.float32)), _p(c(bounds, np.int32)), _p(c(bg, np.float32)), I(R),
                            _p(c(d_colors, np.float32)), opt(d_disp), opt(d_depth), opt(d_weights), F(gs_progress),
                            _p(d_logit), _p(d_rgb))
    return d_logit, d_rgb


def flex_sum(val, bounds):
    vec = 1 if val.ndim == 1 else val.shape[1]
    out = np.zeros((bounds.shape[0],) if val.ndim == 1 else (bounds.shape[0], vec), np.float32)
    lib().orc_flex_sum(_p(c(val, np.float32)), I(vec), _p(c(bounds, np.int32)), I(bounds.shape[0]), _p(out))
    return out


def flex_accumulate(val, bounds, include_this):
    out = np.zeros_like(val, dtype=np.float32)
    lib().orc_flex_accumulate(_p(c(val, np.float32)), _p(c(bounds, np.int32)), I(bounds.shape[0]), I(int(include_this)), _p(out))
    return out


def weight_var(w, bounds, dl_dvars=None):
    R = bounds.shape[0]
    out = np.zeros(R, np.float32)
    dw = np.zeros_like(w, dtype=np.float32) if dl_dvars is not None else None
    lib().orc_weight_var(_p(c(w, np.float32)), _p(c(bounds, np.int32)), I(R),
                         _p(c(dl_dvars, np.float32)) if dl_dvars is not None else None, _p(out), _p(dw))
    return out, dw


def img2world_rays(poses, intri, dist_params, cam_indices, ij):
    n = cam_indices.shape[0]
    rays_o, rays_d = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.float32)
    lib().orc_img2world_rays(_p(c(poses, np.float32)), _p(c(intri, np.float32)), _p(c(dist_params, np.float32)),
                             _p(c(cam_indices, np.int32)), _p(c(ij, np.int32)), I(n), _p(rays_o), _p(rays_d))
    return rays_o, rays_d


def octree_proc(nodes, wstat, astat, visit, subdivide, brute_force=False):
    """-> (nodes_out bytes [n_out*64], wstat_out, astat_out)"""
    n = nodes.size // 64
    out = np.zeros(9 * n * 64, np.uint8)
    w, a = np.zeros(9 * n, np.int32), np.zeros(9 * n, np.int32)
    lib().orc_octree_proc.restype = ctypes.c_int
    m = lib().orc_octree_proc(_p(c(nodes, np.uint8)), _p(c(wstat, np.int32)), _p(c(astat, np.int32)), _p(c(visit, np.int32)),
                              I(n), I(int(subdivide)), I(int(brute_force)), _p(out), _p(w), _p(a))
    return out[:m * 64].copy(), w[:m].copy(), a[:m].copy()


def num_threads():
    return int(lib().orc_num_threads())


def mark_invisible(nodes, intri, w2c, bound):
    """PersOctree::MarkInvisibleNodes restated (oracle/f2_oracle.c: orc_mark_invisible) -> nodes bytes with trans_idx = -1
    on every node no camera sees."""
    out = c(nodes, np.uint8).copy()
    intri, w2c, bound = c(intri, np.float32), c(w2c, np.float32), c(bound, np.float32)
    lib().orc_mark_invisible(_p(out), I(out.size // 64), _p(intri), _p(w2c), _p(bound), I(bound.size // 2))
    return out
