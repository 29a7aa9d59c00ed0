"""CUDA path (through the C ABI) against the CPU oracle on identical seeded inputs.

Bars: bit-exact for every integer / index output and for fp32 stages that contain no transcendental
(sampler, edge samples, hash encode with the device's own level scales, compaction, octree votes,
FlexOps); 1e-4 relative (BASELINE.json north_star) for fp32 stages downstream of exp(); fp16-storage
stages (MLP) within 2 fp16 ulp of the fp32-accumulate oracle on the same fp16 operands.
"""
import numpy as np
import pytest
import torch

from conftest import make_rays

pytestmark = pytest.mark.gpu

DEV = "cuda"


def T(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.to(DEV).contiguous()


def N(t):
    return t.detach().cpu().numpy()


def assert_close(a, b, rtol=1e-4, atol_frac=1e-4, name=""):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (name, a.shape, b.shape)
    scale = max(np.abs(b).max(), 1e-30) if b.size else 1.0
    err = np.abs(a - b)
    tol = rtol * np.abs(b) + atol_frac * scale
    assert (err <= tol).all(), f"{name}: max err {err.max():.3e} at {np.unravel_index(err.argmax(), err.shape)} " \
                               f"(ref {b.flat[err.argmax()]:.6e}, scale {scale:.3e})"


def half_ulp(b):
    """fp16 ulp at max(|b|, 2^-14)."""
    mag = np.maximum(np.abs(np.asarray(b, np.float32)), 2.0 ** -14)
    return 2.0 ** (np.floor(np.log2(mag)) - 10)


def half_ulps(a, b):
    """max |a-b| in units of fp16 ulp at max(|b|, 2^-14)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return float((np.abs(a - b) / half_ulp(b)).max()) if a.size else 0.0


# ----------------------------------------------------------------------------------- sampler ---
def run_sampler_gpu(scene, o, dn, noise, near, sample_l, scale_by_dis, max_hits=1024):
    from f2nerf_b200 import ops
    args = (T(scene["nodes"]), T(scene["trans"]), T(o), T(dn), T(noise), near, 1e8, sample_l, scale_by_dis, max_hits)
    bounds, totals = ops.sampler_count(*args)
    n_pts, n_hits = (int(v) for v in totals.tolist())
    pts, dirs, dt, t, anchors, first = ops.sampler_fill(*args, bounds, n_pts)
    return dict(pts=N(pts), dirs=N(dirs), dt=N(dt), t=N(t), anchors=N(anchors), bounds=N(bounds),
                first_oct_dis=N(first), n_hits=n_hits)


@pytest.mark.parametrize("n_rays,scale_by_dis,noise_kind,sample_l", [
    (256, False, "ones", 1 / 256), (1000, True, "rand", 1 / 256), (64, True, "rand", 1 / 32), (4096, False, "rand", 1 / 256)])
def test_sampler_bit_exact(scene, oracle, n_rays, scale_by_dis, noise_kind, sample_l):
    o, d, dn, _ = make_rays(scene, n_rays, seed=n_rays)
    rng = np.random.default_rng(5)
    noise = np.ones(1024 + n_rays + 10, np.float32) if noise_kind == "ones" else \
        (rng.random(1024 + n_rays + 10, dtype=np.float32) - .5 + 1.).astype(np.float32)
    ref = oracle.sampler(scene["nodes"], scene["trans"], o, dn, noise, 0.05, 1e8, sample_l, scale_by_dis, 1024)
    got = run_sampler_gpu(scene, o, dn, noise, 0.05, sample_l, scale_by_dis)
    assert got["n_hits"] == ref["n_hits"]
    np.testing.assert_array_equal(got["bounds"], ref["bounds"])
    for k in ("first_oct_dis", "t", "dt", "dirs", "pts"):
        np.testing.assert_array_equal(got[k].view(np.uint32), ref[k].view(np.uint32), err_msg=k)   # bit-exact fp32
    np.testing.assert_array_equal(got["anchors"], ref["anchors"])


def test_sampler_one_pass_equals_two_pass(scene, oracle):
    """f2b_sampler_march + f2b_sampler_gather (one march into scratch slots) == count + fill, bit for bit."""
    from f2nerf_b200 import ops
    n = 777
    o, d, dn, _ = make_rays(scene, n, seed=3)
    noise = (np.random.default_rng(8).random(1024 + n + 10, dtype=np.float32) + .5).astype(np.float32)
    two = run_sampler_gpu(scene, o, dn, noise, 0.05, 1 / 256, True)
    args = (T(scene["nodes"]), T(scene["trans"]), T(o), T(dn), T(noise), 0.05, 1e8, 1 / 256, True, 1024)
    cap = n * 1024
    f = lambda *s: torch.empty(s, dtype=torch.float32, device=DEV)
    scratch = (f(cap, 3), f(cap), f(cap), torch.empty((cap, 2), dtype=torch.int32, device=DEV))
    bounds, totals, first = ops.sampler_march(*args, scratch, count_all_hits=True)
    assert totals.tolist() == [two["pts"].shape[0], two["n_hits"]]
    pts, dirs, dt, t, anchors = ops.sampler_gather(T(dn), bounds, int(totals[0]), scratch)
    np.testing.assert_array_equal(N(bounds), two["bounds"])
    np.testing.assert_array_equal(N(anchors), two["anchors"])
    for k, v in (("pts", pts), ("dirs", dirs), ("dt", dt), ("t", t), ("first_oct_dis", first)):
        np.testing.assert_array_equal(N(v).view(np.uint32), two[k].view(np.uint32), err_msg=k)


def test_sampler_edge_cases(scene, oracle):
    from f2nerf_b200 import ops
    # rays that miss everything (start far outside, pointing away) and an empty batch
    o = np.array([[600., 600., 600.], [0., 0., 0.2]], np.float32)
    dn = np.array([[0.57735026, 0.57735026, 0.57735026], [0., 0., 1.]], np.float32)
    noise = np.ones(1024 + 2 + 10, np.float32)
    ref = oracle.sampler(scene["nodes"], scene["trans"], o, dn, noise, 0.05, 1e8, 1 / 256, False, 1024)
    got = run_sampler_gpu(scene, o, dn, noise, 0.05, 1 / 256, False)
    np.testing.assert_array_equal(got["bounds"], ref["bounds"])
    assert got["bounds"][0, 0] == got["bounds"][0, 1]                 # ray 0 has no samples
    assert got["first_oct_dis"][0, 0] == np.float32(1e9)
    np.testing.assert_array_equal(got["pts"].view(np.uint32), ref["pts"].view(np.uint32))
    # small hit cap (max_oct_intersect_per_ray) is honoured identically
    ref2 = oracle.sampler(scene["nodes"], scene["trans"], o, dn, noise, 0.05, 1e8, 1 / 256, False, 3)
    got2 = run_sampler_gpu(scene, o, dn, noise, 0.05, 1 / 256, False, max_hits=3)
    np.testing.assert_array_equal(got2["bounds"], ref2["bounds"])
    assert got2["n_hits"] == ref2["n_hits"]
    z = torch.zeros((0, 3), device=DEV)
    b, tot = ops.sampler_count(T(scene["nodes"]), T(scene["trans"]), z, z, T(noise), 0.05, 1e8, 1 / 256, False, 1024)
    assert tot.tolist() == [0, 0] and b.shape == (0, 2)


def test_edge_samples_bit_exact(scene, oracle):
    from f2nerf_b200 import ops
    rng = np.random.default_rng(3)
    n_edges = scene["edges"].size // 64
    idx = rng.integers(0, n_edges, 2048).astype(np.int32)
    coord = (rng.random((2048, 2), dtype=np.float32) * 2 - 1).astype(np.float32)
    rp, ri = oracle.edge_samples(scene["edges"], scene["trans"], idx, coord)
    gp, gi = ops.edge_samples(T(scene["edges"]), T(scene["trans"]), T(idx), T(coord))
    np.testing.assert_array_equal(N(gi), ri)
    np.testing.assert_array_equal(N(gp).view(np.uint32), rp.view(np.uint32))


# -------------------------------------------------------------------------------- hash field ---
def sample_points(scene, oracle, n_rays=128):
    o, d, dn, _ = make_rays(scene, n_rays, seed=11)
    noise = np.ones(1024 + n_rays + 10, np.float32)
    return oracle.sampler(scene["nodes"], scene["trans"], o, dn, noise, 0.05, 1e8, 1 / 256, False, 1024)


def test_hash_fwd_bit_exact(scene, oracle, hash_params):
    from f2nerf_b200 import ops
    s = sample_points(scene, oracle)
    hp = hash_params
    scales = ops.hash_level_scales().numpy()
    np.testing.assert_allclose(scales, oracle.level_scales(), rtol=6e-7)        # MUFU.EX2 vs libm: <= 2 ulp
    ref = oracle.hash_fwd(hp["table"], hp["prim"], hp["bias"], hp["V"], hp["local_size"], scales, s["pts"], s["anchors"], 3)
    got = ops.hash_fwd(T(hp["table"]), T(hp["prim"]), T(hp["bias"]), hp["V"], hp["local_size"], T(s["pts"]),
                       T(s["anchors"]), 3)
    np.testing.assert_array_equal(N(got).view(np.uint16), ref.view(np.uint16))
    # extreme coordinates: negative / huge values exercise the saturating float->u32 conversion
    pts = np.array([[-5000., 3., 7e9], [1e-3, -1e-3, 0.], [123456.7, -98765.4, 4e9]], np.float32)
    vol = np.array([0, 1, hp["V"] - 1], np.int32)
    ref = oracle.hash_fwd(hp["table"], hp["prim"], hp["bias"], hp["V"], hp["local_size"], scales, pts, vol)
    got = ops.hash_fwd(T(hp["table"]), T(hp["prim"]), T(hp["bias"]), hp["V"], hp["local_size"], T(pts), T(vol), 1)
    np.testing.assert_array_equal(N(got).view(np.uint16), ref.view(np.uint16))


def test_hash_bwd_matches_exact_sum(scene, oracle, hash_params):
    from f2nerf_b200 import ops
    s = sample_points(scene, oracle, 32)
    hp = hash_params
    n = s["pts"].shape[0]
    rng = np.random.default_rng(9)
    g = (rng.standard_normal((n, 32)).astype(np.float32) * 1e-3)
    g[::7] = 0.                                                   # zero rows are skipped
    scales = ops.hash_level_scales().numpy()
    ref = oracle.hash_bwd(hp["prim"], hp["bias"], hp["V"], hp["local_size"], scales, s["pts"], s["anchors"], 3, g, 0.5, hp["pool"])
    for as_half in (False, True):
        gt = T(g.astype(np.float16)) if as_half else T(g)
        gref = ref if not as_half else oracle.hash_bwd(hp["prim"], hp["bias"], hp["V"], hp["local_size"], scales, s["pts"],
                                                        s["anchors"], 3, g.astype(np.float16).astype(np.float32), 0.5, hp["pool"])
        table = torch.zeros((hp["pool"], 2), dtype=torch.float32, device=DEV)
        ops.hash_bwd(T(hp["prim"]), T(hp["bias"]), hp["V"], hp["local_size"], T(s["pts"]), T(s["anchors"]), 3, gt, 0.5, table)
        assert_close(N(table), gref, rtol=1e-4, atol_frac=1e-5, name=f"hash_bwd half={as_half}")
        # the quirk: only the first 17/32 of the pool is ever touched
        assert float(table[(17 * hp["local_size"]) // 2 + 1:].abs().max()) == 0.0


# -------------------------------------------------------------------------------------- MLP ----
@pytest.mark.parametrize("nh", [0, 1])
def test_mlp_fwd_bwd(oracle, nh):
    from f2nerf_b200 import ops
    rng = np.random.default_rng(21 + nh)
    n = 1000                                                       # ragged: not a multiple of 128
    x = (rng.standard_normal((n, 32)) * 0.5).astype(np.float16)
    params = (oracle.mlp_init(32, nh) * 2).astype(np.float16)
    ref_out, ref_hid = oracle.mlp_fwd(x, params, nh, save_hidden=True)
    out, hid = ops.mlp_fwd(T(x), T(params), nh, save_hidden=True)
    assert half_ulps(N(hid)[0].astype(np.float32), ref_hid[0].astype(np.float32)) <= 2.0      # first layer: same operands
    if nh:   # second layer sees first-layer outputs that may differ by an ulp: compare at the tensor's scale
        assert_close(N(hid)[1].astype(np.float32), ref_hid[1].astype(np.float32), rtol=4e-3, atol_frac=2e-3, name="hidden 1")
    assert_close(N(out).astype(np.float32), ref_out.astype(np.float32), rtol=2e-3, atol_frac=1e-3, name="mlp out")
    # backward on the ORACLE's saved activations so both sides see identical operands
    dout = (rng.standard_normal((n, 16)) * 0.1).astype(np.float16)
    rdin, rdp = oracle.mlp_bwd(dout, x, ref_hid, params, nh)
    din, dp = ops.mlp_bwd(T(dout), T(x), T(ref_hid), T(params), nh, need_din=True)
    assert_close(N(din).astype(np.float32), rdin.astype(np.float32), rtol=4e-3, atol_frac=2e-3, name="mlp din")
    assert_close(N(dp), rdp, rtol=2e-3, atol_frac=2e-3, name="mlp dparams")


@pytest.mark.parametrize("nh", [0, 1])
def test_mlp_tc_tiles_and_f32_output(oracle, nh):
    """Persistent-tile path of the tensor-core forward: sizes below / across / far beyond one tile per CTA (double-buffered
    cp.async input, coalesced hidden copy-out), tc == the CPU oracle within fp16 noise, fp32 output == widened fp16."""
    from f2nerf_b200 import ops
    rng = np.random.default_rng(77 + nh)
    params_h = (oracle.mlp_init(32, nh) * 2).astype(np.float16)
    params = T(params_h)
    for n in (1, 127, 128, 129, 5000, 148 * 5 * 128 * 2 + 333):
        x_h = (rng.standard_normal((n, 32)) * 0.5).astype(np.float16)
        x = T(x_h)
        out, hid = ops.mlp_fwd(x, params, nh, save_hidden=True)
        ref_out, ref_hid = oracle.mlp_fwd(x_h, params_h, nh, save_hidden=True)
        # fp32 accumulation order differs (tensor core vs serial): fp16 roundings may flip on cancellation-small values
        assert_close(N(hid)[0].astype(np.float32), ref_hid[0].astype(np.float32), rtol=2e-3, atol_frac=1e-3, name=f"hidden n={n}")
        assert_close(N(out).astype(np.float32), ref_out.astype(np.float32), rtol=4e-3, atol_frac=2e-3, name=f"tc vs oracle n={n}")
        out32, out16, hid2 = ops.mlp_fwd_f32(x, params, nh, save_hidden=True, want_f16=True)
        np.testing.assert_array_equal(N(out16).view(np.uint16), N(out).view(np.uint16))
        np.testing.assert_array_equal(N(out32), N(out).astype(np.float32))
        np.testing.assert_array_equal(N(hid2).view(np.uint16), N(hid).view(np.uint16))
        out32b, none16, _ = ops.mlp_fwd_f32(x, params, nh, save_hidden=False)
        assert none16 is None
        np.testing.assert_array_equal(N(out32b), N(out32))
        # backward over the same tiles (double-buffered operand prefetch, in-place activation gradients,
        # weight gradients resident in registers across the CTA's tiles) against the oracle, both on the oracle's activations
        dout_h = (rng.standard_normal((n, 16)) * 0.1).astype(np.float16)
        din, dp = ops.mlp_bwd(T(dout_h), x, T(ref_hid), params, nh, need_din=True)
        rdin, rdp = oracle.mlp_bwd(dout_h, x_h, ref_hid, params_h, nh)
        assert_close(N(din).astype(np.float32), rdin.astype(np.float32), rtol=4e-3, atol_frac=2e-3, name=f"din n={n}")
        assert_close(N(dp), rdp, rtol=3e-3, atol_frac=2e-3, name=f"dparams n={n}")


@pytest.mark.parametrize("nh", [0, 1])
def test_mlp_bwd_recompute_equals_saved(oracle, nh):
    """f2b_mlp_bwd2 with hidden0 == NULL rebuilds the hidden activations on the tensor pipe from the input rows (no 128 / 256 B
    per sample saved by the forward): dL/dinput must equal the saved-activation kernel's BIT FOR BIT (same MMAs on the same
    operands), the weight gradients up to the order of the fp32 atomics that flush them."""
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    rng = np.random.default_rng(310 + nh)
    params = T((oracle.mlp_init(32, nh) * 2).astype(np.float16))
    for n in (1, 127, 128, 129, 5000, 148 * 4 * 128 * 2 + 77):
        x = T((rng.standard_normal((n, 32)) * 0.5).astype(np.float16))
        dout = T((rng.standard_normal((n, 16)) * 0.1).astype(np.float16))
        _, hid = ops.mlp_fwd(x, params, nh, save_hidden=True)
        outs = []
        for h0, h1 in ((hid[0], hid[1] if nh else None), (None, None)):
            din = torch.empty((n, 32), dtype=torch.float16, device="cuda")
            dp = torch.zeros(params.numel(), dtype=torch.float32, device="cuda")
            call("f2b_mlp_bwd2", dout, x, h0, h1, params, nh, n, din, dp, stream())
            outs.append((N(din), N(dp)))
        np.testing.assert_array_equal(outs[0][0].view(np.uint16), outs[1][0].view(np.uint16))
        assert_close(outs[1][1], outs[0][1], rtol=1e-5, atol_frac=1e-6, name=f"dparams recompute n={n}")


def test_fused_epilogues_match_operator_sequence(oracle):
    """f2b_field_shade_fwd == mlp_fwd_f32 -> shading-input assembly and f2b_shader_mlp_rgb_fwd == mlp_fwd -> shader_act, bit for
    bit (ragged sizes, with and without appearance embedding, across several tiles per CTA).  The assembly is restated in numpy
    with shade_row's roundings, fp16([1, out[1:16]] + emb) by one fp32 add and RNE, next to fp16(sh_encode(dirs)): sh_encode
    runs the same sh4 device function as the epilogue."""
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    rng = np.random.default_rng(55)
    fp = T((oracle.mlp_init(32, 0) * 3).astype(np.float16))
    sp = T((oracle.mlp_init(32, 1) * 2).astype(np.float16))
    emb = T((rng.standard_normal((11, 16)) * .1).astype(np.float32))
    for n in (1, 129, 4000, 148 * 5 * 128 + 77):
        feat = T((rng.standard_normal((n, 32)) * 0.5).astype(np.float16))
        d = rng.standard_normal((n, 3)).astype(np.float32); d /= np.linalg.norm(d, axis=-1, keepdims=True)
        dirs, idx = T(d), T(rng.integers(0, 11, n).astype(np.int32))
        out32, _, hid = ops.mlp_fwd_f32(feat, fp, 0, save_hidden=True)
        sh = N(ops.sh_encode(dirs)).astype(np.float16)
        for use_emb in (False, True):
            head = N(out32)
            head[:, 0] = 1.0
            if use_emb:
                head = head + N(emb)[N(idx)]
            want_in = T(np.concatenate([head.astype(np.float16), sh], 1))
            logit = torch.empty((n,), device=DEV); mlp_in = torch.empty((n, 32), dtype=torch.float16, device=DEV)
            hid2 = torch.empty((1, n, 64), dtype=torch.float16, device=DEV)
            call("f2b_field_shade_fwd", feat, fp, dirs, emb if use_emb else None, idx if use_emb else None, n, logit, mlp_in, hid2, stream())
            np.testing.assert_array_equal(N(mlp_in).view(np.uint16), N(want_in).view(np.uint16))
            np.testing.assert_array_equal(N(logit), N(out32)[:, 0])
            np.testing.assert_array_equal(N(hid2).view(np.uint16), N(hid).view(np.uint16))
        raw_w, shid_w = ops.mlp_fwd(want_in, sp, 1, save_hidden=True)
        rgb_w = ops.shader_act(raw_w)
        raw = torch.empty((n, 16), dtype=torch.float16, device=DEV); rgb = torch.empty((n, 3), device=DEV)
        shid = torch.empty((2, n, 64), dtype=torch.float16, device=DEV)
        call("f2b_shader_mlp_rgb_fwd", want_in, sp, n, raw, rgb, shid, stream())
        np.testing.assert_array_equal(N(raw).view(np.uint16), N(raw_w).view(np.uint16))
        np.testing.assert_array_equal(N(rgb), N(rgb_w))
        np.testing.assert_array_equal(N(shid).view(np.uint16), N(shid_w).view(np.uint16))


def test_fused_field_matches_unfused(scene, oracle, hash_params):
    """f2b_field_fwd (encode fused into the tensor-core MLP) == f2b_hash_fwd -> f2b_mlp_fwd, bit for bit."""
    from f2nerf_b200 import ops
    s = sample_points(scene, oracle, 100)
    hp = hash_params
    params = T((oracle.mlp_init(32, 0) * 3).astype(np.float16))
    tab, prim, bias, pts, anc = T(hp["table"]), T(hp["prim"]), T(hp["bias"]), T(s["pts"]), T(s["anchors"])
    feat = ops.hash_fwd(tab, prim, bias, hp["V"], hp["local_size"], pts, anc, 3)
    out16, hid = ops.mlp_fwd(feat, params, 0, save_hidden=True)
    out, f2, h2 = ops.field_fwd(tab, prim, bias, hp["V"], hp["local_size"], params, pts, anc, 3, save=True)
    np.testing.assert_array_equal(N(f2).view(np.uint16), N(feat).view(np.uint16))
    np.testing.assert_array_equal(N(h2).view(np.uint16), N(hid).view(np.uint16))
    np.testing.assert_array_equal(N(out), N(out16).astype(np.float32))
    logit, _, _ = ops.field_fwd(tab, prim, bias, hp["V"], hp["local_size"], params, pts, anc, 3, logit_only=True)
    np.testing.assert_array_equal(N(logit), N(out)[:, 0])


def test_mlp_init_matches_tcnn_stream(oracle):
    from f2nerf_b200.field import tcnn_xavier_params
    for nh_layers in (1, 2):
        np.testing.assert_array_equal(tcnn_xavier_params(32, nh_layers).numpy(), oracle.mlp_init(32, nh_layers - 1))


# ----------------------------------------------------------------------------------- shader ----
def test_shader_prep_and_act(oracle):
    """The shading input f2b_field_shade_fwd assembles in its epilogue against the oracle's shader_prep of the same call's fp32
    field output; SH encode, colour activation and its backward against the oracle / autograd."""
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    rng = np.random.default_rng(31)
    n = 777
    feat = T((rng.standard_normal((n, 32)) * 0.5).astype(np.float16))
    fp = T((oracle.mlp_init(32, 0) * 3).astype(np.float16))
    out32 = N(ops.mlp_fwd_f32(feat, fp, 0)[0])
    d = rng.standard_normal((n, 3)).astype(np.float32); d /= np.linalg.norm(d, axis=-1, keepdims=True)
    emb = (rng.standard_normal((9, 16)) * .1).astype(np.float32)
    idx = rng.integers(0, 9, n).astype(np.int32)
    for use in (False, True):
        ref = oracle.shader_prep(out32, d, emb if use else None, idx if use else None)
        logit, got = torch.empty((n,), device=DEV), torch.empty((n, 32), dtype=torch.float16, device=DEV)
        call("f2b_field_shade_fwd", feat, fp, T(d), T(emb) if use else None, T(idx) if use else None, n, logit, got, None, stream())
        assert half_ulps(N(got).astype(np.float32), ref.astype(np.float32)) <= 1.0
    assert_close(N(ops.sh_encode(T(d), 4)), oracle.sh4(d), rtol=1e-5, atol_frac=1e-6, name="sh4")
    raw = (rng.standard_normal((n, 16)) * 3).astype(np.float16)
    assert_close(N(ops.shader_act(T(raw))), oracle.shader_act(raw), rtol=1e-5, atol_frac=1e-6, name="rgb")
    # activation backward against autograd of the same formula
    r = torch.from_numpy(raw[:, :3].astype(np.float32)).requires_grad_(True)
    rgb = (1. + 2e-3) / (1. + torch.exp(-r)) - 1e-3
    g = torch.from_numpy(rng.standard_normal((n, 3)).astype(np.float32))
    rgb.backward(g)
    got = N(ops.shader_act_bwd(T(raw), T(g.numpy()), 128.0)).astype(np.float32)
    assert_close(got[:, :3] / 128.0, r.grad.numpy(), rtol=2e-3, atol_frac=1e-3, name="act bwd")
    assert (got[:, 3:] == 0).all()


def test_rng_burn_matches_torch_rand():
    """rng.burn_rand must leave the CUDA generator exactly where a real torch.rand / rand_like leaves it."""
    from f2nerf_b200.rng import burn_mlp_output, burn_rand
    for numel, dt in ((1, torch.float16), (255, torch.float32), (1024 * 16, torch.float16), (4_190_123 * 3, torch.float32),
                      (1184 * 256 * 4 + 1, torch.float16), (33_554_432 + 16, torch.float16)):
        torch.manual_seed(5)
        torch.rand(numel, dtype=dt, device=DEV)
        a = torch.rand(8, device=DEV)
        torch.manual_seed(5)
        burn_rand(numel, DEV)
        b = torch.rand(8, device=DEV)
        assert torch.equal(a, b), numel
    torch.manual_seed(6)
    torch.rand((128 * 3, 16), dtype=torch.float16, device=DEV)
    a = torch.randint(0, 1000, (16,), device=DEV)
    torch.manual_seed(6)
    burn_mlp_output(257, DEV)                                     # 257 rows -> padded to 384
    assert torch.equal(a, torch.randint(0, 1000, (16,), device=DEV))


@pytest.mark.parametrize("use_emb", [False, True])
def test_shader_prep_bwd_f16(use_emb):
    """f2b_shader_prep_bwd_f16 bit for bit against numpy's roundings, fp16(fp32(g) * inv_s * f_scale) with column 0 =
    fp16(d_logit * f_scale), for two loss-scale pairs and rays that include an empty and a one-sample ray; rows past the
    rays' samples (edge points) untouched; the appearance-embedding gradient against a float64 sum."""
    from f2nerf_b200 import ops
    rng = np.random.default_rng(34)
    n_emb = 17
    lens = rng.integers(0, 150, 200).astype(np.int32); lens[0] = 0; lens[7] = 1
    bounds = np.stack([np.cumsum(lens) - lens, np.cumsum(lens)], -1).astype(np.int32)
    n = int(lens.sum())
    g = (rng.standard_normal((n, 32)) * 3).astype(np.float16)
    d_logit = (rng.standard_normal(n) * 1e-3).astype(np.float32)
    ray_idx = rng.integers(0, n_emb, 200).astype(np.int32)
    for s_scale, f_scale in ((128.0, 128.0), (64.0, 128.0)):
        gs = g[:, :16].astype(np.float32) * np.float32(1 / s_scale)
        want = gs * np.float32(f_scale)
        want[:, 0] = d_logit * np.float32(f_scale)
        out = torch.full((n + 5, 16), 9.0, dtype=torch.float16, device=DEV)
        d_app = torch.zeros((n_emb, 16), device=DEV) if use_emb else None
        ops.shader_prep_bwd_f16(T(g), T(d_logit), T(bounds), T(ray_idx) if use_emb else None, 1 / s_scale, f_scale, out, d_app)
        np.testing.assert_array_equal(N(out)[:n].view(np.uint16), want.astype(np.float16).view(np.uint16))
        assert (N(out)[n:] == 9.0).all()                           # rows past the rays' samples (edge points) untouched
        if use_emb:
            ref = np.zeros((n_emb, 16), np.float64)
            np.add.at(ref, np.repeat(ray_idx, lens), gs.astype(np.float64))
            assert_close(N(d_app), ref, rtol=1e-4, atol_frac=1e-5, name="d_app_emb")


# -------------------------------------------------------------------------------- composite ----
def composite_inputs(scene, oracle, n_rays=300, seed=41):
    s = sample_points(scene, oracle, n_rays)
    rng = np.random.default_rng(seed)
    P = s["pts"].shape[0]
    # density logits that make some rays saturate (early stop) and others stay transparent
    ray_of = np.repeat(np.arange(n_rays), s["bounds"][:, 1] - s["bounds"][:, 0])
    logit = (rng.standard_normal(P) * 2 + (ray_of % 5) * 2.5).astype(np.float32)
    feat = rng.standard_normal((P, 16)).astype(np.float32)
    feat[:, 0] = logit
    rgb = rng.random((P, 3), dtype=np.float32)
    bg = rng.random((n_rays, 3), dtype=np.float32)
    return s, feat, rgb, bg


def test_early_stop_and_compaction(scene, oracle):
    """f2b_early_stop_rays on logits at stride 16, f2b_count_scan of its survivor counts -> the compacted bounds."""
    from f2nerf_b200 import ops
    s, feat, rgb, bg = composite_inputs(scene, oracle)
    rw, ra, rkeep, rnb, rtot = oracle.early_stop(feat, 16, s["dt"], s["bounds"])
    P, R = s["dt"].shape[0], s["bounds"].shape[0]
    w, a = torch.empty(P, device=DEV), torch.empty(P, device=DEV)
    keep, counts = torch.empty(P, dtype=torch.uint8, device=DEV), torch.empty(R, dtype=torch.int32, device=DEV)
    ops.early_stop_rays(T(feat), 16, T(s["dt"]), T(s["bounds"]), w, a, keep, counts)
    nb, tot = ops.count_scan(counts, R)
    assert_close(N(w), rw, rtol=1e-4, atol_frac=1e-6, name="weights")
    assert_close(N(a), ra, rtol=1e-4, atol_frac=1e-6, name="alphas")
    # the keep mask may differ only where trans is within fp32 noise of the 1e-4 threshold
    diff = N(keep) != rkeep
    assert diff.mean() < 1e-4
    assert 0 < rtot < s["pts"].shape[0], "test inputs must exercise early stop"
    # integer outputs are bit-exact GIVEN the mask: bounds, total
    gb, gtot = oracle.filter_bounds(N(keep), s["bounds"])
    np.testing.assert_array_equal(N(nb), gb)
    assert int(tot.item()) == gtot


def test_composite_fwd_bwd(scene, oracle):
    """Forward composite, and f2b_composite_act_bwd: d_logit against the oracle, d_raw against the oracle's d_rgb through the
    colour activation's backward, within d_rgb's bar carried through the activation's slope plus 2 fp16 ulp."""
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    s, feat, rgb, bg = composite_inputs(scene, oracle, n_rays=200, seed=43)
    ref = oracle.composite_fwd(feat, 16, rgb, s["dt"], s["t"], s["bounds"], bg)
    got = ops.composite_fwd(T(feat), 16, T(rgb), T(s["dt"]), T(s["t"]), T(s["bounds"]), T(bg))
    for g, r, name in zip(got, ref, ("colors", "disparity", "depth", "weights")):
        assert_close(N(g), r, rtol=1e-4, atol_frac=1e-6, name=name)
    rng = np.random.default_rng(47)
    R, P = bg.shape[0], rgb.shape[0]
    dc, dd, dz = (rng.standard_normal((R, 3)).astype(np.float32), rng.standard_normal(R).astype(np.float32) * .1,
                  rng.standard_normal(R).astype(np.float32) * .1)
    dw = rng.standard_normal(P).astype(np.float32) * .01
    raw = T((rng.standard_normal((P, 16)) * 2).astype(np.float16))
    rgb_a = ops.shader_act(raw)
    sg = 1.0 / (1.0 + np.exp(-N(raw)[:, :3].astype(np.float32)))       # fp32 sigmoid, like the reference's autograd
    for gs, dz_or_none in ((1.0, dz), (0.25, dz), (0.25, None)):
        rl, rr = oracle.composite_bwd(feat, 16, N(rgb_a), s["dt"], s["t"], s["bounds"], bg, dc, dd, dz_or_none, dw, gs)
        d_scene = torch.zeros((P, 16), device=DEV)
        d_raw = torch.empty((P, 16), dtype=torch.float16, device=DEV)
        call("f2b_composite_act_bwd", T(feat), 16, rgb_a, T(s["dt"]), T(s["t"]), T(s["bounds"]), T(bg), R, T(dc), T(dd),
             None if dz_or_none is None else T(dz_or_none), T(dw), gs, raw, 128.0, d_scene, 16, d_raw, stream())
        name = f"gs={gs} d_depth={'None' if dz_or_none is None else 'given'}"
        assert_close(N(d_scene)[:, 0], rl, rtol=2e-4, atol_frac=2e-5, name=f"d_logit {name}")
        assert float(d_scene[:, 1:].abs().max()) == 0.0
        # d_rgb's bar (1e-4 relative, 1e-5 of the largest |d_rgb|: the kernel's fp32 1 - exp(-tau) cancels at tiny tau, the
        # float64 oracle's does not) through the activation's slope, plus 2 fp16 ulp for the activation backward's rounding
        slope = (1.0 + 2e-3) * sg * (1.0 - sg) * 128.0
        gr, want = N(d_raw).astype(np.float32), rr * slope
        err, tol = np.abs(gr[:, :3] - want), (1e-4 * np.abs(rr) + 1e-5 * np.abs(rr).max()) * slope + 2 * half_ulp(want)
        assert (err <= tol).all(), f"d_raw {name}: max err / tol {(err / tol).max():.3f}"
        assert (gr[:, 3:] == 0).all()


def test_composite_bwd_against_autograd(scene, oracle):
    """The oracle's analytic backward itself, checked against autograd of a plain torch fp64 composite."""
    from f2nerf_b200 import CustomOps
    s, feat, rgb, bg = composite_inputs(scene, oracle, n_rays=8, seed=49)
    b = s["bounds"]
    x = torch.tensor(feat[:, 0], dtype=torch.float64, requires_grad=True)
    c = torch.tensor(rgb, dtype=torch.float64, requires_grad=True)
    dt, t = torch.tensor(s["dt"], dtype=torch.float64), torch.tensor(s["t"], dtype=torch.float64) + 1e-2
    loss = 0
    rng = np.random.default_rng(1)
    dc, dd, dz = rng.standard_normal((8, 3)), rng.standard_normal(8), rng.standard_normal(8)
    for r in range(8):
        sl = slice(b[r, 0], b[r, 1])
        tau = CustomOps.TruncExp.apply(x[sl] - 3) * dt[sl]          # exp forward, exponent clamped to <= 5 backward
        A = torch.cumsum(tau, 0) - tau
        w = torch.exp(-A) * (1 - torch.exp(-tau))
        lt = torch.exp(-tau.sum())
        col = (w[:, None] * c[sl]).sum(0) + lt * torch.tensor(bg[r], dtype=torch.float64)
        disp = (w / t[sl]).sum()
        depth = (w * t[sl]).sum() / (1 - lt + 1e-4)
        loss = loss + (col * torch.tensor(dc[r])).sum() + disp * dd[r] + depth * dz[r]
    loss.backward()
    rl, rr = oracle.composite_bwd(feat, 16, rgb, s["dt"], s["t"], b, bg, dc.astype(np.float32), dd.astype(np.float32),
                                  dz.astype(np.float32), None, 1.0)
    assert_close(rl, x.grad.numpy(), rtol=1e-5, atol_frac=1e-6, name="oracle d_logit vs autograd")
    assert_close(rr, c.grad.numpy(), rtol=1e-5, atol_frac=1e-6, name="oracle d_rgb vs autograd")


def test_flex_ops_bit_exact(scene, oracle):
    from f2nerf_b200 import FlexOps
    s, feat, rgb, bg = composite_inputs(scene, oracle, n_rays=100, seed=51)
    b = s["bounds"]
    v = feat[:, 1].copy()
    np.testing.assert_array_equal(N(FlexOps.Sum(T(v), T(b))).view(np.uint32), oracle.flex_sum(v, b).view(np.uint32))
    np.testing.assert_array_equal(N(FlexOps.Sum(T(rgb), T(b))).view(np.uint32), oracle.flex_sum(rgb, b).view(np.uint32))
    for inc in (False, True):
        np.testing.assert_array_equal(N(FlexOps.AccumulateSum(T(v), T(b), inc)).view(np.uint32),
                                      oracle.flex_accumulate(v, b, inc).view(np.uint32))
    # autograd of the wrappers (reverse scan / broadcast) against a torch fp64 reference
    vt = T(v).requires_grad_(True)
    out = FlexOps.AccumulateSum(vt, T(b), False)
    gsel = torch.linspace(0, 1, out.numel(), device=DEV)
    (out * gsel).sum().backward()
    ref = np.zeros_like(v, dtype=np.float64)
    gn = gsel.cpu().double().numpy()
    for r in range(b.shape[0]):
        sl = slice(b[r, 0], b[r, 1])
        ref[sl] = np.cumsum(gn[sl][::-1])[::-1] - gn[sl]
    assert_close(N(vt.grad), ref, rtol=1e-4, atol_frac=1e-5, name="accumulate bwd")


def test_weight_var(scene, oracle):
    from f2nerf_b200 import CustomOps
    s, feat, rgb, bg = composite_inputs(scene, oracle, n_rays=64, seed=53)
    w = np.abs(feat[:, 2]).astype(np.float32) * 0.01
    g = np.linspace(0.5, 1.5, 64).astype(np.float32)
    rv, rdw = oracle.weight_var(w, s["bounds"], g)
    wt = T(w).requires_grad_(True)
    out = CustomOps.WeightVar(wt, T(s["bounds"]))
    (out * T(g)).sum().backward()
    assert_close(N(out), rv, rtol=2e-4, atol_frac=1e-5, name="weight var")
    assert_close(N(wt.grad), rdw, rtol=2e-3, atol_frac=2e-4, name="weight var bwd")


# ---------------------------------------------------------------------------- octree votes ----
def test_octree_votes_bit_exact(scene, oracle):
    from f2nerf_b200 import GlobalDataPool, PersSampler, SampleResultFlex
    s, feat, rgb, bg = composite_inputs(scene, oracle, n_rays=500, seed=57)
    w, a, keep, nb, tot = oracle.early_stop(feat, 16, s["dt"], s["bounds"])
    n_nodes = scene["nodes"].size // 64
    rng = np.random.default_rng(2)
    sw0 = rng.integers(-3, 4, n_nodes).astype(np.int32)          # stats near zero: visited-but-empty nodes get pruned
    sa0 = rng.integers(-3, 4, n_nodes).astype(np.int32)
    # oracle
    vc = np.zeros(n_nodes, np.int32)
    vw, va, mk = oracle.mark_visit(s["bounds"], s["anchors"].reshape(-1)[1:].copy(), 3, w, a, n_nodes, vc)
    nodes_ref, sw, sa = scene["nodes"].copy(), sw0.copy(), sa0.copy()
    oracle.update_stats(vw, va, mk, sw, sa, nodes_ref)
    # CUDA through the operator mirror
    ps = PersSampler(GlobalDataPool(), scene["nodes"], scene["trans"], scene["edges"])
    ps.tree_weight_stats_.copy_(T(sw0)); ps.tree_alpha_stats_.copy_(T(sa0))
    sr = SampleResultFlex(T(s["pts"]), T(s["dirs"]), T(s["dt"]), T(s["t"]), T(s["anchors"]), T(s["bounds"]), T(s["first_oct_dis"]))
    ps.UpdateOctNodes(sr, T(w), T(a))
    gw, ga, gm = (N(x) for x in ps.last_votes_)
    np.testing.assert_array_equal(gw, vw); np.testing.assert_array_equal(ga, va); np.testing.assert_array_equal(gm, mk)
    np.testing.assert_array_equal(N(ps.tree_visit_cnt_), vc)
    np.testing.assert_array_equal(N(ps.tree_weight_stats_), sw)
    np.testing.assert_array_equal(N(ps.tree_alpha_stats_), sa)
    np.testing.assert_array_equal(N(ps.tree_nodes_gpu_), nodes_ref)          # trans_idx = -1 pruning, byte for byte
    assert (nodes_ref != scene["nodes"]).any(), "test inputs must prune at least one node"


# ---------------------------------------------------------------------- optimizer (SURVEY 8f N1) ----
def aten_adam_step(p, g, m, v, step, lr, b1, b2, eps, wd):
    """torch::optim::Adam::step of the C++ frontend (torch/csrc/api/src/optim/adam.cpp), op for op: the very ATen
    kernels the reference runs (src/ExpRunner.cpp:136)."""
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    if wd != 0:
        g = g.add(p, alpha=wd)
    m.mul_(b1).add_(g, alpha=1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    denom = (v.sqrt() / (bc2 ** 0.5)).add_(eps)
    p.addcdiv_(m, denom, value=-(lr / bc1))


@pytest.mark.parametrize("wd", [0.0, 1e-6])
def test_fused_adam_bit_exact_vs_aten_sequence(wd):
    from f2nerf_b200._lib import call, stream
    gen = torch.Generator(device=DEV).manual_seed(3)
    n = 1 << 20
    p0 = (torch.rand(n, device=DEV, generator=gen) * 2 - 1) * 1e-2
    pa, pf = p0.clone(), p0.clone()
    ma, va, mf, vf = (torch.zeros(n, device=DEV) for _ in range(4))
    shadow = torch.zeros(n, dtype=torch.float16, device=DEV)
    for step in range(1, 6):
        g = torch.randn(n, device=DEV, generator=gen) * 10.0 ** float(torch.randint(-8, -2, (1,)).item())
        g[torch.rand(n, device=DEV, generator=gen) < 0.7] = 0.0          # mostly-empty gradient, like the hash table's
        lr = 1e-2 * (0.5 + 0.1 * step)
        aten_adam_step(pa, g, ma, va, step, lr, 0.9, 0.99, 1e-15, wd)
        call("f2b_adam_step", pf, g, mf, vf, n, n, lr, 0.9, 0.99, 1e-15, wd, step, shadow, stream())
        for a, b, name in ((pa, pf, "param"), (ma, mf, "exp_avg"), (va, vf, "exp_avg_sq")):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (name, step, wd)
        assert torch.equal(shadow, pf.to(torch.float16))


def test_fused_adam_table_live_prefix_and_shadow(scene):
    """FusedAdam on a real field: the table's dead 15/32 stays untouched, the cached fp16 shadow equals a fresh cast,
    and three training steps give bit-identical parameters to the ATen sequence applied to the same gradients."""
    from f2nerf_b200 import FusedAdam, TRAIN
    from test_gpu_render import build
    from conftest import make_rays
    gdp, sampler, field, shader, renderer = build(scene)
    gdp.mode_, gdp.learning_rate_ = TRAIN, 1e-2
    opt = FusedAdam(renderer.OptimParamGroups(), table_field=field)
    ref = {id(p): (p.detach().clone(), torch.zeros_like(p), torch.zeros_like(p)) for g in opt.param_groups for p in g["params"]}
    dead0 = field.feat_pool_.detach().reshape(-1)[17 * field.local_size_:].clone()
    o, d, dn, cam = make_rays(scene, 96, seed=4)
    for step in range(1, 4):
        opt.zero_grad()
        torch.manual_seed(step)
        r = renderer.Render(T(o), T(d), None, T(cam))
        loss = (r.colors ** 2).mean() + 0.1 * ((r.edge_feats[:, 0] - r.edge_feats[:, 1]) ** 2).mean()
        loss.backward()
        for g in opt.param_groups:
            for p in g["params"]:
                pr, m, v = ref[id(p)]
                pr.copy_(p.detach())                                     # same starting point (guards against drift bookkeeping)
                aten_adam_step(pr, p.grad, m, v, step, g["lr"], *g["betas"], g["eps"], g.get("weight_decay", 0.0))
        opt.step()
        for g in opt.param_groups:
            for p in g["params"]:
                assert torch.equal(p.detach().view(torch.int32), ref[id(p)][0].view(torch.int32)), (step, tuple(p.shape))
        assert torch.equal(field.table_f16(), field.feat_pool_.detach().to(torch.float16))
    assert torch.equal(field.feat_pool_.detach().reshape(-1)[17 * field.local_size_:], dead0)
    assert float((field.feat_pool_.grad.reshape(-1)[17 * field.local_size_:]).abs().max()) == 0.0


# ---------------------------------------------------------------------- ray generation (SURVEY 8f N3) ----
def test_img2world_rays_and_gather_vs_oracle(oracle):
    """f2b_img2world_rays == the oracle (bit for bit) on cameras WITH lens distortion (the Newton iteration runs),
    f2b_gather_pixels == index arithmetic; RayGenerator draws on the CPU generator like Dataset::RandRaysData."""
    from f2nerf_b200 import RayGenerator
    rng = np.random.default_rng(8)
    n_cam, H, W, n = 7, 60, 90, 5000
    poses = rng.standard_normal((n_cam, 3, 4)).astype(np.float32)
    intri = np.zeros((n_cam, 3, 3), np.float32)
    intri[:, 0, 0] = 80 + 10 * rng.random(n_cam); intri[:, 1, 1] = 80 + 10 * rng.random(n_cam)
    intri[:, 0, 2] = W / 2 + rng.random(n_cam); intri[:, 1, 2] = H / 2 + rng.random(n_cam); intri[:, 2, 2] = 1
    dist = (rng.standard_normal((n_cam, 4)) * np.array([0.1, 0.02, 1e-3, 1e-3])).astype(np.float32)
    dist[0] = 0                                                       # one undistorted camera
    bounds = rng.random((n_cam, 2)).astype(np.float32)
    images = rng.random((n_cam, H, W, 3)).astype(np.float32)
    gen = RayGenerator(poses, intri, dist, bounds, images=images, train_set=[0, 2, 3, 5, 6], test_set=[1, 4])
    cam = rng.integers(0, n_cam, n).astype(np.int32)
    ij = np.stack([rng.integers(0, H, n), rng.integers(0, W, n)], -1).astype(np.int32)
    ro, rd = gen.Img2WorldRayFlex(T(cam), T(ij))
    wo, wd = oracle.img2world_rays(poses, intri, dist, cam, ij)
    np.testing.assert_array_equal(N(ro).view(np.uint32), wo.view(np.uint32))
    np.testing.assert_array_equal(N(rd).view(np.uint32), wd.view(np.uint32))
    torch.manual_seed(11)
    (ro, rd, b), gt, cams = gen.RandRaysData(4096)
    torch.manual_seed(11)
    cur = torch.tensor([0, 2, 3, 5, 6], dtype=torch.int32)
    c = cur[torch.randint(5, (4096,), dtype=torch.int64)].numpy()
    i = torch.randint(0, H, (4096,), dtype=torch.int64).numpy(); j = torch.randint(0, W, (4096,), dtype=torch.int64).numpy()
    np.testing.assert_array_equal(N(cams), c)
    np.testing.assert_array_equal(N(gt), images[c, i, j])
    np.testing.assert_array_equal(N(b), bounds[c])
    wo, wd = oracle.img2world_rays(poses, intri, dist, c.astype(np.int32), np.stack([i, j], -1).astype(np.int32))
    np.testing.assert_array_equal(N(rd).view(np.uint32), wd.view(np.uint32))


# ---------------------------------------------------------------------- octree maintenance (SURVEY 8f N2) ----
def _damage_tree(nodes_bytes, rng, frac):
    """mark a random subset of the valid leaves dead (trans_idx = -1), like MarkInvalidNodes does over training"""
    t = nodes_bytes.copy().view(np.int32).reshape(-1, 16)
    is_leaf = nodes_bytes.reshape(-1, 64)[:, 52] != 0
    leaves = np.nonzero(is_leaf & (t[:, 14] >= 0))[0]
    dead = rng.choice(leaves, int(len(leaves) * frac), replace=False)
    t[dead, 14] = -1
    return t.reshape(-1).view(np.uint8), dead


@pytest.mark.parametrize("frac", [0.0, 0.3, 0.8])
def test_octree_proc_matches_oracle(scene, oracle, frac):
    """f2b_octree_proc == the sequential ProcOctree restatement, byte for byte: compaction alone, subdivision of the
    visited leaves, brute-force subdivision, and a second round on the result (deeper tree, collapsed chains)."""
    from test_gpu_render import build
    rng = np.random.default_rng(int(frac * 10) + 1)
    gdp, sampler, field, shader, renderer = build(scene)
    nodes, dead = _damage_tree(scene["nodes"], rng, frac)
    n = nodes.size // 64
    w = rng.integers(-100, 2000, n).astype(np.int32); a = rng.integers(-100, 2000, n).astype(np.int32)
    visit = rng.integers(0, 12, n).astype(np.int32)
    for subdivide, brute in ((False, False), (True, False), (True, True)):
        sampler.tree_nodes_gpu_, sampler.tree_weight_stats_, sampler.tree_alpha_stats_ = T(nodes), T(w), T(a)
        sampler.tree_visit_cnt_ = T(visit)
        m = sampler.ProcOctree(True, subdivide, brute)
        on, ow, oa = oracle.octree_proc(nodes, w, a, visit, subdivide, brute)
        assert m == on.size // 64 and (frac == 0.0 or subdivide or m < n)
        np.testing.assert_array_equal(N(sampler.tree_nodes_gpu_), on)
        np.testing.assert_array_equal(N(sampler.tree_weight_stats_), ow)
        np.testing.assert_array_equal(N(sampler.tree_alpha_stats_), oa)
        assert int(sampler.tree_visit_cnt_.abs().sum()) == 0 and sampler.tree_visit_cnt_.shape[0] == m
        if subdivide and not brute:                                  # second round on the subdivided tree
            n2, d2 = _damage_tree(on, rng, 0.5)
            v2 = rng.integers(0, 12, m).astype(np.int32)
            sampler.tree_nodes_gpu_, sampler.tree_visit_cnt_ = T(n2), T(v2)
            m2 = sampler.ProcOctree(True, True, False)
            on2, ow2, oa2 = oracle.octree_proc(n2, ow, oa, v2, True, False)
            assert m2 == on2.size // 64
            np.testing.assert_array_equal(N(sampler.tree_nodes_gpu_), on2)
            np.testing.assert_array_equal(N(sampler.tree_weight_stats_), ow2)
    # the maintained tree still renders: march it
    o, d, dn, cam = make_rays_for(scene, 64)
    sr = sampler.GetSamples(T(o), T(d))
    assert sr.pts.shape[0] > 0 and int(sr.anchors[:, 1].max()) < sampler.n_nodes


def make_rays_for(scene, n):
    from conftest import make_rays
    return make_rays(scene, n, seed=3)


def test_octree_mark_invisible_matches_oracle(scene, oracle):
    """f2b_octree_mark_invisible (PersSampler.cu:617-680) == the sequential restatement, byte for byte: cameras that see the
    scene, cameras that see nothing (looking away / depth window beyond it), and a camera sitting inside a node's sphere."""
    from f2nerf_b200 import GlobalDataPool, PersSampler
    sc = scene["scene"]
    c2w = np.asarray(sc.c2w, np.float32)[:, :3, :4]
    R, t = c2w[:, :, :3], c2w[:, :, 3]
    w2c = np.concatenate([R.transpose(0, 2, 1), -(R.transpose(0, 2, 1) @ t[:, :, None])], 2).astype(np.float32)
    n = w2c.shape[0]
    intri = np.tile(np.array([[255., 0, 100.], [0, 255., 56.], [0, 0, 1]], np.float32), (n, 1, 1))
    for keep, bnd in ((slice(0, n), (0.05, 6.0)), (slice(0, 3), (0.05, 0.6)), (slice(0, 2), (50., 60.)), (slice(0, 0), (0.05, 6.0))):
        bound = np.tile(np.array(bnd, np.float32), (n, 1))[keep]
        gdp = GlobalDataPool()
        sampler = PersSampler(gdp, scene["nodes"], scene["trans"], scene["edges"])
        if bound.shape[0]:
            sampler.MarkInvisibleNodes(intri[keep], w2c[keep], bound)
        else:                                                    # no cameras: every node is invisible
            from f2nerf_b200._lib import call, stream
            z = torch.zeros(1, device="cuda")
            call("f2b_octree_mark_invisible", sampler.tree_nodes_gpu_, sampler.n_nodes, z, z, z, 0, stream())
        want = oracle.mark_invisible(scene["nodes"], intri[keep], w2c[keep], bound)
        np.testing.assert_array_equal(N(sampler.tree_nodes_gpu_), want.reshape(-1))
    ti = want.view(np.int32).reshape(-1, 16)[:, 14]
    assert (ti < 0).all()


def test_hash_level_range_entry_points(scene, oracle, hash_params):
    """f2b_hash_fwd_levels / f2b_hash_bwd_levels: the level groups, run one after the other, reproduce the full encode bit for
    bit and the full scatter to fp32 summation order; a group touches only its own output columns / its own table slab
    [lo*S, (lo+n+1)*S)."""
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    hp = hash_params
    rng = np.random.default_rng(3)
    n = 5000
    pts = T((rng.random((n, 3), dtype=np.float32) * 2 - 1))
    vol = T(rng.integers(0, hp["V"], n).astype(np.int32))
    table, prim, bias = T(hp["table"]), T(hp["prim"]), T(hp["bias"])
    full = ops.hash_fwd(table, prim, bias, hp["V"], hp["local_size"], pts, vol, 1)
    out = torch.full((n, 32), float("nan"), dtype=torch.float16, device=DEV)
    for lo, nl in ((0, 4), (4, 4), (8, 8)):
        call("f2b_hash_fwd_levels", table, prim, bias, hp["V"], hp["local_size"], pts, vol, 1, n, lo, nl, out, stream())
        assert torch.isnan(out[:, 2 * (lo + nl):]).all()
    np.testing.assert_array_equal(N(out).view(np.uint16), N(full).view(np.uint16))
    g = T((rng.standard_normal((n, 32)) * 0.01).astype(np.float16))
    S = hp["local_size"]
    want = torch.zeros((hp["pool"], 2), device=DEV)
    ops.hash_bwd(prim, bias, hp["V"], S, pts, vol, 1, g, 0.5, want)
    got = torch.zeros((hp["pool"], 2), device=DEV)
    for lo in (12, 8, 4, 0):
        before = got.clone()
        call("f2b_hash_bwd_levels", prim, bias, hp["V"], S, pts, vol, 1, n, g, 1, 0.5, got, lo, 4, stream())
        changed = (got != before).view(-1).nonzero().view(-1)
        assert changed.numel() > 0 and int(changed.min()) >= lo * S and int(changed.max()) < (lo + 5) * S
    np.testing.assert_allclose(N(got), N(want), rtol=1e-5, atol=1e-7)
