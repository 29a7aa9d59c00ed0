"""The forward kernels of the march's slot layout (f2b_field_fwd_slots, f2b_slot_bounds, f2b_early_stop_rays, f2b_count_scan,
f2b_compact_slots) and the fused forward renderer (f2b_render_fwd_fused, f2b_gather_kept_weights) against the CPU oracle, on a
slot layout built by hand: no march, so every ray's sample count and the sample at which it turns opaque are chosen.

Planned early stops: the oracle's density logit of each sample fixes dt = tau / exp(logit - 3) for a chosen optical depth tau.
The taus in front of a ray's stop sum to at most 4, so every kept sample has T >= exp(-4) > 1e-2, even on a ray of 1024 samples
that never stops; the stop sample gets tau = 14, so every sample behind it has T <= exp(-14) < 1e-6.  Both are 100x away from
the 1e-4 threshold, far more than the <= 2 fp16-ulp logit differences of DESIGN.md §5 can move T: the keep mask, the kept counts
and every bound are exact expectations.

Counts 0, 1, 31..33, 127..129, 255..257, S-1, S and stops at samples 0, 31, 32, 126..129, 255, 256 and count-1 put the stop on
both sides of the 32-sample chunks (composite.cu) and the 128-sample tiles (field.cu, fused_fwd.cu), in a ray's last tile and in
front of tiles that are never walked.  S = 1024 is the renderer's slot size; S = 384 is a multiple of the tile that is not a
power of two.  A batch holds more than 24 rays per SM (the fused kernel's three resident walkers per SM, eight times over) and
more than 1024 rays (several per thread of the one-block count scan); the longest rays come first and last, so late tickets
draw long rays, and empty rays are interleaved.  Every slot past a ray's count is NaN (a valid volume id in the anchors) and
every output buffer starts as NaN (0xAA for keep), so what a kernel must not write is checked too."""
import numpy as np
import pytest
import torch

from test_gpu_parity import N, T, assert_close, half_ulps

gpu = pytest.mark.gpu

TILE = 128                    # rows per tile of field.cu / fused_fwd.cu
SLOTS = (1024, 384)
H100_SMS = 132                # the SM count the CPU rehearsal plans for (H100 SXM)
N_LONG = 400                  # rays of S samples at each end of the ray order
PAD = 300                     # rows past the kept total in every packed output buffer
FRONT_DEPTH = 4.0             # most optical depth in front of a ray's stop
STOP_TAU = 14.0
T_KEEP = 1e-4                 # the early-stop threshold (Renderer.cpp:125)
LOSS_SCALE = 128.0
NAN = float("nan")


def n_rays(sms):
    return max(3300, 24 * sms + 100)


# ------------------------------------------------------------------------------------------------------------ layout ----
def ray_cases(S):
    """every (count, stop) pair of the listed counts and stop samples; stop -1: the ray never turns opaque"""
    out = set()
    for c in (0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 257, S - 1, S):
        for k in (-1, 0, 31, 32, 126, 127, 128, 129, 255, 256, c - 1):
            if k < c:
                out.add((c, k))
    return sorted(out)


def ray_plan(S, R, rng):
    """-> count [R], stop [R]: N_LONG rays of S samples first and last; in between every case of ray_cases, as many rays of
    random count with a random stop (or none), and an empty ray in every third place"""
    cases = ray_cases(S)
    long = [ck for ck in cases if ck[0] == S]
    n_mid = R - 2 * N_LONG
    empty = np.zeros(n_mid, bool)
    empty[::3] = True
    body = []
    while len(body) < n_mid - empty.sum():
        body += [cases[i] for i in rng.permutation(len(cases))]
        c = rng.integers(1, S + 1, len(cases))
        k = np.where(rng.random(len(cases)) < 0.3, -1, (rng.random(len(cases)) * c).astype(np.int64))
        body += list(zip(c.tolist(), k.tolist()))
    mid = np.zeros((n_mid, 2), np.int64)
    mid[:, 1] = -1
    mid[~empty] = body[: n_mid - empty.sum()]
    plan = np.concatenate([[long[i % len(long)] for i in range(N_LONG)], mid, [long[-1 - i % len(long)] for i in range(N_LONG)]])
    return plan[:, 0].astype(np.int32), plan[:, 1]


def build_layout(oracle, hp, S, R):
    """the slot layout of R rays and its plan.  Arrays in slot order ([R*S, ...]); logit_cpu: the oracle's logits with its own
    level scales (the ones the plan used)"""
    rng = np.random.default_rng(1000 + S)
    V = hp["V"]
    count, stop = ray_plan(S, R, rng)
    j = np.arange(S)
    valid = j < count[:, None]
    kept = np.where(stop >= 0, stop + 1, count).astype(np.int32)
    keep = j < kept[:, None]
    d = rng.standard_normal((R, 3))
    rays_d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    step = rng.uniform(2e-4, 2e-3, R)
    pts = np.clip(rng.uniform(-0.9, 0.9, (R, 1, 3)) + rays_d[:, None, :] * (step[:, None] * j)[:, :, None], -1, 1).astype(np.float32)
    t = (rng.uniform(0.05, 1.0, (R, 1)) + step[:, None] * (j + 1)).astype(np.float32)
    cut = np.where(rng.random(R) < 0.2, rng.integers(1, S, R), S)                 # the volume id changes inside some rays
    vol = np.where(j < cut[:, None], rng.integers(0, V, (R, 1)), rng.integers(0, V, (R, 1)))
    anchors = np.stack([vol, rng.integers(0, V, (R, S))], -1).astype(np.int32)
    front = np.where(stop >= 0, stop, count)
    # taus in [1e-3, cap] in front of the stop: they sum to <= FRONT_DEPTH, and tau >= 1e-3 keeps the fp32 1 - exp(-tau) within
    # 1e-4 relative (cap >= 4/1024 > 1e-3)
    cap = np.minimum(2.0, FRONT_DEPTH / np.maximum(front, 1))
    tau = 1e-3 + rng.random((R, S)) * (cap[:, None] - 1e-3)
    tau = np.where((stop[:, None] >= 0) & (j > stop[:, None]), rng.uniform(1e-3, 3.0, (R, S)), tau)
    stopped = np.nonzero(stop >= 0)[0]
    tau[stopped, stop[stopped]] = STOP_TAU
    fp16 = (oracle.mlp_init(32, 0) * 3).astype(np.float16)
    feat = oracle.hash_fwd(hp["table"], hp["prim"], hp["bias"], V, hp["local_size"], oracle.level_scales(), pts[valid],
                           anchors[valid], 2)
    logit = np.full((R, S), np.nan, np.float32)
    logit[valid] = oracle.mlp_fwd(feat, fp16, 0)[0][:, 0]
    dt = np.full((R, S), np.nan, np.float32)
    dt[valid] = (tau[valid] / np.exp(logit[valid].astype(np.float64) - 3.0)).astype(np.float32)
    pts[~valid] = np.nan
    t[~valid] = np.nan
    anchors[~valid, 0] = V - 1
    excl = np.cumsum(tau, 1) - tau
    return dict(S=S, R=R, count=count, stop=stop, kept=kept, valid=valid, keep=keep & valid, T_plan=np.exp(-excl),
                pts=pts.reshape(-1, 3), dt=dt.reshape(-1), t=t.reshape(-1), anchors=anchors.reshape(-1, 2), rays_d=rays_d,
                bg=rng.random((R, 3), dtype=np.float32), logit_cpu=logit.reshape(-1), fp16=fp16,
                sp16=(oracle.mlp_init(32, 1) * 2).astype(np.float16))


_LAYOUTS = {}


def layout(oracle, hp, S, R):
    if (S, R) not in _LAYOUTS:
        _LAYOUTS[(S, R)] = build_layout(oracle, hp, S, R)
    return _LAYOUTS[(S, R)]


def slot_bounds(L):
    b = np.arange(L["R"], dtype=np.int32) * L["S"]
    return np.stack([b, b + L["count"]], 1).astype(np.int32)


def packed_bounds(counts):
    c = np.cumsum(counts)
    return np.stack([c - counts, c], 1).astype(np.int32)


# ---------------------------------------------------------------------------------------------------------- CPU part ----
@pytest.mark.parametrize("S", SLOTS)
def test_planned_stops_exact_under_oracle(oracle, hash_params, S):
    """the planner's layout: exactly the requested counts and stops under the oracle's own early stop, every planned T at least
    100x away from the threshold, every case present, long rays at both ends, empty rays interleaved"""
    R = n_rays(H100_SMS)
    L = layout(oracle, hash_params, S, R)
    v, keep, Tp = L["valid"], L["keep"], L["T_plan"]
    w, a, got, nb, total = oracle.early_stop(L["logit_cpu"], 1, L["dt"], slot_bounds(L))
    got = got.reshape(R, S).astype(bool)
    assert (got[v] == keep[v]).all(), f"{int((got[v] != keep[v]).sum())} keep bits off the plan"
    np.testing.assert_array_equal(nb, packed_bounds(L["kept"]))
    assert total == int(L["kept"].sum())
    assert Tp[keep].min() >= 100 * T_KEEP and Tp[v & ~keep].max() <= T_KEEP / 100
    assert set(zip(L["count"].tolist(), L["stop"].tolist())) >= set(ray_cases(S))
    assert R >= 24 * H100_SMS and R > 1024
    assert (L["count"][:N_LONG] == S).all() and (L["count"][-N_LONG:] == S).all()
    mid = L["count"][N_LONG:-N_LONG]
    assert (mid[::3] == 0).all() and (mid > 0).mean() > 0.6
    stop, last_tile = L["stop"], (L["count"] - 1) // TILE
    assert ((stop >= 0) & (stop // TILE == last_tile) & (stop < L["count"] - 1)).any()      # a stop inside the last tile
    assert ((stop >= 0) & (last_tile - stop // TILE >= 2)).sum() > 100                      # stops in front of unwalked tiles
    assert L["kept"].max() == S


# ----------------------------------------------------------------------------------------------------------- kernels ----
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def device_inputs(oracle, hp, S):
    """the layout of this device's batch size, its tensors on the device, and the oracle's features / logits of the valid samples
    with the device's level scales (what the kernels encode with)"""
    from f2nerf_b200 import ops
    L = layout(oracle, hp, S, n_rays(sms()))
    if "dev" not in L:
        scales = ops.hash_level_scales().numpy()
        v = L["valid"].reshape(-1)
        feat = oracle.hash_fwd(hp["table"], hp["prim"], hp["bias"], hp["V"], hp["local_size"], scales, L["pts"][v], L["anchors"][v], 2)
        L["ref_feat"], L["ref_out"] = feat, oracle.mlp_fwd(feat, L["fp16"], 0)[0].astype(np.float32)
        L["dev"] = {k: T(L[k]) for k in ("pts", "dt", "t", "anchors", "count", "rays_d", "bg", "fp16", "sp16")}
        L["dev"].update(table=T(hp["table"]), prim=T(hp["prim"]), bias=T(hp["bias"]))
    return L, L["dev"]


def full(shape, fill, dtype=torch.float32):
    return torch.full(shape, fill, dtype=dtype, device="cuda")


def run_field(L, D, hp):
    from f2nerf_b200 import ops
    RS = L["R"] * L["S"]
    logit, feat = full((RS,), NAN), full((RS, 32), NAN, torch.float16)
    ops.field_fwd_slots(D["table"], D["prim"], D["bias"], hp["V"], hp["local_size"], D["fp16"], D["pts"], D["anchors"], D["count"],
                        L["R"], L["S"], logit, feat)
    return logit, feat


def run_phase1(L, D, hp):
    """the early-stop half of a TRAIN step on the slots (csrc/render.cu phase 1 + the compaction of phase 2).  The slot bounds are
    made in two ray chunks, the second with first_ray != 0, as the chunked march makes them."""
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    R, S = L["R"], L["S"]
    logit, feat = run_field(L, D, hp)
    sb = full((R, 2), -7, torch.int32)
    h = R // 2 + 5
    call("f2b_slot_bounds", D["count"][:h], h, S, 0, sb[:h], stream())
    call("f2b_slot_bounds", D["count"][h:], R - h, S, h, sb[h:], stream())
    w, a = full((R * S,), NAN), full((R * S,), NAN)
    keep, kc = full((R * S,), 0xAA, torch.uint8), full((R,), -7, torch.int32)
    ops.early_stop_rays(logit, 1, D["dt"], sb, w, a, keep, kc)
    nb, total = ops.count_scan(kc, R)
    P = int(total)
    o = dict(pts=full((P + PAD, 3), NAN), dirs=full((P + PAD, 3), NAN), dt=full((P + PAD,), NAN), t=full((P + PAD,), NAN),
             anchors=full((P + PAD, 3), -7, torch.int32), feat=full((P + PAD, 32), NAN, torch.float16))
    ops.compact_slots(keep, sb, nb, D["rays_d"], D["pts"], D["dt"], D["t"], D["anchors"], feat,
                      tuple(o[k][:P] for k in ("pts", "dirs", "dt", "t", "anchors")), o["feat"][:P])
    torch.cuda.synchronize()
    return dict(logit_s=logit, feat_s=feat, slot_bounds=sb, w=w, a=a, keep=keep, kept_counts=kc, new_bounds=nb, total=total, P=P, **o)


def run_chain(D, p):
    """the operator chain of phase 2 on the compacted rows: field MLP + shading input, shader MLP + colour activation, composite"""
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    P = p["P"]
    logit, mlp_in = full((P,), NAN), full((P, 32), NAN, torch.float16)
    raw, rgb = full((P, 16), NAN, torch.float16), full((P, 3), NAN)
    call("f2b_field_shade_fwd", p["feat"][:P], D["fp16"], p["dirs"][:P], None, None, P, logit, mlp_in, None, stream())
    call("f2b_shader_mlp_rgb_fwd", mlp_in, D["sp16"], P, raw, rgb, None, stream())
    colors, disp, depth, weights = ops.composite_fwd(logit, 1, rgb, p["dt"][:P], p["t"][:P], p["new_bounds"], D["bg"])
    torch.cuda.synchronize()
    return dict(logit=logit, raw=raw, rgb=rgb, colors=colors, disparity=disp, depth=depth, weights=weights)


def run_fused(L, D, hp, with_weights, total_all):
    from f2nerf_b200._lib import call, stream
    R, S = L["R"], L["S"]
    o = dict(colors=full((R, 3), NAN), disparity=full((R,), NAN), depth=full((R,), NAN), kept=full((R,), -7, torch.int32),
             w_slots=full((R * S,), NAN) if with_weights else None)
    tot = torch.tensor([total_all], dtype=torch.int32, device="cuda") if total_all is not None else None
    call("f2b_render_fwd_fused", D["table"], D["prim"], D["bias"], hp["V"], hp["local_size"], D["fp16"], D["sp16"], D["pts"], D["dt"],
         D["t"], D["anchors"], D["count"], D["rays_d"], D["bg"], R, S, tot, torch.empty(1, dtype=torch.int32, device="cuda"),
         o["colors"], o["disparity"], o["depth"], o["kept"], o["w_slots"], stream())
    torch.cuda.synchronize()
    return o


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32}[a.dtype.itemsize])


def eq_bits(got, want, what):
    g, w = bits(got), bits(want)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = g != w
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} differ; first at {np.argwhere(bad)[0].tolist()}"


# ------------------------------------------------------------------------------------------------------------- tests ----
@gpu
@pytest.mark.parametrize("S", SLOTS)
def test_field_fwd_slots(oracle, hash_params, S):
    """encoded features bit for bit, logits within the MLP-output bar of test_mlp_fwd_bwd; logit slots past a ray's count and
    feature rows of tiles wholly past it stay NaN.  The tile holding a ray's last sample is written whole: its rows past the
    count are zero rows (encode of no sample)."""
    L, D = device_inputs(oracle, hash_params, S)
    R, v = L["R"], L["valid"]
    logit, feat = (N(x) for x in run_field(L, D, hash_params))
    rows = feat.reshape(R, S, 32)
    eq_bits(rows[v], L["ref_feat"], "feature rows")
    lg = logit.reshape(R, S)
    assert_close(lg[v], L["ref_out"][:, 0], rtol=2e-3, atol_frac=1e-3, name="logits")
    assert np.isnan(lg[~v]).all(), "logit slots past a ray's count written"
    tile_end = -(-L["count"] // TILE) * TILE
    j = np.arange(S)
    partial = ~v & (j < tile_end[:, None])
    assert partial.any() and (bits(rows[partial]) == 0).all(), "rows past the count in a ray's last tile are not zero rows"
    assert np.isnan(rows[j >= tile_end[:, None]]).all(), "feature rows of a tile past a ray's count written"


@gpu
@pytest.mark.parametrize("S", SLOTS)
def test_early_stop_bounds_scan_compaction(oracle, hash_params, S):
    """slot bounds, the per-ray early stop on the kernel's own logits (keep mask = the plan = the oracle's, exactly), the count
    scan and the compaction out of the slots, bit for bit"""
    L, D = device_inputs(oracle, hash_params, S)
    R, v, keep_plan = L["R"], L["valid"], L["keep"]
    p = run_phase1(L, D, hash_params)
    sb = slot_bounds(L)
    np.testing.assert_array_equal(N(p["slot_bounds"]), sb)
    keep = N(p["keep"]).reshape(R, S)
    assert (keep[v] == keep_plan[v]).all(), f"{int((keep[v] != keep_plan[v]).sum())} keep bits off the plan"
    rw, ra, rkeep, rnb, rtot = oracle.early_stop(N(p["logit_s"]), 1, L["dt"], sb)
    assert (rkeep.reshape(R, S)[v] == keep[v]).all()
    w, a = N(p["w"]).reshape(R, S), N(p["a"]).reshape(R, S)
    assert_close(w[v], rw.reshape(R, S)[v], rtol=1e-4, atol_frac=1e-6, name="weights")
    assert_close(a[v], ra.reshape(R, S)[v], rtol=1e-4, atol_frac=1e-6, name="alphas")
    assert (keep[~v] == 0xAA).all() and np.isnan(w[~v]).all() and np.isnan(a[~v]).all(), "early stop wrote past a ray's count"
    np.testing.assert_array_equal(N(p["kept_counts"]), L["kept"])
    nb = packed_bounds(L["kept"])
    np.testing.assert_array_equal(N(p["new_bounds"]), nb)
    np.testing.assert_array_equal(rnb, nb)
    P = p["P"]
    assert P == int(L["kept"].sum()) == rtot
    m = keep_plan.reshape(-1)
    ray = np.repeat(np.arange(R), S)[m]
    for k, want in (("pts", L["pts"][m]), ("dt", L["dt"][m]), ("t", L["t"][m]), ("dirs", L["rays_d"][ray])):
        got = N(p[k])
        eq_bits(got[:P], want, f"compacted {k}")
        assert np.isnan(got[P:]).all(), f"compaction wrote {k} rows past the kept total"
    anc = N(p["anchors"])
    np.testing.assert_array_equal(anc[:P, :2], L["anchors"][m])
    assert (anc[:P, 2] == 0).all(), "compacted anchors[:, 2] != 0"
    assert (anc[P:] == -7).all()
    fq = N(p["feat"])
    eq_bits(fq[:P], N(p["feat_s"])[m], "compacted feature rows")
    assert np.isnan(fq[P:]).all()


@gpu
@pytest.mark.parametrize("S", SLOTS)
def test_render_fwd_fused(oracle, hash_params, S):
    """the fused forward == the operator chain on the compacted rows, bit for bit (colours, disparity, depth, the kept samples'
    weights at their slots and packed), with and without weights_slots; kept counts = the plan; the chain's composite against
    the oracle on its own logits / rgb, and the colours against the oracle's whole chain"""
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    L, D = device_inputs(oracle, hash_params, S)
    R = L["R"]
    p = run_phase1(L, D, hash_params)
    P = p["P"]
    ch = {k: N(x) for k, x in run_chain(D, p).items()}
    f = run_fused(L, D, hash_params, True, int(L["count"].sum()))
    f0 = run_fused(L, D, hash_params, False, None)
    np.testing.assert_array_equal(N(f["kept"]), L["kept"])
    for k in ("colors", "disparity", "depth"):
        eq_bits(N(f[k]), ch[k], f"fused {k} vs operator chain")
        eq_bits(N(f0[k]), N(f[k]), f"fused {k} without weights_slots")
    np.testing.assert_array_equal(N(f0["kept"]), L["kept"])
    keep = L["keep"]
    ws = N(f["w_slots"]).reshape(R, S)
    eq_bits(ws[keep], ch["weights"], "fused weights_slots vs operator chain")
    assert np.isnan(ws[~keep]).all(), "weights_slots written past a ray's kept count"
    bounds, total = ops.count_scan(f["kept"], R)
    assert int(total) == P
    wp = full((P + PAD,), NAN)
    call("f2b_gather_kept_weights", f["w_slots"], bounds, R, S, wp[:P], stream())
    wp = N(wp)
    eq_bits(wp[:P], ch["weights"], "gathered weights")
    assert np.isnan(wp[P:]).all()
    empty = L["count"] == 0
    assert empty.sum() > 500
    assert (ch["colors"][empty] == L["bg"][empty]).all() and (ch["depth"][empty] == 0).all() and (ch["disparity"][empty] == 0).all()
    nb = packed_bounds(L["kept"])
    ref = oracle.composite_fwd(ch["logit"], 1, ch["rgb"], N(p["dt"])[:P], N(p["t"])[:P], nb, L["bg"])
    for k, r in zip(("colors", "disparity", "depth", "weights"), ref):
        assert_close(ch[k], r, rtol=1e-4, atol_frac=1e-6, name=f"chain {k} vs oracle composite")
    # the oracle's whole chain: features -> field MLP -> (plan's keep) -> shading input -> shader MLP -> activation -> composite
    m = keep[L["valid"]]
    out = L["ref_out"][m]
    ray = np.repeat(np.arange(R), S)[keep.reshape(-1)]
    raw = oracle.mlp_fwd(oracle.shader_prep(out, L["rays_d"][ray]), L["sp16"], 1)[0]
    colors = oracle.composite_fwd(out, 16, oracle.shader_act(raw), L["dt"][keep.reshape(-1)], L["t"][keep.reshape(-1)], nb, L["bg"])[0]
    err = np.abs(ch["colors"] - colors)
    assert err.max() <= 2e-3 and np.median(err) <= 1e-5, f"colours vs the oracle chain: max {err.max():.3e}, median {np.median(err):.3e}"


@gpu
def test_render_fwd_fused_empty_batch(hash_params):
    """a batch without a single sample (total_all = 0): the background, depth 512, disparity 0, no kept sample, no weight written"""
    from f2nerf_b200._lib import call, stream
    hp = hash_params
    R, S = 24 * sms() + 5, 384
    rng = np.random.default_rng(5)
    bg = T(rng.random((R, 3), dtype=np.float32))
    d = rng.standard_normal((R, 3))
    rays_d = T((d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32))
    nan = full((R * S,), NAN)
    anchors = full((R * S, 2), hp["V"] - 1, torch.int32)
    fp16, sp16 = T((np.ones(64 * 32 + 16 * 64) * 0.01).astype(np.float16)), T((np.ones(64 * 32 + 64 * 64 + 16 * 64) * 0.01).astype(np.float16))
    for with_weights in (True, False):
        colors, disp, depth = full((R, 3), NAN), full((R,), NAN), full((R,), NAN)
        kept, ws = full((R,), -7, torch.int32), full((R * S,), NAN) if with_weights else None
        call("f2b_render_fwd_fused", T(hp["table"]), T(hp["prim"]), T(hp["bias"]), hp["V"], hp["local_size"], fp16, sp16,
             full((R * S, 3), NAN), nan, nan, anchors, torch.zeros(R, dtype=torch.int32, device="cuda"), rays_d, bg, R, S,
             torch.zeros(1, dtype=torch.int32, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda"), colors, disp, depth,
             kept, ws, stream())
        torch.cuda.synchronize()
        assert torch.equal(colors, bg) and bool((depth == 512).all()) and bool((disp == 0).all()) and bool((kept == 0).all())
        assert ws is None or bool(torch.isnan(ws).all())


@gpu
def test_composite_act_bwd_long_rays(oracle, hash_params):
    """f2b_composite_act_bwd on the compacted rows of rays with up to 1024 kept samples (32 chunks of the reverse scan) against
    O.composite_bwd: d_logit within the bar of test_composite_fwd_bwd, d_raw = the oracle's d_rgb through the colour activation's
    backward (tests/oracle_pipeline.py) within 2 fp16 ulp"""
    from f2nerf_b200._lib import call, stream
    L, D = device_inputs(oracle, hash_params, 1024)
    R = L["R"]
    assert L["kept"].max() == 1024
    p = run_phase1(L, D, hash_params)
    P = p["P"]
    ch = run_chain(D, p)
    rng = np.random.default_rng(61)
    dc, dd, dz = (rng.standard_normal((R, 3)).astype(np.float32), (rng.standard_normal(R) * .1).astype(np.float32),
                  (rng.standard_normal(R) * .1).astype(np.float32))
    dw = (rng.standard_normal(P) * .01).astype(np.float32)
    # the activation's backward as the oracle pipeline's shader backward takes it: fp32 sigmoid, like the reference's autograd
    # (its 1 - sigmoid cancels for raw above ~9, where a float64 sigmoid would differ by tens of fp16 ulp)
    o3 = N(ch["raw"])[:, :3].astype(np.float32)
    sg = 1.0 / (1.0 + np.exp(-o3))
    assert sg.dtype == np.float32 and o3.max() > 9
    for gs in (1.0, 0.3):
        d_logit, d_raw = full((P + PAD,), NAN), full((P + PAD, 16), NAN, torch.float16)
        call("f2b_composite_act_bwd", ch["logit"], 1, ch["rgb"], p["dt"][:P], p["t"][:P], p["new_bounds"], D["bg"], R, T(dc), T(dd),
             T(dz), T(dw), float(gs), ch["raw"], LOSS_SCALE, d_logit[:P], 1, d_raw[:P], stream())
        torch.cuda.synchronize()
        rl, rr = oracle.composite_bwd(N(ch["logit"]), 1, N(ch["rgb"]), N(p["dt"])[:P], N(p["t"])[:P], N(p["new_bounds"]), L["bg"],
                                      dc, dd, dz, dw, gs)
        gl, gr = N(d_logit), N(d_raw).astype(np.float32)
        assert_close(gl[:P], rl, rtol=2e-4, atol_frac=2e-5, name=f"d_logit gs={gs}")
        want = rr * (1.0 + 2e-3) * sg * (1.0 - sg) * LOSS_SCALE
        assert half_ulps(gr[:P, :3], want) <= 2.0, f"d_raw gs={gs}: {half_ulps(gr[:P, :3], want)} fp16 ulp"
        assert (gr[:P, 3:] == 0).all()
        assert np.isnan(gl[P:]).all() and np.isnan(gr[P:]).all()
