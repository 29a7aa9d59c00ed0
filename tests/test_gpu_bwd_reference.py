"""The training backward kernels (f2b_shade_field_bwd_scatter, f2b_field_bwd_scatter, f2b_mlp_bwd2, f2b_hash_bwd, f2b_hash_bwd_levels)
against references that run no project kernel: torch float64 for the MLP parts, the CPU oracle's double-precision scatter
(oracle.hash_bwd) for the table gradient.

Exact-operand regime: every weight matrix has at most two nonzeros (+-1) per row and per column, the inputs and output gradients
are in {-1, 0, 1} (d_logit in {-1, 0, 1} * 2^-6) and the loss scales are powers of two.  Every activation, activation gradient
and fp16 row is then a small dyadic value, every fp16 rounding is the identity, and as long as each sum's sum of |terms| stays
below 2^22 steps every fp32 partial sum is exact in any order.  So the debug rows, the weight gradients and d_app must equal the
float64 reference exactly, whatever the tile schedule.  The table gradient has non-dyadic corner weights: it is held per entry,
|got - exact| <= 2^-12 * sum|contributions| (untouched entries exactly 0).

Sizes are chosen from the SM count so that the persistent schedules are reached on purpose: the shade kernel runs min(tiles, SMs)
CTAs, so tiles = SMs + 1 gives one CTA a second tile and 2 SMs + 1 gives one a third (ring slot 0 reused); the field kernel and
f2b_mlp_bwd2 run SMs x resident CTAs (at most 4 per SM), so 12 SMs + 5 tiles give every CTA at least three.  Every size ends in a
partial tile.  Every per-sample input is the first n rows of a longer buffer whose tail is NaN (a valid volume / camera id for
integers), and every output row buffer has a NaN tail that must stay untouched."""
import numpy as np
import pytest
import torch

from test_gpu_parity import N, T

pytestmark = pytest.mark.gpu

BT = 128                      # rows per tile of the persistent kernels
PAD = 300                     # rows past n in every per-sample buffer
EXACT_STEPS = 2.0 ** 22       # sum|terms| bound, in units of the terms' step, for an order-independent fp32 sum
TABLE_TOL = 2.0 ** -12        # per-entry table bar, relative to the entry's sum of |contributions|
N_EMB = 7
S_SCALE, F_SCALE, GRAD_MUL = 128.0, 64.0, 1.0 / 64.0
TILES = {"sms+1": lambda s: s + 1, "2sms": lambda s: 2 * s, "2sms+1": lambda s: 2 * s + 1, "5sms+3": lambda s: 5 * s + 3,
         "12sms+5": lambda s: 12 * s + 5, "8192": lambda s: 8192}          # 8192 tiles: ~1 M samples
F64 = dict(dtype=torch.float64, device="cuda")


def n_of(tiles):
    return BT * TILES[tiles](torch.cuda.get_device_properties(0).multi_processor_count) - 77


# ------------------------------------------------------------------------------------------------------------ inputs ----
def prefix(a, fill):
    """numpy rows a as the first len(a) rows of a device buffer with PAD more rows of `fill`"""
    full = np.full((a.shape[0] + PAD,) + a.shape[1:], fill, dtype=a.dtype)
    full[: a.shape[0]] = a
    return T(full)[: a.shape[0]]


def out_rows(n, cols):
    """NaN-filled fp16 output rows with a PAD-row tail (returned whole: the kernel gets [:n], the tail is checked afterwards)"""
    return torch.full((n + PAD, cols), float("nan"), dtype=torch.float16, device="cuda")


def ray_layout(n, V, rng):
    """n ray-like samples: rays of 1..200 consecutive samples along a line in [-1, 1]^3 (steps 1e-3..1e-2), a volume id constant
    per ray except for an occasional change inside a ray, a camera index that differs between adjacent rays.
    -> pts [n,3] f32, anchors [n,3] i32 (volume id in column 0: stride 3), camera index per sample [n] i32"""
    lens = rng.integers(1, 201, n // 50 + 8)
    R = int(np.searchsorted(np.cumsum(lens), n)) + 1
    lens = lens[:R]
    ray = np.repeat(np.arange(R), lens)[:n]
    pos = np.arange(n) - np.concatenate([[0], np.cumsum(lens)[:-1]])[ray]
    o = rng.uniform(-0.9, 0.9, (R, 3))
    d = rng.standard_normal((R, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    step = rng.uniform(1e-3, 1e-2, R)
    pts = np.clip(o[ray] + d[ray] * (step[ray] * pos)[:, None], -1, 1).astype(np.float32)
    cut = np.where(rng.random(R) < 0.1, rng.integers(1, 201, R), 1 << 30)
    vol = np.where(pos >= cut[ray], rng.integers(0, V, R)[ray], rng.integers(0, V, R)[ray])
    anchors = np.stack([vol, rng.integers(0, V, n), rng.integers(0, V, n)], 1).astype(np.int32)
    cam = (np.cumsum(rng.integers(1, N_EMB, R)) % N_EMB).astype(np.int32)
    emb = cam[ray]
    groups = emb[: n - n % 32].reshape(-1, 32)
    assert (groups[:, 1:] != groups[:, :-1]).any(1).sum() > 0                 # groups with two camera runs
    return pts, anchors, emb


def edge_layout(n, V, rng):
    """edge-like point pairs with a flat volume id per pair (stride 1)"""
    a = rng.uniform(-1, 1, (n // 2 + 1, 3))
    b = np.clip(a + rng.standard_normal(a.shape) * 1e-3, -1, 1)
    pts = np.stack([a, b], 1).reshape(-1, 3)[:n].astype(np.float32)
    return pts, np.repeat(rng.integers(0, V, n // 2 + 1), 2)[:n].astype(np.int32)


def sparse_pm1(rows, cols, rng):
    """[rows, cols] in {-1, 0, 1}, at most two nonzeros per row and per column (two partial signed permutations)"""
    w = np.zeros((rows, cols))
    k = min(rows, cols)
    for _ in range(2):
        r, c = rng.permutation(rows)[:k], rng.permutation(cols)[:k]
        free = w[r, c] == 0
        w[r[free], c[free]] = rng.choice([-1.0, 1.0], int(free.sum()))
    return w


def tern(shape, rng, density=0.5):
    return rng.choice([-1.0, 0.0, 1.0], shape, p=[density / 2, 1 - density, density / 2])


def params16(ws):
    return np.concatenate([w.ravel() for w in ws if w is not None]).astype(np.float16)


def exact_operands(n, rng, dead=None):
    """exact-regime shader + field operands; `dead` rows get all-zero shader dL/dout and d_logit (all-zero field rows)"""
    d_raw = tern((n, 16), rng)
    d_raw[rng.random(n) < 0.2] = 0                                            # all-zero shader dL/dout rows
    d_logit = tern(n, rng) * 2.0 ** -6
    if dead is not None:
        d_raw[dead] = 0
        d_logit[dead] = 0
    return dict(sw=[sparse_pm1(64, 32, rng), sparse_pm1(64, 64, rng), sparse_pm1(16, 64, rng)],
                fw=[sparse_pm1(64, 32, rng), None, sparse_pm1(16, 64, rng)],
                mlp_in=tern((n, 32), rng), feat=tern((n, 32), rng), d_raw=d_raw, d_logit=d_logit)


# -------------------------------------------------------------------------------------------------------- references ----
def f16_exact(t, what):
    assert torch.equal(t, t.to(torch.float16).to(torch.float64)), f"{what}: not exact in fp16 (operands outside the exact regime)"


def sum_exact(abssum, step, what):
    assert float(abssum.max()) / step < EXACT_STEPS, f"{what}: sum|terms| {float(abssum.max())} too large for an exact fp32 sum"


def mlp_bwd_ref(dout, x, ws, step):
    """float64 backward of relu(x W0^T) [-> relu(. Wh^T)] -> . Wout^T (ws = [W0, Wh | None, Wout], rows = outputs).
    -> dL/dinput, dparams in f2b_mlp_bwd2's layout, forward activations [H0, H1 | None].  Asserts that every intermediate is
    exact in fp16 and every weight-gradient sum exact in fp32 (terms are multiples of `step`)."""
    W0, Wh, Wo = (torch.as_tensor(w, **F64) if w is not None else None for w in ws)
    h0 = (x @ W0.T).clamp_min(0)
    hl = (h0 @ Wh.T).clamp_min(0) if Wh is not None else h0
    dhl = (dout @ Wo) * (hl > 0)                                               # the mask is "> 0": exact zeros are masked
    grads, sums = [dout.T @ hl], [dout.abs().T @ hl]
    if Wh is not None:
        dh0 = (dhl @ Wh) * (h0 > 0)
        grads.insert(0, dhl.T @ h0)
        sums.insert(0, dhl.abs().T @ h0)
    else:
        dh0 = dhl
    grads.insert(0, dh0.T @ x)
    sums.insert(0, dh0.abs().T @ x.abs())
    din = dh0 @ W0
    for t, what in ((h0, "H0"), (hl, "H_last"), (dhl, "dH_last"), (dh0, "dH0"), (din, "dIn")):
        f16_exact(t, what)
    sum_exact(torch.cat([s.ravel() for s in sums]), step, "weight gradient")
    return din, torch.cat([g.ravel() for g in grads]), [h0, hl if Wh is not None else None]


def shade_ref(op, emb):
    """f2b_shade_field_bwd_scatter's outputs in float64: shader dIn, field dL/dout, field dL/dfeat, both dparams, d_app"""
    x = {k: torch.as_tensor(op[k], **F64) for k in ("mlp_in", "feat", "d_raw", "d_logit")}
    din, dsp, _ = mlp_bwd_ref(x["d_raw"], x["mlp_in"], op["sw"], 1.0)
    g = din[:, :16] / S_SCALE
    fdo = g.clone()
    fdo[:, 0] = x["d_logit"]
    fdo *= F_SCALE
    f16_exact(fdo, "field dL/dout")
    dfeat, dfp, _ = mlp_bwd_ref(fdo, x["feat"], op["fw"], 0.5)                 # field dL/dout is a multiple of 1/2
    app = None
    if emb is not None:
        e = torch.as_tensor(emb, dtype=torch.long, device=F64["device"])
        app = torch.zeros((N_EMB, 16), **F64).index_add_(0, e, g)
        sum_exact(torch.zeros((N_EMB, 16), **F64).index_add_(0, e, g.abs()), 1.0 / S_SCALE, "d_app")
    return dict(din=din, scene=fdo, dfeat=dfeat, dsp=dsp, dfp=dfp, app=app)


def check_table(oracle, hp, got, pts, vol, stride, dfeat, grad_mul, tag):
    """per entry: |got - exact| <= 2^-12 * sum|contributions|; untouched entries (and the unused 15/32 of the pool) exactly 0"""
    from f2nerf_b200 import ops
    scales = ops.hash_level_scales().numpy()
    args = (hp["prim"], hp["bias"], hp["V"], hp["local_size"], scales, pts, vol, stride)
    g = np.ascontiguousarray(dfeat, np.float32)
    exact = oracle.hash_bwd(*args, g, grad_mul, hp["pool"])
    abssum = oracle.hash_bwd(*args, np.abs(g), grad_mul, hp["pool"])          # corner weights are >= 0
    got = np.asarray(got, np.float64)
    err = np.abs(got - exact)
    bad = ~(err <= TABLE_TOL * abssum)
    assert (abssum > 0).any()
    assert not bad.any(), (f"table {tag}: {int(bad.sum())} entries off, worst at {int(np.argmax(np.where(bad, err, 0)))}: "
                           f"err {err[bad].max():.3e}; untouched entries nonzero: {int((bad & (abssum == 0)).sum())}")
    assert not got[(17 * hp["local_size"]) // 2 + 1:].any()


def eq(got, ref, what):
    """got (kernel output, any float dtype) == ref (float64) exactly, element for element"""
    got = torch.as_tensor(got).to("cuda", torch.float64)
    bad = ~(got == ref)
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {bad.numel()} differ; first at {tuple(bad.nonzero()[0].tolist())}: "
                                 f"got {float(got[bad][0])}, exact {float(ref[bad][0])}")


def tail_untouched(buf, n, what):
    assert bool(torch.isnan(buf[n:].float()).all()), f"{what}: rows past n written"


# ------------------------------------------------------------------------------------------------------------ kernels ----
def run_shade(hp, op, pts, anchors, emb, side_work=None):
    """f2b_shade_field_bwd_scatter on poisoned-tail inputs -> outputs as tensors (debug rows with their tails)"""
    from f2nerf_b200._lib import call, stream
    n, V = pts.shape[0], hp["V"]
    nan = np.float32("nan")
    z = lambda *s: torch.zeros(s, dtype=torch.float32, device="cuda")
    o = dict(din=out_rows(n, 32), scene=out_rows(n, 16), dfeat=out_rows(n, 32), dsp=z(64 * 32 + 64 * 64 + 16 * 64),
             dfp=z(64 * 32 + 16 * 64), table=z(hp["pool"], 2), app=z(N_EMB, 16) if emb is not None else None)
    args = (prefix(op["d_raw"].astype(np.float16), nan), prefix(op["mlp_in"].astype(np.float16), nan), T(params16(op["sw"])),
            prefix(op["d_logit"].astype(np.float32), nan), prefix(emb, N_EMB - 1) if emb is not None else None, 1.0 / S_SCALE, F_SCALE,
            prefix(op["feat"].astype(np.float16), nan), T(params16(op["fw"])), n, prefix(pts, nan), prefix(anchors, V - 1), 3,
            T(hp["prim"]), T(hp["bias"]), V, hp["local_size"], GRAD_MUL, o["dsp"], o["dfp"], o["table"], o["app"],
            torch.empty((1,), dtype=torch.int32, device="cuda"), o["din"][:n], o["scene"][:n], o["dfeat"][:n])
    torch.cuda.synchronize()
    if side_work is not None:
        side_work()                                                            # queued on another stream, not waited for
    call("f2b_shade_field_bwd_scatter", *args, stream())
    torch.cuda.synchronize()
    return o


def check_shade(oracle, hp, op, pts, anchors, emb, o, tag):
    n = pts.shape[0]
    ref = shade_ref(op, emb)
    for k, what in (("din", "shader dIn rows"), ("scene", "field dL/dout rows"), ("dfeat", "field dL/dfeat rows")):
        eq(o[k][:n], ref[k], f"{what} {tag}")
        tail_untouched(o[k], n, f"{what} {tag}")
    eq(o["dsp"], ref["dsp"], f"shader dparams {tag}")
    eq(o["dfp"], ref["dfp"], f"field dparams {tag}")
    if emb is not None:
        assert bool(ref["app"].abs().max() > 0)
        eq(o["app"], ref["app"], f"d_app {tag}")
    check_table(oracle, hp, N(o["table"]), pts, anchors, 3, N(ref["dfeat"]), GRAD_MUL, tag)


def run_field(hp, dout, feat, fw, pts, vol, stride, grad_mul=0.5):
    from f2nerf_b200._lib import call, stream
    n, nan = pts.shape[0], np.float32("nan")
    din = out_rows(n, 32)
    dp = torch.zeros(64 * 32 + 16 * 64, dtype=torch.float32, device="cuda")
    table = torch.zeros((hp["pool"], 2), dtype=torch.float32, device="cuda")
    call("f2b_field_bwd_scatter", prefix(dout.astype(np.float16), nan), prefix(feat.astype(np.float16), nan), T(params16(fw)), n,
         prefix(pts, nan), prefix(vol, hp["V"] - 1), stride, T(hp["prim"]), T(hp["bias"]), hp["V"], hp["local_size"], grad_mul, dp,
         table, din[:n], stream())
    torch.cuda.synchronize()
    return din, dp, table


def check_field(oracle, hp, dout, feat, fw, pts, vol, stride, tag):
    n = pts.shape[0]
    din, dp, table = run_field(hp, dout, feat, fw, pts, vol, stride)
    ref_din, ref_dp, _ = mlp_bwd_ref(torch.as_tensor(dout, **F64), torch.as_tensor(feat, **F64), fw, 1.0)
    eq(din[:n], ref_din, f"field dL/dfeat rows {tag}")
    tail_untouched(din, n, f"field dL/dfeat rows {tag}")
    eq(dp, ref_dp, f"field dparams {tag}")
    check_table(oracle, hp, N(table), pts, vol, stride, N(ref_din), 0.5, tag)


# -------------------------------------------------------------------------------------------------------------- tests ----
@pytest.mark.parametrize("tiles,emb", [("sms+1", False), ("sms+1", True), ("2sms", True), ("2sms+1", False), ("2sms+1", True),
                                       ("5sms+3", True), ("8192", True)])
def test_shade_field_bwd_scatter_exact(oracle, hash_params, tiles, emb):
    n = n_of(tiles)
    rng = np.random.default_rng(n + emb)
    pts, anchors, cam = ray_layout(n, hash_params["V"], rng)
    op = exact_operands(n, rng)
    e = cam if emb else None
    check_shade(oracle, hash_params, op, pts, anchors, e, run_shade(hash_params, op, pts, anchors, e), f"tiles={tiles} emb={emb}")


@pytest.mark.parametrize("tiles,stride", [("12sms+5", 3), ("12sms+5", 1), ("8192", 3)])
def test_field_bwd_scatter_exact(oracle, hash_params, tiles, stride):
    n = n_of(tiles)
    rng = np.random.default_rng(n + stride)
    if stride == 3:
        pts, vol, _ = ray_layout(n, hash_params["V"], rng)
    else:
        pts, vol = edge_layout(n, hash_params["V"], rng)
    dout = tern((n, 16), rng)
    dout[rng.random(n) < 0.2] = 0
    fw = [sparse_pm1(64, 32, rng), None, sparse_pm1(16, 64, rng)]
    check_field(oracle, hash_params, dout, tern((n, 32), rng), fw, pts, vol, stride, f"tiles={tiles} stride={stride}")


@pytest.mark.parametrize("nh", [0, 1])
@pytest.mark.parametrize("saved", [True, False])
def test_mlp_bwd2_exact(nh, saved):
    from f2nerf_b200._lib import call, stream
    n = n_of("12sms+5")
    rng = np.random.default_rng(500 + 2 * nh + saved)
    ws = [sparse_pm1(64, 32, rng), sparse_pm1(64, 64, rng) if nh else None, sparse_pm1(16, 64, rng)]
    dout, x = tern((n, 16), rng), tern((n, 32), rng)
    dout[rng.random(n) < 0.2] = 0
    ref_din, ref_dp, hid = mlp_bwd_ref(torch.as_tensor(dout, **F64), torch.as_tensor(x, **F64), ws, 1.0)
    nan = np.float32("nan")
    h0 = prefix(N(hid[0]).astype(np.float16), nan) if saved else None
    h1 = prefix(N(hid[1]).astype(np.float16), nan) if saved and nh else None
    din = out_rows(n, 32)
    dp = torch.zeros(ref_dp.numel(), dtype=torch.float32, device="cuda")
    call("f2b_mlp_bwd2", prefix(dout.astype(np.float16), nan), prefix(x.astype(np.float16), nan), h0, h1, T(params16(ws)), nh, n,
         din[:n], dp, stream())
    torch.cuda.synchronize()
    eq(din[:n], ref_din, f"dIn nh={nh} saved={saved}")
    tail_untouched(din, n, "dIn")
    eq(dp, ref_dp, f"dparams nh={nh} saved={saved}")


def test_shade_field_bwd_scatter_table_realistic(oracle, hash_params):
    """realistic fp16 values (as the fused-vs-unfused tests use): the table gradient of the kernel's own dL/dfeat rows, per entry"""
    hp = hash_params
    n = n_of("2sms+1")
    rng = np.random.default_rng(77)
    pts, anchors, cam = ray_layout(n, hp["V"], rng)
    d_raw = (rng.standard_normal((n, 16)) * 0.1).astype(np.float16)
    d_raw[1::5] = 0
    d_logit = (rng.standard_normal(n) * 0.05).astype(np.float32)
    d_logit[1::10] = 0
    op = dict(sw=[oracle.mlp_init(32, 1) * 2], fw=[oracle.mlp_init(32, 0) * 2], mlp_in=rng.standard_normal((n, 32)) * 0.5,
              feat=rng.standard_normal((n, 32)) * 0.5, d_raw=d_raw, d_logit=d_logit)
    o = run_shade(hp, op, pts, anchors, cam)
    dfeat = N(o["dfeat"][:n]).astype(np.float32)
    assert np.isfinite(dfeat).all() and (dfeat != 0).any()
    check_table(oracle, hp, N(o["table"]), pts, anchors, 3, dfeat, GRAD_MUL, "realistic")


def test_shade_field_bwd_scatter_skewed_schedule(oracle, hash_params):
    """one call right behind large matmuls queued on a second stream: CTAs start late, some may find no tile left"""
    n = n_of("5sms+3")
    rng = np.random.default_rng(91)
    pts, anchors, cam = ray_layout(n, hash_params["V"], rng)
    op = exact_operands(n, rng)
    side = torch.cuda.Stream()
    a = torch.randn((8192, 8192), dtype=torch.float16, device="cuda")
    keep = []

    def side_work():
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            keep.extend([a @ a, a @ a])

    o = run_shade(hash_params, op, pts, anchors, cam, side_work)
    check_shade(oracle, hash_params, op, pts, anchors, cam, o, "skewed")


# ------------------------------------------------------------------------------------------- scatter_level run layouts ----
LEVEL = 4                     # the level whose cells the layout is built on


def cells_at(hp, scales, pts, vol, l):
    """integer cell coordinates of each point at level l (the kernels' float32 arithmetic; the floor has a >= 0.1 margin)"""
    x = (pts.astype(np.float32) + np.float32(1)) * np.float32(0.5)
    b = hp["bias"].reshape(16, hp["V"], 3)[l, vol].astype(np.float64)
    return np.maximum(np.floor(x.astype(np.float64) * float(scales[l]) + b), 0).astype(np.int64)


def run_layout(hp, scales, rng):
    """32-sample groups of chosen run patterns at level LEVEL -> pts, volume ids, gradient rows [n,32] f32 (fp16 values), group names"""
    V, L = hp["V"], LEVEL
    bias = hp["bias"].reshape(16, V, 3)[L].astype(np.float64)
    va, vb = 0, V - 1
    base = np.floor(bias[va])
    fresh = iter(range(1, 10 ** 6))
    rows, names = [], []                                        # row: (point, volume, dead) dead in {None, "all", "L"}

    def at(cell, v=va, dead=None):
        u = rng.uniform(0.15, 0.85, 3)                          # a point inside the cell, away from its faces
        return ((base + cell + u - bias[v]) / float(scales[L]) * 2 - 1, v, dead)

    def new_cell():
        i = next(fresh)
        return np.array([1 + i % 8, 1 + (i // 8) % 8, 1 + i // 64], np.float64)

    def runs(lengths):
        out = []
        for k in lengths:
            c = new_cell()
            out += [at(c) for _ in range(k)]
        return out

    def group(name, lanes):
        assert len(lanes) == 32 or name == "partial"
        names.append(name)
        rows.extend(lanes)

    c = new_cell()
    group("run32", [at(c) for _ in range(32)])
    group("heads24", runs([2] * 8 + [1] * 16))
    group("heads25", runs([2] * 7 + [1] * 18))
    group("singletons", runs([1] * 32))
    a_, b_ = new_cell(), new_cell()
    group("abab", [at(a_ if i % 2 == 0 else b_) for i in range(32)])
    c = new_cell()
    group("volume_breaks", [at(c, va if (i // 4) % 2 == 0 else vb) for i in range(32)])
    c = new_cell()
    group("zero_rows", [at(c, dead="all" if i in (5, 6, 17) else None) for i in range(32)])
    c = new_cell()
    group("dead_at_L", [at(c, dead="L" if 8 <= i < 24 else None) for i in range(32)])
    c = new_cell()
    group("cross_a", runs([1] * 26) + [at(c) for _ in range(6)])
    group("cross_b", [at(c) for _ in range(6)] + runs([2] * 13))
    sat = [(np.full(3, -1000.0 - 0.37 * i), va, None) for i in range(12)]      # negative: cell 0 at every level
    group("saturated", runs([1] * 10) + sat + runs([3] * 3 + [1]))
    c = new_cell()
    group("partial", runs([1] * 8) + [at(c) for _ in range(12)])
    pts = np.array([r[0] for r in rows], np.float32)
    vol = np.array([r[1] for r in rows], np.int32)
    g = rng.standard_normal((len(rows), 32)).astype(np.float16).astype(np.float32)
    g[g == 0] = 1.0
    dead = np.array([r[2] for r in rows], object)
    g[dead == "all"] = 0
    g[dead == "L", 2 * L: 2 * L + 2] = 0
    return pts, vol, g, names


def assert_layout_coverage(hp, scales, pts, vol, g, names):
    """every pattern the layout is meant to hold really occurs at level LEVEL (coverage only: correctness comes from the oracle)"""
    L, n = LEVEL, pts.shape[0]
    cells = cells_at(hp, scales, pts, vol, L)
    live = (g[:, 2 * L] != 0) | (g[:, 2 * L + 1] != 0)
    same = np.zeros(n, bool)
    same[1:] = (cells[1:] == cells[:-1]).all(1) & (vol[1:] == vol[:-1]) & live[1:] & live[:-1]
    head = ~same
    head[::32] = True
    by = {}
    for k, name in enumerate(names):
        s = slice(32 * k, min(32 * k + 32, n))
        by[name] = dict(heads=int(head[s].sum()), live=live[s], same=same[s], cells=cells[s], vol=vol[s])
    assert by["run32"]["heads"] == 1 and by["run32"]["same"][31]                      # one run, ending at lane 31
    assert by["heads24"]["heads"] == 24 and by["heads25"]["heads"] == 25             # both sides of kDirectHeads
    assert by["singletons"]["heads"] == 32 and by["abab"]["heads"] == 32
    vb = by["volume_breaks"]
    assert vb["heads"] == 8 and (vb["cells"] == vb["cells"][0]).all()               # broken by the volume id alone
    zr = by["zero_rows"]
    assert zr["heads"] == 6 and (~zr["live"]).sum() == 3                            # dead lanes inside a run
    dl = by["dead_at_L"]
    assert (~dl["live"]).sum() == 16 and dl["heads"] == 18
    assert all(((g[32 * names.index("dead_at_L"): 32 * names.index("dead_at_L") + 32, 2 * l: 2 * l + 2] != 0).any(1)).all()
               for l in range(16) if l != L)                                         # ... and live at every other level
    assert same[32 * (names.index("cross_a") + 1)]                                  # a run crosses the group boundary
    sat = by["saturated"]
    assert (sat["cells"][10:22] == 0).all() and not sat["same"][10] and sat["same"][11:22].all()
    s = slice(32 * names.index("saturated") + 10, 32 * names.index("saturated") + 22)
    assert all((cells_at(hp, scales, pts[s], vol[s], l) == 0).all() for l in range(16))
    p = by["partial"]
    assert n % 32 == 20 and p["same"][-11:].all() and p["live"][-1]                  # the run meets the end of the samples
    return by


def layout(oracle, hp):
    rng = np.random.default_rng(4242)
    scales = oracle.level_scales()                               # (the device's scales differ by <= 2 ulp: the cells do not)
    pts, vol, g, names = run_layout(hp, scales, rng)
    assert_layout_coverage(hp, scales, pts, vol, g, names)
    return pts, vol, g, names


@pytest.mark.parametrize("stride", [1, 3])
@pytest.mark.parametrize("half", [False, True])
def test_hash_bwd_run_layouts(oracle, hash_params, stride, half):
    from f2nerf_b200 import ops
    hp = hash_params
    pts, vol, g, _ = layout(oracle, hp)
    v = vol if stride == 1 else np.stack([vol, vol[::-1], vol], 1).astype(np.int32)
    table = torch.zeros((hp["pool"], 2), dtype=torch.float32, device="cuda")
    gt = prefix(g.astype(np.float16) if half else g, np.float16("nan") if half else np.float32("nan"))
    ops.hash_bwd(T(hp["prim"]), T(hp["bias"]), hp["V"], hp["local_size"], prefix(pts, np.float32("nan")), prefix(v, hp["V"] - 1),
                 stride, gt, 0.5, table)
    torch.cuda.synchronize()
    check_table(oracle, hp, N(table), pts, v, stride, g, 0.5, f"hash_bwd stride={stride} half={half}")


@pytest.mark.parametrize("stride", [1, 3])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("group", [1, 2, 4, 8, "renderer"])
def test_hash_bwd_levels_run_layouts(oracle, hash_params, group, stride, half):
    """level groups high to low; "renderer": the data-parallel backward's own groups (renderer.slab_groups), which it scatters
    with stride-3 anchors and fp16 rows"""
    from f2nerf_b200._lib import call, stream
    from f2nerf_b200.renderer import slab_groups
    hp = hash_params
    pts, vol, g, _ = layout(oracle, hp)
    n = pts.shape[0]
    v = vol if stride == 1 else np.stack([vol, vol[::-1], vol], 1).astype(np.int32)
    table = torch.zeros((hp["pool"], 2), dtype=torch.float32, device="cuda")
    gt = prefix(g.astype(np.float16) if half else g, np.float16("nan") if half else np.float32("nan"))
    args = (T(hp["prim"]), T(hp["bias"]), hp["V"], hp["local_size"], prefix(pts, np.float32("nan")), prefix(v, hp["V"] - 1), stride,
            n, gt, int(half), 0.5, table)
    groups = slab_groups() if group == "renderer" else [(lo, group) for lo in reversed(range(0, 16, group))]
    for lo, nl in groups:
        call("f2b_hash_bwd_levels", *args, lo, nl, stream())
    torch.cuda.synchronize()
    check_table(oracle, hp, N(table), pts, v, stride, g, 0.5, f"hash_bwd_levels group={group} stride={stride} half={half}")


@pytest.mark.parametrize("stride", [1, 3])
def test_field_bwd_scatter_run_layouts(oracle, hash_params, stride):
    hp = hash_params
    pts, vol, g, _ = layout(oracle, hp)
    n = pts.shape[0]
    rng = np.random.default_rng(17 + stride)
    dout = tern((n, 16), rng, 0.8)
    dout[(g == 0).all(1)] = 0
    v = vol if stride == 1 else np.stack([vol, vol, vol], 1).astype(np.int32)
    fw = [sparse_pm1(64, 32, rng), None, sparse_pm1(16, 64, rng)]
    check_field(oracle, hp, dout, tern((n, 32), rng, 0.8), fw, pts, v, stride, f"run layouts stride={stride}")


def test_shade_field_bwd_scatter_run_layouts(oracle, hash_params):
    hp = hash_params
    pts, vol, g, _ = layout(oracle, hp)
    n = pts.shape[0]
    rng = np.random.default_rng(23)
    op = exact_operands(n, rng, dead=(g == 0).all(1))
    anchors = np.stack([vol, vol, vol], 1).astype(np.int32)
    cam = (np.arange(n) // 13 % N_EMB).astype(np.int32)
    check_shade(oracle, hp, op, pts, anchors, cam, run_shade(hp, op, pts, anchors, cam), "run layouts")
