"""The packed-layout tensor-core forwards (f2b_mlp_fwd, f2b_mlp_fwd_f32, f2b_field_shade_fwd, f2b_shader_mlp_rgb_fwd, all on
mlp_fwd_tc_kernel; f2b_field_fwd, the hash encode fused in front of the field MLP) and the dtype casts (f2b_cast_f32_to_f16,
f2b_cast_f16_to_f32, f2b_table_to_half) against references that run no project kernel: torch float64 for the MLPs, the
epilogues and the encode, ATen's own conversions for the casts.

Sizes.  launch_fwd runs min(tiles, SMs x per_sm) CTAs of 128 rows, per_sm from the occupancy calculator.  Shared memory alone
allows 5 CTAs per SM for NH = 0 (TcSmem<0>::BYTES = 39,936) and 3 for NH = 1 (64,512).  ptxas -v (CUDA 12.9, sm_90a) reports
102 registers for the NH = 0 plain kernel (4 CTAs of 128 threads per SM), 90 for the NH = 0 EPI_SHADE kernel (5) and 152 for
both NH = 1 kernels (3), so registers bind the plain NH = 0 kernel only and every resident count is at most the shared-memory
bound B.  The tile counts B SMs + 1 (some CTA gets a second tile), 2 B SMs + 1 (some CTA gets a third, which reuses ring
slot 0) and (3 B + 1) SMs + 5 (every CTA gets at least three) hold for any resident count up to B; 8192 tiles are ~1 M rows.
f2b_field_fwd runs SMs x 4 CTAs (kFieldDefaultMinB, 123 / 128 registers fit 4): B = 4 there.  SMs comes from the device.  Every
size is 77 rows short of whole tiles, and n = 1, 127, 128, 129 are run too.

Buffers.  Every per-sample input is the first n rows of a buffer with a 300-row NaN tail (a valid camera / volume id for
integers); every output starts NaN with the same tail, which must still be NaN after the call, and no valid row may hold NaN.
hidden_save of NH = 1 is [2, n, 64] with the tail after the second layer: a first-layer row written past n lands in the second
layer's rows, which the exact and per-element checks then see.

Exact-operand regime (the one test_gpu_bwd_reference.py uses): weight matrices with at most two +-1 per row and per column,
inputs in {-1, 0, 1} x 2^e for e in -3..3, appearance embeddings in {0, +-2^-1 .. +-2^-4}.  Every activation and output is a
multiple of 2^-4 below 2^6 (at most eight terms of 2^3 for NH = 1), so every fp32 sum is exact in any order and every fp16
rounding is the identity (the reference asserts both).  The kernels must then equal the float64 forward bit for bit.

Generic operands (seeded fp16 inputs, xavier-uniform weights), each layer on the kernel's own saved input to it:
    |got - exact| <= delta + 1/2 ulp_fp16(|exact| + delta),    delta = 4 K 2^-24 sum_k |x_k w_k|
where exact = relu?(x W^T) in float64 and K is the layer's input width.  Derivation of delta: products of fp16 operands are
exact in fp32 (22 significant bits); the tensor core adds them in k16 blocks aligned to the block's largest exponent, and the
published measurements of NVIDIA tensor cores (Fasi, Higham, Mikaitis, Pranesh 2021, and later work on Hopper) find the
alignment and the normalisation truncate instead of rounding.  So each of the K products and each block's accumulator input
loses less than one fp32 ulp (2^-23) of a magnitude <= sum|terms|, and each of the K/16 normalisations another:
(K + 2 K / 16) 2^-23 S <= 2 K 2^-23 S = 4 K 2^-24 S.  The bar rests on that published behaviour, not on a figure measured here.
The ReLU does not widen an error; the fp16 rounding of the fp32 value adds half an fp16 ulp at that value (2^-25 below 2^-14).
A dropped k-slice, a wrong weight chunk or a stale ring slot moves an element by the size of whole terms, far above the bar.

Epilogues.
  * SH4 (mlp_in[:, 16:32]) against the float64 polynomial of the fp32 dirs: each component is at most six fp32 roundings
    (constant, products, one FMA) of quantities bounded by S = the component's sum of |terms|, so delta = 8 x 2^-24 S, then half
    an fp16 ulp as above.  Below 1 fp16 ulp wherever |value| >= 2^-9.
  * colour: rgb against (1 + 2e-3) sigmoid(raw) - 1e-3 in float64 on the kernel's own raw, |err| <= 9 x 2^-24.  shade_act is
    fsub(fdiv(c, fadd(1, expf(-o))), 1e-3f): c = fp32(1.002) (2^-24 relative), expf (2 fp32 ulp, the CUDA Programming Guide's
    maximum error, not measured here), fadd and fdiv (1/2 ulp each) give <= 1.002 x 7 x 2^-24 on the quotient (<= 1.002);
    1e-3f is off by < 2^-34 and the final fsub rounds by <= 2^-24: 8.02 x 2^-24 < 9 x 2^-24.
  * logit = out[:, 0] widened; mlp_in[:, 0:16] = fp16([1, out[1:16]] + app_emb[cam]) exactly in the exact regime.
f2b_field_fwd: feat_save against a float64 encode with the device's level scales (f2b_hash_level_scales).  The cell and the
fractions come from the kernel's fp32 arithmetic restated exactly ((p + 1) / 2, a correctly rounded fp32 FMA, floor); the
corner weights and the blend are float64.  The kernel rounds each weight twice and blends with one fp32 FMA chain of eight
terms: delta = (2 + 8 + 1) 2^-24 sum|w f|, then half an fp16 ulp.  The MLP part is checked per element on feat_save as above.

No bar is relative to a tensor's maximum."""
import numpy as np
import pytest
import torch

from test_gpu_bwd_reference import BT, PAD, f16_exact, out_rows, params16, prefix, ray_layout, sparse_pm1, sum_exact, tail_untouched, tern
from test_gpu_parity import N, T

gpu = pytest.mark.gpu

SMEM_BOUND = {0: 5, 1: 3}     # resident CTAs per SM that shared memory allows (TcSmem<0>, TcSmem<1>)
FIELD_CTAS = 4                # f2b_field_fwd: SMs x kFieldDefaultMinB CTAs
SIZES = ["1", "127", "128", "129", "2nd", "3rd", "all3", "1M"]
N_EMB = 9
USED_EMB = [0, 2, 3, 5, N_EMB - 1]                    # the other rows of app_emb are NaN
U = 2.0 ** -24
COLOUR_BAR = 9 * U
SH_C = (0.28209479177387814, 0.48860251190291987, 1.0925484305920792, 0.94617469575755997, 0.31539156525251999,
        0.54627421529603959, 0.59004358992664352, 2.8906114426405538, 0.45704579946446572, 0.3731763325901154,
        1.4453057213202769)
F64 = torch.float64


def n_rows(size, bound):
    """rows for a size name; `bound` = the most CTAs per SM the kernel can have resident"""
    if size.isdigit():
        return int(size)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = {"2nd": bound * sms + 1, "3rd": 2 * bound * sms + 1, "all3": (3 * bound + 1) * sms + 5, "1M": 8192}[size]
    return BT * tiles - 77


# ------------------------------------------------------------------------------------------------ float64 references ----
def r16(t):
    return t.to(torch.float16).to(F64)


def ulp16(a):
    """fp16 ulp at |a| (float64): 2^(floor(log2|a|) - 10), 2^-24 in the subnormal range"""
    _, e = torch.frexp(a.abs().clamp_min(2.0 ** -14))
    return torch.ldexp(torch.ones_like(a), e - 11)


def f16_bar(exact, delta):
    """bar of an fp16 result whose fp32 value is within delta of exact"""
    return delta + 0.5 * ulp16(exact.abs() + delta)


def acc_delta(sum_abs, k):
    """fp32 tensor-core accumulation bound of a K-wide dot product (derivation in the module docstring)"""
    return 4 * k * U * sum_abs


def wt(w, dev):
    return None if w is None else torch.as_tensor(np.asarray(w, np.float64), dtype=F64, device=dev)


def mlp_ref(x, ws, exact=False):
    """float64 forward: relu(x W0^T) [-> relu(. Wh^T)] -> . Wout^T, fp16 rounding at each layer boundary, as the kernel stores
    them.  ws = [W0, Wh | None, Wout] (rows = outputs).  -> out, [H0, H1 | None].  exact: assert every rounding is the
    identity and every sum exact in fp32 (the exact-operand regime)."""
    W0, Wh, Wo = (wt(w, x.device) for w in ws)
    pre = [(x @ W0.T).clamp_min(0)]
    sums = [x.abs() @ W0.abs().T]
    h = [r16(pre[0])]
    if Wh is not None:
        pre.append((h[0] @ Wh.T).clamp_min(0))
        sums.append(h[0].abs() @ Wh.abs().T)
        h.append(r16(pre[1]))
    pre.append(h[-1] @ Wo.T)
    sums.append(h[-1].abs() @ Wo.abs().T)
    if exact:
        for t, what in zip(pre, ("H0", "H1", "out") if Wh is not None else ("H0", "out")):
            f16_exact(t, what)
        sum_exact(torch.cat([s.ravel() for s in sums]), 2.0 ** -3, "forward")
    return r16(pre[-1]), h + ([None] if Wh is None else [])


def layer_ref(x, W, relu):
    """one layer on its input rows x (float64): exact relu?(x W^T) and its per-element bar"""
    z = x @ W.T
    if relu:
        z = z.clamp_min(0)
    return z, f16_bar(z, acc_delta(x.abs() @ W.abs().T, x.shape[1]))


def sh4_ref(d):
    """degree-4 real SH of dirs [n,3] (float64, tiny-cuda-nn ordering) -> values [n,16], sum of |terms| per component"""
    c0, c1, c2, c3, c4, c5, c6, c7, c8, c9, c10 = SH_C
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    ax, ay, az = x.abs(), y.abs(), z.abs()
    x2, y2, z2 = x * x, y * y, z * z
    one = torch.ones_like(x)
    v = [c0 * one, -c1 * y, c1 * z, -c1 * x, c2 * x * y, -c2 * y * z, c3 * z2 - c4, -c2 * x * z, c5 * x2 - c5 * y2,
         c6 * y * (-3 * x2 + y2), c7 * x * y * z, c8 * y * (1 - 5 * z2), c9 * z * (5 * z2 - 3), c8 * x * (1 - 5 * z2),
         c10 * z * (x2 - y2), c6 * x * (-x2 + 3 * y2)]
    s = [c0 * one, c1 * ay, c1 * az, c1 * ax, c2 * ax * ay, c2 * ay * az, c3 * z2 + c4, c2 * ax * az, c5 * (x2 + y2),
         c6 * ay * (3 * x2 + y2), c7 * ax * ay * az, c8 * ay * (1 + 5 * z2), c9 * az * (5 * z2 + 3), c8 * ax * (1 + 5 * z2),
         c10 * az * (x2 + y2), c6 * ax * (x2 + 3 * y2)]
    return torch.stack(v, 1), torch.stack(s, 1)


def sh4_bar(d):
    v, s = sh4_ref(d)
    return v, f16_bar(v, 8 * U * s)


def colour_ref(raw):
    return (1 + 2e-3) / (1 + torch.exp(-raw)) - 1e-3


def fma32(a, b, c):
    """fp32 fma(a, b, c) correctly rounded, from float32 tensors (-> float32).  The product is exact in float64 (24 + 24 bits);
    TwoSum keeps the float64 sum's rounding error e.  Rounding the float64 sum s to fp32 can differ from rounding the exact
    s + e only when s lies on an fp32 midpoint, and then e decides the side."""
    p = a.to(F64) * b.to(F64)
    c = c.to(F64)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.to(torch.float32)
    other = torch.nextafter(r, torch.where(s > r.to(F64), torch.full_like(r, np.inf), torch.full_like(r, -np.inf)))
    mid = (s != r.to(F64)) & (2 * s == r.to(F64) + other.to(F64))
    # on a midpoint the tie went to r; the exact value is on other's side when e points that way
    away = mid & (e != 0) & ((e > 0) == (other > r))
    return torch.where(away, other, r)


def encode_ref(table16, prim, bias, n_volumes, local_size, scales, pts, vol):
    """float64 16-level anchored hash encode (tensors on one device: table16 [pool,2] f16, prim [16,V,3] i32, bias [16*V,3] f32,
    scales [16] f32, pts [n,3] f32, vol [n] i32) -> feat [n,32] float64, bar [n,32].  Cells and fractions restate the kernel's
    fp32 arithmetic exactly; weights and blend are float64 (bar: module docstring)."""
    dev = pts.device
    tab = table16.reshape(-1).to(F64)
    x = (pts + torch.ones((), device=dev)) * torch.full((), 0.5, device=dev)        # fp32, as the kernel rounds it
    v = vol.long()
    feat = torch.empty((pts.shape[0], 32), dtype=F64, device=dev)
    bar = torch.empty_like(feat)
    mask = local_size - 1
    assert local_size & mask == 0
    for l in range(16):
        pr = prim.reshape(16, n_volumes, 3)[l].long()[v] & 0xFFFFFFFF
        bi = bias.reshape(16, n_volumes, 3)[l][v]
        px = fma32(x, scales[l].expand_as(x), bi)
        fx = torch.floor(px)
        ix = fx.long()
        frac = (px - fx).to(F64)                                                     # exact in fp32
        h0 = (ix * pr) & 0xFFFFFFFF
        h1 = (h0 + pr) & 0xFFFFFFFF
        acc = torch.zeros((pts.shape[0], 2), dtype=F64, device=dev)
        sabs = torch.zeros_like(acc)
        for k in range(8):
            bx, by, bz = (k >> 2) & 1, (k >> 1) & 1, k & 1                         # z fastest, as hash.cuh's corners()
            idx = ((h1[:, 0] if bx else h0[:, 0]) ^ (h1[:, 1] if by else h0[:, 1]) ^ (h1[:, 2] if bz else h0[:, 2])) & mask
            w = torch.ones_like(frac[:, 0])
            for j, bit in enumerate((bx, by, bz)):
                w = w * (frac[:, j] if bit else 1 - frac[:, j])
            f = torch.stack([tab[l * local_size + 2 * idx], tab[l * local_size + 2 * idx + 1]], 1)
            acc += w[:, None] * f
            sabs += (w[:, None] * f).abs()
        feat[:, 2 * l: 2 * l + 2] = acc
        bar[:, 2 * l: 2 * l + 2] = f16_bar(acc, 11 * U * sabs)
    return feat, bar


# ------------------------------------------------------------------------------------------------------------ inputs ----
def pow2_tern(shape, rng):
    """{-1, 0, 1} x 2^e, e in -3..3"""
    return tern(shape, rng) * 2.0 ** rng.integers(-3, 4, shape)


def exact_ws(nh, rng):
    return [sparse_pm1(64, 32, rng), sparse_pm1(64, 64, rng) if nh else None, sparse_pm1(16, 64, rng)]


def xavier(rows, cols, rng):
    b = np.sqrt(6.0 / (rows + cols))
    return rng.uniform(-b, b, (rows, cols)).astype(np.float16).astype(np.float64)


def generic_ws(nh, rng):
    return [xavier(64, 32, rng), xavier(64, 64, rng) if nh else None, xavier(16, 64, rng)]


def unit_dirs(n, rng):
    d = rng.standard_normal((n, 3))
    return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def camera_ids(n, rng):
    """runs of 1..40 samples (so ids change inside every tile) over the used rows; the last sample has id N_EMB - 1"""
    lens = rng.integers(1, 41, n)
    ids = np.repeat(rng.choice(USED_EMB, lens.shape[0]), lens)[:n].astype(np.int32)
    ids[-1] = N_EMB - 1
    return ids


def exact_emb(rng):
    e = rng.choice([-1.0, 1.0], (N_EMB, 16)) * 2.0 ** -rng.integers(1, 5, (N_EMB, 16))
    e[rng.random((N_EMB, 16)) < 0.2] = 0
    unused = np.setdiff1d(np.arange(N_EMB), USED_EMB)
    e[unused] = np.nan
    return e.astype(np.float32)


def f32_rows(n, cols=None):
    """NaN-filled fp32 output rows with a PAD-row tail"""
    return torch.full((n + PAD,) if cols is None else (n + PAD, cols), float("nan"), dtype=torch.float32, device="cuda")


def rows_ok(buf, n, what):
    """rows [n:] still NaN, rows [:n] free of NaN"""
    tail_untouched(buf, n, what)
    bad = torch.isnan(buf[:n].float())
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} NaN in the valid rows, first at {tuple(bad.nonzero()[0].tolist())}"


def eq(got, ref, what):
    got = torch.as_tensor(got).to(ref.device, F64)
    bad = ~(got == ref)
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {bad.numel()} differ; first at {tuple(bad.nonzero()[0].tolist())}: "
                                 f"got {float(got[bad][0])}, exact {float(ref[bad][0])}")


def within(got, exact, bar, what):
    got = torch.as_tensor(got).to(exact.device, F64)
    err = (got - exact).abs()
    bad = ~(err <= bar)                                                  # NaN is bad
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        worst = float(torch.nan_to_num(err[bad] / bar[bad], nan=np.inf).max())
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} beyond the bar (worst {worst:.3g} x bar); first at {i}: "
                             f"got {float(got[i])}, exact {float(exact[i])}, bar {float(bar[i]):.3e}")


def dev64(a):
    return torch.as_tensor(np.asarray(a, np.float64), dtype=F64, device="cuda")


# ------------------------------------------------------------------------------------------------------------ kernels ----
def run_mlp(x16, ws, nh, n, mode):
    """mode "f32" / "f16" / "both": f2b_mlp_fwd_f32 with those outputs; "fwd": f2b_mlp_fwd.  Every call saves the hidden
    activations.  -> dict of whole buffers (tails included) and the hidden rows per layer"""
    from f2nerf_b200._lib import call, stream
    o = dict(out32=f32_rows(n, 16) if mode in ("f32", "both") else None,
             out16=out_rows(n, 16) if mode in ("f16", "both", "fwd") else None, hid=out_rows((nh + 1) * n, 64))
    v = {k: (b[: (nh + 1) * n] if k == "hid" else b[:n]) if b is not None else None for k, b in o.items()}
    if mode == "fwd":
        call("f2b_mlp_fwd", x16, T(params16(ws)), nh, n, v["out16"], v["hid"], stream())
    else:
        call("f2b_mlp_fwd_f32", x16, T(params16(ws)), nh, n, v["out32"], v["out16"], v["hid"], stream())
    torch.cuda.synchronize()
    for k, b in o.items():
        if b is not None:
            rows_ok(b, (nh + 1) * n if k == "hid" else n, f"{k} nh={nh} n={n} mode={mode}")
    o["layers"] = [o["hid"][l * n:(l + 1) * n] for l in range(nh + 1)]
    return o


def run_field_shade(x16, ws, dirs, emb, ids, n):
    from f2nerf_b200._lib import call, stream
    nan = np.float32("nan")
    o = dict(logit=f32_rows(n), mlp_in=out_rows(n, 32), hid=out_rows(n, 64))
    call("f2b_field_shade_fwd", x16, T(params16(ws)), prefix(dirs, nan), T(emb) if emb is not None else None,
         prefix(ids, N_EMB - 1) if emb is not None else None, n, o["logit"][:n], o["mlp_in"][:n], o["hid"][:n], stream())
    torch.cuda.synchronize()
    for k, b in o.items():
        rows_ok(b, n, f"{k} n={n} emb={emb is not None}")
    return o


def run_shader(x16, ws, n):
    from f2nerf_b200._lib import call, stream
    o = dict(raw=out_rows(n, 16), rgb=f32_rows(n, 3), hid=out_rows(2 * n, 64))
    call("f2b_shader_mlp_rgb_fwd", x16, T(params16(ws)), n, o["raw"][:n], o["rgb"][:n], o["hid"][: 2 * n], stream())
    torch.cuda.synchronize()
    for k, b in o.items():
        rows_ok(b, 2 * n if k == "hid" else n, f"{k} n={n}")
    o["layers"] = [o["hid"][:n], o["hid"][n: 2 * n]]
    return o


def check_sh(mlp_in, dirs, what):
    v, bar = sh4_bar(dev64(dirs))
    within(mlp_in[:, 16:32], v, bar, f"SH4 {what}")


# ------------------------------------------------------------------------------------------------ exact-operand tests ----
@gpu
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("nh", [0, 1])
def test_mlp_fwd_exact(nh, size):
    """f2b_mlp_fwd_f32 in all three output modes and f2b_mlp_fwd: out, widened out_f32 and both hidden layers bit for bit"""
    n = n_rows(size, SMEM_BOUND[nh])
    rng = np.random.default_rng(100 + 10 * nh + SIZES.index(size))
    x, ws = pow2_tern((n, 32), rng), exact_ws(nh, rng)
    out, hid = mlp_ref(dev64(x), ws, exact=True)
    x16 = prefix(x.astype(np.float16), np.float16("nan"))
    for mode in ("f32", "f16", "both", "fwd"):
        o = run_mlp(x16, ws, nh, n, mode)
        tag = f"nh={nh} n={n} mode={mode}"
        for l in range(nh + 1):
            eq(o["layers"][l], hid[l], f"hidden {l} {tag}")
        if o["out32"] is not None:
            eq(o["out32"][:n], out, f"out_f32 {tag}")
        if o["out16"] is not None:
            eq(o["out16"][:n], out, f"out {tag}")


@gpu
@pytest.mark.parametrize("emb", [False, True])
@pytest.mark.parametrize("size", SIZES)
def test_field_shade_fwd_exact(size, emb):
    """logit, mlp_in[:, 0:16] (with the appearance-embedding add) and the hidden layer bit for bit; SH4 within its bar"""
    n = n_rows(size, SMEM_BOUND[0])
    rng = np.random.default_rng(200 + 2 * SIZES.index(size) + emb)
    x, ws, dirs = pow2_tern((n, 32), rng), exact_ws(0, rng), unit_dirs(n, rng)
    app, ids = (exact_emb(rng), camera_ids(n, rng)) if emb else (None, None)
    out, hid = mlp_ref(dev64(x), ws, exact=True)
    lead = out[:, :16].clone()
    lead[:, 0] = 1
    if emb:
        lead += dev64(app)[torch.as_tensor(ids, device="cuda").long()]
        f16_exact(lead, "mlp_in[:, 0:16]")
    o = run_field_shade(prefix(x.astype(np.float16), np.float16("nan")), ws, dirs, app, ids, n)
    tag = f"n={n} emb={emb}"
    eq(o["hid"][:n], hid[0], f"hidden {tag}")
    eq(o["logit"][:n], out[:, 0], f"logit {tag}")
    eq(o["mlp_in"][:n, :16], lead, f"mlp_in[:, 0:16] {tag}")
    check_sh(o["mlp_in"][:n], dirs, tag)


@gpu
@pytest.mark.parametrize("size", SIZES)
def test_shader_mlp_rgb_fwd_exact(size):
    """raw and both hidden layers bit for bit; rgb against the float64 activation of raw"""
    n = n_rows(size, SMEM_BOUND[1])
    rng = np.random.default_rng(300 + SIZES.index(size))
    x, ws = pow2_tern((n, 32), rng), exact_ws(1, rng)
    out, hid = mlp_ref(dev64(x), ws, exact=True)
    o = run_shader(prefix(x.astype(np.float16), np.float16("nan")), ws, n)
    for l in range(2):
        eq(o["layers"][l], hid[l], f"hidden {l} n={n}")
    eq(o["raw"][:n], out, f"raw n={n}")
    within(o["rgb"][:n], colour_ref(out[:, :3]), torch.full_like(out[:, :3], COLOUR_BAR), f"rgb n={n}")


# ----------------------------------------------------------------------------------------------- generic operands ----
def check_mlp_layers(layers, out, x, ws, tag):
    """each layer per element on the kernel's own input to it; out: the output layer's fp16 values (float64)"""
    inp = x
    for l, W in enumerate(w for w in ws[:2] if w is not None):
        z, bar = layer_ref(inp, wt(W, x.device), True)
        within(layers[l], z, bar, f"hidden {l} {tag}")
        inp = layers[l].to(x.device, F64)
    z, bar = layer_ref(inp, wt(ws[2], x.device), False)
    within(out, z[:, : out.shape[1]], bar[:, : out.shape[1]], f"out {tag}")


@gpu
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("nh", [0, 1])
def test_mlp_fwd_generic(nh, size):
    n = n_rows(size, SMEM_BOUND[nh])
    rng = np.random.default_rng(400 + 10 * nh + SIZES.index(size))
    x = (rng.standard_normal((n, 32)) * 0.5).astype(np.float16)
    ws = generic_ws(nh, rng)
    x16 = prefix(x, np.float16("nan"))
    o = run_mlp(x16, ws, nh, n, "both")
    tag = f"nh={nh} n={n}"
    check_mlp_layers(o["layers"], o["out16"][:n].to(F64), dev64(x), ws, tag)
    eq(o["out32"][:n], o["out16"][:n].to(F64), f"out_f32 == widened out {tag}")
    for mode in ("f32", "f16", "fwd"):                                 # the other output modes: the same values
        m = run_mlp(x16, ws, nh, n, mode)
        eq(m["out32"][:n] if mode == "f32" else m["out16"][:n], o["out16"][:n].to(F64), f"out {tag} mode={mode}")
        eq(m["hid"][: (nh + 1) * n], o["hid"][: (nh + 1) * n].to(F64), f"hidden {tag} mode={mode}")


@gpu
@pytest.mark.parametrize("size", SIZES)
def test_field_shade_fwd_generic(size):
    n = n_rows(size, SMEM_BOUND[0])
    rng = np.random.default_rng(500 + SIZES.index(size))
    x = (rng.standard_normal((n, 32)) * 0.5).astype(np.float16)
    ws, dirs = generic_ws(0, rng), unit_dirs(n, rng)
    o = run_field_shade(prefix(x, np.float16("nan")), ws, dirs, None, None, n)
    lead = o["mlp_in"][:n, :16].to(F64)
    assert bool((lead[:, 0] == 1).all()), "mlp_in[:, 0] != 1"
    lead[:, 0] = o["logit"][:n].to(F64)
    check_mlp_layers([o["hid"][:n]], lead, dev64(x), ws, f"n={n}")
    eq(o["logit"][:n], o["logit"][:n].half().to(F64), f"logit is an fp16 value n={n}")
    check_sh(o["mlp_in"][:n], dirs, f"n={n}")


@gpu
@pytest.mark.parametrize("size", SIZES)
def test_shader_mlp_rgb_fwd_generic(size):
    n = n_rows(size, SMEM_BOUND[1])
    rng = np.random.default_rng(600 + SIZES.index(size))
    x = (rng.standard_normal((n, 32)) * 0.5).astype(np.float16)
    ws = generic_ws(1, rng)
    ws[2] = ws[2] * 4                                                    # raw spreads over the sigmoid's range
    o = run_shader(prefix(x, np.float16("nan")), ws, n)
    raw = o["raw"][:n].to(F64)
    check_mlp_layers(o["layers"], raw, dev64(x), ws, f"n={n}")
    within(o["rgb"][:n], colour_ref(raw[:, :3]), torch.full_like(raw[:, :3], COLOUR_BAR), f"rgb n={n}")


# ------------------------------------------------------------------------------------------------ packed field_fwd ----
@gpu
@pytest.mark.parametrize("size,stride", [(s, 3) for s in SIZES] + [("3rd", 1), ("1M", 1)])
def test_field_fwd(hash_params, size, stride):
    """encode + field MLP: feat_save against the float64 encode, the hidden layer and out per element on the kernel's own
    feat_save / hidden rows; logit_only == out[:, 0] and the same feat_save, bit for bit"""
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    hp = hash_params
    n = n_rows(size, FIELD_CTAS)
    rng = np.random.default_rng(700 + 2 * SIZES.index(size) + stride)
    pts, anchors, _ = ray_layout(max(n, 4096), hp["V"], rng)             # (ray_layout wants a few dozen rays)
    pts, anchors = pts[:n], anchors[:n]
    vol = anchors if stride == 3 else np.ascontiguousarray(anchors[:, 0])
    ws = generic_ws(0, rng)
    ws[0] = ws[0] * 4                                                    # features are ~0.1: hidden rows well above 0
    nan = np.float32("nan")
    args = (T(hp["table"]), T(hp["prim"]), T(hp["bias"]), hp["V"], hp["local_size"], T(params16(ws)), prefix(pts, nan),
            prefix(vol, hp["V"] - 1), stride, n)
    out, feat, hid = f32_rows(n, 16), out_rows(n, 32), out_rows(n, 64)
    call("f2b_field_fwd", *args, 0, out[:n], feat[:n], hid[:n], stream())
    logit, feat2, hid2 = f32_rows(n), out_rows(n, 32), out_rows(n, 64)
    call("f2b_field_fwd", *args, 1, logit[:n], feat2[:n], hid2[:n], stream())
    torch.cuda.synchronize()
    tag = f"n={n} stride={stride}"
    for b, what in ((out, "out"), (feat, "feat_save"), (hid, "hidden_save"), (logit, "logit_only"), (feat2, "logit_only feat_save")):
        rows_ok(b, n, f"{what} {tag}")
    assert bool(torch.isnan(hid2.float()).all()), f"logit_only wrote hidden_save {tag}"
    scales = ops.hash_level_scales().cuda()
    ref, bar = encode_ref(T(hp["table"]), T(hp["prim"]), T(hp["bias"]), hp["V"], hp["local_size"], scales, T(pts),
                          T(np.ascontiguousarray(anchors[:, 0])))
    within(feat[:n], ref, bar, f"feat_save {tag}")
    check_mlp_layers([hid[:n]], out[:n].to(F64), feat[:n].to(F64), ws, tag)
    eq(out[:n], out[:n].half().to(F64), f"out is fp16-rounded {tag}")
    eq(logit[:n], out[:n, 0].to(F64), f"logit_only {tag}")
    eq(feat2[:n], feat[:n].to(F64), f"logit_only feat_save {tag}")


# ---------------------------------------------------------------------------------------------------------- casts ----
def special_f32(rng, n):
    """fp32 values: +-0, NaN, +-inf, fp16 overflow (65504 stays, 65520 and beyond round to inf), fp16 subnormals and their
    ties, the fp16 normal/subnormal edge, then log-uniform magnitudes over 2^-30 .. 2^20 of either sign"""
    edge = [0.0, -0.0, np.nan, np.inf, -np.inf, 65504.0, 65519.99, 65520.0, -65520.0, 70000.0, 1e6, -3.4e38,
            2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25, 2.0 ** -26, -2.0 ** -24, 2.0 ** -14, 2.0 ** -14 - 2.0 ** -25, 1e-7, 5.9e-8,
            1.0, -1.0, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11]
    v = rng.choice([-1.0, 1.0], n) * 2.0 ** rng.uniform(-30, 20, n)
    v[: min(n, len(edge))] = edge[: min(n, len(edge))]
    return rng.permutation(v).astype(np.float32) if n > len(edge) else v.astype(np.float32)


def same_bits(got, ref, what):
    """bit-equal, except that any NaN matches any NaN"""
    g, r = got.cpu(), ref.cpu()
    ok = (g.view(torch.int16 if g.dtype == torch.float16 else torch.int32) == r.view(torch.int16 if r.dtype == torch.float16 else torch.int32)) \
        | (torch.isnan(g) & torch.isnan(r))
    assert bool(ok.all()), (f"{what}: {int((~ok).sum())} of {ok.numel()} differ; first at {int((~ok).nonzero()[0])}: "
                            f"got {float(g[~ok][0])!r}, ATen {float(r[~ok][0])!r}")


CAST_N = [1, 3, 4, 5, 255, 1029, (1 << 20) + 3]


@gpu
@pytest.mark.parametrize("scale", [1.0, 2.0 ** -7, 16.0])
@pytest.mark.parametrize("n", CAST_N)
def test_cast_f32_to_f16(n, scale):
    from f2nerf_b200._lib import call, stream
    v = special_f32(np.random.default_rng(n), n)
    out = out_rows(n, 1).view(-1)
    call("f2b_cast_f32_to_f16", prefix(v, np.float32("nan")), out[:n], n, scale, stream())
    torch.cuda.synchronize()
    tail_untouched(out, n, f"cast_f32_to_f16 n={n}")
    ref = (torch.from_numpy(v) * torch.tensor(scale, dtype=torch.float32)).to(torch.float16)
    same_bits(out[:n], ref, f"cast_f32_to_f16 n={n} scale={scale}")


@gpu
@pytest.mark.parametrize("scale", [1.0, 2.0 ** -7])
@pytest.mark.parametrize("n", CAST_N + [65536 + 3])
def test_cast_f16_to_f32(n, scale):
    """every fp16 bit pattern (subnormals, +-0, +-inf, NaNs) in a seeded order, repeated up to n"""
    from f2nerf_b200._lib import call, stream
    bits = np.random.default_rng(n).permutation(np.arange(65536, dtype=np.uint32).astype(np.uint16))
    v = np.resize(bits, n).view(np.float16)
    out = f32_rows(n)
    call("f2b_cast_f16_to_f32", prefix(v, np.float16("nan")), out[:n], n, scale, stream())
    torch.cuda.synchronize()
    tail_untouched(out, n, f"cast_f16_to_f32 n={n}")
    ref = torch.from_numpy(v.copy()).to(torch.float32) * torch.tensor(scale, dtype=torch.float32)
    same_bits(out[:n], ref, f"cast_f16_to_f32 n={n} scale={scale}")


@gpu
@pytest.mark.parametrize("live", [1, 4097, (1 << 19) * 2 - 6])
def test_table_to_half(live):
    """the table shadow: the live prefix of a [pool, 2] fp32 table converted, everything past it untouched"""
    from f2nerf_b200 import ops
    from f2nerf_b200._lib import call, stream
    pool = 1 << 19
    t = special_f32(np.random.default_rng(live), 2 * pool).reshape(pool, 2)
    out = torch.full((2 * pool + PAD,), float("nan"), dtype=torch.float16, device="cuda")
    call("f2b_table_to_half", T(t), out[:live], live, stream())
    torch.cuda.synchronize()
    tail_untouched(out, live, f"table_to_half live={live}")
    same_bits(out[:live], torch.from_numpy(t.reshape(-1)[:live].copy()).to(torch.float16), f"table_to_half live={live}")
    whole = ops.table_to_half(T(t))
    same_bits(whole.view(-1), torch.from_numpy(t.reshape(-1).copy()).to(torch.float16), "table_to_half whole table")


# ------------------------------------------------------------------------- CPU self-checks of the float64 references ----
@pytest.mark.parametrize("nh", [0, 1])
def test_reference_exact_regime_matches_oracle(oracle, nh):
    """the exact-regime float64 forward == the CPU oracle's fp32 forward on the same operands, bit for bit"""
    rng = np.random.default_rng(11 + nh)
    n = 3000
    x, ws = pow2_tern((n, 32), rng), exact_ws(nh, rng)
    out, hid = mlp_ref(torch.as_tensor(x), ws, exact=True)
    o_out, o_hid = oracle.mlp_fwd(x.astype(np.float16), params16(ws), nh, save_hidden=True)
    np.testing.assert_array_equal(o_out.astype(np.float64), out.numpy())
    for l in range(nh + 1):
        np.testing.assert_array_equal(o_hid[l].astype(np.float64), hid[l].numpy())


@pytest.mark.parametrize("nh", [0, 1])
def test_reference_generic_bars_hold_for_oracle(oracle, nh):
    """the per-element bars hold for the oracle's serial fp32 forward, and are not loose: with one k16 slice of the input
    dropped, most rows leave the layer-0 bar"""
    rng = np.random.default_rng(21 + nh)
    n = 4000
    x = (rng.standard_normal((n, 32)) * 0.5).astype(np.float16)
    ws = generic_ws(nh, rng)
    o_out, o_hid = oracle.mlp_fwd(x, params16(ws), nh, save_hidden=True)
    xt = torch.as_tensor(x.astype(np.float64))
    hid = [torch.as_tensor(h.astype(np.float64)) for h in o_hid]
    check_mlp_layers(hid, torch.as_tensor(o_out.astype(np.float64)), xt, ws, f"oracle nh={nh}")
    W0 = torch.as_tensor(ws[0])
    z, bar = layer_ref(xt, W0, True)
    cut = xt.clone()
    cut[:, 16:] = 0
    moved = ((r16((cut @ W0.T).clamp_min(0)) - z).abs() > bar).any(1)
    assert float(moved.double().mean()) > 0.9


def test_reference_sh4_and_colour(oracle):
    """SH4: the oracle's fp32 polynomial (same operation sequence as the kernel) within the fp32 part of the bar, its fp16
    rounding within the whole bar; colour: the oracle's activation within COLOUR_BAR"""
    rng = np.random.default_rng(31)
    d = unit_dirs(20000, rng)
    d[:6] = [[1, 0, 0], [0, -1, 0], [0, 0, 1], [0.6, 0.8, 0], [0, 0.6, -0.8], [0.48, 0.6, 0.64]]
    v, s = sh4_ref(torch.as_tensor(d.astype(np.float64)))
    o = torch.as_tensor(oracle.sh4(d).astype(np.float64))
    assert bool(((o - v).abs() <= 8 * U * s).all())
    v, bar = sh4_bar(torch.as_tensor(d.astype(np.float64)))
    assert bool(((o.half().double() - v).abs() <= bar).all())
    raw = (rng.standard_normal((20000, 16)) * 4).astype(np.float16)
    raw[:4, 0] = [0, -17, 12, np.float16(-0.0)]
    r = torch.as_tensor(raw[:, :3].astype(np.float64))
    assert bool(((torch.as_tensor(oracle.shader_act(raw).astype(np.float64)) - colour_ref(r)).abs() <= COLOUR_BAR).all())


def test_reference_encode_matches_oracle(oracle, hash_params):
    """the float64 encode holds the oracle's fp32 encode (the kernel's operation sequence) within its bar, on ray-like points
    and on points at the corners of the domain; fma32 is correctly rounded on random operands (exact rational arithmetic)"""
    from fractions import Fraction
    hp = hash_params
    rng = np.random.default_rng(41)
    pts, anchors, _ = ray_layout(5000, hp["V"], rng)
    pts[:8] = [[-1, -1, -1], [1, 1, 1], [-1, 1, -1], [0, 0, 0], [1, -1, 1], [0.5, -0.5, 0.25], [-1, 0, 1], [1, 1, -1]]
    vol = np.ascontiguousarray(anchors[:, 0])
    scales = oracle.level_scales()
    got = oracle.hash_fwd(hp["table"], hp["prim"], hp["bias"], hp["V"], hp["local_size"], scales, pts, vol, 1)
    ref, bar = encode_ref(torch.as_tensor(hp["table"]), torch.as_tensor(hp["prim"]), torch.as_tensor(hp["bias"]), hp["V"],
                          hp["local_size"], torch.as_tensor(scales), torch.as_tensor(pts), torch.as_tensor(vol))
    err = (torch.as_tensor(got.astype(np.float64)) - ref).abs()
    assert bool((err <= bar).all()), f"{int((err > bar).sum())} off, worst {float((err / bar).max()):.2f} x bar"

    def round32(q):
        """Fraction -> nearest fp32 (ties to even)"""
        if q == 0:
            return 0.0
        e = abs(q.numerator).bit_length() - abs(q.denominator).bit_length()
        while abs(q) >= Fraction(2) ** (e + 1):
            e += 1
        while abs(q) < Fraction(2) ** e:
            e -= 1
        step = Fraction(2) ** (e - 23)
        return float(round(q / step) * step)

    a = rng.uniform(0, 1, 3000).astype(np.float32) * (2.0 ** -rng.integers(0, 30, 3000)).astype(np.float32)
    b = rng.uniform(8, 1024, 3000).astype(np.float32)
    c = rng.uniform(100, 1100, 3000).astype(np.float32)
    r = fma32(torch.as_tensor(a), torch.as_tensor(b), torch.as_tensor(c)).numpy()
    want = np.array([round32(Fraction(float(p)) * Fraction(float(q)) + Fraction(float(s))) for p, q, s in zip(a, b, c)], np.float32)
    np.testing.assert_array_equal(r.view(np.uint32), want.view(np.uint32))
