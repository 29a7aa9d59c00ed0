"""The C++ operator-level drop-in (f2nerf_b200/shim/B200Ops.cpp: B200HashField::AnchoredQuery, B200Shader::Query) by gradient
magnitude, against float64 autograd, the Python operators and the reference's own operators.

``ref_driver_b200 --ops`` runs the two operators of this library inside the reference's program, ``ref_driver --ops`` the
reference's own (tiny-cuda-nn), each followed by (out * g).sum().backward() on inputs this test writes (oracle/ref_driver.cpp).
Gradients are compared by size, not only by direction: a loss-scale mistake (a missing / scale, a wrong grad_mul or cast scale)
multiplies a group by the scale and leaves every cosine unchanged.

Finite cases: 1, 129, 2 SMs 128 + 77 and 128 (12 SMs + 5) - 77 ray-like points (so every CTA of the saved-activation MLP
backward, at most 4 resident per SM, takes at least three 128-row tiles), each at field/shader loss scales 128 (the default),
1 and 1024.  Per case:
  * B200 against the float64 twin (tests/autograd_twin.py) pinned to its forward: the bars of test_autograd_twin_cpu per group
    (field MLP, shader MLP, shading input, table per level slab) and per table entry;
  * B200 against the Python operators on the same inputs: field output bit-identical, field gradients to fp32 atomic order;
    rgb against the float64 activation of the MLP's own fp16 output;
  * B200 against tiny-cuda-nn: forward at fp16 resolution, per-group gradient norm ratio, and the CUDA generator's state after
    each operator (the torch::rand that stands in for tcnn's output allocation).
Non-finite cases, where the reference arm's backward_nan_ and loss scales are the expected values: (i) an inf in one row of
dL/dout (field) or dL/drgb (shader); (ii) only dL/dinput overflows in fp16 while dL/dparams stay finite.
"""
import json
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import autograd_twin as AT
from test_autograd_twin_cpu import COS_BAR, REL_BAR, group_errors
from test_gpu_bwd_reference import ray_layout
from test_gpu_grad_autograd import ENTRY_BAR, hash_args
from test_gpu_parity import N, T
from workloads import diag_path, load_golden

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "ref_driver")
B200 = os.path.join(ROOT, "oracle", "_ref", "ref_driver_b200")
CONFIG = os.path.join(ROOT, "oracle", "ref_config_ngp_fox.yaml")
F64 = torch.float64
OPS_SEED = 52000                     # ref_driver.cpp kOpsSeed: the field operator's seed, the shader's is one more
SIZES = ("one", "ragged", "past_a_wave", "three_tiles")
SCALES = (128.0, 1.0, 1024.0)
NONFINITE = ("i_field", "i_shader", "ii_field", "ii_shader")
G_STD = 0.01                         # dL/dout and dL/drgb: N(0, G_STD^2); tcnn's fp16 dL/dparams stay finite at 1024 x 200k rows

# rgb = (1 + 2e-3) / (1 + expf(-raw)) - 1e-3 in fp32 (shader.cuh shade_act) against float64 on the same fp16 raw: expf is within
# 2 ulp (carried through 1 + e unchanged in relative terms), the add, the divide and the constant 1.002f each add 2^-24
# relative to a quotient of at most 1.002; the final subtraction rounds at half an ulp of a value below 1.002 (2^-24) and
# 1e-3f is 1e-3 within 2^-24 relative.  Derived, not measured.
ACT_BAR = 1.002 * (2 * 2. ** -23 + 3 * 2. ** -24) + 2. ** -24 + 1e-3 * 2. ** -24
# B200 against the Python operator: the same kernels and call sequence; only the order of the fp32 atomics (hash scatter,
# dL/dparams across CTAs) differs.  Measured on an H100 (80 GB HBM3, 132 SMs): at most 4.5e-7 (field MLP, 203 315 points).
FIELD_PY_BAR = 2e-6
# |log(||B200|| / ||tcnn||)| per group (field MLP, shader MLP, shading input, table level slab).  A loss-scale mistake moves a
# group by log(scale) >= log 2 = 0.69 (the mutations tried moved one by 4.85 .. 6.93).  Measured on an H100 (80 GB HBM3):
# at most 7.7e-3 (table level 0, 129 points: tcnn's fp16 atomics), 1e-3 elsewhere.
NORM_RATIO_BAR = 2e-2


def sizes():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return dict(one=1, ragged=129, past_a_wave=2 * sms * 128 + 77, three_tiles=128 * (12 * sms + 5) - 77)


def case_name(size, scale):
    return f"{size}_s{int(scale)}"


def _golden():
    return load_golden("ref_ngp_fox")


def _inputs(n, V, seed, scale):
    rng = np.random.default_rng(seed)
    pts, anchors, _ = ray_layout(max(n, 4096), V, rng)           # ray-like runs: the scatter merges consecutive rows
    dirs = rng.standard_normal((n, 3))
    return dict(points=np.ascontiguousarray(pts[:n]), anchors=np.ascontiguousarray(anchors[:n, 0]),
                d_out=(rng.standard_normal((n, 16)) * G_STD).astype(np.float32),
                feats=rng.standard_normal((n, 16)).astype(np.float32),
                dirs=(dirs / np.linalg.norm(dirs, axis=1, keepdims=True)).astype(np.float32),
                d_rgb=(rng.standard_normal((n, 3)) * G_STD).astype(np.float32),
                loss_scales=np.array([scale, scale], np.float32))


def _nonfinite_inputs(kind, V, base):
    """(i): an inf in one dL/dout (dL/drgb) row.  (ii): dL/dinput alone overflows.  Field: positive table entries, W0 = +1 and
    W_out[0, :] = 2 make every hidden unit live (h = sum of the 32 features), so dL/dout[0] * 128 = 1000 in one row gives
    dH = 2000 (finite in fp16) and dL/dfeat = 64 * 2000 = 128000 (inf), while dL/dW_out <= 1000 * h and dL/dW0 <= 2000 * feat
    stay finite.  Shader: W0 = 1/8 on the 16 feature columns (0 on the SH columns), W1 = 1/8, W_out[0, :] = 1/8 and features
    0.005 put raw[0] at 0.64 (sigmoid' = 0.23): dL/drgb[0] = 1000 gives d_raw = 2.9e4, dH2 = 3.6e3, dH1 = 2.9e4 and
    dL/dinput = 64 * 2.9e4 / 8 = 2.3e5 (inf), dL/dparams <= 2.9e4.  n = 129 keeps tcnn's fp16 dL/dparams sums of the other
    rows small."""
    x = _inputs(129, V, 7000 + NONFINITE.index(kind), 128.0)
    if kind == "i_field":
        x["d_out"][5, 0] = np.inf
    elif kind == "i_shader":
        x["d_rgb"][5, 0] = np.inf
    elif kind == "ii_field":
        x["feat_pool"] = np.abs(base["feat_pool"])
        p = base["field_params"].copy()
        p[:64 * 32] = 1.0
        p[64 * 32:64 * 32 + 64] = 2.0
        x["field_params"] = p
        x["d_out"][0] = 0
        x["d_out"][0, 0] = 1000. / 128.
    else:
        p = base["shader_params"].copy()
        w0 = np.zeros((64, 32), np.float32)
        w0[:, :16] = 0.125
        p[:64 * 32] = w0.reshape(-1)
        p[64 * 32:64 * 96] = 0.125
        p[64 * 96:64 * 96 + 64] = 0.125
        x["shader_params"] = p
        x["feats"][:] = 0.005
        x["d_rgb"][0] = [1000., 0., 0.]
    return x


_state = {}


def _setup():
    """Writes every case, runs both binaries once over all of them -> (inputs, {arm: {case: dumps}}, scene dumps)."""
    if _state:
        return _state["inputs"], _state["runs"], _state["scene"]
    for b in (REF, B200):
        if not os.path.exists(b):
            pytest.skip(f"{b} not built (build() makes it from the reference's sources)")
    g = _golden()
    V, pool = int(g["scalars"][4]), int(g["scalars"][5])
    gen = torch.Generator().manual_seed(1234)                   # the scene's table: ref_driver.cpp make_scene's U(-1, 1)
    base = dict(feat_pool=(torch.rand((pool, 2), generator=gen) * 2. - 1.).numpy(),
                field_params=g["field_mlp_params"].astype(np.float32), shader_params=g["shader_mlp_params"].astype(np.float32))
    inputs = {}
    for size, n in sizes().items():
        for s in SCALES:
            inputs[case_name(size, s)] = _inputs(n, V, n * 7 + int(s), s)
    for kind in NONFINITE:
        inputs[kind] = _nonfinite_inputs(kind, V, base)
    tmp = tempfile.mkdtemp(prefix="f2b_ops_")
    try:
        in_dir = os.path.join(tmp, "in")
        for k, v in base.items():
            os.makedirs(in_dir, exist_ok=True)
            np.save(os.path.join(in_dir, k + ".npy"), v)
        for c, x in inputs.items():
            os.makedirs(os.path.join(in_dir, c))
            for k, v in x.items():
                np.save(os.path.join(in_dir, c, k + ".npy"), v)
        runs, scene = {}, None
        for arm, binary in (("ref", REF), ("b200", B200)):
            out = os.path.join(tmp, arm)
            env = {k: v for k, v in os.environ.items() if k not in ("F2B_SHIM", "F2B_RENDER")}
            r = subprocess.run([binary, "--ops", CONFIG, in_dir, out], cwd=ROOT, capture_output=True, text=True, timeout=1200,
                               env=env)
            open(diag_path(f"ops_{arm}.log"), "w").write(r.stdout[-8000:] + "\n--- stderr ---\n" + r.stderr[-8000:])
            assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
            if arm == "b200":
                assert "replaced by the B200 subclasses" in r.stdout
            runs[arm] = {c: {f[:-4]: np.load(os.path.join(out, c, f)) for f in os.listdir(os.path.join(out, c))} for c in inputs}
            if scene is None:
                scene = {f[:-4]: np.load(os.path.join(out, f)) for f in os.listdir(out) if f.endswith(".npy")}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    for k in ("prim_pool", "bias_pool"):
        np.testing.assert_array_equal(scene[k], g[k], err_msg=k)
    np.testing.assert_array_equal(scene["scalars"][:7], g["scalars"][:7])       # [7]: the ray count of the golden run
    inputs["_base"] = base
    _state.update(inputs=inputs, runs=runs, scene=scene)
    return inputs, runs, scene


_py = {}


def _python_ops(x, base):
    """The Python operators (Hash3DAnchored / SHShader on the golden scene) with the case's parameters and loss scales."""
    if not _py:
        from test_ref_parity import build_from_ref
        gdp, _, field, shader, _ = build_from_ref(_golden())
        _py.update(gdp=gdp, field=field, shader=shader)
    gdp, field, shader = _py["gdp"], _py["field"], _py["shader"]
    field.feat_pool_.data.copy_(T(x.get("feat_pool", base["feat_pool"])))
    field.mlp_.params_.data.copy_(T(x.get("field_params", base["field_params"])))
    shader.mlp_.params_.data.copy_(T(x.get("shader_params", base["shader_params"])))
    field.mlp_.loss_scale_, shader.mlp_.loss_scale_ = float(x["loss_scales"][0]), float(x["loss_scales"][1])
    for p in (field.feat_pool_, field.mlp_.params_, shader.mlp_.params_):
        p.grad = None
    return gdp, field, shader


def _run_python(x, base):
    """Both operators as ref_driver.cpp runs them -> dumps in the binary's names."""
    gdp, field, shader = _python_ops(x, base)
    flags = lambda: np.array([float(gdp.backward_nan_), field.mlp_.loss_scale_, shader.mlp_.loss_scale_], np.float32)
    d = {}
    gdp.backward_nan_ = False
    torch.manual_seed(OPS_SEED)
    out = field.AnchoredQuery(T(x["points"]), T(x["anchors"]))
    (out * T(x["d_out"])).sum().backward()
    d.update(field_out=N(out), field_grad_table=N(field.feat_pool_.grad), field_grad_params=N(field.mlp_.params_.grad),
             field_flags=flags(), field_probe=N(torch.rand(4, device="cuda")))
    gdp.backward_nan_ = False
    torch.manual_seed(OPS_SEED + 1)
    feats = T(x["feats"]).requires_grad_(True)
    rgb = shader.Query(feats, T(x["dirs"]))
    (rgb * T(x["d_rgb"])).sum().backward()
    d.update(rgb=N(rgb), shader_grad_params=N(shader.mlp_.params_.grad), feats_grad=N(feats.grad), shader_flags=flags(),
             shader_probe=N(torch.rand(4, device="cuda")))
    return d


def dense_table(dump, pool):
    g = np.zeros(pool * 2, np.float32)
    g[dump["field_grad_table_nz_idx"].astype(np.int64)] = dump["field_grad_table_nz_val"]
    return g.reshape(pool, 2)


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64).reshape(-1), np.asarray(b, np.float64).reshape(-1)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-300))


def grad_groups(d, pool, local_size):
    """{group: gradient}: the two MLPs, the shading input, the table per level slab of its live prefix."""
    t = dense_table(d, pool) if "field_grad_table_nz_idx" in d else d["field_grad_table"]
    S = int(local_size)
    live = 17 * S // 2
    out = dict(field=d["field_grad_params"], shader=d["shader_grad_params"], feats=d["feats_grad"])
    for l in range((live + S - 1) // S):
        out[f"table[{l}]"] = t[l * S:min((l + 1) * S, live)]
    return out


def log_norm_ratios(a, b):
    """{group: log(||a|| / ||b||)} over the groups where b is nonzero (a must then be nonzero too)."""
    out = {}
    for k in b:
        nb, na = float(np.linalg.norm(np.asarray(b[k], np.float64))), float(np.linalg.norm(np.asarray(a[k], np.float64)))
        if nb > 0:
            out[k] = float(np.log(na / nb)) if na > 0 else float("-inf")
    return out


def twin_errors(x, d, field, shader, pool):
    """B200's gradients against the float64 twin pinned to the forward of the same fp16 kernels -> (errors, entry ratio, pins)."""
    from f2nerf_b200 import ops
    pts, vol, g_out = T(x["points"]), T(x["anchors"]), T(x["d_out"])
    scale_f, scale_s = float(x["loss_scales"][0]), float(x["loss_scales"][1])
    hp = hash_args(field, ops.hash_level_scales().cuda())
    tab = field.feat_pool_.detach().to(F64).requires_grad_(True)
    fpar = field.mlp_.params_.detach().to(F64).requires_grad_(True)
    pins = AT.Pins()
    with torch.no_grad():
        mag_feat = AT.hash_encode(AT.round16(tab).abs(), pts, vol, hp)
    feat = pins.pin("feat", AT.hash_encode(AT.round16(tab), pts, vol, hp),
                    ops.hash_fwd(field.table_f16(), field.prim_pool_, field.bias_pool_, field.n_volumes_, field.local_size_, pts, vol),
                    mag_feat)
    o, mag = AT.mlp(feat, AT.round16(fpar), 0, magnitude=True)
    o = pins.pin("out", o, T(d["field_out"]), mag)
    (o * g_out.to(F64)).sum().backward()
    got_table = dense_table(d, pool)
    errs = group_errors(dict(field=d["field_grad_params"], shader=np.ones(1), table=got_table),
                        dict(field=N(fpar.grad), shader=np.ones(1), table=N(tab.grad)), field.local_size_)
    # per table entry: the magnitude each fp16 row of the backward (loss-scaled dL/dout, dH, dL/dfeat) was rounded at, taken
    # back to dL/dfeat through |W| and the ReLU mask, each stage with its fp16 subnormal spacing (2^-24 / scale)
    qf = 2. ** -24 / scale_f
    p16 = field.mlp_.params_.detach().half().to(F64)
    W0, Wo = p16[:64 * 32].view(64, 32), p16[64 * 32:].view(16, 64)
    live = (feat.detach() @ W0.T) > 0
    m_feat = (((g_out.to(F64).abs() + qf) @ Wo.abs()) * live + qf) @ W0.abs() + qf
    bound = N(AT.abs_table_contributions(tuple(field.feat_pool_.shape), pts, vol, hp, m_feat, device="cuda"))
    entry = float((np.abs(got_table - N(tab.grad)) / (bound + 1e-300)).max())
    del tab, fpar, feat, o
    # shader: pinned to the fp16 MLP output of the same kernel
    feats, dirs, g_rgb = T(x["feats"]), T(x["dirs"]), T(x["d_rgb"])
    sh = shader.SHEncode(dirs)
    with torch.no_grad():
        raw_dev = shader.mlp_.Query(torch.cat([feats, sh], -1))
    spar = shader.mlp_.params_.detach().to(F64).requires_grad_(True)
    f64 = feats.to(F64).requires_grad_(True)
    raw, mag = AT.mlp(AT.round16(torch.cat([f64, sh.to(F64)], 1)), AT.round16(spar), 1, magnitude=True)
    raw = pins.pin("raw", raw[:, :3], raw_dev, mag[:, :3])
    (AT.shader_act(raw) * g_rgb.to(F64)).sum().backward()
    for name, a, b in (("shader", d["shader_grad_params"], N(spar.grad)), ("feats", d["feats_grad"], N(f64.grad))):
        errs[name] = dict(rel=rel_l2(a, b), cos=float((a.astype(np.float64) * b).sum() / (np.linalg.norm(a) * np.linalg.norm(b))),
                          norm=float(np.linalg.norm(b)))
    # the fp16 rows the loss scale is for: how many nonzero loss-scaled dL/dout entries fall below 2^-14 (subnormal)
    act = AT.shader_act(raw_dev[:, :3].to(F64))
    d_raw16 = (g_rgb.to(F64) * scale_s * (1. + 2e-3) * torch.sigmoid(raw_dev[:, :3].to(F64)) *
               (1 - torch.sigmoid(raw_dev[:, :3].to(F64)))).abs()
    d_out16 = g_out.to(F64).abs() * scale_f
    sub = lambda v: float((v[v > 0] < 2. ** -14).double().mean()) if bool((v > 0).any()) else 0.0
    extra = dict(act_err=float((T(d["rgb"]).to(F64) - act).abs().max()), subnormal_d_out=sub(d_out16), subnormal_d_raw=sub(d_raw16))
    return errs, entry, pins.stats, extra


CASES = [(s, sc) for s in SIZES for sc in SCALES]


@pytest.mark.parametrize("size,scale", CASES, ids=[case_name(s, sc) for s, sc in CASES])
def test_cpp_operators(size, scale):
    inputs, runs, scene = _setup()
    c = case_name(size, scale)
    x, base = inputs[c], inputs["_base"]
    b, r = runs["b200"][c], runs["ref"][c]
    pool = base["feat_pool"].shape[0]
    py = _run_python(x, base)
    gdp, field, shader = _py["gdp"], _py["field"], _py["shader"]
    S = field.local_size_
    # no flag at any scale, the generators where the reference leaves them
    for arm, d in (("b200", b), ("ref", r), ("python", py)):
        np.testing.assert_array_equal(d["field_flags"], [0, scale, scale], err_msg=arm)
        np.testing.assert_array_equal(d["shader_flags"], [0, scale, scale], err_msg=arm)
        for k in ("field_probe", "shader_probe"):
            np.testing.assert_array_equal(d[k], r[k], err_msg=f"{arm} {k}: RNG stream differs from the reference's")
    # against float64 autograd
    errs, entry, pins, extra = twin_errors(x, b, field, shader, pool)
    # against the Python operators: field_fwd (fused) vs hash_fwd + mlp_fwd, the same backward kernels
    np.testing.assert_array_equal(b["field_out"].view(np.uint32), py["field_out"].view(np.uint32))
    field_py = dict(params=rel_l2(b["field_grad_params"], py["field_grad_params"]),
                    table=rel_l2(dense_table(b, pool), py["field_grad_table"]))
    # against tiny-cuda-nn
    fscale = float(np.abs(r["field_out"]).max())
    ferr = np.abs(b["field_out"] - r["field_out"])
    ratios = log_norm_ratios(grad_groups(b, pool, S), grad_groups(r, pool, S))
    rec = dict(case=c, n=int(x["points"].shape[0]), scale=scale, pins=pins, errors=errs, table_entry_ratio_max=entry,
               field_vs_python=field_py, log_norm_ratio=ratios, fwd_vs_tcnn=dict(field_max=float(ferr.max() / fscale),
               field_median=float(np.median(ferr) / fscale), rgb_max=float(np.abs(b["rgb"] - r["rgb"]).max())), **extra,
               bars=dict(rel_l2=REL_BAR, one_minus_cos=COS_BAR, entry=ENTRY_BAR, act=ACT_BAR, field_python=FIELD_PY_BAR,
                         log_norm_ratio=NORM_RATIO_BAR))
    with open(diag_path(f"ops_{c}.json"), "w") as f:
        json.dump(rec, f, indent=1)
    bad = {k: v for k, v in errs.items() if v["norm"] > 0 and (v["rel"] > REL_BAR or v["cos"] < 1 - COS_BAR)}
    assert not bad, (c, bad)
    assert entry <= ENTRY_BAR, (c, entry)
    assert extra["act_err"] <= ACT_BAR, (c, extra["act_err"])
    assert max(field_py.values()) <= FIELD_PY_BAR, (c, field_py)
    assert ferr.max() <= 0.02 * fscale and np.median(ferr) <= 2e-3 * fscale, rec["fwd_vs_tcnn"]
    assert rec["fwd_vs_tcnn"]["rgb_max"] <= 0.02, rec["fwd_vs_tcnn"]
    worst = max(ratios.items(), key=lambda kv: abs(kv[1]))
    assert abs(worst[1]) <= NORM_RATIO_BAR, (c, worst)


@pytest.mark.parametrize("kind", NONFINITE)
def test_cpp_operators_nonfinite(kind):
    """The reference arm decides: which operator flags backward_nan_ and whose loss scale halves."""
    inputs, runs, _ = _setup()
    x, base = inputs[kind], inputs["_base"]
    r, b = runs["ref"][kind], runs["b200"][kind]
    py = _run_python(x, base)
    flagged_field = kind.endswith("field")
    exp_field = [1., 64., 128.] if flagged_field else [0., 128., 128.]
    exp_shader = [0., 64., 128.] if flagged_field else [1., 128., 64.]
    np.testing.assert_array_equal(r["field_flags"], exp_field)
    np.testing.assert_array_equal(r["shader_flags"], exp_shader)
    if kind.startswith("ii"):
        # only dL/dinput overflowed: the reference's dL/dparams are finite, its table gradient (field) or dL/dfeats (shader)
        # are not
        if flagged_field:
            assert np.isfinite(r["field_grad_params"]).all() and not np.isfinite(r["field_grad_table_nz_val"]).all()
            assert np.isfinite(b["field_grad_params"]).all() and not np.isfinite(b["field_grad_table_nz_val"]).all()
        else:
            assert np.isfinite(r["shader_grad_params"]).all() and not np.isfinite(r["feats_grad"]).all()
            assert np.isfinite(b["shader_grad_params"]).all() and not np.isfinite(b["feats_grad"]).all()
    for arm, d in (("b200", b), ("python", py)):
        np.testing.assert_array_equal(d["field_flags"], r["field_flags"], err_msg=f"{kind}: {arm} field operator")
        np.testing.assert_array_equal(d["shader_flags"], r["shader_flags"], err_msg=f"{kind}: {arm} shader operator")
