"""The free and large-table configurations against the reference program, through both hosts.

tests/test_ref_parity.py and tests/test_shim_dropin.py compare this library with the unmodified reference on the wanjinyou
settings only (oracle/ref_config_ngp_fox.yaml).  bench.py's other configurations take paths those runs never reach:

  free   (oracle/ref_config_free.yaml, nerf360 shares it)  near 0.05, scale_by_dis off, no appearance embedding, at the
         fineness 4 and gradient-scaling progress 1 that ExpRunner::UpdateAdaParams gives it at iteration 0
  big20  (oracle/ref_config_big20.yaml)  wanjinyou with a 2^20-entry table
  big22  (oracle/ref_config_big22.yaml)  wanjinyou with a 2^22-entry table: level offsets past 2^26 halves, a 512 MB gradient

Per config the seeded 512-ray script of oracle/ref_driver.cpp runs in three arms — ``ref`` (oracle/_ref/ref_driver, the
unmodified reference), ``fused`` (oracle/_ref/ref_driver_b200, the fused C++ host) and ``ops`` (the same with F2B_SHIM=ops,
the operator-level drop-in) — and the Python host replays it.  Each comparison is the one tests/test_ref_parity.py /
tests/test_shim_dropin.py make on wanjinyou, at the same bars.  The big-table runs skip the dense table gradient
(dump_full_grads 0): their table gradients are compared through the non-zero entries each arm dumps.  So on big20 / big22
test_render_train_vs_reference takes its stored-run branch: the Python host's table gradient is held against the
reference's fp16-noisy non-zero entries (cosine 0.97, slab norms within [0.8, 1.25]) and not against the exact oracle, which
only the free and wanjinyou runs reach.  What covers the big tables more tightly is transitive: the Python host equals the
fused arm to 1e-5 (test_fused_cpp_host_equals_python_host), and the fused arm matches the reference per level slab at cosine
0.999 (test_big_table_gradient_per_level_slab).

The free reference run is also stored (tests/golden/ref_free_512_*.npz, oracle/make_golden.py --config free), so its
reference-against-Python checks run where the binaries were not built; every other case skips then, naming the binary.

Beyond the shared checks:
  * without an embedding no arm produces an embedding gradient, the Python host leaves app_emb_.grad empty and the shader
    input's column 0 is exactly 1 (tests/test_shim_dropin.py:check_fused_cpp_host_equals_python_host);
  * big20 / big22: per level slab [l*S, (l+1)*S), l < 17, the table gradient's cosine and norm ratio against the
    reference's non-zero entries, and no arm writes a float at or past 17*S;
  * f2b_adam_step over the whole 2^27-float big22 table (live prefix 17/32, fp16 shadow) equals the ATen sequence of
    torch::optim::Adam bit for bit over two steps and leaves the dead tail untouched.

Measured margins go to workloads.diag_path as refcfg_<config>_<arm>_*.json.
"""
import json

import numpy as np
import pytest
import torch

import test_ref_parity as RP
import test_shim_dropin as SD
from test_gpu_parity import aten_adam_step
from workloads import diag_path, load_golden

pytestmark = pytest.mark.gpu

# oracle/<yaml> and ref_driver's trailing arguments [n_time_iters, dump_full_grads, fineness, gs_progress] per config
RUNS = {"free": ("ref_config_free.yaml", ("0", "1", "4", "1")),
        "big20": ("ref_config_big20.yaml", ("0", "0")),
        "big22": ("ref_config_big22.yaml", ("0", "0"))}
BIG = ("big20", "big22")
# Per level slab of a big table, the arm's gradient on the reference's non-zero entries against the reference's: cosine at
# least SLAB_COS_BAR and |log(norm ratio)| at most SD.STEP_NORM_RATIO_BAR, the whole-group bar of tests/test_shim_dropin.py.
# Measured on an H100 80GB HBM3 at 700 W, both arms, big20 and big22: cosine 0.99997 at the lowest (over 52 k reference
# entries per slab at least), |log(norm ratio)| 0.0043 (big20) and 0.0097 (big22, level 0) at the highest.  The reference's
# table gradient is the noisy side (fp16 products and fp16 atomics, Hash3DAnchored.cu:145-151).
SLAB_COS_BAR = 0.999
_refs = {}


def ref_run(config, source):
    """The reference's dumps of ``config``: "live" runs oracle/_ref/ref_driver, "golden" loads the stored free run"""
    key = (config, source)
    if key not in _refs:
        d = load_golden("ref_free_512") if source == "golden" else dict(SD._run("ref", *RUNS[config]))
        d = {k: (v.astype(np.float32) if v.dtype == np.float16 else v) for k, v in d.items()}
        d["_tag"] = f"refcfg_{config}_{source}"
        _refs[key] = d
    return _refs[key]


@pytest.fixture(params=[("free", "golden"), ("free", "live"), ("big20", "live"), ("big22", "live")], ids=lambda p: "-".join(p))
def ref(request):
    d = ref_run(*request.param)
    want = {"free": (False, 4.0, 1.0)}.get(request.param[0], (True, 1.0, 0.25))
    assert RP.run_settings(d) == want, (request.param, RP.run_settings(d))          # the run is the configuration it claims
    return d


# ---- the reference against the Python host: tests/test_ref_parity.py's checks --------------------------------------------
def test_sampler_validate_bit_exact(ref):
    RP.test_sampler_validate_bit_exact(ref)


def test_field_and_shader_vs_tcnn(ref):
    RP.test_field_and_shader_vs_tcnn(ref)


def test_render_validate_vs_reference(ref):
    RP.test_render_validate_vs_reference(ref)


def test_edge_samples_vs_reference(ref):
    RP.test_edge_samples_vs_reference(ref)


def test_render_train_vs_reference(ref):
    """the TRAIN sampler bit-exact (noise x fineness included), the octree votes, the loss and the gradient groups"""
    RP.test_render_train_vs_reference(ref)


# ---- the three arms of the reference program: tests/test_shim_dropin.py's checks ------------------------------------------
@pytest.fixture(params=[(c, k) for c in RUNS for k in ("fused", "ops")], ids=lambda p: "-".join(p))
def arms(request):
    config, kind = request.param
    return SD._run("ref", *RUNS[config]), SD._run(kind, *RUNS[config]), config, kind


def test_arms_same_scene_and_sampler(arms):
    a, b, _, _ = arms
    SD.check_same_scene(a, b)
    SD.check_sampler(a, b)


def test_arms_render(arms):
    a, b, _, kind = arms
    SD.check_render(a, b, kind)


def test_arms_step_gradient_magnitudes(arms):
    a, b, config, kind = arms
    SD.check_step_gradient_magnitudes(a, b, f"refcfg_{config}_{kind}_norm_ratio.json")
    for d in (a, b):                                        # the dead tail of the table takes no gradient in any arm
        assert int(SD.grad_of(d, "grad_feat_pool")[0].max()) < 17 * slab_size(d), (config, kind)


@pytest.mark.parametrize("config", list(RUNS))
def test_ops_arm_equals_fused_arm(config):
    SD.check_ops_arm_equals_fused_arm(SD._run("ops", *RUNS[config]), SD._run("fused", *RUNS[config]),
                                      f"refcfg_{config}_ops_vs_fused.json")


@pytest.mark.parametrize("config", list(RUNS))
def test_fused_cpp_host_equals_python_host(config):
    c = SD._run("fused", *RUNS[config])
    renderer = SD.check_fused_cpp_host_equals_python_host(c)
    g = renderer.scene_field_.feat_pool_.grad.reshape(-1)
    assert not bool(g[17 * renderer.scene_field_.local_size_:].any())         # the dead tail of the table takes no gradient


# ---- the large tables, level slab by level slab ---------------------------------------------------------------------------
def slab_size(d):
    return ((int(d["scalars"][5]) // 16) >> 4) << 4          # Hash3DAnchored's local_size_: fp32 elements per level slab


@pytest.mark.parametrize("config", BIG)
def test_big_table_gradient_per_level_slab(config):
    a = SD._run("ref", *RUNS[config])
    S = slab_size(a)
    assert a["scalars"][5] * 2 == 32 * S                     # 32 slabs of S floats: the levels' halves overlap
    ia, va = SD.grad_of(a, "grad_feat_pool")
    margins = {}
    for kind in ("fused", "ops"):
        b = SD._run(kind, *RUNS[config])
        ib, vb = SD.grad_of(b, "grad_feat_pool")
        for name, idx in (("ref", ia), (kind, ib)):
            assert idx.size > 0 and int(idx.max()) < 17 * S, (config, name, int(idx.max()), 17 * S)
        # the arm on the reference's non-zero entries (where the arm has none, its value is 0)
        pos = np.searchsorted(ib, ia)
        hit = (pos < ib.size) & (ib[np.minimum(pos, ib.size - 1)] == ia)
        mine = np.where(hit, vb[np.minimum(pos, ib.size - 1)], 0.)
        slabs = []
        for l in range(17):
            m = (ia >= l * S) & (ia < (l + 1) * S)
            x, y = mine[m], va[m]
            slabs.append(dict(slab=l, nnz_ref=int(m.sum()), nnz_arm=int(((ib >= l * S) & (ib < (l + 1) * S)).sum()),
                              cos=SD.cos(x, y), log_norm_ratio=float(np.log(np.linalg.norm(x) / np.linalg.norm(y)))))
        margins[kind] = slabs
    open(diag_path(f"refcfg_{config}_table_slabs.json"), "w").write(json.dumps(margins, indent=1))
    for kind, slabs in margins.items():
        for s in slabs:
            assert s["nnz_ref"] > 0 and s["cos"] >= SLAB_COS_BAR and abs(s["log_norm_ratio"]) <= SD.STEP_NORM_RATIO_BAR, (config, kind, s)


def test_big22_adam_full_table_live_prefix_and_shadow():
    """f2b_adam_step on big22's whole table (2^27 floats, live prefix 17 of 32 slabs, fp16 shadow) against the ATen sequence of
    torch::optim::Adam on the live prefix, two steps: bit-identical parameters, moments and shadow.  Every float of the dead
    tail is a sentinel in the fused arm — NaN gradient and moments, the parameter's own bits — and must be left as it was."""
    from f2nerf_b200._lib import call, stream
    dev = "cuda"
    n = (1 << 22) * 16 * 2                                   # the [pool, 2] float table of a 2^22-entry hash grid
    S = ((n // 2 // 16) >> 4) << 4
    live = 17 * S
    assert live == n * 17 // 32 and live > 1 << 26
    gen = torch.Generator(device=dev).manual_seed(22)
    p0 = torch.rand(n, device=dev, generator=gen) * 2 - 1
    pa, pf = p0[:live].clone(), p0.clone()
    ma, va = torch.zeros(live, device=dev), torch.zeros(live, device=dev)
    mf, vf = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    mf[live:], vf[live:] = float("nan"), float("nan")
    shadow = p0.to(torch.float16)
    shadow_tail = shadow[live:].clone()
    for step, lr in ((1, 1e-2), (2, 9e-3)):
        g = torch.randn(live, device=dev, generator=gen) * 10.0 ** -step
        g[torch.rand(live, device=dev, generator=gen) < 0.7] = 0.0          # mostly empty, like a table gradient
        gf = torch.full((n,), float("nan"), device=dev)
        gf[:live] = g
        aten_adam_step(pa, g, ma, va, step, lr, 0.9, 0.99, 1e-15, 0.0)
        call("f2b_adam_step", pf, gf, mf, vf, n, live, lr, 0.9, 0.99, 1e-15, 0.0, step, shadow, stream())
        del gf
        torch.cuda.synchronize()
        for want, got, name in ((pa, pf, "param"), (ma, mf, "exp_avg"), (va, vf, "exp_avg_sq")):
            assert torch.equal(want.view(torch.int32), got[:live].view(torch.int32)), (name, step)
        assert torch.equal(shadow[:live], pa.to(torch.float16)), step
        assert torch.equal(pf[live:].view(torch.int32), p0[live:].view(torch.int32)), step
        assert bool(torch.isnan(mf[live:]).all()) and bool(torch.isnan(vf[live:]).all()), step
        assert torch.equal(shadow[live:], shadow_tail), step
    assert not torch.equal(pa, p0[:live])
