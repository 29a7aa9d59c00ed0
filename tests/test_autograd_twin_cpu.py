"""The CPU oracle's hand-written TRAIN backward (oracle_pipeline.render_train) against float64 autograd of the reference's
Render and loss (tests/autograd_twin.py), one loss term at a time, on the synthetic scene.

The twin is pinned to the oracle's forward values, so what is compared is the backward alone.  The remaining distance is the
fp16 rounding of the rows the oracle's backward writes (loss-scaled dL/dout, dH, dL/dfeat), as the CUDA backward does.
Deliberately broken twins (autograd_twin.BROKEN) must fail the same comparison: that shows the bars are tight enough to
catch a mistake of their size in any one term.
"""
import numpy as np
import pytest
import torch

import autograd_twin as AT
from conftest import make_rays

F64 = torch.float64
LOSS_W = dict(color=(1, 0, 0, 0, 0), var=(0, 1, 0, 0, 0), disp=(0, 0, 1, 0, 0), tv=(0, 0, 0, 1, 0), depth=(0, 0, 0, 0, 1),
              mix=(1.0, 0.01, 0.01, 0.1, 0))
# the groups a term's gradient reaches; the others must be exactly zero
REACH = dict(color=("field", "shader", "app_emb", "table"), var=("field", "table"), disp=("field", "table"),
             tv=("field", "table"), depth=("field", "table"), mix=("field", "shader", "app_emb", "table"))
# bars: relative L2 and 1 - cosine per group (the table: per level slab, the appearance embedding: per camera row).  The
# measured errors are 2e-5 .. 7.3e-4 in rel L2 and <= 2.6e-7 in 1 - cos (the fp16 rows of the backward); every broken twin
# moves some group by > 1e-2
REL_BAR, COS_BAR = 4e-3, 2e-6


def twin_weights(term):
    return dict(zip(("color", "var", "disp", "tv", "depth"), LOSS_W[term]))


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64).reshape(-1), np.asarray(b, np.float64).reshape(-1)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-300))


def cos(a, b):
    a, b = np.asarray(a, np.float64).reshape(-1), np.asarray(b, np.float64).reshape(-1)
    return float((a * b).sum() / (np.linalg.norm(a) * np.linalg.norm(b) + 1e-300))


def group_errors(got, twin, local_size):
    """got / twin: dict(field, shader, app_emb (or None), table [pool, 2]) of numpy gradients -> {group: dict(rel, cos, norm)}.
    The table is compared per level slab [l S, (l + 1) S) of its live prefix [0, 17 S / 2) rows; its dead tail must be 0.
    The appearance embedding is compared per camera row; rows no sample used must be 0 on both sides."""
    out = {}
    for k in ("field", "shader"):
        out[k] = dict(rel=rel_l2(got[k], twin[k]), cos=cos(got[k], twin[k]), norm=float(np.linalg.norm(twin[k])))
    if twin.get("app_emb") is not None:
        for r in range(twin["app_emb"].shape[0]):
            g, t = got["app_emb"][r], twin["app_emb"][r]
            if np.abs(t).max() == 0:
                assert np.abs(g).max() == 0, f"app_emb row {r}: gradient where the twin has none"
                continue
            out[f"app_emb[{r}]"] = dict(rel=rel_l2(g, t), cos=cos(g, t), norm=float(np.linalg.norm(t)))
    S = int(local_size)
    live = 17 * S // 2
    tail = np.asarray(got["table"])[live:]
    assert (tail == 0).all(), f"table gradient in the dead tail [{live}, ...): {int((tail != 0).sum())} entries"
    assert (np.asarray(twin["table"])[live:] == 0).all()
    for l in range((live + S - 1) // S):
        sl = slice(l * S, min((l + 1) * S, live))
        g, t = np.asarray(got["table"])[sl], np.asarray(twin["table"])[sl]
        out[f"table[{l}]"] = dict(rel=rel_l2(g, t), cos=cos(g, t), norm=float(np.linalg.norm(t)))
    return out


def worst(errs, prefix):
    sel = [v for k, v in errs.items() if k.split("[")[0] == prefix and v["norm"] > 0]
    if not sel:
        return None
    return dict(rel=max(v["rel"] for v in sel), cos=min(v["cos"] for v in sel), norm=max(v["norm"] for v in sel))


def passes(errs, rel_bar=REL_BAR, cos_bar=COS_BAR):
    return all(v["rel"] <= rel_bar and v["cos"] >= 1 - cos_bar for v in errs.values() if v["norm"] > 0)


def run_twin(leaves0, inp, hp, dev, gt, term, broken=(), device="cpu"):
    """Fresh float64 leaves, the twin's forward pinned to ``dev`` and the term's backward -> (numpy grads, render output)."""
    leaves = {k: (None if v is None else v.detach().clone().to(device).requires_grad_(True)) for k, v in leaves0.items()}
    out = AT.render(leaves, inp, hp, dev=dev, broken=broken)
    L = AT.loss(out, gt, twin_weights(term), broken=broken)
    L.backward()
    grads = {k: (None if v is None else (v.grad.cpu().numpy() if v.grad is not None else np.zeros(v.shape))) for k, v in leaves.items()}
    return grads, out, float(L.detach())


# ------------------------------------------------------------------------------------------------------ the CPU problem
def cpu_problem(scene, oracle, hash_params, n_rays, seed, use_emb, gs, term, miss=0):
    """The synthetic scene with test_gpu_render.build-like parameters (table U(-1, 1); the field MLP at 8x its init, so that
    early stop cuts most rays short and the TruncExp clamp acts on several % of the kept samples), through the oracle
    pipeline with the term's loss weights."""
    import oracle_pipeline as OP
    O = oracle
    sc = dict(nodes=scene["nodes"], trans=scene["trans"], edges=scene["edges"], near=0.05, sample_l=1 / 64, scale_by_dis=True,
              max_hits=1024)
    hp = hash_params
    rng = np.random.default_rng(seed)
    o, d, dn, cam = make_rays(scene, n_rays, seed=seed)
    if miss:                                             # every miss-th ray starts outside the octree and points away
        o[::miss] = 600.
        dn[::miss] = 1. / np.sqrt(3.)
    field_params = (O.mlp_init(32, 0) * 8).astype(np.float32)
    shader_params = O.mlp_init(32, 1)
    app_emb = (rng.standard_normal((24, 16)) * .1).astype(np.float32) if use_emb else None
    noise = rng.random(1024 + n_rays + 10, dtype=np.float32)
    bg = rng.random((n_rays, 3), dtype=np.float32)
    gt = rng.random((n_rays, 3), dtype=np.float32)
    n_edges = scene["edges"].size // 64
    e_idx = rng.integers(0, n_edges, 8192).astype(np.int32)
    e_coord = (rng.random((8192, 2), dtype=np.float32) * 2 - 1).astype(np.float32)
    fld = dict(table16=hp["table"], prim=hp["prim"], bias=hp["bias"], V=hp["V"], local_size=hp["local_size"], mlp_params=field_params)
    scales = O.level_scales()
    ref = OP.render_train(sc, o, dn, noise, bg, fld, shader_params, app_emb, cam if use_emb else None, (e_idx, e_coord), gt,
                          scales=scales, gs_progress=gs, loss_w=LOSS_W[term])
    nk = ref["n_kept"]
    t = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a)) if dt is None else torch.from_numpy(np.ascontiguousarray(a)).to(dt)
    inp = dict(pts=t(ref["pts"]), vol=t(ref["q_vol"][:nk]), dt=t(ref["dt"]), t=t(ref["t"]), bounds=t(ref["bounds"]), bg=t(bg),
               cam=t(cam) if use_emb else None, sh=t(ref["mlp_in"][:, 16:].astype(np.float32)), e_pts=t(ref["q_pts"][nk:]),
               e_vol=t(ref["q_vol"][nk:]), gs_progress=gs)
    dev = dict(feat=t(ref["feat16"]), logit=t(ref["scene_feat"][:nk, 0]), mlp_in=t(ref["mlp_in"]), raw=t(ref["raw"]),
               rgb=t(ref["rgb"]), edge=t(ref["scene_feat"][nk:]))
    hpt = dict(prim=t(hp["prim"].reshape(-1, 3), torch.int64) & 0xFFFFFFFF, bias=t(hp["bias"].reshape(-1, 3)), scales=t(scales),
               n_volumes=hp["V"], local_size=hp["local_size"])
    leaves = dict(table=t(hp["table"].astype(np.float32), F64), field=t(field_params, F64), shader=t(shader_params, F64),
                  app_emb=t(app_emb, F64) if use_emb else None)
    got = dict(field=ref["grad_field_mlp"], shader=ref["grad_shader_mlp"], app_emb=ref.get("grad_app_emb"),
               table=ref["grad_feat_pool"])
    return dict(ref=ref, inp=inp, dev=dev, hp=hpt, leaves=leaves, got=got, gt=t(gt), cam=cam)


def check_regime(P, gs, use_emb):
    """The case exercises what it is meant to: the TruncExp clamp, long rays under GradientScaling, several cameras."""
    ref, nk = P["ref"], P["ref"]["n_kept"]
    x = ref["scene_feat"][:nk, 0].astype(np.float64) - 3
    assert (x > 5).mean() >= 0.01, f"only {(x > 5).mean():.4f} of the kept samples have logit - 3 > 5"
    cnt = ref["bounds"][:, 1] - ref["bounds"][:, 0]
    if gs < 1:
        assert (cnt >= 32).any(), cnt.max()
    if use_emb:
        assert len(np.unique(P["cam"][cnt > 0])) >= 2
    assert ref["n_kept"] < ref["sample"]["pts"].shape[0], "early stop must act"


CASES = [(n, gs, emb, miss, term) for (n, gs, emb, miss) in ((128, 1.0, True, 0), (128, 0.3, True, 0), (96, 0.3, False, 0),
                                                            (129, 0.3, False, 3))
         for term in ("color", "var", "disp", "tv", "depth", "mix")]


@pytest.mark.parametrize("n_rays,gs,use_emb,miss,term", CASES,
                         ids=[f"{n}-gs{gs}-{'emb' if e else 'noemb'}{'-missed' if m else ''}-{t}" for n, gs, e, m, t in CASES])
def test_oracle_backward_matches_float64_autograd(scene, oracle, hash_params, n_rays, gs, use_emb, miss, term):
    """``miss``: every miss-th ray starts outside the octree and points away, so rays without samples sit between the others."""
    P = cpu_problem(scene, oracle, hash_params, n_rays, 5, use_emb, gs, term, miss=miss)
    check_regime(P, gs, use_emb)
    if miss:
        b = P["ref"]["bounds"]
        assert (b[::miss, 1] == b[::miss, 0]).all()
    twin, out, L = run_twin(P["leaves"], P["inp"], P["hp"], P["dev"], P["gt"], term)
    assert abs(L - P["ref"]["loss"]) <= 1e-5 * abs(P["ref"]["loss"]) + 1e-12, (L, P["ref"]["loss"])
    for k in ("field", "shader", "app_emb", "table"):
        if twin.get(k) is None:
            continue
        if k in REACH[term]:
            assert np.abs(twin[k]).max() > 0 and np.abs(P["got"][k]).max() > 0, f"{term}: no gradient in {k}"
        else:
            assert np.abs(twin[k]).max() == 0 and np.abs(P["got"][k]).max() == 0, f"{term}: gradient in {k}"
    errs = group_errors(P["got"], twin, P["hp"]["local_size"])
    bad = {k: v for k, v in errs.items() if v["norm"] > 0 and (v["rel"] > REL_BAR or v["cos"] < 1 - COS_BAR)}
    assert not bad, bad


# a broken twin, the case where its mistake acts, and the term it shows in
BROKEN_CASES = [("gs_linear", 0.3, True, "color"), ("gs_linear", 0.3, True, "disp"), ("truncexp_noclamp", 1.0, True, "mix"),
                ("emb_15ch", 1.0, True, "color"), ("disp_no_eps", 1.0, False, "disp")]


@pytest.mark.parametrize("broken,gs,use_emb,term", BROKEN_CASES, ids=[f"{b}-{t}" for b, _, _, t in BROKEN_CASES])
def test_broken_twin_fails(scene, oracle, hash_params, broken, gs, use_emb, term):
    P = cpu_problem(scene, oracle, hash_params, 128, 5, use_emb, gs, term)
    twin, _, _ = run_twin(P["leaves"], P["inp"], P["hp"], P["dev"], P["gt"], term, broken=(broken,))
    errs = group_errors(P["got"], twin, P["hp"]["local_size"])
    moved = max(v["rel"] for v in errs.values() if v["norm"] > 0)
    assert not passes(errs), f"{broken}: passes the bars (largest group error {moved:.2e})"
    assert moved > 2.5 * REL_BAR, (broken, moved)


def test_weightvar_backward_follows_the_reference(oracle):
    """WeightVar's backward (CustomOps.cu:38-66) per element against the oracle's restatement, on rays whose total weight runs
    from 1e-8 to 1: the twin's reference rule agrees, the exact derivative (x_j - mean) does not.  The two differ by
    tmp * mean / W with tmp = 2e-6 mean, so only rays whose total weight is near 1e-6 tell them apart."""
    rng = np.random.default_rng(3)
    n = rng.integers(1, 40, 64)
    total = 10.0 ** rng.uniform(-8, 0, 64)
    w = np.concatenate([rng.dirichlet(np.ones(k)) * s for k, s in zip(n, total)]).astype(np.float32)
    b = np.stack([np.cumsum(n) - n, np.cumsum(n)], 1).astype(np.int32)
    g = rng.uniform(.5, 1.5, 64).astype(np.float32)
    var_ref, dw_ref = oracle.weight_var(w, b, g)
    seg = AT.segments(torch.from_numpy(b))
    for centered in (False, True):
        wt = torch.from_numpy(w).to(F64).requires_grad_(True)
        var = AT.WeightVar.apply(wt, seg, centered)
        (var * torch.from_numpy(g).to(F64)).sum().backward()
        np.testing.assert_allclose(var.detach().numpy(), var_ref, rtol=1e-5, atol=1e-7)
        err = np.abs(wt.grad.numpy() - dw_ref) / (np.abs(dw_ref) + 1e-3 * np.abs(dw_ref).max())
        if centered:
            assert err.max() > 0.1, err.max()
        else:
            assert err.max() <= 1e-3, err.max()
