"""The ray march (march16_kernel: several lanes per ray, several rays per warp) against the CPU oracle, bit for bit, in all
three modes: count (f2b_sampler_count), fill (f2b_sampler_fill) and the one-pass march into scratch slots (f2b_sampler_march +
f2b_sampler_gather).

The cases are the ones a lane split can get wrong: ray counts that leave a warp partly filled (1, 3, 5, 7, 9, 4095, 4097 cover
one ray short of and past 2, 4 and 8 rays per warp), rays that miss the scene between rays that hit it, rays that stop at the
1024-sample cap next to rays that stop early, leaf hops that land several steps ahead, scale_by_dis 0 / 1 and count_all_hits.
Each case first checks on the oracle's output that the batch does contain what it is meant to cover."""
import numpy as np
import pytest
import torch

from conftest import make_rays

pytestmark = pytest.mark.gpu

DEV = "cuda"
CAP = 1024


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV).contiguous()


def N(t):
    return t.detach().cpu().numpy()


def batch(scene, n, seed, miss_every=7):
    """n seeded rays through the scene; every `miss_every`-th ray starts far outside and points away."""
    o, _, dn, _ = make_rays(scene, n, seed=seed)
    o, dn = o.copy(), dn.copy()
    if miss_every:
        o[::miss_every] = np.float32(600.)
        dn[::miss_every] = np.float32(0.57735026)
    rng = np.random.default_rng(seed)
    noise = (rng.random(CAP + n + 10, dtype=np.float32) * .5 + .75).astype(np.float32)
    return o, dn, noise


def hops(ref):
    """Per ray, the largest t step across a leaf change over the t step just before it (a leaf hop of n steps gives ~n)."""
    b, t, node = ref["bounds"], ref["t"], ref["anchors"][:, 1]
    best = 0.
    for beg, end in b:
        if end - beg < 3:
            continue
        dtt = np.diff(t[beg:end].astype(np.float64))
        jump = np.nonzero(node[beg + 1:end] != node[beg:end - 1])[0]
        jump = jump[jump >= 1]
        if jump.size:
            best = max(best, float((dtt[jump] / np.maximum(dtt[jump - 1], 1e-30)).max()))
    return best


def check_all_modes(scene, oracle, o, dn, noise, sample_l, scale_by_dis, max_hits=CAP):
    from f2nerf_b200 import ops
    ref = oracle.sampler(scene["nodes"], scene["trans"], o, dn, noise, 0.05, 1e8, sample_l, scale_by_dis, max_hits)
    n = o.shape[0]
    args = (T(scene["nodes"]), T(scene["trans"]), T(o), T(dn), T(noise), 0.05, 1e8, sample_l, scale_by_dis, max_hits)
    # MODE 0 (count), with and without count_all_hits, then MODE 1 (fill)
    bounds, totals = ops.sampler_count(*args, count_all_hits=True)
    n_pts, n_hits = (int(v) for v in totals.tolist())
    assert n_hits == ref["n_hits"]
    np.testing.assert_array_equal(N(bounds), ref["bounds"])
    b2, tot2 = ops.sampler_count(*args, count_all_hits=False)
    np.testing.assert_array_equal(N(b2), ref["bounds"])
    assert int(tot2[0]) == n_pts and 0 < int(tot2[1]) <= n_hits
    pts, dirs, dt, t, anchors, first = ops.sampler_fill(*args, bounds, n_pts)
    got = dict(pts=N(pts), dirs=N(dirs), dt=N(dt), t=N(t), first_oct_dis=N(first))
    for k in ("first_oct_dis", "t", "dt", "dirs", "pts"):
        np.testing.assert_array_equal(got[k].view(np.uint32), ref[k].view(np.uint32), err_msg=f"fill {k}")
    np.testing.assert_array_equal(N(anchors), ref["anchors"])
    # MODE 2: one pass into per-ray slots, then the gather into the compact layout
    f = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device=DEV)
    scratch = (f(n * CAP, 3), f(n * CAP), f(n * CAP), torch.full((n * CAP, 2), -7, dtype=torch.int32, device=DEV))
    for cah in (True, False):
        b3, tot3, first3 = ops.sampler_march(*args, scratch, count_all_hits=cah)
        np.testing.assert_array_equal(N(b3), ref["bounds"])
        assert int(tot3[0]) == n_pts
        assert int(tot3[1]) == n_hits if cah else 0 < int(tot3[1]) <= n_hits
        np.testing.assert_array_equal(N(first3).view(np.uint32), ref["first_oct_dis"].view(np.uint32))
    # nothing was written past a ray's count in its slot
    cnt = np.diff(ref["bounds"], axis=1)[:, 0]
    s_dt = N(scratch[1]).reshape(n, CAP)
    assert np.isnan(s_dt[np.arange(CAP)[None, :] >= cnt[:, None]]).all()
    g = ops.sampler_gather(T(dn), b3, n_pts, scratch)
    for k, v in zip(("pts", "dirs", "dt", "t"), g[:4]):
        np.testing.assert_array_equal(N(v).view(np.uint32), ref[k].view(np.uint32), err_msg=f"march {k}")
    np.testing.assert_array_equal(N(g[4]), ref["anchors"])
    return ref


@pytest.mark.parametrize("n", [1, 3, 5, 7, 9, 4095, 4097])
@pytest.mark.parametrize("scale_by_dis", [False, True])
def test_march_ray_counts(scene, oracle, n, scale_by_dis):
    o, dn, noise = batch(scene, n, seed=100 + n, miss_every=7 if n > 1 else 0)
    ref = check_all_modes(scene, oracle, o, dn, noise, 1 / 256, scale_by_dis)
    cnt = np.diff(ref["bounds"], axis=1)[:, 0]
    assert cnt.max() > 0
    if n >= 7:
        assert (cnt[::7] == 0).all()                  # the rays pointing away from the scene


def test_march_sample_cap(scene, oracle):
    """Rays that stop at the 1024-sample cap, warp-mates of rays that end earlier."""
    o, dn, noise = batch(scene, 333, seed=11, miss_every=5)
    ref = check_all_modes(scene, oracle, o, dn, noise, 1 / 256, True)
    cnt = np.diff(ref["bounds"], axis=1)[:, 0]
    assert (cnt == CAP).sum() >= 16 and ((cnt > 0) & (cnt < CAP)).sum() >= 16


def test_march_leaf_hops(scene, oracle):
    """Long steps: rays cross many leaves and the leaf hop lands several steps past the current t."""
    o, dn, noise = batch(scene, 517, seed=12, miss_every=0)
    ref = check_all_modes(scene, oracle, o, dn, noise, 1 / 16, False)
    nodes_per_ray = [len(np.unique(ref["anchors"][b:e, 1])) for b, e in ref["bounds"]]
    assert max(nodes_per_ray) >= 8
    assert hops(ref) >= 3.


def test_march_hit_cap(scene, oracle):
    """max_oct_intersect_per_ray cuts rays off after a few leaves, in every lane of the ray alike."""
    o, dn, noise = batch(scene, 100, seed=13)
    check_all_modes(scene, oracle, o, dn, noise, 1 / 256, True, max_hits=3)
