"""World-size-2 gloo test (CPU) of the data-parallel exchange step in f2nerf_b200/dist.py."""
import os
import socket
from datetime import timedelta
from types import SimpleNamespace

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _mock_renderer(rank, local, pool):
    field = SimpleNamespace(feat_pool_=torch.zeros(pool, 2, requires_grad=True), local_size_=local,
                            mlp_=SimpleNamespace(params_=torch.zeros(3072, requires_grad=True)))
    shader = SimpleNamespace(mlp_=SimpleNamespace(params_=torch.zeros(7168, requires_grad=True)))
    return SimpleNamespace(scene_field_=field, shader_=shader, app_emb_=torch.zeros(5, 16, requires_grad=True),
                           nonfinite_flag_=torch.tensor([rank == 1, False]))


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timedelta(seconds=60))
    from f2nerf_b200 import dist as fd
    from f2nerf_b200.renderer import slab_groups
    from f2nerf_b200.sampler import GlobalDataPool
    local = 1 << 8
    pool = local * 16
    renderer = _mock_renderer(rank, local, pool)
    field, shader = renderer.scene_field_, renderer.shader_
    g = torch.Generator().manual_seed(rank)
    live = fd.live_rows(field)
    assert live == 17 * local // 2
    field.feat_pool_.grad = torch.zeros(pool, 2)
    field.feat_pool_.grad[:live] = torch.rand(live, 2, generator=g)
    field.mlp_.params_.grad = torch.rand(3072, generator=g)
    shader.mlp_.params_.grad = torch.rand(7168, generator=g)
    renderer.app_emb_.grad = torch.rand(5, 16, generator=g) if rank == 0 else None   # a rank with no gradient (empty batch)
    zero_if_none = lambda t, like: torch.zeros_like(like) if t is None else t.clone()
    mine = [field.feat_pool_.grad.clone(), field.mlp_.params_.grad.clone(), shader.mlp_.params_.grad.clone(), zero_if_none(renderer.app_emb_.grad, renderer.app_emb_)]
    sent = fd.allreduce_grads(renderer)
    got = [field.feat_pool_.grad, field.mlp_.params_.grad, shader.mlp_.params_.grad, renderer.app_emb_.grad]
    # octree votes: MAX across ranks
    sampler = SimpleNamespace(vote_allreduce_=None)
    fd.install_vote_sync(sampler)
    vw = torch.tensor([-1, 512, -1, -1], dtype=torch.int32) if rank == 0 else torch.tensor([-1, -1, 512, -1], dtype=torch.int32)
    va = torch.tensor([32, -1, -1, -1], dtype=torch.int32) if rank == 0 else torch.tensor([-1, -1, -1, -1], dtype=torch.int32)
    mk = torch.tensor([1, 1, 0, 0], dtype=torch.int32) if rank == 0 else torch.tensor([0, 0, 1, 0], dtype=torch.int32)
    vc = torch.tensor([3, 7, 0, 0], dtype=torch.int32) if rank == 0 else torch.tensor([0, 9, 4, 0], dtype=torch.int32)
    sampler.vote_allreduce_(vw, va, mk, vc)
    # slab-wise overlapped all-reduce of the table gradient (install_grad_overlap): the hook sequence the backward issues
    fd.install_grad_overlap(renderer)
    assert renderer.grad_premul_ == 0.5
    gs = torch.Generator().manual_seed(100 + rank)
    slab = torch.rand(pool, 2, generator=gs)
    slab0 = slab.clone()
    for lo in (12, 8, 4, 0):
        renderer.grad_slab_hook_(slab, lo, local)
    renderer.grad_slab_finish_()
    assert renderer.table_grad_reduced_
    # the overlap installed on both ranks, but rank 1's shard is empty: its backward never runs, so it calls no hook and has
    # no gradient at all.  allreduce_grads must still issue the slab all-reduces rank 0 issued from inside its backward
    empty = _mock_renderer(rank, local, pool)
    fd.install_grad_overlap(empty)
    ge = torch.Generator().manual_seed(200)
    own = torch.zeros(pool, 2)
    if rank == 0:
        own[:live] = torch.rand(live, 2, generator=ge) * empty.grad_premul_      # the backward's 1/world pre-scaled scatter
        empty.scene_field_.feat_pool_.grad = own.clone()
        for lo, _ in slab_groups():
            empty.grad_slab_hook_(empty.scene_field_.feat_pool_.grad, lo, local)
        empty.grad_slab_finish_()
        for p in (empty.scene_field_.mlp_.params_, empty.shader_.mlp_.params_, empty.app_emb_):
            p.grad = torch.rand(p.shape, generator=ge)
    e_sent = fd.allreduce_grads(empty)
    e_got = [empty.scene_field_.feat_pool_.grad, empty.scene_field_.mlp_.params_.grad, empty.shader_.mlp_.params_.grad,
             empty.app_emb_.grad]
    gdp = GlobalDataPool()
    gdp.sampled_pts_per_ray_ = 100.0 + 50 * rank
    fd.sync_emas(gdp)
    q.put((rank, [t.numpy() for t in mine], [t.numpy() for t in got], renderer.nonfinite_flag_.tolist(), sent,
           vw.tolist(), va.tolist(), mk.tolist(), vc.tolist(), gdp.sampled_pts_per_ray_, slab0.numpy(), slab.numpy(),
           own.numpy(), [t.numpy() for t in e_got], e_sent, empty.table_grad_reduced_))
    dist.destroy_process_group()


def test_allreduce_step_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = sorted([q.get(timeout=120) for _ in range(2)], key=lambda x: x[0])
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)
    (r0, m0, g0, f0, s0, *v0), (r1, m1, g1, f1, s1, *v1) = res
    for a, b, ga, gb in zip(m0, m1, g0, g1):
        np.testing.assert_allclose(ga, (a + b) / 2, rtol=1e-6)           # averaged gradient, identical on both ranks
        np.testing.assert_array_equal(ga, gb)
    assert f0 == f1 == [True, False]                                    # NaN flags are OR-ed per MLP; same collectives on both ranks
    assert s0 == s1 == (17 * 256 // 2) * 2 * 4 + (3072 + 7168 + 80 + 2) * 4   # only the live prefix of the table travels
    assert v0[0] == v1[0] == [-1, 512, 512, -1] and v0[1] == v1[1] == [32, -1, -1, -1]
    assert v0[2] == v1[2] == [1, 1, 1, 0] and v0[3] == v1[3] == [3, 9, 4, 0]
    assert abs(v0[4] - 125.0) < 1e-9 and v0[4] == v1[4]
    live = 17 * 256 // 2                                                # slabs cover exactly the live prefix, once each
    np.testing.assert_allclose(v0[6][:live], v0[5][:live] + v1[5][:live], rtol=1e-6)
    np.testing.assert_array_equal(v0[6][:live], v1[6][:live])
    np.testing.assert_array_equal(v0[6][live:], v0[5][live:])
    # an empty rank under the overlap: same slab all-reduces, so both ranks end with rank 0's pre-scaled contribution (the
    # average of it and a zero gradient), bit for bit, and report the same bytes sent
    own0, e0, e1 = v0[7], v0[8], v1[8]
    assert (own0[:live] != 0).all() and not v1[7].any()
    np.testing.assert_array_equal(e0[0], own0)
    for a, b in zip(e0, e1):
        np.testing.assert_array_equal(a, b)
    assert v0[9] == v1[9] == s0
    assert not v0[10] and not v1[10]
