"""Data-parallel plumbing: rays are sharded across ranks (one process per GPU), the hash table, MLPs,
appearance embedding and octree are replicated; after backward exactly one exchange step runs
(SURVEY.md §8e).  No collective sits inside the data path (forward / backward kernels).

  * SUM all-reduce of the hash-table gradient — only the live prefix: level l occupies halves
    [l*S, l*S + 2S) so rows >= 17*S/2 of the [pool,2] gradient are identically zero (the reference's
    overlapping-level quirk) and are never sent;
  * one flattened SUM all-reduce for the two MLP gradients + the appearance-embedding gradient;
  * MAX all-reduce (int32) of the octree votes BEFORE the stat update, so every rank prunes the same
    nodes (PersSampler.cu:579-603 would otherwise diverge across ranks); a rank whose batch has no sample takes part with
    neutral votes (Renderer._neutral_votes);
  * OR of the NaN flag, MEAN of the samples-per-ray EMAs that size the next batch (ExpRunner.cpp:86).
Gradients are averaged (losses are means over the global batch).
"""
import torch
import torch.distributed as dist

from .renderer import slab_groups


def live_rows(field):
    return min(field.feat_pool_.shape[0], (17 * field.local_size_) // 2)


def install_vote_sync(sampler):
    """Make UpdateOctNodes all-reduce its votes (MAX) across ranks before applying them."""
    def sync(vote_w, vote_a, mark, visit_cnt):
        n = vote_w.numel()
        flat = torch.cat([vote_w, vote_a, mark, visit_cnt])
        dist.all_reduce(flat, op=dist.ReduceOp.MAX)
        vote_w.copy_(flat[:n]); vote_a.copy_(flat[n:2 * n]); mark.copy_(flat[2 * n:3 * n]); visit_cnt.copy_(flat[3 * n:])
    sampler.vote_allreduce_ = sync


def install_grad_overlap(renderer):
    """Overlap the table-gradient all-reduce with the scatter that produces it.  The renderer's backward then scatters per
    level group, top-down (f2b_hash_bwd_levels), and calls the hook after each group; level l writes only floats
    [l*S, (l+2)*S) of the gradient, so after the group starting at level ``lo`` everything from float (lo+1)*S up to the
    previous boundary is final and its SUM all-reduce is issued at once (async, on NCCL's stream, ordered behind the scatter
    stream) while the lower groups still run.  Only the last slab ([0, 5S) of 17S) is exposed.  The 1/world averaging is folded
    into the scatter's gradient multiplier; the backward's last act is to make its stream wait for the slab all-reduces, so
    the gradient autograd hands to ``.grad`` is already the global average and ``allreduce_grads`` skips the table.  A rank
    whose backward did not run (an empty shard) issues the same slab all-reduces from ``allreduce_grads`` instead."""
    world = dist.get_world_size()
    renderer.grad_premul_ = 1.0 / world
    st = dict(hi=None, works=[], table=None)

    def hook(d_table, level_lo, local_size):
        flat = d_table.view(-1)
        if st["table"] is not d_table:                                   # first group of this backward (finish() clears the slot)
            st.update(hi=min(flat.numel(), 17 * local_size), works=[], table=d_table)
        lo = (level_lo + 1) * local_size if level_lo > 0 else 0
        if st["hi"] > lo:
            st["works"].append(dist.all_reduce(flat[lo:st["hi"]], async_op=True))
        st["hi"] = lo

    def finish():
        for w in st["works"]:
            w.wait()                                                      # the current (main) stream waits; no host block
        st.update(works=[], table=None)
        renderer.table_grad_reduced_ = True

    renderer.grad_slab_hook_, renderer.grad_slab_finish_ = hook, finish
    renderer.table_grad_reduced_ = False


def allreduce_grads(renderer):
    """The post-backward exchange step; returns the number of bytes each rank contributed.  Every rank issues the SAME
    fixed-shape collectives whether or not its own batch produced gradients (a rank whose rays all missed the octree, or
    whose shard is empty, contributes zeros), so ranks can never disagree on the collective sequence."""
    world = dist.get_world_size()
    field, shader = renderer.scene_field_, renderer.shader_
    params = (field.mlp_.params_, shader.mlp_.params_, renderer.app_emb_)
    sent = 0
    hook = getattr(renderer, "grad_slab_hook_", None)
    if hook is not None and not getattr(renderer, "table_grad_reduced_", False):
        # overlap installed but no backward of this step called the hook (an empty shard: no graph): issue the same slab
        # all-reduces the other ranks issued from inside their backward, on a zero contribution
        if field.feat_pool_.grad is None:
            field.feat_pool_.grad = torch.zeros_like(field.feat_pool_)
        for lo, _ in slab_groups():
            hook(field.feat_pool_.grad, lo, int(field.local_size_))
        renderer.grad_slab_finish_()
    if getattr(renderer, "table_grad_reduced_", False) and field.feat_pool_.grad is not None:
        renderer.table_grad_reduced_ = False             # averaged slab by slab inside the backward (install_grad_overlap)
        sent += live_rows(field) * 2 * 4
    else:
        if field.feat_pool_.grad is None:
            field.feat_pool_.grad = torch.zeros_like(field.feat_pool_)
        g = field.feat_pool_.grad[:live_rows(field)]
        dist.all_reduce(g)
        g.div_(world)
        sent += g.numel() * g.element_size()
    dev = field.feat_pool_.device
    flag = getattr(renderer, "nonfinite_flag_", None)
    flag = torch.zeros(2, device=dev) if flag is None else flag.reshape(-1).float().expand(2) if flag.numel() == 1 else flag.float()
    flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in params] + [flag * world])
    dist.all_reduce(flat)
    flat.div_(world)
    off = 0
    for p in params:
        n = p.numel()
        if p.grad is None:
            p.grad = torch.empty_like(p)
        p.grad.copy_(flat[off:off + n].view_as(p)); off += n
    renderer.nonfinite_flag_ = flat[off:off + 2] > 0        # OR across ranks, per MLP
    sent += flat.numel() * 4
    return sent


def sync_emas(gdp):
    t = torch.tensor([gdp.sampled_oct_per_ray_, gdp.sampled_pts_per_ray_, gdp.meaningful_sampled_pts_per_ray_], dtype=torch.float64)
    if dist.get_backend() == "nccl":
        t = t.cuda()
    dist.all_reduce(t)
    t = (t / dist.get_world_size()).tolist()
    gdp.sampled_oct_per_ray_, gdp.sampled_pts_per_ray_, gdp.meaningful_sampled_pts_per_ray_ = t


def allreduce_step(prob):
    """bench.py hook: the exchange step of one training iteration."""
    allreduce_grads(prob["renderer"])
