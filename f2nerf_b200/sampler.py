"""PersSampler — host-side mirror of the reference's perspective-warp octree sampler operator
(``src/PtsSampler/PersSampler.h:75-96``, ``PersSampler.cu:317-615``) over the C ABI.

Same method names and argument meaning as the reference class (``GetSamples``, ``GetEdgeSamples``,
``UpdateOctNodes``, ``States``, ``LoadStates``); tensors are CUDA, contiguous, f32 / i32 like the
reference's ``CUDAFloat`` / ``CUDAInt``.  RNG draws use the same torch calls in the same order as the
reference so that a shared ``torch.manual_seed`` reproduces its noise (``PersSampler.cu:377,456-457``).
Octree (re)construction / compaction (``PersOctree::ProcOctree``) is out of scope (SURVEY §8f N2):
blobs come from a reference checkpoint / dump or from ``tests/synth_scene.py`` (synthetic scenes for tests and the bench).
"""
from dataclasses import dataclass

import torch

from . import ops
from ._lib import call, stream

MAX_SAMPLE_PER_RAY = 1024
INIT_NODE_STAT = 1000
TRAIN, VALIDATE = 0, 1


@dataclass
class SampleResultFlex:
    """``struct SampleResultFlex`` (src/PtsSampler/PtsSampler.h:13-22)."""
    pts: torch.Tensor              # [n_all_pts, 3] warped coordinates
    dirs: torch.Tensor             # [n_all_pts, 3]
    dt: torch.Tensor               # [n_all_pts]
    t: torch.Tensor                # [n_all_pts]
    anchors: torch.Tensor          # [n_all_pts, 3] i32: trans_idx, node idx, 0
    pts_idx_bounds: torch.Tensor   # [n_rays, 2] i32 start, end
    first_oct_dis: torch.Tensor    # [n_rays, 1]


class SlotSamples:
    """Result of the one-pass march in its native layout: ray ``r`` owns slots ``[r*1024, r*1024 + counts[r])`` of
    the sampler's persistent scratch (pts, dt, t, anchors[0:2]; 28 B/sample).  The renderer runs the early-stop pass
    on this layout directly, so the cumsum / host sync / gather of ``PersSampler::GetSamples`` (PersSampler.cu:395-434)
    only happens when somebody asks for the reference's ``SampleResultFlex`` (:meth:`PersSampler.materialize`).
    Valid until the sampler's next march."""
    slot = MAX_SAMPLE_PER_RAY

    def __init__(self, sampler, rays_o, rays_d, noise, bufs, generation):
        self.sampler, self.rays_o, self.rays_d, self.noise, self.generation = sampler, rays_o, rays_d, noise, generation
        self.n_rays = rays_o.shape[0]
        n = self.n_rays * self.slot
        self.s_pts, self.s_dt, self.s_t, self.s_anchors = bufs[0][:n], bufs[1][:n], bufs[2][:n], bufs[3][:n]
        dev = rays_o.device
        R = max(self.n_rays, 1)
        self.counts = torch.empty((R,), dtype=torch.int32, device=dev)
        self.chunk_bounds = torch.empty((R, 2), dtype=torch.int32, device=dev)      # the march's cumsum bounds (unused by the renderer)
        self.slot_bounds = torch.empty((self.n_rays, 2), dtype=torch.int32, device=dev)
        self.first_oct_dis = torch.empty((self.n_rays, 1), dtype=torch.float32, device=dev)
        self.totals = torch.empty((2,), dtype=torch.int32, device=dev)              # [samples, octree hits], written by the march


class LazySampleResult:
    """``Renderer::sample_result_`` on demand: attribute access materialises the reference-layout SampleResultFlex
    (one scan + host sync + gather) from the slot layout; the training path never touches it."""

    def __init__(self, slots):
        object.__setattr__(self, "_slots", slots)
        object.__setattr__(self, "_flex", None)

    def _get(self):
        if self._flex is None:
            object.__setattr__(self, "_flex", self._slots.sampler.materialize(self._slots))
        return self._flex

    def __getattr__(self, name):
        return getattr(self._get(), name)


class GlobalDataPool:
    """The cross-module scalars of ``GlobalDataPool`` (src/Utils/GlobalDataPool.h:10-32) the path reads/writes."""

    def __init__(self):
        self.mode_ = TRAIN
        self.n_volumes_ = 1
        self.iter_step_ = 0
        self.sampled_oct_per_ray_ = 16.0
        self.sampled_pts_per_ray_ = 512.0
        self.meaningful_sampled_pts_per_ray_ = 512.0
        self.learning_rate_ = 1.0
        self.ray_march_fineness_ = 1.0
        self.gradient_scaling_progress_ = 1.0
        self.backward_nan_ = False


class PersSampler:
    def __init__(self, global_data_pool, tree_nodes, pers_trans, edge_pool=None, *, near=0.05, sample_l=1.0 / 256,
                 scale_by_dis=False, max_oct_intersect_per_ray=1024, device="cuda"):
        self.global_data_pool_ = global_data_pool
        dev = torch.device(device)
        as_u8 = lambda b: torch.as_tensor(b, dtype=torch.uint8).reshape(-1).to(dev).contiguous()
        self.tree_nodes_gpu_ = as_u8(tree_nodes)
        self.pers_trans_gpu_ = as_u8(pers_trans)
        self.edge_pool_gpu_ = as_u8(edge_pool) if edge_pool is not None else torch.zeros(0, dtype=torch.uint8, device=dev)
        if self.tree_nodes_gpu_.numel() % 64 or self.pers_trans_gpu_.numel() % 544 or self.edge_pool_gpu_.numel() % 64:
            raise ValueError("PersSampler: blob sizes must be multiples of sizeof(TreeNode)=64 / TransInfo=544 / EdgePool=64")
        n_nodes = self.tree_nodes_gpu_.numel() // 64
        self.tree_weight_stats_ = torch.full((n_nodes,), INIT_NODE_STAT, dtype=torch.int32, device=dev)
        self.tree_alpha_stats_ = torch.full((n_nodes,), INIT_NODE_STAT, dtype=torch.int32, device=dev)
        self.tree_visit_cnt_ = torch.zeros((n_nodes,), dtype=torch.int32, device=dev)
        self.global_near_, self.sample_l_, self.scale_by_dis_ = float(near), float(sample_l), bool(scale_by_dis)
        self.max_oct_intersect_per_ray_ = int(max_oct_intersect_per_ray)
        self.sub_div_milestones_ = []
        self.exact_oct_stat_ = False         # True: run the traversal to exhaustion for the exact "OctSamples" log EMA
        self.vote_allreduce_ = None          # set by f2nerf_b200.dist.install_vote_sync under data parallelism
        global_data_pool.n_volumes_ = self.pers_trans_gpu_.numel() // 544

    @property
    def n_nodes(self):
        return self.tree_nodes_gpu_.numel() // 64

    @property
    def n_edges(self):
        return self.edge_pool_gpu_.numel() // 64

    def make_noise(self, n_rays, device):
        gdp = self.global_data_pool_
        n = MAX_SAMPLE_PER_RAY + n_rays + 10
        if gdp.mode_ == VALIDATE:
            noise = torch.ones(n, dtype=torch.float32, device=device)
        else:
            noise = ((torch.rand(n, dtype=torch.float32, device=device) - .5) + 1.).contiguous()
        return noise.mul_(gdp.ray_march_fineness_)

    def GetSamples(self, rays_o_raw, rays_d_raw, bounds_raw=None, rays_noise=None):
        """PersSampler::GetSamples (PersSampler.cu:317-434).  ``bounds_raw`` is ignored like in the
        reference (it marches [global_near_, 1e8]).  One host sync (sample total) instead of two."""
        slots = self.begin_march(rays_o_raw, rays_d_raw, rays_noise)
        self.march_rays(slots)
        return self.materialize(slots)

    # ---- slot-layout pieces (used by Renderer.Render; GetSamples = begin_march + march_rays + materialize) ----------
    def begin_march(self, rays_o_raw, rays_d_raw, rays_noise=None, normalised=False, lane=0):
        """Normalise directions, draw the noise (PersSampler.cu:373-380) and bind the scratch; launches no march yet.
        ``lane`` > 0 selects an additional scratch set (whole-image rendering keeps two chunks in flight on two streams);
        lane 0 is the training scratch whose results die with the next lane-0 march."""
        rays_o = rays_o_raw.contiguous()
        rays_d = rays_d_raw if normalised else (rays_d_raw / torch.linalg.norm(rays_d_raw, 2, -1, True)).contiguous()
        n_rays = rays_o.shape[0]
        if rays_noise is None:
            rays_noise = self.make_noise(n_rays, rays_o.device)
        if lane:
            return SlotSamples(self, rays_o, rays_d, rays_noise, self._scratch(n_rays, rays_o.device, lane), -int(lane))
        self._generation = getattr(self, "_generation", 0) + 1
        return SlotSamples(self, rays_o, rays_d, rays_noise, self._scratch(n_rays, rays_o.device), self._generation)

    def march_rays(self, slots):
        """March the batch into its slots on the CURRENT stream (no host sync)."""
        n = slots.n_rays
        if n <= 0:
            return
        call("f2b_sampler_march", self.tree_nodes_gpu_, self.n_nodes, self.pers_trans_gpu_, self.pers_trans_gpu_.numel() // 544,
             slots.rays_o, slots.rays_d, slots.noise, n, float(self.global_near_), 1e8, float(self.sample_l_),
             int(self.scale_by_dis_), int(self.max_oct_intersect_per_ray_), int(bool(self.exact_oct_stat_)),
             slots.s_pts, slots.s_dt, slots.s_t, slots.s_anchors, slots.counts, slots.chunk_bounds, slots.totals,
             slots.first_oct_dis, stream())
        call("f2b_slot_bounds", slots.counts, n, slots.slot, 0, slots.slot_bounds, stream())

    # ---- software pipelining of the march (it reads no trainable state: only rays, noise and the octree) ------------------
    def prefetch_march(self, rays_o_raw, rays_d_raw, stream, pending_rand_numel=()):
        """March the NEXT batch now, on ``stream`` (a side stream that already carries this iteration's octree votes, so the
        march sees the pruned tree exactly as a march issued at the start of the next ``Render`` would), while the caller's
        main stream runs loss + backward of the current batch.  The next ``begin_march`` with the same ray tensors picks the
        result up instead of marching.

        RNG-stream parity: the noise is drawn from the Philox position it will have when the next Render starts —
        ``pending_rand_numel`` lists the ``torch.rand`` sizes still to be consumed before then (the GradientScaling burns of
        the coming backward) — and the generator is then put back, so a prefetched run draws the very same numbers as an
        unpipelined one under the same seed."""
        from .rng import rand_philox_offset
        dev = rays_o_raw.device
        main = torch.cuda.current_stream(dev)
        n_rays = rays_o_raw.shape[0]
        gen = torch.cuda.default_generators[dev.index if dev.index is not None else torch.cuda.current_device()]
        here = gen.get_offset()
        ahead = sum(rand_philox_offset(int(n), dev) for n in pending_rand_numel)
        gen.set_offset(here + ahead)
        noise = self.make_noise(n_rays, dev)                       # drawn on the main stream (tiny), consumed by the side stream
        noise_inc = gen.get_offset() - (here + ahead)
        gen.set_offset(here)
        rays_o = rays_o_raw.contiguous()
        rays_d = (rays_d_raw / torch.linalg.norm(rays_d_raw, 2, -1, True)).contiguous()
        slots = self.begin_march(rays_o, rays_d, noise, normalised=True)
        ev = torch.cuda.Event()
        ev.record(main)                                            # the ray upload / noise draw queued so far precede the march (the
        stream.wait_event(ev)                                      # scratch it writes is the OTHER set: no reader to wait for)
        with torch.cuda.stream(stream):
            self.march_rays(slots)
            ring = self.__dict__.setdefault("_pinned_totals", [torch.empty((2,), dtype=torch.int32).pin_memory() for _ in range(4)])
            self._pinned_turn = (getattr(self, "_pinned_turn", -1) + 1) % len(ring)
            host_totals = ring[self._pinned_turn]
            host_totals.copy_(slots.totals, non_blocking=True)         # [samples, octree hits] of the batch, on the host by the
            done = torch.cuda.Event()                                  # time the consuming Render asks (it waits on `done`)
            done.record(stream)
        # no record_stream: every tensor the side stream touches stays referenced from the prefetch record / the slots until the
        # consuming Render has made the main stream wait on ``done``, so it cannot be recycled under the march
        self._prefetched = dict(key=(rays_o_raw.data_ptr(), rays_d_raw.data_ptr(), n_rays, rays_o_raw._version, rays_d_raw._version),
                                slots=slots, done=done, noise_inc=noise_inc, host_totals=host_totals, tree=self._tree_id(),
                                mode=self.global_data_pool_.mode_, fineness=self.global_data_pool_.ray_march_fineness_)

    def _tree_id(self):
        """The octree a march ran on: the tensor itself and its version counter, not its address.  ProcOctree and LoadStates
        replace the tensor (a freed tree's block can come back from the caching allocator for a later one, so an address proves
        nothing; the record also keeps the marched tree alive until the side stream is done reading it); a host-side in-place
        write (``copy_``) bumps the version.  The votes' pruning (apply_votes) writes through the raw pointer and bumps nothing:
        it precedes the prefetched march on its stream.  MarkInvisibleNodes, the other raw-pointer writer, drops the prefetch."""
        return self.tree_nodes_gpu_, self.tree_nodes_gpu_._version

    def take_prefetched(self, rays_o_raw, rays_d_raw):
        """The prefetched march for exactly these ray tensors (and an unchanged octree / mode / fineness), or None."""
        pf, self._prefetched = getattr(self, "_prefetched", None), None
        if pf is None:
            return None
        gdp = self.global_data_pool_
        key = (rays_o_raw.data_ptr(), rays_d_raw.data_ptr(), rays_o_raw.shape[0], rays_o_raw._version, rays_d_raw._version)
        tree, version = pf["tree"]
        if (key != pf["key"] or tree is not self.tree_nodes_gpu_ or version != tree._version or pf["mode"] != gdp.mode_
                or pf["fineness"] != gdp.ray_march_fineness_ or pf["slots"].generation != getattr(self, "_generation", 0)):
            # (a march in between took the other scratch set and bumped the generation: the prefetched slots are stale by order)
            torch.cuda.current_stream(rays_o_raw.device).wait_event(pf["done"])      # its buffers are released behind the march
            return None
        return pf

    def note_totals(self, n_rays, n_all_oct):
        """EMA of octree intersections per ray (PersSampler.cu:378-379); called once the host knows the totals."""
        gdp = self.global_data_pool_
        if gdp.mode_ != VALIDATE and n_rays > 0:
            gdp.sampled_oct_per_ray_ = gdp.sampled_oct_per_ray_ * .9 + (n_all_oct / n_rays) * .1

    def materialize(self, slots):
        """Slot layout -> the reference's SampleResultFlex (cumsum bounds, gathered arrays).  One host sync."""
        if slots.generation >= 0 and slots.generation < getattr(self, "_generation", 0) - 1:
            raise RuntimeError("SampleResult: the sampler has marched twice since; this result's scratch slots were overwritten")
        R, dev = slots.n_rays, slots.rays_o.device
        bounds = torch.empty((R, 2), dtype=torch.int32, device=dev)
        total = torch.zeros((1,), dtype=torch.int32, device=dev)
        call("f2b_count_scan", slots.counts, R, bounds, total, stream())
        n_all_pts, _, n_all_oct = torch.cat([total, slots.totals]).tolist()              # the one sync
        if not getattr(slots, "noted", False):
            self.note_totals(R, n_all_oct)
            slots.noted = True
        pts, dirs, dt, t, anchors = ops.sampler_gather(slots.rays_d, bounds, n_all_pts,
                                                       (slots.s_pts, slots.s_dt, slots.s_t, slots.s_anchors))
        return SampleResultFlex(pts, dirs, dt, t, anchors, bounds, slots.first_oct_dis)

    def _scratch(self, n_rays, dev, lane=0):
        """Persistent one-pass march scratch: a 1024-sample slot per ray (28 B/sample), grown on demand."""
        cap = max(n_rays, 1) * MAX_SAMPLE_PER_RAY
        f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        if lane:
            pool = self.__dict__.setdefault("_scratch_lanes", {})
            b = pool.get(lane)
            if b is None or b[1].numel() < cap or b[0].device != dev:
                b = pool[lane] = (f(cap, 3), f(cap), f(cap), torch.empty((cap, 2), dtype=torch.int32, device=dev))
            return b
        # two sets, used alternately: the march of batch i+1 can be issued while batch i's samples are still being read
        # (Renderer.Render launches it right behind the occupancy votes, before the compaction of batch i has run)
        sets = self.__dict__.setdefault("_scratch_sets", [None, None])
        self._scratch_turn = 1 - getattr(self, "_scratch_turn", 1)
        b = sets[self._scratch_turn]
        if b is None or b[1].numel() < cap or b[0].device != dev:
            b = sets[self._scratch_turn] = (f(cap, 3), f(cap), f(cap), torch.empty((cap, 2), dtype=torch.int32, device=dev))
        return b

    def GetEdgeSamples(self, n_pts):
        """PersSampler::GetEdgeSamples (PersSampler.cu:454-473): (out_pts [n,2,3], out_idx [n,2])."""
        if self.n_edges <= 0:
            raise RuntimeError("GetEdgeSamples: empty edge pool (needs >= 2 face-adjacent valid leaves)")
        dev = self.tree_nodes_gpu_.device
        edge_idx = torch.randint(0, self.n_edges, (n_pts,), dtype=torch.int32, device=dev).contiguous()
        edge_coord = (torch.rand((n_pts, 2), dtype=torch.float32, device=dev) * 2. - 1.).contiguous()
        return ops.edge_samples(self.edge_pool_gpu_, self.pers_trans_gpu_, edge_idx, edge_coord)

    def UpdateOctNodes(self, sample_result, sampled_weight, sampled_alpha):
        """PersSampler::UpdateOctNodes (PersSampler.cu:536-603) without the milestone/compaction calls."""
        n_pts = sample_result.anchors.shape[0]
        if sampled_weight.shape[0] != n_pts or sampled_alpha.shape[0] != n_pts:
            raise ValueError("UpdateOctNodes: weight/alpha length must equal the number of samples")
        self.update_oct_nodes_raw(sample_result.pts_idx_bounds, sample_result.anchors, sampled_weight.contiguous(),
                                  sampled_alpha.contiguous())

    def update_oct_nodes_raw(self, bounds, anchors, sampled_weight, sampled_alpha):
        """Same on any sample layout: ``bounds`` [R,2] index rows of ``anchors`` [*, 2 or 3] (node index in column 1)
        and of the weight / alpha arrays (the renderer passes the march's slot layout)."""
        n_nodes, n_rays = self.n_nodes, bounds.shape[0]
        dev = self.tree_nodes_gpu_.device
        vote_w = torch.full((n_nodes,), -1, dtype=torch.int32, device=dev)
        vote_a = torch.full((n_nodes,), -1, dtype=torch.int32, device=dev)
        mark = torch.zeros((n_nodes,), dtype=torch.int32, device=dev)
        stride = anchors.shape[1]
        oct_idx = anchors.reshape(-1)[1:]                                        # anchors[:,1] with the row stride
        call("f2b_oct_mark_visit", bounds, n_rays, oct_idx.data_ptr(), stride,
             sampled_weight, sampled_alpha, vote_w, vote_a, mark, self.tree_visit_cnt_, stream())
        if self.vote_allreduce_ is not None:                                     # DP: identical pruning on every rank
            self.vote_allreduce_(vote_w, vote_a, mark, self.tree_visit_cnt_)
        self.last_votes_ = (vote_w, vote_a, mark)
        self.apply_votes(vote_w, vote_a, mark)

    # ---- octree maintenance on the device (SURVEY 8f N2) --------------------------------------------------------
    def ProcOctree(self, compact=True, subdivide=False, brute_force=False):
        """PersOctree::ProcOctree (PersSampler.cpp:120-330) without leaving the device: prune dead leaves, collapse
        single-child chains, renumber, optionally split every leaf visited more than 4 times (or all, ``brute_force``).
        Same numbering / links / statistics as the reference; one 4-byte readback (the new node count)."""
        if not compact:
            raise NotImplementedError("ProcOctree(compact=False): every call site of the reference compacts (PersSampler.cu:604-614)")
        n, dev = self.n_nodes, self.tree_nodes_gpu_.device
        work_nodes = torch.empty((n * 64,), dtype=torch.uint8, device=dev)
        work_i32 = torch.empty((5 * n + 2,), dtype=torch.int32, device=dev)
        cap = 9 * n if subdivide else n
        nodes_out = torch.empty((cap * 64,), dtype=torch.uint8, device=dev)
        w_out = torch.empty((cap,), dtype=torch.int32, device=dev)
        a_out = torch.empty((cap,), dtype=torch.int32, device=dev)
        n_out = torch.zeros((1,), dtype=torch.int32, device=dev)
        call("f2b_octree_proc", self.tree_nodes_gpu_, self.tree_weight_stats_, self.tree_alpha_stats_, self.tree_visit_cnt_, n,
             int(bool(subdivide)), int(bool(brute_force)), work_nodes, work_i32, nodes_out, w_out, a_out, n_out, stream())
        m = int(n_out.item())                                                    # the only host round trip
        self.tree_nodes_gpu_ = nodes_out[:m * 64].clone()
        self.tree_weight_stats_, self.tree_alpha_stats_ = w_out[:m].clone(), a_out[:m].clone()
        self.tree_visit_cnt_ = torch.zeros((m,), dtype=torch.int32, device=dev)
        return m

    def MarkInvisibleNodes(self, intri, w2c, bounds):
        """PersOctree::MarkInvisibleNodes (PersSampler.cu:645-680): intri [n,3,3], w2c [n,3,4], bounds [n,2] of the
        training cameras (the reference keeps them in PersOctree; here the caller passes them)."""
        f = lambda t: torch.as_tensor(t, dtype=torch.float32).to(self.tree_nodes_gpu_.device).contiguous()
        intri, w2c, bounds = f(intri), f(w2c), f(bounds)
        pf, self._prefetched = getattr(self, "_prefetched", None), None
        if pf is not None:                                                       # a prefetched march reads the tree written below
            torch.cuda.current_stream(self.tree_nodes_gpu_.device).wait_event(pf["done"])
        call("f2b_octree_mark_invisible", self.tree_nodes_gpu_, self.n_nodes, intri, w2c, bounds, intri.shape[0], stream())

    def maintain(self, cameras=None, compact_freq=1000):
        """The tail of PersSampler::UpdateOctNodes (PersSampler.cu:604-614): subdivision milestones, then the periodic
        compaction.  ``cameras`` = (intri, w2c, bounds) for MarkInvisibleNodes (skipped when None)."""
        it = self.global_data_pool_.iter_step_
        while self.sub_div_milestones_ and self.sub_div_milestones_[-1] <= it:
            self.ProcOctree(True, True, self.sub_div_milestones_[-1] <= 0)
            if cameras is not None:
                self.MarkInvisibleNodes(*cameras)
            self.ProcOctree(True, False, False)
            self.sub_div_milestones_.pop()
        if compact_freq and it % compact_freq == 0:
            self.ProcOctree(True, False, False)

    def apply_votes(self, vote_w, vote_a, mark):
        call("f2b_oct_update_stats", vote_w, vote_a, mark, self.tree_weight_stats_, self.tree_alpha_stats_,
             self.tree_nodes_gpu_, self.n_nodes, stream())

    def States(self):
        """PersSampler::States (PersSampler.cpp:692-701): same order / dtypes as the reference checkpoint."""
        ms = torch.tensor(self.sub_div_milestones_, dtype=torch.int32, device=self.tree_nodes_gpu_.device)
        return [self.tree_nodes_gpu_, self.pers_trans_gpu_, self.tree_visit_cnt_, ms]

    def LoadStates(self, states, idx):
        dev = self.tree_nodes_gpu_.device
        self.tree_nodes_gpu_ = states[idx].clone().to(dev).contiguous(); idx += 1
        self.pers_trans_gpu_ = states[idx].clone().to(dev).contiguous(); idx += 1
        self.tree_visit_cnt_ = states[idx].clone().to(dev).contiguous(); idx += 1
        self.sub_div_milestones_ = states[idx].cpu().tolist(); idx += 1
        n_nodes = self.n_nodes
        self.tree_weight_stats_ = torch.full((n_nodes,), INIT_NODE_STAT, dtype=torch.int32, device=dev)
        self.tree_alpha_stats_ = torch.full((n_nodes,), INIT_NODE_STAT, dtype=torch.int32, device=dev)
        self.global_data_pool_.n_volumes_ = self.pers_trans_gpu_.numel() // 544
        return idx
