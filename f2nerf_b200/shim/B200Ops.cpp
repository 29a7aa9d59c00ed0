// B200Ops.cpp — see B200Ops.h.  Host code stays C++/LibTorch; every kernel is behind the C ABI.
#include "B200Ops.h"
#include <ATen/cuda/CUDAContext.h>
#include "Common.h"
#include "f2nerf_b200.h"

using Tensor = torch::Tensor;

#define F2B_CHECK(expr)                                                            \
  do {                                                                             \
    int f2b_rc_ = (expr);                                                          \
    CHECK(f2b_rc_ == 0) << #expr << " -> " << f2b_rc_ << ": " << f2b_last_error(); \
  } while (0)

static void* cur_stream() { return (void*) at::cuda::getCurrentCUDAStream().stream(); }

// ------------------------------------------------------------------------------ sampler ---------
SampleResultFlex B200Sampler::GetSamples(const Tensor& rays_o_raw, const Tensor& rays_d_raw, const Tensor&) {
  Tensor rays_o = rays_o_raw.contiguous();
  Tensor rays_d = (rays_d_raw / torch::linalg_norm(rays_d_raw, 2, -1, true)).contiguous();
  const int n_rays = rays_o.size(0);
  Tensor noise;                                                        // same RNG draw as PersSampler.cu:373-381
  if (global_data_pool_->mode_ == RunningMode::VALIDATE) noise = torch::ones({1024 + n_rays + 10}, CUDAFloat);
  else noise = ((torch::rand({1024 + n_rays + 10}, CUDAFloat) - .5f) + 1.f).contiguous();
  noise.mul_(global_data_pool_->ray_march_fineness_);
  Tensor& nodes = pers_octree_->tree_nodes_gpu_;
  Tensor& trans = pers_octree_->pers_trans_gpu_;
  Tensor counts = torch::empty({std::max(n_rays, 1)}, CUDAInt), bounds = torch::empty({n_rays, 2}, CUDAInt);
  Tensor totals = torch::empty({2}, CUDAInt);
  F2B_CHECK(f2b_sampler_count(nodes.data_ptr(), nodes.numel() / 64, trans.data_ptr(), trans.numel() / 544,
                              rays_o.data_ptr<float>(), rays_d.data_ptr<float>(), noise.data_ptr<float>(), n_rays,
                              global_near_, 1e8f, sample_l_, scale_by_dis_, max_oct_intersect_per_ray_, /*count_all_hits=*/1,
                              counts.data_ptr<int>(), bounds.data_ptr<int>(), totals.data_ptr<int>(), cur_stream()));
  Tensor totals_cpu = totals.to(torch::kCPU);                           // the one host sync
  const int n_pts = totals_cpu[0].item<int>(), n_oct = totals_cpu[1].item<int>();
  if (global_data_pool_->mode_ != RunningMode::VALIDATE)
    global_data_pool_->sampled_oct_per_ray_ = global_data_pool_->sampled_oct_per_ray_ * .9f + (float(n_oct) / float(n_rays)) * .1f;
  Tensor pts = torch::empty({n_pts, 3}, CUDAFloat), dirs = torch::empty({n_pts, 3}, CUDAFloat);
  Tensor dt = torch::empty({n_pts}, CUDAFloat), t = torch::empty({n_pts}, CUDAFloat);
  Tensor anchors = torch::empty({n_pts, 3}, CUDAInt), first = torch::empty({n_rays, 1}, CUDAFloat);
  F2B_CHECK(f2b_sampler_fill(nodes.data_ptr(), nodes.numel() / 64, trans.data_ptr(), trans.numel() / 544,
                             rays_o.data_ptr<float>(), rays_d.data_ptr<float>(), noise.data_ptr<float>(), n_rays,
                             global_near_, 1e8f, sample_l_, scale_by_dis_, max_oct_intersect_per_ray_,
                             bounds.data_ptr<int>(), pts.data_ptr<float>(), dirs.data_ptr<float>(), dt.data_ptr<float>(),
                             t.data_ptr<float>(), anchors.data_ptr<int>(), first.data_ptr<float>(), cur_stream()));
  return {pts, dirs, dt, t, anchors, bounds, first};
}

std::tuple<Tensor, Tensor> B200Sampler::GetEdgeSamples(int n_pts) {
  const int n_edges = pers_octree_->edge_pool_.size();
  Tensor edge_idx = torch::randint(0, n_edges, {n_pts}, CUDAInt).contiguous();
  Tensor edge_coord = (torch::rand({n_pts, 2}, CUDAFloat) * 2.f - 1.f).contiguous();
  Tensor out_pts = torch::empty({n_pts, 2, 3}, CUDAFloat), out_idx = torch::empty({n_pts, 2}, CUDAInt);
  F2B_CHECK(f2b_edge_samples(pers_octree_->edge_pool_gpu_.data_ptr(), pers_octree_->pers_trans_gpu_.data_ptr(),
                             edge_idx.data_ptr<int>(), edge_coord.data_ptr<float>(), n_pts, out_pts.data_ptr<float>(),
                             out_idx.data_ptr<int>(), cur_stream()));
  return {out_pts, out_idx};
}

void B200Sampler::UpdateOctNodes(const SampleResultFlex& s, const Tensor& w, const Tensor& a) {
  const int n_nodes = pers_octree_->tree_nodes_.size(), n_rays = s.pts_idx_bounds.size(0);
  Tensor vote_w = torch::full({n_nodes}, -1, CUDAInt), vote_a = torch::full({n_nodes}, -1, CUDAInt);
  Tensor mark = torch::zeros({n_nodes}, CUDAInt);
  Tensor wc = w.contiguous(), ac = a.contiguous();
  F2B_CHECK(f2b_oct_mark_visit(s.pts_idx_bounds.data_ptr<int>(), n_rays, s.anchors.data_ptr<int>() + 1, 3,
                               wc.data_ptr<float>(), ac.data_ptr<float>(), vote_w.data_ptr<int>(), vote_a.data_ptr<int>(),
                               mark.data_ptr<int>(), pers_octree_->tree_visit_cnt_.data_ptr<int>(), cur_stream()));
  F2B_CHECK(f2b_oct_update_stats(vote_w.data_ptr<int>(), vote_a.data_ptr<int>(), mark.data_ptr<int>(),
                                 pers_octree_->tree_weight_stats_.data_ptr<int>(), pers_octree_->tree_alpha_stats_.data_ptr<int>(),
                                 pers_octree_->tree_nodes_gpu_.data_ptr(), n_nodes, cur_stream()));
  // milestones / compaction stay the reference's host code (PersSampler.cu:605-614)
  while (!sub_div_milestones_.empty() && sub_div_milestones_.back() <= global_data_pool_->iter_step_) {
    pers_octree_->ProcOctree(true, true, sub_div_milestones_.back() <= 0);
    pers_octree_->MarkInvisibleNodes();
    pers_octree_->ProcOctree(true, false, false);
    sub_div_milestones_.pop_back();
  }
  if (global_data_pool_->iter_step_ % compact_freq_ == 0) pers_octree_->ProcOctree(true, false, false);
}

// ------------------------------------------------------------------------------ field -----------
namespace {
struct FieldCtx : torch::CustomClassHolder {
  B200HashField* f = nullptr;
  Tensor params16, points, anchors, feat16, hidden;
};

class FieldFn : public torch::autograd::Function<FieldFn> {
public:
  static torch::autograd::variable_list forward(torch::autograd::AutogradContext* ctx, Tensor feat_pool, Tensor params,
                                                Tensor points, Tensor anchors, int64_t self_ptr) {
    auto* f = reinterpret_cast<B200HashField*>(self_ptr);
    const int n = points.size(0);
    const int local_size = ((f->pool_size_ / N_LEVELS) >> 4) << 4;
    Tensor table16 = torch::empty_like(feat_pool, CUDAHalf), params16 = torch::empty_like(params, CUDAHalf);
    F2B_CHECK(f2b_table_to_half(feat_pool.data_ptr<float>(), table16.data_ptr(), feat_pool.numel(), cur_stream()));
    F2B_CHECK(f2b_cast_f32_to_f16(params.data_ptr<float>(), params16.data_ptr(), params.numel(), 1.f, cur_stream()));
    Tensor feat16 = torch::empty({n, 32}, CUDAHalf), out16 = torch::empty({n, 16}, CUDAHalf), hidden = torch::empty({1, n, 64}, CUDAHalf);
    F2B_CHECK(f2b_hash_fwd(table16.data_ptr(), f->prim_pool_.data_ptr<int>(), f->bias_pool_.data_ptr<float>(), f->n_volumes_,
                           local_size, points.data_ptr<float>(), anchors.data_ptr<int>(), 1, n, feat16.data_ptr(), cur_stream()));
    // RNG-stream parity: the reference allocates the MLP output with torch::rand (TCNNWP.cpp:143), which the draws
    // that follow (edge samples, next iteration's noise) depend on.  Same call, result discarded.
    (void)torch::rand({(n + 127) / 128 * 128, 16}, CUDAHalf);
    F2B_CHECK(f2b_mlp_fwd(feat16.data_ptr(), params16.data_ptr(), 0, n, out16.data_ptr(), hidden.data_ptr(), cur_stream()));
    Tensor out = torch::empty({n, 16}, CUDAFloat);
    F2B_CHECK(f2b_cast_f16_to_f32(out16.data_ptr(), out.data_ptr<float>(), out.numel(), 1.f, cur_stream()));
    ctx->save_for_backward({params16, points, anchors, feat16, hidden, feat_pool});
    ctx->saved_data["self"] = self_ptr;
    return {out};
  }
  static torch::autograd::variable_list backward(torch::autograd::AutogradContext* ctx, torch::autograd::variable_list g) {
    auto sv = ctx->get_saved_variables();
    auto* f = reinterpret_cast<B200HashField*>(ctx->saved_data["self"].toInt());
    Tensor &params16 = sv[0], &points = sv[1], &anchors = sv[2], &feat16 = sv[3], &hidden = sv[4];
    const int n = points.size(0);
    const int local_size = ((f->pool_size_ / N_LEVELS) >> 4) << 4;
    const float scale = f->mlp_->loss_scale_;
    Tensor d = g[0].contiguous(), d16 = torch::empty({n, 16}, CUDAHalf), dfeat16 = torch::empty({n, 32}, CUDAHalf);
    Tensor dparams = torch::zeros({params16.numel()}, CUDAFloat), dtable = torch::zeros_like(sv[5]);
    F2B_CHECK(f2b_cast_f32_to_f16(d.data_ptr<float>(), d16.data_ptr(), d.numel(), scale, cur_stream()));
    F2B_CHECK(f2b_mlp_bwd(d16.data_ptr(), feat16.data_ptr(), hidden.data_ptr(), params16.data_ptr(), 0, n, dfeat16.data_ptr(),
                          dparams.data_ptr<float>(), cur_stream()));
    F2B_CHECK(f2b_hash_bwd(f->prim_pool_.data_ptr<int>(), f->bias_pool_.data_ptr<float>(), f->n_volumes_, local_size,
                           points.data_ptr<float>(), anchors.data_ptr<int>(), 1, n, dfeat16.data_ptr(), 1, 1.f / scale,
                           dtable.data_ptr<float>(), cur_stream()));
    dparams = dparams / scale;
    // TCNNWP.cpp:231-240: dL/dinput (the fp16 dL/dfeat rows, which overflow before the fp32 dL/dparams do) or dL/dparams
    if (!torch::all(torch::isfinite(dfeat16)).item<bool>() || !torch::all(torch::isfinite(dparams)).item<bool>()) {
      f->global_data_pool_->backward_nan_ = true;
      f->mlp_->loss_scale_ = std::max(f->mlp_->loss_scale_ / 2.f, 1.f);
    }
    return {dtable, dparams, Tensor(), Tensor(), Tensor()};
  }
};
}  // namespace

Tensor B200HashField::AnchoredQuery(const Tensor& points, const Tensor& anchors) {
  return FieldFn::apply(feat_pool_, mlp_->params_, points.contiguous(), anchors.contiguous(), reinterpret_cast<int64_t>(this))[0];
}

// ------------------------------------------------------------------------------ shader ----------
namespace {
class ShaderFn : public torch::autograd::Function<ShaderFn> {
public:
  static torch::autograd::variable_list forward(torch::autograd::AutogradContext* ctx, Tensor feats, Tensor params,
                                                Tensor dirs, int64_t self_ptr) {
    const int n = feats.size(0);
    Tensor params16 = torch::empty_like(params, CUDAHalf);
    F2B_CHECK(f2b_cast_f32_to_f16(params.data_ptr<float>(), params16.data_ptr(), params.numel(), 1.f, cur_stream()));
    // feats already hold the constant-1 channel / appearance embedding (Renderer.cpp:179-187): cast + SH only
    Tensor sh = torch::empty({n, 16}, CUDAFloat);
    F2B_CHECK(f2b_sh_encode(dirs.data_ptr<float>(), n, 4, sh.data_ptr<float>(), cur_stream()));
    Tensor x = torch::cat({feats, sh}, -1).contiguous(), x16 = torch::empty({n, 32}, CUDAHalf);
    F2B_CHECK(f2b_cast_f32_to_f16(x.data_ptr<float>(), x16.data_ptr(), x.numel(), 1.f, cur_stream()));
    Tensor raw = torch::empty({n, 16}, CUDAHalf), hidden = torch::empty({2, n, 64}, CUDAHalf), rgb = torch::empty({n, 3}, CUDAFloat);
    (void)torch::rand({(n + 127) / 128 * 128, 16}, CUDAHalf);      // RNG-stream parity (TCNNWP.cpp:143), see FieldFn
    F2B_CHECK(f2b_mlp_fwd(x16.data_ptr(), params16.data_ptr(), 1, n, raw.data_ptr(), hidden.data_ptr(), cur_stream()));
    F2B_CHECK(f2b_shader_act(raw.data_ptr(), n, rgb.data_ptr<float>(), cur_stream()));
    ctx->save_for_backward({params16, x16, hidden, raw});
    ctx->saved_data["self"] = self_ptr;
    return {rgb};
  }
  static torch::autograd::variable_list backward(torch::autograd::AutogradContext* ctx, torch::autograd::variable_list g) {
    auto sv = ctx->get_saved_variables();
    auto* s = reinterpret_cast<B200Shader*>(ctx->saved_data["self"].toInt());
    const int n = sv[1].size(0);
    const float scale = s->mlp_->loss_scale_;
    Tensor d = g[0].contiguous(), draw = torch::empty({n, 16}, CUDAHalf), din16 = torch::empty({n, 32}, CUDAHalf);
    Tensor dparams = torch::zeros({sv[0].numel()}, CUDAFloat), din = torch::empty({n, 32}, CUDAFloat);
    F2B_CHECK(f2b_shader_act_bwd(sv[3].data_ptr(), d.data_ptr<float>(), n, scale, draw.data_ptr(), cur_stream()));
    F2B_CHECK(f2b_mlp_bwd(draw.data_ptr(), sv[1].data_ptr(), sv[2].data_ptr(), sv[0].data_ptr(), 1, n, din16.data_ptr(),
                          dparams.data_ptr<float>(), cur_stream()));
    F2B_CHECK(f2b_cast_f16_to_f32(din16.data_ptr(), din.data_ptr<float>(), din.numel(), 1.f / scale, cur_stream()));
    dparams = dparams / scale;
    if (!torch::all(torch::isfinite(din)).item<bool>() || !torch::all(torch::isfinite(dparams)).item<bool>()) {   // as FieldFn
      s->global_data_pool_->backward_nan_ = true;
      s->mlp_->loss_scale_ = std::max(s->mlp_->loss_scale_ / 2.f, 1.f);
    }
    return {din.index({Slc(), Slc(0, 16)}).contiguous(), dparams, Tensor(), Tensor()};
  }
};
}  // namespace

Tensor B200Shader::Query(const Tensor& feats, const Tensor& dirs) {
  return ShaderFn::apply(feats.contiguous(), mlp_->params_, dirs.contiguous(), reinterpret_cast<int64_t>(this))[0];
}
