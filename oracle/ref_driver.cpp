// ref_driver.cpp — harness around the UNMODIFIED reference operators (Totoro97/f2-nerf @98f0daa),
// linked from the reference's own sources by oracle/Makefile.ref into oracle/_ref/ref_driver.
//
// TEST INFRASTRUCTURE ONLY (see oracle/f2_oracle.c header).  It constructs the reference's
// GlobalDataPool / Dataset / Renderer exactly like ExpRunner::ExpRunner does (src/ExpRunner.cpp:17-63),
// then (1) dumps the octree / warp / hash blobs, (2) runs PersSampler::GetSamples,
// Hash3DAnchored::AnchoredQuery, SHShader::Query and Renderer::Render (+ backward) on fixed seeded
// inputs and dumps every boundary tensor as .npy, (3) times Render + backward with CUDA events.
// The dumps pin oracle/f2_oracle.c and the CUDA kernels (tests/golden/, tests/test_ref_parity.py).
//
//   ref_driver <runtime_config.yaml> <out_dir> <n_rays> [n_time_iters=0] [dump_full_grads=0] [fineness=1] [gs_progress=0.25]
//       the seeded VALIDATE and TRAIN batches run at ray-march fineness `fineness` and gradient-scaling progress `gs_progress`
//       (ExpRunner::UpdateAdaParams' values at iteration 0 of the free configs are 4 and 1); `scalars` records them with
//       use_app_emb: [near, sample_l, scale_by_dis, max_hits, n_volumes, pool_size, n_images, n_rays, use_app_emb, fineness,
//       gs_progress].  Readers take a vector of the first 8 only as use_app_emb 1, fineness 1, progress 0.25.
//   ref_driver --train <runtime_config.yaml>      what the reference's main.cpp does: ExpRunner(conf).Execute() — the
//                                                 unmodified trainer (train to end_iter, then TestImages -> mean PSNR)
//   ref_driver --steps <runtime_config.yaml> <out_dir> <n_iters> [fixed_batch=0]
//       n_iters iterations of the body of ExpRunner::Train (src/ExpRunner.cpp:81-175) from iter_step_ = 0 on the
//       deterministic parameters below: batch size from the meaningful-samples EMA (:86, or fixed_batch), RandRaysData,
//       Render, the losses with the config's schedule weights, zero_grad / backward / the backward_nan_ skip / Adam step,
//       iter_step_++ and UpdateAdaParams (:221-254).  So octree maintenance (compaction, subdivision milestones) runs
//       inside Render on the iterations the config names.  It deviates from the trainer in two ways: both torch
//       generators are reseeded (kStepSeed + k) at the start of iteration k, so that every iteration can be replayed from
//       its dumped state alone; and after each iteration a small probe is drawn from each generator and dumped — equal
//       probes mean the iteration consumed the same draws.  Per iteration, <out_dir>/it<k>/ holds the state before the
//       step, the Render outputs, the loss, the gradients (d_weights: dL/dweights as the loss hands it to Render's backward,
//       the var-loss term through the reference's WeightVar), the octree after the step and the probes.
//   ref_driver --march <runtime_config.yaml> <dir>
//       PersSampler::GetSamples alone on trees and rays a test wrote.  Every subdirectory <case> of dir holding params.npy is one
//       case, run in name order: tree_nodes.npy and pers_trans.npy (u8 blobs) replace the scene's octree and warps, rays_o /
//       rays_d [n,3] f32 are the rays (GetSamples normalises rays_d itself; rays_d_used is what it marched), params [6] f32 =
//       [train, near, sample_l, scale_by_dis, max_oct_intersect_per_ray, seed].  VALIDATE (train 0) marches with noise 1; TRAIN
//       seeds the CUDA generator with `seed` and dumps the noise GetSamples draws (fineness 1).  <case> gets pts, dirs, dt, t,
//       anchors [n,2] (the reference leaves the third column unwritten), bounds and first_oct_dis.
//   ref_driver --ops <runtime_config.yaml> <in_dir> <out_dir>
//       the two MLP operators alone, on inputs a test wrote: Hash3DAnchored::AnchoredQuery and SHShader::Query, each followed
//       by (out * g).sum().backward().  In ref_driver these are the reference's own (tiny-cuda-nn); in ref_driver_b200 always
//       this library's operator subclasses, whatever F2B_SHIM says.  Every subdirectory <case> of in_dir holding points.npy is
//       one case, run in name order on the one scene; a case reads <in_dir>/<case>/<name>.npy, or <in_dir>/<name>.npy when it
//       has none: feat_pool [pool,2], field_params, shader_params, loss_scales [2] (field, shader), points [n,3],
//       anchors [n] i32, d_out [n,16], feats [n,16], dirs [n,3], d_rgb [n,3].  The generators are seeded right before each
//       operator.  <out_dir>/<case>/ gets the outputs, the gradients (the table's as nonzero index / value), the flags
//       [backward_nan_, field loss scale, shader loss scale] after each operator's backward and a 4-value torch::rand probe of
//       the CUDA generator after each operator; <out_dir> itself gets the scene blobs.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include <iostream>
#include <experimental/filesystem>
#include <torch/torch.h>
#include <cuda_runtime.h>
#ifdef F2B_WITH_SHIM
#include "../f2nerf_b200/shim/B200Ops.h"
#include "../f2nerf_b200/shim/B200Renderer.h"
#endif
#include "ExpRunner.h"
#include "Common.h"
#include "Utils/GlobalDataPool.h"
#include "Utils/cnpy.h"
#include "Utils/CustomOps/CustomOps.h"
#include "Dataset/Dataset.h"
#include "Renderer/Renderer.h"
#include "PtsSampler/PersSampler.h"
#include "Field/Hash3DAnchored.h"
#include "Shader/SHShader.h"

namespace fs = std::experimental::filesystem::v1;
using Tensor = torch::Tensor;

static std::string g_out;

static void dump(const std::string& name, const Tensor& t_in) {
  Tensor t = t_in.detach().to(torch::kCPU).contiguous();
  std::vector<size_t> shape;
  for (auto s : t.sizes()) shape.push_back((size_t)s);
  if (shape.empty()) shape.push_back(1);
  const std::string path = g_out + "/" + name + ".npy";
  switch (t.scalar_type()) {
    case torch::kFloat32: cnpy::npy_save(path, t.data_ptr<float>(), shape); break;
    case torch::kInt32: cnpy::npy_save(path, t.data_ptr<int>(), shape); break;
    case torch::kInt64: cnpy::npy_save(path, t.data_ptr<int64_t>(), shape); break;
    case torch::kUInt8: cnpy::npy_save(path, t.data_ptr<uint8_t>(), shape); break;
    case torch::kBool: { Tensor u = t.to(torch::kUInt8); cnpy::npy_save(path, u.data_ptr<uint8_t>(), shape); break; }
    default: std::cerr << "dump: unsupported dtype for " << name << std::endl; std::exit(2);
  }
}
static void dump_scalar(const std::string& name, float v) { dump(name, torch::full({1}, v, CPUFloat)); }

// The reference's objects as ExpRunner::ExpRunner builds them, with the deterministic parameters below and, in
// ref_driver_b200, this library's drop-in installed.
struct Scene {
  std::unique_ptr<GlobalDataPool> gdp;
  std::unique_ptr<Dataset> dataset;
  std::unique_ptr<Renderer> renderer;
  PersSampler* sampler = nullptr;
  Hash3DAnchored* field = nullptr;
  SHShader* shader = nullptr;
};

static Scene make_scene(const std::string& conf_path, bool fixed_lr, bool ops_level = false) {
  Scene sc;
  torch::manual_seed(2022);   // main.cpp:8
  sc.gdp = std::make_unique<GlobalDataPool>(conf_path);
  GlobalDataPool* gdp = sc.gdp.get();
  gdp->base_exp_dir_ = gdp->config_["base_exp_dir"].as<std::string>();
  fs::create_directories(gdp->base_exp_dir_);
  if (fixed_lr) gdp->learning_rate_ = 1e-2f;
  sc.dataset = std::make_unique<Dataset>(gdp);
  sc.renderer = std::make_unique<Renderer>(gdp, sc.dataset->n_images_);
  auto& dataset = sc.dataset;
  auto& renderer = sc.renderer;
  auto* sampler = dynamic_cast<PersSampler*>(renderer->pts_sampler_.get());
  auto* field = dynamic_cast<Hash3DAnchored*>(renderer->scene_field_.get());
  auto* shader = dynamic_cast<SHShader*>(renderer->shader_.get());
  CHECK(sampler && field && shader);

  // ---- deterministic, non-trivial parameters (reproducible from the CPU generator in Python) ----
  {
    auto g = at::detail::createCPUGenerator(1234);
    Tensor feat = (torch::rand({field->pool_size_, 2}, g, CPUFloat) * 2.f - 1.f);      // U(-1,1)
    field->feat_pool_.data().copy_(feat.to(torch::kCUDA));
    field->mlp_->params_.data().mul_(4.f);          // wider density range so early stop triggers
    renderer->app_emb_.data().copy_((torch::rand({dataset->n_images_, 16}, g, CPUFloat) * .2f - .1f).to(torch::kCUDA));
  }

#ifdef F2B_WITH_SHIM
  // ---- ref_driver_b200 only.  Default (F2B_SHIM unset or "fused"): the body of Renderer::Render is the fused B200 host
  // (f2nerf_b200/shim/B200Renderer.cpp) working on the reference's own operator objects.  F2B_SHIM=ops: the operator-level
  // drop-in — the reference's OWN Renderer::Render / autograd / loss drive this library's subclasses (INTEGRATION.md): same octree
  // object, same parameters.  Either way every dump below is directly comparable with the pure-reference run of
  // oracle/_ref/ref_driver.  Never built into ref_driver (the reference arm stays unmodified).  ``ops_level`` (--ops) installs
  // the operator subclasses whatever F2B_SHIM says.
  const char* shim_env = std::getenv("F2B_SHIM");
  const bool shim_ops = ops_level || (shim_env && std::string(shim_env) == "ops");
  if (shim_ops) {
    f2b_render_use_reference(true);
    auto b_sampler = std::make_unique<B200Sampler>(gdp);
    b_sampler->pers_octree_ = std::move(sampler->pers_octree_);          // the very same octree / warps / edge pool
    auto b_field = std::make_unique<B200HashField>(gdp);
    b_field->LoadStates(field->States(), 0);
    auto b_shader = std::make_unique<B200Shader>(gdp);
    b_shader->LoadStates(shader->States(), 0);
    // Renderer::OptimParamGroups / States / LoadStates walk the sub-pipes the constructor registered (Renderer.cpp:28-35,
    // Pipe.cpp): point them at the replacements, or they would reach the destroyed originals
    for (auto& p : renderer->sub_pipes_) {
      if (p == sampler) p = b_sampler.get();
      else if (p == field) p = b_field.get();
      else if (p == shader) p = b_shader.get();
    }
    renderer->pts_sampler_ = std::move(b_sampler);
    renderer->scene_field_ = std::move(b_field);
    renderer->shader_ = std::move(b_shader);
    sampler = dynamic_cast<PersSampler*>(renderer->pts_sampler_.get());
    field = dynamic_cast<Hash3DAnchored*>(renderer->scene_field_.get());
    shader = dynamic_cast<SHShader*>(renderer->shader_.get());
    CHECK(sampler && field && shader);
    std::printf("ref_driver_b200: PersSampler / Hash3DAnchored / SHShader replaced by the B200 subclasses\n");
  } else {
    f2b_render_keep_samples(true);                                       // the dumps read renderer->sample_result_
    std::printf("ref_driver_b200: Renderer::Render replaced by the fused B200 host\n");
  }
#endif
  sc.sampler = sampler; sc.field = field; sc.shader = shader;
  return sc;
}

static void dump_scene(const Scene& sc, int n_rays) {
  auto* sampler = sc.sampler; auto* field = sc.field; auto* shader = sc.shader;
  dump("tree_nodes", sampler->pers_octree_->tree_nodes_gpu_);
  dump("pers_trans", sampler->pers_octree_->pers_trans_gpu_);
  dump("edge_pool", sampler->pers_octree_->edge_pool_gpu_);
  dump("search_order", sampler->pers_octree_->node_search_order_);
  dump("prim_pool", field->prim_pool_);
  dump("bias_pool", field->bias_pool_);
  dump("field_mlp_params", field->mlp_->params_);
  dump("shader_mlp_params", shader->mlp_->params_);
  dump("app_emb", sc.renderer->app_emb_);
  Tensor s = torch::zeros({11}, CPUFloat);
  s[0] = sampler->global_near_; s[1] = sampler->sample_l_; s[2] = sampler->scale_by_dis_ ? 1.f : 0.f;
  s[3] = float(sampler->max_oct_intersect_per_ray_); s[4] = float(field->n_volumes_);
  s[5] = float(field->pool_size_); s[6] = float(sc.dataset->n_images_); s[7] = float(n_rays);
  s[8] = sc.renderer->use_app_emb_ ? 1.f : 0.f;
  s[9] = sc.gdp->ray_march_fineness_; s[10] = sc.gdp->gradient_scaling_progress_;
  dump("scalars", s);
}

static int run_steps(const std::string& conf_path, const std::string& out_root, int n_iters, int fixed_batch);
static int run_ops(const std::string& conf_path, const std::string& in_dir, const std::string& out_root);
static int run_march(const std::string& conf_path, const std::string& dir);

int main(int argc, char** argv) {
  if (argc >= 4 && std::string(argv[1]) == "--march") return run_march(argv[2], argv[3]);
  if (argc >= 5 && std::string(argv[1]) == "--ops") return run_ops(argv[2], argv[3], argv[4]);
  if (argc >= 3 && std::string(argv[1]) == "--train") {     // main.cpp:6-13 verbatim in behaviour
    torch::manual_seed(2022);
    auto exp_runner = std::make_unique<ExpRunner>(argv[2]);
    exp_runner->Execute();
    return 0;
  }
  if (argc >= 5 && std::string(argv[1]) == "--steps")
    return run_steps(argv[2], argv[3], std::atoi(argv[4]), argc > 5 ? std::atoi(argv[5]) : 0);
  if (argc < 4) {
    std::fprintf(stderr, "usage: ref_driver <config.yaml> <out_dir> <n_rays> [n_time_iters] [dump_full_grads] [fineness] [gs_progress]\n"
                         "       ref_driver --steps <config.yaml> <out_dir> <n_iters> [fixed_batch]\n"
                         "       ref_driver --ops <config.yaml> <in_dir> <out_dir>\n"
                         "       ref_driver --march <config.yaml> <dir>\n");
    return 1;
  }
  const std::string conf_path = argv[1];
  g_out = argv[2];
  const int n_rays = std::atoi(argv[3]);
  const int n_time = argc > 4 ? std::atoi(argv[4]) : 0;
  const int full_grads = argc > 5 ? std::atoi(argv[5]) : 0;
  const float fineness = argc > 6 ? std::strtof(argv[6], nullptr) : 1.f;
  const float gs_progress = argc > 7 ? std::strtof(argv[7], nullptr) : 0.25f;   // < 1 exercises GradientScaling
  fs::create_directories(g_out);

  Scene sc = make_scene(conf_path, true);
  GlobalDataPool* gdp = sc.gdp.get();
  auto& dataset = sc.dataset;
  auto& renderer = sc.renderer;
  auto* sampler = sc.sampler;
  auto* field = sc.field;
  auto* shader = sc.shader;

  // ---- scene blobs & scalars (the fineness and progress both seeded batches run at are part of them) ----------------
  gdp->ray_march_fineness_ = fineness;
  gdp->gradient_scaling_progress_ = gs_progress;
  dump_scene(sc, n_rays);

  // ---- rays ---------------------------------------------------------------------------------------
  torch::manual_seed(2023);
  auto [rays, gt_colors, emb_idx] = dataset->RandRaysData(n_rays, DATA_TRAIN_SET);
  Tensor rays_o = rays.origins.contiguous(), rays_d = rays.dirs.contiguous(), bounds = rays.bounds.contiguous();
  dump("rays_o", rays_o); dump("rays_d", rays_d); dump("gt_colors", gt_colors); dump("emb_idx", emb_idx);
  dump("rays_d_normed", (rays_d / torch::linalg_norm(rays_d, 2, -1, true)).contiguous());
  {   // ray generation (SURVEY 8f N3): the camera tables and a replay of RandRaysData's CPU draws (Dataset.cpp:287-289)
    dump("ds_poses", dataset->poses_.reshape({-1, 12})); dump("ds_intri", dataset->intri_.reshape({-1, 9}));
    dump("ds_dist_params", dataset->dist_params_); dump("ds_bounds", dataset->bounds_); dump("ray_bounds", bounds);
    Tensor hw = torch::zeros({2}, CUDAFloat); hw[0] = float(dataset->height_); hw[1] = float(dataset->width_);
    dump("ds_hw", hw);
    Tensor tset = torch::from_blob(dataset->train_set_.data(), {int(dataset->train_set_.size())}, CPUInt).clone().to(torch::kCUDA);
    dump("ds_train_set", tset);
    torch::manual_seed(2023);
    Tensor cam = torch::randint(int(dataset->train_set_.size()), {n_rays}, CPULong);
    Tensor ri = torch::randint(0, dataset->height_, n_rays, CPULong);
    Tensor rj = torch::randint(0, dataset->width_, n_rays, CPULong);
    dump("ray_ij", torch::stack({ri, rj}, -1).to(torch::kInt32).to(torch::kCUDA).contiguous());
    dump("ray_cam_draw", cam.to(torch::kInt32).to(torch::kCUDA).contiguous());
  }

  // ---- edge samples: the operator alone, with its RNG draws replayed next to it --------------------
  {
    torch::manual_seed(4242);
    auto [edge_pts, edge_anchors] = sampler->GetEdgeSamples(8192);
    dump("edge_pts", edge_pts); dump("edge_anchors", edge_anchors);
    torch::manual_seed(4242);
    int n_edges = sampler->pers_octree_->edge_pool_.size();
    Tensor edge_idx = torch::randint(0, n_edges, {8192}, CUDAInt);                                 // PersSampler.cu:456
    Tensor edge_coord = torch::rand({8192, 2}, CUDAFloat) * 2.f - 1.f;                             // :457
    dump("edge_idx", edge_idx); dump("edge_coord", edge_coord);
  }

  // ---- sampler, VALIDATE mode (noise == 1) --------------------------------------------------------
  gdp->iter_step_ = 1;
  gdp->mode_ = RunningMode::VALIDATE;
  {
    torch::NoGradGuard ng;
    auto s = sampler->GetSamples(rays_o, rays_d, bounds);
    dump("val_pts", s.pts); dump("val_dirs", s.dirs); dump("val_dt", s.dt); dump("val_t", s.t);
    dump("val_anchors", s.anchors.index({Slc(), Slc(0, 2)}).contiguous());
    dump("val_bounds", s.pts_idx_bounds); dump("val_first_oct_dis", s.first_oct_dis);
    Tensor feat = field->AnchoredQuery(s.pts, s.anchors.index({"...", 0}).contiguous());
    dump("val_scene_feat", feat);
    Tensor shading = torch::cat({torch::ones_like(feat.index({Slc(), Slc(0, 1)})), feat.index({Slc(), Slc(1, None)})}, 1);
    dump("val_rgb", shader->Query(shading, s.dirs));
    dump("val_sh", shader->SHEncode(s.dirs));
    auto r = renderer->Render(rays_o, rays_d, bounds, Tensor());
    dump("val_colors", r.colors); dump("val_disparity", r.disparity); dump("val_depth", r.depth);
    dump("val_weights", r.weights); dump("val_idx_start_end", r.idx_start_end);
  }

  // ---- TRAIN mode: seeded RNG, replayed once to expose the internal draws -------------------------
  gdp->mode_ = RunningMode::TRAIN;
  const int64_t seed = 777;
  Tensor stats_w0 = sampler->pers_octree_->tree_weight_stats_.clone();
  {
    torch::manual_seed(seed);
    auto r = renderer->Render(rays_o, rays_d, bounds, emb_idx);
    dump("train_colors", r.colors); dump("train_disparity", r.disparity); dump("train_depth", r.depth);
    dump("train_weights", r.weights); dump("train_idx_start_end", r.idx_start_end);
    dump("train_first_oct_dis", r.first_oct_dis); dump("train_edge_feats", r.edge_feats);
    const auto& s = renderer->sample_result_;
    dump("train_pts", s.pts); dump("train_dt", s.dt); dump("train_t", s.t);
    dump("train_anchors", s.anchors.index({Slc(), Slc(0, 2)}).contiguous()); dump("train_bounds", s.pts_idx_bounds);
    dump("train_tree_nodes_after", sampler->pers_octree_->tree_nodes_gpu_);
    dump("train_weight_stats_after", sampler->pers_octree_->tree_weight_stats_);
    dump("train_alpha_stats_after", sampler->pers_octree_->tree_alpha_stats_);
    dump("train_visit_cnt_after", sampler->pers_octree_->tree_visit_cnt_);

    // losses as ExpRunner::Train (src/ExpRunner.cpp:94-118), fixed weights
    Tensor color_loss = torch::sqrt((r.colors - gt_colors).square() + 1e-4f).mean();
    Tensor disparity_loss = r.disparity.square().mean();
    Tensor tv_loss = (r.edge_feats.index({Slc(), 0}) - r.edge_feats.index({Slc(), 1})).square().mean();
    Tensor var_loss = (CustomOps::WeightVar(r.weights, r.idx_start_end) + 1e-2).sqrt().mean();
    Tensor loss = color_loss + var_loss * 1e-2f + disparity_loss * 1e-2f + tv_loss * 1e-1f;
    dump("train_loss", loss.reshape({1}));
    loss.backward();
    dump("grad_field_mlp", field->mlp_->params_.grad());
    dump("grad_shader_mlp", shader->mlp_->params_.grad());
    if (renderer->app_emb_.grad().defined()) dump("grad_app_emb", renderer->app_emb_.grad());   // undefined when use_app_emb is false
    Tensor g = field->feat_pool_.grad().reshape({-1});
    if (full_grads) dump("grad_feat_pool", g);
    Tensor nz = torch::nonzero(g).reshape({-1});
    dump("grad_feat_pool_nz_idx", nz.to(torch::kInt32));
    dump("grad_feat_pool_nz_val", g.index({nz}));
    dump_scalar("backward_nan", gdp->backward_nan_ ? 1.f : 0.f);
    // ---- the optimizer step the trainer takes next (ExpRunner.cpp:54,136): torch::optim::Adam over the field's groups
    if (full_grads) {
      dump("feat_pool_before_adam", field->feat_pool_.detach().reshape({-1}));
      dump("field_mlp_before_adam", field->mlp_->params_.detach().reshape({-1}));
      torch::optim::Adam opt(field->OptimParamGroups());
      for (int it = 0; it < 2; it++) opt.step();                 // same gradient twice: exercises step 1 and step 2 bias corrections
      dump("feat_pool_after_adam", field->feat_pool_.detach().reshape({-1}));
      dump("field_mlp_after_adam", field->mlp_->params_.detach().reshape({-1}));
      dump_scalar("adam_lr", gdp->learning_rate_);
    }
  }
  {   // replay of the RNG draws Render made, in its order.  Every TCNNWP forward allocates its output with
      // torch::rand (TCNNWP.cpp:143), so the early-stop MLP call sits between the background and the edge draws.
    const int64_t n_all = renderer->sample_result_.pts.size(0);
    torch::manual_seed(seed);
    Tensor noise = ((torch::rand({1024 + n_rays + 10}, CUDAFloat) - .5f) + 1.f).contiguous();   // PersSampler.cu:377
    noise.mul_(gdp->ray_march_fineness_);
    Tensor bg = torch::rand({n_rays, 3}, CUDAFloat);                                               // Renderer.cpp:73
    Tensor burn = torch::rand({(n_all + 127) / 128 * 128, 16}, torch::TensorOptions().dtype(torch::kFloat16).device(torch::kCUDA));
    int n_edges = sampler->pers_octree_->edge_pool_.size();
    Tensor edge_idx = torch::randint(0, n_edges, {8192}, CUDAInt);                                 // PersSampler.cu:456
    Tensor edge_coord = torch::rand({8192, 2}, CUDAFloat) * 2.f - 1.f;                             // :457
    dump("train_noise", noise); dump("train_bg", bg); dump("train_edge_idx", edge_idx); dump("train_edge_coord", edge_coord);
  }

  // ---- timing: Render + backward, CUDA events on the default stream ------------------------------
  if (n_time > 0) {
#ifdef F2B_WITH_SHIM
    f2b_render_keep_samples(false);
#endif
    std::vector<float> ms_fwd, ms_all;
    cudaEvent_t e0, e1, e2;
    cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventCreate(&e2);
    double samples = 0, kept = 0;
    for (int it = 0; it < n_time + 5; it++) {
      gdp->iter_step_ = 1 + it * 2 + 1;      // never a multiple of compact_freq / milestone
      field->feat_pool_.mutable_grad() = Tensor(); field->mlp_->params_.mutable_grad() = Tensor();
      shader->mlp_->params_.mutable_grad() = Tensor(); renderer->app_emb_.mutable_grad() = Tensor();
      torch::cuda::synchronize();
      cudaEventRecord(e0, 0);
      auto r = renderer->Render(rays_o, rays_d, bounds, emb_idx);
      cudaEventRecord(e1, 0);
      Tensor color_loss = torch::sqrt((r.colors - gt_colors).square() + 1e-4f).mean();
      Tensor tv_loss = (r.edge_feats.index({Slc(), 0}) - r.edge_feats.index({Slc(), 1})).square().mean();
      Tensor var_loss = (CustomOps::WeightVar(r.weights, r.idx_start_end) + 1e-2).sqrt().mean();
      Tensor loss = color_loss + var_loss * 1e-2f + tv_loss * 1e-1f;
      loss.backward();
      cudaEventRecord(e2, 0);
      torch::cuda::synchronize();
      float a, b; cudaEventElapsedTime(&a, e0, e1); cudaEventElapsedTime(&b, e0, e2);
      if (it >= 5) { ms_fwd.push_back(a); ms_all.push_back(b); samples += renderer->sample_result_.pts.size(0); kept += r.weights.size(0); }
    }
    std::sort(ms_fwd.begin(), ms_fwd.end()); std::sort(ms_all.begin(), ms_all.end());
    const float mf = ms_fwd[ms_fwd.size() / 2], ma = ms_all[ms_all.size() / 2];
    // forward only, as ExpRunner::RenderWholeImage drives it (VALIDATE mode, NoGradGuard; ExpRunner.cpp:257-293)
    std::vector<float> ms_val;
    {
      torch::NoGradGuard ng;
      gdp->mode_ = RunningMode::VALIDATE;
      for (int it = 0; it < n_time + 5; it++) {
        torch::cuda::synchronize();
        cudaEventRecord(e0, 0);
        auto r = renderer->Render(rays_o, rays_d, bounds, Tensor());
        cudaEventRecord(e1, 0);
        torch::cuda::synchronize();
        float a; cudaEventElapsedTime(&a, e0, e1);
        if (it >= 5) ms_val.push_back(a);
      }
      gdp->mode_ = RunningMode::TRAIN;
    }
    std::sort(ms_val.begin(), ms_val.end());
    const float mv = ms_val[ms_val.size() / 2];
    std::printf("{\"ref_timing\": {\"n_rays\": %d, \"iters\": %d, \"ms_fwd_median\": %.4f, \"ms_fwd_bwd_median\": %.4f, "
                "\"samples_per_ray\": %.2f, \"kept_per_ray\": %.2f, \"rays_per_s\": %.1f, \"ms_validate_median\": %.4f}}\n",
                n_rays, n_time, mf, ma, samples / n_time / n_rays, kept / n_time / n_rays, n_rays / (ma * 1e-3), mv);
    FILE* f = std::fopen((g_out + "/ref_timing.json").c_str(), "w");
    std::fprintf(f, "{\"n_rays\": %d, \"iters\": %d, \"ms_fwd_median\": %.4f, \"ms_fwd_bwd_median\": %.4f, "
                 "\"samples_per_ray\": %.2f, \"kept_per_ray\": %.2f, \"rays_per_s\": %.1f, \"ms_validate_median\": %.4f}\n",
                 n_rays, n_time, mf, ma, samples / n_time / n_rays, kept / n_time / n_rays, n_rays / (ma * 1e-3), mv);
    std::fclose(f);
  }
  // ---- octree maintenance (SURVEY 8f N2): ProcOctree / MarkInvisibleNodes on a deterministically damaged tree -------
  if (full_grads) {
    auto& oct = *sampler->pers_octree_;
    const int n = (int)oct.tree_nodes_.size();
    Tensor nodes_cpu = oct.tree_nodes_gpu_.to(torch::kCPU).clone();
    TreeNode* tn = reinterpret_cast<TreeNode*>(nodes_cpu.data_ptr());
    int k = 0;
    for (int u = 0; u < n; u++)
      if (tn[u].is_leaf_node && tn[u].trans_idx >= 0 && (k++ % 5 == 0)) tn[u].trans_idx = -1;     // as MarkInvalidNodes would
    oct.tree_nodes_gpu_ = nodes_cpu.to(torch::kCUDA).contiguous();
    oct.tree_visit_cnt_ = ((torch::arange(n, CUDAInt) * 7) % 11).to(torch::kInt32).contiguous();
    dump("oct_nodes_in", oct.tree_nodes_gpu_); dump("oct_w_in", oct.tree_weight_stats_); dump("oct_a_in", oct.tree_alpha_stats_);
    dump("oct_visit_in", oct.tree_visit_cnt_);
    dump("oct_intri", oct.intri_.reshape({-1, 9})); dump("oct_w2c", oct.w2c_.reshape({-1, 12})); dump("oct_bound", oct.bound_);
    oct.ProcOctree(true, true, false);
    dump("oct_nodes_sub", oct.tree_nodes_gpu_); dump("oct_w_sub", oct.tree_weight_stats_); dump("oct_a_sub", oct.tree_alpha_stats_);
    oct.MarkInvisibleNodes();
    dump("oct_nodes_invis", oct.tree_nodes_gpu_);
    oct.ProcOctree(true, false, false);
    dump("oct_nodes_final", oct.tree_nodes_gpu_); dump("oct_w_final", oct.tree_weight_stats_); dump("oct_a_final", oct.tree_alpha_stats_);
  }
  std::printf("ref_driver: done, dumps in %s\n", g_out.c_str());
  return 0;
}

// ==================================================================================================== --steps ===
static const int64_t kStepSeed = 31000;

static void dump_octree(const std::string& prefix, PersSampler* sampler) {
  auto& oct = *sampler->pers_octree_;
  dump(prefix + "tree_nodes", oct.tree_nodes_gpu_);
  dump(prefix + "weight_stats", oct.tree_weight_stats_); dump(prefix + "alpha_stats", oct.tree_alpha_stats_);
  dump(prefix + "visit_cnt", oct.tree_visit_cnt_);
  // [count, the remaining milestones as the sampler holds them: reversed, the next one last (PersSampler.cpp:674)]
  const auto& ms = sampler->sub_div_milestones_;
  Tensor t = torch::zeros({int64_t(ms.size()) + 1}, CPUInt);
  t[0] = int(ms.size());
  for (size_t i = 0; i < ms.size(); i++) t[i + 1] = ms[i];
  dump(prefix + "milestones", t);
}

static int run_steps(const std::string& conf_path, const std::string& out_root, int n_iters, int fixed_batch) {
  Scene sc = make_scene(conf_path, false);
  GlobalDataPool* gdp = sc.gdp.get();
  Dataset* dataset = sc.dataset.get();
  Renderer* renderer = sc.renderer.get();
  auto* sampler = sc.sampler; auto* field = sc.field; auto* shader = sc.shader;
  const auto& tc = gdp->config_["train"];                                                  // ExpRunner.cpp:28-45
  const int pts_batch_size = tc["pts_batch_size"].as<int>(), end_iter = tc["end_iter"].as<int>();
  const float learning_rate = tc["learning_rate"].as<float>(), learning_rate_alpha = tc["learning_rate_alpha"].as<float>();
  const int warm_up_end_iter = tc["learning_rate_warm_up_end_iter"].as<int>();
  const float init_fineness = tc["ray_march_init_fineness"].as<float>();
  const int fineness_decay_end_iter = tc["ray_march_fineness_decay_end_iter"].as<int>();
  const float tv_loss_weight = tc["tv_loss_weight"].as<float>(), disp_loss_weight = tc["disp_loss_weight"].as<float>();
  const float var_loss_weight_max = tc["var_loss_weight"].as<float>();
  const int var_loss_start = tc["var_loss_start"].as<int>(), var_loss_end = tc["var_loss_end"].as<int>();
  const int gs_start = tc["gradient_scaling_start"].as<int>(), gs_end = tc["gradient_scaling_end"].as<int>();
  torch::optim::Adam optimizer(renderer->OptimParamGroups());                                // :54
  int iter_step = 0;
  auto update_ada_params = [&]() {                                                          // :221-254
    if (iter_step >= fineness_decay_end_iter) {
      gdp->ray_march_fineness_ = 1.f;
    } else {
      float progress = float(iter_step) / float(fineness_decay_end_iter);
      gdp->ray_march_fineness_ = std::exp(std::log(1.f) * progress + std::log(init_fineness) * (1.f - progress));
    }
    float lr_factor;
    if (iter_step >= warm_up_end_iter) {
      float progress = float(iter_step - warm_up_end_iter) / float(end_iter - warm_up_end_iter);
      lr_factor = (1.f - learning_rate_alpha) * (std::cos(progress * float(M_PI)) * .5f + .5f) + learning_rate_alpha;
    } else {
      lr_factor = float(iter_step) / float(warm_up_end_iter);
    }
    for (auto& g : optimizer.param_groups()) g.options().set_lr(learning_rate * lr_factor);
    float progress = 1.f;
    if (iter_step < gs_end) progress = std::max(0.f, (float(iter_step) - gs_start) / (gs_end - gs_start + 1e-9f));
    gdp->gradient_scaling_progress_ = progress;
  };

  gdp->mode_ = RunningMode::TRAIN;                                                          // :66
  update_ada_params();                                                                      // :76
  gdp->iter_step_ = iter_step;                                                              // :80
  g_out = out_root;
  fs::create_directories(g_out);
  dump_scene(sc, fixed_batch);
  {
    auto& oct = *sampler->pers_octree_;                  // the cameras MarkInvisibleNodes tests against
    dump("oct_intri", oct.intri_.reshape({-1, 9})); dump("oct_w2c", oct.w2c_.reshape({-1, 12})); dump("oct_bound", oct.bound_);
    dump("ds_poses", dataset->poses_.reshape({-1, 12})); dump("ds_intri", dataset->intri_.reshape({-1, 9}));
    dump("ds_dist_params", dataset->dist_params_); dump("ds_bounds", dataset->bounds_);
    Tensor hw = torch::zeros({2}, CPUFloat); hw[0] = float(dataset->height_); hw[1] = float(dataset->width_);
    dump("ds_hw", hw);
    dump("ds_train_set", torch::from_blob(dataset->train_set_.data(), {int(dataset->train_set_.size())}, CPUInt).clone());
    Tensor run = torch::zeros({4}, CPUFloat);
    run[0] = float(sampler->compact_freq_); run[1] = float(pts_batch_size); run[2] = float(kStepSeed); run[3] = float(n_iters);
    dump("run", run);
  }

  for (int k = 0; k < n_iters; k++) {
    g_out = out_root + "/it" + std::to_string(k);
    fs::create_directories(g_out);
    gdp->backward_nan_ = false;                                                             // :82
    torch::manual_seed(kStepSeed + k);                                                      // harness: replayable iterations
    const int n_rays = fixed_batch > 0 ? fixed_batch
                                       : int(pts_batch_size / gdp->meaningful_sampled_pts_per_ray_) >> 4 << 4;    // :86
    float var_loss_weight = 0.f;                                                            // :108-114
    if (iter_step > var_loss_end) var_loss_weight = var_loss_weight_max;
    else if (iter_step > var_loss_start)
      var_loss_weight = float(iter_step - var_loss_start) / float(var_loss_end - var_loss_start) * var_loss_weight_max;

    // ---- the state the step starts from
    dump("feat_pool", field->feat_pool_); dump("field_mlp_params", field->mlp_->params_);
    dump("shader_mlp_params", shader->mlp_->params_); dump("app_emb", renderer->app_emb_);
    dump_octree("", sampler);
    const int64_t nodes_before = sampler->pers_octree_->tree_nodes_gpu_.numel() / 64;
    {
      Tensor st = torch::zeros({12}, CPUFloat);
      st[0] = float(gdp->iter_step_); st[1] = float(n_rays); st[2] = gdp->ray_march_fineness_; st[3] = gdp->gradient_scaling_progress_;
      st[4] = field->mlp_->loss_scale_; st[5] = shader->mlp_->loss_scale_; st[6] = gdp->sampled_oct_per_ray_;
      st[7] = gdp->sampled_pts_per_ray_; st[8] = gdp->meaningful_sampled_pts_per_ray_; st[9] = var_loss_weight;
      st[10] = disp_loss_weight; st[11] = tv_loss_weight;
      dump("state", st);
    }

    // ---- the step
    auto [train_rays, gt_colors, emb_idx] = dataset->RandRaysData(n_rays, DATA_TRAIN_SET);   // :87
    dump("rays_o", train_rays.origins); dump("rays_d", train_rays.dirs); dump("gt_colors", gt_colors); dump("emb_idx", emb_idx);
    auto r = renderer->Render(train_rays.origins, train_rays.dirs, train_rays.bounds, emb_idx);   // :93
    if (k == 0) {
      const auto& s = renderer->sample_result_;
      dump("sample_pts", s.pts); dump("sample_dt", s.dt); dump("sample_t", s.t); dump("sample_bounds", s.pts_idx_bounds);
      dump("sample_anchors", s.anchors.index({Slc(), Slc(0, 2)}).contiguous());
    }
    Tensor pred_colors = r.colors.index({Slc(0, n_rays)});                                 // :94-118
    Tensor color_loss = torch::sqrt((pred_colors - gt_colors).square() + 1e-4f).mean();
    Tensor disparity_loss = r.disparity.square().mean();
    Tensor tv_loss = (r.edge_feats.index({Slc(), 0}) - r.edge_feats.index({Slc(), 1})).square().mean();
    Tensor var_loss = (CustomOps::WeightVar(r.weights, r.idx_start_end) + 1e-2).sqrt().mean();
    Tensor loss = color_loss + var_loss * var_loss_weight + disparity_loss * disp_loss_weight + tv_loss * tv_loss_weight;
    dump("colors", pred_colors); dump("disparity", r.disparity); dump("depth", r.depth); dump("weights", r.weights);
    dump("idx_start_end", r.idx_start_end); dump("edge_feats", r.edge_feats); dump("first_oct_dis", r.first_oct_dis);
    dump("loss", loss.reshape({1}));
    bool stepped = false;
    if (loss.requires_grad()) {                                                             // :128-138
      optimizer.zero_grad();
      if (r.weights.requires_grad()) r.weights.retain_grad();
      loss.backward();
      if (r.weights.grad().defined()) dump("d_weights", r.weights.grad());
      dump("grad_field_mlp", field->mlp_->params_.grad()); dump("grad_shader_mlp", shader->mlp_->params_.grad());
      if (renderer->app_emb_.grad().defined()) dump("grad_app_emb", renderer->app_emb_.grad());
      Tensor g = field->feat_pool_.grad().reshape({-1});
      Tensor nz = torch::nonzero(g).reshape({-1});
      dump("grad_feat_pool_nz_idx", nz.to(torch::kInt32)); dump("grad_feat_pool_nz_val", g.index({nz}));
      if (!gdp->backward_nan_) { optimizer.step(); stepped = true; }
    }
    const bool nan_skip = gdp->backward_nan_;                                               // :131-134: `continue`
    if (!nan_skip) {
      iter_step++;                                                                          // :142-143
      gdp->iter_step_ = iter_step;
      update_ada_params();                                                                  // :175
    }

    // ---- after the step: the octree (maintained inside Render), the EMAs, the two generators
    dump_octree("after_", sampler);
    long reused = 0, fresh = 0;
#ifdef F2B_WITH_SHIM
    f2b_render_grad_storage_counts(&reused, &fresh);
#endif
    Tensor af = torch::zeros({8}, CPUFloat);
    af[0] = float(gdp->iter_step_); af[1] = gdp->sampled_oct_per_ray_; af[2] = gdp->sampled_pts_per_ray_;
    af[3] = gdp->meaningful_sampled_pts_per_ray_; af[4] = nan_skip ? 1.f : 0.f; af[5] = float(reused); af[6] = float(fresh);
    af[7] = stepped ? 1.f : 0.f;
    dump("after", af);
    dump("probe_cpu", torch::rand({4}, CPUFloat));
    dump("probe_cuda", torch::rand({4}, CUDAFloat));
    std::printf("{\"step\": %d, \"iter_step\": %d, \"n_rays\": %d, \"loss\": %.6f, \"nodes\": [%lld, %lld], \"backward_nan\": %d, "
                "\"grad_storage\": {\"reused\": %ld, \"fresh\": %ld}}\n", k, int(gdp->iter_step_), n_rays, loss.item<float>(),
                (long long) nodes_before, (long long) (sampler->pers_octree_->tree_nodes_gpu_.numel() / 64), int(nan_skip), reused, fresh);
  }
  std::printf("ref_driver: done, %d steps in %s\n", n_iters, out_root.c_str());
  return 0;
}

// ====================================================================================================== --ops ===
static const int64_t kOpsSeed = 52000;

static int run_ops(const std::string& conf_path, const std::string& in_dir, const std::string& out_root) {
  Scene sc = make_scene(conf_path, true, /*ops_level=*/true);
  GlobalDataPool* gdp = sc.gdp.get();
  auto* field = sc.field; auto* shader = sc.shader;
  gdp->mode_ = RunningMode::TRAIN;
  g_out = out_root;
  fs::create_directories(g_out);
  dump_scene(sc, 0);
  std::vector<std::string> cases;
  for (const auto& e : fs::directory_iterator(in_dir))
    if (fs::is_directory(e.path()) && fs::exists(e.path() / "points.npy")) cases.push_back(e.path().filename().string());
  std::sort(cases.begin(), cases.end());
  const auto opts_of = [](bool is_int) { return is_int ? CPUInt : CPUFloat; };

  for (const auto& c : cases) {
    const auto in = [&](const std::string& name, bool is_int = false) {
      std::string p = in_dir + "/" + c + "/" + name + ".npy";
      if (!fs::exists(p)) p = in_dir + "/" + name + ".npy";
      cnpy::NpyArray a = cnpy::npy_load(p);
      CHECK(a.word_size == 4 && !a.fortran_order) << p;
      std::vector<int64_t> shape(a.shape.begin(), a.shape.end());
      return torch::from_blob(a.data<char>(), shape, opts_of(is_int)).clone().to(torch::kCUDA).contiguous();
    };
    g_out = out_root + "/" + c;
    fs::create_directories(g_out);
    field->feat_pool_.data().copy_(in("feat_pool"));
    field->mlp_->params_.data().copy_(in("field_params"));
    shader->mlp_->params_.data().copy_(in("shader_params"));
    Tensor scales = in("loss_scales").to(torch::kCPU);
    field->mlp_->loss_scale_ = scales[0].item<float>();
    shader->mlp_->loss_scale_ = scales[1].item<float>();
    field->feat_pool_.mutable_grad() = Tensor(); field->mlp_->params_.mutable_grad() = Tensor();
    shader->mlp_->params_.mutable_grad() = Tensor();
    const auto flags = [&]() {
      Tensor f = torch::zeros({3}, CPUFloat);
      f[0] = gdp->backward_nan_ ? 1.f : 0.f; f[1] = field->mlp_->loss_scale_; f[2] = shader->mlp_->loss_scale_;
      return f;
    };

    // field: hash encode + field MLP
    gdp->backward_nan_ = false;
    torch::manual_seed(kOpsSeed);
    Tensor out = field->AnchoredQuery(in("points"), in("anchors", true));
    (out * in("d_out")).sum().backward();
    dump("field_out", out);
    Tensor g = field->feat_pool_.grad().reshape({-1});
    Tensor nz = torch::nonzero(g).reshape({-1});
    dump("field_grad_table_nz_idx", nz.to(torch::kInt32)); dump("field_grad_table_nz_val", g.index({nz}));
    dump("field_grad_params", field->mlp_->params_.grad());
    Tensor ff = flags();
    dump("field_flags", ff);
    dump("field_probe", torch::rand({4}, CUDAFloat));

    // shader: SH encode + shader MLP + colour activation
    gdp->backward_nan_ = false;
    torch::manual_seed(kOpsSeed + 1);
    Tensor feats = in("feats").requires_grad_(true);
    Tensor rgb = shader->Query(feats, in("dirs"));
    (rgb * in("d_rgb")).sum().backward();
    dump("rgb", rgb);
    dump("shader_grad_params", shader->mlp_->params_.grad());
    dump("feats_grad", feats.grad());
    Tensor sf = flags();
    dump("shader_flags", sf);
    dump("shader_probe", torch::rand({4}, CUDAFloat));
    std::printf("{\"ops_case\": \"%s\", \"n\": %d, \"field_flags\": [%g, %g, %g], \"shader_flags\": [%g, %g, %g]}\n", c.c_str(),
                int(out.size(0)), ff[0].item<float>(), ff[1].item<float>(), ff[2].item<float>(), sf[0].item<float>(),
                sf[1].item<float>(), sf[2].item<float>());
  }
  std::printf("ref_driver: done, %d operator cases in %s\n", int(cases.size()), out_root.c_str());
  return 0;
}

// ==================================================================================================== --march ===
static int run_march(const std::string& conf_path, const std::string& root) {
  Scene sc = make_scene(conf_path, true);
  GlobalDataPool* gdp = sc.gdp.get();
  PersSampler* sampler = sc.sampler;
  std::vector<std::string> cases;
  for (const auto& e : fs::directory_iterator(root))
    if (fs::is_directory(e.path()) && fs::exists(e.path() / "params.npy")) cases.push_back(e.path().string());
  std::sort(cases.begin(), cases.end());
  for (const auto& dir : cases) {
    const auto in = [&](const std::string& name, torch::TensorOptions opts) {
      cnpy::NpyArray a = cnpy::npy_load(dir + "/" + name + ".npy");
      CHECK(!a.fortran_order && a.word_size == size_t(opts.dtype().itemsize())) << name;
      std::vector<int64_t> shape(a.shape.begin(), a.shape.end());
      return torch::from_blob(a.data<char>(), shape, opts).clone().to(torch::kCUDA).contiguous();
    };
    sampler->pers_octree_->tree_nodes_gpu_ = in("tree_nodes", CPUUInt8).reshape({-1});
    sampler->pers_octree_->pers_trans_gpu_ = in("pers_trans", CPUUInt8).reshape({-1});
    Tensor rays_o = in("rays_o", CPUFloat), rays_d = in("rays_d", CPUFloat);
    Tensor params = in("params", CPUFloat).to(torch::kCPU);
    const bool train = params[0].item<float>() != 0.f;
    sampler->global_near_ = params[1].item<float>();
    sampler->sample_l_ = params[2].item<float>();
    sampler->scale_by_dis_ = params[3].item<float>() != 0.f;
    sampler->max_oct_intersect_per_ray_ = int(params[4].item<float>());
    const int64_t seed = int64_t(params[5].item<float>());
    gdp->ray_march_fineness_ = 1.f;
    gdp->mode_ = train ? RunningMode::TRAIN : RunningMode::VALIDATE;
    g_out = dir;
    const int n_rays = int(rays_o.size(0));
    torch::NoGradGuard ng;
    dump("rays_d_used", rays_d / torch::linalg_norm(rays_d, 2, -1, true));
    if (train) {   // the draw GetSamples makes first (PersSampler.cu:377, MAX_SAMPLE_PER_RAY 1024), replayed from the same seed
      torch::manual_seed(seed);
      dump("noise", (torch::rand({ 1024 + n_rays + 10 }, CUDAFloat) - .5f) + 1.f);
      torch::manual_seed(seed);
    }
    auto s = sampler->GetSamples(rays_o, rays_d, Tensor());
    dump("pts", s.pts); dump("dirs", s.dirs); dump("dt", s.dt); dump("t", s.t);
    dump("anchors", s.anchors.index({Slc(), Slc(0, 2)}).contiguous());
    dump("bounds", s.pts_idx_bounds); dump("first_oct_dis", s.first_oct_dis);
    std::printf("{\"march_case\": \"%s\", \"rays\": %d, \"samples\": %d}\n", dir.c_str(), n_rays, int(s.pts.size(0)));
  }
  std::printf("ref_driver: done, %d march cases in %s\n", int(cases.size()), root.c_str());
  return 0;
}
