// ref_resume.cpp — the reference program's RESUME path (is_continue: true), with the same seeded TRAIN step and dumps as
// oracle/ref_driver.cpp.  TEST INFRASTRUCTURE ONLY, linked by oracle/Makefile.resume against the UNMODIFIED reference objects
// into oracle/_ref/ref_resume, and with this library's fused C++ host as the body of Renderer::Render into
// oracle/_ref/ref_resume_b200.
//
//   ref_resume <runtime_config.yaml with is_continue: true> <out_dir> <n_rays>
//
// ExpRunner's own constructor builds the scene exactly as a resumed run does (ExpRunner.cpp:17-62): Dataset, Renderer (whose
// PersSampler builds the initial octree, warps and edge pool from the training cameras), the optimizer, and LoadCheckpoint on
// <base_exp_dir>/checkpoints/latest (the checkpoint's octree and warps replace the initial ones, UpdateAdaParams sets the
// saved iteration's fineness and gradient-scaling progress; the edge pool stays the initial one).  Then:
//   * the renderer state a resumed run trains with: edge pool, octree and warp bytes, iteration, fineness, progress;
//   * the edge-sample operator under a fixed seed, with its RNG draws replayed next to it;
//   * one seeded TRAIN Render + the loss of oracle/ref_driver.cpp + backward, on RandRaysData rays: outputs and gradients.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include <iostream>
#include <experimental/filesystem>
#include <torch/torch.h>
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
    case torch::kUInt8: cnpy::npy_save(path, t.data_ptr<uint8_t>(), shape); break;
    default: std::cerr << "dump: unsupported dtype for " << name << std::endl; std::exit(2);
  }
}

int main(int argc, char** argv) {
  if (argc < 4) { std::fprintf(stderr, "usage: ref_resume <config.yaml> <out_dir> <n_rays>\n"); return 1; }
  g_out = argv[2];
  const int n_rays = std::atoi(argv[3]);
  fs::create_directories(g_out);

  torch::manual_seed(2022);   // main.cpp:8
  auto runner = std::make_unique<ExpRunner>(argv[1]);
  CHECK(runner->global_data_pool_->config_["is_continue"].as<bool>());
  GlobalDataPool* gdp = runner->global_data_pool_.get();
  Dataset* dataset = runner->dataset_.get();
  Renderer* renderer = runner->renderer_.get();
  auto* sampler = dynamic_cast<PersSampler*>(renderer->pts_sampler_.get());
  auto* field = dynamic_cast<Hash3DAnchored*>(renderer->scene_field_.get());
  auto* shader = dynamic_cast<SHShader*>(renderer->shader_.get());
  CHECK(sampler && field && shader);
#ifdef F2B_WITH_SHIM
  std::printf("ref_resume_b200: Renderer::Render replaced by the fused B200 host\n");
#endif

  // ---- the resumed renderer state ------------------------------------------------------------------------------------
  dump("edge_pool", sampler->pers_octree_->edge_pool_gpu_);
  dump("tree_nodes", sampler->pers_octree_->tree_nodes_gpu_);
  dump("pers_trans", sampler->pers_octree_->pers_trans_gpu_);
  {
    Tensor sc = torch::zeros({3}, CPUFloat);
    sc[0] = float(runner->iter_step_); sc[1] = gdp->ray_march_fineness_; sc[2] = gdp->gradient_scaling_progress_;
    dump("resume_scalars", sc);
  }

  // ---- rays, as oracle/ref_driver.cpp draws them -------------------------------------------------------------------------
  torch::manual_seed(2023);
  auto [rays, gt_colors, emb_idx] = dataset->RandRaysData(n_rays, DATA_TRAIN_SET);
  Tensor rays_o = rays.origins.contiguous(), rays_d = rays.dirs.contiguous(), bounds = rays.bounds.contiguous();
  dump("rays_o", rays_o); dump("rays_d", rays_d); dump("gt_colors", gt_colors); dump("emb_idx", emb_idx);

  // ---- edge samples over the resumed pool and warps, with the RNG draws replayed ---------------------------------------
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

  // ---- one TRAIN step at the saved iteration (ExpRunner::Train sets iter_step_ before its loop, ExpRunner.cpp:80) --------
  gdp->iter_step_ = runner->iter_step_;
  gdp->mode_ = RunningMode::TRAIN;
  gdp->backward_nan_ = false;
  torch::manual_seed(777);
  auto r = renderer->Render(rays_o, rays_d, bounds, emb_idx);
  dump("train_colors", r.colors); dump("train_disparity", r.disparity); dump("train_depth", r.depth);
  dump("train_weights", r.weights); dump("train_idx_start_end", r.idx_start_end);
  dump("train_first_oct_dis", r.first_oct_dis); dump("train_edge_feats", r.edge_feats);
  Tensor color_loss = torch::sqrt((r.colors - gt_colors).square() + 1e-4f).mean();
  Tensor disparity_loss = r.disparity.square().mean();
  Tensor tv_loss = (r.edge_feats.index({Slc(), 0}) - r.edge_feats.index({Slc(), 1})).square().mean();
  Tensor var_loss = (CustomOps::WeightVar(r.weights, r.idx_start_end) + 1e-2).sqrt().mean();
  Tensor loss = color_loss + var_loss * 1e-2f + disparity_loss * 1e-2f + tv_loss * 1e-1f;
  dump("train_loss", loss.reshape({1}));
  loss.backward();
  dump("grad_field_mlp", field->mlp_->params_.grad());
  dump("grad_shader_mlp", shader->mlp_->params_.grad());
  dump("grad_app_emb", renderer->app_emb_.grad());
  dump("grad_feat_pool", field->feat_pool_.grad().reshape({-1}));
  dump("backward_nan", torch::full({1}, gdp->backward_nan_ ? 1.f : 0.f, CPUFloat));
  std::printf("ref_resume: iteration %u, %d edges, dumps in %s\n", runner->iter_step_,
              int(sampler->pers_octree_->edge_pool_.size()), g_out.c_str());
  return 0;
}
