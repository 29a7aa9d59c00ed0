// ref_camrays.cpp — harness around the UNMODIFIED reference's Dataset (Totoro97/f2-nerf @98f0daa), linked from the reference's
// own objects by oracle/Makefile.camrays into oracle/_ref/ref_camrays.
//
// TEST INFRASTRUCTURE ONLY.  It constructs the reference's GlobalDataPool and Dataset as ExpRunner::ExpRunner does
// (src/ExpRunner.cpp:17-40) and dumps, as .npy, the whole-camera rays of the evaluation modes (ExpRunner::TestImages /
// RenderPath, src/ExpRunner.cpp:322-391): Dataset::RaysOfCamera(test_set_[0]) and Dataset::RaysFromPose(render_poses_[0], 2) /
// (render_poses_[5], 3) (src/Dataset/Dataset.cpp:177-218), with the camera tables, render poses and test split they come from.
// The dumps pin f2b_camera_rays and oracle/camera_rays.c (tests/golden/ref_ngp_fox_camrays.npz, tests/test_gpu_eval.py).
//
//   ref_camrays <runtime_config.yaml> <out_dir>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include <iostream>
#include <experimental/filesystem>
#include <torch/torch.h>
#include "Common.h"
#include "Utils/GlobalDataPool.h"
#include "Utils/cnpy.h"
#include "Dataset/Dataset.h"

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
    default: std::cerr << "dump: unsupported dtype for " << name << std::endl; std::exit(2);
  }
}

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: ref_camrays <config.yaml> <out_dir>\n"); return 1; }
  g_out = argv[2];
  fs::create_directories(g_out);
  torch::manual_seed(2022);   // main.cpp:8
  auto gdp = std::make_unique<GlobalDataPool>(argv[1]);
  gdp->base_exp_dir_ = gdp->config_["base_exp_dir"].as<std::string>();
  fs::create_directories(gdp->base_exp_dir_);
  auto dataset = std::make_unique<Dataset>(gdp.get());
  CHECK(dataset->render_poses_.defined() && dataset->render_poses_.size(0) > 5 && !dataset->test_set_.empty());

  dump("ds_poses", dataset->poses_.reshape({-1, 12})); dump("ds_intri", dataset->intri_.reshape({-1, 9}));
  dump("ds_dist_params", dataset->dist_params_); dump("ds_bounds", dataset->bounds_);
  Tensor hw = torch::zeros({2}, CPUFloat); hw[0] = float(dataset->height_); hw[1] = float(dataset->width_);
  dump("ds_hw", hw);
  dump("cam_render_poses", dataset->render_poses_.reshape({-1, 12}).contiguous());
  dump("cam_test_set", torch::from_blob(dataset->test_set_.data(), {int(dataset->test_set_.size())}, CPUInt).clone());
  auto put = [](const std::string& tag, const BoundedRays& r) {
    dump("cam_" + tag + "_rays_o", r.origins); dump("cam_" + tag + "_rays_d", r.dirs); dump("cam_" + tag + "_bounds", r.bounds);
  };
  put("test0", dataset->RaysOfCamera(dataset->test_set_[0]));
  put("path0_reso2", dataset->RaysFromPose(dataset->render_poses_[0], 2));
  put("path5_reso3", dataset->RaysFromPose(dataset->render_poses_[5], 3));
  std::printf("ref_camrays: done, dumps in %s\n", g_out.c_str());
  return 0;
}
