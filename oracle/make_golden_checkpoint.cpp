// Writes the checkpoint-reader fixtures tests/golden/libtorch_states.pt and libtorch_scalars.pt with LibTorch's own
// torch::save, the call the reference's ExpRunner::SaveCheckpoint makes (ExpRunner.cpp:203-219):
//   libtorch_states.pt   torch::save(std::vector<Tensor>): a miniature Renderer::States() of 11 entries (so that the keys
//                        "10" and "2" are both present and string order differs from index order)
//   libtorch_scalars.pt  torch::save(Tensor): the one-element float iter_step tensor
// Every value is an exact function of its index, restated in tests/test_checkpoint_cpu.py.
// Built and run by oracle/make_golden_checkpoint.sh.
#include <torch/torch.h>

#include <cstdint>
#include <string>
#include <vector>

using torch::Tensor;

static Tensor u8_blob(int64_t n, int mul, int add) {
  std::vector<uint8_t> v(n);
  for (int64_t i = 0; i < n; i++) v[i] = uint8_t((i * mul + add) % 256);
  return torch::from_blob(v.data(), {n}, torch::kUInt8).clone();
}

static Tensor i32(std::vector<int32_t> v, std::vector<int64_t> shape) {
  return torch::from_blob(v.data(), shape, torch::kInt32).clone();
}

// ((i * mul) % 2001 - 1000) / 1024: exact in float
static Tensor f32(std::vector<int64_t> shape, int64_t mul) {
  int64_t n = 1;
  for (auto s : shape) n *= s;
  std::vector<float> v(n);
  for (int64_t i = 0; i < n; i++) v[i] = float((i * mul) % 2001 - 1000) / 1024.f;
  return torch::from_blob(v.data(), shape, torch::kFloat32).clone();
}

int main(int argc, char** argv) {
  const std::string out = argc > 1 ? argv[1] : "tests/golden";
  const int64_t V = 2, log2_table = 4, n_images = 5;
  std::vector<int32_t> prims(16 * V * 3);
  for (size_t i = 0; i < prims.size(); i++) prims[i] = int32_t((1 << 28) + 7 * int32_t(i));
  std::vector<Tensor> states = {
      u8_blob(2 * 64, 37, 11),                           // PersSampler: tree_nodes_gpu_ (2 TreeNode)
      u8_blob(V * 544, 13, 5),                           //              pers_trans_gpu_ (V TransInfo)
      i32({3, -7}, {2}),                                 //              tree_visit_cnt_
      i32({2000, 4000, 6000, 8000, 10000}, {5}),         //              sub_div_milestones_
      f32({(1 << log2_table) * 16, 2}, 7919),            // Hash3DAnchored: feat_pool_
      i32(prims, {16, V, 3}),                            //                 prim_pool_
      f32({16 * V, 3}, 104729),                          //                 bias_pool_
      i32({int32_t(V)}, {1}),                            //                 n_volumes_ (a CPU tensor in the reference too)
      f32({32 * 64 + 64 * 16}, 31),                      //                 mlp_->params_
      f32({32 * 64 + 64 * 64 + 64 * 16}, 17),            // SHShader: mlp_->params_
      f32({n_images, 16}, 523),                          // Renderer: app_emb_
  };
  torch::save(states, out + "/libtorch_states.pt");
  Tensor scalars = torch::empty({1}, torch::kFloat32);
  scalars.index_put_({0}, float(1234));
  torch::save(scalars, out + "/libtorch_scalars.pt");
  return 0;
}
