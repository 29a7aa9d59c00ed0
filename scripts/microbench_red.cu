// microbench_red.cu — issue rate of global-memory reductions on this GPU, the roofline that governs f2b_hash_bwd.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/red scripts/microbench_red.cu && /tmp/red > red_rate.json
//
// Every lane issues `red.global.add` to pseudo-random addresses inside a buffer of the hash table's live size (34 MB of
// fp32 pairs: L2-resident, like the real gradient table), for three flavours:
//   v2f32   red.global.add.v2.f32   (8 B: what hash_bwd issues, one per (sample, level, corner))
//   f32     red.global.add.f32      (4 B)
//   f16x2   red.global.add.noftz.f16x2 (4 B: both channels of one table entry in fp16 — the reference's own format)
// and two address patterns: `spread` (every lane a different random entry — the fine levels) and `same_line` (the 32 lanes
// of a warp hit 32 consecutive entries of one random 256 B block — best case coalescing).
// Output: one JSON object; rates in G lane-reductions/s and the equivalent cycles per lane-reduction per SM.
#include <cstdio>
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t mix(uint32_t x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }

template <int KIND, int SPREAD>
__global__ void red_kernel(float* __restrict__ buf, uint32_t n_entries, int iters, uint32_t seed) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31, warp = tid >> 5;
  uint32_t s = mix(tid * 2654435761u + seed);
  for (int i = 0; i < iters; i++) {
    s = mix(s + i);
    uint32_t e;
    if (SPREAD) e = s % n_entries;
    else e = ((mix(warp * 977u + i * 131071u + seed) % (n_entries / 32)) * 32 + lane);
    float* p = buf + 2 * size_t(e);
    const float a = 1e-6f * (s & 255), b = 1e-6f * ((s >> 8) & 255);
    if (KIND == 0) asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
    else if (KIND == 1) asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(a) : "memory");
    else {
      const __half2 h = __floats2half2_rn(a, b);
      asm volatile("red.global.add.noftz.f16x2 [%0], %1;" ::"l"(p), "r"(*reinterpret_cast<const uint32_t*>(&h)) : "memory");
    }
  }
}

template <int KIND, int SPREAD>
static double run(float* buf, uint32_t n_entries, int blocks, int threads, int iters) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  red_kernel<KIND, SPREAD><<<blocks, threads>>>(buf, n_entries, iters, 1u);          // warm-up
  cudaDeviceSynchronize();
  float best = 1e30f;
  for (int rep = 0; rep < 5; rep++) {
    cudaEventRecord(e0);
    red_kernel<KIND, SPREAD><<<blocks, threads>>>(buf, n_entries, iters, 7u + rep);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  return double(blocks) * threads * iters / (best * 1e-3) / 1e9;                     // G lane-reductions / s
}

int main() {
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
  int clk_khz = 0; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
  const uint32_t n_entries = 17u * (1u << 19) / 2;          // the live prefix of a log2-19 table, in (ch0,ch1) entries
  float* buf; cudaMalloc(&buf, size_t(n_entries) * 8); cudaMemset(buf, 0, size_t(n_entries) * 8);
  const int sms = prop.multiProcessorCount, iters = 256;
  printf("{\"gpu\": \"%s\", \"sms\": %d, \"sm_clock_mhz\": %.0f, \"buffer_mb\": %.1f, \"iters_per_lane\": %d,\n \"rows\": [\n", prop.name, sms,
         clk_khz / 1e3, n_entries * 8 / 1e6, iters);
  const char* names[3] = {"v2f32", "f32", "f16x2"};
  bool first = true;
  for (int threads_per_sm : {256, 512, 1024, 2048}) {
    const int threads = 256, blocks = sms * (threads_per_sm / threads);
    double r[3][2];
    r[0][1] = run<0, 1>(buf, n_entries, blocks, threads, iters); r[0][0] = run<0, 0>(buf, n_entries, blocks, threads, iters);
    r[1][1] = run<1, 1>(buf, n_entries, blocks, threads, iters); r[1][0] = run<1, 0>(buf, n_entries, blocks, threads, iters);
    r[2][1] = run<2, 1>(buf, n_entries, blocks, threads, iters); r[2][0] = run<2, 0>(buf, n_entries, blocks, threads, iters);
    for (int k = 0; k < 3; k++)
      for (int sp = 1; sp >= 0; sp--) {
        const double cyc = double(sms) * (clk_khz * 1e3) / (r[k][sp] * 1e9);
        printf("%s  {\"kind\": \"%s\", \"pattern\": \"%s\", \"threads_per_sm\": %d, \"g_lane_red_per_s\": %.1f, \"cycles_per_lane_red_per_sm\": %.3f}",
               first ? "" : ",\n", names[k], sp ? "spread" : "same_line", threads_per_sm, r[k][sp], cyc);
        first = false;
      }
  }
  printf("\n ]}\n");
  cudaFree(buf);
  return 0;
}
