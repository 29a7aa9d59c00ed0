// microbench_gather.cu — rate of random 4-byte gathers from an L2-resident table on this GPU: the roofline that governs the
// hash encode (f2b_field_fwd / f2b_hash_fwd: 128 half2 gathers per sample from the 17 MB live prefix of the fp16 table).
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/gather scripts/microbench_gather.cu && /tmp/gather > gather_rate.json
//
// Patterns: `spread` — every lane its own random entry (the fine levels: every sample in its own cell);
//           `warp_same` — all 32 lanes of a warp read the same 8 random entries (the coarse levels: a warp's samples share a cell);
// 8 independent loads in flight per thread and iteration, like the kernel's 8 corner gathers of one level.
// Output: G lane-gathers/s, and the L2->SM sector traffic that implies (32 B per distinct sector).
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t mix(uint32_t x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }
__device__ __forceinline__ uint32_t ldg_nc_u32(const void* p) { uint32_t v; asm volatile("ld.global.nc.b32 %0, [%1];" : "=r"(v) : "l"(p)); return v; }

template <int SPREAD>
__global__ void gather_kernel(const uint32_t* __restrict__ table, uint32_t n_entries, int iters, uint32_t seed, uint32_t* __restrict__ sink) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, warp = tid >> 5;
  uint32_t s = mix((SPREAD ? tid : warp) * 2654435761u + seed), acc = 0;
  for (int i = 0; i < iters; i++) {
    uint32_t v[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { s = mix(s + k + i * 8); v[k] = ldg_nc_u32(table + (s % n_entries)); }
#pragma unroll
    for (int k = 0; k < 8; k++) acc ^= v[k];
  }
  if (acc == 0x12345678u) sink[0] = acc;
}

template <int SPREAD>
static double run(const uint32_t* table, uint32_t n_entries, int blocks, int threads, int iters, uint32_t* sink) {
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  gather_kernel<SPREAD><<<blocks, threads>>>(table, n_entries, iters, 1u, sink);
  cudaDeviceSynchronize();
  float best = 1e30f;
  for (int rep = 0; rep < 5; rep++) {
    cudaEventRecord(e0);
    gather_kernel<SPREAD><<<blocks, threads>>>(table, n_entries, iters, 7u + rep, sink);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  return double(blocks) * threads * iters * 8 / (best * 1e-3) / 1e9;
}

int main() {
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
  int clk_khz = 0; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
  const int sms = prop.multiProcessorCount, iters = 64;
  printf("{\"gpu\": \"%s\", \"sms\": %d, \"sm_clock_mhz\": %.0f, \"rows\": [\n", prop.name, sms, clk_khz / 1e3);
  bool first = true;
  for (double mb : {17.0, 34.0, 272.0}) {                     // live fp16 table at log2 19 / 20 / 23-equivalent (beyond L2)
    const uint32_t n_entries = uint32_t(mb * 1e6 / 4);
    uint32_t *table, *sink; cudaMalloc(&table, size_t(n_entries) * 4); cudaMemset(table, 1, size_t(n_entries) * 4); cudaMalloc(&sink, 4);
    for (int threads_per_sm : {512, 1024, 2048}) {
      const int threads = 128, blocks = sms * (threads_per_sm / threads);
      const double sp = run<1>(table, n_entries, blocks, threads, iters, sink), ws = run<0>(table, n_entries, blocks, threads, iters, sink);
      printf("%s  {\"table_mb\": %.0f, \"threads_per_sm\": %d, \"spread_g_lane_gathers_per_s\": %.1f, \"spread_lanes_per_clk_per_sm\": %.3f, "
             "\"spread_sector_tb_per_s\": %.2f, \"warp_same_g_lane_gathers_per_s\": %.1f}", first ? "" : ",\n", mb, threads_per_sm, sp,
             sp * 1e9 / (double(sms) * clk_khz * 1e3), sp * 32 / 1e3, ws);
      first = false;
    }
    cudaFree(table); cudaFree(sink);
  }
  printf("\n ]}\n");
  return 0;
}
