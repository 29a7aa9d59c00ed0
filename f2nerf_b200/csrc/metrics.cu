// metrics.cu — the image-quality numbers F2-NeRF is judged by, for one test view on the device: the 8-bit PSNR and the SSIM of the
// reference's evaluation script (scripts/eval.py), which reads the 8-bit PNGs ExpRunner::TestImages writes (ExpRunner.cpp:343-391,
// Utils::WriteImageTensor, ImageIO.cpp:28-32) and scores them with skimage's peak_signal_noise_ratio and rgb_ssim (the mip-NeRF SSIM).
//
// One CTA takes a 32 x 16 tile of SSIM outputs: it converts the 42 x 26 x 3 input window of both images to bytes in shared memory,
// then per channel blurs x, y, x^2, y^2, xy with the 11 taps down the columns into shared memory and along the rows into registers,
// in float64 (the fp32 E[x^2] - mu^2 cancels at 1e-4-sized variances).  Nothing but the inputs and the CTAs' partial sums touches
// HBM.  The grid is at most F2B_METRICS_BLOCKS CTAs striding over the tiles; every CTA reduces its sums in a fixed order and a
// one-CTA kernel adds the partials in a fixed order, so a given image pair gives the same bits on every run.
#include "common.cuh"

namespace f2b {

constexpr int MT_X = 32, MT_Y = 16;                          // SSIM outputs per tile
constexpr int MT_R = 5, MT_K = 2 * MT_R + 1;                 // filter radius, taps
constexpr int MT_IX = MT_X + 2 * MT_R, MT_IY = MT_Y + 2 * MT_R;
constexpr int MT_THREADS = 256;
static_assert(F2B_METRICS_WORK_BYTES >= F2B_METRICS_BLOCKS * (sizeof(double) + sizeof(long long)), "metrics scratch layout");

struct SsimTaps { double w[MT_K]; };

// The writer's cast of quantify's output, (x * 255).clip(0, 255).to(uint8): truncation.  fmaxf maps NaN to 0.
__device__ __forceinline__ unsigned pred_u8(float x) { return __float2uint_rz(fmul(fminf(fmaxf(x, 0.f), 1.f), 255.f)); }
// Ground truth loaded as u8 / 255.f: rounding to nearest gives the stored byte back.
__device__ __forceinline__ unsigned gt_u8(float x) { return __float2uint_rn(fmul(fminf(fmaxf(x, 0.f), 1.f), 255.f)); }

// rgb_ssim's map at one pixel from the blurred means and second moments (k1 = 0.01, k2 = 0.03, max_val = 1).
__device__ __forceinline__ double ssim_px(double mu0, double mu1, double e00, double e11, double e01) {
  const double c1 = 0.01 * 0.01, c2 = 0.03 * 0.03;
  const double mu00 = mu0 * mu0, mu11 = mu1 * mu1, mu01 = mu0 * mu1;
  const double s00 = fmax(0., e00 - mu00), s11 = fmax(0., e11 - mu11);
  const double s01r = e01 - mu01;
  const double s01 = copysign(fmin(sqrt(s00 * s11), fabs(s01r)), s01r);
  return ((2. * mu01 + c1) * (2. * s01 + c2)) / ((mu00 + mu11 + c1) * (s00 + s11 + c2));
}

// Sum over the CTA in a fixed order; the result is valid in thread 0.
template <class T>
__device__ __forceinline__ T block_sum(T v, T* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  T s = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < MT_THREADS / 32; w++) s += red[w];
  return s;
}

__global__ void __launch_bounds__(MT_THREADS)
image_metrics_kernel(const float* __restrict__ pred, const float* __restrict__ gt, int height, int width, int tiles_x, int tiles_y,
                     SsimTaps taps, double* __restrict__ part_ssim, long long* __restrict__ part_sse) {
  __shared__ uint8_t sp[MT_IY][MT_IX * 3], sg[MT_IY][MT_IX * 3];
  __shared__ double lut[256];                                // byte / 255., as the script divides the PNG's bytes
  __shared__ double vb[5][MT_Y][MT_IX];                      // column blur of x, y, x^2, y^2, xy for one channel
  __shared__ double red_d[MT_THREADS / 32];
  __shared__ long long red_i[MT_THREADS / 32];
  for (int i = threadIdx.x; i < 256; i += MT_THREADS) lut[i] = double(i) / 255.;
  const int n_tiles = tiles_x * tiles_y, out_h = height - 2 * MT_R, out_w = width - 2 * MT_R;
  double ssim_acc = 0.;
  long long sse_acc = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
    const int y0 = ty * MT_Y, x0 = tx * MT_X;
    // every pixel's squared difference is counted by exactly one tile: the one whose outputs start at its row / column, and the
    // last tile row / column also takes the image's last 2R rows / columns, which start no output
    const int own_rows = ty == tiles_y - 1 ? MT_IY : MT_Y, own_vals = (tx == tiles_x - 1 ? MT_IX : MT_X) * 3;
    __syncthreads();                                         // the previous tile's readers of sp / sg / vb are done
    for (int i = threadIdx.x; i < MT_IY * MT_IX * 3; i += MT_THREADS) {
      const int r = i / (MT_IX * 3), c = i - r * (MT_IX * 3);
      unsigned p = 0, g = 0;
      if (y0 + r < height && x0 * 3 + c < width * 3) {
        const size_t a = (size_t(y0 + r) * width + x0) * 3 + c;
        p = pred_u8(__ldg(pred + a));
        g = gt_u8(__ldg(gt + a));
        if (r < own_rows && c < own_vals) sse_acc += (long long)((int(p) - int(g)) * (int(p) - int(g)));
      }
      sp[r][c] = uint8_t(p);
      sg[r][c] = uint8_t(g);
    }
    __syncthreads();
    for (int ch = 0; ch < 3; ch++) {
      for (int i = threadIdx.x; i < MT_Y * MT_IX; i += MT_THREADS) {
        const int r = i / MT_IX, c = i - r * MT_IX;
        double m0 = 0., m1 = 0., e00 = 0., e11 = 0., e01 = 0.;
#pragma unroll
        for (int k = 0; k < MT_K; k++) {
          const double w = taps.w[MT_K - 1 - k];             // a convolution: the taps run backwards (they are symmetric)
          const double x = lut[sp[r + k][c * 3 + ch]], y = lut[sg[r + k][c * 3 + ch]];
          m0 += w * x; m1 += w * y; e00 += w * (x * x); e11 += w * (y * y); e01 += w * (x * y);
        }
        vb[0][r][c] = m0; vb[1][r][c] = m1; vb[2][r][c] = e00; vb[3][r][c] = e11; vb[4][r][c] = e01;
      }
      __syncthreads();
      for (int i = threadIdx.x; i < MT_Y * MT_X; i += MT_THREADS) {
        const int r = i / MT_X, c = i - r * MT_X;
        if (y0 + r >= out_h || x0 + c >= out_w) continue;
        double q[5] = {0., 0., 0., 0., 0.};
#pragma unroll
        for (int k = 0; k < MT_K; k++) {
          const double w = taps.w[MT_K - 1 - k];
#pragma unroll
          for (int j = 0; j < 5; j++) q[j] += w * vb[j][r][c + k];
        }
        ssim_acc += ssim_px(q[0], q[1], q[2], q[3], q[4]);
      }
      __syncthreads();                                       // before the next channel overwrites vb
    }
  }
  const double s = block_sum(ssim_acc, red_d);
  const long long e = block_sum(sse_acc, red_i);
  if (threadIdx.x == 0) {
    part_ssim[blockIdx.x] = s;
    part_sse[blockIdx.x] = e;
  }
}

__global__ void __launch_bounds__(MT_THREADS)
image_metrics_finish_kernel(const double* __restrict__ part_ssim, const long long* __restrict__ part_sse, int n,
                            int64_t* __restrict__ sse, double* __restrict__ ssim_sum) {
  __shared__ double red_d[MT_THREADS / 32];
  __shared__ long long red_i[MT_THREADS / 32];
  double s = 0.;
  long long e = 0;
  for (int i = threadIdx.x; i < n; i += MT_THREADS) {
    s += part_ssim[i];
    e += part_sse[i];
  }
  s = block_sum(s, red_d);
  e = block_sum(e, red_i);
  if (threadIdx.x == 0) {
    *sse = e;
    *ssim_sum = s;
  }
}

}  // namespace f2b

using namespace f2b;

extern "C" int f2b_image_metrics(const float* pred, const float* gt, int height, int width, const double* taps_host, void* work,
                                 int64_t* sse, double* ssim_sum, void* stream) {
  F2B_REQUIRE(pred && gt && taps_host && work && sse && ssim_sum, "f2b_image_metrics: null pointer");
  F2B_REQUIRE(height >= MT_K && width >= MT_K, "f2b_image_metrics: %d x %d image is smaller than the %d x %d SSIM window", height,
              width, MT_K, MT_K);
  F2B_REQUIRE(int64_t(height) * width < (int64_t(1) << 31), "f2b_image_metrics: %d x %d pixels overflow int32", height, width);
  F2B_REQUIRE(reinterpret_cast<uintptr_t>(work) % 8 == 0, "f2b_image_metrics: work must be 8-byte aligned");
  SsimTaps taps;
  for (int k = 0; k < MT_K; k++) taps.w[k] = taps_host[k];
  const int tiles_x = div_up(width - 2 * MT_R, MT_X), tiles_y = div_up(height - 2 * MT_R, MT_Y);
  const int grid = int(tiles_x * int64_t(tiles_y) < F2B_METRICS_BLOCKS ? tiles_x * tiles_y : F2B_METRICS_BLOCKS);
  double* part_ssim = static_cast<double*>(work);
  long long* part_sse = reinterpret_cast<long long*>(part_ssim + F2B_METRICS_BLOCKS);
  image_metrics_kernel<<<grid, MT_THREADS, 0, as_stream(stream)>>>(pred, gt, height, width, tiles_x, tiles_y, taps, part_ssim,
                                                                  part_sse);
  image_metrics_finish_kernel<<<1, MT_THREADS, 0, as_stream(stream)>>>(part_ssim, part_sse, grid, sse, ssim_sum);
  return check_launch("f2b_image_metrics");
}
