// metrics.cu -- per-image MSE / PSNR / SSIM of generated views against ground truth (xunet_image_metrics).
//
// One CTA scores one image, so the grid is (B) and nothing crosses CTAs: no scratch, no atomics, and an image's numbers do not
// depend on B or on its position in the batch.  Every value is mapped to u = clamp((v + 1) / 2, 0, 1) in fp64 (exact for fp32
// inputs), and everything after the loads is fp64:
//   * MSE: each thread sums (u_p - u_t)^2 over a fixed stride of the S*S*3 values, then a fixed warp-shuffle / shared-memory
//     tree adds the thread sums.
//   * SSIM: a separable 11-tap Gaussian filter of the five moments (u_p, u_t, u_p^2, u_t^2, u_p u_t), per channel.  A ring of
//     METRICS_BAND + 10 horizontally filtered rows lives in shared memory; each pass filters the next METRICS_BAND input rows
//     into it, then filters the ring vertically into METRICS_BAND output rows and adds their SSIM terms to per-thread sums.
//     fp64 moments keep sigma^2 = E[u^2] - mu^2 accurate to ~1e-16 where it cancels (near-white backgrounds), far below C2.
#include "xunet_b200.h"
#include "common.cuh"
#include "kernels.h"

#define METRICS_THREADS 512
#define METRICS_BAND 8                        // output rows per pass
#define METRICS_RING (METRICS_BAND + 10)      // horizontally filtered rows kept in shared memory

struct MetricsWindow { double w[11]; };   // the normalised 1-D Gaussian weights of the SSIM window

static size_t metrics_smem_bytes(int S) { return sizeof(double) * 5 * METRICS_RING * (size_t)(S - 10); }

__device__ __forceinline__ double metrics_u(float v) { return fmin(fmax(((double)v + 1.0) * 0.5, 0.0), 1.0); }

// 512 threads; red: 16 doubles of shared memory.  Fixed order: butterfly within each warp, then warps 0..15 in order.
__device__ __forceinline__ double metrics_block_sum(double x, double* red) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = x;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < METRICS_THREADS / 32; ++w) t += red[w];
  __syncthreads();
  return t;   // valid in thread 0
}

__global__ void __launch_bounds__(METRICS_THREADS) image_metrics_kernel(const float* __restrict__ pred,
                                                                        const float* __restrict__ target, int S,
                                                                        MetricsWindow win, float* __restrict__ mse_out,
                                                                        float* __restrict__ psnr_out,
                                                                        float* __restrict__ ssim_out) {
  xu_grid_dep_sync();
  extern __shared__ double ring[];   // [5][METRICS_RING][So]: mu_p, mu_t, E[p^2], E[t^2], E[pt]
  __shared__ double red[METRICS_THREADS / 32];
  const int So = S - 10;
  const long long per = (long long)S * S * 3;
  const float* P = pred + (long long)blockIdx.x * per;
  const float* T = target + (long long)blockIdx.x * per;
  const int plane = METRICS_RING * So;

  double se = 0.0;
  for (long long i = threadIdx.x; i < per; i += METRICS_THREADS) {
    const double d = metrics_u(__ldg(P + i)) - metrics_u(__ldg(T + i));
    se = fma(d, d, se);
  }

  double ss = 0.0;
  for (int c = 0; c < 3; ++c) {
    for (int yo0 = 0; yo0 < So; yo0 += METRICS_BAND) {
      // input rows [y0, y1) enter the ring at slot y % METRICS_RING; they replace rows the previous pass no longer needs
      const int y0 = yo0 == 0 ? 0 : yo0 + 10, y1 = min(yo0 + METRICS_RING, S);
      for (int it = threadIdx.x; it < (y1 - y0) * So; it += METRICS_THREADS) {
        const int y = y0 + it / So, x = it % So;
        const long long base = ((long long)y * S + x) * 3 + c;
        double mp = 0.0, mt = 0.0, pp = 0.0, tt = 0.0, pt = 0.0;
#pragma unroll
        for (int j = 0; j < 11; ++j) {
          const double p = metrics_u(__ldg(P + base + 3 * j)), t = metrics_u(__ldg(T + base + 3 * j)), w = win.w[j];
          mp = fma(w, p, mp);
          mt = fma(w, t, mt);
          pp = fma(w, p * p, pp);
          tt = fma(w, t * t, tt);
          pt = fma(w, p * t, pt);
        }
        double* r = ring + (y % METRICS_RING) * So + x;
        r[0] = mp; r[plane] = mt; r[2 * plane] = pp; r[3 * plane] = tt; r[4 * plane] = pt;
      }
      __syncthreads();
      const int nout = min(METRICS_BAND, So - yo0);
      for (int it = threadIdx.x; it < nout * So; it += METRICS_THREADS) {
        const int yo = yo0 + it / So, x = it % So;
        double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
        for (int i = 0; i < 11; ++i) {
          const double* r = ring + ((yo + i) % METRICS_RING) * So + x;
#pragma unroll
          for (int k = 0; k < 5; ++k) m[k] = fma(win.w[i], r[k * plane], m[k]);
        }
        const double vp = m[2] - m[0] * m[0], vt = m[3] - m[1] * m[1], cpt = m[4] - m[0] * m[1];
        const double C1 = 1e-4, C2 = 9e-4;   // (0.01 L)^2, (0.03 L)^2 with data range L = 1
        ss += (2.0 * m[0] * m[1] + C1) * (2.0 * cpt + C2) / ((m[0] * m[0] + m[1] * m[1] + C1) * (vp + vt + C2));
      }
      __syncthreads();
    }
  }

  const double se_sum = metrics_block_sum(se, red);
  const double ss_sum = metrics_block_sum(ss, red);
  if (threadIdx.x == 0) {
    const double mse = se_sum / (double)per;
    mse_out[blockIdx.x] = (float)mse;
    psnr_out[blockIdx.x] = (float)(-10.0 * log10(mse));   // +inf when mse == 0
    ssim_out[blockIdx.x] = (float)(ss_sum / (3.0 * So * So));
  }
}

// exp(-i^2 / (2 * 1.5^2)), i = -5..5, normalised to sum 1
static MetricsWindow metrics_window() {
  MetricsWindow win;
  double sum = 0.0;
  for (int i = 0; i < 11; ++i) sum += win.w[i] = exp(-(double)((i - 5) * (i - 5)) / (2.0 * 1.5 * 1.5));
  for (int i = 0; i < 11; ++i) win.w[i] /= sum;
  return win;
}

extern "C" int xunet_image_metrics(const float* pred, const float* target, int B, int S, float* mse_out, float* psnr_out,
                                   float* ssim_out, void* stream) {
  if (!pred || !target || !mse_out || !psnr_out || !ssim_out) return xu_fail("xunet_image_metrics: NULL pointer argument");
  if (B < 1) return xu_fail("xunet_image_metrics: B = %d, need B >= 1", B);
  if (S < 11 || S > XUNET_METRICS_MAX_SIDE)
    return xu_fail("xunet_image_metrics: S = %d outside [11, %d]", S, XUNET_METRICS_MAX_SIDE);
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(image_metrics_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)metrics_smem_bytes(XUNET_METRICS_MAX_SIDE));
    configured = true;
  }
  static const MetricsWindow win = metrics_window();
  xu_launch(image_metrics_kernel, B, METRICS_THREADS, metrics_smem_bytes(S), (cudaStream_t)stream, pred, target, S, win, mse_out,
            psnr_out, ssim_out);
  return xu_launched("image_metrics");
}
