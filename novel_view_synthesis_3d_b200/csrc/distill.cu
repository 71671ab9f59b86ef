// distill.cu -- the teacher half of a progressive-distillation training step (Salimans & Ho 2022, Alg. 2):
// xunet_distill_teacher_step and xunet_distill_target.
//
// Sample b of the micro-batch sits at student grid position m_b (drawn by xunet_srn_batch_distill), i.e. at the teacher's
// timestep t = G_T[2 m_b].  The teacher takes two DDIM (eta = 0) steps from there, rows 2 m_b and 2 m_b + 1 of its sampler
// table, each exactly the fixed-clip table step of sampler_step_table_kernel (the common.cuh helpers, sigma = 0):
//   teacher step:  z' = step(row 2 m_b, out_1, z_t)              -> the teacher's z rows, and log-SNR(t') = row[5]
//   target:        z'' = step(row 2 m_b + 1, out_2, z')
//                  x~ = c_a z'' - c_b z_t,   v = (alpha_t z_t - x~) / sigma_t   -> the student's regression target
// with the target-table row m_b = {c_a, c_b, alpha_t, sigma_t}: c_a = 1 / (alpha'' - (sigma'' / sigma_t) alpha_t),
// c_b = (sigma'' / sigma_t) c_a, computed in fp64 on the host and rounded once.  x~ and v use intrinsics, so each product,
// difference and the division is rounded once.  A guided teacher (copies = 2) has the [cond ; uncond] output of a 2B batch
// and its new z goes to both halves; an unguided one (copies = 1) a B batch.  One thread per element, no atomics.
#include "xunet_b200.h"
#include "common.cuh"
#include "kernels.h"

template <bool GUIDED>
__global__ void __launch_bounds__(256) distill_teacher_step_kernel(const float* __restrict__ out_t, float w,
                                                                   const float* __restrict__ ttab, const int* __restrict__ m_dev,
                                                                   long long per, long long n, int B, int copies,
                                                                   float* __restrict__ tz, float* __restrict__ tlogsnr) {
  xu_grid_dep_sync();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i < (long long)B * copies) tlogsnr[i] = ttab[8LL * (2 * m_dev[i % B]) + 5];
  if (i >= n) return;
  const float* t = ttab + 8LL * (2 * m_dev[i / per]);
  const float e = GUIDED ? xu_step_guided(w, out_t[i], out_t[n + i]) : out_t[i];
  const float zi = tz[i];
  const float x0 = xu_step_x0(t, zi, e);
  const float zn = xu_step_z(t, x0, zi, 0.f);
  tz[i] = zn;
  if constexpr (GUIDED) tz[n + i] = zn;
}

template <bool GUIDED>
__global__ void __launch_bounds__(256) distill_target_kernel(const float* __restrict__ out_t, float w,
                                                             const float* __restrict__ ttab, const float* __restrict__ gtab,
                                                             const int* __restrict__ m_dev, const float* __restrict__ z_t,
                                                             const float* __restrict__ tz, long long per, long long n,
                                                             float* __restrict__ v_out) {
  xu_grid_dep_sync();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const int m = m_dev[i / per];
  const float* t = ttab + 8LL * (2 * m + 1);
  const float* g = gtab + 4LL * m;
  const float e = GUIDED ? xu_step_guided(w, out_t[i], out_t[n + i]) : out_t[i];
  const float zp = tz[i];
  const float x0 = xu_step_x0(t, zp, e);
  const float z2 = xu_step_z(t, x0, zp, 0.f);
  const float zt = z_t[i];
  const float xt = __fsub_rn(__fmul_rn(g[0], z2), __fmul_rn(g[1], zt));
  v_out[i] = __fdiv_rn(__fsub_rn(__fmul_rn(g[2], zt), xt), g[3]);
}

void launch_distill_teacher_step(const float* out_t, float w, int copies, const float* ttab, const int* m_dev, int B,
                                 long long per, float* tz, float* tlogsnr, cudaStream_t s) {
  const long long n = (long long)B * per;
  const int grid = cdiv(n > (long long)B * copies ? n : (long long)B * copies, 256);
  xu_launch(copies == 2 ? distill_teacher_step_kernel<true> : distill_teacher_step_kernel<false>, grid, 256, 0, s, out_t, w,
            ttab, m_dev, per, n, B, copies, tz, tlogsnr);
}

void launch_distill_target(const float* out_t, float w, int copies, const float* ttab, const float* gtab, const int* m_dev,
                           const float* z_t, const float* tz, int B, long long per, float* v_out, cudaStream_t s) {
  const long long n = (long long)B * per;
  xu_launch(copies == 2 ? distill_target_kernel<true> : distill_target_kernel<false>, cdiv(n, 256), 256, 0, s, out_t, w, ttab,
            gtab, m_dev, z_t, tz, per, n, v_out);
}
