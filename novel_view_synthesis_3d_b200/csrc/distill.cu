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

extern "C" int xunet_distill_teacher_step(const float* out_t, float w, int teacher_copies, const float* teacher_table,
                                          const int* m_dev, int B, long long per, const xunet_batch* teacher, void* stream) {
  if (!out_t || !teacher_table || !m_dev || !teacher || !teacher->z || !teacher->logsnr)
    return xu_fail("xunet_distill_teacher_step: NULL pointer argument");
  if (B < 1 || per < 1) return xu_fail("xunet_distill_teacher_step: B = %d, per = %lld, need both >= 1", B, per);
  if (teacher_copies != 1 && teacher_copies != 2)
    return xu_fail("xunet_distill_teacher_step: teacher_copies = %d, need 1 or 2", teacher_copies);
  const long long n = (long long)B * per;
  const int grid = cdiv(n > (long long)B * teacher_copies ? n : (long long)B * teacher_copies, 256);
  xu_launch(teacher_copies == 2 ? distill_teacher_step_kernel<true> : distill_teacher_step_kernel<false>, grid, 256, 0,
            (cudaStream_t)stream, out_t, w, teacher_table, m_dev, per, n, B, teacher_copies, const_cast<float*>(teacher->z),
            const_cast<float*>(teacher->logsnr));
  return xu_launched("distill_teacher_step");
}

extern "C" int xunet_distill_target(const float* out_t, float w, int teacher_copies, const float* teacher_table,
                                    const float* target_table, const int* m_dev, const float* z_t, const float* teacher_z, int B,
                                    long long per, float* v_out, void* stream) {
  if (!out_t || !teacher_table || !target_table || !m_dev || !z_t || !teacher_z || !v_out)
    return xu_fail("xunet_distill_target: NULL pointer argument");
  if (B < 1 || per < 1) return xu_fail("xunet_distill_target: B = %d, per = %lld, need both >= 1", B, per);
  if (teacher_copies != 1 && teacher_copies != 2)
    return xu_fail("xunet_distill_target: teacher_copies = %d, need 1 or 2", teacher_copies);
  const long long n = (long long)B * per;
  xu_launch(teacher_copies == 2 ? distill_target_kernel<true> : distill_target_kernel<false>, cdiv(n, 256), 256, 0,
            (cudaStream_t)stream, out_t, w, teacher_table, target_table, m_dev, z_t, teacher_z, per, n, v_out);
  return xu_launched("distill_target");
}
