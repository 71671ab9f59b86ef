// cd.cu -- the teacher half of a consistency-distillation training step (Song et al. 2023, Consistency Models, Alg. 2,
// with a guided teacher as in LCM): xunet_cd_teacher_step and xunet_cd_target.
//
// Sample b of the micro-batch sits at grid position n = m_b (drawn by xunet_srn_batch_distill on the teacher grid G of N
// timesteps), i.e. at t_n = G[n].  The teacher takes one DDIM (eta = 0) step from there, row n of its sampler table, exactly
// the fixed-clip table step of sampler_step_table_kernel (the common.cuh helpers, sigma = 0); the target network (the
// student's own weights, run by the caller between the two entries) maps the result to x0; the regression target is the v
// whose x0 is that one:
//   teacher step:  z^ = step(row n, out_t, z_t)           -> z_out, and log-SNR(t_{n+1}) = row[5] -> logsnr_out
//   target:        x0- = clip(a z^ - b v-, -1, 1),   v* = (alpha_n z_t - x0-) / sigma_n   -> the student's regression target
// with the target-table row n = {a, b, alpha_n, sigma_n}: a = alpha_{n+1}, b = sigma_{n+1}, and (a, b) = (1, 0) on the last
// row (t_{n+1} = clean), where x0- = z^, the teacher's clipped x0 (the boundary condition f(., clean) = identity).  The
// table is computed in fp64 on the host and rounded once.  x0- is the sampler's x0 expression (xu_step_x0 on a row whose
// first two columns are {a, b}); v* uses intrinsics, so the product, the difference and the division are each rounded once.
// A guided teacher (copies = 2) has the [cond ; uncond] output of a 2B batch, an unguided one (copies = 1) a B batch.  One
// thread per element, no atomics.
#include "xunet_b200.h"
#include "common.cuh"
#include "kernels.h"

template <bool GUIDED>
__global__ void __launch_bounds__(256) cd_teacher_step_kernel(const float* __restrict__ out_t, float w,
                                                              const float* __restrict__ ttab, const int* __restrict__ m_dev,
                                                              long long per, long long n, int B, const float* __restrict__ z_t,
                                                              float* __restrict__ z_out, float* __restrict__ logsnr_out) {
  xu_grid_dep_sync();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i < B) logsnr_out[i] = ttab[8LL * m_dev[i] + 5];
  if (i >= n) return;
  const float* t = ttab + 8LL * m_dev[i / per];
  const float e = GUIDED ? xu_step_guided(w, out_t[i], out_t[n + i]) : out_t[i];
  const float zi = z_t[i];
  const float x0 = xu_step_x0(t, zi, e);
  z_out[i] = xu_step_z(t, x0, zi, 0.f);
}

__global__ void __launch_bounds__(256) cd_target_kernel(const float* __restrict__ v_minus, const float* __restrict__ gtab,
                                                        const int* __restrict__ m_dev, const float* __restrict__ z_t,
                                                        const float* __restrict__ z_hat, long long per, long long n,
                                                        float* __restrict__ v_out) {
  xu_grid_dep_sync();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const float* g = gtab + 4LL * m_dev[i / per];
  const float x0 = xu_step_x0(g, z_hat[i], v_minus[i]);
  v_out[i] = __fdiv_rn(__fsub_rn(__fmul_rn(g[2], z_t[i]), x0), g[3]);
}

extern "C" int xunet_cd_teacher_step(const float* out_t, float w, int teacher_copies, const float* teacher_table,
                                     const int* m_dev, int B, long long per, const float* z_t, float* z_out, float* logsnr_out,
                                     void* stream) {
  if (!out_t || !teacher_table || !m_dev || !z_t || !z_out || !logsnr_out)
    return xu_fail("xunet_cd_teacher_step: NULL pointer argument");
  if (B < 1 || per < 1) return xu_fail("xunet_cd_teacher_step: B = %d, per = %lld, need both >= 1", B, per);
  if (teacher_copies != 1 && teacher_copies != 2)
    return xu_fail("xunet_cd_teacher_step: teacher_copies = %d, need 1 or 2", teacher_copies);
  const long long n = (long long)B * per;
  xu_launch(teacher_copies == 2 ? cd_teacher_step_kernel<true> : cd_teacher_step_kernel<false>, cdiv(n > B ? n : B, 256), 256,
            0, (cudaStream_t)stream, out_t, w, teacher_table, m_dev, per, n, B, z_t, z_out, logsnr_out);
  return xu_launched("cd_teacher_step");
}

extern "C" int xunet_cd_target(const float* v_minus, const float* target_table, const int* m_dev, const float* z_t,
                               const float* z_hat, int B, long long per, float* v_out, void* stream) {
  if (!v_minus || !target_table || !m_dev || !z_t || !z_hat || !v_out) return xu_fail("xunet_cd_target: NULL pointer argument");
  if (B < 1 || per < 1) return xu_fail("xunet_cd_target: B = %d, per = %lld, need both >= 1", B, per);
  const long long n = (long long)B * per;
  xu_launch(cd_target_kernel, cdiv(n, 256), 256, 0, (cudaStream_t)stream, v_minus, target_table, m_dev, z_t, z_hat, per, n,
            v_out);
  return xu_launched("cd_target");
}
