// sampler.cu -- one sampler step with the schedule on the device, and the C entries that launch it
// (xunet_sampler_step_table, _multistep, _dynamic, _cond and _guide): sampler_step_table_kernel clips x0 to [-1, 1],
// sampler_step_dynamic_kernel thresholds it per view (dynamic thresholding, Saharia et al. 2022, Imagen section 2.3).
//
// The dynamic step is sampler_step_table_kernel's with the fixed clip of x0 to [-1, 1] replaced by a per-view one:
//   s = max(1, quantile_p(|x0|)) over the per = S*S*3 values of the view;   x0 <- clip(x0, -s, s) / s.
// quantile_p is numpy's np.quantile(a, p) with the default 'linear' method, evaluated in fp64 on the fp32 values a = |x0|
// sorted ascending (a[0] <= ... <= a[per-1]):
//   idx = (per - 1) p,  lo = floor(idx),  hi = min(lo + 1, per - 1),  g = idx - lo,  d = a[hi] - a[lo],
//   q = g < 0.5 ? a[lo] + d g : a[hi] - d (1 - g),
// each operation rounded once (__dmul_rn / __dsub_rn / __dadd_rn: no fma contraction, as numpy), then s = fmaxf(fp32(q), 1).
// With s = 1 the thresholded value is clip(x0, -1, 1) exactly, and e, x0 and z' use the same fp32 operations in the same
// order as sampler_step_table_kernel (spelled out with intrinsics), so such a view gets the static step's bits.
//
// Layout: one thread-block cluster of DYN_CLUSTER CTAs per view (grid B * DYN_CLUSTER).  CTA r of the cluster owns the
// contiguous slice [r*chunk, min((r+1)*chunk, per)) of its view, chunk = ceil(per / DYN_CLUSTER), and keeps the guided,
// unclipped x0 of the slice in shared memory.  The order statistic a[lo] is found by a radix select on the bit patterns of
// |x0| (for non-negative floats the order of the bit patterns is the order of the values): four passes of 8-bit digits,
// high to low; per pass every CTA counts the digits of its candidates in a shared-memory histogram, the cluster syncs, and
// every CTA adds the DYN_CLUSTER histograms through distributed shared memory and derives the digit from the merged counts.
// The counts are integers, so every CTA derives the same digit with no broadcast, and s does not depend on B, on the view's
// position in the batch or on the order of any addition.  a[hi] is a[lo] when more than lo + 1 values are at or below it,
// else the cluster minimum of the keys above a[lo].  Each CTA then finishes the step for its slice from shared memory.
// No atomics outside shared memory, no scratch buffer, one launch.
#include <cooperative_groups.h>

#include "xunet_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace cg = cooperative_groups;

// One ancestral step with the schedule ON THE DEVICE (sampling.py:128-151): the coefficients of loop position k = *pos_dev come
// from a table (k = 0 is the first executed step = highest t), and the kernel also writes the NEXT forward's inputs (z into
// both halves of the [cond ; uncond] batch, the lagging log-SNR), so one CUDA graph = forward + this kernel + counter++ is
// replayed per step with no host arithmetic or copies in between.
// tab row: {c_recip, c_recipm1, c_x0, c_z, sigma, logsnr_next, c_prev, -}
// The noise of step k is noise[k*n .. k*n+n) if `noise` is set, else the hash normal of (*seed_dev - k).
// HIST = false (DDPM, DDIM): z' = c_x0 x0 + c_z z + sigma noise, as the compiler contracts it (the bits of the original
// single-step kernel).  HIST = true (multistep solvers, DPM-Solver++(2M)) fixes the order, one rounding per fma:
//   z' = fma(sigma, noise, fma(c_prev, x0_hist[i], fma(c_x0, x0, c_z * z))), the c_prev term skipped when c_prev == 0,
// then x0_hist[i] = x0.  A row with c_prev == 0 never reads x0_hist (the first step needs no initialised history).
// NEG selects where the guidance's negative output comes from:
//   NEG_HALF (classifier-free guidance): eps2 is the [cond ; uncond] output of a 2B batch, the negative is eps2[n + i], and the
//            new z goes to both halves of inp_z;
//   NEG_NONE (a model whose guidance is in its weights, e.g. a distilled student): eps2 is the B-batch conditional output, read
//            as is, and the new z goes to inp_z's n values;
//   NEG_PTR  (autoguidance): eps2 is the B-batch output of the main model, the negative is neg[i], the B-batch output of a
//            second (guide) model on the same inputs, and the new z goes to inp_z's n values.
// NEG_HALF and NEG_PTR combine the two outputs with the same fp32 operations (xu_step_guided); neg is read only by NEG_PTR.
enum SamplerNeg { NEG_NONE = 0, NEG_HALF = 1, NEG_PTR = 2 };

template <bool HIST, int NEG>
__global__ void __launch_bounds__(256) sampler_step_table_kernel(const float* __restrict__ eps2, float* __restrict__ z,
                                                                 const float* __restrict__ noise, long long n, float w,
                                                                 const float* __restrict__ tab, const int* __restrict__ pos_dev,
                                                                 const unsigned long long* __restrict__ seed_dev, float* __restrict__ inp_z,
                                                                 float* __restrict__ inp_logsnr, int B2, float* __restrict__ x0_hist,
                                                                 const float* __restrict__ neg) {
  xu_grid_dep_sync();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  const int k = *pos_dev;
  const float* t = tab + 8LL * k;
  if (i < B2) inp_logsnr[i] = t[5];
  if (i >= n) return;
  const float e = NEG == NEG_NONE ? eps2[i] : xu_step_guided(w, eps2[i], NEG == NEG_HALF ? eps2[n + i] : neg[i]);
  const float zi = z[i];
  const float x0 = xu_step_x0(t, zi, e);
  const float nz = noise != nullptr ? noise[k * n + i] : xu_hash_normal(*seed_dev - (unsigned long long)k, (uint64_t)i);
  float zn;
  if constexpr (HIST) {
    const float c_prev = t[6];
    zn = fmaf(t[2], x0, __fmul_rn(t[3], zi));
    if (c_prev != 0.f) zn = fmaf(c_prev, x0_hist[i], zn);
    zn = fmaf(t[4], nz, zn);
    x0_hist[i] = x0;
  } else {
    zn = xu_step_z(t, x0, zi, nz);
  }
  z[i] = zn;
  inp_z[i] = zn;
  if constexpr (NEG == NEG_HALF) inp_z[n + i] = zn;
}
static void launch_sampler_step_table(const float* eps2, float* z, const float* noise, long long n, float w, const float* tab,
                                      const int* pos_dev, const unsigned long long* seed_dev, float* inp_z, float* inp_logsnr,
                                      int B2, float* x0_hist, int neg_mode, const float* neg, cudaStream_t s) {
  const int grid = cdiv(n > B2 ? n : B2, 256);
  static void (*const kernels[2][3])(const float*, float*, const float*, long long, float, const float*, const int*,
                                     const unsigned long long*, float*, float*, int, float*, const float*) = {
      {sampler_step_table_kernel<false, NEG_NONE>, sampler_step_table_kernel<false, NEG_HALF>,
       sampler_step_table_kernel<false, NEG_PTR>},
      {sampler_step_table_kernel<true, NEG_NONE>, sampler_step_table_kernel<true, NEG_HALF>,
       sampler_step_table_kernel<true, NEG_PTR>}};
  xu_launch(kernels[x0_hist != nullptr][neg_mode], grid, 256, 0, s, eps2, z, noise, n, w, tab, pos_dev, seed_dev, inp_z,
            inp_logsnr, B2, x0_hist, neg);
}

#define DYN_CLUSTER 8
#define DYN_THREADS 256    // = the number of histogram bins: thread t owns bin t of the merged histogram

static constexpr int kDynMaxChunk = (XUNET_SAMPLER_DYN_MAX_PER + DYN_CLUSTER - 1) / DYN_CLUSTER;

// The fp64 'linear' quantile of the sorted values a[lo] = lo_v, a[hi] = hi_v (see the header of this file)
__device__ __forceinline__ float dyn_threshold_scale(float lo_v, float hi_v, double g) {
  const double alo = (double)lo_v, ahi = (double)hi_v;
  const double d = __dsub_rn(ahi, alo);
  const double q = g < 0.5 ? __dadd_rn(alo, __dmul_rn(d, g)) : __dsub_rn(ahi, __dmul_rn(d, __dsub_rn(1.0, g)));
  return fmaxf(__double2float_rn(q), 1.f);
}

// NEG as in sampler_step_table_kernel: NEG_HALF reads the negative from eps2[n + i] and writes both halves of inp_z, NEG_NONE
// reads eps2 as is, NEG_PTR reads the negative from neg[i]; the last two write inp_z's n values only
template <bool HIST, int NEG>
__global__ void __cluster_dims__(DYN_CLUSTER, 1, 1) __launch_bounds__(DYN_THREADS)
sampler_step_dynamic_kernel(const float* __restrict__ eps2, float* __restrict__ z, const float* __restrict__ noise, long long n,
                            float w, const float* __restrict__ tab, const int* __restrict__ pos_dev,
                            const unsigned long long* __restrict__ seed_dev, float* __restrict__ inp_z,
                            float* __restrict__ inp_logsnr, int B2, float* __restrict__ x0_hist, int per, double p,
                            float* __restrict__ scale_out, const float* __restrict__ neg) {
  extern __shared__ float xs[];                 // the guided, unclipped x0 of this CTA's slice
  __shared__ unsigned hist[2][DYN_THREADS];     // digit counts of this CTA's candidates, double-buffered across passes
  __shared__ unsigned wsum[DYN_THREADS / 32];
  __shared__ unsigned sel[3];                   // the pass's digit, the merged count below it, the merged count of it
  __shared__ unsigned minkey;                   // the smallest key above a[lo] (this CTA's, then the cluster's)
  xu_grid_dep_sync();
  cg::cluster_group cluster = cg::this_cluster();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned rank = cluster.block_rank();
  const long long view = blockIdx.x / DYN_CLUSTER;
  const int chunk = (per + DYN_CLUSTER - 1) / DYN_CLUSTER;
  const int start = min((int)rank * chunk, per), len = min(chunk, per - start);
  const long long base = view * per + start;
  const int k = *pos_dev;
  const float* t = tab + 8LL * k;
  for (long long j = (long long)blockIdx.x * DYN_THREADS + tid; j < B2; j += (long long)gridDim.x * DYN_THREADS)
    inp_logsnr[j] = t[5];

  // guided x0, as sampler_step_table_kernel contracts it: e = fma(1 + w, eps_c, -(w eps_u)), x0 = fma(c_recip, z, -(c_recipm1 e))
  const float c_recip = t[0], c_recipm1 = t[1], wp1 = __fadd_rn(1.f, w);
  for (int j = tid; j < len; j += DYN_THREADS) {
    const long long i = base + j;
    const float e = NEG == NEG_NONE ? eps2[i] : fmaf(wp1, eps2[i], -__fmul_rn(w, NEG == NEG_HALF ? eps2[n + i] : neg[i]));
    xs[j] = fmaf(c_recip, z[i], -__fmul_rn(c_recipm1, e));
  }
  hist[0][tid] = 0u;
  __syncthreads();

  // radix select of rank lo: after the pass at `shift`, the candidates are the keys whose bits above shift equal `prefix`
  const double idx = __dmul_rn((double)(per - 1), p);
  const int lo = (int)floor(idx), hi = min(lo + 1, per - 1);
  const double g = __dsub_rn(idx, (double)lo);
  unsigned prefix = 0u, mask = 0u, r = (unsigned)lo, cnt = 0u;
#pragma unroll 1
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass, buf = pass & 1;
    for (int j0 = 0; j0 < len; j0 += DYN_THREADS) {     // uniform trip count: every lane takes part in the match
      const int j = j0 + tid;
      unsigned d = DYN_THREADS;
      if (j < len) {
        const unsigned key = __float_as_uint(xs[j]) & 0x7FFFFFFFu;
        if ((key & mask) == prefix) d = (key >> shift) & 0xFFu;
      }
      const unsigned peers = __match_any_sync(0xFFFFFFFFu, d);
      if (d < DYN_THREADS && lane == __ffs(peers) - 1) atomicAdd(&hist[buf][d], (unsigned)__popc(peers));
    }
    cluster.sync();
    unsigned c = 0u;
#pragma unroll
    for (int q = 0; q < DYN_CLUSTER; ++q) c += *cluster.map_shared_rank(&hist[buf][tid], q);
    // every CTA has finished reading the other buffer (the previous pass) before this pass's cluster.sync
    hist[buf ^ 1][tid] = 0u;
    unsigned incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    unsigned excl = incl - c;
    for (int q = 0; q < warp; ++q) excl += wsum[q];
    if (excl <= r && r < excl + c) {
      sel[0] = (unsigned)tid;
      sel[1] = excl;
      sel[2] = c;
    }
    __syncthreads();
    prefix |= sel[0] << shift;
    mask |= 0xFFu << shift;
    r -= sel[1];
    cnt = sel[2];
  }
  // prefix = a[lo]'s key; lo - r keys lie below it and cnt are equal to it
  unsigned key_hi = prefix;
  if (hi != lo && (unsigned)lo - r + cnt <= (unsigned)hi) {    // a[hi] is the next larger key (the same branch in every CTA)
    unsigned m = 0xFFFFFFFFu;
    for (int j = tid; j < len; j += DYN_THREADS) {
      const unsigned key = __float_as_uint(xs[j]) & 0x7FFFFFFFu;
      if (key > prefix) m = min(m, key);
    }
    m = __reduce_min_sync(0xFFFFFFFFu, m);
    if (lane == 0) wsum[warp] = m;
    __syncthreads();
    if (tid == 0) {
      unsigned b = wsum[0];
      for (int q = 1; q < DYN_THREADS / 32; ++q) b = min(b, wsum[q]);
      minkey = b;
    }
    cluster.sync();
    if (tid == 0) {
      unsigned b = 0xFFFFFFFFu;
      for (int q = 0; q < DYN_CLUSTER; ++q) b = min(b, *cluster.map_shared_rank(&minkey, q));
      wsum[0] = b;
    }
    __syncthreads();
    key_hi = wsum[0];
  }
  // no CTA may exit while another still reads its shared memory
  auto arrived = cluster.barrier_arrive();
  const float s = dyn_threshold_scale(__uint_as_float(prefix), __uint_as_float(key_hi), g);
  if (scale_out != nullptr && rank == 0 && tid == 0) scale_out[view] = s;

  for (int j = tid; j < len; j += DYN_THREADS) {
    const long long i = base + j;
    const float x0 = __fdiv_rn(fminf(fmaxf(xs[j], -s), s), s);
    const float zi = z[i];
    const float nz = noise != nullptr ? noise[k * n + i] : xu_hash_normal(*seed_dev - (unsigned long long)k, (uint64_t)i);
    float zn = fmaf(t[2], x0, __fmul_rn(t[3], zi));
    if constexpr (HIST) {
      const float c_prev = t[6];
      if (c_prev != 0.f) zn = fmaf(c_prev, x0_hist[i], zn);
      x0_hist[i] = x0;
    }
    zn = fmaf(t[4], nz, zn);
    z[i] = zn;
    inp_z[i] = zn;
    if constexpr (NEG == NEG_HALF) inp_z[n + i] = zn;
  }
  cluster.barrier_wait(std::move(arrived));
}

// n / B <= XUNET_SAMPLER_DYN_MAX_PER values per view (the entries check it)
static void launch_sampler_step_dynamic(const float* eps2, float* z, const float* noise, long long n, float w, const float* tab,
                                        const int* pos_dev, const unsigned long long* seed_dev, float* inp_z, float* inp_logsnr,
                                        int B2, float* x0_hist, int B, double p, float* scale_out, int neg_mode,
                                        const float* neg, cudaStream_t s) {
  static void (*const kernels[2][3])(const float*, float*, const float*, long long, float, const float*, const int*,
                                     const unsigned long long*, float*, float*, int, float*, int, double, float*,
                                     const float*) = {
      {sampler_step_dynamic_kernel<false, NEG_NONE>, sampler_step_dynamic_kernel<false, NEG_HALF>,
       sampler_step_dynamic_kernel<false, NEG_PTR>},
      {sampler_step_dynamic_kernel<true, NEG_NONE>, sampler_step_dynamic_kernel<true, NEG_HALF>,
       sampler_step_dynamic_kernel<true, NEG_PTR>}};
  static bool configured = false;
  if (!configured) {
    for (auto& row : kernels)
      for (auto kernel : row)
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(float) * kDynMaxChunk));
    configured = true;
  }
  const int per = (int)(n / B);
  const size_t smem = sizeof(float) * (size_t)((per + DYN_CLUSTER - 1) / DYN_CLUSTER);
  const dim3 grid((unsigned)B * DYN_CLUSTER);
  xu_launch(kernels[x0_hist != nullptr][neg_mode], grid, DYN_THREADS, smem, s, eps2, z, noise, n, w, tab, pos_dev, seed_dev,
            inp_z, inp_logsnr, B2, x0_hist, per, p, scale_out, neg);
}

extern "C" int xunet_sampler_step_table(const float* eps2, float* z, const float* noise, long long n, float w, const float* table,
                                        const int* pos_dev, const unsigned long long* seed_dev, float* next_z2, float* next_logsnr2,
                                        int batch2, void* stream) {
  if (!eps2 || !z || !table || !pos_dev || !seed_dev || !next_z2 || !next_logsnr2 || n <= 0 || batch2 <= 0) return xu_fail("xunet_sampler_step_table: bad argument");
  launch_sampler_step_table(eps2, z, noise, n, w, table, pos_dev, seed_dev, next_z2, next_logsnr2, batch2, nullptr, NEG_HALF,
                            nullptr, (cudaStream_t)stream);
  return xu_launched("sampler_step_table");
}

extern "C" int xunet_sampler_step_multistep(const float* eps2, float* z, const float* noise, long long n, float w,
                                            const float* table, const int* pos_dev, const unsigned long long* seed_dev,
                                            float* x0_hist, float* next_z2, float* next_logsnr2, int batch2, void* stream) {
  if (!eps2 || !z || !table || !pos_dev || !seed_dev || !x0_hist || !next_z2 || !next_logsnr2 || n <= 0 || batch2 <= 0)
    return xu_fail("xunet_sampler_step_multistep: bad argument");
  launch_sampler_step_table(eps2, z, noise, n, w, table, pos_dev, seed_dev, next_z2, next_logsnr2, batch2, x0_hist, NEG_HALF,
                            nullptr, (cudaStream_t)stream);
  return xu_launched("sampler_step_multistep");
}

extern "C" int xunet_sampler_step_dynamic(const float* eps2, float* z, const float* noise, long long n, float w,
                                          const float* table, const int* pos_dev, const unsigned long long* seed_dev,
                                          float* x0_hist, int batch, double percentile, float* scale_out, float* next_z2,
                                          float* next_logsnr2, int batch2, void* stream) {
  if (!eps2 || !z || !table || !pos_dev || !seed_dev || !next_z2 || !next_logsnr2)
    return xu_fail("xunet_sampler_step_dynamic: NULL pointer argument");
  if (n <= 0 || batch2 <= 0) return xu_fail("xunet_sampler_step_dynamic: n = %lld, batch2 = %d, need both >= 1", n, batch2);
  if (batch < 1) return xu_fail("xunet_sampler_step_dynamic: batch = %d, need batch >= 1", batch);
  if (n % batch != 0) return xu_fail("xunet_sampler_step_dynamic: n = %lld is not a multiple of batch = %d", n, batch);
  if (n / batch > XUNET_SAMPLER_DYN_MAX_PER)
    return xu_fail("xunet_sampler_step_dynamic: %lld values per view, more than XUNET_SAMPLER_DYN_MAX_PER = %d", n / batch,
                   XUNET_SAMPLER_DYN_MAX_PER);
  if (!(percentile > 0.0 && percentile <= 1.0))
    return xu_fail("xunet_sampler_step_dynamic: percentile %g outside (0, 1]", percentile);
  launch_sampler_step_dynamic(eps2, z, noise, n, w, table, pos_dev, seed_dev, next_z2, next_logsnr2, batch2, x0_hist, batch,
                              percentile, scale_out, NEG_HALF, nullptr, (cudaStream_t)stream);
  return xu_launched("sampler_step_dynamic");
}

extern "C" int xunet_sampler_step_cond(const float* out, float* z, const float* noise, long long n, const float* table,
                                       const int* pos_dev, const unsigned long long* seed_dev, float* x0_hist, int batch,
                                       double percentile, float* scale_out, float* next_z, float* next_logsnr, void* stream) {
  if (!out || !z || !table || !pos_dev || !seed_dev || !next_z || !next_logsnr)
    return xu_fail("xunet_sampler_step_cond: NULL pointer argument");
  if (n <= 0 || batch < 1) return xu_fail("xunet_sampler_step_cond: n = %lld, batch = %d, need both >= 1", n, batch);
  if (n % batch != 0) return xu_fail("xunet_sampler_step_cond: n = %lld is not a multiple of batch = %d", n, batch);
  if (percentile != 0.0) {
    if (n / batch > XUNET_SAMPLER_DYN_MAX_PER)
      return xu_fail("xunet_sampler_step_cond: %lld values per view, more than XUNET_SAMPLER_DYN_MAX_PER = %d", n / batch,
                     XUNET_SAMPLER_DYN_MAX_PER);
    if (!(percentile > 0.0 && percentile <= 1.0))
      return xu_fail("xunet_sampler_step_cond: percentile %g outside (0, 1] (0 selects the fixed clip)", percentile);
    launch_sampler_step_dynamic(out, z, noise, n, 0.f, table, pos_dev, seed_dev, next_z, next_logsnr, batch, x0_hist, batch,
                                percentile, scale_out, NEG_NONE, nullptr, (cudaStream_t)stream);
  } else {
    launch_sampler_step_table(out, z, noise, n, 0.f, table, pos_dev, seed_dev, next_z, next_logsnr, batch, x0_hist, NEG_NONE,
                              nullptr, (cudaStream_t)stream);
  }
  return xu_launched("sampler_step_cond");
}

extern "C" int xunet_sampler_step_guide(const float* out_main, const float* out_guide, float* z, const float* noise, long long n,
                                        float w, const float* table, const int* pos_dev, const unsigned long long* seed_dev,
                                        float* x0_hist, int batch, double percentile, float* scale_out, float* next_z,
                                        float* next_logsnr, void* stream) {
  if (!out_main || !out_guide || !z || !table || !pos_dev || !seed_dev || !next_z || !next_logsnr)
    return xu_fail("xunet_sampler_step_guide: NULL pointer argument");
  if (n <= 0 || batch < 1) return xu_fail("xunet_sampler_step_guide: n = %lld, batch = %d, need both >= 1", n, batch);
  if (n % batch != 0) return xu_fail("xunet_sampler_step_guide: n = %lld is not a multiple of batch = %d", n, batch);
  if (percentile != 0.0) {
    if (n / batch > XUNET_SAMPLER_DYN_MAX_PER)
      return xu_fail("xunet_sampler_step_guide: %lld values per view, more than XUNET_SAMPLER_DYN_MAX_PER = %d", n / batch,
                     XUNET_SAMPLER_DYN_MAX_PER);
    if (!(percentile > 0.0 && percentile <= 1.0))
      return xu_fail("xunet_sampler_step_guide: percentile %g outside (0, 1] (0 selects the fixed clip)", percentile);
    launch_sampler_step_dynamic(out_main, z, noise, n, w, table, pos_dev, seed_dev, next_z, next_logsnr, batch, x0_hist, batch,
                                percentile, scale_out, NEG_PTR, out_guide, (cudaStream_t)stream);
  } else {
    launch_sampler_step_table(out_main, z, noise, n, w, table, pos_dev, seed_dev, next_z, next_logsnr, batch, x0_hist, NEG_PTR,
                              out_guide, (cudaStream_t)stream);
  }
  return xu_launched("sampler_step_guide");
}
