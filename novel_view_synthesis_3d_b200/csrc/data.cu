// data.cu -- one training micro-batch drawn from an SRN store in device memory, gathered and forward-diffused (xunet_srn_batch,
// xunet_srn_batch_v for v-prediction, and xunet_srn_batch_distill for progressive distillation).
//
// Grid (chunks, B): CTA (c, b) handles sample b.  Its thread 0 reads the step counter and derives the sample's draw -- source
// item, target view, diffusion seed and timestep -- into shared memory; the CTA then streams its share of the S*S*3 values:
// x from the source view, z and noise (and v, xunet_srn_batch_v) from the target view (the arithmetic of
// xunet_forward_diffusion, common.cuh), four values per thread with 16-byte stores (4-byte loads from a uint8 store) when
// the layout allows.  CTA 0 of each sample also
// writes the sample's poses, K, logsnr, cond_mask, loss weight and the optional idx / t outputs.  Every output element has one
// writer and no value is reduced, so the result is deterministic and independent of the grid.
//
// The distillation instance (TARGET == XU_TARGET_DISTILL) draws the same pairs, seeds and noise, but the timestep of sample b
// is grid_t[m_b] with m_b = (sample hash) mod n_grid, cond_mask is 1, no target is stored, and the same x, poses, K, z and
// logsnr also go to each of the teacher's `copies` row blocks (copy c of sample b = teacher row c B + b), with m_b to m_out.
//
// The draw functions below are restated in numpy by srn_data.draw_indices / diffusion_seed: change both together.
#include "xunet_b200.h"
#include "common.cuh"
#include "kernels.h"

#define SRN_THREADS 256

// xunet_srn_batch_distill: the draw of xunet_srn_batch with t = grid_t[m], m = (sample hash) mod n_grid, cond_mask 1, no
// target, and the sample's inputs copied into the teacher's `copies` row blocks
struct XuDistillDraw {
  xunet_batch teacher;    // x, z, logsnr, R1, t1, R2, t2, K of the teacher's batch (copies * B rows; cond_mask, rays unused)
  int copies;             // 2: a guided [cond ; uncond] teacher batch, 1: an unguided one
  const int* grid_t;      // the student's timesteps, loop order
  int n_grid;
  int* m_out;             // (B) the drawn grid positions
};

// key of round r of the permutation of epoch `epoch`
__host__ __device__ __forceinline__ uint64_t srn_round_key(uint64_t seed, uint64_t epoch, int r) {
  return xu_mix64(xu_mix64(seed ^ 0x243F6A8885A308D3ULL) + epoch * 4ULL + (uint64_t)r);
}
// P_{seed,epoch}(x) for x in [0, n): a 4-round Feistel network on 2h bits (4^h >= n, h >= 1), cycle-walked back into [0, n)
__host__ __device__ __forceinline__ uint64_t srn_permute(uint64_t x, uint64_t n, uint64_t seed, uint64_t epoch) {
  int h = 1;
  while ((1ULL << (2 * h)) < n) ++h;
  const uint64_t mask = (1ULL << h) - 1ULL;
  uint64_t key[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) key[r] = srn_round_key(seed, epoch, r);
  do {
    uint64_t L = x >> h, R = x & mask;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const uint64_t F = xu_mix64(R ^ key[r]) & mask;
      const uint64_t nl = R;
      R = L ^ F;
      L = nl;
    }
    x = (L << h) | R;
  } while (x >= n);
  return x;
}
// target-view hash of draw g
__host__ __device__ __forceinline__ uint64_t srn_view_hash(uint64_t seed, uint64_t g) {
  return xu_mix64(xu_mix64(seed ^ 0x13198A2E03707344ULL) + g);
}
// diffusion seed of micro-batch mb = c k + j on rank r
__host__ __device__ __forceinline__ uint64_t srn_diffusion_seed(uint64_t seed, uint64_t mb, uint64_t rank) {
  return xu_mix64(xu_mix64(xu_mix64(seed ^ 0xA4093822299F31D0ULL) + mb) + rank);
}

__device__ __forceinline__ float srn_u8(unsigned int u) { return __fmul_rn(__fsub_rn(__fdiv_rn((float)u, 255.f), .5f), 2.f); }

template <int PIX> __device__ __forceinline__ float4 srn_load4(const void* px, long long off) {
  if (PIX == XUNET_PIXELS_U8) {
    const uchar4 u = *reinterpret_cast<const uchar4*>(static_cast<const uint8_t*>(px) + off);
    return make_float4(srn_u8(u.x), srn_u8(u.y), srn_u8(u.z), srn_u8(u.w));
  }
  return *reinterpret_cast<const float4*>(static_cast<const float*>(px) + off);
}
template <int PIX> __device__ __forceinline__ float srn_load1(const void* px, long long off) {
  if (PIX == XUNET_PIXELS_U8) return srn_u8(static_cast<const uint8_t*>(px)[off]);
  return static_cast<const float*>(px)[off];
}

// TARGET == XU_TARGET_V also stores v = xu_fd_v(..) to v_out (the last parameter, so the eps instances keep their parameter
// layout and code), and `noise` may then be NULL.  TARGET == XU_TARGET_DISTILL reads `dd` (the last parameter) and takes
// noise == v_out == NULL.
template <int PIX, int TARGET>
__global__ void __launch_bounds__(SRN_THREADS) srn_batch_kernel(xunet_srn_store st, const long long* __restrict__ step_dev,
                                                                unsigned long long seed, int j, int k, int rank, int world,
                                                                const float* __restrict__ sqrt_ac,
                                                                const float* __restrict__ sqrt_1mac, float p_uncond,
                                                                const float* __restrict__ snr_weight, xunet_batch out,
                                                                float* __restrict__ noise, float* __restrict__ loss_weight,
                                                                int* __restrict__ idx_out, int* __restrict__ t_out, int vec,
                                                                float* __restrict__ v_out, XuDistillDraw dd) {
  constexpr bool V = TARGET == XU_TARGET_V, D = TARGET == XU_TARGET_DISTILL;
  __shared__ long long s_src, s_tgt;
  __shared__ unsigned long long s_seed, s_hb;
  __shared__ int s_inst, s_v, s_v2, s_t, s_m;
  xu_grid_dep_sync();
  const int b = blockIdx.y, B = gridDim.y;
  if (threadIdx.x == 0) {
    const uint64_t c = (uint64_t)(*step_dev - 1);
    const uint64_t mb = c * (uint64_t)k + (uint64_t)j;
    const uint64_t g = (mb * (uint64_t)world + (uint64_t)rank) * (uint64_t)B + (uint64_t)b;
    const uint64_t n = (uint64_t)st.n_items;
    const long long item = (long long)srn_permute(g % n, n, seed, g / n);
    const int inst = st.item_inst[item];
    const int v2 = (int)(srn_view_hash(seed, g) % (uint64_t)st.count[inst]);
    const uint64_t s = srn_diffusion_seed(seed, mb, (uint64_t)rank);
    const uint64_t hb = xu_fd_sample_hash(s, b);
    s_src = item;
    s_tgt = (long long)st.first[inst] + v2;
    s_inst = inst;
    s_v = (int)(item - st.first[inst]);
    s_v2 = v2;
    s_seed = s;
    s_hb = hb;
    if constexpr (D) {
      s_m = (int)(hb % (uint64_t)dd.n_grid);
      s_t = dd.grid_t[s_m];
    } else {
      s_t = xu_fd_timestep(hb);
    }
  }
  __syncthreads();
  const long long per = 3LL * st.S * st.S;
  const long long src = s_src * per, tgt = s_tgt * per, ob = (long long)b * per;
  const uint64_t s = s_seed;
  const int t = s_t;
  const float sa = sqrt_ac[t], sb = sqrt_1mac[t];
  float* x = const_cast<float*>(out.x);
  float* z = const_cast<float*>(out.z);
  const long long stride = (long long)gridDim.x * SRN_THREADS;
  if (vec) {
    for (long long q = (long long)blockIdx.x * SRN_THREADS + threadIdx.x; q < per / 4; q += stride) {
      const long long i = 4 * q;
      const float4 xs = srn_load4<PIX>(st.pixels, src + i);
      const float4 xt = srn_load4<PIX>(st.pixels, tgt + i);
      float4 nz, zz;
      nz.x = xu_hash_normal(s, (uint64_t)(ob + i));
      nz.y = xu_hash_normal(s, (uint64_t)(ob + i + 1));
      nz.z = xu_hash_normal(s, (uint64_t)(ob + i + 2));
      nz.w = xu_hash_normal(s, (uint64_t)(ob + i + 3));
      if constexpr (V || D) {
        zz.x = xu_fd_z_rn(sa, xt.x, sb, nz.x);
        zz.y = xu_fd_z_rn(sa, xt.y, sb, nz.y);
        zz.z = xu_fd_z_rn(sa, xt.z, sb, nz.z);
        zz.w = xu_fd_z_rn(sa, xt.w, sb, nz.w);
      } else {
        zz.x = xu_fd_z(sa, xt.x, sb, nz.x);
        zz.y = xu_fd_z(sa, xt.y, sb, nz.y);
        zz.z = xu_fd_z(sa, xt.z, sb, nz.z);
        zz.w = xu_fd_z(sa, xt.w, sb, nz.w);
      }
      *reinterpret_cast<float4*>(x + ob + i) = xs;
      *reinterpret_cast<float4*>(z + ob + i) = zz;
      if constexpr (V) {
        float4 vv;
        vv.x = xu_fd_v(sa, nz.x, sb, xt.x);
        vv.y = xu_fd_v(sa, nz.y, sb, xt.y);
        vv.z = xu_fd_v(sa, nz.z, sb, xt.z);
        vv.w = xu_fd_v(sa, nz.w, sb, xt.w);
        *reinterpret_cast<float4*>(v_out + ob + i) = vv;
        if (noise != nullptr) *reinterpret_cast<float4*>(noise + ob + i) = nz;
      } else if constexpr (D) {
        for (int c = 0; c < dd.copies; ++c) {
          const long long tb = (long long)c * B * per + ob + i;
          *reinterpret_cast<float4*>(const_cast<float*>(dd.teacher.x) + tb) = xs;
          *reinterpret_cast<float4*>(const_cast<float*>(dd.teacher.z) + tb) = zz;
        }
      } else {
        *reinterpret_cast<float4*>(noise + ob + i) = nz;
      }
    }
  } else {
    for (long long i = (long long)blockIdx.x * SRN_THREADS + threadIdx.x; i < per; i += stride) {
      const float nz = xu_hash_normal(s, (uint64_t)(ob + i));
      x[ob + i] = srn_load1<PIX>(st.pixels, src + i);
      if constexpr (V) {
        const float xt = srn_load1<PIX>(st.pixels, tgt + i);
        z[ob + i] = xu_fd_z_rn_scalar(sa, xt, sb, nz);
        v_out[ob + i] = xu_fd_v(sa, nz, sb, xt);
        if (noise != nullptr) noise[ob + i] = nz;
      } else if constexpr (D) {
        const float xt = srn_load1<PIX>(st.pixels, tgt + i), zi = xu_fd_z_rn_scalar(sa, xt, sb, nz);
        const float xi = srn_load1<PIX>(st.pixels, src + i);
        z[ob + i] = zi;
        for (int c = 0; c < dd.copies; ++c) {
          const long long tb = (long long)c * B * per + ob + i;
          const_cast<float*>(dd.teacher.x)[tb] = xi;
          const_cast<float*>(dd.teacher.z)[tb] = zi;
        }
      } else {
        z[ob + i] = xu_fd_z(sa, srn_load1<PIX>(st.pixels, tgt + i), sb, nz);
        noise[ob + i] = nz;
      }
    }
  }
  if (blockIdx.x == 0) {
    const int tid = threadIdx.x;
    if (tid < 9) {
      const_cast<float*>(out.R1)[b * 9 + tid] = st.R[s_src * 9 + tid];
      const_cast<float*>(out.R2)[b * 9 + tid] = st.R[s_tgt * 9 + tid];
      const_cast<float*>(out.K)[b * 9 + tid] = st.K[s_inst * 9 + tid];
    } else if (tid < 12) {
      const_cast<float*>(out.t1)[b * 3 + tid - 9] = st.t[s_src * 3 + tid - 9];
      const_cast<float*>(out.t2)[b * 3 + tid - 9] = st.t[s_tgt * 3 + tid - 9];
    } else if (tid == 12) {
      const_cast<float*>(out.logsnr)[b] = xu_fd_logsnr(t);
      const_cast<float*>(out.cond_mask)[b] = D ? 1.f : xu_fd_cond_mask(s_hb, p_uncond);
      if (loss_weight != nullptr) loss_weight[b] = snr_weight != nullptr ? snr_weight[t] : 1.f;
      if (t_out != nullptr) t_out[b] = t;
      if (idx_out != nullptr) {
        idx_out[b * 3 + 0] = s_inst;
        idx_out[b * 3 + 1] = s_v;
        idx_out[b * 3 + 2] = s_v2;
      }
    }
    if constexpr (D) {     // the same values into the teacher's rows, and m_b
      for (int c = 0; c < dd.copies; ++c) {
        const int tb = c * B + b;
        if (tid < 9) {
          const_cast<float*>(dd.teacher.R1)[tb * 9 + tid] = st.R[s_src * 9 + tid];
          const_cast<float*>(dd.teacher.R2)[tb * 9 + tid] = st.R[s_tgt * 9 + tid];
          const_cast<float*>(dd.teacher.K)[tb * 9 + tid] = st.K[s_inst * 9 + tid];
        } else if (tid < 12) {
          const_cast<float*>(dd.teacher.t1)[tb * 3 + tid - 9] = st.t[s_src * 3 + tid - 9];
          const_cast<float*>(dd.teacher.t2)[tb * 3 + tid - 9] = st.t[s_tgt * 3 + tid - 9];
        } else if (tid == 12) {
          const_cast<float*>(dd.teacher.logsnr)[tb] = xu_fd_logsnr(t);
        }
      }
      if (tid == 12) dd.m_out[b] = s_m;
    }
  }
}

static bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

template <int TARGET>
static void launch_srn_batch_target(const xunet_srn_store& st, const long long* step_dev, unsigned long long seed, int j, int k,
                                    int rank, int world, int B, const float* sqrt_ac, const float* sqrt_1mac, float p_uncond,
                                    const float* snr_weight, const xunet_batch& out, float* noise, float* loss_weight,
                                    int* idx_out, int* t_out, float* v_out, const XuDistillDraw& dd, cudaStream_t s) {
  const long long per = 3LL * st.S * st.S;
  const size_t px_align = st.pixel_kind == XUNET_PIXELS_U8 ? 4 : 16;
  const int vec = per % 4 == 0 && ((uintptr_t)st.pixels % px_align) == 0 && aligned16(out.x) && aligned16(out.z) &&
                  aligned16(noise) && aligned16(v_out) && aligned16(dd.teacher.x) && aligned16(dd.teacher.z);
  const long long work = vec ? per / 4 : per;
  const dim3 grid((unsigned)cdiv(work, SRN_THREADS), (unsigned)B);
  if (st.pixel_kind == XUNET_PIXELS_U8)
    xu_launch(srn_batch_kernel<XUNET_PIXELS_U8, TARGET>, grid, SRN_THREADS, 0, s, st, step_dev, seed, j, k, rank, world,
              sqrt_ac, sqrt_1mac, p_uncond, snr_weight, out, noise, loss_weight, idx_out, t_out, vec, v_out, dd);
  else
    xu_launch(srn_batch_kernel<XUNET_PIXELS_F32, TARGET>, grid, SRN_THREADS, 0, s, st, step_dev, seed, j, k, rank, world,
              sqrt_ac, sqrt_1mac, p_uncond, snr_weight, out, noise, loss_weight, idx_out, t_out, vec, v_out, dd);
}

// the argument checks of xunet_srn_batch / _v; the ε buffer `noise` is checked by the caller (optional in the v form)
static int srn_batch_check(const char* fn, const xunet_srn_store* store, const long long* step_dev, int j, int k, int rank,
                           int world, int B, const float* sqrt_ac, const float* sqrt_1mac, const xunet_batch* out) {
  if (!store || !step_dev || !sqrt_ac || !sqrt_1mac || !out || !store->pixels || !store->R || !store->t || !store->K ||
      !store->first || !store->count || !store->item_inst || !out->x || !out->z || !out->logsnr || !out->R1 || !out->t1 ||
      !out->R2 || !out->t2 || !out->K || !out->cond_mask)
    return xu_fail("%s: NULL pointer argument", fn);
  if (B < 1 || k < 1 || world < 1) return xu_fail("%s: B = %d, k = %d, world = %d, need all >= 1", fn, B, k, world);
  if (rank < 0 || rank >= world || j < 0 || j >= k)
    return xu_fail("%s: rank = %d of world = %d, j = %d of k = %d out of range", fn, rank, world, j, k);
  if (store->n_items < 1 || store->n_instances < 1 || store->S < 1)
    return xu_fail("%s: empty store (n_items = %lld, n_instances = %d, S = %d)", fn, store->n_items, store->n_instances, store->S);
  if (store->pixel_kind != XUNET_PIXELS_U8 && store->pixel_kind != XUNET_PIXELS_F32)
    return xu_fail("%s: unknown pixel_kind %d", fn, store->pixel_kind);
  return 0;
}

extern "C" int xunet_srn_batch(const xunet_srn_store* store, const long long* step_dev, unsigned long long seed, int j, int k,
                               int rank, int world, int B, const float* sqrt_ac, const float* sqrt_1mac, float p_uncond,
                               const float* snr_weight, const xunet_batch* out, float* noise, float* loss_weight, int* idx_out,
                               int* t_out, void* stream) {
  if (!noise) return xu_fail("xunet_srn_batch: NULL pointer argument");
  if (const int rc = srn_batch_check("xunet_srn_batch", store, step_dev, j, k, rank, world, B, sqrt_ac, sqrt_1mac, out)) return rc;
  launch_srn_batch_target<XU_TARGET_EPS>(*store, step_dev, seed, j, k, rank, world, B, sqrt_ac, sqrt_1mac, p_uncond, snr_weight,
                                         *out, noise, loss_weight, idx_out, t_out, nullptr, XuDistillDraw{}, (cudaStream_t)stream);
  return xu_launched("srn_batch");
}

extern "C" int xunet_srn_batch_v(const xunet_srn_store* store, const long long* step_dev, unsigned long long seed, int j, int k,
                                 int rank, int world, int B, const float* sqrt_ac, const float* sqrt_1mac, float p_uncond,
                                 const float* snr_weight, const xunet_batch* out, float* noise, float* v_out,
                                 float* loss_weight, int* idx_out, int* t_out, void* stream) {
  if (!v_out) return xu_fail("xunet_srn_batch_v: NULL pointer argument");
  if (const int rc = srn_batch_check("xunet_srn_batch_v", store, step_dev, j, k, rank, world, B, sqrt_ac, sqrt_1mac, out)) return rc;
  launch_srn_batch_target<XU_TARGET_V>(*store, step_dev, seed, j, k, rank, world, B, sqrt_ac, sqrt_1mac, p_uncond, snr_weight,
                                       *out, noise, loss_weight, idx_out, t_out, v_out, XuDistillDraw{}, (cudaStream_t)stream);
  return xu_launched("srn_batch_v");
}

extern "C" int xunet_srn_batch_distill(const xunet_srn_store* store, const long long* step_dev, unsigned long long seed, int j,
                                       int k, int rank, int world, int B, const float* sqrt_ac, const float* sqrt_1mac,
                                       const int* grid_t, int n_grid, const xunet_batch* out, const xunet_batch* teacher,
                                       int teacher_copies, int* m_out, int* idx_out, int* t_out, void* stream) {
  if (!grid_t || !teacher || !m_out || !teacher->x || !teacher->z || !teacher->logsnr || !teacher->R1 || !teacher->t1 ||
      !teacher->R2 || !teacher->t2 || !teacher->K)
    return xu_fail("xunet_srn_batch_distill: NULL pointer argument");
  if (const int rc = srn_batch_check("xunet_srn_batch_distill", store, step_dev, j, k, rank, world, B, sqrt_ac, sqrt_1mac, out))
    return rc;
  if (n_grid < 1) return xu_fail("xunet_srn_batch_distill: n_grid = %d, need >= 1", n_grid);
  if (teacher_copies != 1 && teacher_copies != 2)
    return xu_fail("xunet_srn_batch_distill: teacher_copies = %d, need 1 or 2", teacher_copies);
  const XuDistillDraw dd = {*teacher, teacher_copies, grid_t, n_grid, m_out};
  launch_srn_batch_target<XU_TARGET_DISTILL>(*store, step_dev, seed, j, k, rank, world, B, sqrt_ac, sqrt_1mac, 0.f, nullptr,
                                             *out, nullptr, nullptr, idx_out, t_out, nullptr, dd, (cudaStream_t)stream);
  return xu_launched("srn_batch_distill");
}
