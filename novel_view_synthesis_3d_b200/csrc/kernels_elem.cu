// kernels_elem.cu -- HBM-bound kernels of the X-UNet path: joint-frame GroupNorm (+SiLU/FiLM/dropout/
// resample) forward and backward, conditioning (log-SNR embedding, camera-ray NeRF posenc), resample,
// channel copies, loss, Adam, forward diffusion.  All 128-bit (fp32) / 64-bit (bf16) vectorised along C.
// The C entries of Adam, the gradient norm, forward diffusion and the dropout mask launch their kernels here.
#include "common.cuh"
#include "kernels.h"
#include <string.h>

#include <map>
#include <utility>
#include <vector>

static thread_local char g_kernel_error[256] = "";
const char* xu_kernel_error() { return g_kernel_error; }
void xu_set_kernel_error(const char* msg) {
  strncpy(g_kernel_error, msg, sizeof(g_kernel_error) - 1);
  g_kernel_error[sizeof(g_kernel_error) - 1] = 0;
}

// ---- order-insensitive accumulation (kernels.h) --------------------------------------------------------------------------
struct XuDetScratch {
  struct Region { double* p = nullptr; long long n = 0; };
  bool stream_ordered = false;
  int device = -1;                                       // engine owner: the device of its first allocation
  cudaStream_t zero_stream = nullptr;                    // engine owner: zeroes new regions outside any capture
  std::map<cudaStream_t, Region> regions;                // engine owner: one region per stream
  std::vector<double*> retired;                          // engine owner: outgrown regions (a captured graph may still use them)
  std::vector<std::pair<double*, cudaStream_t>> taken;   // call-scoped owner: stream-ordered allocations to release
};
static thread_local XuDetScratch* t_det = nullptr;

XuDetScratch* xu_det_create(bool stream_ordered) {
  XuDetScratch* d = new XuDetScratch();
  d->stream_ordered = stream_ordered;
  return d;
}
void xu_det_destroy(XuDetScratch* d) {
  if (d == nullptr) return;
  for (auto& t : d->taken) cudaFreeAsync(t.first, t.second);
  if (d->device >= 0) {
    int cur = -1;
    cudaGetDevice(&cur);
    cudaSetDevice(d->device);
    for (auto& r : d->regions) cudaFree(r.second.p);    // waits for the work that still uses the region
    for (double* p : d->retired) cudaFree(p);
    if (d->zero_stream != nullptr) cudaStreamDestroy(d->zero_stream);
    cudaSetDevice(cur);
  }
  delete d;
}
XuDetBind::XuDetBind(XuDetScratch* d) : prev(t_det) { t_det = d; }
XuDetBind::~XuDetBind() { t_det = prev; }

double* xu_det_scratch(cudaStream_t s, long long n) {
  XuDetScratch* d = t_det;
  if (d == nullptr) {
    xu_set_kernel_error("xu_det_scratch: no reduction scratch is bound to this call");
    return nullptr;
  }
  const size_t bytes = sizeof(double) * (size_t)n;
  if (d->stream_ordered) {
    double* p = nullptr;
    if (cudaMallocAsync(&p, bytes, s) != cudaSuccess || cudaMemsetAsync(p, 0, bytes, s) != cudaSuccess) {
      xu_set_kernel_error("xu_det_scratch: stream-ordered allocation failed");
      return nullptr;
    }
    d->taken.emplace_back(p, s);
    return p;
  }
  int dev = -1;
  cudaGetDevice(&dev);
  if (d->device < 0) d->device = dev;
  if (dev != d->device) {
    xu_set_kernel_error("xu_det_scratch: the engine is used on a different device than it was first run on");
    return nullptr;
  }
  XuDetScratch::Region& r = d->regions[s];
  if (n <= r.n) return r.p;
  // a larger region replaces the old one, which stays allocated until the owner goes.  cudaMalloc is legal during stream capture in relaxed mode, and the new region is zeroed
  // on the owner's private stream, outside any graph.
  const long long want = n < (1LL << 16) ? (1LL << 16) : n;
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  cudaThreadExchangeStreamCaptureMode(&mode);
  double* p = nullptr;
  const bool ok = (d->zero_stream != nullptr || cudaStreamCreateWithFlags(&d->zero_stream, cudaStreamNonBlocking) == cudaSuccess) &&
                  cudaMalloc(&p, sizeof(double) * want) == cudaSuccess &&
                  cudaMemsetAsync(p, 0, sizeof(double) * want, d->zero_stream) == cudaSuccess &&
                  cudaStreamSynchronize(d->zero_stream) == cudaSuccess;
  cudaThreadExchangeStreamCaptureMode(&mode);
  if (!ok) {
    xu_set_kernel_error("xu_det_scratch: allocating the reduction scratch failed");
    return nullptr;
  }
  if (r.p != nullptr) d->retired.push_back(r.p);
  r.p = p; r.n = want;
  return p;
}

__global__ void __launch_bounds__(256) det_fold_kernel(float* __restrict__ dst, double* __restrict__ acc, long long n) {
  xu_grid_dep_sync();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  dst[i] += (float)acc[i];
  acc[i] = 0.0;
}
void xu_det_fold(float* dst, double* acc, long long n, cudaStream_t s) {
  if (n > 0 && acc != nullptr) xu_launch(det_fold_kernel, cdiv(n, 256), 256, 0, s, dst, acc, n);
}

// lanes l, l' of a warp hold partial sums of the same channel vector iff (l - l') % TPB == 0 (when TPB divides 32):
// fold them with xor-shuffles so that only the first TPB lanes touch shared memory (cuts smem-atomic contention 4-32x)
__device__ __forceinline__ bool fold_same_channel_lanes(float (&v)[4], int TPB) {
  if (TPB >= 32 || (32 % TPB) != 0) return true;
  for (int off = TPB; off < 32; off <<= 1) {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] += __shfl_xor_sync(0xffffffffu, v[j], off);
  }
  return (threadIdx.x & 31) < TPB;
}

// ======================================================================================================
// GroupNorm  (model/xunet.py:46-52: nn.GroupNorm(32) on (B,2,H,W,C) -> statistics over F,H,W,C/32 jointly)
// ======================================================================================================
static void gn_grid(int C, int P, int B, dim3& grid, int& ppb) {
  int C4 = C / 4;
  int TPB = C4 < 256 ? C4 : 256;
  int PL = 256 / TPB;
  ppb = PL * 8;
  // enough blocks to cover the memory latency (reductions are latency-bound), but not absurdly many atomics
  while ((long long)cdiv(P, ppb) * B > xu_device_sms() * 8 && ppb < P) ppb *= 2;
  grid = dim3(cdiv(P, ppb), B);
}

// Per-(sample, channel) statistics for tensors whose producer cannot emit them in its epilogue: channel sums kept in shared
// memory, one interleaved [sum, sumsq] red per channel and block.
template <typename T>
__global__ void __launch_bounds__(256) gn_cstats_kernel(const T* __restrict__ x, double* __restrict__ cstats, int P, int C,
                                                        int ppb) {
  xu_grid_dep_sync();
  extern __shared__ double scsd[];   // [C][2]
  const int tid = threadIdx.x, b = blockIdx.y;
  for (int i = tid; i < 2 * C; i += 256) scsd[i] = 0.0;
  __syncthreads();
  const int C4 = C >> 2;
  const int TPB = C4 < 256 ? C4 : 256;
  const int PL = 256 / TPB;
  const int cv0 = tid % TPB, pl = tid / TPB;
  const int pbeg = blockIdx.x * ppb;
  const int pend = min(pbeg + ppb, P);
  for (int cv = cv0; cv < C4; cv += TPB) {
    float s[4] = {0.f, 0.f, 0.f, 0.f}, ss[4] = {0.f, 0.f, 0.f, 0.f};
    const T* base = x + ((long long)b * P) * C + cv * 4;
    if (pl < PL)
#pragma unroll 4
      for (int p = pbeg + pl; p < pend; p += PL) {
        float v[4];
        Vec4<T>::ldg(base + (long long)p * C, v);
#pragma unroll
        for (int j = 0; j < 4; ++j) { s[j] += v[j]; ss[j] = fmaf(v[j], v[j], ss[j]); }
      }
    const bool owner = fold_same_channel_lanes(s, TPB);
    fold_same_channel_lanes(ss, TPB);
    if (owner && pl < PL) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        xu_det_add(&scsd[(cv * 4 + j) * 2 + 0], s[j]);
        xu_det_add(&scsd[(cv * 4 + j) * 2 + 1], ss[j]);
      }
    }
  }
  __syncthreads();
  double* dst = cstats + (long long)b * C * 2;
  for (int i = tid; i < 2 * C; i += 256) atomicAdd(&dst[i], scsd[i]);
}

void launch_gn_cstats(int dtype, const void* x, float* cstats, int N, int H, int W, int C, cudaStream_t s) {
  const int B = N / 2, P = 2 * H * W;
  dim3 grid; int ppb;
  gn_grid(C, P, B, grid, ppb);
  const size_t smem = sizeof(double) * 2 * C;
  double* acc = xu_det_scratch(s, (long long)B * C * 2);
  if (acc == nullptr) return;
  if (dtype == XU_F32) xu_launch(gn_cstats_kernel<float>, grid, 256, smem, s, (const float*)x, acc, P, C, ppb);
  else xu_launch(gn_cstats_kernel<bf16>, grid, 256, smem, s, (const bf16*)x, acc, P, C, ppb);
  xu_det_fold(cstats, acc, (long long)B * C * 2, s);
}

struct GnDev {
  const void* x; void* y; const void* e; const void* dy; void* de;
  const float* gamma; const float* beta; float* dgamma; float* dbeta; float* stats; float* bstats;
  int N, H, W, C, Ho, Wo, mode, rs, train, op_index, accumulate, de_accumulate;
  float drop_rate, inv_cnt;
  int cpg, cpg_shift;   // channels per group; log2 if a power of two, else -1
  const void* extra; float extra_alpha;
  const unsigned long long* seed_dev;
  const float* cstatsA; const float* cstatsB; int csA;
  float4* params_out; const float* bcs;
  double* acc;          // gn_bwd_reduce: fp64 sums [dgamma C][dbeta C][bstats (N/2) x groups x 2] (xu_det_scratch)
};

static GnDev gn_dev(const GnArgs& a) {
  GnDev d;
  d.x = a.x; d.y = a.y; d.e = a.e; d.dy = a.dy; d.de = a.de; d.gamma = a.gamma; d.beta = a.beta;
  d.dgamma = a.dgamma; d.dbeta = a.dbeta; d.stats = a.stats; d.bstats = a.bstats;
  d.N = a.N; d.H = a.H; d.W = a.W; d.C = a.C;
  d.Ho = a.rs == RS_DOWN ? a.H / 2 : (a.rs == RS_UP ? a.H * 2 : a.H);
  d.Wo = a.rs == RS_DOWN ? a.W / 2 : (a.rs == RS_UP ? a.W * 2 : a.W);
  d.mode = a.mode; d.rs = a.rs; d.train = a.train; d.op_index = a.op_index; d.accumulate = a.accumulate;
  d.de_accumulate = a.de_accumulate;
  d.drop_rate = a.drop_rate;
  d.inv_cnt = 1.f / (2.f * a.H * a.W * (a.C / XU_GROUPS));
  d.cpg = a.C / XU_GROUPS;
  d.cpg_shift = -1;
  for (int sft = 0; sft < 12; ++sft) if ((1 << sft) == d.cpg) d.cpg_shift = sft;
  d.seed_dev = a.seed_dev;
  d.extra = a.extra; d.extra_alpha = a.extra_alpha;
  d.cstatsA = a.cstatsA; d.cstatsB = a.cstatsB; d.csA = a.csA;
  d.params_out = reinterpret_cast<float4*>(a.params_out); d.bcs = a.bcs;
  return d;
}

__device__ __forceinline__ int gn_group(const GnDev& d, int c) { return d.cpg_shift >= 0 ? (c >> d.cpg_shift) : c / d.cpg; }
__device__ __forceinline__ void gn_mean_rstd(const GnDev& d, int b, int c, float& mean, float& rstd) {
  const int g = gn_group(d, c);
  const float s = d.stats[(b * XU_GROUPS + g) * 2 + 0], q = d.stats[(b * XU_GROUPS + g) * 2 + 1];
  mean = s * d.inv_cnt;
  float var = fmaxf(q * d.inv_cnt - mean * mean, 0.f);
  rstd = rsqrtf(var + XU_GN_EPS);
}

// normalised+affine value of 4 channels of input pixel (n,y,x); optionally returns xhat
template <typename T>
__device__ __forceinline__ void gn_yhat4(const GnDev& d, int n, int y, int x, int c0, const float (&mean)[4],
                                         const float (&rstd)[4], const float (&gm)[4], const float (&bt)[4],
                                         float (&yh)[4], float (&xh)[4]) {
  float v[4];
  Vec4<T>::ldg(reinterpret_cast<const T*>(d.x) + (((long long)n * d.H + y) * d.W + x) * d.C + c0, v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    xh[j] = (v[j] - mean[j]) * rstd[j];
    yh[j] = fmaf(xh[j], gm[j], bt[j]);
  }
}

// group sums of sample b into s_grp: the producers of x emitted per-channel sums, folded here into the 32 group sums (8 lanes
// per group) -- there is no statistics pass over x.  Block 0 of each sample also stores the group sums where the backward
// kernels read them.
template <typename T>
__device__ __forceinline__ void gn_group_prologue(const GnDev& d, int b, float (*s_grp)[2]) {
  const int tid = threadIdx.x;
  const int g = tid >> 3, sub = tid & 7;
  float s = 0.f, q = 0.f;
  for (int k = sub; k < d.cpg; k += 8) {
    const int c = g * d.cpg + k;
    const float* src = c < d.csA ? d.cstatsA + ((long long)b * d.csA + c) * 2
                                 : d.cstatsB + ((long long)b * (d.C - d.csA) + (c - d.csA)) * 2;
    const float2 v = *reinterpret_cast<const float2*>(src);
    s += v.x; q += v.y;
  }
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
  if (sub == 0) {
    s_grp[g][0] = s; s_grp[g][1] = q;
    if (blockIdx.x == 0) { d.stats[(b * XU_GROUPS + g) * 2 + 0] = s; d.stats[(b * XU_GROUPS + g) * 2 + 1] = q; }
  }
  __syncthreads();
}
__device__ __forceinline__ void gn_group_mean_rstd(const GnDev& d, const float (*s_grp)[2], int c, float& mean, float& rstd) {
  const int g = gn_group(d, c);
  mean = s_grp[g][0] * d.inv_cnt;
  rstd = rsqrtf(fmaxf(s_grp[g][1] * d.inv_cnt - mean * mean, 0.f) + XU_GN_EPS);
}

// GroupNorm (+ swish) with resampling: RS_DOWN averages 2x2 pixels of the activation, RS_UP repeats each pixel 2x2 (the
// first norm of a ResnetBlock that resamples).
// grid (pixel chunks of the OUTPUT, B): every thread owns a fixed 4-channel vector, so the per-channel constants
// (mean, rstd, gamma, beta) are formed once and the inner loop is load -> fma -> activation -> store.
template <typename T>
__global__ void __launch_bounds__(256) gn_apply_kernel(GnDev d, int ppb) {
  xu_grid_dep_sync();
  const int tid = threadIdx.x, b = blockIdx.y;
  __shared__ float s_grp[XU_GROUPS][2];
  gn_group_prologue<T>(d, b, s_grp);
  const int C4 = d.C >> 2;
  const int TPB = C4 < 256 ? C4 : 256;
  const int PL = 256 / TPB;
  const int cv0 = tid % TPB, pl = tid / TPB;
  if (pl >= PL) return;
  const int HWo = d.Ho * d.Wo, P = 2 * HWo;
  const int pbeg = blockIdx.x * ppb;
  const int pend = min(pbeg + ppb, P);
  for (int cv = cv0; cv < C4; cv += TPB) {
    const int c0 = cv * 4;
    float mean[4], rstd[4], gm[4], bt[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      gn_group_mean_rstd(d, s_grp, c0 + j, mean[j], rstd[j]);
      gm[j] = d.gamma[c0 + j];
      bt[j] = d.beta[c0 + j];
    }
#pragma unroll 2
    for (int p = pbeg + pl; p < pend; p += PL) {
      const int f = p / HWo, r = p - f * HWo;
      const int oy = r / d.Wo, ox = r - oy * d.Wo, n = b * 2 + f;
      const long long pix = (long long)(2 * b) * HWo + p;
      float out[4], yh[4], xh[4];
      if (d.rs == RS_DOWN) {
#pragma unroll
        for (int j = 0; j < 4; ++j) out[j] = 0.f;
        for (int i = 0; i < 2; ++i)
          for (int k = 0; k < 2; ++k) {
            gn_yhat4<T>(d, n, oy * 2 + i, ox * 2 + k, c0, mean, rstd, gm, bt, yh, xh);
#pragma unroll
            for (int j = 0; j < 4; ++j) out[j] += (d.mode == GN_SWISH) ? swishf_(yh[j]) : yh[j];
          }
#pragma unroll
        for (int j = 0; j < 4; ++j) out[j] *= 0.25f;
      } else {
        gn_yhat4<T>(d, n, oy >> 1, ox >> 1, c0, mean, rstd, gm, bt, yh, xh);
#pragma unroll
        for (int j = 0; j < 4; ++j) out[j] = (d.mode == GN_SWISH) ? swishf_(yh[j]) : yh[j];
      }
      Vec4<T>::st(reinterpret_cast<T*>(d.y) + pix * d.C + c0, out);
    }
  }
}

// pixels per block for the elementwise GroupNorm passes: ~16 pixels per thread, >= 2 waves of blocks when possible
static void gn_apply_grid(int C, int P, int B, dim3& grid, int& ppb) {
  int C4 = C / 4;
  int TPB = C4 < 256 ? C4 : 256;
  int PL = 256 / TPB;
  ppb = PL * 16;   // the per-thread prologue (statistics -> scale/shift) is ~200 instructions: amortise it over >= 8 pixels
  // down to 4 pixels per thread (measured: 4 beats 8 and 2; latency-bound: more blocks in flight)
  while (ppb > PL * 4 && (long long)cdiv(P, ppb) * B < xu_device_sms() * 4) ppb /= 2;
  grid = dim3(cdiv(P, ppb), B);
}

// ---- no-resample fast paths: 16-byte accesses for both dtypes (8 bf16 / 4 fp32 channels per thread), U pixels of loads in
// flight per thread before the first use, per-channel affine folded to one fma: yhat = x * a + b -----------------------------
template <typename T, bool FILM>
__global__ void __launch_bounds__(256, FILM ? 2 : 3) gn_apply_vec_kernel(GnDev d, int ppb) {
  xu_grid_dep_sync();
  constexpr int VW = VecW<T>::W;
  constexpr int U = FILM ? 4 : 8;
  const int tid = threadIdx.x, b = blockIdx.y;
  __shared__ float s_grp[XU_GROUPS][2];
  gn_group_prologue<T>(d, b, s_grp);
  if (d.params_out != nullptr && blockIdx.x == 0) {
    for (int c = tid; c < d.C; c += 256) {
      float mean, rstd;
      gn_group_mean_rstd(d, s_grp, c, mean, rstd);
      d.params_out[(long long)b * d.C + c] = make_float4(rstd, -mean * rstd, d.gamma[c], d.beta[c]);
    }
  }
  const int CV = d.C / VW;
  const int TPB = CV < 256 ? CV : 256;
  const int PL = 256 / TPB;
  const int cv0 = tid % TPB, pl = tid / TPB;
  if (pl >= PL) return;
  const int HW = d.H * d.W, P = 2 * HW;
  const int pbeg = blockIdx.x * ppb;
  const int pend = min(pbeg + ppb, P);
  constexpr bool film = FILM;
  const bool swish = d.mode != GN_PLAIN;
  const bool drop = film && d.train && d.drop_rate > 0.f;
  const unsigned long long seed = drop ? *d.seed_dev : 0ULL;
  const float keep_scale = 1.f / (1.f - d.drop_rate);
  const long long pix0 = (long long)(2 * b) * HW;
  for (int cv = cv0; cv < CV; cv += TPB) {
    const int c0 = cv * VW;
    float ka[VW], kb[VW];
#pragma unroll
    for (int j = 0; j < VW; ++j) {
      float mean, rstd;
      gn_group_mean_rstd(d, s_grp, c0 + j, mean, rstd);
      ka[j] = rstd * d.gamma[c0 + j];
      kb[j] = fmaf(-mean, ka[j], d.beta[c0 + j]);
    }
    const T* X = reinterpret_cast<const T*>(d.x) + pix0 * d.C + c0;
    const T* E = film ? reinterpret_cast<const T*>(d.e) + pix0 * (2LL * d.C) + c0 : nullptr;
    T* Y = reinterpret_cast<T*>(d.y) + pix0 * d.C + c0;
    for (int p0 = pbeg + pl; p0 < pend; p0 += U * PL) {
      typename VecW<T>::raw xr[U], scr[FILM ? U : 1], shr[FILM ? U : 1];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int p = p0 + u * PL;
        if (p < pend) {
          xr[u] = VecW<T>::ldg(X + (long long)p * d.C);
          if constexpr (film) {
            scr[u] = VecW<T>::ldg(E + (long long)p * (2 * d.C));
            shr[u] = VecW<T>::ldg(E + (long long)p * (2 * d.C) + d.C);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int p = p0 + u * PL;
        if (p >= pend) break;
        float v[VW], out[VW];
        VecW<T>::unpack(xr[u], v);
        if constexpr (film) {
          float sc[VW], sh[VW];
          VecW<T>::unpack(scr[u], sc);
          VecW<T>::unpack(shr[u], sh);
          uint32_t km = 0xFFu;
          if (drop) {
            const unsigned long long e4 = (unsigned long long)((pix0 + p) * d.C + c0) >> 2;
            km = xu_keep4(seed, d.op_index, e4, d.drop_rate);
            if (VW == 8) km |= xu_keep4(seed, d.op_index, e4 + 1, d.drop_rate) << 4;
          }
#pragma unroll
          for (int j = 0; j < VW; ++j) {
            const float yh = fmaf(v[j], ka[j], kb[j]);
            float sv = swishf_(fmaf(yh, 1.f + sc[j], sh[j]));
            if (drop) sv = ((km >> j) & 1u) ? sv * keep_scale : 0.f;
            out[j] = sv;
          }
        } else {
#pragma unroll
          for (int j = 0; j < VW; ++j) {
            const float yh = fmaf(v[j], ka[j], kb[j]);
            out[j] = swish ? swishf_(yh) : yh;
          }
        }
        VecW<T>::st(Y + (long long)p * d.C, out);
      }
    }
  }
}

// pixels per block for the vector kernels
static void gn_vec_grid(int C, int VW, int P, int B, dim3& grid, int& ppb) {
  const int CV = C / VW;
  const int TPB = CV < 256 ? CV : 256;
  const int PL = 256 / TPB;
  ppb = PL * 32;                    // several batches of U pixels per thread when the tensor is large
  while (ppb > PL * 4 && (long long)cdiv(P, ppb) * B < xu_device_sms() * 4) ppb /= 2;
  grid = dim3(cdiv(P, ppb), B);
}

void launch_gn_apply(int dtype, const GnArgs& a, cudaStream_t s) {
  GnDev d = gn_dev(a);
  dim3 grid; int ppb;
  if (a.rs == RS_NONE) {
    const bool film = a.mode == GN_FILM;
    if (dtype == XU_F32) {
      gn_vec_grid(d.C, 4, 2 * d.H * d.W, d.N / 2, grid, ppb);
      if (film) xu_launch(gn_apply_vec_kernel<float, true>, grid, 256, 0, s, d, ppb);
      else xu_launch(gn_apply_vec_kernel<float, false>, grid, 256, 0, s, d, ppb);
    } else {
      gn_vec_grid(d.C, 8, 2 * d.H * d.W, d.N / 2, grid, ppb);
      if (film) xu_launch(gn_apply_vec_kernel<bf16, true>, grid, 256, 0, s, d, ppb);
      else xu_launch(gn_apply_vec_kernel<bf16, false>, grid, 256, 0, s, d, ppb);
    }
    return;
  }
  if (a.mode == GN_FILM || a.params_out != nullptr) {
    xu_set_kernel_error("gn_apply: a resampling norm has no FiLM and no fused backward");
    return;
  }
  gn_apply_grid(d.C, 2 * d.Ho * d.Wo, d.N / 2, grid, ppb);
  if (dtype == XU_F32) xu_launch(gn_apply_kernel<float>, grid, 256, 0, s, d, ppb);
  else xu_launch(gn_apply_kernel<bf16>, grid, 256, 0, s, d, ppb);
}

// gradient w.r.t. yhat (the GroupNorm output before activation/FiLM) for 4 channels of INPUT pixel (n,y,x).
// For GN_FILM also returns du (grad wrt pre-swish u) so the caller can emit de.
template <typename T>
__device__ __forceinline__ void gn_dyhat4(const GnDev& d, int n, int y, int x, int c0, const float (&yh)[4],
                                          unsigned long long seed, float (&dyh)[4], float (&du)[4]) {
  const T* dout = reinterpret_cast<const T*>(d.dy);
  float g[4];
  if (d.rs == RS_NONE) {
    Vec4<T>::ldg(dout + (((long long)n * d.H + y) * d.W + x) * d.C + c0, g);
  } else if (d.rs == RS_DOWN) {
    // forward averaged 2x2 -> each input pixel receives 0.25 * dout[y/2, x/2] (odd trailing row/col gets none)
    const int oy = y >> 1, ox = x >> 1;
    if (oy < d.Ho && ox < d.Wo) {
      Vec4<T>::ldg(dout + (((long long)n * d.Ho + oy) * d.Wo + ox) * d.C + c0, g);
#pragma unroll
      for (int j = 0; j < 4; ++j) g[j] *= 0.25f;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) g[j] = 0.f;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) g[j] = 0.f;
    for (int i = 0; i < 2; ++i)
      for (int k = 0; k < 2; ++k) {
        float t[4];
        Vec4<T>::ldg(dout + (((long long)n * d.Ho + (2 * y + i)) * d.Wo + (2 * x + k)) * d.C + c0, t);
#pragma unroll
        for (int j = 0; j < 4; ++j) g[j] += t[j];
      }
  }
  if (d.mode == GN_PLAIN) {
#pragma unroll
    for (int j = 0; j < 4; ++j) { dyh[j] = g[j]; du[j] = 0.f; }
  } else if (d.mode == GN_SWISH) {
#pragma unroll
    for (int j = 0; j < 4; ++j) { dyh[j] = g[j] * swish_gradf_(yh[j]); du[j] = 0.f; }
  } else {
    const long long pix = ((long long)n * d.H + y) * d.W + x;
    const T* e = reinterpret_cast<const T*>(d.e) + pix * (2LL * d.C);
    float sc[4], sh[4];
    Vec4<T>::ldg(e + c0, sc);
    Vec4<T>::ldg(e + d.C + c0, sh);
    const bool drop = d.train && d.drop_rate > 0.f;
    const float keep_scale = 1.f / (1.f - d.drop_rate);
    const uint32_t km = drop ? xu_keep4(seed, d.op_index, (unsigned long long)(pix * d.C + c0) >> 2, d.drop_rate) : 0xFu;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float u = fmaf(yh[j], 1.f + sc[j], sh[j]);
      float gs = g[j];
      if (drop) gs = ((km >> j) & 1u) ? gs * keep_scale : 0.f;
      du[j] = gs * swish_gradf_(u);
      dyh[j] = du[j] * (1.f + sc[j]);
    }
  }
}

// compute-only part of gn_dyhat4 for the no-resample fast path (operands already in registers)
__device__ __forceinline__ void gn_dyhat_compute(int mode, const float (&g)[4], const float (&yh)[4], const float (&sc)[4],
                                                 const float (&sh)[4], uint32_t km, bool drop, float keep_scale,
                                                 float (&dyh)[4], float (&du)[4]) {
  if (mode == GN_PLAIN) {
#pragma unroll
    for (int j = 0; j < 4; ++j) { dyh[j] = g[j]; du[j] = 0.f; }
  } else if (mode == GN_SWISH) {
#pragma unroll
    for (int j = 0; j < 4; ++j) { dyh[j] = g[j] * swish_gradf_(yh[j]); du[j] = 0.f; }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float u = fmaf(yh[j], 1.f + sc[j], sh[j]);
      float gs = g[j];
      if (drop) gs = ((km >> j) & 1u) ? gs * keep_scale : 0.f;
      du[j] = gs * swish_gradf_(u);
      dyh[j] = du[j] * (1.f + sc[j]);
    }
  }
}

// pass A: per-channel sums  A_c = sum dyh*xhat (-> dgamma),  B_c = sum dyh (-> dbeta); group sums S1,S2; FiLM de.
template <typename T>
__global__ void __launch_bounds__(256) gn_bwd_reduce_kernel(GnDev d, int ppb) {
  xu_grid_dep_sync();
  extern __shared__ double smd[];  // sA[C], sB[C]
  double* sA = smd;
  double* sB = smd + d.C;
  const int tid = threadIdx.x, b = blockIdx.y;
  for (int i = tid; i < 2 * d.C; i += 256) smd[i] = 0.0;
  __syncthreads();
  const int C4 = d.C >> 2;
  const int TPB = C4 < 256 ? C4 : 256;
  const int PL = 256 / TPB;
  const int cv0 = tid % TPB, pl = tid / TPB;
  const int P = 2 * d.H * d.W, HW = d.H * d.W;
  const int pbeg = blockIdx.x * ppb;
  const int pend = min(pbeg + ppb, P);
  const unsigned long long seed = (d.mode == GN_FILM && d.train && d.drop_rate > 0.f) ? *d.seed_dev : 0ULL;
  {
    for (int cv = cv0; cv < C4; cv += TPB) {
      const int c0 = cv * 4;
      float mean[4], rstd[4], gm[4], bt[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        gn_mean_rstd(d, b, c0 + j, mean[j], rstd[j]);
        gm[j] = d.gamma[c0 + j];
        bt[j] = d.beta[c0 + j];
      }
      float A[4] = {0.f, 0.f, 0.f, 0.f}, Bc[4] = {0.f, 0.f, 0.f, 0.f};
      if (pl < PL && d.rs == RS_NONE) {
        // fast path (no resampling): 4 pixels per trip, all loads issued before the first use
        constexpr int U = 4;
        const bool film = d.mode == GN_FILM;
        const bool drop = film && d.train && d.drop_rate > 0.f;
        const float keep_scale = 1.f / (1.f - d.drop_rate);
        const long long pix0 = (long long)(2 * b) * HW;
        const T* X = reinterpret_cast<const T*>(d.x) + pix0 * d.C + c0;
        const T* G = reinterpret_cast<const T*>(d.dy) + pix0 * d.C + c0;
        const T* E = film ? reinterpret_cast<const T*>(d.e) + pix0 * (2LL * d.C) + c0 : nullptr;
        T* DE = film ? reinterpret_cast<T*>(d.de) + pix0 * (2LL * d.C) + c0 : nullptr;
        for (int p0 = pbeg + pl; p0 < pend; p0 += U * PL) {
          typename Vec4<T>::raw xr[U], gr[U], scr[U], shr[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int p = p0 + u * PL;
            if (p < pend) {
              xr[u] = Vec4<T>::ldg_raw(X + (long long)p * d.C);
              gr[u] = Vec4<T>::ldg_raw(G + (long long)p * d.C);
              if (film) {
                scr[u] = Vec4<T>::ldg_raw(E + (long long)p * (2 * d.C));
                shr[u] = Vec4<T>::ldg_raw(E + (long long)p * (2 * d.C) + d.C);
              }
            }
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int p = p0 + u * PL;
            if (p >= pend) break;
            float v[4], g[4], sc[4] = {0.f, 0.f, 0.f, 0.f}, sh[4] = {0.f, 0.f, 0.f, 0.f}, xh[4], yh[4], dyh[4], du[4];
            Vec4<T>::unpack(xr[u], v);
            Vec4<T>::unpack(gr[u], g);
            if (film) { Vec4<T>::unpack(scr[u], sc); Vec4<T>::unpack(shr[u], sh); }
#pragma unroll
            for (int j = 0; j < 4; ++j) { xh[j] = (v[j] - mean[j]) * rstd[j]; yh[j] = fmaf(xh[j], gm[j], bt[j]); }
            const uint32_t km = drop ? xu_keep4(seed, d.op_index, (unsigned long long)((pix0 + p) * d.C + c0) >> 2, d.drop_rate) : 0xFu;
            gn_dyhat_compute(d.mode, g, yh, sc, sh, km, drop, keep_scale, dyh, du);
#pragma unroll
            for (int j = 0; j < 4; ++j) { A[j] = fmaf(dyh[j], xh[j], A[j]); Bc[j] += dyh[j]; }
            if (film) {
              T* de = DE + (long long)p * (2 * d.C);
              float dsc[4], dsh[4];
#pragma unroll
              for (int j = 0; j < 4; ++j) { dsc[j] = du[j] * yh[j]; dsh[j] = du[j]; }
              if (d.de_accumulate) {
                float o1[4], o2[4];
                Vec4<T>::ld(de, o1);
                Vec4<T>::ld(de + d.C, o2);
#pragma unroll
                for (int j = 0; j < 4; ++j) { dsc[j] += o1[j]; dsh[j] += o2[j]; }
              }
              Vec4<T>::st(de, dsc);
              Vec4<T>::st(de + d.C, dsh);
            }
          }
        }
      } else if (pl < PL)
#pragma unroll 2
      for (int p = pbeg + pl; p < pend; p += PL) {
        int n = 2 * b, y = 0, x = p;             // linear addressing unless the op resamples
        if (d.rs != RS_NONE) {
          const int f = p / HW, r = p - f * HW;
          y = r / d.W; x = r - y * d.W; n = b * 2 + f;
        }
        float yh[4], xh[4], dyh[4], du[4];
        gn_yhat4<T>(d, n, y, x, c0, mean, rstd, gm, bt, yh, xh);
        gn_dyhat4<T>(d, n, y, x, c0, yh, seed, dyh, du);
#pragma unroll
        for (int j = 0; j < 4; ++j) { A[j] = fmaf(dyh[j], xh[j], A[j]); Bc[j] += dyh[j]; }
        if (d.mode == GN_FILM) {
          T* de = reinterpret_cast<T*>(d.de) + (((long long)n * d.H + y) * d.W + x) * (2LL * d.C);
          float dsc[4], dsh[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) { dsc[j] = du[j] * yh[j]; dsh[j] = du[j]; }
          if (d.de_accumulate) {
            float o1[4], o2[4];
            Vec4<T>::ld(de + c0, o1);
            Vec4<T>::ld(de + d.C + c0, o2);
#pragma unroll
            for (int j = 0; j < 4; ++j) { dsc[j] += o1[j]; dsh[j] += o2[j]; }
          }
          Vec4<T>::st(de + c0, dsc);
          Vec4<T>::st(de + d.C + c0, dsh);
        }
      }
      const bool owner = fold_same_channel_lanes(A, TPB);
      fold_same_channel_lanes(Bc, TPB);
      if (owner && pl < PL) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          xu_det_add(&sA[c0 + j], A[j]);
          xu_det_add(&sB[c0 + j], Bc[j]);
        }
      }
    }
  }
  __syncthreads();
  const int cpg = d.C / XU_GROUPS;
  double* gacc = d.acc;
  double* bacc = d.acc + 2 * d.C;
  for (int c = tid; c < d.C; c += 256) {
    atomicAdd(&gacc[c], sA[c]);
    atomicAdd(&gacc[d.C + c], sB[c]);
  }
  if (tid < XU_GROUPS) {
    double s1 = 0.0, s2 = 0.0;
    for (int k = 0; k < cpg; ++k) {
      const int c = tid * cpg + k;
      const double gmc = d.gamma[c];
      s1 += gmc * sB[c];
      s2 += gmc * sA[c];
    }
    atomicAdd(&bacc[(b * XU_GROUPS + tid) * 2 + 0], s1);
    atomicAdd(&bacc[(b * XU_GROUPS + tid) * 2 + 1], s2);
  }
}

void launch_gn_bwd_reduce(int dtype, const GnArgs& a, cudaStream_t s) {
  GnDev d = gn_dev(a);
  const int B = a.N / 2, P = 2 * a.H * a.W;
  if (!a.skip_zero) cudaMemsetAsync(a.bstats, 0, sizeof(float) * B * XU_GROUPS * 2, s);
  dim3 grid; int ppb;
  gn_grid(a.C, P, B, grid, ppb);
  size_t smem = sizeof(double) * 2 * a.C;
  d.acc = xu_det_scratch(s, 2LL * a.C + (long long)B * XU_GROUPS * 2);
  if (d.acc == nullptr) return;
  if (dtype == XU_F32) xu_launch(gn_bwd_reduce_kernel<float>, grid, 256, smem, s, d, ppb);
  else xu_launch(gn_bwd_reduce_kernel<bf16>, grid, 256, smem, s, d, ppb);
  xu_det_fold(a.dgamma, d.acc, a.C, s);
  xu_det_fold(a.dbeta, d.acc + a.C, a.C, s);
  xu_det_fold(a.bstats, d.acc + 2 * a.C, (long long)B * XU_GROUPS * 2, s);
}

// pass B: dx = rstd * (gamma*dyh - S1/cnt - xhat*S2/cnt); same thread <-> channel-vector mapping as gn_apply_kernel
template <typename T>
__global__ void __launch_bounds__(256) gn_bwd_apply_kernel(GnDev d, int ppb) {
  xu_grid_dep_sync();
  const int tid = threadIdx.x, b = blockIdx.y;
  const int C4 = d.C >> 2;
  const int TPB = C4 < 256 ? C4 : 256;
  const int PL = 256 / TPB;
  const int cv0 = tid % TPB, pl = tid / TPB;
  if (pl >= PL) return;
  const int HW = d.H * d.W, P = 2 * HW;
  const int pbeg = blockIdx.x * ppb;
  const int pend = min(pbeg + ppb, P);
    const unsigned long long seed = (d.mode == GN_FILM && d.train && d.drop_rate > 0.f) ? *d.seed_dev : 0ULL;
  for (int cv = cv0; cv < C4; cv += TPB) {
    const int c0 = cv * 4;
    float mean[4], rstd[4], gm[4], bt[4], s1[4], s2[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      gn_mean_rstd(d, b, c0 + j, mean[j], rstd[j]);
      gm[j] = d.gamma[c0 + j];
      bt[j] = d.beta[c0 + j];
      const int g = gn_group(d, c0 + j);
      s1[j] = d.bstats[(b * XU_GROUPS + g) * 2 + 0] * d.inv_cnt;
      s2[j] = d.bstats[(b * XU_GROUPS + g) * 2 + 1] * d.inv_cnt;
    }
    if (d.rs == RS_NONE) {
      constexpr int U = 4;
      const bool film = d.mode == GN_FILM;
      const bool drop = film && d.train && d.drop_rate > 0.f;
      const float keep_scale = 1.f / (1.f - d.drop_rate);
      const long long pix0 = (long long)(2 * b) * HW;
      const T* X = reinterpret_cast<const T*>(d.x) + pix0 * d.C + c0;
      const T* G = reinterpret_cast<const T*>(d.dy) + pix0 * d.C + c0;
      const T* E = film ? reinterpret_cast<const T*>(d.e) + pix0 * (2LL * d.C) + c0 : nullptr;
      T* DX = reinterpret_cast<T*>(d.y) + pix0 * d.C + c0;
      for (int p0 = pbeg + pl; p0 < pend; p0 += U * PL) {
        typename Vec4<T>::raw xr[U], gr[U], scr[U], shr[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int p = p0 + u * PL;
          if (p < pend) {
            xr[u] = Vec4<T>::ldg_raw(X + (long long)p * d.C);
            gr[u] = Vec4<T>::ldg_raw(G + (long long)p * d.C);
            if (film) {
              scr[u] = Vec4<T>::ldg_raw(E + (long long)p * (2 * d.C));
              shr[u] = Vec4<T>::ldg_raw(E + (long long)p * (2 * d.C) + d.C);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int p = p0 + u * PL;
          if (p >= pend) break;
          float v[4], g[4], sc[4] = {0.f, 0.f, 0.f, 0.f}, sh[4] = {0.f, 0.f, 0.f, 0.f}, xh[4], yh[4], dyh[4], du[4], out[4];
          Vec4<T>::unpack(xr[u], v);
          Vec4<T>::unpack(gr[u], g);
          if (film) { Vec4<T>::unpack(scr[u], sc); Vec4<T>::unpack(shr[u], sh); }
#pragma unroll
          for (int j = 0; j < 4; ++j) { xh[j] = (v[j] - mean[j]) * rstd[j]; yh[j] = fmaf(xh[j], gm[j], bt[j]); }
          const uint32_t km = drop ? xu_keep4(seed, d.op_index, (unsigned long long)((pix0 + p) * d.C + c0) >> 2, d.drop_rate) : 0xFu;
          gn_dyhat_compute(d.mode, g, yh, sc, sh, km, drop, keep_scale, dyh, du);
#pragma unroll
          for (int j = 0; j < 4; ++j) out[j] = rstd[j] * (gm[j] * dyh[j] - s1[j] - xh[j] * s2[j]);
          if (d.extra != nullptr) {   // fused residual-branch gradient (replaces a separate axpy pass over dx)
            float ex[4];
            Vec4<T>::ldg(reinterpret_cast<const T*>(d.extra) + pix0 * d.C + c0 + (long long)p * d.C, ex);
#pragma unroll
            for (int j = 0; j < 4; ++j) out[j] = fmaf(d.extra_alpha, ex[j], out[j]);
          }
          T* dx = DX + (long long)p * d.C;
          if (d.accumulate) {
            float o[4];
            Vec4<T>::ld(dx, o);
#pragma unroll
            for (int j = 0; j < 4; ++j) out[j] += o[j];
          }
          Vec4<T>::st(dx, out);
        }
      }
    } else
#pragma unroll 2
    for (int p = pbeg + pl; p < pend; p += PL) {
      int n = 2 * b, y = 0, x = p;
      if (d.rs != RS_NONE) {
        const int f = p / HW, r = p - f * HW;
        y = r / d.W; x = r - y * d.W; n = b * 2 + f;
      }
      float yh[4], xh[4], dyh[4], du[4], out[4];
      gn_yhat4<T>(d, n, y, x, c0, mean, rstd, gm, bt, yh, xh);
      gn_dyhat4<T>(d, n, y, x, c0, yh, seed, dyh, du);
#pragma unroll
      for (int j = 0; j < 4; ++j) out[j] = rstd[j] * (gm[j] * dyh[j] - s1[j] - xh[j] * s2[j]);
      if (d.extra != nullptr) {
        float ex[4];
        Vec4<T>::ldg(reinterpret_cast<const T*>(d.extra) + ((long long)(2 * b) * HW + p) * d.C + c0, ex);
#pragma unroll
        for (int j = 0; j < 4; ++j) out[j] = fmaf(d.extra_alpha, ex[j], out[j]);
      }
      T* dx = reinterpret_cast<T*>(d.y) + ((long long)(2 * b) * HW + p) * d.C + c0;
      if (d.accumulate) {
        float o[4];
        Vec4<T>::ld(dx, o);
#pragma unroll
        for (int j = 0; j < 4; ++j) out[j] += o[j];
      }
      Vec4<T>::st(dx, out);
    }
  }
}

// Only pass of the GroupNorm backward when the consumer conv's data-gradient epilogue has already stored dyh (in a.dy) and
// accumulated the per-(sample, channel) sums [A = sum dyh*xhat, B = sum dyh] (a.bcs): fold them (dgamma, dbeta, group sums
// S1 = sum_c gamma B, S2 = sum_c gamma A), then dx = rstd * (gamma*dyh - S1/cnt - xhat*S2/cnt) [+ fused residual gradient].
template <typename T>
__global__ void __launch_bounds__(256, 2) gn_bwd_apply_pre_kernel(GnDev d, int ppb) {
  xu_grid_dep_sync();
  constexpr int VW = VecW<T>::W;
  constexpr int U = 4;
  const int tid = threadIdx.x, b = blockIdx.y;
  __shared__ float s_s12[XU_GROUPS][2];
  __shared__ float s_grp[XU_GROUPS][2];
  {
    const int g = tid >> 3, sub = tid & 7;
    float s1 = 0.f, s2 = 0.f;
    for (int k = sub; k < d.cpg; k += 8) {
      const int c = g * d.cpg + k;
      const float2 ab = *reinterpret_cast<const float2*>(d.bcs + ((long long)b * d.C + c) * 2);
      const float gmc = d.gamma[c];
      s1 = fmaf(gmc, ab.y, s1);
      s2 = fmaf(gmc, ab.x, s2);
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if (sub == 0) { s_s12[g][0] = s1 * d.inv_cnt; s_s12[g][1] = s2 * d.inv_cnt; }
    if (tid < XU_GROUPS) {
      s_grp[tid][0] = d.stats[(b * XU_GROUPS + tid) * 2 + 0];
      s_grp[tid][1] = d.stats[(b * XU_GROUPS + tid) * 2 + 1];
    }
    if (blockIdx.x == 0 && b == 0) {     // one block adds the channel sums of every sample, in sample order, to the parameter gradients
      for (int c = tid; c < d.C; c += 256) {
        float ga = 0.f, gb = 0.f;
        for (int bb = 0; bb < d.N / 2; ++bb) {
          const float2 ab = *reinterpret_cast<const float2*>(d.bcs + ((long long)bb * d.C + c) * 2);
          ga += ab.x; gb += ab.y;
        }
        d.dgamma[c] += ga;
        d.dbeta[c] += gb;
      }
    }
    __syncthreads();
  }
  const int CV = d.C / VW;
  const int TPB = CV < 256 ? CV : 256;
  const int PL = 256 / TPB;
  const int cv0 = tid % TPB, pl = tid / TPB;
  if (pl >= PL) return;
  const int HW = d.H * d.W, P = 2 * HW;
  const int pbeg = blockIdx.x * ppb;
  const int pend = min(pbeg + ppb, P);
  const long long pix0 = (long long)(2 * b) * HW;
  for (int cv = cv0; cv < CV; cv += TPB) {
    const int c0 = cv * VW;
    // dx = rstd*(gamma*dyh - S1 - xhat*S2)  with xhat = (x-mean)*rstd   ==   dyh*kg + x*kx + k0
    float kg[VW], kx[VW], k0[VW];
#pragma unroll
    for (int j = 0; j < VW; ++j) {
      float mean, rstd;
      gn_group_mean_rstd(d, s_grp, c0 + j, mean, rstd);
      const int g = gn_group(d, c0 + j);
      const float s1 = s_s12[g][0], s2 = s_s12[g][1];
      kg[j] = rstd * d.gamma[c0 + j];
      kx[j] = -rstd * rstd * s2;
      k0[j] = rstd * (mean * rstd * s2 - s1);
    }
    const T* X = reinterpret_cast<const T*>(d.x) + pix0 * d.C + c0;
    const T* G = reinterpret_cast<const T*>(d.dy) + pix0 * d.C + c0;
    const T* EX = d.extra ? reinterpret_cast<const T*>(d.extra) + pix0 * d.C + c0 : nullptr;
    T* DX = reinterpret_cast<T*>(d.y) + pix0 * d.C + c0;
    for (int p0 = pbeg + pl; p0 < pend; p0 += U * PL) {
      typename VecW<T>::raw xr[U], gr[U], er[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int p = p0 + u * PL;
        if (p < pend) {
          xr[u] = VecW<T>::ldg(X + (long long)p * d.C);
          gr[u] = VecW<T>::ldg(G + (long long)p * d.C);
          if (EX) er[u] = VecW<T>::ldg(EX + (long long)p * d.C);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int p = p0 + u * PL;
        if (p >= pend) break;
        float v[VW], g[VW], out[VW];
        VecW<T>::unpack(xr[u], v);
        VecW<T>::unpack(gr[u], g);
#pragma unroll
        for (int j = 0; j < VW; ++j) out[j] = fmaf(g[j], kg[j], fmaf(v[j], kx[j], k0[j]));
        if (EX) {
          float ex[VW];
          VecW<T>::unpack(er[u], ex);
#pragma unroll
          for (int j = 0; j < VW; ++j) out[j] = fmaf(d.extra_alpha, ex[j], out[j]);
        }
        T* dx = DX + (long long)p * d.C;
        if (d.accumulate) {
          float o[VW];
          VecW<T>::unpack(VecW<T>::ld(dx), o);
#pragma unroll
          for (int j = 0; j < VW; ++j) out[j] += o[j];
        }
        VecW<T>::st(dx, out);
      }
    }
  }
}

void launch_gn_bwd_apply_pre(int dtype, const GnArgs& a, cudaStream_t s) {
  GnDev d = gn_dev(a);
  dim3 grid; int ppb;
  gn_vec_grid(d.C, dtype == XU_F32 ? 4 : 8, 2 * d.H * d.W, d.N / 2, grid, ppb);
  if (dtype == XU_F32) xu_launch(gn_bwd_apply_pre_kernel<float>, grid, 256, 0, s, d, ppb);
  else xu_launch(gn_bwd_apply_pre_kernel<bf16>, grid, 256, 0, s, d, ppb);
}

void launch_gn_bwd_apply(int dtype, const GnArgs& a, cudaStream_t s) {
  GnDev d = gn_dev(a);
  dim3 grid; int ppb;
  gn_apply_grid(d.C, 2 * d.H * d.W, d.N / 2, grid, ppb);
  if (dtype == XU_F32) xu_launch(gn_bwd_apply_kernel<float>, grid, 256, 0, s, d, ppb);
  else xu_launch(gn_bwd_apply_kernel<bf16>, grid, 256, 0, s, d, ppb);
}

// ======================================================================================================
// log-SNR embedding  (model/xunet.py:153-157, posenc_ddpm :23-35)
// ======================================================================================================
// One Dense layer of the log-SNR MLP for one sample and 32 output columns per CTA: lane <-> column (128-byte coalesced weight rows),
// the 8 warps split K and are reduced through shared memory in a fixed order (deterministic).  FIRST: the input vector is the
// DDPM sinusoidal encoding of logsnr[b], built in shared memory (and exported to `pe` for the backward); otherwise swish(h1[b]).
// grid (E/32, B): E = 1024 -> 32*B CTAs instead of the B CTAs x 2E serial FMAs per thread of round 1.
template <bool FIRST>
__global__ void __launch_bounds__(256) logsnr_dense_kernel(const float* __restrict__ logsnr, const float* __restrict__ in,
                                                            const float* __restrict__ w, const float* __restrict__ bias,
                                                            float* __restrict__ pe, float* __restrict__ out, int E) {
  xu_grid_dep_sync();
  extern __shared__ float sm[];  // sv[E] input vector, red[8][32]
  float* sv = sm;
  float* red = sm + E;
  const int b = blockIdx.y;
  const int j0 = blockIdx.x * 32;
  if (FIRST) {
    float l = fminf(fmaxf(logsnr[b], -20.f), 20.f);
    float t = 2.f * atanf(expf(-l * 0.5f)) / 3.14159265358979323846f;
    t *= 1000.f;  // posenc_ddpm(max_time=1.): timesteps *= 1000/max_time
    const int half = E / 2;
    const float c = (float)(-9.210340371976184 / (double)(half - 1));  // -log(10000)/(half-1)
    for (int k = threadIdx.x; k < E; k += blockDim.x) {
      int kk = k < half ? k : k - half;
      float f = expf((float)kk * c);
      float arg = t * f;
      float v = k < half ? sinf(arg) : cosf(arg);
      if (k >= 2 * half) v = 0.f;
      sv[k] = v;
      if (k >= j0 && k < j0 + 32) pe[b * E + k] = v;
    }
  } else {
    for (int k = threadIdx.x; k < E; k += blockDim.x) sv[k] = swishf_(in[b * E + k]);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int j = j0 + lane;
  const int kper = (E + 7) / 8;
  const int k0 = wp * kper, k1 = min(E, k0 + kper);
  float acc = 0.f;
  if (j < E) {
#pragma unroll 8
    for (int k = k0; k < k1; ++k) acc = fmaf(sv[k], w[(size_t)k * E + j], acc);
  }
  red[wp * 32 + lane] = acc;
  __syncthreads();
  if (wp == 0 && j < E) {
    float r = bias[j];
#pragma unroll
    for (int q = 0; q < 8; ++q) r += red[q * 32 + lane];
    out[b * E + j] = r;
  }
}

void launch_logsnr_emb(const float* logsnr, const float* w0, const float* b0, const float* w1, const float* b1, float* pe,
                       float* h1, float* lemb, int B, int E, cudaStream_t s) {
  dim3 grid(cdiv(E, 32), B);
  const size_t smem = (size_t)(E + 256) * sizeof(float);
  xu_launch(logsnr_dense_kernel<true>, grid, 256, smem, s, logsnr, (const float*)nullptr, w0, b0, pe, h1, E);
  xu_launch(logsnr_dense_kernel<false>, grid, 256, smem, s, logsnr, (const float*)h1, w1, b1, pe, lemb, E);
}

// dh1[b,k] = swish'(h1[b,k]) * sum_j w1[k][j] dlemb[b,j]
__global__ void logsnr_bwd_dh1_kernel(const float* __restrict__ dlemb, const float* __restrict__ w1,
                                      const float* __restrict__ h1, float* __restrict__ dh1, int E) {
  xu_grid_dep_sync();
  const int b = blockIdx.y;
  const int k = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (k >= E) return;
  float acc = 0.f;
  for (int j = lane; j < E; j += 32) acc = fmaf(w1[k * E + j], dlemb[b * E + j], acc);
  acc = warp_sum(acc);
  if (lane == 0) dh1[b * E + k] = acc * swish_gradf_(h1[b * E + k]);
}
// dw1[k][j] = sum_b swish(h1[b,k]) dlemb[b,j];  dw0[k][j] = sum_b pe[b,k] dh1[b,j];  biases.  ACC: added to the gradients instead
template <bool ACC>
__global__ void logsnr_bwd_w_kernel(const float* __restrict__ dlemb, const float* __restrict__ pe,
                                    const float* __restrict__ h1, const float* __restrict__ dh1, float* __restrict__ dw0,
                                    float* __restrict__ db0, float* __restrict__ dw1, float* __restrict__ db1, int B,
                                    int E) {
  xu_grid_dep_sync();
  const int k = blockIdx.x;
  for (int j = threadIdx.x; j < E; j += blockDim.x) {
    float a1 = 0.f, a0 = 0.f, s1 = 0.f, s0 = 0.f;
    for (int b = 0; b < B; ++b) {
      const float dl = dlemb[b * E + j], dh = dh1[b * E + j];
      a1 = fmaf(swishf_(h1[b * E + k]), dl, a1);
      a0 = fmaf(pe[b * E + k], dh, a0);
      s1 += dl;
      s0 += dh;
    }
    if (ACC) {
      dw1[k * E + j] += a1;
      dw0[k * E + j] += a0;
      if (k == 0) { db1[j] += s1; db0[j] += s0; }
    } else {
      dw1[k * E + j] = a1;
      dw0[k * E + j] = a0;
      if (k == 0) { db1[j] = s1; db0[j] = s0; }
    }
  }
}

void launch_logsnr_emb_bwd(const float* dlemb, const float* w1, const float* pe, const float* h1, float* dh1, float* dw0,
                           float* db0, float* dw1, float* db1, int B, int E, int accumulate, cudaStream_t s) {
  dim3 g1(cdiv(E, 8), B);
  xu_launch(logsnr_bwd_dh1_kernel, g1, 256, 0, s, dlemb, w1, h1, dh1, E);
  int threads = E < 256 ? ((E + 31) / 32) * 32 : 256;
  if (accumulate) xu_launch(logsnr_bwd_w_kernel<true>, E, threads, 0, s, dlemb, pe, h1, dh1, dw0, db0, dw1, db1, B, E);
  else xu_launch(logsnr_bwd_w_kernel<false>, E, threads, 0, s, dlemb, pe, h1, dh1, dw0, db0, dw1, db1, B, E);
}

// ======================================================================================================
// camera rays + NeRF positional encoding  (model/xunet.py:159-194, posenc_nerf :37-44)
// ======================================================================================================
__global__ void kinv_kernel(const float* __restrict__ K, float* __restrict__ kinv, int B) {
  xu_grid_dep_sync();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double m[9];
  for (int i = 0; i < 9; ++i) m[i] = (double)K[b * 9 + i];
  double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
  double det = m[0] * c00 + m[1] * c01 + m[2] * c02;
  double id = 1.0 / det;
  double inv[9];
  inv[0] = c00 * id; inv[1] = (m[2] * m[7] - m[1] * m[8]) * id; inv[2] = (m[1] * m[5] - m[2] * m[4]) * id;
  inv[3] = c01 * id; inv[4] = (m[0] * m[8] - m[2] * m[6]) * id; inv[5] = (m[2] * m[3] - m[0] * m[5]) * id;
  inv[6] = c02 * id; inv[7] = (m[1] * m[6] - m[0] * m[7]) * id; inv[8] = (m[0] * m[4] - m[1] * m[3]) * id;
  for (int i = 0; i < 9; ++i) kinv[b * 9 + i] = (float)inv[i];
}

// One block = 64 pixels of one frame.  The 93 position channels depend only on the frame (camera centre t), so they are
// evaluated once per block (their arguments reach 2^14 |t|: the slow range-reduction path of sinf) and broadcast; the ray
// direction of each pixel is formed once and shared by its 51 direction channels.
constexpr int kPosePix = 64;
__device__ __forceinline__ float pose_channel(int jj, int nd, const float (&v)[3]) {
  // posenc_nerf layout: [x (3) | sin(2^k x) k<nd (3 nd) | sin(2^k x + pi/2) (3 nd)]
  if (jj < 3) return v[jj];
  int k = jj - 3;
  const int phase = k >= 3 * nd;
  if (phase) k -= 3 * nd;
  const int sc = k / 3, d = k - sc * 3;
  float xb = v[d] * (float)(1 << sc);              // exact in fp32
  if (phase) xb = xb + 1.57079632679489661923f;    // fp32 add of pi/2, then accurate sin (not cos)
  return sinf(xb);
}

template <typename T>
__global__ void __launch_bounds__(256) pose_emb_kernel(const float* __restrict__ R1, const float* __restrict__ t1,
                                                       const float* __restrict__ R2, const float* __restrict__ t2,
                                                       const float* __restrict__ kinv, const float* __restrict__ cond_mask,
                                                       const float* __restrict__ pos_emb, const float* __restrict__ ref_first,
                                                       const float* __restrict__ ref_other, T* __restrict__ out, int B, int S,
                                                       int convention, const float* __restrict__ rays) {
  xu_grid_dep_sync();
  __shared__ float s_pos[93];
  __shared__ float s_dir[kPosePix][3];
  __shared__ float s_ppos[kPosePix][3];   // explicit-rays entry only: per-pixel ray origin
  const int tid = threadIdx.x;
  const int n = blockIdx.y, b = n >> 1, f = n & 1;
  const int HW = S * S;
  const int pix0 = blockIdx.x * kPosePix;
  const bool on = cond_mask[b] != 0.f;
  if (on && rays != nullptr) {
    // caller-supplied rays (B, 2, S, S, 6): v3d.Camera.rays() output fed straight in (model/xunet.py:159-161)
    if (tid < kPosePix && pix0 + tid < HW) {
      const float* r = rays + ((long long)n * HW + pix0 + tid) * 6;
      s_ppos[tid][0] = r[0]; s_ppos[tid][1] = r[1]; s_ppos[tid][2] = r[2];
      s_dir[tid][0] = r[3]; s_dir[tid][1] = r[4]; s_dir[tid][2] = r[5];
    }
  } else if (on) {
    const float* R = (f == 0 ? R1 : R2) + b * 9;
    const float* t = (f == 0 ? t1 : t2) + b * 3;
    if (tid < 93) {
      const float tv[3] = {t[0], t[1], t[2]};
      s_pos[tid] = pose_channel(tid, 15, tv);
    } else if (tid >= 128 && tid < 128 + kPosePix && pix0 + tid - 128 < HW) {
      const int pix = pix0 + tid - 128;
      const int row = pix / S, col = pix - row * S;
      float d[3];
      xu_ray_dir(kinv + b * 9, R, row, col, convention, d);
      s_dir[tid - 128][0] = d[0]; s_dir[tid - 128][1] = d[1]; s_dir[tid - 128][2] = d[2];
    }
  }
  __syncthreads();
  const int npix = min(kPosePix, HW - pix0);
  T* o = out + ((long long)n * HW + pix0) * XU_POSE_DIM;
  const float* pe = pos_emb ? pos_emb + (long long)pix0 * XU_POSE_DIM : nullptr;
  const float* rf = ref_first ? (f == 0 ? ref_first : ref_other) : nullptr;
  for (int i = tid; i < npix * XU_POSE_DIM; i += 256) {
    const int pl = i / XU_POSE_DIM, j = i - pl * XU_POSE_DIM;
    float val = 0.f;
    if (on) {
      if (j < 93) {
        if (rays != nullptr) {
          const float pv[3] = {s_ppos[pl][0], s_ppos[pl][1], s_ppos[pl][2]};
          val = pose_channel(j, 15, pv);
        } else val = s_pos[j];
      } else {
        const float dv[3] = {s_dir[pl][0], s_dir[pl][1], s_dir[pl][2]};
        val = pose_channel(j - 93, 8, dv);
      }
    }
    if (pe) val += pe[i];
    if (rf) val += rf[j];
    stf(o + i, val);
  }
}

void launch_pose_emb(int dtype, const float* R1, const float* t1, const float* R2, const float* t2, const float* K,
                     const float* cond_mask, const float* pos_emb, const float* ref_first, const float* ref_other,
                     float* kinv_scratch, void* out, int B, int S, int convention, const float* rays, cudaStream_t s) {
  if (rays == nullptr) xu_launch(kinv_kernel, cdiv(B, 64), 64, 0, s, K, kinv_scratch, B);
  const dim3 grid(cdiv(S * S, kPosePix), 2 * B);
  if (dtype == XU_F32)
    xu_launch(pose_emb_kernel<float>, grid, 256, 0, s, R1, t1, R2, t2, kinv_scratch, cond_mask, pos_emb, ref_first,
                                                           ref_other, (float*)out, B, S, convention, rays);
  else
    xu_launch(pose_emb_kernel<bf16>, grid, 256, 0, s, R1, t1, R2, t2, kinv_scratch, cond_mask, pos_emb, ref_first,
                                                          ref_other, (bf16*)out, B, S, convention, rays);
}

// ACC: dpos_emb is added to instead of stored (the ref_pose_emb leaves are folded, which always adds)
template <typename T, bool ACC>
__global__ void pose_emb_bwd_kernel(const T* __restrict__ dpose, float* __restrict__ dpos_emb,
                                    double* __restrict__ dref_first, double* __restrict__ dref_other, int B, int S) {
  xu_grid_dep_sync();
  const long long per = (long long)S * S * XU_POSE_DIM;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= per) return;
  const int j = (int)(idx % XU_POSE_DIM);
  float s0 = 0.f, s1 = 0.f;
  for (int b = 0; b < B; ++b) {
    s0 += ldf(dpose + (long long)(2 * b) * per + idx);
    s1 += ldf(dpose + (long long)(2 * b + 1) * per + idx);
  }
  if (dpos_emb != nullptr) {
    if (ACC) dpos_emb[idx] += s0 + s1;
    else dpos_emb[idx] = s0 + s1;
  }
  if (dref_first != nullptr) { xu_det_add(&dref_first[j], s0); xu_det_add(&dref_other[j], s1); }
}

void launch_pose_emb_bwd(int dtype, const void* dpose, float* dpos_emb, float* dref_first, float* dref_other, int B, int S,
                         int accumulate, cudaStream_t s) {
  const long long per = (long long)S * S * XU_POSE_DIM;
  double* acc = nullptr;
  if (dref_first != nullptr && (acc = xu_det_scratch(s, 2 * XU_POSE_DIM)) == nullptr) return;
  double* acc2 = acc ? acc + XU_POSE_DIM : nullptr;
  const int nb = cdiv(per, 256);
  if (dtype == XU_F32) {
    if (accumulate) xu_launch(pose_emb_bwd_kernel<float, true>, nb, 256, 0, s, (const float*)dpose, dpos_emb, acc, acc2, B, S);
    else xu_launch(pose_emb_bwd_kernel<float, false>, nb, 256, 0, s, (const float*)dpose, dpos_emb, acc, acc2, B, S);
  } else {
    if (accumulate) xu_launch(pose_emb_bwd_kernel<bf16, true>, nb, 256, 0, s, (const bf16*)dpose, dpos_emb, acc, acc2, B, S);
    else xu_launch(pose_emb_bwd_kernel<bf16, false>, nb, 256, 0, s, (const bf16*)dpose, dpos_emb, acc, acc2, B, S);
  }
  if (acc != nullptr) {
    xu_det_fold(dref_first, acc, XU_POSE_DIM, s);
    xu_det_fold(dref_other, acc2, XU_POSE_DIM, s);
  }
}

// ======================================================================================================
// emb = swish(logsnr_emb[b] + pose_emb_level)   (FiLM's nonlinearity(emb), model/xunet.py:59,233)
// ======================================================================================================
template <typename T>
__global__ void __launch_bounds__(256) emb_fwd_kernel(const float* __restrict__ lemb, const T* __restrict__ pe,
                                                      T* __restrict__ semb, int N, int HW, int E) {
  xu_grid_dep_sync();
  const int E4 = E >> 2;
  const long long total = (long long)N * HW * E4;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= total) return;
  const int cv = (int)(idx % E4);
  const long long pix = idx / E4;
  const int b = (int)(pix / HW) >> 1;
  float v[4];
  Vec4<T>::ld(pe + pix * E + cv * 4, v);
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = swishf_(v[j] + lemb[b * E + cv * 4 + j]);
  Vec4<T>::st(semb + pix * E + cv * 4, v);
}

void launch_emb_fwd(int dtype, const float* lemb, const void* pe, void* semb, int N, int HW, int E, cudaStream_t s) {
  const long long total = (long long)N * HW * (E / 4);
  if (dtype == XU_F32) xu_launch(emb_fwd_kernel<float>, cdiv(total, 256), 256, 0, s, lemb, (const float*)pe, (float*)semb, N, HW, E);
  else xu_launch(emb_fwd_kernel<bf16>, cdiv(total, 256), 256, 0, s, lemb, (const bf16*)pe, (bf16*)semb, N, HW, E);
}

// grid (chunks, B): dz = dsemb * swish'(lemb+pe); dpe = dz (optional); dlemb[b,c] += sum over this block's pixels
template <typename T>
__global__ void __launch_bounds__(256) emb_bwd_kernel(const float* __restrict__ lemb, const T* __restrict__ pe,
                                                      const T* __restrict__ dsemb, T* __restrict__ dpe,
                                                      double* __restrict__ dlemb, int P, int E, int ppb, int write_dpe) {
  xu_grid_dep_sync();
  extern __shared__ double saccd[];  // E
  const int tid = threadIdx.x, b = blockIdx.y;
  for (int i = tid; i < E; i += 256) saccd[i] = 0.0;
  __syncthreads();
  const int E4 = E >> 2;
  const int TPB = E4 < 256 ? E4 : 256;
  const int PL = 256 / TPB;
  const int cv0 = tid % TPB, pl = tid / TPB;
  const int pbeg = blockIdx.x * ppb, pend = min(pbeg + ppb, P);
  {
    for (int cv = cv0; cv < E4; cv += TPB) {
      float le[4], acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int j = 0; j < 4; ++j) le[j] = lemb[b * E + cv * 4 + j];
      if (pl < PL)
      for (int p = pbeg + pl; p < pend; p += PL) {
        const long long off = ((long long)b * P + p) * E + cv * 4;
        float v[4], g[4];
        Vec4<T>::ld(pe + off, v);
        Vec4<T>::ld(dsemb + off, g);
#pragma unroll
        for (int j = 0; j < 4; ++j) { g[j] *= swish_gradf_(v[j] + le[j]); acc[j] += g[j]; }
        if (write_dpe) Vec4<T>::st(dpe + off, g);
      }
      if (fold_same_channel_lanes(acc, TPB) && pl < PL) {
#pragma unroll
        for (int j = 0; j < 4; ++j) xu_det_add(&saccd[cv * 4 + j], acc[j]);
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < E; i += 256) atomicAdd(&dlemb[b * E + i], saccd[i]);
}

void launch_emb_bwd(int dtype, const float* lemb, const void* pe, const void* dsemb, void* dpe, float* dlemb, int N, int HW,
                    int E, int write_dpe, cudaStream_t s) {
  const int B = N / 2, P = 2 * HW;
  dim3 grid; int ppb;
  gn_grid(E, P, B, grid, ppb);
  size_t smem = sizeof(double) * E;
  double* acc = xu_det_scratch(s, (long long)B * E);
  if (acc == nullptr) return;
  if (dtype == XU_F32)
    xu_launch(emb_bwd_kernel<float>, grid, 256, smem, s, lemb, (const float*)pe, (const float*)dsemb, (float*)dpe, acc, P, E, ppb, write_dpe);
  else
    xu_launch(emb_bwd_kernel<bf16>, grid, 256, smem, s, lemb, (const bf16*)pe, (const bf16*)dsemb, (bf16*)dpe, acc, P, E, ppb, write_dpe);
  xu_det_fold(dlemb, acc, (long long)B * E, s);
}

// ======================================================================================================
// plumbing
// ======================================================================================================
template <typename T>
__global__ void pack_input_kernel(const float* __restrict__ x, const float* __restrict__ z, T* __restrict__ out, int B,
                                  long long per) {
  xu_grid_dep_sync();
  const long long total = (long long)B * 2 * per;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= total) return;
  const long long n = idx / per, r = idx - n * per;
  const long long b = n >> 1;
  stf(out + idx, (n & 1) ? z[b * per + r] : x[b * per + r]);
}
void launch_pack_input(int dtype, const float* x, const float* z, void* out, int B, int S, cudaStream_t s) {
  const long long per = (long long)S * S * 3, total = 2 * B * per;
  if (dtype == XU_F32) xu_launch(pack_input_kernel<float>, cdiv(total, 256), 256, 0, s, x, z, (float*)out, B, per);
  else xu_launch(pack_input_kernel<bf16>, cdiv(total, 256), 256, 0, s, x, z, (bf16*)out, B, per);
}

template <typename T>
__global__ void __launch_bounds__(256) resample_kernel(const T* __restrict__ x, T* __restrict__ y, int N, int Hi, int Wi,
                                                       int C, int pool, float scale, int accumulate) {
  xu_grid_dep_sync();
  const int Ho = pool ? Hi / 2 : Hi * 2, Wo = pool ? Wi / 2 : Wi * 2;
  const int C4 = C >> 2;
  const long long total = (long long)N * Ho * Wo * C4;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= total) return;
  const int cv = (int)(idx % C4);
  const long long pix = idx / C4;
  const int ox = (int)(pix % Wo);
  const int oy = (int)((pix / Wo) % Ho);
  const int n = (int)(pix / ((long long)Wo * Ho));
  float out[4] = {0.f, 0.f, 0.f, 0.f};
  if (pool) {
    for (int i = 0; i < 2; ++i)
      for (int k = 0; k < 2; ++k) {
        float v[4];
        Vec4<T>::ld(x + (((long long)n * Hi + 2 * oy + i) * Wi + 2 * ox + k) * C + cv * 4, v);
#pragma unroll
        for (int j = 0; j < 4; ++j) out[j] += v[j];
      }
  } else {
    Vec4<T>::ld(x + (((long long)n * Hi + (oy >> 1)) * Wi + (ox >> 1)) * C + cv * 4, out);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) out[j] *= scale;
  T* dst = y + pix * C + cv * 4;
  if (accumulate) {
    float o[4];
    Vec4<T>::ld(dst, o);
#pragma unroll
    for (int j = 0; j < 4; ++j) out[j] += o[j];
  }
  Vec4<T>::st(dst, out);
}
void launch_resample(int dtype, const void* x, void* y, int N, int Hi, int Wi, int C, int pool, float scale, int accumulate,
                     cudaStream_t s) {
  const int Ho = pool ? Hi / 2 : Hi * 2, Wo = pool ? Wi / 2 : Wi * 2;
  const long long total = (long long)N * Ho * Wo * (C / 4);
  if (dtype == XU_F32) xu_launch(resample_kernel<float>, cdiv(total, 256), 256, 0, s, (const float*)x, (float*)y, N, Hi, Wi, C, pool, scale, accumulate);
  else xu_launch(resample_kernel<bf16>, cdiv(total, 256), 256, 0, s, (const bf16*)x, (bf16*)y, N, Hi, Wi, C, pool, scale, accumulate);
}

template <typename T>
__global__ void __launch_bounds__(256) copy_channels_kernel(const T* __restrict__ src, T* __restrict__ dst, long long npix,
                                                            int Cs, int Cd, int so, int doff, int Cc, int accumulate) {
  xu_grid_dep_sync();
  const int C4 = Cc >> 2;
  const long long total = npix * C4;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= total) return;
  const int cv = (int)(idx % C4);
  const long long pix = idx / C4;
  float v[4];
  Vec4<T>::ld(src + pix * Cs + so + cv * 4, v);
  T* d = dst + pix * Cd + doff + cv * 4;
  if (accumulate) {
    float o[4];
    Vec4<T>::ld(d, o);
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] += o[j];
  }
  Vec4<T>::st(d, v);
}
void launch_copy_channels(int dtype, const void* src, void* dst, long long npix, int Cs, int Cd, int src_off, int dst_off,
                          int Cc, int accumulate, cudaStream_t s) {
  const long long total = npix * (Cc / 4);
  if (dtype == XU_F32)
    xu_launch(copy_channels_kernel<float>, cdiv(total, 256), 256, 0, s, (const float*)src, (float*)dst, npix, Cs, Cd, src_off, dst_off, Cc, accumulate);
  else
    xu_launch(copy_channels_kernel<bf16>, cdiv(total, 256), 256, 0, s, (const bf16*)src, (bf16*)dst, npix, Cs, Cd, src_off, dst_off, Cc, accumulate);
}

template <typename T>
__global__ void __launch_bounds__(256) scale_add_kernel(const T* __restrict__ src, T* __restrict__ dst, long long n4,
                                                        float alpha, int accumulate) {
  xu_grid_dep_sync();
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= n4) return;
  float v[4];
  Vec4<T>::ld(src + idx * 4, v);
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] *= alpha;
  if (accumulate) {
    float o[4];
    Vec4<T>::ld(dst + idx * 4, o);
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] += o[j];
  }
  Vec4<T>::st(dst + idx * 4, v);
}
void launch_scale_add(int dtype, const void* src, void* dst, long long n, float alpha, int accumulate, cudaStream_t s) {
  const long long n4 = n / 4;  // all activation tensors here have C % 4 == 0
  if (dtype == XU_F32) xu_launch(scale_add_kernel<float>, cdiv(n4, 256), 256, 0, s, (const float*)src, (float*)dst, n4, alpha, accumulate);
  else xu_launch(scale_add_kernel<bf16>, cdiv(n4, 256), 256, 0, s, (const bf16*)src, (bf16*)dst, n4, alpha, accumulate);
}

template <typename T>
__global__ void extract_frame1_kernel(const T* __restrict__ o, float* __restrict__ eps, int B, long long per) {
  xu_grid_dep_sync();
  const long long total = (long long)B * per;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= total) return;
  const long long b = idx / per, r = idx - b * per;
  eps[idx] = ldf(o + (2 * b + 1) * per + r);
}
void launch_extract_frame1(int dtype, const void* o, float* eps, int B, int S, cudaStream_t s) {
  const long long per = (long long)S * S * 3, total = B * per;
  if (dtype == XU_F32) xu_launch(extract_frame1_kernel<float>, cdiv(total, 256), 256, 0, s, (const float*)o, eps, B, per);
  else xu_launch(extract_frame1_kernel<bf16>, cdiv(total, 256), 256, 0, s, (const bf16*)o, eps, B, per);
}

// loss = ||eps - noise||_F  (train.py:67)
__global__ void __launch_bounds__(256) loss_sumsq_kernel(const float* __restrict__ eps, const float* __restrict__ noise,
                                                         long long n, double* __restrict__ sumsq) {
  xu_grid_dep_sync();
  __shared__ float sw[8];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    float r = eps[i] - noise[i];
    acc = fmaf(r, r, acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 8) {
    float v = sw[threadIdx.x];
    for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0xffu, v, o);
    if (threadIdx.x == 0) xu_det_add(sumsq, v);
  }
}
template <typename T>
__global__ void loss_grad_kernel(const float* __restrict__ eps, const float* __restrict__ noise,
                                 const float* __restrict__ sumsq, float* __restrict__ loss_out, T* __restrict__ dO, int B,
                                 long long per) {
  xu_grid_dep_sync();
  const long long total = (long long)B * 2 * per;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  const float loss = sqrtf(*sumsq);
  if (idx == 0) *loss_out = loss;
  if (idx >= total) return;
  const long long n = idx / per, r = idx - n * per;
  float g = 0.f;
  if (n & 1) {
    const long long i = (n >> 1) * per + r;
    g = loss > 0.f ? (eps[i] - noise[i]) / loss : 0.f;
  }
  stf(dO + idx, g);
}
void launch_loss(int dtype, const float* eps, const float* noise, float* sumsq_scratch, float* loss_out, void* dO, int B,
                 int S, cudaStream_t s) {
  const long long per = (long long)S * S * 3, n = B * per;
  cudaMemsetAsync(sumsq_scratch, 0, sizeof(float), s);
  int blocks = cdiv(n, 256 * 4);
  if (blocks > 592) blocks = 592;
  double* acc = xu_det_scratch(s, 1);
  if (acc == nullptr) return;
  xu_launch(loss_sumsq_kernel, blocks, 256, 0, s, eps, noise, n, acc);
  xu_det_fold(sumsq_scratch, acc, 1, s);
  const long long total = 2 * n;
  if (dtype == XU_F32) xu_launch(loss_grad_kernel<float>, cdiv(total, 256), 256, 0, s, eps, noise, sumsq_scratch, loss_out, (float*)dO, B, per);
  else xu_launch(loss_grad_kernel<bf16>, cdiv(total, 256), 256, 0, s, eps, noise, sumsq_scratch, loss_out, (bf16*)dO, B, per);
}

// the caller's dL/d(eps_hat) as the output gradient (xunet_backward_vjp), in the layout loss_grad_kernel writes:
// dO frame 1 = round_T(d_eps[b]), dO frame 0 = 0
template <typename T>
__global__ void vjp_seed_kernel(const float* __restrict__ d_eps, T* __restrict__ dO, int B, long long per) {
  xu_grid_dep_sync();
  const long long total = (long long)B * 2 * per;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= total) return;
  const long long n = idx / per, r = idx - n * per;
  stf(dO + idx, (n & 1) ? d_eps[(n >> 1) * per + r] : 0.f);
}
void launch_vjp_seed(int dtype, const float* d_eps, void* dO, int B, int S, cudaStream_t s) {
  const long long per = (long long)S * S * 3, total = 2 * B * per;
  if (dtype == XU_F32) xu_launch(vjp_seed_kernel<float>, cdiv(total, 256), 256, 0, s, d_eps, (float*)dO, B, per);
  else xu_launch(vjp_seed_kernel<bf16>, cdiv(total, 256), 256, 0, s, d_eps, (bf16*)dO, B, per);
}

__device__ __forceinline__ double block_sum_fixed(double x, double* red);

// loss = (1/B) sum_b w_b (1/P) sum_i r_bi^2, r = eps - noise (P = S*S*3 per sample; w == nullptr: all 1).  The gradient does
// not depend on the loss, so one pass writes the output gradient and the per-sample sums of squares:
//   dO frame 1 = round_T(fl(c_b * fl(eps - noise))), c_b = fl32(2 w_b / (B P)) formed in double;  dO frame 0 = 0.
// CTA (j, b) sums elements j, j + parts*256, ... of sample b in fp64 and stores its partial: the grid depends on (B, P) only
// and nothing is added atomically, so the loss has the same bits on every run by construction.
template <typename T>
__global__ void __launch_bounds__(256) mse_grad_sumsq_kernel(const float* __restrict__ eps, const float* __restrict__ noise,
                                                             const float* __restrict__ w, T* __restrict__ dO, int B,
                                                             long long per, double* __restrict__ partials) {
  xu_grid_dep_sync();
  __shared__ double red[8];
  const int b = blockIdx.y, parts = gridDim.x;
  const float c = (float)(2.0 * (w != nullptr ? (double)w[b] : 1.0) / ((double)B * (double)per));
  const float* e = eps + (long long)b * per;
  const float* nz = noise + (long long)b * per;
  T* d0 = dO + 2LL * b * per;
  T* d1 = d0 + per;
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < per; i += (long long)parts * 256) {
    const float r = __fsub_rn(e[i], nz[i]);
    acc = fma((double)r, (double)r, acc);
    stf(d1 + i, __fmul_rn(c, r));
    stf(d0 + i, 0.f);
  }
  const double t = block_sum_fixed(acc, red);
  if (threadIdx.x == 0) partials[(long long)b * parts + blockIdx.x] = t;
}
// *loss_out = fl32( sum_b w_b * S_b / (B P) ), S_b the partials of sample b summed in a fixed order, everything in fp64.
// The partials are re-zeroed (the reduction scratch is handed back all-zero, kernels.h).
__global__ void __launch_bounds__(256) mse_loss_final_kernel(double* __restrict__ partials, int parts,
                                                             const float* __restrict__ w, int B, long long per,
                                                             float* __restrict__ loss_out) {
  xu_grid_dep_sync();
  __shared__ double red[8];
  double total = 0.0;   // valid in thread 0
  for (int b = 0; b < B; ++b) {
    double acc = 0.0;
    for (int i = threadIdx.x; i < parts; i += 256) {
      acc += partials[(long long)b * parts + i];
      partials[(long long)b * parts + i] = 0.0;
    }
    const double sb = block_sum_fixed(acc, red);
    if (threadIdx.x == 0) total += (w != nullptr ? (double)w[b] : 1.0) * sb;
    __syncthreads();   // red is rewritten by the next sample
  }
  if (threadIdx.x == 0) *loss_out = (float)(total / ((double)B * (double)per));
}
void launch_loss_mse(int dtype, const float* eps, const float* noise, const float* weight, float* loss_out, void* dO, int B,
                     int S, cudaStream_t s) {
  const long long per = (long long)S * S * 3;
  const int parts = cdiv(per, 256 * 4);
  double* partials = xu_det_scratch(s, (long long)B * parts);
  if (partials == nullptr) return;
  const dim3 grid(parts, B);
  if (dtype == XU_F32) xu_launch(mse_grad_sumsq_kernel<float>, grid, 256, 0, s, eps, noise, weight, (float*)dO, B, per, partials);
  else xu_launch(mse_grad_sumsq_kernel<bf16>, grid, 256, 0, s, eps, noise, weight, (bf16*)dO, B, per, partials);
  xu_launch(mse_loss_final_kernel, 1, 256, 0, s, partials, parts, weight, B, per, loss_out);
}

// optax.adam (train.py:45, 74-76).  (1-b1), (1-b2) and the bias corrections are formed in double (optax forms them
// from python floats) and only then rounded to fp32.
// AVG == 1 also folds the weight EMA into the same pass: ema = d*ema + (1-d)*p_new with p_new still in registers (8 more
// bytes per parameter instead of 12 for a separate pass).  The _rn intrinsics forbid FMA contraction, so a float32 numpy
// restatement matches bit for bit.
// AVG == 2 keeps two power-function averages instead (EDM2's post-hoc EMA): with the Adam count t, thread 0 forms
// beta_k = (1 - 1/t)^(gamma_k + 1) and 1 - beta_k in double and rounds each to fp32 once; ema_k = beta_k*ema_k +
// (1-beta_k)*p_new, rounded like the EMA.  beta_1 = 0, so the first update overwrites both averages with p_new.
// CLIP = true adds a linear learning-rate warm-up and clipping by a global norm read from the device.  Thread 0 of each CTA
// also forms lr_t = lr * min(step - 1, W) / W in double rounded once (optax.linear_schedule(0, lr, W) evaluated at the
// schedule's count, which lags Adam's by one), and the clip decision of optax.clip_by_global_norm: g' = g if norm < max_norm,
// else fl(fl(g / norm) * max_norm).  A non-finite norm skips the step: every CTA returns before touching p / m / v / ema and
// CTA 0 counts it in *skipped.  norm == nullptr: no clipping and no guard.  With g' == g and lr_t == lr both instantiations
// give the same bits; CLIP is a template parameter so that plain Adam keeps its 40 registers (6 CTAs per SM, 46 with CLIP).
template <int AVG, bool CLIP>
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, float* __restrict__ ema, long long n, long long step,
                                                   const long long* __restrict__ step_dev, double lr, double b1d, double b2d,
                                                   float eps, float gs, double decay, const float* __restrict__ norm_dev,
                                                   float max_norm, long long warmup, long long* __restrict__ skipped,
                                                   float* __restrict__ ema_b, double gamma_a, double gamma_b) {
  xu_grid_dep_sync();
  constexpr int NSC = CLIP ? 4 : 2;   // sc[NSC..NSC+3]: beta_a, 1-beta_a, beta_b, 1-beta_b of the power averages
  __shared__ float sc[NSC + (AVG == 2 ? 4 : 0)];
  __shared__ int mode;   // CLIP: 0 plain gradient, 1 clipped, 2 skip the step
  if (threadIdx.x == 0) {
    const long long st = step_dev != nullptr ? *step_dev : step;
    sc[0] = (float)(1.0 / (1.0 - pow(b1d, (double)st)));
    sc[1] = (float)(1.0 / (1.0 - pow(b2d, (double)st)));
    if constexpr (CLIP) {
      const long long c = st - 1;
      sc[2] = warmup > 0 ? (float)(lr * (double)(c < warmup ? c : warmup) / (double)warmup) : (float)lr;
      int md = 0;
      sc[3] = 1.f;
      if (norm_dev != nullptr) {
        const float nrm = *norm_dev;
        sc[3] = nrm;
        md = !isfinite(nrm) ? 2 : (nrm < max_norm ? 0 : 1);
        if (md == 2 && blockIdx.x == 0) *skipped += 1;
      }
      mode = md;
    }
    if constexpr (AVG == 2) {
      const double keep = 1.0 - 1.0 / (double)st;
      const double ba = pow(keep, gamma_a + 1.0), bb = pow(keep, gamma_b + 1.0);
      sc[NSC] = (float)ba;
      sc[NSC + 1] = (float)(1.0 - ba);
      sc[NSC + 2] = (float)bb;
      sc[NSC + 3] = (float)(1.0 - bb);
    }
  }
  __syncthreads();
  int md = 0;
  if constexpr (CLIP) {
    md = mode;
    if (md == 2) return;
  }
  const float c1 = sc[0], c2 = sc[1];
  const float b1 = (float)b1d, b2 = (float)b2d, omb1 = (float)(1.0 - b1d), omb2 = (float)(1.0 - b2d);
  float lrf = (float)lr, nrm = 1.f;
  if constexpr (CLIP) {
    lrf = sc[2];
    nrm = sc[3];
  }
  float d = (float)decay, omd = (float)(1.0 - decay), db = 0.f, omdb = 0.f;
  if constexpr (AVG == 2) {
    d = sc[NSC];
    omd = sc[NSC + 1];
    db = sc[NSC + 2];
    omdb = sc[NSC + 3];
  }
  // 16-byte accesses (7 streams of n floats: 4 read, 3 written; 9 with the EMA: 5 read, 4 written; 11 with the two power
  // averages: 6 read, 5 written -- the kernel is pure HBM traffic); scalar path for a ragged tail or unaligned sub-ranges
  uintptr_t addr_or = reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                      reinterpret_cast<uintptr_t>(v);
  if (AVG >= 1) addr_or |= reinterpret_cast<uintptr_t>(ema);
  if (AVG == 2) addr_or |= reinterpret_cast<uintptr_t>(ema_b);
  const bool vec = (addr_or & 15) == 0;
  const long long n4 = vec ? (n >> 2) : 0;
  auto upd = [&](float gi, float& mi, float& vi, float& pi) {
    gi *= gs;
    if (CLIP && md == 1) gi = __fmul_rn(__fdiv_rn(gi, nrm), max_norm);
    mi = b1 * mi + omb1 * gi;
    vi = b2 * vi + omb2 * gi * gi;
    pi -= lrf * (mi * c1) / (sqrtf(vi * c2) + eps);
  };
  auto avg = [](float& ei, float pi, float dk, float omdk) { ei = __fadd_rn(__fmul_rn(dk, ei), __fmul_rn(omdk, pi)); };
  auto avg4 = [&](float* buf, long long i, const float4& p4, float dk, float omdk) {
    float4 e4 = reinterpret_cast<float4*>(buf)[i];
    avg(e4.x, p4.x, dk, omdk); avg(e4.y, p4.y, dk, omdk); avg(e4.z, p4.z, dk, omdk); avg(e4.w, p4.w, dk, omdk);
    reinterpret_cast<float4*>(buf)[i] = e4;
  };
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    const float4 g4 = __ldg(reinterpret_cast<const float4*>(g) + i);
    float4 m4 = reinterpret_cast<float4*>(m)[i], v4 = reinterpret_cast<float4*>(v)[i], p4 = reinterpret_cast<float4*>(p)[i];
    upd(g4.x, m4.x, v4.x, p4.x); upd(g4.y, m4.y, v4.y, p4.y); upd(g4.z, m4.z, v4.z, p4.z); upd(g4.w, m4.w, v4.w, p4.w);
    reinterpret_cast<float4*>(m)[i] = m4;
    reinterpret_cast<float4*>(v)[i] = v4;
    reinterpret_cast<float4*>(p)[i] = p4;
    if (AVG >= 1) avg4(ema, i, p4, d, omd);
    if (AVG == 2) avg4(ema_b, i, p4, db, omdb);
  }
  for (long long i = n4 * 4 + (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    float mi = m[i], vi = v[i], pi = p[i];
    upd(g[i], mi, vi, pi);
    m[i] = mi; v[i] = vi; p[i] = pi;
    if (AVG >= 1) {
      float ei = ema[i];
      avg(ei, pi, d, omd);
      ema[i] = ei;
    }
    if (AVG == 2) {
      float ei = ema_b[i];
      avg(ei, pi, db, omdb);
      ema_b[i] = ei;
    }
  }
}
// ema == nullptr: no EMA; ema_b != nullptr: ema and ema_b are the power averages of exponents gamma_a / gamma_b (decay is
// then unused).  norm_dev == nullptr and warmup == 0: plain Adam, without the clip / warm-up prologue
static void launch_adam(float* p, const float* g, float* m, float* v, long long n, long long step, const long long* step_dev,
                        double lr, double b1, double b2, double eps, double grad_scale, float* ema, double decay,
                        const float* norm_dev, double max_norm, long long warmup, long long* skipped, cudaStream_t s,
                        float* ema_b = nullptr, double gamma_a = 0.0, double gamma_b = 0.0) {
  int blocks = cdiv(n, 256 * 4);   // one float4 per thread and pass
  if (blocks > xu_num_sms() * 8) blocks = xu_num_sms() * 8;
  if (blocks < 1) blocks = 1;
  const bool clip = norm_dev != nullptr || warmup > 0;
  auto kernel = ema_b != nullptr ? (clip ? adam_kernel<2, true> : adam_kernel<2, false>)
                : ema == nullptr ? (clip ? adam_kernel<0, true> : adam_kernel<0, false>)
                                 : (clip ? adam_kernel<1, true> : adam_kernel<1, false>);
  xu_launch(kernel, blocks, 256, 0, s, p, g, m, v, ema, n, step, step_dev, lr, b1, b2, (float)eps, (float)grad_scale,
            decay, norm_dev, (float)max_norm, warmup, skipped, ema_b, gamma_a, gamma_b);
}

extern "C" int xunet_adam_step(float* params, const float* grads, float* m, float* v, long long n, long long step,
                               const long long* step_dev, double lr, double b1, double b2, double eps, double grad_scale,
                               void* stream) {
  if (!params || !grads || !m || !v || n < 0) return xu_fail("xunet_adam_step: bad argument");
  launch_adam(params, grads, m, v, n, step, step_dev, lr, b1, b2, eps, grad_scale, nullptr, 0.0, nullptr, 0.0, 0, nullptr,
              (cudaStream_t)stream);
  return xu_launched("adam");
}

extern "C" int xunet_adam_ema_step(float* params, const float* grads, float* m, float* v, float* ema, long long n,
                                   long long step, const long long* step_dev, double lr, double b1, double b2, double eps,
                                   double grad_scale, double ema_decay, void* stream) {
  if (!params || !grads || !m || !v || n < 0) return xu_fail("xunet_adam_ema_step: bad argument");
  if (!ema) return xu_fail("xunet_adam_ema_step: ema is NULL (use xunet_adam_step without an EMA)");
  if (!(ema_decay >= 0.0 && ema_decay <= 1.0)) return xu_fail("xunet_adam_ema_step: ema_decay %g outside [0, 1]", ema_decay);
  launch_adam(params, grads, m, v, n, step, step_dev, lr, b1, b2, eps, grad_scale, ema, ema_decay, nullptr, 0.0, 0, nullptr,
              (cudaStream_t)stream);
  return xu_launched("adam_ema");
}

extern "C" int xunet_adam_clip_step(float* params, const float* grads, float* m, float* v, float* ema, long long n,
                                    long long step, const long long* step_dev, double lr, double b1, double b2, double eps,
                                    double grad_scale, double ema_decay, const float* norm_dev, double max_norm,
                                    long long warmup_steps, long long* skipped_dev, void* stream) {
  if (!params || !grads || !m || !v || n < 0) return xu_fail("xunet_adam_clip_step: bad argument");
  if (ema && !(ema_decay >= 0.0 && ema_decay <= 1.0)) return xu_fail("xunet_adam_clip_step: ema_decay %g outside [0, 1]", ema_decay);
  if (warmup_steps < 0) return xu_fail("xunet_adam_clip_step: warmup_steps %lld < 0", warmup_steps);
  if (norm_dev) {
    if (!(max_norm > 0.0)) return xu_fail("xunet_adam_clip_step: max_norm %g must be > 0", max_norm);
    if (!skipped_dev) return xu_fail("xunet_adam_clip_step: skipped_dev is NULL (needed with norm_dev)");
  }
  launch_adam(params, grads, m, v, n, step, step_dev, lr, b1, b2, eps, grad_scale, ema, ema ? ema_decay : 0.0, norm_dev,
              max_norm, warmup_steps, skipped_dev, (cudaStream_t)stream);
  return xu_launched("adam_clip");
}

extern "C" int xunet_adam_posthoc_step(float* params, const float* grads, float* m, float* v, float* ema_a, float* ema_b,
                                       long long n, long long step, const long long* step_dev, double lr, double b1,
                                       double b2, double eps, double grad_scale, double gamma_a, double gamma_b,
                                       const float* norm_dev, double max_norm, long long warmup_steps,
                                       long long* skipped_dev, void* stream) {
  if (!params || !grads || !m || !v || n < 0) return xu_fail("xunet_adam_posthoc_step: bad argument");
  if (!ema_a || !ema_b) return xu_fail("xunet_adam_posthoc_step: ema_a and ema_b must both be given");
  if (ema_a == ema_b) return xu_fail("xunet_adam_posthoc_step: ema_a and ema_b are the same buffer");
  if (!(isfinite(gamma_a) && gamma_a > -1.0) || !(isfinite(gamma_b) && gamma_b > -1.0))
    return xu_fail("xunet_adam_posthoc_step: gamma_a %g / gamma_b %g must be finite and > -1", gamma_a, gamma_b);
  if (!step_dev && step < 1) return xu_fail("xunet_adam_posthoc_step: step %lld < 1", step);
  if (warmup_steps < 0) return xu_fail("xunet_adam_posthoc_step: warmup_steps %lld < 0", warmup_steps);
  if (norm_dev) {
    if (!(max_norm > 0.0)) return xu_fail("xunet_adam_posthoc_step: max_norm %g must be > 0", max_norm);
    if (!skipped_dev) return xu_fail("xunet_adam_posthoc_step: skipped_dev is NULL (needed with norm_dev)");
  }
  launch_adam(params, grads, m, v, n, step, step_dev, lr, b1, b2, eps, grad_scale, ema_a, 0.0, norm_dev, max_norm,
              warmup_steps, skipped_dev, (cudaStream_t)stream, ema_b, gamma_a, gamma_b);
  return xu_launched("adam_posthoc");
}

// ---- global gradient norm (optax.clip_by_global_norm) ----------------------------------------------------------------------
// Deterministic by construction: the grid depends on n only, each CTA sums a fixed share of the buffer in a fixed order (per
// thread in index order, then a fixed shuffle / shared-memory tree), and one CTA adds the per-CTA partials the same way.  Each
// scaled gradient fp32(g_i * gs) is squared and accumulated in fp64 (the square of an fp32 value is exact in fp64).
__device__ __forceinline__ double block_sum_fixed(double x, double* red) {   // 256 threads; red: 8 doubles of shared memory
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = x;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < 8; ++w) t += red[w];
  return t;   // valid in thread 0
}

__global__ void __launch_bounds__(256) grad_sumsq_partial_kernel(const float* __restrict__ g, long long n, float gs,
                                                                 double* __restrict__ partials) {
  xu_grid_dep_sync();
  __shared__ double red[8];
  const bool vec = (reinterpret_cast<uintptr_t>(g) & 15) == 0;
  const long long n4 = vec ? (n >> 2) : 0;
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    const float4 g4 = __ldg(reinterpret_cast<const float4*>(g) + i);
    const double x = g4.x * gs, y = g4.y * gs, z = g4.z * gs, w = g4.w * gs;
    acc = fma(x, x, acc); acc = fma(y, y, acc); acc = fma(z, z, acc); acc = fma(w, w, acc);
  }
  for (long long i = n4 * 4 + (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const double x = __ldg(g + i) * gs;
    acc = fma(x, x, acc);
  }
  const double t = block_sum_fixed(acc, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = t;
}

__global__ void __launch_bounds__(256) grad_norm_final_kernel(double* __restrict__ partials, int nparts,
                                                              float* __restrict__ norm_out) {
  xu_grid_dep_sync();
  __shared__ double red[8];
  double acc = 0.0;
  for (int i = threadIdx.x; i < nparts; i += 256) acc += partials[i];
  const double t = block_sum_fixed(acc, red);
  if (threadIdx.x == 0) {
    partials[0] = t;   // the fp64 sum of squares stays readable in scratch[0]
    *norm_out = (float)sqrt(t);
  }
}

static int grad_norm_partials(long long n) {
  long long b = (n + 4095) / 4096;   // at least 16 elements per thread
  if (b > XUNET_GRAD_NORM_SCRATCH) b = XUNET_GRAD_NORM_SCRATCH;
  return b < 1 ? 1 : (int)b;
}
extern "C" int xunet_grad_global_norm(const float* grads, long long n, double grad_scale, double* scratch, float* norm_out,
                                      void* stream) {
  if (!grads || !scratch || !norm_out || n < 0) return xu_fail("xunet_grad_global_norm: bad argument");
  const int parts = grad_norm_partials(n);
  xu_launch(grad_sumsq_partial_kernel, parts, 256, 0, (cudaStream_t)stream, grads, n, (float)grad_scale, scratch);
  xu_launch(grad_norm_final_kernel, 1, 256, 0, (cudaStream_t)stream, scratch, parts, norm_out);
  return xu_launched("grad_global_norm");
}

// dataset/data_loader.py:92-110 on the device.  TARGET == XU_TARGET_V also stores v = xu_fd_v(..) to v_out (the last
// parameter, so the eps instance keeps its parameter layout and code).
template <int TARGET>
__global__ void __launch_bounds__(256) forward_diffusion_kernel(const float* __restrict__ x0, const float* __restrict__ noise_in,
                                                                const int* __restrict__ t_in, unsigned long long seed,
                                                                const float* __restrict__ sqrt_ac, const float* __restrict__ sqrt_1mac,
                                                                float p_uncond, float* __restrict__ z, float* __restrict__ noise_out,
                                                                float* __restrict__ logsnr_out, int* __restrict__ t_out,
                                                                float* __restrict__ cond_mask_out, int B, long long per,
                                                                float* __restrict__ v_out) {
  xu_grid_dep_sync();
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= (long long)B * per) return;
  const int b = (int)(idx / per);
  const uint64_t hb = xu_fd_sample_hash(seed, b);
  const int t = t_in != nullptr ? t_in[b] : xu_fd_timestep(hb);
  const float nz = noise_in != nullptr ? noise_in[idx] : xu_hash_normal(seed, (uint64_t)idx);
  if constexpr (TARGET == XU_TARGET_V) {
    const float sa = sqrt_ac[t], sb = sqrt_1mac[t], x = x0[idx];
    z[idx] = xu_fd_z_rn(sa, x, sb, nz);
    v_out[idx] = xu_fd_v(sa, nz, sb, x);
  } else {
    z[idx] = xu_fd_z(sqrt_ac[t], x0[idx], sqrt_1mac[t], nz);
  }
  if (noise_out != nullptr) noise_out[idx] = nz;
  if (idx == (long long)b * per) {
    logsnr_out[b] = xu_fd_logsnr(t);
    if (t_out != nullptr) t_out[b] = t;
    if (cond_mask_out != nullptr) cond_mask_out[b] = xu_fd_cond_mask(hb, p_uncond);
  }
}
extern "C" int xunet_forward_diffusion(const float* x0, const float* noise_in, const int* t_in, unsigned long long seed,
                                       const float* sqrt_ac, const float* sqrt_1mac, float p_uncond, float* z, float* noise_out,
                                       float* logsnr_out, int* t_out, float* cond_mask_out, int B, long long per, void* stream) {
  if (!x0 || !sqrt_ac || !sqrt_1mac || !z || !logsnr_out || B < 1 || per < 1) return xu_fail("xunet_forward_diffusion: bad argument");
  xu_launch(forward_diffusion_kernel<XU_TARGET_EPS>, cdiv((long long)B * per, 256), 256, 0, (cudaStream_t)stream, x0, noise_in,
            t_in, seed, sqrt_ac, sqrt_1mac, p_uncond, z, noise_out, logsnr_out, t_out, cond_mask_out, B, per, nullptr);
  return xu_launched("forward_diffusion");
}

extern "C" int xunet_forward_diffusion_v(const float* x0, const float* noise_in, const int* t_in, unsigned long long seed,
                                         const float* sqrt_ac, const float* sqrt_1mac, float p_uncond, float* z,
                                         float* noise_out, float* v_out, float* logsnr_out, int* t_out, float* cond_mask_out,
                                         int B, long long per, void* stream) {
  if (!x0 || !sqrt_ac || !sqrt_1mac || !z || !v_out || !logsnr_out) return xu_fail("xunet_forward_diffusion_v: NULL pointer argument");
  if (B < 1 || per < 1) return xu_fail("xunet_forward_diffusion_v: B = %d, per = %lld, need both >= 1", B, per);
  xu_launch(forward_diffusion_kernel<XU_TARGET_V>, cdiv((long long)B * per, 256), 256, 0, (cudaStream_t)stream, x0, noise_in,
            t_in, seed, sqrt_ac, sqrt_1mac, p_uncond, z, noise_out, logsnr_out, t_out, cond_mask_out, B, per, v_out);
  return xu_launched("forward_diffusion_v");
}

__global__ void dropout_mask_kernel(float* __restrict__ out, long long n, int op_index, unsigned long long seed, float rate) {
  xu_grid_dep_sync();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i < n) out[i] = xu_keep(seed, op_index, (unsigned long long)i, rate) ? 1.f : 0.f;
}
extern "C" int xunet_dropout_mask(float* mask_out, long long n, int op_index, unsigned long long seed, float rate,
                                  void* stream) {
  if (!mask_out || n <= 0) return xu_fail("xunet_dropout_mask: bad argument");
  xu_launch(dropout_mask_kernel, cdiv(n, 256), 256, 0, (cudaStream_t)stream, mask_out, n, op_index, seed, rate);
  return xu_launched("dropout_mask");
}
