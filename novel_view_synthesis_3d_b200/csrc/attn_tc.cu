// attn_tc.cu -- wgmma / TMA flash attention over frames for sm_90a (bf16 operands, fp32 softmax state and accumulators).
//
// Replaces nn.dot_product_attention (model/xunet.py:103: two einsums + a materialised (B,h,L,L) fp32 score tensor) and
// the AttnBlock residual (model/xunet.py:127) for BOTH attention flavours: kv_frame = frame ^ cross (model/xunet.py:114-121).
//
// Forward: one CTA = one (frame n, head h, 64-query tile) = one consumer warpgroup + one TMA producer warp.  Per 64-key block j:
//   S_j[64q,64k] = Q K_j^T            (wgmma, Q and K_j K-major from TMA-swizzled smem, fp32 accumulators in registers)
//   online softmax on the accumulator fragment (a row lives in the 4 lanes of a quad), P_j -> bf16 A-operand registers
//   O = O * corr + P_j V_j            (wgmma with A from registers, B = V_j MN-major straight from the TMA box)
// Epilogue: out = (O / l + residual) / sqrt(2), lse = m + log(l) for the backward.
// Backward (FlashAttention-2 order): one CTA = one (query frame n, head h, 64-key tile); it streams the 64-query blocks of the
// frame and accumulates dK, dV in registers; the dQ contributions of its keys are summed in an fp64 buffer (xu_det_scratch),
// so the result does not depend on the order in which the key tiles finish.  attn_bwd_prep_kernel forms D = rowsum(dO * O),
// attn_bwd_dq_store_kernel rounds dQ to bf16 and re-zeroes the fp64 buffer.
#include "kernels.h"
#include "tc_common.cuh"

namespace {

constexpr int kBlk = 64;          // queries per forward CTA, keys per backward CTA, keys / queries per streamed block
constexpr int kAttnThreads = 160; // one consumer warpgroup + one producer warp

__host__ __device__ constexpr int attn_cw(int hd) { return hd < 64 ? hd : 64; }     // channel chunk = one swizzle span
__host__ __device__ constexpr int attn_stages(int hd) { return hd <= 32 ? 4 : 2; }

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
// accumulator fragment of a 64 x 64 tile (32 floats) -> the four 16-column A-operand slices of the next wgmma
__device__ __forceinline__ void frag_to_a(const float (&x)[32], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int q = 0; q < 4; ++q) a[kk][q] = pack_bf16(x[8 * kk + 2 * q], x[8 * kk + 2 * q + 1]);
}

struct AttnTcParams {
  const bf16* res;
  bf16* out;
  float* lse;
  int L, C, heads, cross;
  float scale_log2;   // log2(e) / sqrt(hd)
  double* cstats;     // optional: per-(sample, channel) [sum, sumsq] of the stored output (N/2, C, 2) -- the next GroupNorm's statistics,
                      // accumulated in fp64 (xu_det_scratch) and folded into the caller's fp32 buffer after the kernel
};

template <int HD>
__global__ void __launch_bounds__(kAttnThreads) attn_fwd_tc_kernel(const __grid_constant__ CUtensorMap tmQKV, const AttnTcParams p) {
  constexpr int CW = attn_cw(HD);
  constexpr int NCH = HD / CW;
  constexpr int TILE = kBlk * CW * 2;         // [64 rows][CW] bf16
  constexpr int ST = attn_stages(HD);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smQ = base;
  uint8_t* smK = smQ + NCH * TILE;            // ST x NCH tiles
  uint8_t* smV = smK + ST * NCH * TILE;
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smV + ST * NCH * TILE);
  uint64_t* kv_full = q_full + 1;
  uint64_t* kv_empty = kv_full + ST;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kBlk, h = blockIdx.y, n = blockIdx.z;
  const int nkv = p.cross ? (n ^ 1) : n;
  const int nkb = p.L / kBlk;
  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < ST; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmQKV) : "memory");
  }
  __syncthreads();
  xu_grid_dep_sync();

  if (warp == 4) {
    if (lane == 0) {
      mbar_expect_tx(q_full, NCH * TILE);
      for (int c = 0; c < NCH; ++c) tma_load_3d(smQ + c * TILE, &tmQKV, q_full, h * HD + c * CW, q0, n);
      for (int j = 0; j < nkb; ++j) {
        const int s = j % ST;
        mbar_wait(&kv_empty[s], ((j / ST) & 1) ^ 1);
        mbar_expect_tx(&kv_full[s], 2 * NCH * TILE);
        for (int c = 0; c < NCH; ++c) {
          tma_load_3d(smK + (s * NCH + c) * TILE, &tmQKV, &kv_full[s], p.C + h * HD + c * CW, j * kBlk, nkv);
          tma_load_3d(smV + (s * NCH + c) * TILE, &tmQKV, &kv_full[s], 2 * p.C + h * HD + c * CW, j * kBlk, nkv);
        }
      }
    }
    return;
  }
  // ===== consumer warpgroup: thread rows 16 warp + g and + 8 (g = lane / 4), columns 8 i + 2 t (+1) =====
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};     // m in log2 units; l = this thread's partial row sums
  mbar_wait(q_full, 0);
  for (int j = 0; j < nkb; ++j) {
    const int s = j % ST;
    mbar_wait(&kv_full[s], (j / ST) & 1);
    float sc[32];
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int kk = 0; kk < CW / 16; ++kk)
        Wgmma<64>::template ss<0, 0>(sc, make_kmajor_desc<CW>(smem_u32(smQ + c * TILE) + kk * 32),
                                     make_kmajor_desc<CW>(smem_u32(smK + (s * NCH + c) * TILE) + kk * 32), (c > 0 || kk > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    float corr[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 8; ++i) mx = fmaxf(mx, fmaxf(sc[4 * i + 2 * hh], sc[4 * i + 2 * hh + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(m[hh], mx * p.scale_log2);      // scale > 0: max commutes with the scaling
      corr[hh] = ex2_approx(m[hh] - mn);                      // m = -inf on the first block -> 0
      m[hh] = mn;
      float rs = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float pv = ex2_approx(fmaf(sc[4 * i + 2 * hh + e], p.scale_log2, -mn));
          sc[4 * i + 2 * hh + e] = pv;
          rs += pv;
        }
      l[hh] = l[hh] * corr[hh] + rs;
    }
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
      o[4 * i] *= corr[0]; o[4 * i + 1] *= corr[0];
      o[4 * i + 2] *= corr[1]; o[4 * i + 3] *= corr[1];
    }
    uint32_t pa[4][4];
    frag_to_a(sc, pa);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      Wgmma<HD>::template rs<1>(o, pa[kk], make_mnmajor_desc<CW>(smem_u32(smV + s * NCH * TILE) + kk * 16 * (CW * 2), TILE), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&kv_empty[s]);
  }
  // epilogue: (O / l + residual) / sqrt2
  float inv[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    inv[hh] = 1.f / l[hh];
  }
  const int g = lane >> 2, t = lane & 3;
  const long long row0 = (long long)n * p.L + q0 + 16 * warp + g;
  double* cs_row = p.cstats ? p.cstats + ((long long)(n >> 1) * p.C + h * HD) * 2 : nullptr;   // both frames of a sample pool
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) {
    const int col = 8 * i + 2 * t;
    float sum0 = 0.f, sum1 = 0.f, sq0 = 0.f, sq1 = 0.f;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const long long off = (row0 + 8 * hh) * p.C + h * HD + col;
      const __nv_bfloat162 r2 = *reinterpret_cast<const __nv_bfloat162*>(p.res + off);
      const __nv_bfloat162 o2 = __floats2bfloat162_rn((o[4 * i + 2 * hh] * inv[hh] + __low2float(r2)) * XU_RSQRT2,
                                                      (o[4 * i + 2 * hh + 1] * inv[hh] + __high2float(r2)) * XU_RSQRT2);
      *reinterpret_cast<__nv_bfloat162*>(p.out + off) = o2;
      const float a = __low2float(o2), b = __high2float(o2);   // statistics of the rounded, stored values
      sum0 += a; sum1 += b; sq0 += a * a; sq1 += b * b;
    }
    if (cs_row != nullptr) {     // CTA-uniform branch: reduce over the 8 row groups of the warp, one red per channel and warp
#pragma unroll
      for (int sh = 4; sh < 32; sh <<= 1) {
        sum0 += __shfl_xor_sync(0xffffffffu, sum0, sh); sum1 += __shfl_xor_sync(0xffffffffu, sum1, sh);
        sq0 += __shfl_xor_sync(0xffffffffu, sq0, sh); sq1 += __shfl_xor_sync(0xffffffffu, sq1, sh);
      }
      if (g == 0) {
        xu_det_add(cs_row + col * 2, sum0); xu_det_add(cs_row + col * 2 + 1, sq0);
        xu_det_add(cs_row + col * 2 + 2, sum1); xu_det_add(cs_row + col * 2 + 3, sq1);
      }
    }
  }
  // natural-log LSE of the scaled scores (what the backward expects): m is in log2 units
  if (t == 0) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
      p.lse[((long long)n * p.heads + h) * p.L + q0 + 16 * warp + g + 8 * hh] = m[hh] * 0.69314718055994530942f + __logf(l[hh]);
  }
}

// ================================================================================================================
// backward.  dO = dout / sqrt2 (the AttnBlock residual scale), D = rowsum(dO * O), P = exp(S*scale - lse),
// dS = P * (dP - D) * scale.
// ================================================================================================================
struct AttnBwdParams {
  const bf16* res; const bf16* out; const bf16* dout;
  const float* lse; float* Dbuf; double* dq64; bf16* dqkv;
  int L, C, heads, cross;
  float scale, scale_log2;
};

template <int HD>
__global__ void __launch_bounds__(kAttnThreads) attn_bwd_tc_kernel(const __grid_constant__ CUtensorMap tmQKV,
                                                                   const __grid_constant__ CUtensorMap tmG, const AttnBwdParams p) {
  constexpr int CW = attn_cw(HD);
  constexpr int NCH = HD / CW;
  constexpr int TILE = kBlk * CW * 2;
  constexpr int ST = attn_stages(HD);
  constexpr int DQN = HD <= 64 ? HD : 64;     // dQ is formed DQN columns at a time (register budget at head_dim 128)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smK = base;                        // resident key / value tiles of this CTA
  uint8_t* smV = smK + NCH * TILE;
  uint8_t* smDS = smV + NCH * TILE;           // dS^T [64 keys][64 queries] bf16, 128B-swizzled (MN-major A operand of dQ)
  uint8_t* smQ = smDS + kBlk * kBlk * 2;      // ST x NCH tiles
  uint8_t* smG = smQ + ST * NCH * TILE;       // ST x NCH tiles of dout
  uint64_t* kv_full = reinterpret_cast<uint64_t*>(smG + ST * NCH * TILE);
  uint64_t* full = kv_full + 1;
  uint64_t* empty = full + ST;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = blockIdx.x * kBlk, h = blockIdx.y, n = blockIdx.z;     // n = query frame
  const int nkv = p.cross ? (n ^ 1) : n;
  const int nqb = p.L / kBlk;
  if (threadIdx.x == 0) {
    mbar_init(kv_full, 1);
    for (int s = 0; s < ST; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmQKV) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmG) : "memory");
  }
  __syncthreads();
  xu_grid_dep_sync();

  if (warp == 4) {
    if (lane == 0) {
      mbar_expect_tx(kv_full, 2 * NCH * TILE);
      for (int c = 0; c < NCH; ++c) {
        tma_load_3d(smK + c * TILE, &tmQKV, kv_full, p.C + h * HD + c * CW, k0, nkv);
        tma_load_3d(smV + c * TILE, &tmQKV, kv_full, 2 * p.C + h * HD + c * CW, k0, nkv);
      }
      for (int j = 0; j < nqb; ++j) {
        const int s = j % ST;
        mbar_wait(&empty[s], ((j / ST) & 1) ^ 1);
        mbar_expect_tx(&full[s], 2 * NCH * TILE);
        for (int c = 0; c < NCH; ++c) {
          tma_load_3d(smQ + (s * NCH + c) * TILE, &tmQKV, &full[s], h * HD + c * CW, j * kBlk, n);
          tma_load_3d(smG + (s * NCH + c) * TILE, &tmG, &full[s], h * HD + c * CW, j * kBlk, n);
        }
      }
    }
    return;
  }
  const int g = lane >> 2, t = lane & 3;
  float dv[HD / 2], dk[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  const float* lse_row = p.lse + ((long long)n * p.heads + h) * p.L;
  const float* D_row = p.Dbuf + ((long long)n * p.heads + h) * p.L;
  mbar_wait(kv_full, 0);
  for (int j = 0; j < nqb; ++j) {
    const int s = j % ST;
    // per-query operands of the 16 columns this thread holds (L1 / L2 hits: 64 floats per block)
    float lq[16], dq_[16];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int q = j * kBlk + 8 * i + 2 * t + e;
        lq[2 * i + e] = __ldg(lse_row + q) * 1.4426950408889634f;
        dq_[2 * i + e] = __ldg(D_row + q);
      }
    mbar_wait(&full[s], (j / ST) & 1);
    const uint32_t q_addr = smem_u32(smQ + s * NCH * TILE), g_addr = smem_u32(smG + s * NCH * TILE);
    float st[32], dpt[32];
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int kk = 0; kk < CW / 16; ++kk) {
        // S^T = K Q^T  and  dP^T = V dout^T  (every operand K-major: head_dim contiguous)
        Wgmma<64>::template ss<0, 0>(st, make_kmajor_desc<CW>(smem_u32(smK + c * TILE) + kk * 32),
                                     make_kmajor_desc<CW>(q_addr + c * TILE + kk * 32), (c > 0 || kk > 0) ? 1u : 0u);
        Wgmma<64>::template ss<0, 0>(dpt, make_kmajor_desc<CW>(smem_u32(smV + c * TILE) + kk * 32),
                                     make_kmajor_desc<CW>(g_addr + c * TILE + kk * 32), (c > 0 || kk > 0) ? 1u : 0u);
      }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * i + 2 * hh + e;
          const float pv = ex2_approx(fmaf(st[x], p.scale_log2, -lq[2 * i + e]));
          st[x] = pv;
          dpt[x] = pv * (dpt[x] * XU_RSQRT2 - dq_[2 * i + e]) * p.scale;
        }
    uint32_t pa[4][4], da[4][4];
    frag_to_a(st, pa);
    frag_to_a(dpt, da);
    // dS^T -> shared memory (row = key, 128-byte rows of 64 queries, 16-byte chunks XOR-swizzled by row)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int R = 16 * warp + g + 8 * hh;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t v = pack_bf16(dpt[4 * i + 2 * hh], dpt[4 * i + 2 * hh + 1]);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(smem_u32(smDS + R * 128 + ((i ^ (R & 7)) << 4) + 4 * t)), "r"(v) : "memory");
      }
    }
    fence_async_smem();
    named_bar_sync(1, 128);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      // dV += P^T dout,  dK += dS^T Q   (B = the query-block tiles, MN-major: head_dim contiguous)
      Wgmma<HD>::template rs<1>(dv, pa[kk], make_mnmajor_desc<CW>(g_addr + kk * 16 * (CW * 2), TILE), 1u);
      Wgmma<HD>::template rs<1>(dk, da[kk], make_mnmajor_desc<CW>(q_addr + kk * 16 * (CW * 2), TILE), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    // dQ[64 q][HD] += dS K: A = dS^T in shared memory read MN-major (M = queries), B = the resident key tile (MN-major)
    const long long qrow0 = (long long)n * p.L + j * kBlk + 16 * warp + g;
#pragma unroll
    for (int c2 = 0; c2 < HD / DQN; ++c2) {
      float dq[DQN / 2];
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        Wgmma<DQN>::template ss<1, 1>(dq, make_mnmajor_desc<64>(smem_u32(smDS) + kk * 16 * 128, 8192),
                                      make_mnmajor_desc<CW>(smem_u32(smK + c2 * TILE) + kk * 16 * (CW * 2), TILE), kk > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < DQN / 8; ++i)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          double* d = p.dq64 + (qrow0 + 8 * hh) * p.C + h * HD + c2 * DQN + 8 * i + 2 * t;
          xu_det_add(d, dq[4 * i + 2 * hh]);
          xu_det_add(d + 1, dq[4 * i + 2 * hh + 1]);
        }
    }
    if (lane == 0) mbar_arrive(&empty[s]);
    named_bar_sync(1, 128);      // every warp's dQ MMAs have read smDS before the next block overwrites it
  }
  // dK, dV of this CTA's 64 keys (dV picks up the 1/sqrt2 of dO here)
  const long long krow0 = (long long)nkv * p.L + k0 + 16 * warp + g;
#pragma unroll
  for (int i = 0; i < HD / 8; ++i)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      bf16* d = p.dqkv + (krow0 + 8 * hh) * (3LL * p.C) + h * HD + 8 * i + 2 * t;
      *reinterpret_cast<__nv_bfloat162*>(d + p.C) = __floats2bfloat162_rn(dk[4 * i + 2 * hh], dk[4 * i + 2 * hh + 1]);
      *reinterpret_cast<__nv_bfloat162*>(d + 2 * p.C) =
          __floats2bfloat162_rn(dv[4 * i + 2 * hh] * XU_RSQRT2, dv[4 * i + 2 * hh + 1] * XU_RSQRT2);
    }
}

// D = rowsum(dO * O) per (row, head) (one thread per row and head)
template <int HD>
__global__ void __launch_bounds__(256) attn_bwd_prep_kernel(const AttnBwdParams p, long long total) {
  xu_grid_dep_sync();
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= total) return;
  const int h = (int)(idx % p.heads);
  const long long row = idx / p.heads;
  const long long o = row * p.C + h * HD;
  float D = 0.f;
#pragma unroll
  for (int c0 = 0; c0 < HD; c0 += 8) {
    uint4 gv = *reinterpret_cast<const uint4*>(p.dout + o + c0);
    uint4 ov = *reinterpret_cast<const uint4*>(p.out + o + c0);
    uint4 rv = *reinterpret_cast<const uint4*>(p.res + o + c0);
    const __nv_bfloat162* g2 = reinterpret_cast<const __nv_bfloat162*>(&gv);
    const __nv_bfloat162* o2 = reinterpret_cast<const __nv_bfloat162*>(&ov);
    const __nv_bfloat162* r2 = reinterpret_cast<const __nv_bfloat162*>(&rv);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      D = fmaf(__low2float(g2[q]) * XU_RSQRT2, __low2float(o2[q]) * XU_SQRT2 - __low2float(r2[q]), D);
      D = fmaf(__high2float(g2[q]) * XU_RSQRT2, __high2float(o2[q]) * XU_SQRT2 - __high2float(r2[q]), D);
    }
  }
  const long long n = row / p.L, l = row % p.L;
  p.Dbuf[(n * p.heads + h) * p.L + l] = D;
}

// dq64 -> the q third of dqkv (bf16), 4 channels per thread, re-zeroing dq64.  zero: also clear the n_d D values, so that a
// caller that keeps its scratch buffer all-zero between calls gets it back that way.
__global__ void __launch_bounds__(256) attn_bwd_dq_store_kernel(double* __restrict__ dq64, bf16* __restrict__ dqkv, long long total4,
                                                                int C, float* __restrict__ dbuf, long long n_d, int zero) {
  xu_grid_dep_sync();
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= total4) return;
  const int c4 = (int)(idx % (C / 4));
  const long long row = idx / (C / 4);
  double2* src = reinterpret_cast<double2*>(dq64 + row * C + c4 * 4);
  const double2 v01 = src[0], v23 = src[1];
  src[0] = make_double2(0.0, 0.0);
  src[1] = make_double2(0.0, 0.0);
  __nv_bfloat162 a = __floats2bfloat162_rn((float)v01.x, (float)v01.y), b = __floats2bfloat162_rn((float)v23.x, (float)v23.y);
  uint2 t;
  t.x = *reinterpret_cast<uint32_t*>(&a);
  t.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(dqkv + row * (3LL * C) + c4 * 4) = t;
  if (zero && idx < n_d) dbuf[idx] = 0.f;
}

template <int HD>
void launch_bwd(const AttnArgs& a, cudaStream_t s) {
  constexpr int CW = attn_cw(HD);
  constexpr int NCH = HD / CW;
  constexpr int TILE = kBlk * CW * 2;
  CUtensorMap tq, tg;
  uint64_t qd[3] = {(uint64_t)(3 * a.C), (uint64_t)a.L, (uint64_t)a.N};
  uint64_t qs[2] = {(uint64_t)3 * a.C * 2, (uint64_t)a.L * 3 * a.C * 2};
  uint64_t gd[3] = {(uint64_t)a.C, (uint64_t)a.L, (uint64_t)a.N};
  uint64_t gs[2] = {(uint64_t)a.C * 2, (uint64_t)a.L * a.C * 2};
  uint32_t box[3] = {(uint32_t)CW, (uint32_t)kBlk, 1u};
  if (!xu_encode_bf16_map(&tq, a.qkv, 3, qd, qs, box, CW) || !xu_encode_bf16_map(&tg, a.dout, 3, gd, gs, box, CW)) return;
  AttnBwdParams p;
  p.res = (const bf16*)a.res; p.out = (const bf16*)a.out; p.dout = (const bf16*)a.dout;
  p.lse = a.lse; p.Dbuf = a.dscratch; p.dqkv = (bf16*)a.dqkv;
  const long long rows = (long long)a.N * a.L;
  p.dq64 = xu_det_scratch(s, rows * a.C);                     // [N*L][C] fp64
  if (p.dq64 == nullptr) return;
  p.L = a.L; p.C = a.C; p.heads = a.heads; p.cross = a.cross;
  p.scale = 1.f / sqrtf((float)HD);
  p.scale_log2 = 1.4426950408889634f * p.scale;
  const size_t smem = (size_t)2 * NCH * TILE + kBlk * kBlk * 2 + (size_t)2 * attn_stages(HD) * NCH * TILE + 1024 + 256;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(attn_bwd_tc_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    configured = true;
  }
  xu_launch(attn_bwd_prep_kernel<HD>, cdiv(rows * a.heads, 256), 256, 0, s, p, rows * a.heads);
  xu_launch(attn_bwd_tc_kernel<HD>, dim3(a.L / kBlk, a.heads, a.N), kAttnThreads, smem, s, tq, tg, p);
  xu_launch(attn_bwd_dq_store_kernel, cdiv(rows * a.C / 4, 256), 256, 0, s, p.dq64, p.dqkv, rows * a.C / 4, a.C, p.Dbuf,
            rows * a.heads, a.scratch_zeroed);
}

template <int HD>
void launch_fwd(const AttnArgs& a, cudaStream_t s) {
  constexpr int CW = attn_cw(HD);
  constexpr int NCH = HD / CW;
  constexpr int TILE = kBlk * CW * 2;
  CUtensorMap tq;
  uint64_t dims[3] = {(uint64_t)(3 * a.C), (uint64_t)a.L, (uint64_t)a.N};
  uint64_t strides[2] = {(uint64_t)3 * a.C * 2, (uint64_t)a.L * 3 * a.C * 2};
  uint32_t box[3] = {(uint32_t)CW, (uint32_t)kBlk, 1u};
  if (!xu_encode_bf16_map(&tq, a.qkv, 3, dims, strides, box, CW)) return;
  AttnTcParams p;
  p.res = (const bf16*)a.res; p.out = (bf16*)a.out; p.lse = a.lse;
  p.L = a.L; p.C = a.C; p.heads = a.heads; p.cross = a.cross;
  p.scale_log2 = 1.4426950408889634f / sqrtf((float)HD);
  const long long ncs = a.cstats ? (long long)(a.N / 2) * a.C * 2 : 0;
  p.cstats = nullptr;
  if (ncs > 0 && (p.cstats = xu_det_scratch(s, ncs)) == nullptr) return;
  const size_t smem = (size_t)NCH * TILE + (size_t)2 * attn_stages(HD) * NCH * TILE + 1024 + 256;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(attn_fwd_tc_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    configured = true;
  }
  xu_launch(attn_fwd_tc_kernel<HD>, dim3(a.L / kBlk, a.heads, a.N), kAttnThreads, smem, s, tq, p);
  if (p.cstats != nullptr) xu_det_fold(a.cstats, p.cstats, ncs, s);
}

}  // namespace

bool attn_tc_supported(int dtype, int L, int C, int heads) {
  if (dtype != XU_BF16 || heads <= 0 || C % heads) return false;
  const int hd = C / heads;
  if (hd != 16 && hd != 32 && hd != 64 && hd != 128) return false;
  return L % 128 == 0 && (3 * C) % 8 == 0;
}

void launch_attn_bwd_tc(const AttnArgs& a, cudaStream_t s) {
  switch (a.C / a.heads) {
    case 16: launch_bwd<16>(a, s); break;
    case 32: launch_bwd<32>(a, s); break;
    case 64: launch_bwd<64>(a, s); break;
    case 128: launch_bwd<128>(a, s); break;
    default: xu_set_kernel_error("attn_tc: unsupported head_dim");
  }
}

void launch_attn_fwd_tc(const AttnArgs& a, cudaStream_t s) {
  switch (a.C / a.heads) {
    case 16: launch_fwd<16>(a, s); break;
    case 32: launch_fwd<32>(a, s); break;
    case 64: launch_fwd<64>(a, s); break;
    case 128: launch_fwd<128>(a, s); break;
    default: xu_set_kernel_error("attn_tc: unsupported head_dim");
  }
}
