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
// Backward: two passes without atomics.  attn_bwd_dq_tc_kernel has the forward's grid (one CTA per 64-query tile): it forms
// D = rowsum(dO * O) of its rows, streams the key / value blocks and accumulates dQ in registers.  attn_bwd_dkdv_tc_kernel
// (FlashAttention-2 order: one CTA per 64-key tile) streams the 64-query blocks and accumulates dK, dV in registers.
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
// dS = P * (dP - D) * scale.  Two passes with the forward's warp layout (one consumer warpgroup + one TMA producer warp):
//   attn_bwd_dq_tc_kernel   one CTA = one (query frame n, head h, 64-query tile): forms D of its 64 rows (and stores it for
//                           the second pass), streams the key / value blocks and accumulates dQ = sum_j dS_j K_j in registers
//                           (each block's product in fp32, their sum in fp64).
//   attn_bwd_dkdv_tc_kernel one CTA = one (query frame n, head h, 64-key tile): streams the 64-query blocks and accumulates
//                           dK = sum_j dS_j^T Q_j, dV = sum_j P_j^T dO_j in registers.
// Every gradient element is owned by one CTA and summed in a fixed order: no atomics, deterministic by construction.
// S and dP are recomputed by the second pass (a second round of exponentials) in exchange for that.
// ================================================================================================================
struct AttnBwdParams {
  const bf16* res; const bf16* out; const bf16* dout;
  const float* lse; float* Dbuf; bf16* dqkv;
  int L, C, heads, cross;
  float scale, scale_log2;
};

// CTAs per SM the backward kernels are compiled for (__launch_bounds__ minimum): the largest count whose register budget
// ptxas meets without spilling
__host__ __device__ constexpr int attn_dq_ctas(int hd) { return hd <= 32 ? 3 : (hd == 64 ? 2 : 1); }
__host__ __device__ constexpr int attn_dkdv_ctas(int hd) { return hd == 16 ? 3 : (hd <= 64 ? 2 : 1); }

template <int HD>
__global__ void __launch_bounds__(kAttnThreads, attn_dq_ctas(HD))
    attn_bwd_dq_tc_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmG, const AttnBwdParams p) {
  constexpr int CW = attn_cw(HD);
  constexpr int NCH = HD / CW;
  constexpr int TILE = kBlk * CW * 2;
  constexpr int ST = attn_stages(HD);
  constexpr int DQN = HD <= 64 ? HD : 64;     // dQ_j is formed DQN columns at a time (register budget at head_dim 128)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smQ = base;                        // resident query / dout tiles of this CTA
  uint8_t* smG = smQ + NCH * TILE;
  uint8_t* smK = smG + NCH * TILE;            // ST x NCH tiles
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
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmG) : "memory");
  }
  __syncthreads();
  xu_grid_dep_sync();

  if (warp == 4) {
    if (lane == 0) {
      mbar_expect_tx(q_full, 2 * NCH * TILE);
      for (int c = 0; c < NCH; ++c) {
        tma_load_3d(smQ + c * TILE, &tmQKV, q_full, h * HD + c * CW, q0, n);
        tma_load_3d(smG + c * TILE, &tmG, q_full, h * HD + c * CW, q0, n);
      }
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
  const int g = lane >> 2, t = lane & 3;
  const long long row0 = (long long)n * p.L + q0 + 16 * warp + g;
  const long long srow0 = ((long long)n * p.heads + h) * p.L + q0 + 16 * warp + g;   // (n, h, q) index of lse / D
  // D = rowsum(dO * O) with O = out * sqrt2 - res, one fma per channel in channel order (every lane of the quad forms its
  // rows' D the same way).  D and lse are per-row constants of the whole key loop.
  float Dr[2], lq[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const long long off = (row0 + 8 * hh) * p.C + h * HD;
    float D = 0.f;
#pragma unroll
    for (int c = 0; c < HD; c += 2) {
      const __nv_bfloat162 g2 = *reinterpret_cast<const __nv_bfloat162*>(p.dout + off + c);
      const __nv_bfloat162 o2 = *reinterpret_cast<const __nv_bfloat162*>(p.out + off + c);
      const __nv_bfloat162 r2 = *reinterpret_cast<const __nv_bfloat162*>(p.res + off + c);
      D = fmaf(__low2float(g2) * XU_RSQRT2, __low2float(o2) * XU_SQRT2 - __low2float(r2), D);
      D = fmaf(__high2float(g2) * XU_RSQRT2, __high2float(o2) * XU_SQRT2 - __high2float(r2), D);
    }
    Dr[hh] = D;
    lq[hh] = p.lse[srow0 + 8 * hh] * 1.4426950408889634f;
  }
  if (t == 0) { p.Dbuf[srow0] = Dr[0]; p.Dbuf[srow0 + 8] = Dr[1]; }
  double dq[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) dq[i] = 0.0;
  mbar_wait(q_full, 0);
  for (int j = 0; j < nkb; ++j) {
    const int s = j % ST;
    mbar_wait(&kv_full[s], (j / ST) & 1);
    const uint32_t k_addr = smem_u32(smK + s * NCH * TILE), v_addr = smem_u32(smV + s * NCH * TILE);
    float sc[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int kk = 0; kk < CW / 16; ++kk) {
        // S = Q K_j^T  and  dP = dout V_j^T  (every operand K-major: head_dim contiguous)
        Wgmma<64>::template ss<0, 0>(sc, make_kmajor_desc<CW>(smem_u32(smQ + c * TILE) + kk * 32),
                                     make_kmajor_desc<CW>(k_addr + c * TILE + kk * 32), (c > 0 || kk > 0) ? 1u : 0u);
        Wgmma<64>::template ss<0, 0>(dp, make_kmajor_desc<CW>(smem_u32(smG + c * TILE) + kk * 32),
                                     make_kmajor_desc<CW>(v_addr + c * TILE + kk * 32), (c > 0 || kk > 0) ? 1u : 0u);
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
          const float pv = ex2_approx(fmaf(sc[x], p.scale_log2, -lq[hh]));
          dp[x] = pv * (dp[x] * XU_RSQRT2 - Dr[hh]) * p.scale;
        }
    uint32_t da[4][4];
    frag_to_a(dp, da);
    // dQ_j = dS K_j in fp32 (B = the key tile read MN-major, as the forward reads V), DQN columns at a time, then added to the
    // fp64 dQ in key-block order: fp64 carries 29 more significand bits than the fp32 addends, so the sum is exact unless they
    // span about 29 - log2(L / 64) binary orders of magnitude (DESIGN §4); rounded fp64 -> fp32 -> bf16 once at the end
#pragma unroll
    for (int c2 = 0; c2 < HD / DQN; ++c2) {
      float part[DQN / 2];
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        Wgmma<DQN>::template rs<1>(part, da[kk], make_mnmajor_desc<CW>(k_addr + c2 * TILE + kk * 16 * (CW * 2), TILE), kk > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < DQN / 2; ++i) dq[c2 * (DQN / 2) + i] += (double)part[i];
    }
    if (lane == 0) mbar_arrive(&kv_empty[s]);
  }
#pragma unroll
  for (int c2 = 0; c2 < HD / DQN; ++c2)
#pragma unroll
    for (int i = 0; i < DQN / 8; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const double* v = dq + c2 * (DQN / 2) + 4 * i + 2 * hh;
        *reinterpret_cast<__nv_bfloat162*>(p.dqkv + (row0 + 8 * hh) * (3LL * p.C) + h * HD + c2 * DQN + 8 * i + 2 * t) =
            __floats2bfloat162_rn((float)v[0], (float)v[1]);
      }
}

// runs after attn_bwd_dq_tc_kernel, whose D (Dbuf) it reads
template <int HD>
__global__ void __launch_bounds__(kAttnThreads, attn_dkdv_ctas(HD))
    attn_bwd_dkdv_tc_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmG, const AttnBwdParams p) {
  constexpr int CW = attn_cw(HD);
  constexpr int NCH = HD / CW;
  constexpr int TILE = kBlk * CW * 2;
  constexpr int ST = attn_stages(HD);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smK = base;                        // resident key / value tiles of this CTA
  uint8_t* smV = smK + NCH * TILE;
  uint8_t* smQ = smV + NCH * TILE;            // ST x NCH tiles
  uint8_t* smG = smQ + ST * NCH * TILE;       // ST x NCH tiles of dout
  float* smLD = reinterpret_cast<float*>(smG + ST * NCH * TILE);   // ST x [lse | D] of the 64 queries of a block
  uint64_t* kv_full = reinterpret_cast<uint64_t*>(smLD + ST * 2 * kBlk);
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
      const long long srow = ((long long)n * p.heads + h) * p.L;
      for (int j = 0; j < nqb; ++j) {
        const int s = j % ST;
        mbar_wait(&empty[s], ((j / ST) & 1) ^ 1);
        mbar_expect_tx(&full[s], 2 * NCH * TILE + 2 * kBlk * 4);
        for (int c = 0; c < NCH; ++c) {
          tma_load_3d(smQ + (s * NCH + c) * TILE, &tmQKV, &full[s], h * HD + c * CW, j * kBlk, n);
          tma_load_3d(smG + (s * NCH + c) * TILE, &tmG, &full[s], h * HD + c * CW, j * kBlk, n);
        }
        bulk_load(smLD + s * 2 * kBlk, p.lse + srow + j * kBlk, kBlk * 4, &full[s]);
        bulk_load(smLD + s * 2 * kBlk + kBlk, p.Dbuf + srow + j * kBlk, kBlk * 4, &full[s]);
      }
    }
    return;
  }
  const int g = lane >> 2, t = lane & 3;
  float dv[HD / 2], dk[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  mbar_wait(kv_full, 0);
  for (int j = 0; j < nqb; ++j) {
    const int s = j % ST;
    mbar_wait(&full[s], (j / ST) & 1);
    // per-query operands of the 16 columns this thread holds, from the block's stage
    float lq[16], dq_[16];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float2 l2 = lds_f32x2(smLD + s * 2 * kBlk + 8 * i + 2 * t), d2 = lds_f32x2(smLD + s * 2 * kBlk + kBlk + 8 * i + 2 * t);
      lq[2 * i] = l2.x * 1.4426950408889634f; lq[2 * i + 1] = l2.y * 1.4426950408889634f;
      dq_[2 * i] = d2.x; dq_[2 * i + 1] = d2.y;
    }
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
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      // dV += P^T dout,  dK += dS^T Q   (B = the query-block tiles, MN-major: head_dim contiguous)
      Wgmma<HD>::template rs<1>(dv, pa[kk], make_mnmajor_desc<CW>(g_addr + kk * 16 * (CW * 2), TILE), 1u);
      Wgmma<HD>::template rs<1>(dk, da[kk], make_mnmajor_desc<CW>(q_addr + kk * 16 * (CW * 2), TILE), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&empty[s]);
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
  if (((uintptr_t)a.lse | (uintptr_t)a.dscratch) & 15) {    // the dK/dV kernel bulk-copies lse / D rows
    xu_set_kernel_error("attn_tc: lse and dscratch must be 16-byte aligned");
    return;
  }
  AttnBwdParams p;
  p.res = (const bf16*)a.res; p.out = (const bf16*)a.out; p.dout = (const bf16*)a.dout;
  p.lse = a.lse; p.Dbuf = a.dscratch; p.dqkv = (bf16*)a.dqkv;
  p.L = a.L; p.C = a.C; p.heads = a.heads; p.cross = a.cross;
  p.scale = 1.f / sqrtf((float)HD);
  p.scale_log2 = 1.4426950408889634f * p.scale;
  // both kernels: two resident tiles per chunk + a ring of tile pairs (dK/dV: + the lse / D rows of each stage)
  const size_t smem = (size_t)2 * NCH * TILE + (size_t)2 * attn_stages(HD) * NCH * TILE + 1024 + 256;
  const size_t smem_dkdv = smem + (size_t)attn_stages(HD) * 2 * kBlk * 4;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(attn_bwd_dq_tc_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    cudaFuncSetAttribute(attn_bwd_dkdv_tc_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    configured = true;
  }
  const dim3 grid(a.L / kBlk, a.heads, a.N);
  xu_launch(attn_bwd_dq_tc_kernel<HD>, grid, kAttnThreads, smem, s, tq, tg, p);
  xu_launch(attn_bwd_dkdv_tc_kernel<HD>, grid, kAttnThreads, smem_dkdv, s, tq, tg, p);
  // a caller that keeps its scratch all-zero between calls gets the D rows back cleared
  if (a.scratch_zeroed) cudaMemsetAsync(a.dscratch, 0, sizeof(float) * (size_t)a.N * a.heads * a.L, s);
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
