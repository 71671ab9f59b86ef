// conv_tc.cu -- wgmma / TMA implicit-GEMM convolution for sm_90a (bf16 operands, fp32 accumulate in registers).
//
// Replaces the cuDNN/cuBLAS calls behind flax nn.Conv(3x3, SAME, stride 1) / nn.Dense / nn.DenseGeneral on the
// reference's hot path (model/xunet.py:59,81,85-89,91,100-102) -- forward AND data-gradient.
//
//   D[128 pixels, BN] (registers, fp32)  =  sum over (tap, channel-chunk)  A[128 pixels, BK] (smem)  x  B[BN, BK] (smem)
//
// * A is never materialised as im2col: an M-tile is a TN x TH x TW brick of output pixels of the NHWC tensor and each
//   (tap, chunk) stage is ONE 4-D TMA box load at coordinates (c0, x0+dx-1, y0+dy-1, n0); out-of-bounds rows/cols are
//   zero-filled by the TMA unit, which IS the SAME padding.  The box lands in shared memory in exactly the K-major
//   128B/64B/32B-swizzled layout the GMMA smem descriptor expects.
// * B comes from a bf16 "shadow" of the fp32 master weights, K-major: forward [Co][tap][Ci] (transposed by
//   weight_prep_kernel), data-gradient the plain cast [tap][Ci][Co] (there K = Co is already contiguous).
// * Warp-specialised: warp 8 = TMA producer (one elected lane), warps 0-7 = two consumer warpgroups that issue
//   wgmma.mma_async (64 rows each of every tile, or whole tiles in turn), release ring stages through mbarriers and run the epilogue
//   (+bias (+residual) * alpha -> bf16 -> 16-byte global stores or a TMA store).
#include "conv_tc.h"
#include "tc_common.cuh"

#include <stdio.h>
#include <stdlib.h>

#include <algorithm>

namespace {

struct TcParams {
  int TW, TH, TN, tiles_x, tiles_y;
  int H, W, Co;
  int T, KC, ks, flip, a_seg_stride, b_mode, stride, pad_h, pad_w;
  float alpha;
  int accumulate;
  bf16* y;
  const bf16* res;
  const float* bias;
  int BN, stages;
  int n_tiles, m_tiles, total_tiles;
  int halo;      // 3x3 stride-1: one (TH+2) x TW halo box per (channel chunk, dx) serves the three dy taps
  double* cstats; // fp64 accumulators (xu_det_scratch). EPI 1: per-(sample, channel) [sum, sumsq] of the stored output, (N/2, Co, 2) fp32, accumulated
                 // EPI 2: per-(sample, channel) [sum dyh*xhat, sum dyh] of the GroupNorm backward (same layout)
  const bf16* gx;      // EPI 2: input x of the GroupNorm whose OUTPUT gradient this data-gradient produces, (N,H,W,Co)
  const float4* gnp;   // EPI 2: per-(sample, channel) {rstd, -mean*rstd, gamma, beta} written by the forward gn_apply
  int gn_swish;        // EPI 2: the norm is followed by swish (else plain)
  // EPI 3: the norm is the FiLM one of a ResnetBlock: u = yhat*(1+scale)+shift -> swish -> dropout -> this conv
  const bf16* ge;      // (N,H,W,2*Co) [scale | shift]
  bf16* gde;           // gradient of ge (written: [du*yhat | du])
  float drop_rate; int drop_op; int drop_on; const unsigned long long* seed_dev;
  // output through shared memory + TMA store: the epilogue writes the rounded tile into a swizzled [128 pixels][BN or 64
  // channels] staging buffer (conflict-free 16-byte st.shared) and one thread per buffer issues cp.async.bulk.tensor stores of
  // whole boxes
  int tma_store;
};

// Persistent: each CTA walks tiles  blockIdx.x, blockIdx.x + gridDim.x, ...  (tile = n_tile * m_tiles + m_tile) with the
// smem ring running continuously across tiles; warp 8 is the TMA producer (one elected lane), which fills the ring in tile
// order and runs ahead into the next tile while the consumers drain theirs.  Warps 0-7 are two consumer warpgroups, scheduled
// one of two ways (conv_pingpong):
// * cooperative (BN = 64 and 128): warpgroup wg issues the wgmma for rows 64 wg .. 64 wg + 63 of every tile and then runs
//   the epilogue of those rows.
// * ping-pong (BN = 32, where a tile's few hundred cycles of MMA are dwarfed by its epilogue): warpgroup wg takes whole
//   tiles, the CTA's tiles wg, wg + 2, ..., issuing two m64 wgmmas per k-step (rows 0-63 and 64-127), so that one warpgroup's
//   epilogue (operand loads at DRAM latency, stores, reductions) runs while the other's main loop waits on TMA and the tensor
//   cores.  A ring stage belongs to the warpgroup of its tile.  The main loops take turns in tile order (named barriers
//   4 + wg): a warpgroup starts waiting on the stages of tile j only once the other one has seen every stage of tile j - 1
//   land, so the stage it waits for was last filled for an earlier use that has completed, and the parity of its mbarrier
//   phase cannot alias a phase two uses back.
// The epilogue moves accumulator columns through a shared-memory transpose (fp32, per warpgroup: [64 rows][64 columns]
// cooperative, [128 rows][32 columns] ping-pong) so that a thread owns ONE pixel row and 32 consecutive channels: 16-byte bf16
// stores and per-pixel statistics.
// EPI 1 (forward): the epilogue also emits the GroupNorm input statistics of the tensor it writes (per sample and channel: sum
// and sum of squares of the bf16-rounded outputs), so the consumer norm needs no statistics pass over HBM.
// EPI 2 (data gradient of the conv that consumes a GroupNorm[+swish] output): the epilogue turns dy into the gradient w.r.t.
// the normalised pre-activation, dyh = dy * swish'(xhat*gamma+beta), stores THAT, and emits the per-(sample, channel) sums
// sum(dyh*xhat), sum(dyh) -- the whole first pass of the GroupNorm backward (dgamma, dbeta, group sums) without reading
// x and dy from HBM again (gn_bwd_reduce_kernel disappears for these norms).
// EPI 3: the same for the FiLM norm of a ResnetBlock (model/xunet.py:82-84): dy -> dropout mask -> du = . * swish'(u) with
// u = yhat*(1+scale)+shift, stores dyh = du*(1+scale) and the FiLM gradient [du*yhat | du], emits the same channel sums.
constexpr int kConvThreads = 288;      // two consumer warpgroups + one producer warp
// The ping-pong schedule parks half of a tile's accumulators in registers through the epilogue of the other half once a
// tile has more than one 32-column transpose group: at BN = 64 that does not fit the 96 registers of two CTAs per SM.
__host__ __device__ constexpr bool conv_pingpong(int bn) { return bn < 64; }
// fp32 transpose buffer of one warpgroup: cooperative [64 rows][64 columns] at a pitch of kXP = 68 (16-byte row reads
// without bank conflicts); ping-pong [128 rows][32 columns], either with the 16-byte chunks of row r XOR-swizzled by r % 8
// (the same, in less space than a padded pitch: two CTAs per SM keep their ring depth) or, for the FiLM-backward epilogue
// (EPI 3, one CTA per SM), at a pitch of 36, whose plainer addressing keeps that epilogue within its registers
constexpr int kXP = 68;
__host__ __device__ constexpr int conv_tbuf_floats(int epi, int bn) { return conv_pingpong(bn) ? 128 * (epi == 3 ? 36 : 32) : 64 * kXP; }
__host__ __device__ constexpr int conv_pp_tbuf_at(int epi, int row, int col) {
  return epi == 3 ? row * 36 + col : row * 32 + ((((col >> 2) ^ (row & 7)) << 2) | (col & 3));
}
// Two CTAs per SM (96 registers per thread) for narrow tiles with the plain / statistics epilogues and with the fused
// GroupNorm-backward one (EPI 2, without spills except at BK = 16, BN = 64); the FiLM-backward epilogue (EPI 3) needs more
// registers and runs one CTA per SM.
__host__ __device__ constexpr int conv_ctas_per_sm(int epi, int bn, int bk) {
  return bn <= 64 && (epi < 2 || (epi == 2 && (bn < 64 || bk > 16))) ? 2 : 1;
}
template <int BK, int EPI, int BN>
__global__ void __launch_bounds__(kConvThreads, conv_ctas_per_sm(EPI, BN, BK)) conv_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                               const __grid_constant__ CUtensorMap tmB,
                                                                               const __grid_constant__ CUtensorMap tmY, const TcParams p) {
  extern __shared__ uint8_t smem_raw[];
  constexpr bool PP = conv_pingpong(BN);
  constexpr int NACC = PP ? 2 : 1;                     // m64 accumulator blocks per thread: rows 0-63 and 64-127 (ping-pong)
  constexpr int TBUF = conv_tbuf_floats(EPI, BN);
  // CG accumulator columns per transpose group (= channels of one staged output box), 32 of them per thread
  constexpr int CG = BN < 64 ? BN : 64, CW = 32;
  constexpr int GT = BN / CG * CW;                     // EPI 2/3: norm-table entries per consumer warp (its columns)
  constexpr int B_TILE = BN * BK * 2;
  // halo mode: the A stage holds (TH+2) x TW pixels -- the dy = 0,1,2 operands are the 128-pixel windows starting
  // dy*TW rows in (dy*TW*BK*2 bytes: a whole number of swizzle atoms since TW % 8 == 0) -- and the B stage the 3 dy taps
  const int A_BYTES = p.halo ? (p.TH + 2) * p.TW * BK * 2 : 128 * BK * 2;
  const int B_BYTES = p.halo ? 3 * B_TILE : B_TILE;
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smA = base;
  uint8_t* smB = base + (size_t)p.stages * A_BYTES;
  uint8_t* smY = smB + (size_t)p.stages * B_BYTES;                       // 2 x [128][CG] bf16 staging (tma_store only)
  // a data gradient stages its tile only to accumulate, which the fused GroupNorm-backward epilogues (EPI 2/3) never do:
  // compiling the staging out of them keeps it from costing them registers
  const bool tma_store = EPI < 2 && p.tma_store;
  const int Y_BYTES = tma_store ? 128 * CG * 2 : 0;
  float* smT = reinterpret_cast<float*>(smY + 2 * (size_t)Y_BYTES);      // 2 x TBUF fp32 transpose buffers
  uint64_t* full = reinterpret_cast<uint64_t*>(smT + 2 * TBUF);
  uint64_t* empty = full + p.stages;
  // EPI 2/3: per consumer warp, the {rstd, -mean*rstd, gamma, beta} entries of the GT columns it handles in a tile
  float4* smG = reinterpret_cast<float4*>(empty + p.stages) + (threadIdx.x >> 5) * GT;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_k = p.halo ? 3 * p.KC : p.T * p.KC;

  if (threadIdx.x == 0) {
    // one arrival per consumer warp that reads the stage: both warpgroups (cooperative) or the tile's (ping-pong)
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], PP ? 4 : 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    if (tma_store) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmY) : "memory");
  }
  __syncthreads();
  xu_grid_dep_sync();     // PDL: everything above (barriers) overlaps the previous kernel's tail

  if (warp == 8) {
    if (lane == 0) {
      // ===== TMA producer =====
      int itg = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        // m fastest: the CTAs running at the same time share one weight slab (n_tile) in L2
        const int n_tile = tile / p.m_tiles;
        int t = tile - n_tile * p.m_tiles;
        const int tx = t % p.tiles_x; t /= p.tiles_x;
        const int ty = t % p.tiles_y; t /= p.tiles_y;
        const int x0 = tx * p.TW, y0 = ty * p.TH, n0 = t * p.TN;
        for (int it = 0; it < total_k; ++it, ++itg) {
          const int s = itg % p.stages;
          const uint32_t ph = (itg / p.stages) & 1;
          mbar_wait(&empty[s], ph ^ 1);
          const int tt = it / p.KC, c = it - tt * p.KC;
          if (p.halo) {
            // tt = dx column of the stencil; rows y0-1 .. y0+TH of the input column x0+ox.. arrive in one box
            const int ox = p.flip ? 1 - tt : tt - 1;
            mbar_expect_tx(&full[s], A_BYTES + B_BYTES);
            tma_load_4d(smA + (size_t)s * A_BYTES, &tmA, &full[s], c * BK, x0 + ox, y0 - 1, n0);
#pragma unroll
            for (int j = 0; j < 3; ++j) {            // window j starts at input row y0 - 1 + j  <->  dy = j (dgrad: 2 - j)
              const int tap = (p.flip ? 2 - j : j) * 3 + tt;
              uint8_t* dst = smB + (size_t)s * B_BYTES + j * B_TILE;
              if (p.b_mode == 0) tma_load_3d(dst, &tmB, &full[s], c * BK, tap, n_tile * BN);
              else tma_load_3d(dst, &tmB, &full[s], c * BK, n_tile * BN, tap);
            }
            continue;
          }
          int ox = 0, oy = 0;
          if (p.ks == 3) {
            const int dy = tt / 3, dx = tt - dy * 3;
            oy = p.flip ? 1 - dy : dy - p.pad_h;
            ox = p.flip ? 1 - dx : dx - p.pad_w;
          }
          mbar_expect_tx(&full[s], A_BYTES + B_BYTES);
          tma_load_4d(smA + (size_t)s * A_BYTES, &tmA, &full[s], tt * p.a_seg_stride + c * BK, x0 * p.stride + ox, y0 * p.stride + oy, n0);
          if (p.b_mode == 0) tma_load_3d(smB + (size_t)s * B_BYTES, &tmB, &full[s], c * BK, tt, n_tile * BN);
          else tma_load_3d(smB + (size_t)s * B_BYTES, &tmB, &full[s], c * BK, n_tile * BN, tt);
        }
      }
    }
  } else {
    const int wg = warp >> 2;                            // consumer warpgroup
    const int wq = warp & 3;
    // epilogue mapping: warp wq of the warpgroup owns pixel rows lane_base .. +31 of the tile; cooperative, it takes the
    // 32-column half `ehalf` of every 64-column group of the warpgroup's 64 rows, ping-pong every column of its 32 rows
    const int ehalf = PP ? 0 : wq >> 1;
    const bool bias_vec = (reinterpret_cast<uintptr_t>(p.bias) & 15) == 0;   // leaf offsets are 16-byte aligned in the flat buffer; scalar loads otherwise
    const int lane_base = PP ? wq * 32 : wg * 64 + (wq & 1) * 32;
    const int r = lane_base + lane;                      // row of the 128-pixel tile
    // pixel offset of row r from the tile's first pixel (one register across the tile loop instead of three coordinates)
    const unsigned rofs = (unsigned)((((r / (p.TW * p.TH)) * p.H + (r / p.TW) % p.TH) * p.W + r % p.TW));
    float* tbuf = smT + wg * TBUF;
    const int tr = PP ? r : r - wg * 64;                 // row of the transpose buffer
    const int fr = wq * 16 + (lane >> 2), fc = (lane & 3) * 2;   // accumulator fragment: rows fr, fr + 8; columns 8 i + fc, + 1
    // the thread that issues / retires the TMA stores of a staging buffer: one per warpgroup (ping-pong) or per CTA
    const bool y_issuer = (threadIdx.x & (PP ? 127 : 255)) == 0;
    const int yswz = CG == 64 ? (r & 7) : ((r >> 1) & 3);
    int ybox = 0;                                         // running count of staging boxes (cooperative: selects the buffer)
    float acc[NACC][BN / 2];
    // jt: the tile's index in the CTA's sequence, which fixes its ring iterations jt * total_k ..
    for (int tile = blockIdx.x + (PP ? wg * gridDim.x : 0), jt = PP ? wg : 0; tile < p.total_tiles;
         tile += (PP ? 2 : 1) * gridDim.x, jt += PP ? 2 : 1) {
      // ===== main loop: wgmma over the ring =====
      if (PP && jt > 0) named_bar_sync(4 + wg, 256);    // the other warpgroup has seen every stage of tile jt - 1 land
      int itg = jt * total_k;
      int prev_s = 0;
      for (int it = 0; it < total_k; ++it, ++itg) {
        const int s = itg % p.stages;
        mbar_wait(&full[s], (itg / p.stages) & 1);
        wgmma_fence();
        const uint32_t b_addr = smem_u32(smB + (size_t)s * B_BYTES);
#pragma unroll
        for (int m = 0; m < NACC; ++m) {
          const uint32_t a_addr = smem_u32(smA + (size_t)s * A_BYTES) + (uint32_t)((PP ? m : wg) * 64 * BK * 2);
          if (p.halo) {
            const uint32_t win = (uint32_t)(p.TW * BK * 2);
#pragma unroll
            for (int j = 0; j < 3; ++j)
#pragma unroll
              for (int k = 0; k < BK / 16; ++k)
                Wgmma<BN>::template ss<0, 0>(acc[m], make_kmajor_desc<BK>(a_addr + j * win + k * 32),
                                             make_kmajor_desc<BK>(b_addr + j * B_TILE + k * 32), (it > 0 || j > 0 || k > 0) ? 1u : 0u);
          } else {
#pragma unroll
            for (int k = 0; k < BK / 16; ++k)
              Wgmma<BN>::template ss<0, 0>(acc[m], make_kmajor_desc<BK>(a_addr + k * 32), make_kmajor_desc<BK>(b_addr + k * 32),
                                           (it > 0 || k > 0) ? 1u : 0u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                                 // the previous step's MMAs are done: release its stage
        if (it > 0 && lane == 0) mbar_arrive(&empty[prev_s]);
        prev_s = s;
      }
      if (PP && tile + gridDim.x < p.total_tiles) named_bar_arrive(4 + (wg ^ 1), 256);
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&empty[prev_s]);

      // ===== epilogue =====
      const int n_tile = tile / p.m_tiles;
      int t = tile - n_tile * p.m_tiles;
      const int tx = t % p.tiles_x; t /= p.tiles_x;
      const int ty = t % p.tiles_y; t /= p.tiles_y;
      const int x0 = tx * p.TW, y0 = ty * p.TH, n0 = t * p.TN;
      const long long pix = ((long long)n0 * p.H + y0) * p.W + x0 + rofs;
      bf16* yrow = p.y + pix * p.Co + (long long)n_tile * BN;
      const bf16* rrow = p.res ? p.res + pix * p.Co + (long long)n_tile * BN : nullptr;
      const float* brow = EPI < 2 && p.bias ? p.bias + (long long)n_tile * BN : nullptr;   // a data gradient has no bias
      // The thread's CW columns of a group have their operands held in registers SW at a time: the fused GroupNorm-backward
      // epilogues take 8-column sub-chunks (x, the FiLM operands and the statistics partials of 16 channels live at once),
      // the ping-pong plain / statistics ones 16 columns: this lets them run two CTAs per SM without spilling.
      constexpr int SW = EPI >= 2 ? 8 : (PP ? 16 : CW);
      // STATS: the 32 pixels of this warp belong to one sample (host-checked): b = image of the warp's first row / 2
      double* cs_row = nullptr;
      const long long srow = (long long)((n0 + lane_base / (p.TW * p.TH)) >> 1) * p.Co + (long long)n_tile * BN;
      if constexpr (EPI != 0) cs_row = p.cstats + srow * 2;
      const bf16* gxrow = nullptr;
      const float4* gprow = nullptr;
      if constexpr (EPI >= 2) {
        gxrow = p.gx + pix * p.Co + (long long)n_tile * BN; gprow = p.gnp + srow;
        // stage the norm table of this warp's columns (entry cc / 2 + k <-> column cc + ehalf * CW + k) once per tile: read
        // from shared memory in the column loop instead of being held in registers
        __syncwarp();                   // the warp's reads of the previous tile's entries are done
        for (int k = lane; k < GT; k += 32) smG[k] = __ldg(gprow + (k / CW) * CG + ehalf * CW + k % CW);
        __syncwarp();
      }
      const bf16* gerow = nullptr;
      bf16* gderow = nullptr;
      unsigned long long dseed = 0ULL;
      if constexpr (EPI == 3) {
        gerow = p.ge + pix * (2LL * p.Co) + (long long)n_tile * BN;
        gderow = p.gde + pix * (2LL * p.Co) + (long long)n_tile * BN;
        if (p.drop_on) dseed = *p.seed_dev;
      }
#pragma unroll
      for (int cc = 0; cc < BN; cc += CG) {
        // accumulator columns cc .. cc + CG - 1 of this warpgroup's rows -> transpose buffer
#pragma unroll
        for (int m = 0; m < NACC; ++m) {
#pragma unroll
          for (int i = 0; i < BN / 2; i += 4) {
            const int col = 8 * (i / 4);
            if (col >= cc && col < cc + CG) {
              float* t0 = PP ? tbuf + conv_pp_tbuf_at(EPI, m * 64 + fr, col - cc + fc) : tbuf + fr * kXP + col - cc + fc;
              float* t1 = PP ? tbuf + conv_pp_tbuf_at(EPI, m * 64 + fr + 8, col - cc + fc) : tbuf + (fr + 8) * kXP + col - cc + fc;
              *reinterpret_cast<float2*>(t0) = make_float2(acc[m][i], acc[m][i + 1]);
              *reinterpret_cast<float2*>(t1) = make_float2(acc[m][i + 2], acc[m][i + 3]);
            }
          }
        }
        named_bar_sync(2 + wg, 128);
        float sx[32];     // STATS only (dead otherwise)
#pragma unroll
        for (int h = 0; h < CW; h += SW) {
        const int c0 = cc + ehalf * CW + h;
        const bool active = c0 < BN;
        // the residual operands of the whole sub-chunk are requested before anything waits on them: each is a 16-byte
        // access of a (pixel-pitch strided) row, i.e. a DRAM-latency load per thread when issued one by one
        uint4 rv[SW / 8];
        if (active && EPI < 2 && rrow) {
#pragma unroll
          for (int q = 0; q < SW / 8; ++q) rv[q] = __ldg(reinterpret_cast<const uint4*>(rrow + c0 + 8 * q));
        }
        if constexpr (EPI >= 2) {      // the GroupNorm input of this pixel (rv is free: a data gradient has no residual operand)
          if (active) {
#pragma unroll
            for (int q = 0; q < SW / 8; ++q) rv[q] = __ldg(reinterpret_cast<const uint4*>(gxrow + c0 + 8 * q));
          }
        }
        uint4 scv[SW / 8], shv[SW / 8];
        if constexpr (EPI == 3) {
          if (active) {
#pragma unroll
            for (int q = 0; q < SW / 8; ++q) {
              scv[q] = __ldg(reinterpret_cast<const uint4*>(gerow + c0 + 8 * q));
              shv[q] = __ldg(reinterpret_cast<const uint4*>(gerow + p.Co + c0 + 8 * q));
            }
          }
        }
        float v[SW];
        if (active) {
#pragma unroll
          for (int q = 0; q < SW / 4; ++q) {
            const float* t = PP ? tbuf + conv_pp_tbuf_at(EPI, tr, h + 4 * q) : tbuf + tr * kXP + ehalf * CW + h + 4 * q;
            const float4 t4 = *reinterpret_cast<const float4*>(t);
            v[4 * q] = t4.x; v[4 * q + 1] = t4.y; v[4 * q + 2] = t4.z; v[4 * q + 3] = t4.w;
          }
        }
        // staging buffer: the warpgroup's own (ping-pong), or the CTA's two in turn
        uint8_t* yst = smY + (size_t)(PP ? wg : (ybox & 1)) * Y_BYTES + (size_t)r * (CG * 2);
        if (tma_store && h == 0) {
          // the store that last read this staging buffer must have finished reading before it is overwritten
          if (y_issuer) { if constexpr (PP) bulk_wait_group_read<0>(); else bulk_wait_group_read<1>(); }
          if constexpr (PP) named_bar_sync(2 + wg, 128); else named_bar_sync(1, 256);
        }
        if (active) {
#pragma unroll
          for (int j = 0; j < SW; j += 8) {
            float f[8];
            {
              float4 bq0 = make_float4(0.f, 0.f, 0.f, 0.f), bq1 = bq0;
              if (brow && bias_vec) { bq0 = __ldg(reinterpret_cast<const float4*>(brow + c0 + j)); bq1 = __ldg(reinterpret_cast<const float4*>(brow + c0 + j) + 1); }
              else if (brow) { bq0 = make_float4(brow[c0 + j], brow[c0 + j + 1], brow[c0 + j + 2], brow[c0 + j + 3]); bq1 = make_float4(brow[c0 + j + 4], brow[c0 + j + 5], brow[c0 + j + 6], brow[c0 + j + 7]); }
              const float bq[8] = {bq0.x, bq0.y, bq0.z, bq0.w, bq1.x, bq1.y, bq1.z, bq1.w};
#pragma unroll
              for (int q = 0; q < 8; ++q) f[q] = v[j + q] + bq[q];
            }
            if (EPI < 2 && rrow) {
              const __nv_bfloat162* r2 = reinterpret_cast<const __nv_bfloat162*>(&rv[j >> 3]);
#pragma unroll
              for (int q = 0; q < 4; ++q) { f[2 * q] += __low2float(r2[q]); f[2 * q + 1] += __high2float(r2[q]); }
            }
#pragma unroll
            for (int q = 0; q < 8; ++q) f[q] *= p.alpha;
            float xh[8];
            if constexpr (EPI == 2) {
              const __nv_bfloat162* x2 = reinterpret_cast<const __nv_bfloat162*>(&rv[j >> 3]);
#pragma unroll
              for (int q = 0; q < 8; ++q) {
                const float4 pp = smG[(cc / CG) * CW + h + j + q];
                const float xv = (q & 1) ? __high2float(x2[q >> 1]) : __low2float(x2[q >> 1]);
                xh[q] = fmaf(xv, pp.x, pp.y);
                if (p.gn_swish) f[q] *= swish_gradf_(fmaf(xh[q], pp.z, pp.w));
              }
            }
            if constexpr (EPI == 3) {
              const __nv_bfloat162* x2 = reinterpret_cast<const __nv_bfloat162*>(&rv[j >> 3]);
              const __nv_bfloat162* s2 = reinterpret_cast<const __nv_bfloat162*>(&scv[j >> 3]);
              const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&shv[j >> 3]);
              const long long e0 = pix * p.Co + (long long)n_tile * BN + c0 + j;      // element index of column j in (N,H,W,Co)
              uint32_t km = 0xFFu;
              if (p.drop_on) km = xu_keep4(dseed, p.drop_op, (unsigned long long)e0 >> 2, p.drop_rate) |
                                  (xu_keep4(dseed, p.drop_op, ((unsigned long long)e0 >> 2) + 1, p.drop_rate) << 4);
              const float keep_scale = 1.f / (1.f - p.drop_rate);
              uint4 dsc, dsh;
              __nv_bfloat162* dsc2 = reinterpret_cast<__nv_bfloat162*>(&dsc);
              __nv_bfloat162* dsh2 = reinterpret_cast<__nv_bfloat162*>(&dsh);
              float tsc[8], tsh[8];
#pragma unroll
              for (int q = 0; q < 8; ++q) {
                const float4 pp = smG[(cc / CG) * CW + h + j + q];
                const float xv = (q & 1) ? __high2float(x2[q >> 1]) : __low2float(x2[q >> 1]);
                const float sc = (q & 1) ? __high2float(s2[q >> 1]) : __low2float(s2[q >> 1]);
                const float sh = (q & 1) ? __high2float(h2[q >> 1]) : __low2float(h2[q >> 1]);
                xh[q] = fmaf(xv, pp.x, pp.y);
                const float yh = fmaf(xh[q], pp.z, pp.w);
                const float u = fmaf(yh, 1.f + sc, sh);
                float gs = f[q];
                if (p.drop_on) gs = ((km >> q) & 1u) ? gs * keep_scale : 0.f;
                const float du = gs * swish_gradf_(u);
                f[q] = du * (1.f + sc);
                tsc[q] = du * yh;
                tsh[q] = du;
              }
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                dsc2[q] = __floats2bfloat162_rn(tsc[2 * q], tsc[2 * q + 1]);
                dsh2[q] = __floats2bfloat162_rn(tsh[2 * q], tsh[2 * q + 1]);
              }
              *reinterpret_cast<uint4*>(gderow + c0 + j) = dsc;
              *reinterpret_cast<uint4*>(gderow + p.Co + c0 + j) = dsh;
            }
            uint4 outv;
            __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&outv);
#pragma unroll
            for (int q = 0; q < 4; ++q) o2[q] = __floats2bfloat162_rn(f[2 * q], f[2 * q + 1]);
            if (tma_store) sts128(yst + ((((ehalf * CW + h + j) >> 3) ^ yswz) << 4), outv);
            else *reinterpret_cast<uint4*>(yrow + c0 + j) = outv;
            if constexpr (EPI >= 2) {
              // sums over what is STORED (the second pass reads the rounded dyh back)
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const float a = __low2float(o2[q]), b = __high2float(o2[q]);
                sx[((h + j) & 8) + 2 * q] = a * xh[2 * q];   sx[((h + j) & 8) + 2 * q + 1] = b * xh[2 * q + 1];
                sx[16 + ((h + j) & 8) + 2 * q] = a;          sx[16 + ((h + j) & 8) + 2 * q + 1] = b;
              }
              if ((h + j) & 8) xu_cstats_emit16(sx, lane, cs_row + (c0 + j - 8) * 2);
            }
            if constexpr (EPI == 1) {
              // statistics of what is STORED (rounded), so the consumer's normalisation is exactly zero-mean / unit-variance
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const float a = __low2float(o2[q]), b = __high2float(o2[q]);
                sx[((h + j) & 8) + 2 * q] = a;            sx[((h + j) & 8) + 2 * q + 1] = b;
                sx[16 + ((h + j) & 8) + 2 * q] = a * a;   sx[16 + ((h + j) & 8) + 2 * q + 1] = b * b;
              }
              if ((h + j) & 8) xu_cstats_emit16(sx, lane, cs_row + (c0 + j - 8) * 2);
            }
          }
        }
        }
        if (tma_store) {
          fence_async_smem();                 // generic-proxy writes -> visible to the TMA unit
          if constexpr (PP) named_bar_sync(2 + wg, 128); else named_bar_sync(1, 256);
          if (y_issuer) {
            uint8_t* ybuf = smY + (size_t)(PP ? wg : (ybox & 1)) * Y_BYTES;
            // accumulate: the gradient is ADDED to the destination by the TMA unit (cp.reduce.async.bulk.tensor .add, bf16 at L2)
            if (p.accumulate) tma_reduce_add_4d(ybuf, &tmY, n_tile * BN + cc, x0, y0, n0);
            else tma_store_4d(ybuf, &tmY, n_tile * BN + cc, x0, y0, n0);
            bulk_commit_group();
          }
          ++ybox;
        }
        named_bar_sync(2 + wg, 128);        // transpose buffer read by every warp before the next group overwrites it
      }
    }
    if (tma_store && y_issuer) bulk_wait_group<0>();   // all output boxes written before the CTA retires
  }
}

// ---------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

}  // namespace
bool xu_encode_bf16_map(CUtensorMap* m, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                        const uint32_t* box, int bk, const uint32_t* elem_strides) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { xu_set_kernel_error("conv_tc: cuTensorMapEncodeTiled unavailable"); return false; }
  cuuint64_t gd[5]; cuuint64_t gs[4]; cuuint32_t bx[5]; cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = elem_strides ? elem_strides[i] : 1; }
  for (int i = 0; i + 1 < rank; ++i) gs[i] = strides_bytes[i];
  CUtensorMapSwizzle sw = bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (bk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), gd, gs, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[160];
    snprintf(buf, sizeof(buf), "conv_tc: cuTensorMapEncodeTiled failed (%d) rank %d dims %llu,%llu,%llu box %u,%u,%u", (int)r, rank,
             (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], box[0], box[1], box[2]);
    xu_set_kernel_error(buf);
    return false;
  }
  return true;
}
namespace {
#define encode_bf16 xu_encode_bf16_map

bool pick_tile(int N, int H, int W, int& TW, int& TH, int& TN) {
  if (W >= 128) {
    if (W % 128) return false;
    TW = 128; TH = 1; TN = 1;
    return true;
  }
  if (128 % W) return false;
  TW = W;
  int rem = 128 / W;
  if (H >= rem) {
    if (H % rem) return false;
    TH = rem; TN = 1;
    return true;
  }
  if (rem % H) return false;
  TH = H; TN = rem / H;
  return N % TN == 0;
}

// K-chunk width (= swizzle span / 2 bytes).  K that is a multiple of 16 but not of 32 (the 144 pose-embedding channels)
// uses 64-wide chunks with the tail zero-filled by TMA (both the activation box and the weight-shadow box run out of bounds
// together), which beats 16-wide chunks by 3x fewer pipeline stages.
int pick_bk(int K) { return K % 64 == 0 ? 64 : (K % 32 == 0 ? 32 : (K % 16 == 0 ? (K > 64 ? 64 : 16) : 0)); }

template <int BK, int EPI, int BN>
void launch_tc_bn(const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& y, const TcParams& p, size_t smem, dim3 grid, cudaStream_t s) {
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(conv_tc_kernel<BK, EPI, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    configured = true;
  }
  xu_launch(conv_tc_kernel<BK, EPI, BN>, grid, kConvThreads, smem, s, a, b, y, p);
}
template <int BK, int EPI>
void launch_tc(const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& y, const TcParams& p, size_t smem, dim3 grid, cudaStream_t s) {
  switch (p.BN) {
    case 128: launch_tc_bn<BK, EPI, 128>(a, b, y, p, smem, grid, s); break;
    case 64: launch_tc_bn<BK, EPI, 64>(a, b, y, p, smem, grid, s); break;
    default: launch_tc_bn<BK, EPI, 32>(a, b, y, p, smem, grid, s); break;
  }
}

}  // namespace

// ---- bf16 shadow of the fp32 master weights -----------------------------------------------------------------
// forward : wT[co][tap][ci]            (co over all segments)         from  w[seg][tap][ci][segw]
// dgrad   : wC = plain cast, same index order as the master ([seg|tap][ci][segw])
__global__ void __launch_bounds__(256) weight_prep_kernel(const float* __restrict__ params, uint8_t* __restrict__ ws,
                                                          const __grid_constant__ WeightPrepTable tab) {
  xu_grid_dep_sync();
  // one block = one 64 (ci) x 64 (co) tile of one (segment, tap) slab: 16-byte reads along co, 8-byte writes of the plain cast,
  // 16-byte writes of the transposed shadow along ci.
  __shared__ float tile[64][65];
  const long long t = blockIdx.x;
  int lo = 0, hi = tab.n - 1;
  while (lo < hi) {            // last entry with tprefix <= t
    int mid = (lo + hi + 1) >> 1;
    if (tab.e[mid].tprefix <= t) lo = mid; else hi = mid - 1;
  }
  const WeightPrepEntry& e = tab.e[lo];
  const int segw = e.Co / e.nseg;
  const int tco = (segw + 63) >> 6, tci = (e.Ci + 63) >> 6;
  long long r = t - e.tprefix;
  const int bco = (int)(r % tco); r /= tco;
  const int bci = (int)(r % tci); r /= tci;
  const int tap = (int)(r % e.taps);
  const int seg = (int)(r / e.taps);
  const long long base = ((long long)(seg * e.taps + tap) * e.Ci) * segw;      // master order [seg][tap][ci][segw]
  const bool vecR = (segw & 3) == 0 && (e.src & 3) == 0 && (e.dstC < 0 || (e.dstC & 7) == 0);
  const bool vecT = (e.Ci & 7) == 0 && (e.dstT & 15) == 0;
  bf16* const dC = e.dstC >= 0 ? reinterpret_cast<bf16*>(ws + e.dstC) : nullptr;
  bf16* const dT = e.dstT >= 0 ? reinterpret_cast<bf16*>(ws + e.dstT) : nullptr;
  if (vecR) {
    const int c4 = (threadIdx.x & 15) << 2;
    const int co = bco * 64 + c4;
#pragma unroll
    for (int pass = 0; pass < 4; ++pass) {
      const int row = pass * 16 + (threadIdx.x >> 4);
      const int ci = bci * 64 + row;
      if (ci < e.Ci && co < segw) {
        const long long i = base + (long long)ci * segw + co;
        const float4 v = __ldg(reinterpret_cast<const float4*>(params + e.src + i));
        tile[row][c4] = v.x; tile[row][c4 + 1] = v.y; tile[row][c4 + 2] = v.z; tile[row][c4 + 3] = v.w;
        if (dC) {
          __nv_bfloat162 lo2 = __floats2bfloat162_rn(v.x, v.y), hi2 = __floats2bfloat162_rn(v.z, v.w);
          uint2 o;
          o.x = *reinterpret_cast<uint32_t*>(&lo2); o.y = *reinterpret_cast<uint32_t*>(&hi2);
          *reinterpret_cast<uint2*>(dC + i) = o;
        }
      }
    }
  } else {
    for (int idx = threadIdx.x; idx < 64 * 64; idx += 256) {
      const int row = idx >> 6, col = idx & 63;
      const int ci = bci * 64 + row, co = bco * 64 + col;
      if (ci < e.Ci && co < segw) {
        const long long i = base + (long long)ci * segw + co;
        const float v = params[e.src + i];
        tile[row][col] = v;
        if (dC) dC[i] = __float2bfloat16_rn(v);
      }
    }
  }
  __syncthreads();
  if (!dT) return;
  if (vecT) {
    const int ci8 = (threadIdx.x & 7) << 3;
    const int ci = bci * 64 + ci8;
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
      const int col = pass * 32 + (threadIdx.x >> 3);
      const int co = bco * 64 + col;
      if (ci < e.Ci && co < segw) {
        uint4 o;
        __nv_bfloat162 p0 = __floats2bfloat162_rn(tile[ci8][col], tile[ci8 + 1][col]);
        __nv_bfloat162 p1 = __floats2bfloat162_rn(tile[ci8 + 2][col], tile[ci8 + 3][col]);
        __nv_bfloat162 p2 = __floats2bfloat162_rn(tile[ci8 + 4][col], tile[ci8 + 5][col]);
        __nv_bfloat162 p3 = __floats2bfloat162_rn(tile[ci8 + 6][col], tile[ci8 + 7][col]);
        o.x = *reinterpret_cast<uint32_t*>(&p0); o.y = *reinterpret_cast<uint32_t*>(&p1);
        o.z = *reinterpret_cast<uint32_t*>(&p2); o.w = *reinterpret_cast<uint32_t*>(&p3);
        *reinterpret_cast<uint4*>(dT + ((long long)(seg * segw + co) * e.taps + tap) * e.Ci + ci) = o;
      }
    }
  } else {
    for (int idx = threadIdx.x; idx < 64 * 64; idx += 256) {
      const int col = idx >> 6, row = idx & 63;
      const int ci = bci * 64 + row, co = bco * 64 + col;
      if (ci < e.Ci && co < segw) dT[((long long)(seg * segw + co) * e.taps + tap) * e.Ci + ci] = __float2bfloat16_rn(tile[row][col]);
    }
  }
}

void launch_weight_prep(const WeightPrepTable& tab_in, const float* params, void* ws, cudaStream_t s) {
  if (tab_in.n == 0) return;
  WeightPrepTable tab = tab_in;
  long long tiles = 0;
  for (int i = 0; i < tab.n; ++i) {
    WeightPrepEntry& e = tab.e[i];
    e.tprefix = tiles;
    const int segw = e.Co / e.nseg;
    tiles += (long long)e.nseg * e.taps * ((e.Ci + 63) / 64) * ((segw + 63) / 64);
  }
  xu_launch(weight_prep_kernel, (unsigned)tiles, 256, 0, s, params, reinterpret_cast<uint8_t*>(ws), tab);
}

bool conv_tc_supported(int dtype, int mode, int N, int H, int W, int Ci, int Co, int ks, int stride, int nseg) {
  if (dtype != XU_BF16 || (ks != 1 && ks != 3)) return false;
  if (stride != 1 && (mode != 0 || ks != 3)) return false;    // strided: forward 3x3 only (the pose-embedding convs)
  if (nseg != 1 && ks != 1) return false;
  int TW, TH, TN;
  // H, W are the INPUT dims; the tile is a brick of OUTPUT pixels (SAME: out = ceil(in / stride))
  if (!pick_tile(N, (H + stride - 1) / stride, (W + stride - 1) / stride, TW, TH, TN)) return false;
  if (TW * stride > 256 || TH * stride > 256) return false;
  // GEMM K / N of this mode
  const int K = mode == 0 ? Ci : Co / nseg;
  const int Nn = mode == 0 ? Co : Ci;
  if (pick_bk(K) == 0) return false;
  if (nseg > 1 && K % pick_bk(K) != 0) return false;   // zero-filled tail chunks only without segments
  if (Nn % 32 != 0) return false;
  if (Nn > 256 && Nn % 256 != 0) return false;
  if (Ci % 8 != 0 || Co % 8 != 0) return false;   // 16-byte global strides for the tensor maps / vector epilogue
  return true;
}

// Can the epilogue emit per-(sample, channel) statistics?  Every epilogue warp (32 consecutive rows of the 128-pixel tile) must
// lie inside ONE sample: tiles of >= 32 pixels per image always do; 16-pixel images do when a tile holds whole frame pairs.
bool conv_tc_stats_supported(int mode, int N, int Ho, int Wo) {
  (void)mode;      // forward statistics (mode 0) and the fused GroupNorm backward of a data gradient (mode 1) share the rule
  int TW, TH, TN;
  if (!pick_tile(N, Ho, Wo, TW, TH, TN)) return false;
  // (the halo variant re-tiles to 8 x 16 pixels inside one image: always fine)
  return TW * TH >= 32 || (TW * TH == 16 && TN % 2 == 0);
}

// a: the generic ConvArgs (mode 0 forward: x -> y;  mode 1 dgrad: a.x = dY (N,H,W,wCo), a.y = dX (N,H,W,wCi)).
// wshadow: forward -> wT [wCo][taps][wCi];  dgrad -> wC [seg|tap][wCi][segw]
// N-split rule: BN is halved while the tile count stays below a threshold, in quarters of the SM count: with a long reduction a
// narrower tile only pays under 3/4 of a wave (the narrow MMA is bound by fetching A), short reductions are latency-bound and take
// the full-wave rule.
static int bn_rule(int bn, int k_total) { return (bn > 128 || k_total < 2048) ? 4 : 3; }

static void launch_conv_tc_impl(const ConvArgs& a, const void* wshadow, double* cacc, cudaStream_t s) {
  const int taps = a.ks * a.ks;
  const int nseg = a.wCo / a.segw;
  int TW, TH, TN;
  if (!pick_tile(a.N, a.Ho, a.Wo, TW, TH, TN)) { xu_set_kernel_error("conv_tc: unsupported spatial shape"); return; }
  // halo mode (see the kernel): 3x3, stride 1, SAME, 8 x 16-pixel tiles inside one image; it reads the input 3.75x per
  // output tile instead of 9x (small-channel convolutions are L2-bandwidth-bound on the tap re-reads) and needs a third
  // of the pipeline steps.
  bool halo = a.ks == 3 && a.stride == 1 && nseg == 1 && a.pad_h == 1 && a.pad_w == 1 && a.Wo % 16 == 0 && a.Ho % 8 == 0 &&
              a.Hi == a.Ho && a.Wi == a.Wo;
  TcParams p;
  p.TW = TW; p.TH = TH; p.TN = TN; p.tiles_x = a.Wo / TW; p.tiles_y = a.Ho / TH;
  p.H = a.Ho; p.W = a.Wo; p.Co = a.Co;
  p.ks = a.ks; p.alpha = a.alpha; p.accumulate = a.accumulate;
  p.stride = a.stride; p.pad_h = a.pad_h; p.pad_w = a.pad_w;
  p.y = reinterpret_cast<bf16*>(a.y); p.res = reinterpret_cast<const bf16*>(a.res); p.bias = a.bias;
  int bk;
  CUtensorMap tmA, tmB;
  const int Ca = a.Ci;  // channels of the A-side tensor
  const int Kdim = a.mode == 0 ? a.wCi : a.segw;      // reduction channels per tap (and segment)
  const int Ndim = a.mode == 0 ? a.wCo : a.wCi;       // GEMM N
  bk = pick_bk(Kdim);
  // wgmma N of the kernel: 128, 64 or 32 (the largest that divides the GEMM N).  A 256-column tile would need 128 accumulator
  // registers per thread next to the epilogue's: ptxas caps this 9-warp kernel at 168 and spills ~10 KB per thread.
  p.BN = Ndim % 128 == 0 ? 128 : (Ndim % 64 == 0 ? 64 : 32);
  // small problems are latency-bound: split N so that at least ~one wave of CTAs exists
  { const long long mt = (long long)p.tiles_x * p.tiles_y * (a.N / TN);
    while (p.BN >= 64 && (p.BN / 2) % 32 == 0 && mt * (a.Co / p.BN) * 4 < xu_num_sms() * bn_rule(p.BN, taps * Kdim)) p.BN /= 2; }
  // the halo stage (A: 160 pixels, B: 3 taps) must leave room for a >= 3-deep ring; a 32-channel stage keeps the halo trick for the
  // widest tiles, so the activation tile is fetched 3.75x instead of 9x per output tile (wide convolutions are bound by the L2->SM
  // operand stream).
  if (halo && (size_t)(160 * bk * 2 + 3 * p.BN * bk * 2) > (size_t)56 * 1024) {
    if (bk == 64 && (size_t)(160 * 32 * 2 + 3 * p.BN * 32 * 2) <= (size_t)72 * 1024) bk = 32;
    else halo = false;
  }
  if (a.mode == 0) {
    p.T = taps; p.KC = (a.wCi + bk - 1) / bk; p.flip = 0; p.a_seg_stride = 0; p.b_mode = 0;
    uint64_t bd[3] = {(uint64_t)a.wCi, (uint64_t)taps, (uint64_t)a.wCo};
    uint64_t bs[2] = {(uint64_t)a.wCi * 2, (uint64_t)taps * a.wCi * 2};
    uint32_t bb[3] = {(uint32_t)bk, 1u, (uint32_t)p.BN};
    if (!encode_bf16(&tmB, wshadow, 3, bd, bs, bb, bk)) return;
  } else {
    p.T = taps * nseg; p.KC = (a.segw + bk - 1) / bk; p.flip = 1; p.a_seg_stride = nseg > 1 ? a.segw : 0; p.b_mode = 1;
    uint64_t bd[3] = {(uint64_t)a.segw, (uint64_t)a.wCi, (uint64_t)(taps * nseg)};
    uint64_t bs[2] = {(uint64_t)a.segw * 2, (uint64_t)a.wCi * a.segw * 2};
    uint32_t bb[3] = {(uint32_t)bk, (uint32_t)p.BN, 1u};
    if (!encode_bf16(&tmB, wshadow, 3, bd, bs, bb, bk)) return;
  }
  if (halo) { TW = 16; TH = 8; TN = 1; p.TW = TW; p.TH = TH; p.TN = TN; p.tiles_x = a.Wo / TW; p.tiles_y = a.Ho / TH; }
  const int box_rows = halo ? TH + 2 : TH;
  p.halo = halo ? 1 : 0;
  uint64_t ad[4] = {(uint64_t)Ca, (uint64_t)a.Wi, (uint64_t)a.Hi, (uint64_t)a.N};
  uint64_t as[3] = {(uint64_t)Ca * 2, (uint64_t)a.Wi * Ca * 2, (uint64_t)a.Hi * a.Wi * Ca * 2};
  const uint32_t st = (a.mode == 0) ? (uint32_t)a.stride : 1u;
  uint32_t ab[4] = {(uint32_t)bk, (uint32_t)TW * st, (uint32_t)box_rows * st, (uint32_t)TN};
  uint32_t ae[4] = {1u, st, st, 1u};
  if (!encode_bf16(&tmA, a.x, 4, ad, as, ab, bk, ae)) return;
  const size_t stage = halo ? (size_t)box_rows * TW * bk * 2 + (size_t)3 * p.BN * bk * 2 : (size_t)128 * bk * 2 + (size_t)p.BN * bk * 2;
  const int total = halo ? 3 * p.KC : p.T * p.KC;
  // output path: shared-memory staging + TMA stores, or 16-byte stores from registers.  The per-pixel GEMMs gain from the
  // staged store, the K-heavy 3x3 convolutions lose the pipeline stage the staging buffer costs -> forward 1x1 only.  An
  // accumulating launch (the FiLM Dense data gradients summing into the embedding gradient) always stages its tile and adds
  // it with a TMA reduce-add: the epilogue never reads the destination.
  CUtensorMap tmY = tmA;
  const int cws = p.BN % 64 == 0 ? 64 : 32;         // channels of one staged output box (the kernel's CG)
  {
    p.tma_store = a.accumulate ? 1 : (a.ks == 1 && a.mode == 0);
    if (p.tma_store) {
      uint64_t yd[4] = {(uint64_t)a.Co, (uint64_t)a.Wo, (uint64_t)a.Ho, (uint64_t)a.N};
      uint64_t ys[3] = {(uint64_t)a.Co * 2, (uint64_t)a.Wo * a.Co * 2, (uint64_t)a.Ho * a.Wo * a.Co * 2};
      uint32_t yb[4] = {(uint32_t)cws, (uint32_t)TW, (uint32_t)TH, (uint32_t)TN};
      if (!encode_bf16(&tmY, a.y, 4, yd, ys, yb, cws)) return;
    }
  }
  const size_t ystage = p.tma_store ? (size_t)2 * 128 * cws * 2 : 0;
  p.n_tiles = a.Co / p.BN;
  p.m_tiles = p.tiles_x * p.tiles_y * (a.N / TN);
  p.total_tiles = p.m_tiles * p.n_tiles;
  // CTAs per SM: two where the kernel is compiled for it (conv_ctas_per_sm) and shared
  // memory keeps a >= 3-deep TMA ring for each; one persistent CTA per SM with a 4-deep ring otherwise
  const int epi = a.gn_x == nullptr ? 0 : (a.gn_e != nullptr ? 3 : 2);
  const size_t gtab = epi >= 2 ? (size_t)8 * (p.BN < 64 ? 32 : p.BN / 2) * 16 : 0;      // the EPI 2/3 per-warp norm tables (smG)
  const size_t fixed = ystage + (size_t)2 * conv_tbuf_floats(epi, p.BN) * 4 + 1024 + 256 + gtab;
  int per_sm = 1, stages = 2;
  for (int cand = conv_ctas_per_sm(epi, p.BN, bk); cand >= 1; --cand) {
    const size_t budget = cand == 1 ? (size_t)227 * 1024 : (size_t)112 * 1024;
    int st = (int)((budget - fixed) / stage);
    if (st > 6) st = 6;
    if (st >= 3 || cand == 1) { per_sm = cand; stages = st < 1 ? 1 : st; break; }
  }
  if (per_sm == 1 && stages > 4) stages = 4;
  if (stages > total && total >= 2) stages = total;
  p.stages = stages;
  const size_t smem = stage * stages + fixed + 8 * 2 * stages;
  int ctas = xu_num_sms() * per_sm;
  if (ctas > p.total_tiles) ctas = p.total_tiles;
  dim3 grid((unsigned)ctas);
  {
    static const bool log = getenv("XUNET_CONV_LOG") != nullptr;
    // epi: the epilogue template argument (1: forward with GroupNorm statistics)
    // acc: the output is added to the destination (TMA reduce-add); tma_store: the tile is staged and stored by TMA
    // sched: how the two consumer warpgroups share the tiles (cooperative: both on every tile; pingpong: whole tiles in turn)
    if (log) fprintf(stderr, "conv_tc mode=%d N=%d %dx%d Ci=%d Co=%d ks=%d st=%d wCi=%d wCo=%d segw=%d bk=%d BN=%d KC=%d T=%d halo=%d stages=%d per_sm=%d ctas=%d tiles=%d epi=%d acc=%d tma_store=%d sched=%s\n",
                     a.mode, a.N, a.Ho, a.Wo, a.Ci, a.Co, a.ks, a.stride, a.wCi, a.wCo, a.segw, bk, p.BN, p.KC, p.T, p.halo, p.stages, per_sm, ctas, p.total_tiles,
                     epi != 0 ? epi : (a.cstats != nullptr ? 1 : 0), a.accumulate ? 1 : 0, p.tma_store,
                     conv_pingpong(p.BN) ? "pingpong" : "cooperative");
  }
  p.cstats = cacc;
  p.gx = reinterpret_cast<const bf16*>(a.gn_x); p.gnp = reinterpret_cast<const float4*>(a.gn_params); p.gn_swish = a.gn_swish;
  const bool warp_in_sample = p.TW * p.TH >= 32 || (p.TW * p.TH == 16 && p.TN % 2 == 0);
  if (a.cstats != nullptr && a.gn_x == nullptr) {
    if (a.mode != 0 || a.accumulate || !warp_in_sample) {
      xu_set_kernel_error("conv_tc: fused GroupNorm statistics requested for an unsupported tile shape");
      return;
    }
    if (bk == 64) launch_tc<64, 1>(tmA, tmB, tmY, p, smem, grid, s);
    else if (bk == 32) launch_tc<32, 1>(tmA, tmB, tmY, p, smem, grid, s);
    else launch_tc<16, 1>(tmA, tmB, tmY, p, smem, grid, s);
    return;
  }
  p.ge = reinterpret_cast<const bf16*>(a.gn_e); p.gde = reinterpret_cast<bf16*>(a.gn_de);
  p.drop_rate = a.gn_drop_rate; p.drop_op = a.gn_drop_op; p.seed_dev = a.gn_seed_dev;
  p.drop_on = (a.gn_drop_rate > 0.f && a.gn_train && a.gn_seed_dev != nullptr) ? 1 : 0;
  if (a.gn_x != nullptr) {
    if (a.mode != 1 || a.accumulate || a.bias != nullptr || !warp_in_sample || a.cstats == nullptr || a.gn_params == nullptr) {
      xu_set_kernel_error("conv_tc: fused GroupNorm backward requested for an unsupported configuration");
      return;
    }
    // persistent grid: at most the CTAs that can be resident at once, the loop takes the rest
    if ((int)grid.x > per_sm * xu_num_sms()) grid.x = (unsigned)(per_sm * xu_num_sms());
    if (a.gn_e != nullptr) {
      if (a.gn_de == nullptr) { xu_set_kernel_error("conv_tc: fused FiLM backward needs the FiLM gradient buffer"); return; }
      if (bk == 64) launch_tc<64, 3>(tmA, tmB, tmY, p, smem, grid, s);
      else if (bk == 32) launch_tc<32, 3>(tmA, tmB, tmY, p, smem, grid, s);
      else launch_tc<16, 3>(tmA, tmB, tmY, p, smem, grid, s);
      return;
    }
    if (bk == 64) launch_tc<64, 2>(tmA, tmB, tmY, p, smem, grid, s);
    else if (bk == 32) launch_tc<32, 2>(tmA, tmB, tmY, p, smem, grid, s);
    else launch_tc<16, 2>(tmA, tmB, tmY, p, smem, grid, s);
    return;
  }
  if (bk == 64) launch_tc<64, 0>(tmA, tmB, tmY, p, smem, grid, s);
  else if (bk == 32) launch_tc<32, 0>(tmA, tmB, tmY, p, smem, grid, s);
  else launch_tc<16, 0>(tmA, tmB, tmY, p, smem, grid, s);
}

// the epilogue statistics (a.cstats, (N/2, Co, 2)) are summed in fp64 and folded in once, independent of the tile order
void launch_conv_tc(const ConvArgs& a, const void* wshadow, cudaStream_t s) {
  const long long n = a.cstats ? (long long)(a.N / 2) * a.Co * 2 : 0;
  double* cacc = nullptr;
  if (n > 0 && (cacc = xu_det_scratch(s, n)) == nullptr) return;
  launch_conv_tc_impl(a, wshadow, cacc, s);
  if (cacc != nullptr) xu_det_fold(a.cstats, cacc, n, s);
}
