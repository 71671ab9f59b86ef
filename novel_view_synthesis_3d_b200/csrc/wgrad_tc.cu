// wgrad_tc.cu -- wgmma weight-gradient of the 3x3 / 1x1 convolutions (XLA autodiff of nn.Conv / nn.Dense, train.py:70).
//
//   dW[tap][ci][co] += alpha * sum_pixels X[pixel (+) tap][ci] * dY[pixel][co]
//
// GEMM view: D[M = (tap, ci)][N = co], K = output pixels.  Both operands are "MN-major" for the tensor core -- the
// contiguous index of the NHWC tensors (channels) is the GEMM M / N index -- so the TMA boxes {channels, TW, TH, TN}
// land in shared memory as [128 pixels][channel-chunk] and are consumed through MN-major GMMA descriptors without any
// transposition.  One CTA accumulates a 128 x BN tile of dW (several (tap, ci-chunk) blocks stacked along M) in registers over
// its share of the pixels (split-K across CTAs), then adds it to an fp64 copy of the gradient (xu_det_scratch) that is folded
// into the flat fp32 gradient buffer afterwards, so the split-K sum does not depend on the order in which the CTAs finish.
#include "conv_tc.h"
#include "tc_common.cuh"

#include <stdio.h>
#include <stdlib.h>

namespace {

struct WgTcParams {
  int TW, TH, TN, tiles_x, tiles_y, ptiles;   // pixel tiling (same as conv_tc)
  int Ci, Co, taps, ks, segw, stride, pad_h, pad_w;
  int cpt;          // ci-chunks per tap
  int MB;           // total M-blocks = taps * cpt
  int BN;           // N tile (wgmma N)
  int stages;
  float alpha;
  double* dw;       // fp64 accumulators laid out like the weight / bias gradients (xu_det_scratch), folded in afterwards
  double* dbias;    // if non-null: an all-ones M-block appended after the last (tap, ci) block yields colsum(dY)
};

// One CTA accumulates a 128 x BN tile of dW: warps 0-7 are two consumer warpgroups (M rows 64 wg .. 64 wg + 63, fp32
// accumulators in registers), warp 8 is the TMA producer.  K = pixels, 128 per pipeline step.
constexpr int kWgThreads = 288;
template <int CWA, int CWB, int BN>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmX,
                                                                 const __grid_constant__ CUtensorMap tmDY, const WgTcParams p) {
  constexpr int PT = 128;
  constexpr int G = 128 / CWA;                  // M-blocks stacked per CTA
  constexpr int A_BLOCK = PT * CWA * 2;         // bytes of one [PT pixels][CWA] block
  constexpr int B_BLOCK = PT * CWB * 2;
  constexpr int A_BYTES = G * A_BLOCK;
  constexpr int B_BYTES = (BN / CWB) * B_BLOCK;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smA = base;
  uint8_t* smB = base + (size_t)p.stages * A_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(smB + (size_t)p.stages * B_BYTES);
  uint64_t* empty = full + p.stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile_m = blockIdx.x, n_tile = blockIdx.y;
  const int per = (p.ptiles + gridDim.z - 1) / gridDim.z;
  const int pt_beg = blockIdx.z * per;
  const int pt_end = min(pt_beg + per, p.ptiles);
  const int total = pt_end - pt_beg;
  int nblk = p.MB - tile_m * G;                 // valid M-blocks of this tile
  if (nblk > G) nblk = G;
  if (nblk < 0) nblk = 0;
  // bias gradient: the block right after the last weight block is filled with ones (never touched by TMA)
  const int ones_g = (p.dbias != nullptr && n_tile >= 0 && tile_m == p.MB / G && (p.MB % G != 0 || nblk == 0)) ? nblk : -1;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (ones_g >= 0) {
    const uint32_t ones2 = 0x3F803F80u;          // two bf16 1.0
    for (int st = 0; st < p.stages; ++st) {
      uint32_t* blk = reinterpret_cast<uint32_t*>(smA + (size_t)st * A_BYTES + ones_g * A_BLOCK);
      for (int i = threadIdx.x; i < A_BLOCK / 4; i += blockDim.x) blk[i] = ones2;
    }
    fence_async_smem();
  }
  __syncthreads();
  xu_grid_dep_sync();     // PDL: everything above overlaps the previous kernel's tail
  if (total <= 0) return;

  if (warp == 8) {
    if (lane == 0) {
      for (int it = 0; it < total; ++it) {
        const int s = it % p.stages;
        mbar_wait(&empty[s], ((it / p.stages) & 1) ^ 1);
        int t = pt_beg + it;
        const int tx = t % p.tiles_x; t /= p.tiles_x;
        const int ty = t % p.tiles_y; t /= p.tiles_y;
        const int x0 = tx * p.TW, y0 = ty * p.TH, n0 = t * p.TN;
        mbar_expect_tx(&full[s], nblk * A_BLOCK + B_BYTES);
        for (int g = 0; g < nblk; ++g) {
          const int mb = tile_m * G + g;
          const int tap = mb / p.cpt, chunk = mb - tap * p.cpt;
          int ox = 0, oy = 0;
          if (p.ks == 3) { const int dy = tap / 3; oy = dy - p.pad_h; ox = tap - dy * 3 - p.pad_w; }
          tma_load_4d(smA + (size_t)s * A_BYTES + g * A_BLOCK, &tmX, &full[s], chunk * CWA, x0 * p.stride + ox, y0 * p.stride + oy, n0);
        }
        for (int b = 0; b < BN / CWB; ++b)
          tma_load_4d(smB + (size_t)s * B_BYTES + b * B_BLOCK, &tmDY, &full[s], n_tile * BN + b * CWB, x0, y0, n0);
      }
    }
    return;
  }
  const int wg = warp >> 2, wq = warp & 3;
  const uint32_t a_off = (uint32_t)((64 * wg / CWA) * A_BLOCK);     // this warpgroup's 64 rows of M
  float acc[BN / 2];
  int prev_s = 0;
  for (int it = 0; it < total; ++it) {
    const int s = it % p.stages;
    mbar_wait(&full[s], (it / p.stages) & 1);
    wgmma_fence();
    const uint32_t a_addr = smem_u32(smA + (size_t)s * A_BYTES) + a_off;
    const uint32_t b_addr = smem_u32(smB + (size_t)s * B_BYTES);
#pragma unroll
    for (int k = 0; k < PT / 16; ++k)                     // PT pixels = PT/16 x (K = 16); A and B both MN-major
      Wgmma<BN>::template ss<1, 1>(acc, make_mnmajor_desc<CWA>(a_addr + k * 16 * (CWA * 2), A_BLOCK),
                                   make_mnmajor_desc<CWB>(b_addr + k * 16 * (CWB * 2), B_BLOCK), (it > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    if (it > 0 && lane == 0) mbar_arrive(&empty[prev_s]);
    prev_s = s;
  }
  wgmma_wait<0>();
  if (lane == 0) mbar_arrive(&empty[prev_s]);
  // accumulator fragment -> fp64 adds (rows R and R + 8, column pairs 8 i + 2 t): the split-K sum does not depend on the order
  // in which the CTAs of a tile finish
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int R = 64 * wg + 16 * wq + (lane >> 2) + 8 * h;
    const int g = R / CWA, c = R % CWA;
    const int mb = tile_m * G + g;
    const bool valid = g < nblk;
    const bool bias_row = (g == ones_g) && c == 0;
    const int tap = valid ? mb / p.cpt : 0;
    const int ci = valid ? (mb - tap * p.cpt) * CWA + c : 0;
    double* dst = nullptr;
    if (valid && ci < p.Ci) {
      // segw % 32 == 0 -> both columns of a pair are in one segment
      dst = p.dw + ((long long)tap * p.Ci + ci) * p.segw;
    } else if (bias_row) {
      dst = p.dbias + n_tile * BN;
    }
    if (dst == nullptr) continue;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const int col = 8 * i + 2 * (lane & 3);
      double* d = dst;
      if (!bias_row) {
        const int co = n_tile * BN + col;
        const int seg = co / p.segw;
        d += (long long)seg * p.taps * p.Ci * p.segw + (co - seg * p.segw);
      } else {
        d += col;
      }
      xu_det_add(d, p.alpha * acc[4 * i + 2 * h]);
      xu_det_add(d + 1, p.alpha * acc[4 * i + 2 * h + 1]);
    }
  }
}

bool pick_tile_w(int N, int H, int W, int& TW, int& TH, int& TN, int PT = 128) {
  if (W >= PT) {
    if (W % PT) return false;
    TW = PT; TH = 1; TN = 1;
    return true;
  }
  if (PT % W) return false;
  TW = W;
  int rem = PT / W;
  if (H >= rem) {
    if (H % rem) return false;
    TH = rem; TN = 1;
    return true;
  }
  if (rem % H) return false;
  TH = H; TN = rem / H;
  return N % TN == 0;
}
int pick_cw(int C) { return C % 64 == 0 ? 64 : (C % 32 == 0 ? 32 : (C % 16 == 0 ? (C > 64 ? 64 : 16) : 0)); }   // 144 -> 64-wide blocks, tail zero-filled

template <int CWA, int CWB, int BN>
void launch_wg_bn(const CUtensorMap& x, const CUtensorMap& dy, const WgTcParams& p, size_t smem, dim3 grid, cudaStream_t s) {
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(wgrad_tc_kernel<CWA, CWB, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    configured = true;
  }
  xu_launch(wgrad_tc_kernel<CWA, CWB, BN>, grid, kWgThreads, smem, s, x, dy, p);
}
template <int CWA, int CWB>
void launch_wg(const CUtensorMap& x, const CUtensorMap& dy, const WgTcParams& p, size_t smem, dim3 grid, cudaStream_t s) {
  if (p.BN == 128) launch_wg_bn<CWA, CWB, 128>(x, dy, p, smem, grid, s);
  else if (p.BN == 64) launch_wg_bn<CWA, CWB, 64>(x, dy, p, smem, grid, s);
  else if constexpr (CWB == 32) launch_wg_bn<CWA, 32, 32>(x, dy, p, smem, grid, s);
}

}  // namespace

bool wgrad_tc_supported(int dtype, int N, int H, int W, int Ci, int Co, int ks, int stride, int nseg) {
  if (dtype != XU_BF16 || (ks != 1 && ks != 3)) return false;
  if (stride != 1 && ks != 3) return false;
  if (nseg != 1 && ks != 1) return false;
  int TW, TH, TN;
  if (!pick_tile_w(N, (H + stride - 1) / stride, (W + stride - 1) / stride, TW, TH, TN)) return false;   // tiles of OUTPUT pixels
  if (TW * stride > 256 || TH * stride > 256) return false;
  if (pick_cw(Ci) == 0) return false;
  if (Co % 32 != 0 || (Co / nseg) % 32 != 0) return false;
  if (Co > 256 && Co % 256 != 0) return false;
  return true;
}

void launch_wgrad_tc(const WgradArgs& a, cudaStream_t s) {
  WgTcParams p;
  if (!pick_tile_w(a.N, a.Ho, a.Wo, p.TW, p.TH, p.TN)) { xu_set_kernel_error("wgrad_tc: unsupported spatial shape"); return; }
  p.tiles_x = a.Wo / p.TW; p.tiles_y = a.Ho / p.TH; p.ptiles = p.tiles_x * p.tiles_y * (a.N / p.TN);
  p.Ci = a.Ci; p.Co = a.Co; p.ks = a.ks; p.taps = a.ks * a.ks; p.segw = a.segw;
  p.stride = a.stride; p.pad_h = a.pad_h; p.pad_w = a.pad_w;
  const int cwa = pick_cw(a.Ci);
  const int cwb = a.Co % 64 == 0 ? 64 : 32;
  p.cpt = (a.Ci + cwa - 1) / cwa; p.MB = p.taps * p.cpt;
  // wgmma N: 128, 64 or 32 (a 256-column tile would spill its 128 accumulator registers per thread)
  p.BN = a.Co % 128 == 0 ? 128 : (a.Co % 64 == 0 ? 64 : 32);
  p.alpha = a.alpha;
  const long long ndw = (long long)a.ks * a.ks * a.Ci * a.Co, ndb = a.dbias ? a.Co : 0;
  double* acc = xu_det_scratch(s, ndw + ndb);
  if (acc == nullptr) return;
  p.dw = acc;
  const int G = 128 / cwa;
  p.dbias = a.dbias ? acc + ndw : nullptr;
  const int tiles_m = a.dbias != nullptr ? p.MB / G + 1 : (p.MB + G - 1) / G;   // room for the all-ones bias block
  const int tiles_n = a.Co / p.BN;
  const size_t stage = (size_t)128 * 128 * 2 + (size_t)p.BN * 128 * 2;
  int stages = (int)((225 * 1024) / stage);
  if (stages > 4) stages = 4;
  if (stages < 1) stages = 1;
  p.stages = stages;
  // split-K factor: one CTA per SM (the ring takes all of shared memory), so the launch runs in ceil(tiles*k / SMs) waves of
  // ceil(ptiles / k) pixel tiles each.  Rounding k UP to cover the SMs can cost a whole second wave for a handful of CTAs, so
  // minimise waves x tiles-per-CTA instead (ties -> fewer splits: every split adds M*N fp32 reds).  With SMs reserved
  // (XUNET_SM_RESERVE) the rule alone would pick fewer, longer splits, up to all the pixels in one CTA, whose fp32 sums in the
  // tensor cores' truncating accumulator err past what the whole device's splits do; so k is never below the whole device's.
  const long long T = (long long)tiles_m * tiles_n;
  auto pick_split = [&](long long sms, int kmin) {
    int k_best = kmin;
    long long best = -1;
    const int kmax = p.ptiles < 64 ? p.ptiles : 64;
    for (int k = kmin; k <= (kmax > kmin ? kmax : kmin); ++k) {
      const long long waves = (T * k + sms - 1) / sms, per = (p.ptiles + k - 1) / k;
      const long long cost = waves * (per + 8);        // +8: per-CTA pipeline fill + reds, in pixel-tile units
      if (best < 0 || cost < best) { best = cost; k_best = k; }
    }
    return k_best;
  };
  const int ksplit = pick_split(xu_num_sms(), pick_split(xu_device_sms(), 1));
  CUtensorMap tx, ty;
  uint64_t xd[4] = {(uint64_t)a.Ci, (uint64_t)a.Wi, (uint64_t)a.Hi, (uint64_t)a.N};
  uint64_t xs[3] = {(uint64_t)a.Ci * 2, (uint64_t)a.Wi * a.Ci * 2, (uint64_t)a.Hi * a.Wi * a.Ci * 2};
  const uint32_t st = (uint32_t)a.stride;
  uint32_t xb[4] = {(uint32_t)cwa, (uint32_t)p.TW * st, (uint32_t)p.TH * st, (uint32_t)p.TN};
  uint32_t xe[4] = {1u, st, st, 1u};
  uint64_t yd[4] = {(uint64_t)a.Co, (uint64_t)a.Wo, (uint64_t)a.Ho, (uint64_t)a.N};
  uint64_t ys[3] = {(uint64_t)a.Co * 2, (uint64_t)a.Wo * a.Co * 2, (uint64_t)a.Ho * a.Wo * a.Co * 2};
  uint32_t yb[4] = {(uint32_t)cwb, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
  if (!xu_encode_bf16_map(&tx, a.x, 4, xd, xs, xb, cwa, xe) || !xu_encode_bf16_map(&ty, a.dy, 4, yd, ys, yb, cwb)) return;
  const size_t smem = stage * p.stages + 1024 + 8 * 2 * p.stages + 16;
  dim3 grid((unsigned)tiles_m, (unsigned)tiles_n, (unsigned)ksplit);
  {
    static const bool log = getenv("XUNET_CONV_LOG") != nullptr;      // tools/conv_step_profile.py matches these lines with CUPTI times
    // cwa / cwb: the kernel's <CWA, CWB> (channels per A / B block); MB: the (tap, ci-chunk) blocks of M, G = 128 / cwa per tile
    if (log) fprintf(stderr, "wgrad_tc N=%d %dx%d Ci=%d Co=%d ks=%d st=%d BN=%d ksplit=%d tm=%d tn=%d stages=%d ptiles=%d cwa=%d cwb=%d MB=%d\n", a.N,
                     a.Ho, a.Wo, a.Ci, a.Co, a.ks, a.stride, p.BN, ksplit, tiles_m, tiles_n, p.stages, p.ptiles, cwa, cwb, p.MB);
  }
  if (cwa == 64 && cwb == 64) launch_wg<64, 64>(tx, ty, p, smem, grid, s);
  else if (cwa == 64) launch_wg<64, 32>(tx, ty, p, smem, grid, s);
  else if (cwa == 32 && cwb == 64) launch_wg<32, 64>(tx, ty, p, smem, grid, s);
  else if (cwa == 32) launch_wg<32, 32>(tx, ty, p, smem, grid, s);
  else if (cwb == 64) launch_wg<16, 64>(tx, ty, p, smem, grid, s);
  else launch_wg<16, 32>(tx, ty, p, smem, grid, s);
  xu_det_fold(a.dw, acc, ndw, s);
  if (a.dbias) xu_det_fold(a.dbias, acc + ndw, ndb, s);
}
