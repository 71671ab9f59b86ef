// pose_grad.cu -- gradient of the loss w.r.t. the camera rays and the cameras (xunet_backward_vjp_inputs).
//
// The cameras enter the network through the 144-channel NeRF posenc P(ray) of every pixel of both frames (pose_emb_kernel), read
// by the L pose-embedding convolutions (3x3, 144 -> emb_ch, stride 2^l, XLA SAME padding).  Per level l this file computes the data
// gradient of that convolution, g_l = conv_transpose(grad(pose_emb_l), W_l) (2B, S, S, 144), and never stores it: the posenc is
// elementwise in the ray coordinates at fixed rays, so the epilogue applies the Jacobian transpose at once and keeps six numbers
// per pixel, d_rays = [d pos xyz | d dir xyz] = J(pix)^T g.  For component v of pos (15 scales) or dir (8 scales):
//     J^T g = g[x] + sum_k 2^k cos(fl32(2^k v)) g[sin_k] + 2^k cos(fl32(fl32(2^k v) + pi/2)) g[shifted sin_k]
// with the fp32 arguments the forward formed (posenc_nerf's layout, pose_channel in kernels_elem.cu).
//
// * pose_dgrad_tc_kernel (bf16): wgmma implicit GEMM per level.  Input pixel i receives tap d from output o exactly when
//   s o + d - lo = i, so the pixels are split by phase (i mod s per axis) and each phase is its own GEMM over the taps that hit
//   it (stride 1: all 9; stride 2: 2x2, 2x1, 1x2 or 1x1; strides 4 and 8: one tap for phases 0-2 and none for the rest): no MMA
//   is spent on structural zeros.  A = grad(pose_emb_l) read by TMA boxes of output pixels (K-major, out-of-range rows
//   zero-filled: the SAME padding), B = the forward's bf16 weight shadow [E][tap][144] read as an MN-major operand, D = 128 pixels
//   x 144 channels in registers (m64n144).  Level 0 stores d_rays, later levels add (launch order on one stream).
// * pose_dgrad_simt_kernel: the same contract in fp32 SIMT (fp32 verify mode, and the levels whose forward has no bf16 shadow
//   because it runs on SIMT cores too); it sums its levels' g before one J^T.
// * camera_grad_kernel: generated rays only, d_rays -> dt, dR and dK per sample, in fp64 in a fixed order.
#include "kernels.h"
#include "pose_grad.h"
#include "tc_common.cuh"

#include <stdio.h>

namespace {

// 2^k cos of the argument posenc_nerf formed for scale k (shifted: + pi/2 in fp32), the Jacobian entry of that channel
__device__ __forceinline__ float posenc_coef(float v, int k, int shifted) {
  float xb = v * (float)(1 << k);
  if (shifted) xb = xb + 1.57079632679489661923f;
  return (float)(1 << k) * cosf(xb);
}

// output q of J^T g (q < 3: d pos[q], else d dir[q - 3]); v = that ray component; ctab: the 90 position coefficients of the
// pixel's frame ([sin scales k, xyz | shifted]) or nullptr (computed here)
__device__ __forceinline__ float posenc_jt(const float* g, int q, float v, const float* ctab) {
  const int d = q < 3 ? q : q - 3;
  const int nd = q < 3 ? 15 : 8;
  const float* gg = g + (q < 3 ? 0 : 93);
  float acc = gg[d];
  for (int k = 0; k < nd; ++k) {
    const float cs = ctab ? ctab[3 * k + d] : posenc_coef(v, k, 0);
    const float cc = ctab ? ctab[3 * nd + 3 * k + d] : posenc_coef(v, k, 1);
    acc = fmaf(cs, gg[3 + 3 * k + d], acc);
    acc = fmaf(cc, gg[3 + 3 * nd + 3 * k + d], acc);
  }
  return acc;
}

// ray component q (pos xyz | dir xyz) of pixel (row, col) of frame n
__device__ __forceinline__ float ray_component(const PoseGradArgs& a, int n, int row, int col, int q) {
  if (a.rays) return a.rays[((long long)n * a.S * a.S + (long long)row * a.S + col) * 6 + q];
  const int b = n >> 1, f = n & 1;
  if (q < 3) return ((f == 0 ? a.t1 : a.t2) + b * 3)[q];
  float d[3];
  xu_ray_dir(a.kinv + b * 9, (f == 0 ? a.R1 : a.R2) + b * 9, row, col, a.convention, d);
  return d[q - 3];
}

// taps of phase r along one axis: d with (r + lo - d) = s * off; returns their count, d / off in dd / off
__device__ __forceinline__ int phase_taps(int r, int lo, int s, int (&dd)[3], int (&off)[3]) {
  int n = 0;
  for (int d = 0; d < 3; ++d) {
    const int u = r + lo - d;
    if (((u % s) + s) % s == 0) { dd[n] = d; off[n] = u >= 0 ? u / s : -((-u) / s); ++n; }
  }
  return n;
}

// ================================================================================================ SIMT (fp32 / fallback)
constexpr int kSimtPix = 16, kSimtThreads = 160, kSimtE = 32;
template <typename T, bool RW>
__global__ void __launch_bounds__(kSimtThreads, 4) pose_dgrad_simt_kernel(const PoseGradArgs a, const PoseLevels lv, int accumulate) {
  xu_grid_dep_sync();
  __shared__ float s_dy[kSimtPix][kSimtE + 1];
  __shared__ float s_g[kSimtPix][XU_POSE_DIM + 1];
  const int tid = threadIdx.x;
  const int n = blockIdx.y, b = n >> 1;
  const int HW = a.S * a.S, pix0 = blockIdx.x * kSimtPix;
  const bool on = a.cond_mask[b] != 0.f;
  const int ci = tid;                       // GEMM column of this thread (tid < 144)
  float acc[kSimtPix];
#pragma unroll
  for (int p = 0; p < kSimtPix; ++p) acc[p] = 0.f;
  for (int li = 0; on && li < lv.n; ++li) {
    const PoseLevel& L = lv.l[li];
    const T* dy = reinterpret_cast<const T*>(L.dy);
    for (int tap = 0; tap < 9; ++tap) {
      const int ty = tap / 3, tx = tap - ty * 3;
      for (int e0 = 0; e0 < a.E; e0 += kSimtE) {
        for (int idx = tid; idx < kSimtPix * kSimtE; idx += kSimtThreads) {
          const int p = idx / kSimtE, e = idx - p * kSimtE;
          const int pix = pix0 + p;
          float v = 0.f;
          if (pix < HW && e0 + e < a.E) {
            const int iy = pix / a.S, ix = pix - iy * a.S;
            const int uy = iy + L.lo - ty, ux = ix + L.lo - tx;
            if (uy >= 0 && ux >= 0 && uy % L.s == 0 && ux % L.s == 0 && uy / L.s < L.So && ux / L.s < L.So)
              v = L.alpha * ldf(dy + (((long long)n * L.So + uy / L.s) * L.So + ux / L.s) * a.E + e0 + e);
          }
          s_dy[p][e] = v;
        }
        __syncthreads();
        if (ci < XU_POSE_DIM) {
          // one partial sum per chunk, added to the running sum: the rounding error grows with the chunk count instead of
          // with taps x emb_ch terms in one chain (the J^T after it amplifies relative error by its cancellation)
          float part[kSimtPix];
#pragma unroll
          for (int p = 0; p < kSimtPix; ++p) part[p] = 0.f;
          const float* w = L.w + ((long long)tap * XU_POSE_DIM + ci) * a.E + e0;
          const int ne = min(kSimtE, a.E - e0);
          for (int e = 0; e < ne; ++e) {
            float wv = __ldg(w + e);
            if (RW) wv = __bfloat162float(__float2bfloat16_rn(wv));
#pragma unroll
            for (int p = 0; p < kSimtPix; ++p) part[p] = fmaf(s_dy[p][e], wv, part[p]);
          }
#pragma unroll
          for (int p = 0; p < kSimtPix; ++p) acc[p] += part[p];
        }
        __syncthreads();
      }
    }
  }
  if (ci < XU_POSE_DIM) {
#pragma unroll
    for (int p = 0; p < kSimtPix; ++p) s_g[p][ci] = acc[p];
  }
  __syncthreads();
  if (tid < kSimtPix * 6) {
    const int p = tid / 6, q = tid - p * 6, pix = pix0 + p;
    if (pix < HW) {
      float* o = a.d_rays + ((long long)n * HW + pix) * 6 + q;
      const int row = pix / a.S, col = pix - row * a.S;
      const float r = on ? posenc_jt(s_g[p], q, ray_component(a, n, row, col, q), nullptr) : 0.f;
      if (accumulate) *o += r; else *o = r;
    }
  }
}

// ================================================================================================ wgmma (bf16)
struct TcLevel {
  int So, s, lo, E, KC;
  int TW, TH, TN, tiles_x, tiles_y;
  int nph;          // phases per axis that receive taps
  int stages;
  float alpha;
  int accumulate;
};
constexpr int kTcThreads = 288;          // two consumer warpgroups (64 pixel rows each) + one TMA producer warp
constexpr int kGP = XU_POSE_DIM + 1;     // pitch of the fp32 [128 pixels][144] epilogue buffer
constexpr int kMaxTN = 64;               // images per 128-pixel tile (So = 2 -> 32)
template <int BK>
__global__ void __launch_bounds__(kTcThreads, 1) pose_dgrad_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                       const __grid_constant__ CUtensorMap tmB,
                                                                       const PoseGradArgs a, const TcLevel p) {
  extern __shared__ uint8_t smem_raw[];
  constexpr int A_BYTES = 128 * BK * 2;
  constexpr int B_BLOCK = BK * 64 * 2;      // [BK rows of e][64 channels], 128B-swizzled
  constexpr int B_BYTES = 3 * B_BLOCK;      // channels 0-63, 64-127, 128-143 (+ zero fill)
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smA = base;
  uint8_t* smB = base + (size_t)p.stages * A_BYTES;
  float* sG = reinterpret_cast<float*>(smB + (size_t)p.stages * B_BYTES);      // [128][kGP]
  float* sC = sG + 128 * kGP;                                                  // [TN][90] position coefficients
  uint64_t* full = reinterpret_cast<uint64_t*>(sC + kMaxTN * 90);
  uint64_t* empty = full + p.stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int t = blockIdx.x;
  const int tx = t % p.tiles_x; t /= p.tiles_x;
  const int ty = t % p.tiles_y; t /= p.tiles_y;
  const int qx0 = tx * p.TW, qy0 = ty * p.TH, n0 = t * p.TN;
  const int ry = blockIdx.y / p.nph, rx = blockIdx.y - ry * p.nph;
  int dyy[3], oyy[3], dxx[3], oxx[3];
  const int nty = phase_taps(ry, p.lo, p.s, dyy, oyy);
  const int ntx = phase_taps(rx, p.lo, p.s, dxx, oxx);
  const int total = nty * ntx * p.KC;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  __syncthreads();
  xu_grid_dep_sync();

  if (warp == 8) {
    if (lane == 0) {
      for (int it = 0; it < total; ++it) {
        const int s = it % p.stages;
        mbar_wait(&empty[s], ((it / p.stages) & 1) ^ 1);
        const int c = it % p.KC, tt = it / p.KC;
        const int jy = tt / ntx, jx = tt - jy * ntx;
        const int tap = dyy[jy] * 3 + dxx[jx];
        mbar_expect_tx(&full[s], A_BYTES + B_BYTES);
        tma_load_4d(smA + (size_t)s * A_BYTES, &tmA, &full[s], c * BK, qx0 + oxx[jx], qy0 + oyy[jy], n0);
#pragma unroll
        for (int j = 0; j < 3; ++j) tma_load_3d(smB + (size_t)s * B_BYTES + j * B_BLOCK, &tmB, &full[s], 64 * j, tap, c * BK);
      }
    }
    return;
  }
  // ===== consumers =====
  const int wg = warp >> 2, wq = warp & 3;
  const int ctid = threadIdx.x;              // 0..255
  // position coefficients of the tile's frames (generated rays: the position is the camera centre, one per frame)
  if (a.rays == nullptr) {
    for (int j = ctid; j < p.TN * 90; j += 256) {
      const int tn = j / 90, e = j - tn * 90, n = n0 + tn;
      if (n >= 2 * a.B) continue;
      const int sh = e >= 45, k = (sh ? e - 45 : e) / 3, d = (sh ? e - 45 : e) % 3;
      sC[j] = posenc_coef(((n & 1) == 0 ? a.t1 : a.t2)[(n >> 1) * 3 + d], k, sh);
    }
  }
  float acc[72];
#pragma unroll
  for (int i = 0; i < 72; ++i) acc[i] = 0.f;
  int prev_s = 0;
  for (int it = 0; it < total; ++it) {
    const int s = it % p.stages;
    mbar_wait(&full[s], (it / p.stages) & 1);
    wgmma_fence();
    const uint32_t a_addr = smem_u32(smA + (size_t)s * A_BYTES) + (uint32_t)(wg * 64 * BK * 2);
    const uint32_t b_addr = smem_u32(smB + (size_t)s * B_BYTES);
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)
      Wgmma<144>::template ss<0, 1>(acc, make_kmajor_desc<BK>(a_addr + k * 32), make_mnmajor_desc<64>(b_addr + k * 16 * 128, B_BLOCK),
                                    (it > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    if (it > 0 && lane == 0) mbar_arrive(&empty[prev_s]);
    prev_s = s;
  }
  wgmma_wait<0>();
  // accumulator fragment -> [128 pixels][144] fp32
  {
    const int fr = 64 * wg + 16 * wq + (lane >> 2), fc = (lane & 3) * 2;
#pragma unroll
    for (int i = 0; i < 72; i += 4) {
      const int col = 8 * (i / 4) + fc;
      sG[fr * kGP + col] = p.alpha * acc[i];
      sG[fr * kGP + col + 1] = p.alpha * acc[i + 1];
      sG[(fr + 8) * kGP + col] = p.alpha * acc[i + 2];
      sG[(fr + 8) * kGP + col + 1] = p.alpha * acc[i + 3];
    }
  }
  named_bar_sync(1, 256);
  const int per = p.TW * p.TH;
  for (int idx = ctid; idx < 128 * 6; idx += 256) {
    const int r = idx / 6, q = idx - r * 6;
    const int tn = r / per, rem = r - tn * per;
    const int n = n0 + tn;
    const int qy = qy0 + rem / p.TW, qx = qx0 + rem % p.TW;
    if (n >= 2 * a.B || qy >= p.So || qx >= p.So) continue;
    const int row = p.s * qy + ry, col = p.s * qx + rx;
    float* o = a.d_rays + (((long long)n * a.S + row) * a.S + col) * 6 + q;
    float v = 0.f;
    if (a.cond_mask[n >> 1] != 0.f) {
      const float* ctab = (a.rays == nullptr && q < 3) ? sC + tn * 90 : nullptr;
      v = posenc_jt(sG + r * kGP, q, ctab ? 0.f : ray_component(a, n, row, col, q), ctab);
    }
    if (p.accumulate) *o += v; else *o = v;
  }
}

// ================================================================================================ cameras
// One block per sample: d_rays of both frames -> dt1, dR1, dt2, dR2 and dK.  With c = K^-1 p, w = R c, dir = w / |w|:
//   dt += d pos;  d_w = (d dir - dir (dir . d dir)) / |w|;  dR += d_w c^T;  dK^-1 += (R^T d_w) p^T;  dK = -K^-T (sum dK^-1) K^-T.
// Per-thread fp64 partials over a fixed pixel stride, then a fixed shuffle tree and the warps in order: fixed bits, no atomics.
constexpr int kCamThreads = 256, kCamVals = 33;    // per frame: dt (3), dR (9); shared: dK^-1 (9)
__global__ void __launch_bounds__(kCamThreads) camera_grad_kernel(const float* __restrict__ d_rays, const float* __restrict__ R1,
                                                                  const float* __restrict__ R2, const float* __restrict__ K, int S,
                                                                  int convention, float* dR1, float* dt1, float* dR2, float* dt2,
                                                                  float* dK) {
  xu_grid_dep_sync();
  __shared__ double s_part[kCamThreads / 32][kCamVals];
  __shared__ double s_kinv[9];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) {
    double m[9];
    for (int i = 0; i < 9; ++i) m[i] = (double)K[b * 9 + i];
    const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
    const double id = 1.0 / (m[0] * c00 + m[1] * c01 + m[2] * c02);
    s_kinv[0] = c00 * id; s_kinv[1] = (m[2] * m[7] - m[1] * m[8]) * id; s_kinv[2] = (m[1] * m[5] - m[2] * m[4]) * id;
    s_kinv[3] = c01 * id; s_kinv[4] = (m[0] * m[8] - m[2] * m[6]) * id; s_kinv[5] = (m[2] * m[3] - m[0] * m[5]) * id;
    s_kinv[6] = c02 * id; s_kinv[7] = (m[1] * m[6] - m[0] * m[7]) * id; s_kinv[8] = (m[0] * m[4] - m[1] * m[3]) * id;
  }
  __syncthreads();
  double v[kCamVals];
#pragma unroll
  for (int i = 0; i < kCamVals; ++i) v[i] = 0.0;
  const int HW = S * S;
  for (int f = 0; f < 2; ++f) {
    double Rm[9];
    for (int i = 0; i < 9; ++i) Rm[i] = (double)(f == 0 ? R1 : R2)[b * 9 + i];
    const float* dr = d_rays + (long long)(2 * b + f) * HW * 6;
    for (int pix = tid; pix < HW; pix += kCamThreads) {
      const int row = pix / S, col = pix - row * S;
      const double pp[3] = {(convention == 0 ? row : col) + 0.5, (convention == 0 ? col : row) + 0.5, 1.0};
      double c[3], w[3];
      for (int i = 0; i < 3; ++i) c[i] = s_kinv[3 * i] * pp[0] + s_kinv[3 * i + 1] * pp[1] + s_kinv[3 * i + 2] * pp[2];
      for (int i = 0; i < 3; ++i) w[i] = Rm[3 * i] * c[0] + Rm[3 * i + 1] * c[1] + Rm[3 * i + 2] * c[2];
      const double nw = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
      const double dir[3] = {w[0] / nw, w[1] / nw, w[2] / nw};
      const double dd[3] = {dr[pix * 6 + 3], dr[pix * 6 + 4], dr[pix * 6 + 5]};
      const double dot = dir[0] * dd[0] + dir[1] * dd[1] + dir[2] * dd[2];
      double dw[3];
      for (int i = 0; i < 3; ++i) dw[i] = (dd[i] - dir[i] * dot) / nw;
      double u[3];
      for (int j = 0; j < 3; ++j) u[j] = Rm[j] * dw[0] + Rm[3 + j] * dw[1] + Rm[6 + j] * dw[2];
      double* vf = v + 12 * f;
      for (int i = 0; i < 3; ++i) vf[i] += dr[pix * 6 + i];
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) vf[3 + 3 * i + j] += dw[i] * c[j];
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) v[24 + 3 * i + j] += u[i] * pp[j];
    }
  }
#pragma unroll
  for (int i = 0; i < kCamVals; ++i) {
    double x = v[i];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    v[i] = x;
  }
  if ((tid & 31) == 0)
    for (int i = 0; i < kCamVals; ++i) s_part[tid >> 5][i] = v[i];
  __syncthreads();
  __shared__ double s_tot[kCamVals];
  if (tid < kCamVals) {
    double x = 0.0;
    for (int w = 0; w < kCamThreads / 32; ++w) x += s_part[w][tid];
    s_tot[tid] = x;
  }
  __syncthreads();
  if (tid < 12) {
    float* dt = tid < 3 ? (dt1 ? dt1 + b * 3 + tid : nullptr) : (dR1 ? dR1 + b * 9 + tid - 3 : nullptr);
    if (dt) *dt = (float)s_tot[tid];
  } else if (tid < 24) {
    const int k = tid - 12;
    float* dt = k < 3 ? (dt2 ? dt2 + b * 3 + k : nullptr) : (dR2 ? dR2 + b * 9 + k - 3 : nullptr);
    if (dt) *dt = (float)s_tot[tid];
  } else if (tid < 33 && dK) {
    // dK[i][j] = -sum_{a,c} Kinv[a][i] G[a][c] Kinv[j][c]
    const int i = (tid - 24) / 3, j = (tid - 24) % 3;
    double x = 0.0;
    for (int aa = 0; aa < 3; ++aa)
      for (int cc = 0; cc < 3; ++cc) x += s_kinv[3 * aa + i] * s_tot[24 + 3 * aa + cc] * s_kinv[3 * j + cc];
    dK[b * 9 + 3 * i + j] = (float)(-x);
  }
}

int tc_pick_tile(int N, int So, int& TW, int& TH, int& TN) {
  if (So >= 128) {
    if (So % 128) return 0;
    TW = 128; TH = 1; TN = 1;
    return 1;
  }
  if (128 % So) return 0;
  TW = So;
  const int rem = 128 / So;
  if (So >= rem) { TH = rem; TN = 1; return 1; }
  TH = So; TN = rem / So;
  return TN <= kMaxTN;
  (void)N;
}

template <int BK>
void launch_tc_level(const CUtensorMap& ta, const CUtensorMap& tb, const PoseGradArgs& a, const TcLevel& p, dim3 grid, size_t smem,
                     cudaStream_t s) {
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(pose_dgrad_tc_kernel<BK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    configured = true;
  }
  xu_launch(pose_dgrad_tc_kernel<BK>, grid, kTcThreads, smem, s, ta, tb, a, p);
}

}  // namespace

bool pose_grad_tc_supported(int So, int E) {
  int TW, TH, TN;
  return E % 8 == 0 && tc_pick_tile(0, So, TW, TH, TN);
}

void launch_pose_grad_tc(const PoseGradArgs& a, const PoseLevel& L, const void* wshadow, int accumulate, cudaStream_t s) {
  TcLevel p;
  p.So = L.So; p.s = L.s; p.lo = L.lo; p.E = a.E; p.alpha = L.alpha; p.accumulate = accumulate;
  const int N = 2 * a.B;
  if (!tc_pick_tile(N, L.So, p.TW, p.TH, p.TN) || a.E % 8 != 0) { xu_set_kernel_error("pose_grad: unsupported level shape"); return; }
  p.tiles_x = L.So / p.TW; p.tiles_y = L.So / p.TH;
  const int mt = p.tiles_x * p.tiles_y * cdiv(N, p.TN);
  p.nph = L.s < 3 ? L.s : 3;
  const int bk = (a.E % 64 == 0 || a.E > 64) ? 64 : 32;
  p.KC = cdiv(a.E, bk);
  const size_t stage = (size_t)128 * bk * 2 + (size_t)3 * bk * 64 * 2;
  const size_t fixed = (size_t)128 * kGP * 4 + (size_t)kMaxTN * 90 * 4 + 1024 + 256;
  int st = (int)(((size_t)227 * 1024 - fixed) / stage);
  p.stages = st > 4 ? 4 : st;
  const size_t smem = fixed + stage * p.stages;
  CUtensorMap ta, tb;
  uint64_t ad[4] = {(uint64_t)a.E, (uint64_t)L.So, (uint64_t)L.So, (uint64_t)N};
  uint64_t as[3] = {(uint64_t)a.E * 2, (uint64_t)L.So * a.E * 2, (uint64_t)L.So * L.So * a.E * 2};
  uint32_t ab[4] = {(uint32_t)bk, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
  uint64_t bd[3] = {(uint64_t)XU_POSE_DIM, 9u, (uint64_t)a.E};
  uint64_t bs[2] = {(uint64_t)XU_POSE_DIM * 2, (uint64_t)9 * XU_POSE_DIM * 2};
  uint32_t bb[3] = {64u, 1u, (uint32_t)bk};
  if (!xu_encode_bf16_map(&ta, L.dy, 4, ad, as, ab, bk) || !xu_encode_bf16_map(&tb, wshadow, 3, bd, bs, bb, 64)) return;
  const dim3 grid((unsigned)mt, (unsigned)(p.nph * p.nph));
  if (bk == 64) launch_tc_level<64>(ta, tb, a, p, grid, smem, s);
  else launch_tc_level<32>(ta, tb, a, p, grid, smem, s);
}

void launch_pose_grad_simt(int dtype, const PoseGradArgs& a, const PoseLevels& lv, int accumulate, cudaStream_t s) {
  const dim3 grid(cdiv(a.S * a.S, kSimtPix), 2 * a.B);
  if (dtype == XU_F32) xu_launch(pose_dgrad_simt_kernel<float, false>, grid, kSimtThreads, 0, s, a, lv, accumulate);
  else xu_launch(pose_dgrad_simt_kernel<bf16, true>, grid, kSimtThreads, 0, s, a, lv, accumulate);
}

void launch_camera_grad(const PoseGradArgs& a, float* dR1, float* dt1, float* dR2, float* dt2, float* dK, cudaStream_t s) {
  xu_launch(camera_grad_kernel, a.B, kCamThreads, 0, s, a.d_rays, a.R1, a.R2, a.K, a.S, a.convention, dR1, dt1, dR2, dt2, dK);
}
