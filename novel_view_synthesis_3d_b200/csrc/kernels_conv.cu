// kernels_conv.cu -- SIMT implicit-GEMM convolution (forward / data-gradient / weight-gradient).
//
// This is the exact-fp32 path ("verify mode", XUNET_DTYPE_F32) and the fallback for shapes the tensor-core
// kernel (conv_tc.cu) does not take (Cin=3 input conv, Cout=3 output conv, strided pose convs).
// Replaces flax nn.Conv / nn.Dense / nn.DenseGeneral as called from model/xunet.py:59,81,85-89,91,
// 100-102,199,229,276 and their XLA-autodiff gradients (train.py:70).
#include "common.cuh"
#include "kernels.h"

__device__ __forceinline__ long long conv_waddr(int tap, int ci, int co, int taps, int wCi, int segw) {
  int seg = co / segw;
  return (long long)seg * taps * wCi * segw + ((long long)tap * wCi + ci) * segw + (co - seg * segw);
}

template <typename T, int BM, int BN>
__global__ void __launch_bounds__(256) conv_simt_kernel(ConvArgs a) {
  xu_grid_dep_sync();
  constexpr int BK = 16;
  constexpr int TX = BN / 4;
  __shared__ float As[BK][BM + 1];
  __shared__ __align__(16) float Bs[BK][BN];
  __shared__ int pn[BM], py[BM], px[BM];
  const T* __restrict__ x = reinterpret_cast<const T*>(a.x);
  const int tid = threadIdx.x;
  const long long M = (long long)a.N * a.Ho * a.Wo;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  for (int i = tid; i < BM; i += 256) {
    long long m = m0 + i;
    if (m < M) {
      int ox = (int)(m % a.Wo);
      long long t = m / a.Wo;
      px[i] = ox; py[i] = (int)(t % a.Ho); pn[i] = (int)(t / a.Ho);
    } else {
      pn[i] = -1; py[i] = 0; px[i] = 0;
    }
  }
  __syncthreads();
  const int taps = a.ks * a.ks;
  const int Ktot = taps * a.Ci;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int tx = tid % TX, ty = tid / TX;

  for (int k0 = 0; k0 < Ktot; k0 += BK) {
    {  // A tile: BM pixels x 16 k
      const int kk = tid & 15;
      const int k = k0 + kk;
      const bool kvalid = k < Ktot;
      int tap = 0, ci = 0;
      if (kvalid) { tap = k / a.Ci; ci = k - tap * a.Ci; }
      const int dy = tap / a.ks, dx = tap - dy * a.ks;
#pragma unroll
      for (int r = 0; r < BM / 16; ++r) {
        const int i = (tid >> 4) + 16 * r;
        float v = 0.f;
        const int n = pn[i];
        if (kvalid && n >= 0) {
          int iy, ix;
          bool ok;
          if (a.mode == 0) {
            iy = py[i] * a.stride + dy - a.pad_h;
            ix = px[i] * a.stride + dx - a.pad_w;
            ok = iy >= 0 && iy < a.Hi && ix >= 0 && ix < a.Wi;
          } else {
            int ty_ = py[i] + a.pad_h - dy, tx_ = px[i] + a.pad_w - dx;
            ok = ty_ >= 0 && tx_ >= 0 && (ty_ % a.stride) == 0 && (tx_ % a.stride) == 0;
            iy = ty_ / a.stride; ix = tx_ / a.stride;
            ok = ok && iy < a.Hi && ix < a.Wi;
          }
          if (ok) v = ldf(x + (((long long)n * a.Hi + iy) * a.Wi + ix) * a.Ci + ci);
        }
        As[kk][i] = v;
      }
    }
    {  // B tile: 16 k x BN
#pragma unroll
      for (int r = 0; r < (BK * BN) / 256; ++r) {
        const int idx = tid + 256 * r;
        const int kk = idx / BN, nn = idx - kk * BN;
        const int k = k0 + kk, col = n0 + nn;
        float v = 0.f;
        if (k < Ktot && col < a.Co) {
          int tap = k / a.Ci, kc = k - tap * a.Ci;
          long long wa = (a.mode == 0) ? conv_waddr(tap, kc, col, taps, a.wCi, a.segw)
                                       : conv_waddr(tap, col, kc, taps, a.wCi, a.segw);
          v = a.w[wa];
        }
        Bs[kk][nn] = v;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float av[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[kk][ty * 4 + i];
      float4 b4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      float bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }

  T* __restrict__ y = reinterpret_cast<T*>(a.y);
  const T* __restrict__ res = reinterpret_cast<const T*>(a.res);
  const int c0 = n0 + tx * 4;
  const bool vec = (a.Co % 4 == 0) && (c0 + 3 < a.Co);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= M) continue;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[j] = acc[i][j];
      if (a.bias != nullptr && c0 + j < a.Co) v[j] += a.bias[c0 + j];
    }
    const long long base = m * a.Co + c0;
    if (vec) {
      if (res != nullptr) {
        float rv[4];
        Vec4<T>::ld(res + base, rv);
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] += rv[j];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] *= a.alpha;
      if (a.accumulate) {
        float ov[4];
        Vec4<T>::ld(y + base, ov);
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] += ov[j];
      }
      Vec4<T>::st(y + base, v);
    } else {
      for (int j = 0; j < 4; ++j) {
        if (c0 + j >= a.Co) break;
        float o = v[j];
        if (res != nullptr) o += ldf(res + base + j);
        o *= a.alpha;
        if (a.accumulate) o += ldf(y + base + j);
        stf(y + base + j, o);
      }
    }
  }
}

template <typename T>
static void conv_dispatch(const ConvArgs& a, cudaStream_t s) {
  const long long M = (long long)a.N * a.Ho * a.Wo;
  if (a.Co <= 32) {
    dim3 grid(cdiv(M, 128), cdiv(a.Co, 32));
    xu_launch(conv_simt_kernel<T, 128, 32>, grid, 256, 0, s, a);
  } else {
    dim3 grid(cdiv(M, 64), cdiv(a.Co, 64));
    xu_launch(conv_simt_kernel<T, 64, 64>, grid, 256, 0, s, a);
  }
}

void launch_conv_simt(int dtype, const ConvArgs& a, cudaStream_t s) {
  if (dtype == XU_F32) conv_dispatch<float>(a, s);
  else conv_dispatch<bf16>(a, s);
}

// ------------------------------------------------------------------------------------------------------
// weight gradient: split-K over output pixels, fp32 atomics into the flat gradient buffer
// ------------------------------------------------------------------------------------------------------
template <typename T, int TM, int TN, int RM, int RN>
__global__ void __launch_bounds__(256) wgrad_simt_kernel(WgradArgs a) {
  xu_grid_dep_sync();
  constexpr int PK = 16;
  constexpr int TXN = TN / RN;
  static_assert((TM / RM) * (TN / RN) == 256, "thread tiling");
  __shared__ float As[PK][TM + 1];
  __shared__ float Bs[PK][TN + 1];
  const T* __restrict__ x = reinterpret_cast<const T*>(a.x);
  const T* __restrict__ dy = reinterpret_cast<const T*>(a.dy);
  const int tid = threadIdx.x;
  const int tiles_co = (a.Co + TN - 1) / TN;
  const int tile_ci = blockIdx.x / tiles_co, tile_co = blockIdx.x - tile_ci * tiles_co;
  const int tap = blockIdx.y;
  const int tdy = tap / a.ks, tdx = tap - tdy * a.ks;
  const long long M = (long long)a.N * a.Ho * a.Wo;
  const long long chunks = (M + PK - 1) / PK;
  const long long per = (chunks + gridDim.z - 1) / gridDim.z;
  const long long cbeg = (long long)blockIdx.z * per;
  const long long cend = (cbeg + per < chunks) ? cbeg + per : chunks;
  const int txx = tid % TXN, tyy = tid / TXN;
  float acc[RM][RN];
#pragma unroll
  for (int i = 0; i < RM; ++i)
#pragma unroll
    for (int j = 0; j < RN; ++j) acc[i][j] = 0.f;
  const bool do_bias = (a.dbias != nullptr) && blockIdx.y == 0 && tile_ci == 0;
  float bsum = 0.f;
  const int pp = tid >> 4, lane16 = tid & 15;

  for (long long ch = cbeg; ch < cend; ++ch) {
    const long long m = ch * PK + pp;
    bool ok = false;
    long long xbase = 0;
    if (m < M) {
      int ox = (int)(m % a.Wo);
      long long t = m / a.Wo;
      int oy = (int)(t % a.Ho);
      int n = (int)(t / a.Ho);
      int iy = oy * a.stride + tdy - a.pad_h, ix = ox * a.stride + tdx - a.pad_w;
      ok = iy >= 0 && iy < a.Hi && ix >= 0 && ix < a.Wi;
      xbase = (((long long)n * a.Hi + iy) * a.Wi + ix) * a.Ci;
    }
#pragma unroll
    for (int r = 0; r < TM / 16; ++r) {
      const int c = lane16 + 16 * r;
      const int ci = tile_ci * TM + c;
      float v = 0.f;
      if (ok && ci < a.Ci) v = ldf(x + xbase + ci);
      As[pp][c] = v;
    }
#pragma unroll
    for (int r = 0; r < TN / 16; ++r) {
      const int c = lane16 + 16 * r;
      const int co = tile_co * TN + c;
      float v = 0.f;
      if (m < M && co < a.Co) v = ldf(dy + m * a.Co + co);
      Bs[pp][c] = v;
    }
    __syncthreads();
#pragma unroll
    for (int p = 0; p < PK; ++p) {
      float av[RM], bv[RN];
#pragma unroll
      for (int i = 0; i < RM; ++i) av[i] = As[p][tyy * RM + i];
#pragma unroll
      for (int j = 0; j < RN; ++j) bv[j] = Bs[p][txx * RN + j];
#pragma unroll
      for (int i = 0; i < RM; ++i)
#pragma unroll
        for (int j = 0; j < RN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (do_bias && tid < TN) {
#pragma unroll
      for (int p = 0; p < PK; ++p) bsum += Bs[p][tid];
    }
    __syncthreads();
  }
  const int taps = a.ks * a.ks;
#pragma unroll
  for (int i = 0; i < RM; ++i) {
    const int ci = tile_ci * TM + tyy * RM + i;
    if (ci >= a.Ci) continue;
#pragma unroll
    for (int j = 0; j < RN; ++j) {
      const int co = tile_co * TN + txx * RN + j;
      if (co >= a.Co) continue;
      xu_det_add(a.acc_dw + conv_waddr(tap, ci, co, taps, a.Ci, a.segw), a.alpha * acc[i][j]);
    }
  }
  if (do_bias && tid < TN) {
    const int co = tile_co * TN + tid;
    if (co < a.Co) xu_det_add(a.acc_db + co, a.alpha * bsum);
  }
}

template <typename T>
static void wgrad_dispatch(const WgradArgs& a, cudaStream_t s) {
  const long long M = (long long)a.N * a.Ho * a.Wo;
  const long long chunks = (M + 15) / 16;
  const int taps = a.ks * a.ks;
  if (a.Ci >= 48 && a.Co >= 48) {
    int tiles = cdiv(a.Ci, 64) * cdiv(a.Co, 64);
    long long ks = (4 * xu_num_sms() + (long long)tiles * taps - 1) / ((long long)tiles * taps);
    if (ks < 1) ks = 1;
    if (ks > chunks) ks = chunks;
    if (ks > 65535) ks = 65535;
    dim3 grid(tiles, taps, (unsigned)ks);
    xu_launch(wgrad_simt_kernel<T, 64, 64, 4, 4>, grid, 256, 0, s, a);
  } else {
    int tiles = cdiv(a.Ci, 32) * cdiv(a.Co, 32);
    long long ks = (4 * xu_num_sms() + (long long)tiles * taps - 1) / ((long long)tiles * taps);
    if (ks < 1) ks = 1;
    if (ks > chunks) ks = chunks;
    if (ks > 65535) ks = 65535;
    dim3 grid(tiles, taps, (unsigned)ks);
    xu_launch(wgrad_simt_kernel<T, 32, 32, 2, 2>, grid, 256, 0, s, a);
  }
}

// Runs `launch` with the weight (and bias) gradient accumulated in fp64 scratch and folded into a.dw / a.dbias afterwards, so
// that the result does not depend on the order of the split-K contributions.
template <typename F>
static void det_wgrad(const WgradArgs& a0, cudaStream_t s, F launch) {
  WgradArgs a = a0;
  const long long ndw = (long long)a.ks * a.ks * a.Ci * a.Co, ndb = a.dbias ? a.Co : 0;
  double* acc = xu_det_scratch(s, ndw + ndb);
  if (acc == nullptr) return;
  a.acc_dw = acc;
  a.acc_db = a.dbias ? acc + ndw : nullptr;
  launch(a);
  xu_det_fold(a.dw, acc, ndw, s);
  if (a.dbias) xu_det_fold(a.dbias, acc + ndw, ndb, s);
}

void launch_wgrad_simt(int dtype, const WgradArgs& a, cudaStream_t s) {
  det_wgrad(a, s, [&](const WgradArgs& aa) {
    if (dtype == XU_F32) wgrad_dispatch<float>(aa, s);
    else wgrad_dispatch<bf16>(aa, s);
  });
}

// ======================================================================================================
// Direct kernels for the two 3-channel convolutions: the input conv 3 -> ch (model/xunet.py:229) and the output
// conv ch -> 3 (model/xunet.py:276).  K (resp. N) = 3 is far too thin for a GEMM tile, so these stay on the SIMT
// pipes: one thread per output pixel (x 8-channel group), weights broadcast from shared memory.
// ======================================================================================================
template <typename T>
__global__ void __launch_bounds__(256) conv_cin3_fwd_kernel(ConvArgs a) {
  xu_grid_dep_sync();
  extern __shared__ float sw[];                 // [27][Co] weights + [Co] bias
  const int Co = a.Co;
  for (int i = threadIdx.x; i < 27 * Co; i += 256) sw[i] = a.w[i];
  for (int i = threadIdx.x; i < Co; i += 256) sw[27 * Co + i] = a.bias ? a.bias[i] : 0.f;
  __syncthreads();
  const int G = Co >> 3;
  const long long total = (long long)a.N * a.Ho * a.Wo * G;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int ox = (int)(pix % a.Wo);
  const int oy = (int)((pix / a.Wo) % a.Ho);
  const int n = (int)(pix / ((long long)a.Wo * a.Ho));
  const T* x = reinterpret_cast<const T*>(a.x);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = sw[27 * Co + g * 8 + j];
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const int iy = oy + tap / 3 - 1, ix = ox + tap % 3 - 1;
    if (iy < 0 || iy >= a.Hi || ix < 0 || ix >= a.Wi) continue;
    const T* px = x + (((long long)n * a.Hi + iy) * a.Wi + ix) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = ldf(px + c);
      const float* wr = sw + (tap * 3 + c) * Co + g * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(v, wr[j], acc[j]);
    }
  }
  T* y = reinterpret_cast<T*>(a.y) + pix * Co + g * 8;
  float o0[4] = {acc[0] * a.alpha, acc[1] * a.alpha, acc[2] * a.alpha, acc[3] * a.alpha};
  float o1[4] = {acc[4] * a.alpha, acc[5] * a.alpha, acc[6] * a.alpha, acc[7] * a.alpha};
  Vec4<T>::st(y, o0);
  Vec4<T>::st(y + 4, o1);
}

// dW[27][Co] (+ dbias as row 27) = sum over pixels of patch (x) dY ; one block per chunk of 128 pixels
template <typename T>
__global__ void __launch_bounds__(256) conv_cin3_wgrad_kernel(WgradArgs a) {
  xu_grid_dep_sync();
  constexpr int PPB = 128;
  __shared__ float xs[PPB][28];
  const T* x = reinterpret_cast<const T*>(a.x);
  const T* dy = reinterpret_cast<const T*>(a.dy);
  const long long M = (long long)a.N * a.Ho * a.Wo;
  const long long p0 = (long long)blockIdx.x * PPB;
  for (int i = threadIdx.x; i < PPB * 28; i += 256) {
    const int pp = i / 28, k = i - pp * 28;
    const long long m = p0 + pp;
    float v = 0.f;
    if (m < M) {
      if (k == 27) v = 1.f;
      else {
        const int tap = k / 3, c = k - tap * 3;
        const int ox = (int)(m % a.Wo);
        const int oy = (int)((m / a.Wo) % a.Ho);
        const int n = (int)(m / ((long long)a.Wo * a.Ho));
        const int iy = oy + tap / 3 - 1, ix = ox + tap % 3 - 1;
        if (iy >= 0 && iy < a.Hi && ix >= 0 && ix < a.Wi) v = ldf(x + (((long long)n * a.Hi + iy) * a.Wi + ix) * 3 + c);
      }
    }
    xs[pp][k] = v;
  }
  __syncthreads();
  const int G = a.Co >> 2;
  const int items = 28 * G;
  const int npix = (int)((M - p0) < PPB ? (M - p0) : PPB);
  for (int it = threadIdx.x; it < items; it += 256) {
    const int k = it / G, g = it - k * G;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int pp = 0; pp < npix; ++pp) {
      float d[4];
      Vec4<T>::ld(dy + (p0 + pp) * a.Co + g * 4, d);
      const float xv = xs[pp][k];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = fmaf(xv, d[j], acc[j]);
    }
    double* dst = (k == 27) ? (a.dbias ? a.acc_db + g * 4 : nullptr) : a.acc_dw + (long long)k * a.Co + g * 4;
    if (dst)
#pragma unroll
      for (int j = 0; j < 4; ++j) xu_det_add(dst + j, a.alpha * acc[j]);
  }
}

// Data gradient of the input conv, fused with the un-pack of its (2B,S,S,3) input (the adjoint of pack_input_kernel):
//   dX[n, p, c] = alpha * sum_tap sum_co dY[n, p - tap, co] * W[tap, c, co]     (SAME padding 1)
// row n = 2b goes to dx[b], row 2b + 1 to dz[b], both fp32 (B,S,S,3); fsel = 0 / 1 computes only the dx / dz rows, -1 both.
// A group of LP lanes (a power of two <= 32) owns one pixel: lane l reads the 16-byte chunks l, l + LP, ... of dY at each of the
// 9 neighbours and keeps three fp32 partial sums, tap by tap; the group then adds its lanes with a fixed xor tree.  The order
// depends on Co alone, so the bits depend neither on the grid nor on where a pixel sits in it.  Whole warps iterate together
// (the shuffles need every lane); lanes past the end contribute zeros and store nothing.
template <typename T>
__global__ void __launch_bounds__(256) conv_cin3_dgrad_unpack_kernel(const T* __restrict__ dy, const float* __restrict__ w,
                                                                     float* __restrict__ dx, float* __restrict__ dz, int B, int S,
                                                                     int Co, int LP, float alpha, int fsel) {
  xu_grid_dep_sync();
  extern __shared__ float sw[];                 // [27][Co]: the fp32 kernel (1,3,3,3,Co)
  for (int i = threadIdx.x; i < 27 * Co; i += 256) sw[i] = w[i];
  __syncthreads();
  constexpr int V = VecW<T>::W;
  const int nchunk = Co / V;
  const int lane = threadIdx.x & (LP - 1);
  const int gpw = 32 / LP;                      // pixel groups per warp
  const long long npix = (long long)(fsel < 0 ? 2 * B : B) * S * S;
  const long long wstep = (long long)gridDim.x * (blockDim.x >> 5) * gpw;
  for (long long q0 = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * gpw; q0 < npix; q0 += wstep) {
    const long long q = q0 + ((threadIdx.x & 31) / LP);
    const bool valid = q < npix;
    const long long img = valid ? q / ((long long)S * S) : 0;
    const int pix = valid ? (int)(q - img * S * S) : 0;
    const int iy = pix / S, ix = pix - iy * S;
    const long long b = fsel < 0 ? img >> 1 : img;
    const int f = fsel < 0 ? (int)(img & 1) : fsel;
    const long long n = 2 * b + f;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    if (valid) {
#pragma unroll 1
      for (int tap = 0; tap < 9; ++tap) {
        const int oy = iy + 1 - tap / 3, ox = ix + 1 - tap % 3;
        if (oy < 0 || oy >= S || ox < 0 || ox >= S) continue;
        const T* src = dy + ((n * S + oy) * S + ox) * Co;
        const float* wt = sw + tap * 3 * Co;
        for (int k = lane; k < nchunk; k += LP) {
          float d[V];
          VecW<T>::unpack(VecW<T>::ldg(src + k * V), d);
#pragma unroll
          for (int j4 = 0; j4 < V; j4 += 4) {
            const float4 w0 = *reinterpret_cast<const float4*>(wt + k * V + j4);
            const float4 w1 = *reinterpret_cast<const float4*>(wt + Co + k * V + j4);
            const float4 w2 = *reinterpret_cast<const float4*>(wt + 2 * Co + k * V + j4);
            a0 = fmaf(d[j4], w0.x, a0); a0 = fmaf(d[j4 + 1], w0.y, a0); a0 = fmaf(d[j4 + 2], w0.z, a0); a0 = fmaf(d[j4 + 3], w0.w, a0);
            a1 = fmaf(d[j4], w1.x, a1); a1 = fmaf(d[j4 + 1], w1.y, a1); a1 = fmaf(d[j4 + 2], w1.z, a1); a1 = fmaf(d[j4 + 3], w1.w, a1);
            a2 = fmaf(d[j4], w2.x, a2); a2 = fmaf(d[j4 + 1], w2.y, a2); a2 = fmaf(d[j4 + 2], w2.z, a2); a2 = fmaf(d[j4 + 3], w2.w, a2);
          }
        }
      }
    }
    for (int o = LP >> 1; o > 0; o >>= 1) {     // lanes i and i^o add the same two values: every lane ends with the same bits
      a0 += __shfl_xor_sync(0xffffffffu, a0, o);
      a1 += __shfl_xor_sync(0xffffffffu, a1, o);
      a2 += __shfl_xor_sync(0xffffffffu, a2, o);
    }
    if (valid && lane == 0) {
      float* out = (f ? dz : dx) + ((b * S + iy) * S + ix) * 3;
      out[0] = alpha * a0; out[1] = alpha * a1; out[2] = alpha * a2;
    }
  }
}

void launch_conv_cin3_dgrad_unpack(int dtype, const void* dy, const float* w, float* dx, float* dz, int B, int S, int Co,
                                   float alpha, cudaStream_t s) {
  if (dx == nullptr && dz == nullptr) return;
  const int fsel = (dx != nullptr && dz != nullptr) ? -1 : (dx != nullptr ? 0 : 1);
  const int nchunk = Co / (dtype == XU_F32 ? 4 : 8);
  int LP = 1;
  while (LP * 2 <= nchunk && LP < 32) LP *= 2;
  const long long npix = (long long)(fsel < 0 ? 2 * B : B) * S * S;
  const int grid = (int)std::min<long long>(cdiv(npix, 256 / LP), (long long)xu_num_sms() * 4);
  const size_t sm = sizeof(float) * 27 * Co;
  if (dtype == XU_F32) {
    if (sm > 48 * 1024) cudaFuncSetAttribute(conv_cin3_dgrad_unpack_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    xu_launch(conv_cin3_dgrad_unpack_kernel<float>, grid, 256, sm, s, (const float*)dy, w, dx, dz, B, S, Co, LP, alpha, fsel);
  } else {
    if (sm > 48 * 1024) cudaFuncSetAttribute(conv_cin3_dgrad_unpack_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    xu_launch(conv_cin3_dgrad_unpack_kernel<bf16>, grid, 256, sm, s, (const bf16*)dy, w, dx, dz, B, S, Co, LP, alpha, fsel);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) conv_cout3_fwd_kernel(ConvArgs a) {
  xu_grid_dep_sync();
  extern __shared__ float sw[];                 // [9][Ci][3]
  const int Ci = a.Ci;
  for (int i = threadIdx.x; i < 27 * Ci; i += 256) sw[i] = a.w[i];
  __syncthreads();
  const long long total = (long long)a.N * a.Ho * a.Wo;
  const long long pix = (long long)blockIdx.x * 256 + threadIdx.x;
  if (pix >= total) return;
  const int ox = (int)(pix % a.Wo);
  const int oy = (int)((pix / a.Wo) % a.Ho);
  const int n = (int)(pix / ((long long)a.Wo * a.Ho));
  const T* x = reinterpret_cast<const T*>(a.x);
  float acc[3] = {a.bias ? a.bias[0] : 0.f, a.bias ? a.bias[1] : 0.f, a.bias ? a.bias[2] : 0.f};
  for (int tap = 0; tap < 9; ++tap) {
    const int iy = oy + tap / 3 - 1, ix = ox + tap % 3 - 1;
    if (iy < 0 || iy >= a.Hi || ix < 0 || ix >= a.Wi) continue;
    const T* px = x + (((long long)n * a.Hi + iy) * a.Wi + ix) * Ci;
    const float* wr = sw + tap * Ci * 3;
    for (int c = 0; c < Ci; c += 4) {
      float v[4];
      Vec4<T>::ld(px + c, v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[0] = fmaf(v[j], wr[(c + j) * 3 + 0], acc[0]);
        acc[1] = fmaf(v[j], wr[(c + j) * 3 + 1], acc[1]);
        acc[2] = fmaf(v[j], wr[(c + j) * 3 + 2], acc[2]);
      }
    }
  }
  T* y = reinterpret_cast<T*>(a.y) + pix * 3;
  stf(y, acc[0] * a.alpha); stf(y + 1, acc[1] * a.alpha); stf(y + 2, acc[2] * a.alpha);
}

// dX[pix][ci] (+)= alpha * sum_{tap,co} dO[pix + 1 - tap][co] W[tap][ci][co]      (a.x = dO (N,H,W,3), a.y = dX (N,H,W,Ci=a.Co))
template <typename T>
__global__ void __launch_bounds__(256) conv_cout3_dgrad_kernel(ConvArgs a) {
  xu_grid_dep_sync();
  extern __shared__ float sw[];                 // [9][Ci][3]
  const int Ci = a.Co;
  for (int i = threadIdx.x; i < 27 * Ci; i += 256) sw[i] = a.w[i];
  __syncthreads();
  const int G = Ci >> 3;
  const long long total = (long long)a.N * a.Ho * a.Wo * G;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int ix0 = (int)(pix % a.Wo);
  const int iy0 = (int)((pix / a.Wo) % a.Ho);
  const int n = (int)(pix / ((long long)a.Wo * a.Ho));
  const T* d = reinterpret_cast<const T*>(a.x);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const int oy = iy0 + 1 - tap / 3, ox = ix0 + 1 - tap % 3;
    if (oy < 0 || oy >= a.Hi || ox < 0 || ox >= a.Wi) continue;
    const T* pd = d + (((long long)n * a.Hi + oy) * a.Wi + ox) * 3;
    const float d0 = ldf(pd), d1 = ldf(pd + 1), d2 = ldf(pd + 2);
    const float* wr = sw + (tap * Ci + g * 8) * 3;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += d0 * wr[j * 3] + d1 * wr[j * 3 + 1] + d2 * wr[j * 3 + 2];
  }
  T* y = reinterpret_cast<T*>(a.y) + pix * Ci + g * 8;
  float o0[4], o1[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { o0[j] = acc[j] * a.alpha; o1[j] = acc[4 + j] * a.alpha; }
  if (a.accumulate) {
    float p0[4], p1[4];
    Vec4<T>::ld(y, p0); Vec4<T>::ld(y + 4, p1);
#pragma unroll
    for (int j = 0; j < 4; ++j) { o0[j] += p0[j]; o1[j] += p1[j]; }
  }
  Vec4<T>::st(y, o0);
  Vec4<T>::st(y + 4, o1);
}

// dW[9][Ci][3] += alpha * sum_pix x[pix + tap - 1][ci] dO[pix][co];  dbias[3] += alpha * sum dO
template <typename T>
__global__ void __launch_bounds__(320) conv_cout3_wgrad_kernel(WgradArgs a) {
  xu_grid_dep_sync();
  constexpr int PPB = 128;
  __shared__ float ds[PPB][3];
  __shared__ int sy[PPB], sx[PPB], sn[PPB];
  const T* x = reinterpret_cast<const T*>(a.x);
  const T* dy = reinterpret_cast<const T*>(a.dy);
  const long long M = (long long)a.N * a.Ho * a.Wo;
  const long long p0 = (long long)blockIdx.x * PPB;
  if (threadIdx.x < PPB) {
    const int pp = threadIdx.x;
    const long long m = p0 + pp;
    if (m < M) {
      sx[pp] = (int)(m % a.Wo); sy[pp] = (int)((m / a.Wo) % a.Ho); sn[pp] = (int)(m / ((long long)a.Wo * a.Ho));
      ds[pp][0] = ldf(dy + m * 3); ds[pp][1] = ldf(dy + m * 3 + 1); ds[pp][2] = ldf(dy + m * 3 + 2);
    } else { sn[pp] = -1; ds[pp][0] = ds[pp][1] = ds[pp][2] = 0.f; sx[pp] = sy[pp] = 0; }
  }
  __syncthreads();
  const int items = 9 * a.Ci;
  for (int it = threadIdx.x; it < items; it += blockDim.x) {
    const int tap = it / a.Ci, ci = it - tap * a.Ci;
    const int dyy = tap / 3 - 1, dxx = tap % 3 - 1;
    float acc[3] = {0.f, 0.f, 0.f};
    for (int pp = 0; pp < PPB; ++pp) {
      const int n = sn[pp];
      if (n < 0) break;
      const int iy = sy[pp] + dyy, ix = sx[pp] + dxx;
      if (iy < 0 || iy >= a.Hi || ix < 0 || ix >= a.Wi) continue;
      const float xv = ldf(x + (((long long)n * a.Hi + iy) * a.Wi + ix) * a.Ci + ci);
      acc[0] = fmaf(xv, ds[pp][0], acc[0]); acc[1] = fmaf(xv, ds[pp][1], acc[1]); acc[2] = fmaf(xv, ds[pp][2], acc[2]);
    }
    double* dst = a.acc_dw + (long long)it * 3;
    xu_det_add(dst, a.alpha * acc[0]); xu_det_add(dst + 1, a.alpha * acc[1]); xu_det_add(dst + 2, a.alpha * acc[2]);
  }
  if (a.dbias != nullptr && threadIdx.x < 3) {
    float sacc = 0.f;
    for (int pp = 0; pp < PPB; ++pp) sacc += ds[pp][threadIdx.x];
    xu_det_add(a.acc_db + threadIdx.x, a.alpha * sacc);
  }
}


// ------------------------------------------------------------------------------------------------------
// Round-2 versions of the 3-channel kernels.  The round-1 kernels above reloaded the whole weight matrix into shared memory for
// every 8 pixels, paid one shared-memory load per FMA (8-way bank conflicts on top) and three atomics per (tap, channel, 128 pixels).
// These are persistent,
// register-blocked over 4 pixels (one weight fetch serves 4 pixels), read weights with conflict-free 16-byte LDS, and the weight
// gradients keep their 27 x 2 accumulators in registers over a whole pixel range before one reduction per CTA.
// ------------------------------------------------------------------------------------------------------
template <typename T> struct Io8;   // 8 consecutive elements <-> float[8]
template <> struct Io8<float> {
  static __device__ __forceinline__ void ld(const float* p, float (&v)[8]) {
    float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  static __device__ __forceinline__ void ldrw(const float* p, float (&v)[8]) {
    float4 a = *reinterpret_cast<const float4*>(p), b = *(reinterpret_cast<const float4*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  static __device__ __forceinline__ void st(float* p, const float (&v)[8]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    *(reinterpret_cast<float4*>(p) + 1) = make_float4(v[4], v[5], v[6], v[7]);
  }
};
template <> struct Io8<bf16> {
  static __device__ __forceinline__ void ld(const bf16* p, float (&v)[8]) { VecW<bf16>::unpack(VecW<bf16>::ldg(p), v); }
  static __device__ __forceinline__ void ldrw(const bf16* p, float (&v)[8]) { VecW<bf16>::unpack(VecW<bf16>::ld(p), v); }
  static __device__ __forceinline__ void st(bf16* p, const float (&v)[8]) { VecW<bf16>::st(p, v); }
};
template <typename T> __device__ __forceinline__ void ld2f(const T* p, float& a, float& b);
template <> __device__ __forceinline__ void ld2f<float>(const float* p, float& a, float& b) {
  float2 t = __ldg(reinterpret_cast<const float2*>(p)); a = t.x; b = t.y;
}
template <> __device__ __forceinline__ void ld2f<bf16>(const bf16* p, float& a, float& b) {
  uint32_t t = __ldg(reinterpret_cast<const uint32_t*>(p)); a = __uint_as_float(t << 16); b = __uint_as_float(t & 0xFFFF0000u);
}

// (A) thin -> wide: out[pix][Cw] = alpha * (bias + sum_{window pos, c3} thin[pix + pos - 1][c3] * Wt[pos*3 + c3][Cw])  (+= if accumulate)
//   FLIP = 0: the input convolution (a.x = image (N,H,W,3), a.w = [27][Co] rows (tap, c), bias)
//   FLIP = 1: the data gradient of the output convolution (a.x = dO (N,H,W,3), a.w = [9][Ci][3]; window pos <-> tap 8 - pos)
// work item = 4 consecutive pixels of one row x one group of 8 wide channels (g fastest: a warp stores 512 contiguous bytes per pixel)
template <typename T, int FLIP>
__global__ void __launch_bounds__(256) conv_thin_in_kernel(ConvArgs a) {
  xu_grid_dep_sync();
  extern __shared__ float4 sw4[];               // [28 rows][2 halves][G] float4: row r, channels g*8 + half*4 .. +3 ; row 27 = bias
  const int Cw = a.Co, G = Cw >> 3;
  float* sw = reinterpret_cast<float*>(sw4);
  for (int i = threadIdx.x; i < 28 * Cw; i += 256) {
    const int r = i / Cw, ch = i - r * Cw;
    float v;
    if (r == 27) v = (!FLIP && a.bias) ? a.bias[ch] : 0.f;
    else if (!FLIP) v = a.w[i];
    else { const int pos = r / 3, k = r - pos * 3; v = a.w[((8 - pos) * Cw + ch) * 3 + k]; }
    sw[((r * 2 + ((ch >> 2) & 1)) * G + (ch >> 3)) * 4 + (ch & 3)] = v;
  }
  __syncthreads();
  const int W4 = a.Wo >> 2;
  const long long total = (long long)a.N * a.Ho * W4 * G;
  const T* x = reinterpret_cast<const T*>(a.x);
  for (long long idx = (long long)blockIdx.x * 256 + threadIdx.x; idx < total; idx += (long long)gridDim.x * 256) {
    const int g = (int)(idx % G);
    const long long quad = idx / G;
    const int ox0 = (int)(quad % W4) << 2;
    const int oy = (int)((quad / W4) % a.Ho);
    const int n = (int)(quad / ((long long)W4 * a.Ho));
    float acc[4][8];
    {
      const float4 b0 = sw4[(27 * 2 + 0) * G + g], b1 = sw4[(27 * 2 + 1) * G + g];
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        acc[p][0] = b0.x; acc[p][1] = b0.y; acc[p][2] = b0.z; acc[p][3] = b0.w;
        acc[p][4] = b1.x; acc[p][5] = b1.y; acc[p][6] = b1.z; acc[p][7] = b1.w;
      }
    }
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = oy + ky - 1;
      if (iy < 0 || iy >= a.Hi) continue;
      const T* row = x + ((long long)n * a.Hi + iy) * a.Wi * 3;
      float tv[18];                             // columns ox0-1 .. ox0+4, 3 channels each
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const int ix = ox0 - 1 + c;
        const bool in = ix >= 0 && ix < a.Wi;
#pragma unroll
        for (int k = 0; k < 3; ++k) tv[c * 3 + k] = in ? ldf(row + ix * 3 + k) : 0.f;
      }
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int r = (ky * 3 + kx) * 3 + k;
          const float4 w0 = sw4[(r * 2 + 0) * G + g], w1 = sw4[(r * 2 + 1) * G + g];
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            const float v = tv[(p + kx) * 3 + k];
            acc[p][0] = fmaf(v, w0.x, acc[p][0]); acc[p][1] = fmaf(v, w0.y, acc[p][1]);
            acc[p][2] = fmaf(v, w0.z, acc[p][2]); acc[p][3] = fmaf(v, w0.w, acc[p][3]);
            acc[p][4] = fmaf(v, w1.x, acc[p][4]); acc[p][5] = fmaf(v, w1.y, acc[p][5]);
            acc[p][6] = fmaf(v, w1.z, acc[p][6]); acc[p][7] = fmaf(v, w1.w, acc[p][7]);
          }
        }
      }
    }
    T* y = reinterpret_cast<T*>(a.y) + ((((long long)n * a.Ho + oy) * a.Wo + ox0) * Cw + g * 8);
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = acc[p][j] * a.alpha;
      if (a.accumulate) {
        float old[8];
        Io8<T>::ldrw(y + (long long)p * Cw, old);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += old[j];
      }
      Io8<T>::st(y + (long long)p * Cw, o);
    }
  }
}

// (C) wide -> thin: the output convolution.  L = Ci/8 lanes share 4 consecutive pixels, each lane owning 8 input channels (16-byte
// coalesced loads of the 6 input columns a row of the window touches); the 4 x 3 partial sums are reduced over the L lanes by shuffles.
template <typename T>
__global__ void __launch_bounds__(256) conv_cout3_fwd4_kernel(ConvArgs a) {
  xu_grid_dep_sync();
  extern __shared__ float4 sw4[];               // [9 taps][6][L] float4: the 24 weights (8 channels x 3 outputs) of lane l at tap t
  const int Ci = a.Ci, L = Ci >> 3;
  float* sw = reinterpret_cast<float*>(sw4);
  for (int i = threadIdx.x; i < 27 * Ci; i += 256) {
    const int tap = i / (Ci * 3), rem = i - tap * Ci * 3;      // rem = ci*3 + k
    const int l = rem / 24, e = rem - l * 24;                  // lane, element within the lane's 24 floats
    sw[((tap * 6 + (e >> 2)) * L + l) * 4 + (e & 3)] = a.w[i];
  }
  __syncthreads();
  const int W4 = a.Wo >> 2;
  const long long quads = (long long)a.N * a.Ho * W4;
  const int qpb = 256 / L;                      // quads per block iteration
  const int l = threadIdx.x % L;
  const T* x = reinterpret_cast<const T*>(a.x);
  const float b0 = a.bias ? a.bias[0] : 0.f, b1 = a.bias ? a.bias[1] : 0.f, b2 = a.bias ? a.bias[2] : 0.f;
  const long long iters = (quads + qpb - 1) / qpb;
  for (long long it = blockIdx.x; it < iters; it += gridDim.x) {
    const long long quad = it * qpb + threadIdx.x / L;
    const bool live = quad < quads;              // dead lanes still take part in the shuffles
    const int ox0 = live ? (int)(quad % W4) << 2 : 0;
    const int oy = live ? (int)((quad / W4) % a.Ho) : 0;
    const int n = live ? (int)(quad / ((long long)W4 * a.Ho)) : 0;
    float acc[4][3];
#pragma unroll
    for (int p = 0; p < 4; ++p) acc[p][0] = acc[p][1] = acc[p][2] = 0.f;
    if (live) {
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const int iy = oy + ky - 1;
        if (iy < 0 || iy >= a.Hi) continue;
        const T* row = x + (((long long)n * a.Hi + iy) * a.Wi) * Ci + l * 8;
        float xv[6][8];
#pragma unroll
        for (int c = 0; c < 6; ++c) {
          const int ix = ox0 - 1 + c;
          if (ix >= 0 && ix < a.Wi) Io8<T>::ld(row + (long long)ix * Ci, xv[c]);
          else {
#pragma unroll
            for (int j = 0; j < 8; ++j) xv[c][j] = 0.f;
          }
        }
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          float w[24];
#pragma unroll
          for (int q = 0; q < 6; ++q) {
            const float4 t = sw4[((ky * 3 + kx) * 6 + q) * L + l];
            w[q * 4] = t.x; w[q * 4 + 1] = t.y; w[q * 4 + 2] = t.z; w[q * 4 + 3] = t.w;
          }
#pragma unroll
          for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float v = xv[p + kx][j];
              acc[p][0] = fmaf(v, w[j * 3], acc[p][0]);
              acc[p][1] = fmaf(v, w[j * 3 + 1], acc[p][1]);
              acc[p][2] = fmaf(v, w[j * 3 + 2], acc[p][2]);
            }
        }
      }
    }
    for (int o = L >> 1; o > 0; o >>= 1) {
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int k = 0; k < 3; ++k) acc[p][k] += __shfl_xor_sync(0xffffffffu, acc[p][k], o);
    }
    if (live && l == 0) {
      T* y = reinterpret_cast<T*>(a.y) + (((long long)n * a.Ho + oy) * a.Wo + ox0) * 3;
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        stf(y + p * 3, (acc[p][0] + b0) * a.alpha); stf(y + p * 3 + 1, (acc[p][1] + b1) * a.alpha); stf(y + p * 3 + 2, (acc[p][2] + b2) * a.alpha);
      }
    }
  }
}

// (B) weight gradients of both 3-channel convolutions: acc[pos][c3][ch] = sum_q wide[q][ch] * thin[q + (pos - 1)][c3]
//   FLIP = 0: input conv  (wide = dY (N,H,W,Co), thin = image; dw[(pos*3 + c3)*Co + ch], dbias[ch] = sum dY)
//   FLIP = 1: output conv (wide = x (N,H,W,Ci), thin = dO; dw[((8 - pos)*Ci + ch)*3 + c3], dbias[c3] = sum dO)
// A "stream" = Cw/2 threads (2 wide channels each) walking 32-pixel row segments with the 3 x 3 x 3 window of the thin tensor in
// registers (one new column = 9 uniform loads per pixel); 54 accumulators per thread live over all segments of the stream, then the
// streams of a CTA are summed through shared memory and the CTA issues ONE atomicAdd per weight.
template <typename T, int FLIP>
__global__ void __launch_bounds__(256) wgrad_thin_kernel(WgradArgs a) {
  xu_grid_dep_sync();
  extern __shared__ float red[];                // [256 threads][56]  (54 weights + 2 bias / 3 thin sums)
  const int Cw = FLIP ? a.Ci : a.Co;
  const int TS = Cw >> 1;                       // threads per stream
  const int nstream = 256 / TS;
  const int st = threadIdx.x / TS, tc = threadIdx.x - st * TS;
  const T* wide = reinterpret_cast<const T*>(FLIP ? a.x : a.dy);
  const T* thin = reinterpret_cast<const T*>(FLIP ? a.dy : a.x);
  const int H = a.Ho, Wd = a.Wo;
  const int SEG = Wd < 32 ? Wd : 32;
  const int segs_per_row = Wd / SEG;
  const long long units = (long long)a.N * H * segs_per_row;
  float acc[27][2];
#pragma unroll
  for (int i = 0; i < 27; ++i) acc[i][0] = acc[i][1] = 0.f;
  float ex0 = 0.f, ex1 = 0.f, ex2 = 0.f;        // FLIP=0: bias sums of the 2 channels; FLIP=1: sums of the 3 thin channels
  for (long long u = (long long)blockIdx.x * nstream + st; u < units; u += (long long)gridDim.x * nstream) {
    const int sx = (int)(u % segs_per_row) * SEG;
    const int y = (int)((u / segs_per_row) % H);
    const int n = (int)(u / ((long long)segs_per_row * H));
    const T* trow[3];
    bool rin[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int yy = y + (r - 1);                                // window row r <-> thin row y + (r - 1)
      rin[r] = yy >= 0 && yy < H;
      trow[r] = thin + (((long long)n * H + (rin[r] ? yy : 0)) * Wd) * 3;
    }
    const T* wrow = wide + (((long long)n * H + y) * Wd) * Cw + tc * 2;
    float win[3][9];                            // [column slot][window row * 3 + c3]
    auto load_col = [&](int slot, int xx) {
      const bool cin = xx >= 0 && xx < Wd;
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int k = 0; k < 3; ++k) win[slot][r * 3 + k] = (cin && rin[r]) ? ldf(trow[r] + xx * 3 + k) : 0.f;
    };
    // window column j (0..2) of pixel x is thin column x + (j - 1); slots rotate with x.  (FLIP only renames the result: window
    // position pos is tap 8 - pos of the output convolution, applied when the sums are committed.)
    load_col(0, sx - 1);
    load_col(1, sx);
    for (int xb = 0; xb < SEG; xb += 3) {
#pragma unroll
      for (int uu = 0; uu < 3; ++uu) {
        const int xx = sx + xb + uu;
        if (xb + uu < SEG) {
          load_col((uu + 2) % 3, xx + 1);
          float w0, w1;
          ld2f<T>(wrow + (long long)xx * Cw, w0, w1);
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            const int slot = (uu + j) % 3;
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
              for (int k = 0; k < 3; ++k) {
                const float t = win[slot][r * 3 + k];
                acc[(r * 3 + j) * 3 + k][0] = fmaf(w0, t, acc[(r * 3 + j) * 3 + k][0]);
                acc[(r * 3 + j) * 3 + k][1] = fmaf(w1, t, acc[(r * 3 + j) * 3 + k][1]);
              }
          }
          if (FLIP) { const int c = (uu + 1) % 3; ex0 += win[c][3]; ex1 += win[c][4]; ex2 += win[c][5]; }
          else { ex0 += w0; ex1 += w1; }
        }
      }
    }
  }
  float* mine = red + threadIdx.x * 56;
#pragma unroll
  for (int i = 0; i < 27; ++i) { mine[i * 2] = acc[i][0]; mine[i * 2 + 1] = acc[i][1]; }
  mine[54] = ex0; mine[55] = ex1;
  __syncthreads();
  // sum over the streams of this CTA, one atomic per weight
  for (int i = threadIdx.x; i < 27 * Cw; i += 256) {
    const int pos_c = i / Cw, ch = i - pos_c * Cw;              // pos_c = pos*3 + c3
    float v = 0.f;
    for (int s2 = 0; s2 < nstream; ++s2) v += red[(s2 * TS + (ch >> 1)) * 56 + pos_c * 2 + (ch & 1)];
    const int pos = pos_c / 3, k = pos_c - pos * 3;
    double* dst = FLIP ? a.acc_dw + ((long long)(8 - pos) * Cw + ch) * 3 + k : a.acc_dw + (long long)pos_c * Cw + ch;
    xu_det_add(dst, a.alpha * v);
  }
  if (a.dbias != nullptr) {
    if (!FLIP) {
      for (int ch = threadIdx.x; ch < Cw; ch += 256) {
        float v = 0.f;
        for (int s2 = 0; s2 < nstream; ++s2) v += red[(s2 * TS + (ch >> 1)) * 56 + 54 + (ch & 1)];
        xu_det_add(a.acc_db + ch, a.alpha * v);
      }
    } else {
      // every thread of a stream carries the same three sums: take channel-thread 0 of each stream
      __syncthreads();
      if (tc == 0) { mine[54] = ex0; mine[55] = ex1; mine[53] = ex2; }   // slot 53 = acc[26][1] of this thread, already consumed above
      __syncthreads();
      if (threadIdx.x < 3) {
        float v = 0.f;
        for (int s2 = 0; s2 < nstream; ++s2) v += red[(s2 * TS) * 56 + (threadIdx.x == 2 ? 53 : 54 + threadIdx.x)];
        xu_det_add(a.acc_db + threadIdx.x, a.alpha * v);
      }
    }
  }
}

static bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

bool conv_cin3_supported(int Ci, int Co, int ks, int stride, int nseg, bool res) { return Ci == 3 && ks == 3 && stride == 1 && Co % 8 == 0 && nseg == 1 && !res; }
bool conv_cout3_supported(int Ci, int Co, int ks, int stride, int nseg, bool res) { return Co == 3 && ks == 3 && stride == 1 && Ci % 8 == 0 && 27 * Ci * 4 <= 96 * 1024 && nseg == 1 && !res; }

// exactly one of c (forward, or the Cout=3 data gradient in mode 1) and w (weight gradient) is set
template <typename T>
static void small_dispatch(ConvKernel k, const ConvArgs* c, const WgradArgs* w, cudaStream_t s) {
  const bool cin3 = k == CONV_CIN3;
  // round-2 kernels where their shape rules hold, the round-1 kernels below for every other shape
  if (c && (cin3 || c->mode == 1) && c->Wo % 4 == 0 && c->Co % 8 == 0 && c->Hi == c->Ho && c->Wi == c->Wo) {
    const long long total = (long long)c->N * c->Ho * (c->Wo / 4) * (c->Co / 8);
    const size_t sm = sizeof(float) * 28 * c->Co;
    const int grid = (int)std::min<long long>(cdiv(total, 256), (long long)xu_num_sms() * 4);
    const auto kernel = cin3 ? conv_thin_in_kernel<T, 0> : conv_thin_in_kernel<T, 1>;
    if (sm > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    xu_launch(kernel, grid, 256, sm, s, *c);
    return;
  }
  if (c && !cin3 && c->mode == 0 && c->Wo % 4 == 0 && is_pow2(c->Ci / 8) && c->Ci / 8 <= 32 && c->Hi == c->Ho && c->Wi == c->Wo) {
    const long long quads = (long long)c->N * c->Ho * (c->Wo / 4);
    const int qpb = 256 / (c->Ci / 8);
    const size_t sm = sizeof(float) * 27 * c->Ci;
    const int grid = (int)std::min<long long>(cdiv(quads, qpb), (long long)xu_num_sms() * 4);
    if (sm > 48 * 1024) cudaFuncSetAttribute(conv_cout3_fwd4_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    xu_launch(conv_cout3_fwd4_kernel<T>, grid, 256, sm, s, *c);
    return;
  }
  if (w) {
    const int Cw = cin3 ? w->Co : w->Ci;
    const int SEG = w->Wo < 32 ? w->Wo : 32;
    if (is_pow2(Cw) && Cw >= 2 && Cw <= 512 && w->Wo % SEG == 0 && w->Hi == w->Ho && w->Wi == w->Wo) {
      const int nstream = 256 / (Cw / 2);
      const long long units = (long long)w->N * w->Ho * (w->Wo / SEG);
      const int grid = (int)std::min<long long>(cdiv(units, nstream), (long long)xu_num_sms() * 2);
      const size_t sm = sizeof(float) * 256 * 56;
      const auto kernel = cin3 ? wgrad_thin_kernel<T, 0> : wgrad_thin_kernel<T, 1>;
      cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
      xu_launch(kernel, grid, 256, sm, s, *w);
      return;
    }
  }
  if (c && cin3) {
    const long long total = (long long)c->N * c->Ho * c->Wo * (c->Co / 8);
    const size_t sm = sizeof(float) * 28 * c->Co;
    if (sm > 48 * 1024) cudaFuncSetAttribute(conv_cin3_fwd_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    xu_launch(conv_cin3_fwd_kernel<T>, cdiv(total, 256), 256, sm, s, *c);
  } else if (cin3) {
    const long long M = (long long)w->N * w->Ho * w->Wo;
    xu_launch(conv_cin3_wgrad_kernel<T>, cdiv(M, 128), 256, 0, s, *w);
  } else if (c && c->mode == 0) {
    const long long total = (long long)c->N * c->Ho * c->Wo;
    const size_t sm = sizeof(float) * 27 * c->Ci;
    if (sm > 48 * 1024) cudaFuncSetAttribute(conv_cout3_fwd_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    xu_launch(conv_cout3_fwd_kernel<T>, cdiv(total, 256), 256, sm, s, *c);
  } else if (c) {
    const long long total = (long long)c->N * c->Ho * c->Wo * (c->Co / 8);
    const size_t sm = sizeof(float) * 27 * c->Co;
    if (sm > 48 * 1024) cudaFuncSetAttribute(conv_cout3_dgrad_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    xu_launch(conv_cout3_dgrad_kernel<T>, cdiv(total, 256), 256, sm, s, *c);
  } else {
    const long long M = (long long)w->N * w->Ho * w->Wo;
    const int items = 9 * w->Ci;
    const int threads = items >= 320 ? 320 : ((items + 31) / 32 * 32 < 128 ? 128 : (items + 31) / 32 * 32);
    xu_launch(conv_cout3_wgrad_kernel<T>, cdiv(M, 128), threads, 0, s, *w);
  }
}
void launch_conv_direct(int dtype, ConvKernel k, const ConvArgs& a, cudaStream_t s) {
  if (dtype == XU_F32) small_dispatch<float>(k, &a, nullptr, s);
  else small_dispatch<bf16>(k, &a, nullptr, s);
}
void launch_wgrad_direct(int dtype, ConvKernel k, const WgradArgs& a, cudaStream_t s) {
  det_wgrad(a, s, [&](const WgradArgs& aa) {
    if (dtype == XU_F32) small_dispatch<float>(k, nullptr, &aa, s);
    else small_dispatch<bf16>(k, nullptr, &aa, s);
  });
}
