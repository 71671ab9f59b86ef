// field.cu -- the radiance grid of the 3D consistency score and of lifting: volume rendering of a dense (G, G, G, 4) grid
// (xunet_field_render), one iteration's loss gradient (xunet_field_loss_grad) and the backward of a given image gradient
// (xunet_field_image_grad).  include/xunet_b200.h states the field.
//
// One thread marches one ray; the grid is read with one 16-byte load per corner and stays in L2 (32 MB at G = 128).
// The gradient pass marches a drawn ray twice -- forward to composite C, then front to back again with the residual
// R_{k+1} = C - sum_{j<=k} T_j a_j c_j -- and scatters each sample's gradient into its cell's 8 corners.  Every scattered
// value is rounded to int64 fixed point (XUNET_FIELD_FIXED_ONE per unit) and added with 64-bit integer atomics: integer
// addition is exact and order-free, so the sum has the same bits whatever the schedule and the SM count.  A ray keeps the
// sums of consecutive samples in one cell in registers and flushes them when it leaves the cell (each sample is rounded on
// its own, so this is the same sum), and zero words are never added.  The finish kernel turns the sums into the fp32
// gradient, adds the total-variation stencil, writes the data loss and clears the fixed-point buffer for the next call.
#include "xunet_b200.h"
#include "common.cuh"
#include "kernels.h"

#include <math.h>

#define FIELD_THREADS 128

struct FieldGeom {
  int G;
  float bound, near, step, bg;   // bg = (background + 1) / 2
};

__device__ __forceinline__ float field_softplus(float x) { return x > 20.f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float field_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// The segment of the ray from the camera centre o along d inside [-b, b]^3 and at t >= near: [t0, t0 + L], cut into n pieces.
// false: the segment is empty.
__device__ __forceinline__ bool field_segment(const float (&o)[3], const float (&d)[3], const FieldGeom& g, float& t0, float& L,
                                              int& n) {
  float lo = g.near, hi = INFINITY;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (d[a] == 0.f) {
      if (fabsf(o[a]) > g.bound) return false;
    } else {
      const float t1 = (-g.bound - o[a]) / d[a], t2 = (g.bound - o[a]) / d[a];
      lo = fmaxf(lo, fminf(t1, t2));
      hi = fminf(hi, fmaxf(t1, t2));
    }
  }
  if (!(hi > lo)) return false;
  t0 = lo;
  L = hi - lo;
  n = max(1, (int)ceilf(L / g.step));
  return true;
}

// Sample k of n: its piece length and its position in grid units, clamped to [0, G - 1].
__device__ __forceinline__ float field_sample(const float (&o)[3], const float (&d)[3], float t0, float L, int n, int k,
                                             const FieldGeom& g, float (&u)[3]) {
  const float dk = k < n - 1 ? g.step : L - (float)(n - 1) * g.step;
  const float t = t0 + (float)k * g.step + 0.5f * dk;
  const float s = (float)(g.G - 1) / (2.f * g.bound);
#pragma unroll
  for (int a = 0; a < 3; ++a) u[a] = fminf(fmaxf((o[a] + t * d[a] + g.bound) * s, 0.f), (float)(g.G - 1));
  return dk;
}

// Trilinear interpolation of the raw values at u: cell base index (element offset of corner (i0, j0, k0)), weights of the
// 8 corners in the order (dx, dy, dz) = bits (4, 2, 1) of the corner number, and the interpolated raw vector.
__device__ __forceinline__ int field_interp(const float* __restrict__ grid, int G, const float (&u)[3], float (&w)[8],
                                            float (&v)[4]) {
  int i[3];
  float f[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    i[a] = min((int)u[a], G - 2);
    f[a] = u[a] - (float)i[a];
  }
  const int base = ((i[0] * G + i[1]) * G + i[2]) * 4;
  const int sx = G * G * 4, sy = G * 4;
  v[0] = v[1] = v[2] = v[3] = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const float wx = (c & 4) ? f[0] : 1.f - f[0], wy = (c & 2) ? f[1] : 1.f - f[1], wz = (c & 1) ? f[2] : 1.f - f[2];
    w[c] = wx * wy * wz;
    const float4 q = __ldg(reinterpret_cast<const float4*>(grid + base + ((c & 4) ? sx : 0) + ((c & 2) ? sy : 0) + ((c & 1) ? 4 : 0)));
    v[0] += w[c] * q.x; v[1] += w[c] * q.y; v[2] += w[c] * q.z; v[3] += w[c] * q.w;
  }
  return base;
}

// Front-to-back compositing of one ray: C (in [0, 1]) including the background term T_n bg.
__device__ __forceinline__ void field_composite(const float* __restrict__ grid, const FieldGeom& g, const float (&o)[3],
                                                const float (&d)[3], float (&C)[3]) {
  float t0, L;
  int n;
  float T = 1.f;
  C[0] = C[1] = C[2] = 0.f;
  if (field_segment(o, d, g, t0, L, n)) {
    for (int k = 0; k < n; ++k) {
      float u[3], w[8], v[4];
      const float dk = field_sample(o, d, t0, L, n, k, g, u);
      field_interp(grid, g.G, u, w, v);
      const float a = -expm1f(-field_softplus(v[0] + XUNET_FIELD_DENSITY_SHIFT) * dk);
      const float ta = T * a;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) C[ch] += ta * field_sigmoid(v[1 + ch]);
      T *= 1.f - a;
    }
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) C[ch] += T * g.bg;
}

__device__ __forceinline__ void field_ray(const float* __restrict__ kinv, const float* __restrict__ R,
                                          const float* __restrict__ t, int v, int row, int col, float (&o)[3], float (&d)[3]) {
  xu_ray_dir(kinv + 9 * v, R + 9 * v, row, col, 1, d);   // convention 1 (opencv_uv): SRN's camera model
#pragma unroll
  for (int a = 0; a < 3; ++a) o[a] = t[3 * v + a];
}

__global__ void __launch_bounds__(FIELD_THREADS) field_render_kernel(const float* __restrict__ grid, FieldGeom g,
                                                                      const float* __restrict__ kinv, const float* __restrict__ R,
                                                                      const float* __restrict__ t, int V, int S,
                                                                      float* __restrict__ out) {
  xu_grid_dep_sync();
  const long long p = (long long)blockIdx.x * FIELD_THREADS + threadIdx.x;
  if (p >= (long long)V * S * S) return;
  const int v = (int)(p / ((long long)S * S)), row = (int)(p / S % S), col = (int)(p % S);
  float o[3], d[3], C[3];
  field_ray(kinv, R, t, v, row, col, o, d);
  field_composite(grid, g, o, d, C);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) out[3 * p + ch] = 2.f * C[ch] - 1.f;
}

__device__ __forceinline__ long long field_fix(float x) { return __float2ll_rn(x * (float)XUNET_FIELD_FIXED_ONE); }

// Adds a cell's register sums to the fixed-point buffer (words that are zero are skipped) and clears them.
__device__ __forceinline__ void field_flush(unsigned long long* __restrict__ acc, int base, int G, long long (&s)[8][4]) {
  const int sx = G * G * 4, sy = G * 4;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int off = base + ((c & 4) ? sx : 0) + ((c & 2) ? sy : 0) + ((c & 1) ? 4 : 0);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (s[c][q] != 0) atomicAdd(acc + off + q, (unsigned long long)s[c][q]);
      s[c][q] = 0;
    }
  }
}

// The backward of one ray composited to C: front to back again with the residual R_{k+1} = C - sum_{j<=k} T_j a_j c_j,
// scattering each sample's gradient of sum_ch gC_ch C_ch into its cell's 8 corners of acc (fixed point, flushed per cell).
__device__ __forceinline__ void field_ray_backward(const float* __restrict__ grid, const FieldGeom& g, const float (&o)[3],
                                                   const float (&d)[3], const float (&C)[3], const float (&gC)[3],
                                                   unsigned long long* __restrict__ acc) {
  float t0, L;
  int n;
  if (!field_segment(o, d, g, t0, L, n)) return;
  long long s[8][4];
#pragma unroll
  for (int c = 0; c < 8; ++c)
#pragma unroll
    for (int q = 0; q < 4; ++q) s[c][q] = 0;
  int cell = -1;
  float T = 1.f, Rr[3] = {C[0], C[1], C[2]};
  for (int k = 0; k < n; ++k) {
    float u[3], w[8], raw[4];
    const float dk = field_sample(o, d, t0, L, n, k, g, u);
    const int base = field_interp(grid, g.G, u, w, raw);
    if (base != cell) {
      if (cell >= 0) field_flush(acc, cell, g.G, s);
      cell = base;
    }
    const float sd = field_softplus(raw[0] + XUNET_FIELD_DENSITY_SHIFT);
    const float a = -expm1f(-sd * dk);
    const float ta = T * a, Tn = T * (1.f - a);
    float dsig = 0.f, dc[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float c = field_sigmoid(raw[1 + ch]);
      Rr[ch] -= ta * c;                                   // R_{k+1}
      dsig += gC[ch] * (Tn * c - Rr[ch]);
      dc[ch] = gC[ch] * ta * c * (1.f - c);
    }
    const float draw0 = dsig * dk * field_sigmoid(raw[0] + XUNET_FIELD_DENSITY_SHIFT);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      s[c][0] += field_fix(w[c] * draw0);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) s[c][1 + ch] += field_fix(w[c] * dc[ch]);
    }
    T = Tn;
  }
  field_flush(acc, cell, g.G, s);
}

// One drawn ray per thread: ray r of iteration i = *iter_dev is training pixel
//   xu_mix64(seed * 0x9E3779B97F4A7C15 + i * 0xD1B54A32D192ED03 + r) mod (V S S)     (consistency.draw_rays restates it).
// acc receives the gradient of the per-ray sum sum_ch (C - u)^2 w.r.t. the raw grid, and acc[4 G^3] the sum itself.
__global__ void __launch_bounds__(FIELD_THREADS) field_loss_grad_kernel(const float* __restrict__ grid, FieldGeom g,
                                                                         const float* __restrict__ views,
                                                                         const float* __restrict__ kinv, const float* __restrict__ R,
                                                                         const float* __restrict__ t, int V, int S, int rays,
                                                                         const long long* __restrict__ iter_dev,
                                                                         unsigned long long seed,
                                                                         unsigned long long* __restrict__ acc) {
  xu_grid_dep_sync();
  const int r = blockIdx.x * FIELD_THREADS + threadIdx.x;
  if (r >= rays) return;
  const unsigned long long i = (unsigned long long)*iter_dev;
  const long long npix = (long long)V * S * S;
  const long long p = (long long)(xu_mix64(seed * 0x9E3779B97F4A7C15ULL + i * 0xD1B54A32D192ED03ULL + (unsigned long long)r) %
                                  (unsigned long long)npix);
  const int v = (int)(p / ((long long)S * S)), row = (int)(p / S % S), col = (int)(p % S);
  float o[3], d[3], C[3], gC[3];
  field_ray(kinv, R, t, v, row, col, o, d);
  field_composite(grid, g, o, d, C);
  float lsum = 0.f;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float u = fminf(fmaxf((views[3 * p + ch] + 1.f) * 0.5f, 0.f), 1.f);
    gC[ch] = 2.f * (C[ch] - u);
    lsum += (C[ch] - u) * (C[ch] - u);
  }
  atomicAdd(acc + 4LL * g.G * g.G * g.G, (unsigned long long)field_fix(lsum));
  field_ray_backward(grid, g, o, d, C, gC, acc);
}

// One pixel of V views per thread: acc receives the gradient of sum_ch dC_ch C_ch w.r.t. the raw grid, dC the given image
// gradient (V, S, S, 3) in the caller's unit, a non-finite value read as 0.
__global__ void __launch_bounds__(FIELD_THREADS) field_image_grad_kernel(const float* __restrict__ grid, FieldGeom g,
                                                                          const float* __restrict__ dC,
                                                                          const float* __restrict__ kinv, const float* __restrict__ R,
                                                                          const float* __restrict__ t, int V, int S,
                                                                          unsigned long long* __restrict__ acc) {
  xu_grid_dep_sync();
  const long long p = (long long)blockIdx.x * FIELD_THREADS + threadIdx.x;
  if (p >= (long long)V * S * S) return;
  const int v = (int)(p / ((long long)S * S)), row = (int)(p / S % S), col = (int)(p % S);
  float gC[3];
  bool any = false;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float x = dC[3 * p + ch];
    gC[ch] = isfinite(x) ? x : 0.f;
    any |= gC[ch] != 0.f;
  }
  if (!any) return;                                       // every scattered word would be zero
  float o[3], d[3], C[3];
  field_ray(kinv, R, t, v, row, col, o, d);
  field_composite(grid, g, o, d, C);
  field_ray_backward(grid, g, o, d, C, gC, acc);
}

// grad = acc inv + the total-variation gradient (inv: 1 / (XUNET_FIELD_FIXED_ONE 3N) for the drawn rays' mean, unit /
// XUNET_FIELD_FIXED_ONE for an image gradient in units of `unit`); loss_out[i - 1] = acc[4 G^3] inv when iter_dev is given; acc cleared.
__global__ void __launch_bounds__(256) field_finish_kernel(const float* __restrict__ grid, int G, double inv, float tv_density,
                                                           float tv_color, const long long* __restrict__ iter_dev,
                                                           long long* __restrict__ acc, float* __restrict__ grad,
                                                           float* __restrict__ loss_out, long long loss_len) {
  xu_grid_dep_sync();
  const long long n = 4LL * G * G * G;
  const long long e = (long long)blockIdx.x * 256 + threadIdx.x;
  if (e == 0) {
    if (iter_dev != nullptr) {
      const long long i = *iter_dev;
      if (i >= 1 && i <= loss_len) loss_out[i - 1] = (float)((double)acc[n] * inv);
    }
    acc[n] = 0;
  }
  if (e >= n) return;
  const int q = (int)(e & 3);
  const long long cell = e >> 2;
  const int idx[3] = {(int)(cell / ((long long)G * G)), (int)(cell / G % G), (int)(cell % G)};
  const long long stride[3] = {4LL * G * G, 4LL * G, 4};
  const double x = grid[e];
  double tv = 0.0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (idx[a] > 0) tv += x - (double)grid[e - stride[a]];
    if (idx[a] < G - 1) tv -= (double)grid[e + stride[a]] - x;
  }
  const double lam = q == 0 ? (double)tv_density : (double)tv_color;
  grad[e] = (float)((double)acc[e] * inv + 2.0 * lam / ((double)G * G * G) * tv);
  acc[e] = 0;
}

static FieldGeom field_geom(int G, float bound, float near, float step, float background) {
  return FieldGeom{G, bound, near, step, 0.5f * (background + 1.f)};
}

// The checks both field entries share (include/xunet_b200.h, "Limits"); 0 or the xu_fail() code.
static int field_check(const char* what, int G, float bound, int V, int S, float near, float step, float background) {
  if (G < XUNET_FIELD_MIN_GRID || G > XUNET_FIELD_MAX_GRID)
    return xu_fail("%s: G = %d outside [%d, %d]", what, G, XUNET_FIELD_MIN_GRID, XUNET_FIELD_MAX_GRID);
  if (V < 1 || S < 1) return xu_fail("%s: V = %d, S = %d, need both >= 1", what, V, S);
  if ((long long)V * S * S >= (1LL << 31)) return xu_fail("%s: V S S = %lld pixels, need fewer than 2^31", what, (long long)V * S * S);
  if (!isfinite(bound) || !(bound > 0.f) || bound > XUNET_FIELD_MAX_BOUND)
    return xu_fail("%s: bound = %g outside (0, %g]", what, bound, XUNET_FIELD_MAX_BOUND);
  if (!isfinite(near) || near < 0.f) return xu_fail("%s: near = %g, need a finite near >= 0", what, near);
  if (!isfinite(step) || !(step > 0.f)) return xu_fail("%s: step = %g, need a finite step > 0", what, step);
  if (ceil(2.0 * sqrt(3.0) * bound / step) > XUNET_FIELD_MAX_SAMPLES)
    return xu_fail("%s: step = %g gives more than %d samples on a chord of the cube of bound %g", what, step, XUNET_FIELD_MAX_SAMPLES,
                   bound);
  if (!isfinite(background)) return xu_fail("%s: background = %g is not finite", what, background);
  return 0;
}

extern "C" int xunet_field_render(const float* grid, int G, float bound, const float* R, const float* t, const float* K, float* kinv,
                                  int V, int S, float near, float step, float background, float* out, void* stream) {
  if (!grid || !R || !t || !K || !kinv || !out) return xu_fail("xunet_field_render: NULL pointer argument");
  if (int rc = field_check("xunet_field_render", G, bound, V, S, near, step, background)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  xu_launch(kinv_kernel, cdiv(V, 64), 64, 0, s, K, kinv, V);
  xu_launch(field_render_kernel, cdiv((long long)V * S * S, FIELD_THREADS), FIELD_THREADS, 0, s, grid,
            field_geom(G, bound, near, step, background), (const float*)kinv, R, t, V, S, out);
  return xu_launched("field_render");
}

extern "C" int xunet_field_loss_grad(const float* grid, int G, float bound, const float* views, const float* R, const float* t,
                                     const float* K, float* kinv, int V, int S, float near, float step, float background, int rays,
                                     const long long* iter_dev, unsigned long long seed, float tv_density, float tv_color,
                                     long long* acc, float* grad, float* loss_out, long long loss_len, void* stream) {
  if (!grid || !views || !R || !t || !K || !kinv || !iter_dev || !acc || !grad || !loss_out)
    return xu_fail("xunet_field_loss_grad: NULL pointer argument");
  if (int rc = field_check("xunet_field_loss_grad", G, bound, V, S, near, step, background)) return rc;
  if (rays < 1 || rays > XUNET_FIELD_MAX_RAYS)
    return xu_fail("xunet_field_loss_grad: rays = %d outside [1, %d]", rays, XUNET_FIELD_MAX_RAYS);
  if (!isfinite(tv_density) || !isfinite(tv_color) || tv_density < 0.f || tv_color < 0.f)
    return xu_fail("xunet_field_loss_grad: tv weights %g, %g, need finite weights >= 0", tv_density, tv_color);
  if (loss_len < 0) return xu_fail("xunet_field_loss_grad: loss_len = %lld, need loss_len >= 0", loss_len);
  const cudaStream_t s = (cudaStream_t)stream;
  xu_launch(kinv_kernel, cdiv(V, 64), 64, 0, s, K, kinv, V);
  xu_launch(field_loss_grad_kernel, cdiv(rays, FIELD_THREADS), FIELD_THREADS, 0, s, grid,
            field_geom(G, bound, near, step, background), views, (const float*)kinv, R, t, V, S, rays, iter_dev, seed,
            (unsigned long long*)acc);
  xu_launch(field_finish_kernel, cdiv(4LL * G * G * G, 256), 256, 0, s, grid, G, 1.0 / (XUNET_FIELD_FIXED_ONE * 3.0 * (double)rays),
            tv_density, tv_color, iter_dev, acc, grad, loss_out, loss_len);
  return xu_launched("field_loss_grad");
}

extern "C" int xunet_field_image_grad(const float* grid, int G, float bound, const float* dC, double unit, const float* R,
                                      const float* t, const float* K, float* kinv, int V, int S, float near, float step,
                                      float background, float tv_density, float tv_color, long long* acc, float* grad,
                                      void* stream) {
  if (!grid || !dC || !R || !t || !K || !kinv || !acc || !grad) return xu_fail("xunet_field_image_grad: NULL pointer argument");
  if (int rc = field_check("xunet_field_image_grad", G, bound, V, S, near, step, background)) return rc;
  if ((long long)V * S * S > XUNET_FIELD_MAX_RAYS)
    return xu_fail("xunet_field_image_grad: V S S = %lld pixels, need at most %d", (long long)V * S * S, XUNET_FIELD_MAX_RAYS);
  if (!isfinite(unit) || !(unit > 0.0)) return xu_fail("xunet_field_image_grad: unit = %g, need a finite unit > 0", unit);
  if (!isfinite(tv_density) || !isfinite(tv_color) || tv_density < 0.f || tv_color < 0.f)
    return xu_fail("xunet_field_image_grad: tv weights %g, %g, need finite weights >= 0", tv_density, tv_color);
  const cudaStream_t s = (cudaStream_t)stream;
  xu_launch(kinv_kernel, cdiv(V, 64), 64, 0, s, K, kinv, V);
  xu_launch(field_image_grad_kernel, cdiv((long long)V * S * S, FIELD_THREADS), FIELD_THREADS, 0, s, grid,
            field_geom(G, bound, near, step, background), dC, (const float*)kinv, R, t, V, S, (unsigned long long*)acc);
  xu_launch(field_finish_kernel, cdiv(4LL * G * G * G, 256), 256, 0, s, grid, G, unit / XUNET_FIELD_FIXED_ONE, tv_density, tv_color,
            (const long long*)nullptr, acc, grad, (float*)nullptr, 0LL);
  return xu_launched("field_image_grad");
}
