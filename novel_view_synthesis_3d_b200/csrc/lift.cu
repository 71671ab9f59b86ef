// lift.cu -- the loop around the radiance grid and the guided X-UNet that lifts one view to a grid by score distillation
// (lift.FieldLifter): the per-iteration draw of cameras and timesteps, the noise of the renders, and the guided, weighted
// residual turned into an image gradient for xunet_field_image_grad.  include/xunet_b200.h states the arithmetic.
//
// Rows p and P + p of the engine batch are draw p, conditional and unconditional; view P of the renders is the source camera.
// Every kernel is a function of its inputs alone (no atomics, sums in an order fixed by the shapes), so an iteration has the
// same bits on every run, eagerly or replayed from a graph.
#include "xunet_b200.h"
#include "common.cuh"
#include "kernels.h"

#include <math.h>

#define LIFT_THREADS 256

__device__ __forceinline__ uint64_t lift_hash(unsigned long long seed, unsigned long long i, int p) {
  return xu_mix64((seed ^ XUNET_LIFT_SEED_DOMAIN) * 0x9E3779B97F4A7C15ULL + i * 0xD1B54A32D192ED03ULL + (uint64_t)p);
}

__device__ __forceinline__ int lift_timestep(uint64_t h, int t_min, int t_max) {
  return t_min + (int)(h % (unsigned long long)((long long)t_max - t_min + 1));
}

__device__ __forceinline__ double lift_uniform(uint64_t h, uint64_t k) { return (double)(xu_mix64(h + k) >> 11) * 0x1p-53; }

__device__ __forceinline__ void lift_cross(const double (&a)[3], const double (&b)[3], double (&c)[3]) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// one thread per draw: t_p, the camera centre on the band, the look-at rotation; up and e1 are unit vectors (the entry's)
__global__ void __launch_bounds__(LIFT_THREADS) lift_draw_kernel(int P, int t_min, int t_max, const long long* __restrict__ iter_dev,
                                                                 unsigned long long seed, double3 up_, double3 e1_, double s_lo,
                                                                 double s_hi, double radius, float* __restrict__ R2,
                                                                 float* __restrict__ t2, float* __restrict__ cam_R,
                                                                 float* __restrict__ cam_t, int* __restrict__ t_out) {
  xu_grid_dep_sync();
  const int p = blockIdx.x * LIFT_THREADS + threadIdx.x;
  if (p >= P) return;
  const uint64_t h = lift_hash(seed, (unsigned long long)*iter_dev, p);
  const double up[3] = {up_.x, up_.y, up_.z}, e1[3] = {e1_.x, e1_.y, e1_.z};
  double e2[3];
  lift_cross(up, e1, e2);
  const double s = s_lo + (s_hi - s_lo) * lift_uniform(h, 0x5851F42D4C957F2DULL);
  const double phi = 2.0 * M_PI * lift_uniform(h, 0x14057B7EF767814FULL);
  const double cs = sqrt(fmax(0.0, 1.0 - s * s)), ca = cos(phi), sa = sin(phi);
  double c[3], f[3], right[3], down[3];
  for (int a = 0; a < 3; ++a) c[a] = radius * (s * up[a] + cs * (ca * e1[a] + sa * e2[a]));
  const double cn = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
  for (int a = 0; a < 3; ++a) f[a] = -c[a] / cn;
  lift_cross(f, up, right);
  const double rn = sqrt(right[0] * right[0] + right[1] * right[1] + right[2] * right[2]);
  if (rn < 1e-6) {                                        // f (nearly) parallel to up: e1 made perpendicular to f
    const double ef = e1[0] * f[0] + e1[1] * f[1] + e1[2] * f[2];
    for (int a = 0; a < 3; ++a) right[a] = e1[a] - ef * f[a];
    const double en = sqrt(right[0] * right[0] + right[1] * right[1] + right[2] * right[2]);
    for (int a = 0; a < 3; ++a) right[a] /= en;
  } else {
    for (int a = 0; a < 3; ++a) right[a] /= rn;
  }
  lift_cross(f, right, down);
  for (int a = 0; a < 3; ++a) {
    const float row[3] = {(float)right[a], (float)down[a], (float)f[a]};
    for (int b = 0; b < 3; ++b) {
      R2[9LL * p + 3 * a + b] = row[b];
      R2[9LL * (P + p) + 3 * a + b] = row[b];
      cam_R[9LL * p + 3 * a + b] = row[b];
    }
    t2[3LL * p + a] = t2[3LL * (P + p) + a] = cam_t[3LL * p + a] = (float)c[a];
  }
  t_out[p] = lift_timestep(h, t_min, t_max);
}

// one thread per value k of draw p: the noise, z of both rows of the draw, eps, and (k = 0) the rows' log-SNR
__global__ void __launch_bounds__(LIFT_THREADS) lift_noise_kernel(const float* __restrict__ render, const int* __restrict__ t_draw,
                                                                  int P, long long n, const long long* __restrict__ iter_dev,
                                                                  unsigned long long seed, const float* __restrict__ sqrt_ac,
                                                                  const float* __restrict__ sqrt_1mac, float* __restrict__ z,
                                                                  float* __restrict__ logsnr, float* __restrict__ eps) {
  xu_grid_dep_sync();
  const long long e = (long long)blockIdx.x * LIFT_THREADS + threadIdx.x;
  if (e >= (long long)P * n) return;
  const int p = (int)(e / n);
  const long long k = e - (long long)p * n;
  const uint64_t h = lift_hash(seed, (unsigned long long)*iter_dev, p);
  const int t = t_draw[p];
  const float nz = xu_hash_normal(h, (uint64_t)k);
  const float zv = xu_fd_z_rn(sqrt_ac[t], render[e], sqrt_1mac[t], nz);
  z[e] = zv;
  z[(long long)P * n + e] = zv;
  eps[e] = nz;
  if (k == 0) logsnr[p] = logsnr[P + p] = xu_fd_logsnr(t);
}

// grid (chunks, P + 1): the image gradient of one chunk of view p and the fp64 sum of its squares (r^2, or (C - u)^2 for the
// source view p = P)
template <int PRED_V>
__global__ void __launch_bounds__(LIFT_THREADS) lift_grad_kernel(const float* __restrict__ out, const float* __restrict__ z,
                                                                 const float* __restrict__ eps, const float* __restrict__ render,
                                                                 const float* __restrict__ x, const int* __restrict__ t_draw, int P,
                                                                 long long n, float w, double sds_coef, float recon_coef,
                                                                 const float* __restrict__ sqrt_ac, const float* __restrict__ sqrt_1mac,
                                                                 double* __restrict__ partial, float* __restrict__ dC) {
  xu_grid_dep_sync();
  __shared__ double s_warp[LIFT_THREADS / 32];
  const int c = blockIdx.x, p = blockIdx.y;
  const long long lo = (long long)c * XUNET_POSE_LOSS_CHUNK;
  const long long hi = lo + XUNET_POSE_LOSS_CHUNK < n ? lo + XUNET_POSE_LOSS_CHUNK : n;
  const long long row = (long long)p * n;
  double acc = 0.0;
  if (p < P) {
    const int t = t_draw[p];
    const float sa = sqrt_ac[t], sb = sqrt_1mac[t];
    const float coef = (float)(sds_coef * ((double)sb * (double)sb));
    const float* oc = out + row;
    const float* ou = out + (long long)(P + p) * n;
    for (long long k = lo + threadIdx.x; k < hi; k += LIFT_THREADS) {
      const float og = __fsub_rn(__fmul_rn(1.f + w, oc[k]), __fmul_rn(w, ou[k]));
      const float eh = PRED_V ? __fmaf_rn(sb, z[row + k], __fmul_rn(sa, og)) : og;
      float r = __fsub_rn(eh, eps[row + k]);
      r = isfinite(r) ? fminf(fmaxf(r, -XUNET_LIFT_MAX_RESIDUAL), XUNET_LIFT_MAX_RESIDUAL) : 0.f;
      acc += (double)r * (double)r;
      dC[row + k] = __fmul_rn(coef, r);
    }
  } else {
    for (long long k = lo + threadIdx.x; k < hi; k += LIFT_THREADS) {
      const float C = __fmul_rn(0.5f, __fadd_rn(render[row + k], 1.f));
      const float u = fminf(fmaxf(__fmul_rn(0.5f, __fadd_rn(x[k], 1.f)), 0.f), 1.f);
      const float d = __fsub_rn(C, u);
      acc += (double)d * (double)d;
      dC[row + k] = __fmul_rn(recon_coef, d);
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double sum = 0.0;
    for (int wi = 0; wi < LIFT_THREADS / 32; ++wi) sum += s_warp[wi];
    partial[(long long)p * gridDim.x + c] = sum;
  }
}

// one thread: the diagnostics of iteration i from the partial sums, in order
__global__ void __launch_bounds__(32) lift_finish_kernel(const double* __restrict__ partial, int P, int chunks, long long n,
                                                         const long long* __restrict__ iter_dev, float* __restrict__ sds_out,
                                                         float* __restrict__ loss_out, long long loss_len) {
  xu_grid_dep_sync();
  const long long i = *iter_dev;
  if (threadIdx.x != 0 || i < 1 || i > loss_len) return;
  double sds = 0.0, rec = 0.0;
  for (int p = 0; p < P; ++p)
    for (int c = 0; c < chunks; ++c) sds += partial[(long long)p * chunks + c];
  for (int c = 0; c < chunks; ++c) rec += partial[(long long)P * chunks + c];
  sds_out[i - 1] = (float)(sds / ((double)P * (double)n));
  loss_out[i - 1] = (float)(rec / (double)n);
}

// The shape checks the lift entries share (include/xunet_b200.h, "Lifting"); 0 or the xu_fail() code.
static int lift_check(const char* what, int P, int S) {
  if (P < 1 || S < 1) return xu_fail("%s: P = %d, S = %d, need both >= 1", what, P, S);
  if ((long long)(P + 1) * S * S > XUNET_FIELD_MAX_RAYS)
    return xu_fail("%s: (P + 1) S^2 = %lld pixels, need at most %d", what, (long long)(P + 1) * S * S, XUNET_FIELD_MAX_RAYS);
  return 0;
}

extern "C" int xunet_lift_draw(int P, int t_min, int t_max, const long long* iter_dev, unsigned long long seed, double up_x,
                               double up_y, double up_z, double elev_lo, double elev_hi, double radius, float* R2, float* t2,
                               float* cam_R, float* cam_t, int* t_out, void* stream) {
  if (!iter_dev || !R2 || !t2 || !cam_R || !cam_t || !t_out) return xu_fail("xunet_lift_draw: NULL pointer argument");
  if (P < 1) return xu_fail("xunet_lift_draw: P = %d, need P >= 1", P);
  if (t_min < 0 || t_min > t_max || t_max > XUNET_POSE_MAX_T)
    return xu_fail("xunet_lift_draw: t range [%d, %d], need 0 <= t_min <= t_max <= %d", t_min, t_max, XUNET_POSE_MAX_T);
  const double un = sqrt(up_x * up_x + up_y * up_y + up_z * up_z);
  if (!isfinite(un) || !(un > 0.0)) return xu_fail("xunet_lift_draw: up = (%g, %g, %g), need a finite nonzero vector", up_x, up_y, up_z);
  if (!(elev_lo >= -0.5 * M_PI && elev_lo <= elev_hi && elev_hi <= 0.5 * M_PI))
    return xu_fail("xunet_lift_draw: elevation [%g, %g] rad, need -pi/2 <= lo <= hi <= pi/2", elev_lo, elev_hi);
  if (!isfinite(radius) || !(radius > 0.0)) return xu_fail("xunet_lift_draw: radius = %g, need a finite radius > 0", radius);
  const double up[3] = {up_x / un, up_y / un, up_z / un};
  int j = 0;
  for (int a = 1; a < 3; ++a)
    if (fabs(up[a]) < fabs(up[j])) j = a;
  double e1[3] = {0.0, 0.0, 0.0};
  e1[j] = 1.0;
  const double dot = up[j];
  for (int a = 0; a < 3; ++a) e1[a] -= dot * up[a];
  const double en = sqrt(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
  for (int a = 0; a < 3; ++a) e1[a] /= en;
  xu_launch(lift_draw_kernel, cdiv(P, LIFT_THREADS), LIFT_THREADS, 0, (cudaStream_t)stream, P, t_min, t_max, iter_dev, seed,
            make_double3(up[0], up[1], up[2]), make_double3(e1[0], e1[1], e1[2]), sin(elev_lo), sin(elev_hi), radius, R2, t2, cam_R,
            cam_t, t_out);
  return xu_launched("lift_draw");
}

extern "C" int xunet_lift_noise(const float* render, const int* t_draw, int P, int S, const long long* iter_dev,
                                unsigned long long seed, const float* sqrt_ac, const float* sqrt_1mac, float* z, float* logsnr,
                                float* eps, void* stream) {
  if (!render || !t_draw || !iter_dev || !sqrt_ac || !sqrt_1mac || !z || !logsnr || !eps)
    return xu_fail("xunet_lift_noise: NULL pointer argument");
  if (int rc = lift_check("xunet_lift_noise", P, S)) return rc;
  const long long n = 3LL * S * S;
  xu_launch(lift_noise_kernel, cdiv((long long)P * n, LIFT_THREADS), LIFT_THREADS, 0, (cudaStream_t)stream, render, t_draw, P, n,
            iter_dev, seed, sqrt_ac, sqrt_1mac, z, logsnr, eps);
  return xu_launched("lift_noise");
}

extern "C" int xunet_lift_grad(const float* out, const float* z, const float* eps, const float* render, const float* x,
                               const int* t_draw, int P, int S, float w, int prediction, float sds_weight, float recon_weight,
                               double unit, const float* sqrt_ac, const float* sqrt_1mac, const long long* iter_dev, double* partial, float* dC,
                               float* sds_out, float* loss_out, long long loss_len, void* stream) {
  if (!out || !z || !eps || !render || !x || !t_draw || !sqrt_ac || !sqrt_1mac || !iter_dev || !partial || !dC || !sds_out ||
      !loss_out)
    return xu_fail("xunet_lift_grad: NULL pointer argument");
  if (int rc = lift_check("xunet_lift_grad", P, S)) return rc;
  if (!isfinite(w) || w < 0.f) return xu_fail("xunet_lift_grad: w = %g, need a finite w >= 0", w);
  if (prediction != 0 && prediction != 1) return xu_fail("xunet_lift_grad: prediction = %d, need 0 (eps) or 1 (v)", prediction);
  if (!isfinite(sds_weight) || sds_weight < 0.f) return xu_fail("xunet_lift_grad: sds_weight = %g, need a finite weight >= 0", sds_weight);
  if (!isfinite(recon_weight) || recon_weight < 0.f)
    return xu_fail("xunet_lift_grad: recon_weight = %g, need a finite weight >= 0", recon_weight);
  if (!isfinite(unit) || !(unit > 0.0)) return xu_fail("xunet_lift_grad: unit = %g, need a finite unit > 0", unit);
  const double l1 = (2.0 * XUNET_LIFT_MAX_RESIDUAL * sds_weight + 2.0 * recon_weight) / unit;   // bounds sum |dC|
  if (l1 > XUNET_FIELD_MAX_GRAD_L1)
    return xu_fail("xunet_lift_grad: (32 sds_weight + 2 recon_weight) / unit = %g exceeds %g", l1, XUNET_FIELD_MAX_GRAD_L1);
  if (loss_len < 0) return xu_fail("xunet_lift_grad: loss_len = %lld, need loss_len >= 0", loss_len);
  const long long n = 3LL * S * S;
  const int chunks = cdiv(n, XUNET_POSE_LOSS_CHUNK);
  const double sds_coef = 2.0 * sds_weight / (3.0 * S * S * P * unit);
  const float recon_coef = (float)(2.0 * recon_weight / (3.0 * S * S * unit));
  const cudaStream_t s = (cudaStream_t)stream;
  auto kernel = prediction == 1 ? lift_grad_kernel<1> : lift_grad_kernel<0>;
  xu_launch(kernel, dim3(chunks, P + 1), LIFT_THREADS, 0, s, out, z, eps, render, x, t_draw, P, n, w, sds_coef, recon_coef, sqrt_ac,
            sqrt_1mac, partial, dC);
  xu_launch(lift_finish_kernel, 1, 32, 0, s, (const double*)partial, P, chunks, n, iter_dev, sds_out, loss_out, loss_len);
  return xu_launched("lift_grad");
}
