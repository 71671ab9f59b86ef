// pose_fit.cu -- the loop around the camera gradient that estimates a view's pose by descending the denoising loss
// (pose.PoseEstimator): the per-iteration draw of t and eps, the loss and its seed dL/d(eps_hat), the projection of the camera
// gradient onto each hypothesis's tangent space, and the retraction on SO(3).  include/xunet_b200.h states the arithmetic.
//
// Row b = h P + p of the engine batch is hypothesis h with draw p.  Every kernel is a function of its inputs alone (no atomics,
// sums in an order fixed by the shapes), so an iteration has the same bits on every run, eagerly or replayed from a graph.
// The draw and the loss touch O(B S^2) bytes once; the pose kernels are one thread per hypothesis.
#include "xunet_b200.h"
#include "common.cuh"
#include "kernels.h"

#include <math.h>

#define POSE_THREADS 256

// the hash of draw p of iteration i: it picks the timestep and seeds the draw's noise
__device__ __forceinline__ uint64_t pose_draw_hash(unsigned long long seed, unsigned long long i, int p) {
  return xu_mix64(seed * 0x9E3779B97F4A7C15ULL + i * 0xD1B54A32D192ED03ULL + (uint64_t)p);
}

// one thread per element k of draw p: the noise once, z of the H rows that share the draw, the draw's target, and (k = 0) the
// rows' log-SNR
template <int TARGET>
__global__ void __launch_bounds__(POSE_THREADS) pose_draw_kernel(const float* __restrict__ y, int H, int P, long long n, int t_min,
                                                                 int t_max, int strata, const long long* __restrict__ iter_dev,
                                                                 unsigned long long seed, const float* __restrict__ sqrt_ac,
                                                                 const float* __restrict__ sqrt_1mac, float* __restrict__ z,
                                                                 float* __restrict__ logsnr, float* __restrict__ target,
                                                                 int* __restrict__ t_out) {
  xu_grid_dep_sync();
  const long long e = (long long)blockIdx.x * POSE_THREADS + threadIdx.x;
  if (e >= (long long)P * n) return;
  const int p = (int)(e / n);
  const long long k = e - (long long)p * n;
  const long long i = *iter_dev;
  const uint64_t hp = pose_draw_hash(seed, (unsigned long long)i, p);
  const long long span = (long long)t_max - t_min + 1;
  int t;
  if (strata > 0) {
    const long long g = ((i - 1) * P + p) % strata;
    t = t_min + (int)((2 * g + 1) * span / (2LL * strata));
  } else {
    t = t_min + (int)(hp % (unsigned long long)span);
  }
  const float nz = xu_hash_normal(hp, (uint64_t)k);
  const float sa = sqrt_ac[t], sb = sqrt_1mac[t], x = y[k];
  const float zv = xu_fd_z_rn(sa, x, sb, nz);
  for (int h = 0; h < H; ++h) z[((long long)h * P + p) * n + k] = zv;
  target[e] = TARGET == XU_TARGET_V ? xu_fd_v(sa, nz, sb, x) : nz;
  if (k == 0) {
    const float l = xu_fd_logsnr(t);
    for (int h = 0; h < H; ++h) logsnr[h * P + p] = l;
    if (t_out != nullptr) t_out[p] = t;
  }
}

// grid (chunks, B): the fp64 sum of squared residuals of one chunk of row b, and the seed of that chunk
__global__ void __launch_bounds__(POSE_THREADS) pose_loss_rows_kernel(const float* __restrict__ out, const float* __restrict__ target,
                                                                      int P, long long n, float coef, double* __restrict__ partial,
                                                                      float* __restrict__ d_out) {
  xu_grid_dep_sync();
  __shared__ double s_warp[POSE_THREADS / 32];
  const int c = blockIdx.x, b = blockIdx.y, p = b % P;
  const long long lo = (long long)c * XUNET_POSE_LOSS_CHUNK;
  const long long hi = lo + XUNET_POSE_LOSS_CHUNK < n ? lo + XUNET_POSE_LOSS_CHUNK : n;
  const float* o = out + (long long)b * n;
  const float* tg = target + (long long)p * n;
  float* d = d_out + (long long)b * n;
  double acc = 0.0;
  for (long long k = lo + threadIdx.x; k < hi; k += POSE_THREADS) {
    const float r = __fsub_rn(o[k], tg[k]);
    acc += (double)r * (double)r;
    d[k] = __fmul_rn(coef, r);
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double sum = 0.0;
    for (int w = 0; w < POSE_THREADS / 32; ++w) sum += s_warp[w];
    partial[(long long)b * gridDim.x + c] = sum;
  }
}

// L_h = (sum over p, then chunks, of the partial sums) / (P n), into row i - 1 of the history
__global__ void __launch_bounds__(POSE_THREADS) pose_loss_finish_kernel(const double* __restrict__ partial, int H, int P, int chunks,
                                                                        long long n, const long long* __restrict__ iter_dev,
                                                                        float* __restrict__ loss_out, long long loss_len) {
  xu_grid_dep_sync();
  const long long i = *iter_dev;
  if (i < 1 || i > loss_len) return;
  for (int h = threadIdx.x; h < H; h += POSE_THREADS) {
    double sum = 0.0;
    for (int p = 0; p < P; ++p)
      for (int c = 0; c < chunks; ++c) sum += partial[((long long)h * P + p) * chunks + c];
    loss_out[(i - 1) * H + h] = (float)(sum / ((double)P * (double)n));
  }
}

// one thread per hypothesis: G_R, g_t summed over the draws in p order, N = G_R R^T + g_t t^T, g_omega = vee(N - N^T)
__global__ void __launch_bounds__(POSE_THREADS) pose_tangent_kernel(const float* __restrict__ dR, const float* __restrict__ dt, int H,
                                                                    int P, const double* __restrict__ R, const double* __restrict__ t,
                                                                    int translate, float* __restrict__ grad) {
  xu_grid_dep_sync();
  const int h = blockIdx.x * POSE_THREADS + threadIdx.x;
  if (h >= H) return;
  double G[9], g[3];
  for (int j = 0; j < 9; ++j) G[j] = 0.0;
  for (int j = 0; j < 3; ++j) g[j] = 0.0;
  for (int p = 0; p < P; ++p) {
    const long long b = (long long)h * P + p;
    for (int j = 0; j < 9; ++j) G[j] += (double)dR[b * 9 + j];
    for (int j = 0; j < 3; ++j) g[j] += (double)dt[b * 3 + j];
  }
  const double* Rh = R + 9LL * h;
  const double* th = t + 3LL * h;
  double N[9];
  for (int a = 0; a < 3; ++a)
    for (int c = 0; c < 3; ++c)
      N[3 * a + c] = G[3 * a] * Rh[3 * c] + G[3 * a + 1] * Rh[3 * c + 1] + G[3 * a + 2] * Rh[3 * c + 2] + g[a] * th[c];
  const int D = translate ? 6 : 3;
  float* gr = grad + (long long)h * D;
  gr[0] = (float)(N[7] - N[5]);
  gr[1] = (float)(N[2] - N[6]);
  gr[2] = (float)(N[3] - N[1]);
  if (translate)
    for (int j = 0; j < 3; ++j) gr[3 + j] = (float)g[j];
}

// one thread per hypothesis: E = exp([w]x) by Rodrigues, R <- E R, t <- E t + delta, the fp32 poses into the P rows, step zeroed
__global__ void __launch_bounds__(POSE_THREADS) pose_retract_kernel(float* __restrict__ step, int H, int P, int translate,
                                                                    double* __restrict__ R, double* __restrict__ t,
                                                                    float* __restrict__ R_rows, float* __restrict__ t_rows) {
  xu_grid_dep_sync();
  const int h = blockIdx.x * POSE_THREADS + threadIdx.x;
  if (h >= H) return;
  const int D = translate ? 6 : 3;
  float* st = step + (long long)h * D;
  const double w0 = st[0], w1 = st[1], w2 = st[2];
  const double th2 = w0 * w0 + w1 * w1 + w2 * w2;
  double A, Bc;
  if (th2 < XUNET_POSE_SMALL_ANGLE2) {
    A = 1.0 - th2 / 6.0 + th2 * th2 / 120.0;
    Bc = 0.5 - th2 / 24.0 + th2 * th2 / 720.0;
  } else {
    const double th = sqrt(th2), s = sin(0.5 * th);
    A = sin(th) / th;
    Bc = 2.0 * s * s / th2;
  }
  // W = [w]x, E = I + A W + B W^2 with W^2 = w w^T - th^2 I
  const double W[9] = {0.0, -w2, w1, w2, 0.0, -w0, -w1, w0, 0.0};
  const double wv[3] = {w0, w1, w2};
  double E[9];
  for (int a = 0; a < 3; ++a)
    for (int c = 0; c < 3; ++c)
      E[3 * a + c] = (a == c ? 1.0 : 0.0) + A * W[3 * a + c] + Bc * (wv[a] * wv[c] - (a == c ? th2 : 0.0));
  double* Rh = R + 9LL * h;
  double* th = t + 3LL * h;
  double Rn[9], tn[3];
  for (int a = 0; a < 3; ++a) {
    for (int c = 0; c < 3; ++c) Rn[3 * a + c] = E[3 * a] * Rh[c] + E[3 * a + 1] * Rh[3 + c] + E[3 * a + 2] * Rh[6 + c];
    tn[a] = E[3 * a] * th[0] + E[3 * a + 1] * th[1] + E[3 * a + 2] * th[2] + (translate ? (double)st[3 + a] : 0.0);
  }
  for (int j = 0; j < 9; ++j) Rh[j] = Rn[j];
  for (int j = 0; j < 3; ++j) th[j] = tn[j];
  for (int p = 0; p < P; ++p) {
    const long long b = (long long)h * P + p;
    for (int j = 0; j < 9; ++j) R_rows[b * 9 + j] = (float)Rn[j];
    for (int j = 0; j < 3; ++j) t_rows[b * 3 + j] = (float)tn[j];
  }
  for (int j = 0; j < D; ++j) st[j] = 0.f;
}

// The shape checks the pose entries share (include/xunet_b200.h, "Pose estimation"); 0 or the xu_fail() code.
static int pose_check(const char* what, int H, int P, int S) {
  if (H < 1 || P < 1 || S < 1) return xu_fail("%s: H = %d, P = %d, S = %d, need all >= 1", what, H, P, S);
  if ((long long)H * P * S * S >= (1LL << 31) / 3) return xu_fail("%s: H P S^2 = %lld, need H P S^2 < 2^31 / 3", what, (long long)H * P * S * S);
  return 0;
}

extern "C" int xunet_pose_draw(const float* y, int H, int P, int S, int t_min, int t_max, int strata, const long long* iter_dev,
                               unsigned long long seed, const float* sqrt_ac, const float* sqrt_1mac, int prediction, float* z,
                               float* logsnr, float* target, int* t_out, void* stream) {
  if (!y || !iter_dev || !sqrt_ac || !sqrt_1mac || !z || !logsnr || !target) return xu_fail("xunet_pose_draw: NULL pointer argument");
  if (int rc = pose_check("xunet_pose_draw", H, P, S)) return rc;
  if (t_min < 0 || t_min > t_max || t_max > XUNET_POSE_MAX_T)
    return xu_fail("xunet_pose_draw: t range [%d, %d], need 0 <= t_min <= t_max <= %d", t_min, t_max, XUNET_POSE_MAX_T);
  if (strata < 0) return xu_fail("xunet_pose_draw: strata = %d, need strata >= 0", strata);
  if (prediction != 0 && prediction != 1) return xu_fail("xunet_pose_draw: prediction = %d, need 0 (eps) or 1 (v)", prediction);
  const long long n = 3LL * S * S;
  auto kernel = prediction == 1 ? pose_draw_kernel<XU_TARGET_V> : pose_draw_kernel<XU_TARGET_EPS>;
  xu_launch(kernel, cdiv((long long)P * n, POSE_THREADS), POSE_THREADS, 0, (cudaStream_t)stream, y, H, P, n, t_min, t_max, strata,
            iter_dev, seed, sqrt_ac, sqrt_1mac, z, logsnr, target, t_out);
  return xu_launched("pose_draw");
}

extern "C" int xunet_pose_loss(const float* out, const float* target, int H, int P, int S, const long long* iter_dev, double* partial,
                               float* d_out, float* loss_out, long long loss_len, void* stream) {
  if (!out || !target || !iter_dev || !partial || !d_out || !loss_out) return xu_fail("xunet_pose_loss: NULL pointer argument");
  if (int rc = pose_check("xunet_pose_loss", H, P, S)) return rc;
  if (loss_len < 0) return xu_fail("xunet_pose_loss: loss_len = %lld, need loss_len >= 0", loss_len);
  const long long n = 3LL * S * S;
  const int chunks = cdiv(n, XUNET_POSE_LOSS_CHUNK);
  const float coef = (float)(2.0 / ((double)P * (double)n));
  const cudaStream_t s = (cudaStream_t)stream;
  xu_launch(pose_loss_rows_kernel, dim3(chunks, H * P), POSE_THREADS, 0, s, out, target, P, n, coef, partial, d_out);
  xu_launch(pose_loss_finish_kernel, 1, POSE_THREADS, 0, s, (const double*)partial, H, P, chunks, n, iter_dev, loss_out, loss_len);
  return xu_launched("pose_loss");
}

extern "C" int xunet_pose_tangent(const float* dR, const float* dt, int H, int P, const double* R, const double* t, int translate,
                                  float* grad, void* stream) {
  if (!dR || !dt || !R || !t || !grad) return xu_fail("xunet_pose_tangent: NULL pointer argument");
  if (int rc = pose_check("xunet_pose_tangent", H, P, 1)) return rc;
  if (translate != 0 && translate != 1) return xu_fail("xunet_pose_tangent: translate = %d, need 0 or 1", translate);
  xu_launch(pose_tangent_kernel, cdiv(H, POSE_THREADS), POSE_THREADS, 0, (cudaStream_t)stream, dR, dt, H, P, R, t, translate, grad);
  return xu_launched("pose_tangent");
}

extern "C" int xunet_pose_retract(float* step, int H, int P, int translate, double* R, double* t, float* R_rows, float* t_rows,
                                  void* stream) {
  if (!step || !R || !t || !R_rows || !t_rows) return xu_fail("xunet_pose_retract: NULL pointer argument");
  if (int rc = pose_check("xunet_pose_retract", H, P, 1)) return rc;
  if (translate != 0 && translate != 1) return xu_fail("xunet_pose_retract: translate = %d, need 0 or 1", translate);
  xu_launch(pose_retract_kernel, cdiv(H, POSE_THREADS), POSE_THREADS, 0, (cudaStream_t)stream, step, H, P, translate, R, t, R_rows,
            t_rows);
  return xu_launched("pose_retract");
}
