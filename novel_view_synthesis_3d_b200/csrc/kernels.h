// kernels.h -- what more than one source file needs: the launchers the engine plan runs (all asynchronous on `s`), the
// shared kinv_kernel, and the determinism and error plumbing.  The C entries that run no plan launch their kernels in the
// file that holds them.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "xunet_b200.h"

enum { XU_F32 = 0, XU_BF16 = 1 };

// ---- implicit-GEMM convolution / per-pixel dense (k=1), forward and data-gradient ------------------
// mode 0 (forward):  y[n,oy,ox,co] = alpha * ( sum_{tap,ci} x[n, oy*s+dy-ph, ox*s+dx-pw, ci] W[tap][ci][co] + bias[co] + res )
// mode 1 (dgrad):    y = dX (N,Ho,Wo,Co=wCi),  x = dY (N,Hi,Wi,Ci=wCo):
//                    y[n,iy,ix,ci] (+)= alpha * sum_{tap,co} dY[n,(iy+ph-dy)/s,(ix+pw-dx)/s,co] W[tap][ci][co]
// weights: Flax layout [tap][wCi][wCo] fp32, with wCo split into segments of width segw laid out one after
// the other ([seg][tap][wCi][segw]; nseg>1 only for the fused q|k|v projection with ks==1).
struct ConvArgs {
  const void* x; void* y; const void* res; const float* w; const float* bias;
  int N, Hi, Wi, Ci, Ho, Wo, Co;
  int ks, stride, pad_h, pad_w, mode;
  int wCi, wCo, segw;
  float alpha; int accumulate;
  // optional (tensor-core forward only, see conv_tc_stats_supported): per-(sample, channel) [sum, sumsq] of the STORED output,
  // (N/2, Co, 2) fp32, accumulated with atomics into a zeroed buffer -- the GroupNorm statistics of the consumer norm
  float* cstats = nullptr;
  // optional (tensor-core data gradient, mode 1): this conv consumes the output of a GroupNorm[+swish] without resampling.  The
  // epilogue then stores dyh = dy * swish'(.) instead of dy and accumulates the per-(sample, channel) sums [sum dyh*xhat,
  // sum dyh] into cstats (N/2, Co, 2).  gn_x: the norm's input (N,H,W,Co); gn_params: (N/2, Co) float4 {rstd, -mean*rstd,
  // gamma, beta} written by the forward launch_gn_apply (GnArgs::params_out)
  const void* gn_x = nullptr; const void* gn_params = nullptr; int gn_swish = 0;
  // ... and when that norm is the FiLM norm of a ResnetBlock (u = yhat*(1+scale)+shift -> swish -> dropout -> this conv):
  // gn_e (N,H,W,2*Co) [scale | shift], gn_de its gradient (written), dropout rate / residual-block index / device seed
  const void* gn_e = nullptr; void* gn_de = nullptr;
  float gn_drop_rate = 0.f; int gn_drop_op = 0; const unsigned long long* gn_seed_dev = nullptr; int gn_train = 0;
};
void launch_conv_simt(int dtype, const ConvArgs& a, cudaStream_t s);

// dW[tap][ci][co] += alpha * sum_{n,oy,ox} x[n,oy*s+dy-ph,ox*s+dx-pw,ci] dY[n,oy,ox,co];  dbias[co] += alpha*sum dY
struct WgradArgs {
  const void* x; const void* dy; float* dw; float* dbias;
  int N, Hi, Wi, Ci, Ho, Wo, Co;
  int ks, stride, pad_h, pad_w, segw;
  float alpha;
  // set by the launchers: fp64 accumulators laid out like dw / dbias, folded into them after the kernel (xu_det_scratch)
  double* acc_dw; double* acc_db;
};
void launch_wgrad_simt(int dtype, const WgradArgs& a, cudaStream_t s);
// the kernel a convolution runs in one direction (forward, data gradient or weight gradient)
enum ConvKernel { CONV_SIMT, CONV_TC, CONV_CIN3, CONV_COUT3 };
// direct kernels for the 3-channel convs: CONV_CIN3 (forward, weight gradient) and CONV_COUT3 (forward, data gradient with
// ConvArgs in the mode-1 convention x = dO, y = dX, weight gradient).  Neither takes a residual (res) or segments (nseg > 1).
bool conv_cin3_supported(int Ci, int Co, int ks, int stride, int nseg, bool res);
bool conv_cout3_supported(int Ci, int Co, int ks, int stride, int nseg, bool res);
void launch_conv_direct(int dtype, ConvKernel k, const ConvArgs& a, cudaStream_t s);
void launch_wgrad_direct(int dtype, ConvKernel k, const WgradArgs& a, cudaStream_t s);
// data gradient of the input conv 3 -> Co, un-packed: dy (2B,S,S,Co) activation dtype, w the fp32 kernel (3,3,3,Co); rows 2b go
// to dx (B,S,S,3) fp32, rows 2b+1 to dz; a nullptr output is skipped (both nullptr: nothing is launched)
void launch_conv_cin3_dgrad_unpack(int dtype, const void* dy, const float* w, float* dx, float* dz, int B, int S, int Co,
                                   float alpha, cudaStream_t s);

// ---- GroupNorm(32) over both frames (+ SiLU / FiLM / dropout / resample) -----------------------------
enum { GN_PLAIN = 0, GN_SWISH = 1, GN_FILM = 2 };
enum { RS_NONE = 0, RS_DOWN = 1, RS_UP = 2 };
struct GnArgs {
  const void* x;      // (N,H,W,C) input
  void* y;            // forward output (N,Ho,Wo,C)  /  backward: dx (N,H,W,C)
  const void* e;      // FiLM (N,H,W,2C): [scale | shift]
  const void* dy;     // backward: grad of output (N,Ho,Wo,C)
  void* de;           // backward: grad of e
  const float* gamma; const float* beta;
  float* dgamma; float* dbeta;   // backward (atomic accumulate)
  float* stats;       // (B,32,2) sum, sumsq of x         (forward writes, backward reads)
  // producer-emitted statistics (forward apply only): channels [0, csA) of x come with per-channel sums cstatsA (B, csA, 2),
  // channels [csA, C) with cstatsB (B, C - csA, 2) (a channel concat of two producers).  The apply kernel reduces them to
  // group sums itself and stores them to `stats`.
  const float* cstatsA; const float* cstatsB; int csA;
  float* params_out;   // forward apply, optional: (B, C) float4 {rstd, -mean*rstd, gamma, beta} for the fused backward epilogue
  const float* bcs;    // launch_gn_bwd_apply_pre: per-(sample, channel) [sum dyh*xhat, sum dyh] emitted by that epilogue
  float* bstats;      // (B,32,2) backward group sums S1,S2
  int N, H, W, C;
  int mode, rs;
  float drop_rate; int op_index; const unsigned long long* seed_dev; int train;
  int accumulate;     // backward: dx += instead of =
  int de_accumulate;
  const void* extra;  // backward: optional second gradient stream into dx: dx += extra_alpha * extra  (same shape as x)
  float extra_alpha;
  int skip_zero;      // stats / bstats were already zeroed by the caller (one memset for the whole plan)
};
// per-(sample, channel) [sum, sumsq] of x (N,H,W,C) accumulated into cstats (N/2, C, 2): the stand-alone producer of the
// statistics a conv / attention epilogue emits for free (used after kernels that cannot: 3-channel input conv, SIMT paths)
void launch_gn_cstats(int dtype, const void* x, float* cstats, int N, int H, int W, int C, cudaStream_t s);
// rs == RS_NONE: any mode; a resampling norm is GN_PLAIN or GN_SWISH, without params_out
void launch_gn_apply(int dtype, const GnArgs& a, cudaStream_t s);
void launch_gn_bwd_reduce(int dtype, const GnArgs& a, cudaStream_t s);   // zeroes + fills a.bstats, dgamma/dbeta, de
void launch_gn_bwd_apply(int dtype, const GnArgs& a, cudaStream_t s);
// second (and only) pass of the GroupNorm backward when the consumer conv's data-gradient epilogue already produced dyh and the
// channel sums (a.dy = dyh, a.bcs): folds the sums into dgamma / dbeta / group sums, then dx = rstd*(gamma*dyh - S1 - xhat*S2)
void launch_gn_bwd_apply_pre(int dtype, const GnArgs& a, cudaStream_t s);

// ---- conditioning -------------------------------------------------------------------------------------
// logsnr (B) -> posenc_ddpm -> Dense -> swish -> Dense.  pe,h1: saved (B,E) fp32.  lemb (B,E) fp32
void launch_logsnr_emb(const float* logsnr, const float* w0, const float* b0, const float* w1, const float* b1,
                       float* pe, float* h1, float* lemb, int B, int E, cudaStream_t s);
// accumulate: dw0/db0/dw1/db1 += instead of =
void launch_logsnr_emb_bwd(const float* dlemb, const float* w1, const float* pe, const float* h1, float* dh1,
                           float* dw0, float* db0, float* dw1, float* db1, int B, int E, int accumulate, cudaStream_t s);
// rays + NeRF posenc -> (2B,S,S,144)
void launch_pose_emb(int dtype, const float* R1, const float* t1, const float* R2, const float* t2, const float* K,
                     const float* cond_mask, const float* pos_emb, const float* ref_first, const float* ref_other,
                     float* kinv_scratch, void* out, int B, int S, int convention, const float* rays, cudaStream_t s);
// accumulate: dpos_emb += instead of = (dref_first / dref_other are always added to)
void launch_pose_emb_bwd(int dtype, const void* dpose, float* dpos_emb, float* dref_first, float* dref_other, int B, int S,
                         int accumulate, cudaStream_t s);
// semb = swish(lemb[b] + pe)   /   bwd: dpe (+)= dsemb*swish'(z), dlemb[b] += sum
void launch_emb_fwd(int dtype, const float* lemb, const void* pe, void* semb, int N, int HW, int E, cudaStream_t s);
void launch_emb_bwd(int dtype, const float* lemb, const void* pe, const void* dsemb, void* dpe, float* dlemb, int N, int HW,
                    int E, int write_dpe, cudaStream_t s);

// ---- plumbing -------------------------------------------------------------------------------------------
void launch_pack_input(int dtype, const float* x, const float* z, void* out, int B, int S, cudaStream_t s);
// pool (2x2 sum * scale) or replicate (x2 nearest * scale)
void launch_resample(int dtype, const void* x, void* y, int N, int Hi, int Wi, int C, int pool, float scale, int accumulate,
                     cudaStream_t s);
// dst[:, dst_off : dst_off+Cc] (+)= src[:, src_off : src_off+Cc]
void launch_copy_channels(int dtype, const void* src, void* dst, long long npix, int Cs, int Cd, int src_off, int dst_off,
                          int Cc, int accumulate, cudaStream_t s);
void launch_scale_add(int dtype, const void* src, void* dst, long long n, float alpha, int accumulate, cudaStream_t s);
void launch_extract_frame1(int dtype, const void* o, float* eps, int B, int S, cudaStream_t s);
// loss = ||eps - noise||_F ; dO (2B,S,S,3): frame0 = 0, frame1 = (eps-noise)/loss
void launch_loss(int dtype, const float* eps, const float* noise, float* sumsq_scratch, float* loss_out, void* dO, int B,
                 int S, cudaStream_t s);
// loss = (1/B) sum_b weight_b * mean_i (eps - noise)_bi^2 (weight == nullptr: all 1), reduced in fp64 in a fixed order;
// dO (2B,S,S,3): frame0 = 0, frame1 = fl32(2 weight_b / (B*S*S*3)) * (eps - noise)
void launch_loss_mse(int dtype, const float* eps, const float* noise, const float* weight, float* loss_out, void* dO, int B,
                     int S, cudaStream_t s);
// dO (2B,S,S,3): frame0 = 0, frame1 = d_eps (B,S,S,3) fp32, rounded once to the activation dtype
void launch_vjp_seed(int dtype, const float* d_eps, void* dO, int B, int S, cudaStream_t s);
// K^-1 of B cameras into kinv (B, 9): the pose embedding's rays (kernels_elem.cu) and the radiance field's (field.cu)
__global__ void kinv_kernel(const float* __restrict__ K, float* __restrict__ kinv, int B);

// ---- attention over frames ---------------------------------------------------------------------------------
struct AttnArgs {
  const void* qkv; const void* res; void* out; float* lse;
  const void* dout; float* dscratch; void* dqkv;   // backward
  int N, L, C, heads, cross;
  int scratch_zeroed;   // backward (tensor-core path): dscratch is all-zero on entry and is handed back all-zero
  float* cstats;   // optional (tensor-core forward): per-(sample, channel) [sum, sumsq] of the stored output, (N/2, C, 2) fp32, accumulated
};
void launch_attn_fwd_simt(int dtype, const AttnArgs& a, cudaStream_t s);
void launch_attn_bwd_simt(int dtype, const AttnArgs& a, cudaStream_t s);
// wgmma/TMA versions (bf16; L % 128 == 0; head_dim 16/32/64/128)
bool attn_tc_supported(int dtype, int L, int C, int heads);
void launch_attn_fwd_tc(const AttnArgs& a, cudaStream_t s);
void launch_attn_bwd_tc(const AttnArgs& a, cudaStream_t s);

// Order-insensitive accumulation.  Kernels that sum the contributions of many CTAs (or warps) into one value add them in
// fp64 -- into shared memory, or into a zeroed fp64 scratch obtained from xu_det_scratch -- instead of fp32 atomics on the
// destination; xu_det_fold then adds each fp64 sum to its fp32 destination once and re-zeroes the scratch.  fp64 keeps 29 more
// significand bits than the fp32 addends, so reordering the additions changes an fp64 sum only when its addends span about
// 29 - log2(count) binary orders of magnitude, and the fp32 value folded from it changes only if that fp64 sum then lies at an
// fp32 rounding boundary: the same inputs give the same bits on every run with overwhelming probability, not by construction.
//
// The scratch belongs to an XuDetScratch owner bound to the calling thread (XuDetBind):
//  * an engine handle owns one for its lifetime: one zeroed region per stream, on the handle's device, grown on demand
//    (also during stream capture) and freed with the handle;
//  * operator-level entry points bind a call-scoped owner that takes stream-ordered allocations (cudaMallocAsync) and
//    releases them on the same stream when the call returns.
struct XuDetScratch;
XuDetScratch* xu_det_create(bool stream_ordered);
void xu_det_destroy(XuDetScratch* d);
struct XuDetBind {
  explicit XuDetBind(XuDetScratch* d);
  ~XuDetBind();
  XuDetScratch* prev;
};
double* xu_det_scratch(cudaStream_t s, long long n);   // n zeroed doubles; nullptr (and a kernel error) if unavailable
void xu_det_fold(float* dst, double* acc, long long n, cudaStream_t s);   // dst[i] += (float)acc[i]; acc[i] = 0
__device__ __forceinline__ void xu_det_add(double* acc, float v) { atomicAdd(acc, (double)v); }

const char* xu_kernel_error();  // last launch-configuration error recorded by a launcher ("" if none)
void xu_set_kernel_error(const char* msg);
// xunet_last_error() <- the printf-formatted message; returns 1, the entries' error code
int xu_fail(const char* fmt, ...);
// after an entry's launches: 0, or xu_fail("<what>: CUDA error: <cudaGetLastError()>")
int xu_launched(const char* what);
