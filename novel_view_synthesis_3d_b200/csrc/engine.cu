// engine.cu -- static execution plan of the X-UNet (model/xunet.py:218-280) and its entries of include/xunet_b200.h:
// create, introspection, forward, backward, kernel counting and the gradient-bucket hook, plus the operator-level
// xunet_op_* entries, which share the plan's launch builders.  The C error state (xu_fail, xunet_last_error) lives here
// too.  Entries that run no plan (Adam, samplers, data, distillation, metrics, field, pose) sit beside their kernels.
//
// A config + (B,S,dtype) is compiled ONCE into a flat list of tensor descriptors (arena offsets into the
// caller-owned workspace) and op descriptors; forward() walks the list, backward() walks it in reverse with
// hand-derived gradients (no autograd, no tracing compiler).  All parameters live in ONE flat fp32 buffer whose
// leaves carry the Flax tree names/shapes (SURVEY Appendix A), so the gradient all-reduce and Adam are each a
// single pass over contiguous memory.
#include "xunet_b200.h"
#include "common.cuh"
#include "kernels.h"
#include "conv_tc.h"
#include "pose_grad.h"

#include <algorithm>
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <vector>

static thread_local char g_err[512] = "";
int xu_fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}
int xu_launched(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : xu_fail("%s: CUDA error: %s", what, cudaGetErrorString(e));
}
extern "C" const char* xunet_last_error(void) { return g_err; }
extern "C" int xunet_version(void) { return 112; }

namespace {

struct Leaf {
  std::string name;
  int ndim;
  long long shape[5];
  long long off;
  long long size;
};

struct Tensor {
  int n, h, w, c;
  bool f32;        // element type: fp32 regardless of dtype (else handle dtype)
  bool need_grad;
  bool gwritten;   // backward planning state
  long long off;   // byte offset in workspace
  long long goff;  // byte offset of gradient (-1 none)
  // GroupNorm input statistics of this tensor, per (sample, channel) [sum, sumsq] fp32 (B, C, 2): emitted by the producer's
  // epilogue (cs_fused) or by a stand-alone kernel right after it; -1: nobody normalises this tensor
  long long cstats = -1;
  bool cs_fused = false;
  int producer = -1;        // op that writes the tensor
  // gradient aliasing: a tensor used ONLY as the residual operand of one conv has gradient alpha * grad(conv output) -- instead of
  // materialising it (a scale_add pass), its producer's backward reads grad(galias) and folds gscale into its own alpha
  int galias = -1;
  float gscale = 1.f;
  int cat_a = -1, cat_b = -1;   // channel concat of two tensors (its statistics are the concatenation of theirs)
  std::string tap;
  long long numel() const { return (long long)n * h * w * c; }
};

// a convolution (N,Hi,Wi,Ci) -> (N,Ho,Wo,Co) with SAME padding, its Co outputs in nseg weight segments (conv_shape)
struct ConvShape { int N, Hi, Wi, Ci, Ho, Wo, Co, ks, stride, pad_h, pad_w, nseg; };
struct ConvKernels { ConvKernel fwd = CONV_SIMT, dgrad = CONV_SIMT, wgrad = CONV_SIMT; };

enum OpKind { OP_PACK, OP_LOGSNR, OP_POSE, OP_CONV, OP_EMB, OP_GN, OP_RESAMPLE, OP_CONCAT, OP_ATTN, OP_EXTRACT };

struct Op {
  int kind;
  int x = -1, y = -1, r = -1, e = -1;  // tensors: input, output, second input (residual / concat b), FiLM tensor
  // conv
  ConvShape cs = {};
  ConvKernels k;
  long long wT = -1, wC = -1;         // bf16 weight shadows (workspace byte offsets) for the tensor-core kernels
  long long w = -1, b = -1;            // param offsets (conv W,bias | gn gamma,beta)
  float alpha = 1.f;
  // gn
  int mode = 0, rs = 0, op_index = 0;
  long long stats = -1, bstats = -1;   // aux byte offsets
  // attn
  int cross = 0, heads = 1, impl = 0;   // impl: 1 tensor cores, 0 SIMT
  long long lse = -1, dscr = -1;
  // pose / logsnr params
  long long p0 = -1, p1 = -1, p2 = -1, p3 = -1;
  int fuse_res = 0;    // conv/attn: the residual-branch gradient is added inside the GroupNorm backward of tensor r
  int extra_src = -1;  // GN: tensor whose GRADIENT is added (x extra_alpha) to dx in gn_bwd_apply
  float extra_alpha = 0.f;
  int cs_a = -1, cs_b = -1;   // GN: tensors whose producer-emitted channel statistics cover x (b: second half of a concat)
  // fused GroupNorm backward: the data gradient of the conv that consumes this norm's output does the reduction pass
  int gnb = -1;               // conv: index of that GroupNorm op;  GN: index of the consumer conv (-1: two-kernel backward)
  long long gnp = -1, bcs = -1;   // GN: byte offsets of the (B,C) float4 parameter table and the (B,C,2) channel sums
  int film = 0;        // conv: FiLM Dense over the (pose+logsnr) embedding -- an independent branch (side stream)
  int film_idx = -1;   // GN_FILM: index into handle.film_ops of the conv that produces its `e`
  // backward accumulate flags (decided at plan time)
  int acc_x = 0, acc_r = 0, acc_e = 0;
};

}  // namespace

struct xunet_handle {
  XuDetScratch* det = xu_det_create(false);   // fp64 reduction scratch of this engine (kernels.h), freed with it
  xunet_config cfg;
  int B, S, dtype, training, N;
  size_t esize;
  std::vector<Leaf> leaves;
  long long nparams = 0;
  std::vector<Tensor> tensors;
  std::vector<Op> ops;
  std::vector<int> taps;
  long long ws_bytes = 0;
  // aux (byte offsets)
  long long a_lemb, a_pe, a_h1, a_dlemb, a_dh1, a_kinv, a_sumsq, a_eps;
  int t_in = -1, t_pose = -1, t_out = -1;
  int forward_done_train = 0;
  int static_cond = 0;       // sampler: pose-only ops and weight shadows are reused from the previous forward
  // feature cache (xunet_set_feature_cache): at cache_level L > 0 a forward runs only the ops keep[] marks, reading the
  // tensor cache_t[L] the last full forward left in the workspace
  int cache_level = 0;
  int cache_from = 0;            // the smallest level whose cached tensor is still the last full forward's (0: none)
  std::vector<int> cache_t;      // per level L >= 1: the output of the up ResnetBlock that leaves level L; [0] = -1
  int keep_level = 0;            // the level keep[], keep_fork and keep_clear were derived for
  std::vector<char> keep;        // per op
  int keep_fork = -1;            // the last kept OP_EMB: the FiLM side branch forks after it
  std::vector<std::pair<long long, long long>> keep_clear;   // (offset, bytes): the statistics a cheap forward re-produces
  std::vector<WeightPrepTable> prep;
  // weight-gradient kernels run on a side stream concurrently with the activation-gradient chain (fork/join by events;
  // captured into the same CUDA graph as parallel branches).  Created lazily at the first backward.
  cudaStream_t side = nullptr;
  int side_failed = 0;
  std::vector<int> film_ops;            // op indices of the FiLM Dense convs, forward order
  std::vector<cudaEvent_t> ev_film;     // one event per FiLM conv (forward fork/join)
  cudaEvent_t ev_fork = nullptr;
  int last_emb_op = -1;
  cudaEvent_t ev_pool[16] = {};
  cudaEvent_t ev_join = nullptr;
  int ev_next = 0;
  long long a_stats = 0, stats_bytes = 0, a_bstats = 0, bstats_bytes = 0;   // contiguous GroupNorm statistics regions
  long long a_cstats = 0, cstats_bytes = 0;                                  // contiguous per-channel statistics (one memset)
  long long a_bcs = 0, bcs_bytes = 0;                                        // contiguous backward channel sums (one memset)
  // top-level blocks in forward order (first op index, first parameter offset): the backward finishes the gradient of
  // every leaf at or above blocks[k].leaf_begin once it has walked down to blocks[k].op_begin -> gradient buckets
  struct Block { int op_begin; long long leaf_begin; };
  std::vector<Block> blocks;
  xunet_bucket_fn bucket_fn = nullptr;
  void* bucket_user = nullptr;
  std::vector<Block> bucket_pts;        // emission points, descending op index / offset

  long long alloc(long long bytes) {
    long long o = ws_bytes;
    ws_bytes += (bytes + 255) / 256 * 256;
    return o;
  }
  long long leaf(const std::string& name, std::initializer_list<long long> shape) {
    Leaf l;
    l.name = name;
    l.ndim = (int)shape.size();
    l.size = 1;
    int i = 0;
    for (long long s : shape) { l.shape[i++] = s; l.size *= s; }
    for (; i < 5; ++i) l.shape[i] = 1;
    l.off = nparams;
    nparams += l.size;
    leaves.push_back(l);
    return l.off;
  }
  int tensor(int n, int h, int w, int c, bool need_grad, const std::string& tap = "", bool f32 = false) {
    Tensor t;
    t.n = n; t.h = h; t.w = w; t.c = c; t.f32 = f32; t.need_grad = need_grad && training; t.gwritten = false;
    t.tap = tap;
    size_t es = f32 ? 4 : esize;
    t.off = alloc(t.numel() * es);
    t.goff = t.need_grad ? alloc(t.numel() * es) : -1;
    tensors.push_back(t);
    int id = (int)tensors.size() - 1;
    if (!tap.empty()) taps.push_back(id);
    return id;
  }
};

namespace {

static void same_pad(int in, int k, int s, int& lo, int& out) {
  out = (in + s - 1) / s;
  int total = (out - 1) * s + k - in;
  if (total < 0) total = 0;
  lo = total / 2;
}

// The helpers below choose the kernel of every conv and attention launch, fill its arguments and launch it, and fill the
// launch arguments of the GroupNorm path; the engine and the operator-level entry points (xunet_op_conv, xunet_op_attention,
// xunet_op_groupnorm, ...) both use them, so the operator tests run the launches the engine runs.

static ConvShape conv_shape(int N, int Hi, int Wi, int Ci, int Co, int ks, int stride, int nseg) {
  ConvShape s = {N, Hi, Wi, Ci, Hi, Wi, Co, ks, stride, 0, 0, nseg};
  if (ks == 3) { same_pad(Hi, 3, stride, s.pad_h, s.Ho); same_pad(Wi, 3, stride, s.pad_w, s.Wo); }
  return s;
}

// the kernels the engine runs for a conv of this shape (res: it adds a residual).  The direct 3-channel kernels and the tensor-core
// ones never take the same shape.
static ConvKernels conv_kernels(int dtype, const ConvShape& s, bool res) {
  ConvKernels k;
  if (conv_cin3_supported(s.Ci, s.Co, s.ks, s.stride, s.nseg, res)) k.fwd = k.wgrad = CONV_CIN3;
  if (conv_cout3_supported(s.Ci, s.Co, s.ks, s.stride, s.nseg, res)) k.fwd = k.dgrad = k.wgrad = CONV_COUT3;
  if (conv_tc_supported(dtype, 0, s.N, s.Hi, s.Wi, s.Ci, s.Co, s.ks, s.stride, s.nseg)) k.fwd = CONV_TC;
  if (conv_tc_supported(dtype, 1, s.N, s.Hi, s.Wi, s.Ci, s.Co, s.ks, s.stride, s.nseg)) k.dgrad = CONV_TC;
  if (wgrad_tc_supported(dtype, s.N, s.Hi, s.Wi, s.Ci, s.Co, s.ks, s.stride, s.nseg)) k.wgrad = CONV_TC;
  return k;
}

static ConvArgs conv_fwd_args(const ConvShape& s, const void* x, const float* w, const float* bias, const void* res, void* y,
                              float alpha) {
  ConvArgs a;
  a.x = x; a.y = y; a.res = res; a.w = w; a.bias = bias;
  a.N = s.N; a.Hi = s.Hi; a.Wi = s.Wi; a.Ci = s.Ci; a.Ho = s.Ho; a.Wo = s.Wo; a.Co = s.Co;
  a.ks = s.ks; a.stride = s.stride; a.pad_h = s.pad_h; a.pad_w = s.pad_w; a.mode = 0;
  a.wCi = s.Ci; a.wCo = s.Co; a.segw = s.Co / s.nseg;
  a.alpha = alpha; a.accumulate = 0;
  return a;
}
// the data gradient runs the forward's weights and padding backwards (mode 1): from dY (Ho,Wo,Co) to dX (Hi,Wi,Ci)
static ConvArgs conv_dgrad_args(const ConvShape& s, const void* dy, const float* w, void* dx, float alpha, int accumulate) {
  ConvArgs a = conv_fwd_args(s, dy, w, nullptr, nullptr, dx, alpha);
  a.Hi = s.Ho; a.Wi = s.Wo; a.Ci = s.Co; a.Ho = s.Hi; a.Wo = s.Wi; a.Co = s.Ci;
  a.mode = 1; a.accumulate = accumulate;
  return a;
}
static WgradArgs conv_wgrad_args(const ConvShape& s, const void* x, const void* dy, float* dw, float* dbias, float alpha) {
  WgradArgs a;
  a.x = x; a.dy = dy; a.dw = dw; a.dbias = dbias;
  a.N = s.N; a.Hi = s.Hi; a.Wi = s.Wi; a.Ci = s.Ci; a.Ho = s.Ho; a.Wo = s.Wo; a.Co = s.Co;
  a.ks = s.ks; a.stride = s.stride; a.pad_h = s.pad_h; a.pad_w = s.pad_w; a.segw = s.Co / s.nseg;
  a.alpha = alpha;
  return a;
}
static AttnArgs attn_args(const void* qkv, const void* res, void* out, float* lse, int N, int L, int C, int heads, int cross) {
  AttnArgs a;
  memset(&a, 0, sizeof(a));
  a.qkv = qkv; a.res = res; a.out = out; a.lse = lse;
  a.N = N; a.L = L; a.C = C; a.heads = heads; a.cross = cross;
  return a;
}

// conv forward (a.mode 0) or data gradient (a.mode 1); shadow: the bf16 weight shadow a tensor-core conv reads
static void dispatch_conv(int dtype, ConvKernel k, const ConvArgs& a, const void* shadow, cudaStream_t s) {
  if (k == CONV_TC) launch_conv_tc(a, shadow, s);
  else if (k == CONV_SIMT) launch_conv_simt(dtype, a, s);
  else launch_conv_direct(dtype, k, a, s);
}
static void dispatch_wgrad(int dtype, ConvKernel k, const WgradArgs& a, cudaStream_t s) {
  if (k == CONV_TC) launch_wgrad_tc(a, s);
  else if (k == CONV_SIMT) launch_wgrad_simt(dtype, a, s);
  else launch_wgrad_direct(dtype, k, a, s);
}
static void dispatch_attn_fwd(int dtype, int impl, const AttnArgs& a, cudaStream_t s) {
  if (impl == 1) launch_attn_fwd_tc(a, s);
  else launch_attn_fwd_simt(dtype, a, s);
}
static void dispatch_attn_bwd(int dtype, int impl, const AttnArgs& a, cudaStream_t s) {
  if (impl == 1) launch_attn_bwd_tc(a, s);
  else launch_attn_bwd_simt(dtype, a, s);
}

// appends a conv's weight to a bf16 shadow table: src its element offset in the fp32 parameters, dstT / dstC the byte offsets of
// the forward / data-gradient shadows (-1: none)
static void prep_entry(WeightPrepTable& tab, const ConvShape& s, long long src, long long dstT, long long dstC) {
  WeightPrepEntry& e = tab.e[tab.n++];
  e.src = src; e.dstT = dstT; e.dstC = dstC; e.prefix = tab.total;
  e.Ci = s.Ci; e.Co = s.Co; e.taps = s.ks * s.ks; e.nseg = s.nseg;
  tab.total += (long long)e.taps * e.Ci * e.Co;
}

// a convolution's forward epilogue emits the GroupNorm input statistics of its output (EPI 1); else launch_gn_cstats follows it
static bool conv_emits_stats(ConvKernel k, const ConvShape& s) {
  return k == CONV_TC && s.nseg == 1 && s.stride == 1 && conv_tc_stats_supported(0, s.N, s.Ho, s.Wo);
}
// likewise the tensor-core attention forward; the SIMT one cannot
static bool attn_emits_stats(int impl) { return impl == 1; }
// the data gradient of a conv that consumes a GroupNorm output can also run the norm's first backward pass (set_gn_bwd_epilogue)
static bool dgrad_fuses_gn_bwd(ConvKernel k, const ConvShape& s) {
  return k == CONV_TC && s.stride == 1 && conv_tc_stats_supported(1, s.N, s.Hi, s.Wi);
}

// the data gradient `a` of the conv that consumes a GroupNorm output also runs the norm's first backward pass (EPI 2; EPI 3
// with the FiLM tensor e and its gradient de): it stores dyh and adds the channel sums to bcs
static void set_gn_bwd_epilogue(ConvArgs& a, const void* gn_x, const void* gn_params, int mode, const void* e, void* de,
                                float* bcs, float drop_rate, int op_index, const unsigned long long* seed_dev, int train) {
  a.gn_x = gn_x;
  a.gn_params = gn_params;
  a.gn_swish = mode == GN_SWISH ? 1 : 0;
  a.cstats = bcs;
  if (mode == GN_FILM) {
    a.gn_e = e;
    a.gn_de = de;
    a.gn_drop_rate = drop_rate; a.gn_drop_op = op_index; a.gn_seed_dev = seed_dev; a.gn_train = train;
  }
}

static GnArgs gn_fill(const void* x, void* y, const void* e, const float* gamma, const float* beta, float* stats, int N, int H,
                      int W, int C, int mode, int rs, float drop_rate, int op_index, const unsigned long long* seed_dev, int train) {
  GnArgs a;
  memset(&a, 0, sizeof(a));
  a.x = x; a.y = y; a.e = e;
  a.gamma = gamma; a.beta = beta;
  a.stats = stats;
  a.N = N; a.H = H; a.W = W; a.C = C; a.mode = mode; a.rs = rs;
  a.drop_rate = drop_rate; a.op_index = op_index; a.seed_dev = seed_dev; a.train = train;
  a.skip_zero = 1;
  return a;
}

// the resample launches of an OP_RESAMPLE: the forward averages 2x2 pixels (RS_DOWN) or repeats each pixel 2x2 (RS_UP); the
// backward runs the adjoint on the output's gradient -- replicate x 0.25, or the 2x2 sum -- times that gradient's alias scale
struct ResampleArgs { int pool; float scale; };
static ResampleArgs resample_fwd_args(int rs) { return {rs == RS_DOWN ? 1 : 0, rs == RS_DOWN ? 0.25f : 1.f}; }
static ResampleArgs resample_bwd_args(int rs, float gscale) { return {rs == RS_UP ? 1 : 0, (rs == RS_DOWN ? 0.25f : 1.f) * gscale}; }

// one channel copy of a concat y = [a | b] (ca + cb channels): the forward copies a (second = 0) or b into y, the backward
// copies the matching channels of grad(y) out to grad(a) or grad(b)
struct ChannelCopy { int Cs, Cd, src_off, dst_off, Cc; };
static ChannelCopy concat_copy(int ca, int cb, bool bwd, bool second) {
  const int Cd = ca + cb;
  if (!bwd) return second ? ChannelCopy{cb, Cd, 0, ca, cb} : ChannelCopy{ca, Cd, 0, 0, ca};
  return second ? ChannelCopy{Cd, cb, ca, 0, cb} : ChannelCopy{Cd, ca, 0, 0, ca};
}

struct Builder {
  xunet_handle& H;
  explicit Builder(xunet_handle& h) : H(h) {}
  int res_counter = 0;

  int conv(int x, int cout, int ks, int stride, long long w, long long b, int res, float alpha, int nseg,
           const std::string& tap = "") {
    const Tensor tx = H.tensors[x];   // by value: H.tensor() below may reallocate the vector
    Op o;
    o.kind = OP_CONV; o.x = x; o.r = res; o.w = w; o.b = b; o.alpha = alpha;
    o.cs = conv_shape(tx.n, tx.h, tx.w, tx.c, cout, ks, stride, nseg);
    o.k = conv_kernels(H.dtype, o.cs, res >= 0);
    o.y = H.tensor(tx.n, o.cs.Ho, o.cs.Wo, cout, true, tap);
    if (o.k.fwd == CONV_TC) o.wT = H.alloc((long long)ks * ks * tx.c * cout * 2);
    if (o.k.dgrad == CONV_TC && tx.need_grad) o.wC = H.alloc((long long)ks * ks * tx.c * cout * 2);
    H.ops.push_back(o);
    H.tensors[o.y].producer = (int)H.ops.size() - 1;
    return o.y;
  }
  int gn(int x, int mode, int rs, long long gamma, long long beta, int e, int op_index) {
    const Tensor tx = H.tensors[x];
    int ho = rs == RS_DOWN ? tx.h / 2 : (rs == RS_UP ? tx.h * 2 : tx.h);
    int wo = rs == RS_DOWN ? tx.w / 2 : (rs == RS_UP ? tx.w * 2 : tx.w);
    int y = H.tensor(tx.n, ho, wo, tx.c, true);
    Op o;
    o.kind = OP_GN; o.x = x; o.y = y; o.e = e; o.mode = mode; o.rs = rs; o.w = gamma; o.b = beta; o.op_index = op_index;
    o.stats = -1; o.bstats = -1;   // assigned at the end of build(): one contiguous region -> ONE memset per pass
    // statistics come from whoever produced x (both halves of a concat): no statistics pass over HBM.  build() checks that
    // every norm found its producers.
    const int sa = tx.cat_a >= 0 ? tx.cat_a : x, sb = tx.cat_a >= 0 ? tx.cat_b : -1;
    if (H.tensors[sa].producer >= 0 && (sb < 0 || H.tensors[sb].producer >= 0) && H.tensors[sa].cat_a < 0 &&
        (sb < 0 || H.tensors[sb].cat_a < 0)) {
      o.cs_a = sa; o.cs_b = sb;
      H.tensors[sa].cstats = 0;                      // marked; offsets assigned at the end of build()
      if (sb >= 0) H.tensors[sb].cstats = 0;
    }
    H.ops.push_back(o);
    return y;
  }
  int resample(int x, int rs) {
    const Tensor tx = H.tensors[x];
    int ho = rs == RS_DOWN ? tx.h / 2 : tx.h * 2, wo = rs == RS_DOWN ? tx.w / 2 : tx.w * 2;
    int y = H.tensor(tx.n, ho, wo, tx.c, true);
    Op o;
    o.kind = OP_RESAMPLE; o.x = x; o.y = y; o.rs = rs;
    H.ops.push_back(o);
    return y;
  }
  int concat(int a, int b) {
    const Tensor ta = H.tensors[a];
    const Tensor tb = H.tensors[b];
    int y = H.tensor(ta.n, ta.h, ta.w, ta.c + tb.c, true);
    Op o;
    o.kind = OP_CONCAT; o.x = a; o.r = b; o.y = y;
    H.ops.push_back(o);
    H.tensors[y].cat_a = a; H.tensors[y].cat_b = b;
    return y;
  }
  void gn_leaves(const std::string& p, int c, long long& gamma, long long& beta) {
    gamma = H.leaf(p + "/GroupNorm_0/scale", {c});
    beta = H.leaf(p + "/GroupNorm_0/bias", {c});
  }
  // ResnetBlock  model/xunet.py:63-92
  int resblock(const std::string& p, int x_in, int semb, int features, int rs, const std::string& tap) {
    const int C = H.tensors[x_in].c;
    if (features <= 0) features = C;
    const int E = H.cfg.emb_ch;
    const int op_index = res_counter++;
    long long g0, b0, g1, b1;
    gn_leaves(p + "/GroupNorm_0", C, g0, b0);
    long long w0 = H.leaf(p + "/Conv_0/kernel", {1, 3, 3, C, features});
    long long c0 = H.leaf(p + "/Conv_0/bias", {features});
    gn_leaves(p + "/GroupNorm_1", features, g1, b1);
    long long wf = H.leaf(p + "/FiLM_0/Dense_0/kernel", {E, 2 * features});
    long long bf = H.leaf(p + "/FiLM_0/Dense_0/bias", {2 * features});
    long long w1 = H.leaf(p + "/Conv_1/kernel", {1, 3, 3, features, features});
    long long c1 = H.leaf(p + "/Conv_1/bias", {features});
    long long wd = -1, bd = -1;
    if (C != features) {
      wd = H.leaf(p + "/Dense_0/kernel", {C, features});
      bd = H.leaf(p + "/Dense_0/bias", {features});
    }
    int a = gn(x_in, GN_SWISH, rs, g0, b0, -1, op_index);
    int xin2 = rs != RS_NONE ? resample(x_in, rs) : x_in;
    int h1 = conv(a, features, 3, 1, w0, c0, -1, 1.f, 1);
    int e = conv(semb, 2 * features, 1, 1, wf, bf, -1, 1.f, 1);
    H.ops.back().film = 1;
    H.film_ops.push_back((int)H.ops.size() - 1);
    int h2 = gn(h1, GN_FILM, RS_NONE, g1, b1, e, op_index);
    H.ops.back().film_idx = (int)H.film_ops.size() - 1;
    int sk = xin2;
    if (C != features) sk = conv(xin2, features, 1, 1, wd, bd, -1, 1.f, 1);
    return conv(h2, features, 3, 1, w1, c1, sk, XU_RSQRT2, 1, tap);
  }
  // AttnBlock  model/xunet.py:105-127 (+AttnLayer :94-103)
  int attnblock(const std::string& p, int h_in, int cross, const std::string& tap) {
    const Tensor t = H.tensors[h_in];
    const int C = t.c, heads = H.cfg.attn_heads, hd = C / heads;
    long long g, b;
    gn_leaves(p + "/GroupNorm_0", C, g, b);
    long long wq = H.leaf(p + "/AttnLayer_0/DenseGeneral_0/kernel", {C, heads, hd});
    H.leaf(p + "/AttnLayer_0/DenseGeneral_1/kernel", {C, heads, hd});
    H.leaf(p + "/AttnLayer_0/DenseGeneral_2/kernel", {C, heads, hd});
    long long bq = H.leaf(p + "/AttnLayer_0/DenseGeneral_0/bias", {heads, hd});
    H.leaf(p + "/AttnLayer_0/DenseGeneral_1/bias", {heads, hd});
    H.leaf(p + "/AttnLayer_0/DenseGeneral_2/bias", {heads, hd});
    int gno = gn(h_in, GN_PLAIN, RS_NONE, g, b, -1, 0);
    int qkv = conv(gno, 3 * C, 1, 1, wq, bq, -1, 1.f, 3);
    int y = H.tensor(t.n, t.h, t.w, C, true, tap);
    Op o;
    o.kind = OP_ATTN; o.x = qkv; o.y = y; o.r = h_in; o.cross = cross; o.heads = heads;
    o.impl = attn_tc_supported(H.dtype, t.h * t.w, C, heads) ? 1 : 0;
    o.lse = H.alloc(sizeof(float) * t.n * heads * t.h * t.w);
    o.dscr = H.training ? H.alloc(sizeof(float) * t.n * heads * t.h * t.w) : -1;   // D [N,heads,L]
    H.ops.push_back(o);
    H.tensors[y].producer = (int)H.ops.size() - 1;
    return y;
  }
  bool is_attn_res(int r) {
    for (int i = 0; i < H.cfg.n_attn_resolutions; ++i)
      if (H.cfg.attn_resolutions[i] == r) return true;
    return false;
  }
  int n_xb = 0, n_rb = 0;
  void mark_block() { H.blocks.push_back({(int)H.ops.size(), H.nparams}); }
  int xblock(int x, int semb, int features) {
    mark_block();
    std::string name = "XUNetBlock_" + std::to_string(n_xb++);
    bool use_attn = is_attn_res(H.tensors[x].h);
    int h = resblock(name + "/ResnetBlock_0", x, semb, features, RS_NONE, use_attn ? "" : name);
    if (use_attn) {
      h = attnblock(name + "/AttnBlock_0", h, 0, "");
      h = attnblock(name + "/AttnBlock_1", h, 1, name);
    }
    return h;
  }
  int rblock(int x, int semb, int rs) {
    mark_block();
    std::string name = "ResnetBlock_" + std::to_string(n_rb++);
    return resblock(name, x, semb, -1, rs, name);
  }

  int build() {
    const xunet_config& c = H.cfg;
    const int B = H.B, S = H.S, N = 2 * B, E = c.emb_ch, L = c.n_levels;
    // ---- ConditioningProcessor  model/xunet.py:150-203
    const std::string cp = "ConditioningProcessor_0";
    Op ol;
    ol.kind = OP_LOGSNR;
    ol.p0 = H.leaf(cp + "/Dense_0/kernel", {E, E});
    ol.p1 = H.leaf(cp + "/Dense_0/bias", {E});
    ol.p2 = H.leaf(cp + "/Dense_1/kernel", {E, E});
    ol.p3 = H.leaf(cp + "/Dense_1/bias", {E});
    H.a_lemb = H.alloc(sizeof(float) * B * E);
    H.a_pe = H.alloc(sizeof(float) * B * E);
    H.a_h1 = H.alloc(sizeof(float) * B * E);
    H.a_dlemb = H.alloc(sizeof(float) * B * E);
    H.a_dh1 = H.alloc(sizeof(float) * B * E);
    H.a_kinv = H.alloc(sizeof(float) * B * 9);
    H.a_sumsq = H.alloc(sizeof(float) * 4);
    H.a_eps = H.alloc(sizeof(float) * (long long)B * S * S * 3);
    H.ops.push_back(ol);
    Op op;
    op.kind = OP_POSE;
    if (c.use_pos_emb) op.p0 = H.leaf(cp + "/pos_emb", {S, S, XU_POSE_DIM});
    if (c.use_ref_pose_emb) {
      op.p1 = H.leaf(cp + "/ref_pose_emb_first", {XU_POSE_DIM});
      op.p2 = H.leaf(cp + "/ref_pose_emb_other", {XU_POSE_DIM});
    }
    const bool pose_grad = c.use_pos_emb || c.use_ref_pose_emb;
    H.t_pose = H.tensor(N, S, S, XU_POSE_DIM, pose_grad, "pose_emb");
    op.y = H.t_pose;
    H.ops.push_back(op);
    std::vector<int> semb(L);
    for (int i = 0; i < L; ++i) {
      long long w = H.leaf(cp + "/Conv_" + std::to_string(i) + "/kernel", {1, 3, 3, XU_POSE_DIM, E});
      long long b = H.leaf(cp + "/Conv_" + std::to_string(i) + "/bias", {E});
      int pe = conv(H.t_pose, E, 3, 1 << i, w, b, -1, 1.f, 1, "pose_emb_" + std::to_string(i));
      const Tensor tp = H.tensors[pe];
      int se = H.tensor(tp.n, tp.h, tp.w, E, true);
      Op oe;
      oe.kind = OP_EMB; oe.x = pe; oe.y = se;
      H.ops.push_back(oe);
      H.last_emb_op = (int)H.ops.size() - 1;
      semb[i] = se;
    }
    // ---- input conv  model/xunet.py:228-229
    H.t_in = H.tensor(N, S, S, 3, false);
    Op opk;
    opk.kind = OP_PACK; opk.y = H.t_in;
    H.ops.push_back(opk);
    long long w_in = H.leaf("Conv_0/kernel", {1, 3, 3, 3, c.ch});
    long long b_in = H.leaf("Conv_0/bias", {c.ch});
    int h = conv(H.t_in, c.ch, 3, 1, w_in, b_in, -1, 1.f, 1, "Conv_0");
    std::vector<int> hs;
    hs.push_back(h);
    H.cache_t.assign(L, -1);
    // ---- down  :231-246
    for (int i = 0; i < L; ++i) {
      for (int k = 0; k < c.num_res_blocks; ++k) {
        h = xblock(h, semb[i], c.ch * c.ch_mult[i]);
        hs.push_back(h);
      }
      if (i != L - 1) {
        h = rblock(h, semb[i + 1], RS_DOWN);
        hs.push_back(h);
      }
    }
    // ---- middle  :249-255
    h = xblock(h, semb[L - 1], c.ch * c.ch_mult[L - 1]);
    // ---- up  :257-271
    for (int i = L - 1; i >= 0; --i) {
      for (int k = 0; k < c.num_res_blocks + 1; ++k) {
        int skip = hs.back();
        hs.pop_back();
        int cat = concat(h, skip);
        // use_attn is decided on the skip's resolution (== h's resolution)
        h = xblock(cat, semb[i], c.ch * c.ch_mult[i]);
      }
      if (i != 0) H.cache_t[i] = h = rblock(h, semb[i - 1], RS_UP);
    }
    if (!hs.empty()) return xu_fail("internal: skip stack not empty");
    // ---- head  :275-280
    mark_block();
    long long g, b;
    gn_leaves("GroupNorm_0", H.tensors[h].c, g, b);
    long long w_out = H.leaf("Conv_1/kernel", {1, 3, 3, H.tensors[h].c, 3});
    long long b_out = H.leaf("Conv_1/bias", {3});
    int a = gn(h, GN_SWISH, RS_NONE, g, b, -1, 0);
    H.t_out = conv(a, 3, 3, 1, w_out, b_out, -1, 1.f, 1, "out_both_frames");
    Op ox;
    ox.kind = OP_EXTRACT; ox.x = H.t_out;
    H.ops.push_back(ox);

    {
      const long long per = sizeof(float) * H.B * XU_GROUPS * 2;
      int ngn = 0;
      for (const Op& o : H.ops) ngn += o.kind == OP_GN;
      H.stats_bytes = per * ngn;
      H.a_stats = H.alloc(H.stats_bytes);
      if (H.training) { H.bstats_bytes = per * ngn; H.a_bstats = H.alloc(H.bstats_bytes); }
      int k = 0;
      for (Op& o : H.ops)
        if (o.kind == OP_GN) { o.stats = H.a_stats + per * k; o.bstats = H.training ? H.a_bstats + per * k : -1; ++k; }
    }
    // ---- per-channel GroupNorm statistics: one region (one memset per forward); decide who emits them
    {
      H.cstats_bytes = 0;
      for (Tensor& t : H.tensors) {
        if (t.cstats < 0) continue;
        const long long bytes = (sizeof(float) * 2 * (long long)H.B * t.c + 255) / 256 * 256;
        t.cstats = H.cstats_bytes;
        H.cstats_bytes += bytes;
        const Op& po = H.ops[t.producer];
        if (po.kind == OP_CONV) t.cs_fused = conv_emits_stats(po.k.fwd, po.cs);
        else if (po.kind == OP_ATTN) t.cs_fused = attn_emits_stats(po.impl);
      }
      H.a_cstats = H.alloc(H.cstats_bytes);
      for (Tensor& t : H.tensors) if (t.cstats >= 0) t.cstats += H.a_cstats;
    }
    // ---- bf16 weight shadows for the tensor-core convs: one table-driven cast/transpose kernel per forward
    {
      WeightPrepTable tab;
      tab.n = 0; tab.total = 0;
      for (const Op& o : H.ops) {
        if (o.kind != OP_CONV || (o.wT < 0 && o.wC < 0)) continue;
        if (tab.n == XU_PREP_MAX) { H.prep.push_back(tab); tab.n = 0; tab.total = 0; }
        prep_entry(tab, o.cs, o.w, o.wT, o.wC);
      }
      if (tab.n) H.prep.push_back(tab);
    }
    // ---- fuse "grad(residual) += alpha * grad(y)" into the backward of the GroupNorm that reads the same tensor
    if (H.training) {
      for (size_t i = 0; i < H.ops.size(); ++i) {
        Op& o = H.ops[i];
        const bool is_res_conv = o.kind == OP_CONV && o.r >= 0;
        if (!(is_res_conv || o.kind == OP_ATTN) || !H.tensors[o.r].need_grad) continue;
        for (size_t g = 0; g < i; ++g) {
          Op& gn = H.ops[g];
          if (gn.kind == OP_GN && gn.x == o.r && gn.rs == RS_NONE && gn.extra_src < 0) {
            gn.extra_src = o.y;
            gn.extra_alpha = o.kind == OP_CONV ? o.alpha : XU_RSQRT2;
            o.fuse_res = 1;
            break;
          }
        }
      }
    }
    // ---- fused GroupNorm backward: a norm without resampling, plain or +swish, whose output feeds exactly one tensor-core conv
    // -> that conv's data-gradient epilogue emits dyh and the channel sums; the norm's backward is then ONE elementwise kernel
    if (H.training) {
      H.bcs_bytes = 0;
      for (size_t g = 0; g < H.ops.size(); ++g) {
        Op& gn = H.ops[g];
        if (gn.kind != OP_GN || gn.rs != RS_NONE) continue;
        int consumer = -1, users = 0;
        for (size_t k = g + 1; k < H.ops.size(); ++k) {
          const Op& u = H.ops[k];
          if (u.x == gn.y || u.r == gn.y || u.e == gn.y) { ++users; if (u.kind == OP_CONV && u.x == gn.y) consumer = (int)k; }
        }
        if (users != 1 || consumer < 0) continue;
        Op& cv = H.ops[consumer];
        const Tensor& tx = H.tensors[gn.x];
        if (!dgrad_fuses_gn_bwd(cv.k.dgrad, cv.cs) || !H.tensors[gn.y].need_grad) continue;
        gn.gnb = consumer; cv.gnb = (int)g;
        gn.gnp = H.alloc(sizeof(float) * 4 * (long long)H.B * tx.c);
        gn.bcs = H.bcs_bytes;
        H.bcs_bytes += (sizeof(float) * 2 * (long long)H.B * tx.c + 255) / 256 * 256;
      }
      H.a_bcs = H.alloc(H.bcs_bytes);
      for (Op& o : H.ops) if (o.kind == OP_GN && o.gnb >= 0) o.bcs += H.a_bcs;
    }
    // ---- residual operands whose gradient is just alpha * grad(y): alias instead of a scale_add pass
    if (H.training) {
      for (Op& o : H.ops) {
        if (o.kind != OP_CONV || o.r < 0 || o.fuse_res || !H.tensors[o.r].need_grad) continue;
        Tensor& tr = H.tensors[o.r];
        if (tr.producer < 0 && !tr.tap.empty()) continue;
        int users = 0;
        for (const Op& u : H.ops) users += (u.x == o.r) + (u.r == o.r) + (u.e == o.r) + (u.kind == OP_GN && u.extra_src == o.r);
        bool ok = users == 1 && tr.tap.empty() && tr.cat_a < 0;
        // the producer must be an op whose backward can fold a scale: the 1x1 skip Dense, or the residual-path resample
        int prod = -1;
        for (size_t k = 0; k < H.ops.size(); ++k) if (H.ops[k].y == o.r && (H.ops[k].kind == OP_CONV || H.ops[k].kind == OP_RESAMPLE)) prod = (int)k;
        if (!ok || prod < 0 || H.ops[prod].gnb >= 0) continue;
        tr.galias = o.y;
        tr.gscale = o.alpha;
        o.fuse_res = 2;           // no scale_add, no claim: the gradient of r lives in grad(y)
      }
    }
    // ---- backward planning: first writer of a gradient overwrites, later ones accumulate
    if (H.training) {
      auto claim = [&](int t) -> int {
        if (t < 0 || !H.tensors[t].need_grad) return 0;
        int f = H.tensors[t].gwritten ? 1 : 0;
        H.tensors[t].gwritten = true;
        return f;
      };
      for (int i = (int)H.ops.size() - 1; i >= 0; --i) {
        Op& o = H.ops[i];
        switch (o.kind) {
          case OP_EXTRACT: claim(o.x); break;
          case OP_CONV: o.acc_r = o.fuse_res ? 0 : claim(o.r); o.acc_x = claim(o.x); break;
          case OP_GN: o.acc_e = claim(o.e); o.acc_x = claim(o.x); break;
          case OP_EMB: o.acc_x = claim(o.x); break;
          case OP_RESAMPLE: o.acc_x = claim(o.x); break;
          case OP_CONCAT: o.acc_x = claim(o.x); o.acc_r = claim(o.r); break;
          case OP_ATTN: o.acc_r = o.fuse_res ? 0 : claim(o.r); o.acc_x = claim(o.x); break;
          default: break;
        }
      }
      // the fused GroupNorm backward overwrites its outputs: drop it wherever a gradient would have to accumulate
      for (Op& gn : H.ops) {
        if (gn.kind != OP_GN || gn.gnb < 0) continue;
        Op& cv = H.ops[gn.gnb];
        if (cv.acc_x != 0 || (gn.mode == GN_FILM && gn.acc_e != 0)) { cv.gnb = -1; gn.gnb = -1; }
      }
      // emb_bwd_kernel stores grad(pose-embedding level): each level must feed nothing but its own OP_EMB
      for (const Op& o : H.ops)
        if (o.kind == OP_EMB && o.acc_x) return xu_fail("internal: a pose-embedding level has a gradient writer besides its OP_EMB");
    }
    for (const Op& o : H.ops)
      if (o.kind == OP_GN && o.cs_a < 0) return xu_fail("internal: a GroupNorm input has no producer-emitted statistics");
    return 0;
  }
};

struct Ctx {
  xunet_handle* h;
  const float* params;
  float* grads;
  char* ws;
  const xunet_batch* batch;
  const unsigned long long* seed_dev;
  int train;
  cudaStream_t s;
  cudaStream_t side = nullptr;   // non-null: weight gradients go here
  int acc_grads = 0;             // backward: add the parameter gradient into `grads` (xunet_backward_accumulate)
  int mse = 0;                   // backward: seed with the mean-squared loss instead of the Frobenius norm (xunet_backward_mse)
  const float* loss_weight = nullptr;   // mse: per-sample weights (B), nullptr = all 1
  const float* d_eps = nullptr;  // backward: seed with the caller's dL/d(eps_hat) (B,S,S,3) instead of a loss (xunet_backward_vjp)
  float* dx = nullptr;           // backward: dL/dx and dL/dz (B,S,S,3) fp32 of the two input views, nullptr = not computed
  float* dz = nullptr;
  const xunet_input_grads* cam = nullptr;   // backward: ray / camera gradients (xunet_backward_vjp_inputs), nullptr = none
  void* act(int t) const { return ws + h->tensors[t].off; }
  void* grad(int t) const { const Tensor& x = h->tensors[t]; return ws + (x.galias >= 0 ? h->tensors[x.galias].goff : x.goff); }
  float gscale(int t) const { return h->tensors[t].gscale; }
  float* aux(long long off) const { return reinterpret_cast<float*>(ws + off); }
  const float* P(long long off) const { return off < 0 ? nullptr : params + off; }
  float* G(long long off) const { return off < 0 ? nullptr : grads + off; }
  const void* shadow(long long off) const { return off < 0 ? nullptr : ws + off; }
};

static void destroy_side(xunet_handle* h) {
  if (h->side) cudaStreamDestroy(h->side);
  h->side = nullptr;
  for (int i = 0; i < 16; ++i) { if (h->ev_pool[i]) cudaEventDestroy(h->ev_pool[i]); h->ev_pool[i] = nullptr; }
  if (h->ev_join) cudaEventDestroy(h->ev_join);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  h->ev_join = h->ev_fork = nullptr;
  for (auto& ev : h->ev_film) if (ev) cudaEventDestroy(ev);
  h->ev_film.clear();
}

// side stream + events, created at the first forward/backward (XUNET_NO_SIDE_STREAM=1 keeps everything on one stream)
static cudaStream_t ensure_side(xunet_handle* h) {
  const char* e = getenv("XUNET_NO_SIDE_STREAM");
  if (e && e[0] == '1') return nullptr;
  if (h->side_failed) return nullptr;
  if (h->side == nullptr) {
    // any failure here -> single-stream execution (correct, just without the overlap); never a half-built fork/join
    bool ok = cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; i < 16 && ok; ++i) ok = cudaEventCreateWithFlags(&h->ev_pool[i], cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) == cudaSuccess;
    if (ok) {
      h->ev_film.assign(h->film_ops.size(), nullptr);
      for (auto& ev : h->ev_film) ok = ok && cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) == cudaSuccess;
    }
    if (!ok) {
      cudaGetLastError();
      destroy_side(h);
      h->side_failed = 1;
      return nullptr;
    }
  }
  return h->side;
}

static void run_conv_fwd(const Ctx& c, const Op& o) {
  const Tensor& y = c.h->tensors[o.y];
  ConvArgs a = conv_fwd_args(o.cs, c.act(o.x), c.P(o.w), c.P(o.b), o.r >= 0 ? c.act(o.r) : nullptr, c.act(o.y), o.alpha);
  a.cstats = (y.cstats >= 0 && y.cs_fused) ? reinterpret_cast<float*>(c.ws + y.cstats) : nullptr;
  dispatch_conv(c.h->dtype, o.k.fwd, a, c.shadow(o.wT), c.s);
  if (y.cstats >= 0 && !y.cs_fused)     // producer without a statistics epilogue (3-channel input conv, SIMT paths)
    launch_gn_cstats(c.h->dtype, c.act(o.y), reinterpret_cast<float*>(c.ws + y.cstats), y.n, y.h, y.w, y.c, c.s);
}

static void run_conv_bwd(const Ctx& c, const Op& o) {
  const Tensor& x = c.h->tensors[o.x];
  const Tensor& y = c.h->tensors[o.y];
  const int dt = c.h->dtype;
  if (o.r >= 0 && c.h->tensors[o.r].need_grad && !o.fuse_res)
    launch_scale_add(dt, c.grad(o.y), c.grad(o.r), y.numel(), o.alpha, o.acc_r, c.s);
  cudaStream_t ws = c.s;
  if (c.side != nullptr) {   // fork: everything grad(y) depends on is already ordered on the main stream
    cudaEvent_t ev = c.h->ev_pool[c.h->ev_next];
    c.h->ev_next = (c.h->ev_next + 1) % 16;
    cudaEventRecord(ev, c.s);
    cudaStreamWaitEvent(c.side, ev, 0);
    ws = c.side;
  }
  const float alpha = o.alpha * c.gscale(o.y);
  dispatch_wgrad(dt, o.k.wgrad, conv_wgrad_args(o.cs, c.act(o.x), c.grad(o.y), c.G(o.w), c.G(o.b), alpha), ws);
  if (x.need_grad) {
    // the FiLM branch's data gradient feeds only the embedding backward at the very end: keep it on the side stream
    cudaStream_t ds = (o.film && c.side != nullptr) ? c.side : c.s;
    ConvArgs a = conv_dgrad_args(o.cs, c.grad(o.y), c.P(o.w), c.grad(o.x), alpha, o.acc_x);
    if (o.gnb >= 0) {     // the output is d(GroupNorm output): emit dyh + channel sums instead (see build())
      const Op& gn = c.h->ops[o.gnb];
      const bool film = gn.mode == GN_FILM;
      set_gn_bwd_epilogue(a, c.act(gn.x), c.ws + gn.gnp, gn.mode, film ? c.act(gn.e) : nullptr, film ? c.grad(gn.e) : nullptr,
                          reinterpret_cast<float*>(c.ws + gn.bcs), c.h->cfg.dropout, gn.op_index, c.seed_dev, c.train);
    }
    dispatch_conv(dt, o.k.dgrad, a, c.shadow(o.wC), ds);
  }
}

static GnArgs gn_args(const Ctx& c, const Op& o) {
  const Tensor& x = c.h->tensors[o.x];
  return gn_fill(c.act(o.x), c.act(o.y), o.e >= 0 ? c.act(o.e) : nullptr, c.P(o.w), c.P(o.b), c.aux(o.stats), x.n, x.h, x.w, x.c,
                 o.mode, o.rs, c.h->cfg.dropout, o.op_index, c.seed_dev, c.train);
}

// The ops a cheap forward at feature-cache level `level` runs: a walk from the output back through every op's inputs, with
// the cached tensor as a leaf.  The log-SNR embedding is kept too (the OP_EMBs read it outside the tensor list).  Also derives
// the statistics ranges the kept ops re-produce: the per-op GroupNorm statistics of the kept norms and the per-channel sums
// of the tensors a kept op writes.  The cached tensor's sums are not among them, so they survive for the norm that reads it.
static void plan_feature_cache(xunet_handle* h, int level) {
  const int nops = (int)h->ops.size(), cached = h->cache_t[level];
  std::vector<char> need(h->tensors.size(), 0);
  h->keep.assign(nops, 0);
  h->keep_fork = -1;
  for (int i = nops - 1; i >= 0; --i) {
    const Op& o = h->ops[i];
    if (!(o.kind == OP_EXTRACT || o.kind == OP_LOGSNR || (o.y >= 0 && need[o.y]))) continue;
    h->keep[i] = 1;
    for (int t : {o.x, o.r, o.e, o.cs_a, o.cs_b}) if (t >= 0 && t != cached) need[t] = 1;
    if (o.kind == OP_EMB && h->keep_fork < 0) h->keep_fork = i;
  }
  std::vector<std::pair<long long, long long>> r;
  const long long per = sizeof(float) * h->B * XU_GROUPS * 2;
  for (int i = 0; i < nops; ++i)
    if (h->keep[i] && h->ops[i].kind == OP_GN) r.push_back({h->ops[i].stats, per});
  for (const Tensor& t : h->tensors)
    if (t.cstats >= 0 && h->keep[t.producer])
      r.push_back({t.cstats, (sizeof(float) * 2 * (long long)h->B * t.c + 255) / 256 * 256});
  std::sort(r.begin(), r.end());
  h->keep_clear.clear();
  for (const auto& x : r) {
    auto& last = h->keep_clear;
    if (!last.empty() && last.back().first + last.back().second == x.first) last.back().second += x.second;
    else last.push_back(x);
  }
  h->keep_level = level;
}

static int forward_impl(Ctx& c, float* eps_out) {
  xunet_handle* h = c.h;
  const int dt = h->dtype, B = h->B, S = h->S, E = h->cfg.emb_ch;
  const bool reuse = h->static_cond && h->forward_done_train != 0;
  if (!reuse) for (const WeightPrepTable& t : h->prep) launch_weight_prep(t, c.params, c.ws, c.s);
  const bool cheap = h->cache_level > 0;
  if (cheap) {
    for (const auto& r : h->keep_clear) cudaMemsetAsync(c.ws + r.first, 0, (size_t)r.second, c.s);
  } else {
    if (h->stats_bytes) cudaMemsetAsync(c.ws + h->a_stats, 0, (size_t)h->stats_bytes, c.s);
    if (h->cstats_bytes) cudaMemsetAsync(c.ws + h->a_cstats, 0, (size_t)h->cstats_bytes, c.s);
  }
  const int fork_op = cheap ? h->keep_fork : h->last_emb_op;
  cudaStream_t side = h->film_ops.empty() ? nullptr : ensure_side(h);
  for (int oi = 0; oi < (int)h->ops.size(); ++oi) {
    const Op& o = h->ops[oi];
    if (cheap && !h->keep[oi]) continue;
    switch (o.kind) {
      case OP_LOGSNR:
        launch_logsnr_emb(c.batch->logsnr, c.P(o.p0), c.P(o.p1), c.P(o.p2), c.P(o.p3), c.aux(h->a_pe), c.aux(h->a_h1),
                          c.aux(h->a_lemb), B, E, c.s);
        break;
      case OP_POSE:
        if (reuse) break;
        launch_pose_emb(dt, c.batch->R1, c.batch->t1, c.batch->R2, c.batch->t2, c.batch->K, c.batch->cond_mask, c.P(o.p0),
                        c.P(o.p1), c.P(o.p2), c.aux(h->a_kinv), c.act(o.y), B, S, h->cfg.ray_convention, c.batch->rays, c.s);
        break;
      case OP_PACK: launch_pack_input(dt, c.batch->x, c.batch->z, c.act(o.y), B, S, c.s); break;
      case OP_CONV:
        if (reuse && o.x == h->t_pose) break;   // pose-embedding convs depend on the poses only
        if (o.film && side != nullptr) break;   // already running on the side stream (forked after the last OP_EMB)
        run_conv_fwd(c, o);
        break;
      case OP_EMB: {
        const Tensor& x = h->tensors[o.x];
        launch_emb_fwd(dt, c.aux(h->a_lemb), c.act(o.x), c.act(o.y), x.n, x.h * x.w, x.c, c.s);
        if (oi == fork_op && side != nullptr) {
          // every FiLM Dense depends only on the embeddings: run the whole branch concurrently with the trunk
          cudaEventRecord(h->ev_fork, c.s);
          cudaStreamWaitEvent(side, h->ev_fork, 0);
          Ctx cs = c;
          cs.s = side;
          for (size_t k = 0; k < h->film_ops.size(); ++k) {
            if (cheap && !h->keep[h->film_ops[k]]) continue;   // its norm is skipped too, so nothing waits on its event
            run_conv_fwd(cs, h->ops[h->film_ops[k]]);
            cudaEventRecord(h->ev_film[k], side);
          }
        }
        break;
      }
      case OP_GN: {
        if (o.film_idx >= 0 && side != nullptr) cudaStreamWaitEvent(c.s, h->ev_film[o.film_idx], 0);
        GnArgs a = gn_args(c, o);
        a.cstatsA = reinterpret_cast<const float*>(c.ws + h->tensors[o.cs_a].cstats);
        a.csA = h->tensors[o.cs_a].c;
        a.cstatsB = o.cs_b >= 0 ? reinterpret_cast<const float*>(c.ws + h->tensors[o.cs_b].cstats) : nullptr;
        if (o.gnb >= 0 && h->training) a.params_out = reinterpret_cast<float*>(c.ws + o.gnp);
        launch_gn_apply(dt, a, c.s);
        break;
      }
      case OP_RESAMPLE: {
        const Tensor& x = h->tensors[o.x];
        const ResampleArgs r = resample_fwd_args(o.rs);
        launch_resample(dt, c.act(o.x), c.act(o.y), x.n, x.h, x.w, x.c, r.pool, r.scale, 0, c.s);
        break;
      }
      case OP_CONCAT: {
        const Tensor& a = h->tensors[o.x];
        const Tensor& b = h->tensors[o.r];
        const long long npix = (long long)a.n * a.h * a.w;
        for (int k = 0; k < 2; ++k) {
          const ChannelCopy cc = concat_copy(a.c, b.c, false, k == 1);
          launch_copy_channels(dt, c.act(k ? o.r : o.x), c.act(o.y), npix, cc.Cs, cc.Cd, cc.src_off, cc.dst_off, cc.Cc, 0, c.s);
        }
        break;
      }
      case OP_ATTN: {
        const Tensor& y = h->tensors[o.y];
        AttnArgs a = attn_args(c.act(o.x), c.act(o.r), c.act(o.y), c.aux(o.lse), y.n, y.h * y.w, y.c, o.heads, o.cross);
        a.cstats = (y.cstats >= 0 && y.cs_fused) ? reinterpret_cast<float*>(c.ws + y.cstats) : nullptr;
        dispatch_attn_fwd(dt, o.impl, a, c.s);
        if (y.cstats >= 0 && !y.cs_fused)
          launch_gn_cstats(dt, c.act(o.y), reinterpret_cast<float*>(c.ws + y.cstats), y.n, y.h, y.w, y.c, c.s);
        break;
      }
      case OP_EXTRACT:
        launch_extract_frame1(dt, c.act(o.x), c.aux(h->a_eps), B, S, c.s);
        if (eps_out != nullptr)
          cudaMemcpyAsync(eps_out, c.aux(h->a_eps), sizeof(float) * (size_t)B * S * S * 3, cudaMemcpyDeviceToDevice, c.s);
        break;
    }
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return xu_fail("forward: CUDA error: %s", cudaGetErrorString(e));
  if (xu_kernel_error()[0]) return xu_fail("forward: %s", xu_kernel_error());
  return 0;
}

// ray (and camera) gradient of the backward's OP_POSE step: every grad(pose_emb_l) is final, on this stream.  bf16: the
// levels whose forward runs on the tensor cores (and so has a bf16 weight shadow) run the wgmma kernel one by one, level 0
// storing d_rays and the rest adding; the others (small images, forward on SIMT cores too) follow in one SIMT launch.  fp32:
// one SIMT launch over all levels.
static void run_pose_grad(const Ctx& c) {
  const xunet_handle* h = c.h;
  const xunet_batch* bt = c.batch;
  PoseGradArgs a{bt->R1, bt->t1, bt->R2, bt->t2, bt->K, c.aux(h->a_kinv), bt->rays, bt->cond_mask, c.cam->d_rays,
                 h->B, h->S, h->cfg.emb_ch, h->cfg.ray_convention};
  PoseLevels simt{};
  int stored = 0;
  for (const Op& o : h->ops) {
    if (o.kind != OP_CONV || o.x != h->t_pose) continue;
    const PoseLevel L{c.grad(o.y), c.P(o.w), o.alpha * c.gscale(o.y), o.cs.Ho, o.cs.stride, o.cs.pad_h};
    if (h->dtype == XU_BF16 && o.k.fwd == CONV_TC && pose_grad_tc_supported(L.So, a.E)) {
      launch_pose_grad_tc(a, L, c.shadow(o.wT), stored, c.s);
      stored = 1;
    } else {
      simt.l[simt.n++] = L;
    }
  }
  if (simt.n > 0) launch_pose_grad_simt(h->dtype, a, simt, stored, c.s);
  const xunet_input_grads* g = c.cam;
  if (g->dR1 || g->dt1 || g->dR2 || g->dt2 || g->dK) launch_camera_grad(a, g->dR1, g->dt1, g->dR2, g->dt2, g->dK, c.s);
}

static int backward_impl(Ctx& c, const float* noise, float* loss_out) {
  xunet_handle* h = c.h;
  const int dt = h->dtype, B = h->B, S = h->S, E = h->cfg.emb_ch;
  c.side = ensure_side(h);
  bool emb_joined = false;
  // every parameter-gradient writer below adds its leaf's gradient exactly once (an fp64 fold or a += per element), except the
  // log-SNR Dense and pos_emb kernels, which store unless told to add: zeroing the buffer first makes the backward overwrite it
  if (!c.acc_grads) cudaMemsetAsync(c.grads, 0, sizeof(float) * (size_t)h->nparams, c.s);
  cudaMemsetAsync(c.aux(h->a_dlemb), 0, sizeof(float) * B * E, c.s);
  if (h->bstats_bytes) cudaMemsetAsync(c.ws + h->a_bstats, 0, (size_t)h->bstats_bytes, c.s);
  if (h->bcs_bytes) cudaMemsetAsync(c.ws + h->a_bcs, 0, (size_t)h->bcs_bytes, c.s);
  size_t bp = 0;
  long long bucket_end = h->nparams;
  auto emit_bucket = [&](long long off) {
    if (h->bucket_fn == nullptr || off >= bucket_end) return;
    if (c.side != nullptr) {   // weight gradients of the finished blocks run on the side stream: order them before the hand-over
      cudaEventRecord(h->ev_join, c.side);
      cudaStreamWaitEvent(c.s, h->ev_join, 0);
    }
    h->bucket_fn(h->bucket_user, off, bucket_end - off);
    bucket_end = off;
  };
  for (int i = (int)h->ops.size() - 1; i >= 0; --i) {
    const Op& o = h->ops[i];
    switch (o.kind) {
      case OP_EXTRACT:
        if (c.d_eps) launch_vjp_seed(dt, c.d_eps, c.grad(o.x), B, S, c.s);
        else if (c.mse) launch_loss_mse(dt, c.aux(h->a_eps), noise, c.loss_weight, loss_out, c.grad(o.x), B, S, c.s);
        else launch_loss(dt, c.aux(h->a_eps), noise, c.aux(h->a_sumsq), loss_out, c.grad(o.x), B, S, c.s);
        break;
      case OP_CONV: run_conv_bwd(c, o); break;
      case OP_GN: {
        GnArgs a = gn_args(c, o);
        a.dy = c.grad(o.y);
        a.y = c.grad(o.x);  // dx
        a.de = o.e >= 0 ? c.grad(o.e) : nullptr;
        a.dgamma = c.G(o.w); a.dbeta = c.G(o.b);
        a.bstats = c.aux(o.bstats);
        a.accumulate = o.acc_x; a.de_accumulate = o.acc_e;
        a.extra = o.extra_src >= 0 ? c.grad(o.extra_src) : nullptr;
        a.extra_alpha = o.extra_alpha;
        if (o.gnb >= 0) {   // dy already holds dyh, the channel sums are in bcs (and, FiLM norm, de has been written)
          a.bcs = reinterpret_cast<const float*>(c.ws + o.bcs);
          launch_gn_bwd_apply_pre(dt, a, c.s);
          break;
        }
        launch_gn_bwd_reduce(dt, a, c.s);
        launch_gn_bwd_apply(dt, a, c.s);
        break;
      }
      case OP_EMB: {
        if (c.side != nullptr && !emb_joined) {   // grad(semb) was produced on the side stream
          cudaEventRecord(h->ev_join, c.side);
          cudaStreamWaitEvent(c.s, h->ev_join, 0);
          emb_joined = true;
        }
        const Tensor& x = h->tensors[o.x];
        launch_emb_bwd(dt, c.aux(h->a_lemb), c.act(o.x), c.grad(o.y), x.need_grad ? c.grad(o.x) : nullptr, c.aux(h->a_dlemb),
                       x.n, x.h * x.w, x.c, x.need_grad ? 1 : 0, c.s);
        break;
      }
      case OP_RESAMPLE: {
        const Tensor& y = h->tensors[o.y];
        const ResampleArgs r = resample_bwd_args(o.rs, c.gscale(o.y));
        launch_resample(dt, c.grad(o.y), c.grad(o.x), y.n, y.h, y.w, y.c, r.pool, r.scale, o.acc_x, c.s);
        break;
      }
      case OP_CONCAT: {
        const Tensor& a = h->tensors[o.x];
        const Tensor& b = h->tensors[o.r];
        const long long npix = (long long)a.n * a.h * a.w;
        for (int k = 0; k < 2; ++k) {
          if (!(k ? b : a).need_grad) continue;
          const ChannelCopy cc = concat_copy(a.c, b.c, true, k == 1);
          launch_copy_channels(dt, c.grad(o.y), c.grad(k ? o.r : o.x), npix, cc.Cs, cc.Cd, cc.src_off, cc.dst_off, cc.Cc,
                               k ? o.acc_r : o.acc_x, c.s);
        }
        break;
      }
      case OP_ATTN: {
        const Tensor& y = h->tensors[o.y];
        if (!o.fuse_res) launch_scale_add(dt, c.grad(o.y), c.grad(o.r), y.numel(), XU_RSQRT2, o.acc_r, c.s);
        AttnArgs a = attn_args(c.act(o.x), c.act(o.r), c.act(o.y), c.aux(o.lse), y.n, y.h * y.w, y.c, o.heads, o.cross);
        a.dout = c.grad(o.y); a.dscratch = c.aux(o.dscr); a.dqkv = c.grad(o.x);
        dispatch_attn_bwd(dt, o.impl, a, c.s);
        break;
      }
      case OP_PACK:
        if (c.dx != nullptr || c.dz != nullptr) {
          // adjoint of the pack: the data gradient of the conv that reads the packed views, split back into dx / dz.  Every
          // writer of that conv's output gradient ran on this stream, and its weight gradient only reads it on the side stream.
          int k = i + 1;
          while (h->ops[k].kind != OP_CONV || h->ops[k].x != o.y) ++k;
          const Op& cv = h->ops[k];
          launch_conv_cin3_dgrad_unpack(dt, c.grad(cv.y), c.P(cv.w), c.dx, c.dz, B, S, h->tensors[cv.y].c,
                                        cv.alpha * c.gscale(cv.y), c.s);
        }
        break;
      case OP_POSE:
        if (h->tensors[o.y].need_grad)
          launch_pose_emb_bwd(dt, c.grad(o.y), c.G(o.p0), c.G(o.p1), c.G(o.p2), B, S, c.acc_grads, c.s);
        if (c.cam != nullptr && c.cam->d_rays != nullptr) run_pose_grad(c);
        break;
      case OP_LOGSNR:
        launch_logsnr_emb_bwd(c.aux(h->a_dlemb), c.P(o.p2), c.aux(h->a_pe), c.aux(h->a_h1), c.aux(h->a_dh1), c.G(o.p0),
                              c.G(o.p1), c.G(o.p2), c.G(o.p3), B, E, c.acc_grads, c.s);
        break;
      default: break;
    }
    if (h->bucket_fn != nullptr && bp < h->bucket_pts.size() && h->bucket_pts[bp].op_begin == i) emit_bucket(h->bucket_pts[bp++].leaf_begin);
  }
  if (c.side != nullptr) {   // join
    cudaEventRecord(h->ev_join, c.side);
    cudaStreamWaitEvent(c.s, h->ev_join, 0);
  }
  if (h->bucket_fn != nullptr && bucket_end > 0) {
    h->bucket_fn(h->bucket_user, 0, bucket_end);
    bucket_end = 0;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return xu_fail("backward: CUDA error: %s", cudaGetErrorString(e));
  if (xu_kernel_error()[0]) return xu_fail("backward: %s", xu_kernel_error());
  return 0;
}

}  // namespace

// ======================================================================================================
// C-ABI
// ======================================================================================================
extern "C" int xunet_create(const xunet_config* cfg, int batch, int side, int dtype, int training, xunet_handle** out) {
  if (!cfg || !out) return xu_fail("xunet_create: null argument");
  if (dtype != XUNET_DTYPE_F32 && dtype != XUNET_DTYPE_BF16) return xu_fail("xunet_create: bad dtype %d", dtype);
  if (batch < 1 || side < 1) return xu_fail("xunet_create: bad batch/side");
  if (cfg->n_levels < 1 || cfg->n_levels > XUNET_MAX_LEVELS) return xu_fail("xunet_create: n_levels out of range");
  if (cfg->n_attn_resolutions < 0 || cfg->n_attn_resolutions > XUNET_MAX_LEVELS) return xu_fail("xunet_create: bad attn_resolutions");
  if (cfg->ch % 32 != 0) return xu_fail("xunet_create: ch must be a multiple of 32 (GroupNorm(32), model/xunet.py:51)");
  if (cfg->emb_ch % 4 != 0 || cfg->emb_ch < 4) return xu_fail("xunet_create: emb_ch must be a multiple of 4");
  if (side % (1 << (cfg->n_levels - 1)) != 0) return xu_fail("xunet_create: side must be divisible by 2^(levels-1)");
  if (cfg->dropout < 0.f || cfg->dropout >= 1.f) return xu_fail("xunet_create: dropout must be in [0,1)");
  for (int i = 0; i < cfg->n_levels; ++i) {
    int C = cfg->ch * cfg->ch_mult[i];
    if (cfg->ch_mult[i] < 1) return xu_fail("xunet_create: ch_mult must be >= 1");
    int res = side >> i;
    bool at = false;
    for (int k = 0; k < cfg->n_attn_resolutions; ++k) at |= cfg->attn_resolutions[k] == res;
    if (at) {
      if (C % cfg->attn_heads != 0) return xu_fail("xunet_create: channels not divisible by attn_heads");
      int hd = C / cfg->attn_heads;
      if (hd != 16 && hd != 32 && hd != 64 && hd != 128) return xu_fail("xunet_create: head_dim %d unsupported (16/32/64/128)", hd);
    }
  }
  xunet_handle* h = new xunet_handle();
  h->cfg = *cfg;
  h->B = batch; h->S = side; h->dtype = dtype; h->training = training ? 1 : 0; h->N = 2 * batch;
  h->esize = dtype == XUNET_DTYPE_F32 ? 4 : 2;
  Builder b(*h);
  if (b.build() != 0) { delete h; return 1; }
  *out = h;
  return 0;
}

extern "C" void xunet_destroy(xunet_handle* h) {
  if (!h) return;
  xu_det_destroy(h->det);
  destroy_side(h);
  delete h;
}
extern "C" long long xunet_param_count(const xunet_handle* h) { return h->nparams; }
extern "C" int xunet_param_leaves(const xunet_handle* h) { return (int)h->leaves.size(); }
extern "C" int xunet_param_leaf(const xunet_handle* h, int i, const char** name, int* ndim, long long shape[5],
                                long long* offset) {
  if (i < 0 || i >= (int)h->leaves.size()) return xu_fail("xunet_param_leaf: index out of range");
  const Leaf& l = h->leaves[i];
  *name = l.name.c_str();
  *ndim = l.ndim;
  for (int k = 0; k < 5; ++k) shape[k] = l.shape[k];
  *offset = l.off;
  return 0;
}
extern "C" long long xunet_workspace_bytes(const xunet_handle* h) { return h->ws_bytes; }
extern "C" int xunet_tap_count(const xunet_handle* h) { return (int)h->taps.size() + 1; }
extern "C" int xunet_tap(const xunet_handle* h, int i, const char** name, int dims[4], long long* byte_offset, int* is_f32,
                         long long* grad_byte_offset) {
  if (i < 0 || i > (int)h->taps.size()) return xu_fail("xunet_tap: index out of range");
  if (i == (int)h->taps.size()) {  // the fp32 log-SNR embedding lives in aux storage
    *name = "logsnr_emb";
    dims[0] = h->B; dims[1] = 1; dims[2] = 1; dims[3] = h->cfg.emb_ch;
    *byte_offset = h->a_lemb; *is_f32 = 1; *grad_byte_offset = h->training ? h->a_dlemb : -1;
    return 0;
  }
  const Tensor& t = h->tensors[h->taps[i]];
  *name = t.tap.c_str();
  dims[0] = t.n; dims[1] = t.h; dims[2] = t.w; dims[3] = t.c;
  *byte_offset = t.off; *is_f32 = t.f32 ? 1 : 0; *grad_byte_offset = t.goff;
  return 0;
}

static_assert(XUNET_KERNEL_SIMT == CONV_SIMT && XUNET_KERNEL_TC == CONV_TC && XUNET_KERNEL_CIN3 == CONV_CIN3 &&
              XUNET_KERNEL_COUT3 == CONV_COUT3, "conv kernels");

static bool is_launch(const Op& o) { return o.kind == OP_CONV || o.kind == OP_ATTN; }

extern "C" int xunet_plan_launch_count(const xunet_handle* h) {
  int n = 0;
  for (const Op& o : h->ops) n += is_launch(o);
  return n;
}

// every field comes from the op and the helpers the launch code uses (run_conv_fwd / run_conv_bwd, forward_impl's OP_ATTN)
extern "C" int xunet_plan_launch(const xunet_handle* h, int i, xunet_launch_info* out) {
  if (!h || !out) return xu_fail("xunet_plan_launch: null argument");
  int k = -1;
  for (size_t j = 0; j < h->ops.size() && i >= 0; ++j)
    if (is_launch(h->ops[j]) && i-- == 0) k = (int)j;
  if (k < 0) return xu_fail("xunet_plan_launch: index out of range");
  const Op& o = h->ops[k];
  const Tensor& x = h->tensors[o.x];
  const Tensor& y = h->tensors[o.y];
  xunet_launch_info r;
  memset(&r, 0, sizeof(r));
  r.leaf = -1;
  r.fwd = r.dgrad = r.wgrad = XUNET_KERNEL_NONE;
  r.gn_mode = -1;
  r.emits_stats = y.cstats >= 0 && y.cs_fused;
  if (o.kind == OP_ATTN) {
    r.kind = XUNET_LAUNCH_ATTN;
    r.N = y.n; r.L = y.h * y.w; r.C = y.c; r.heads = o.heads; r.cross = o.cross; r.impl = o.impl;
    *out = r;
    return 0;
  }
  r.kind = XUNET_LAUNCH_CONV;
  for (size_t l = 0; l < h->leaves.size(); ++l)
    if (h->leaves[l].off == o.w) r.leaf = (int)l;
  const ConvShape& s = o.cs;
  r.N = s.N; r.Hi = s.Hi; r.Wi = s.Wi; r.Ci = s.Ci; r.Ho = s.Ho; r.Wo = s.Wo; r.Co = s.Co;
  r.ksize = s.ks; r.stride = s.stride; r.nseg = s.nseg;
  r.residual = o.r >= 0;
  r.alpha = o.alpha;
  r.fwd = o.k.fwd;
  r.bwd_alpha = o.alpha * y.gscale;
  if (h->training) {
    r.wgrad = o.k.wgrad;
    if (x.need_grad) {
      r.dgrad = o.k.dgrad;
      r.accumulate = o.acc_x;
      if (o.gnb >= 0) r.gn_mode = h->ops[o.gnb].mode;
    }
  }
  *out = r;
  return 0;
}

static int plan_op_kind(const Op& o) {
  switch (o.kind) {
    case OP_LOGSNR: return XUNET_PLAN_OP_LOGSNR;
    case OP_POSE: return XUNET_PLAN_OP_POSE;
    case OP_EMB: return XUNET_PLAN_OP_EMB;
    case OP_RESAMPLE: return XUNET_PLAN_OP_RESAMPLE;
    case OP_CONCAT: return XUNET_PLAN_OP_CONCAT;
    case OP_ATTN: return XUNET_PLAN_OP_ATTN_RESIDUAL;
    case OP_EXTRACT: return XUNET_PLAN_OP_LOSS;
    default: return -1;
  }
}

extern "C" int xunet_plan_op_count(const xunet_handle* h) {
  int n = 0;
  for (const Op& o : h->ops) n += plan_op_kind(o) >= 0;
  return n;
}

// every field comes from the op and the helpers forward_impl / backward_impl launch it with
extern "C" int xunet_plan_op(const xunet_handle* h, int i, xunet_op_info* out) {
  if (!h || !out) return xu_fail("xunet_plan_op: null argument");
  int k = -1;
  for (size_t j = 0; j < h->ops.size() && i >= 0; ++j)
    if (plan_op_kind(h->ops[j]) >= 0 && i-- == 0) k = (int)j;
  if (k < 0) return xu_fail("xunet_plan_op: index out of range");
  const Op& o = h->ops[k];
  const bool tr = h->training != 0;
  xunet_op_info r;
  memset(&r, 0, sizeof(r));
  r.kind = plan_op_kind(o);
  r.B = h->B; r.S = h->S; r.E = h->cfg.emb_ch;
  r.N = h->N; r.H = h->S; r.W = h->S;
  r.fwd_scale = r.gscale = r.bwd_scale = r.alpha = 1.f;
  r.need_grad = tr;
  switch (o.kind) {
    case OP_LOGSNR: r.C = h->cfg.emb_ch; break;
    case OP_POSE: {
      const Tensor& y = h->tensors[o.y];
      r.C = y.c;
      r.need_grad = y.need_grad;
      r.pos_emb = o.p0 >= 0; r.ref_pose_emb = o.p1 >= 0; r.ray_convention = h->cfg.ray_convention;
      break;
    }
    case OP_EMB: {
      const Tensor& x = h->tensors[o.x];
      r.N = x.n; r.H = x.h; r.W = x.w; r.C = x.c;
      r.acc_x = o.acc_x;
      r.write_dpe = tr && x.need_grad;
      break;
    }
    case OP_RESAMPLE: {
      const Tensor& x = h->tensors[o.x];
      const Tensor& y = h->tensors[o.y];
      r.N = x.n; r.H = x.h; r.W = x.w; r.C = x.c;
      r.rs = o.rs;
      const ResampleArgs f = resample_fwd_args(o.rs), b = resample_bwd_args(o.rs, y.gscale);
      r.fwd_pool = f.pool; r.fwd_scale = f.scale;
      r.gscale = y.gscale;
      r.bwd_pool = b.pool; r.bwd_scale = b.scale;
      r.acc_x = o.acc_x;
      break;
    }
    case OP_CONCAT: {
      const Tensor& a = h->tensors[o.x];
      const Tensor& b = h->tensors[o.r];
      r.N = a.n; r.H = a.h; r.W = a.w; r.C = a.c; r.C2 = b.c;
      for (int q = 0; q < 4; ++q) {
        const ChannelCopy cc = concat_copy(a.c, b.c, q >= 2, q & 1);
        const int v[5] = {cc.Cs, cc.Cd, cc.src_off, cc.dst_off, cc.Cc};
        memcpy(r.copies[q], v, sizeof(v));
      }
      r.acc_x = o.acc_x; r.acc_r = o.acc_r;
      r.need_grad = tr && a.need_grad;
      r.need_grad_r = tr && b.need_grad;
      break;
    }
    case OP_ATTN: {
      const Tensor& y = h->tensors[o.y];
      r.N = y.n; r.H = y.h; r.W = y.w; r.C = y.c;
      r.alpha = XU_RSQRT2;
      r.acc_r = o.acc_r;
      r.need_grad = tr && !o.fuse_res;   // else the residual gradient is added inside a GroupNorm backward
      break;
    }
    case OP_EXTRACT: r.C = 3; break;
  }
  *out = r;
  return 0;
}

extern "C" int xunet_forward(xunet_handle* h, const float* params, const xunet_batch* batch, int train,
                             const unsigned long long* seed_dev, void* workspace, float* eps_out, void* stream) {
  if (!h || !params || !batch || !workspace) return xu_fail("xunet_forward: null argument");
  if (train && h->cfg.dropout > 0.f && !seed_dev) return xu_fail("xunet_forward: train=1 with dropout needs seed_dev");
  if (h->cache_level > 0 && (h->cache_from == 0 || h->cache_level < h->cache_from))
    return xu_fail("xunet_forward: a cheap forward at feature-cache level %d needs a full forward first (none has completed since "
                   "the handle was created, or a cheap forward at a deeper level has recomputed the cached tensor since)",
                   h->cache_level);
  xu_set_kernel_error("");
  Ctx c{h, params, nullptr, (char*)workspace, batch, seed_dev, train ? 1 : 0, (cudaStream_t)stream};
  XuDetBind bind(h->det);
  int rc = forward_impl(c, eps_out);
  h->forward_done_train = (rc == 0) ? (train ? 1 : 2) : 0;
  // a cheap forward at L recomputes the cached tensors of every level below L
  h->cache_from = rc != 0 ? 0 : h->cache_level == 0 ? 1 : std::max(h->cache_from, h->cache_level);
  return rc;
}

extern "C" int xunet_set_feature_cache(xunet_handle* h, int level) {
  if (!h) return xu_fail("xunet_set_feature_cache: null handle");
  if (h->training)
    return xu_fail("xunet_set_feature_cache: the handle was created with training=1, and a backward needs every activation of a "
                   "full forward");
  if (level < 0 || level > h->cfg.n_levels - 1)
    return xu_fail("xunet_set_feature_cache: level %d outside [0, %d] for a %d-level config", level, h->cfg.n_levels - 1,
                   h->cfg.n_levels);
  if (level > 0 && level != h->keep_level) plan_feature_cache(h, level);
  h->cache_level = level;
  return 0;
}

extern "C" int xunet_set_static_conditioning(xunet_handle* h, int on) {
  if (!h) return xu_fail("xunet_set_static_conditioning: null handle");
  h->static_cond = on ? 1 : 0;
  return 0;
}

extern "C" int xunet_set_grad_bucket_callback(xunet_handle* h, xunet_bucket_fn fn, void* user, long long min_bucket_bytes) {
  if (!h) return xu_fail("xunet_set_grad_bucket_callback: null handle");
  h->bucket_fn = fn;
  h->bucket_user = user;
  h->bucket_pts.clear();
  if (fn == nullptr) return 0;
  const long long min_elems = min_bucket_bytes > 0 ? (min_bucket_bytes + 3) / 4 : 0;
  long long end = h->nparams;
  for (int k = (int)h->blocks.size() - 1; k >= 0; --k) {
    const xunet_handle::Block& b = h->blocks[k];
    if (b.leaf_begin >= end) continue;                       // a block without parameters of its own
    if (end - b.leaf_begin >= min_elems && b.leaf_begin > 0) { h->bucket_pts.push_back(b); end = b.leaf_begin; }
  }
  return 0;
}

extern "C" int xunet_grad_bucket_count(const xunet_handle* h) { return h ? (int)h->bucket_pts.size() + 1 : 0; }

// The preamble of every backward entry (fn: its name in the messages): null arguments, a training handle and a forward to
// differentiate, then backward_impl in the engine's fp64 scratch.  in == nullptr: the loss backward, seeded from noise and
// writing loss_out (the mean-squared loss with mse, weighted by loss_weight); else the VJP of d_eps, with the input and
// camera gradients `in` asks for.
static int backward_entry(const char* fn, xunet_handle* h, const float* params, const xunet_batch* batch, const float* noise,
                          const float* d_eps, const unsigned long long* seed_dev, void* workspace, float* grads, float* loss_out,
                          int accumulate, int mse, const float* loss_weight, const xunet_input_grads* in, void* stream) {
  if (!h || !params || !batch || !workspace || !grads || (in ? !d_eps : (!noise || !loss_out)))
    return xu_fail("%s: null argument", fn);
  if (!h->training) return xu_fail("%s: handle was created with training=0", fn);
  if (!h->forward_done_train) return xu_fail("%s: call xunet_forward first", fn);
  const bool cams = in && (in->dR1 || in->dt1 || in->dR2 || in->dt2 || in->dK);
  if (cams && !in->d_rays) return xu_fail("%s: camera gradients need d_rays", fn);
  if (cams && batch->rays) return xu_fail("%s: camera gradients need generated rays (batch->rays == NULL)", fn);
  xu_set_kernel_error("");
  Ctx c{h, params, grads, (char*)workspace, batch, seed_dev, h->forward_done_train == 1 ? 1 : 0, (cudaStream_t)stream};
  c.acc_grads = accumulate ? 1 : 0;
  c.mse = mse;
  c.loss_weight = loss_weight;
  c.d_eps = d_eps;
  if (in) {
    c.dx = in->dx;
    c.dz = in->dz;
    c.cam = in->d_rays ? in : nullptr;
  }
  XuDetBind bind(h->det);
  return backward_impl(c, noise, loss_out);
}

extern "C" int xunet_backward(xunet_handle* h, const float* params, const xunet_batch* batch, const float* noise,
                              const unsigned long long* seed_dev, void* workspace, float* grads, float* loss_out,
                              void* stream) {
  return backward_entry("xunet_backward", h, params, batch, noise, nullptr, seed_dev, workspace, grads, loss_out, 0, 0, nullptr,
                        nullptr, stream);
}

extern "C" int xunet_backward_accumulate(xunet_handle* h, const float* params, const xunet_batch* batch, const float* noise,
                                         const unsigned long long* seed_dev, void* workspace, float* grads, float* loss_out,
                                         void* stream) {
  return backward_entry("xunet_backward_accumulate", h, params, batch, noise, nullptr, seed_dev, workspace, grads, loss_out, 1, 0,
                        nullptr, nullptr, stream);
}

extern "C" int xunet_backward_mse(xunet_handle* h, const float* params, const xunet_batch* batch, const float* noise,
                                  const float* loss_weight, const unsigned long long* seed_dev, void* workspace, float* grads,
                                  float* loss_out, int accumulate, void* stream) {
  return backward_entry("xunet_backward_mse", h, params, batch, noise, nullptr, seed_dev, workspace, grads, loss_out, accumulate,
                        1, loss_weight, nullptr, stream);
}

extern "C" int xunet_backward_vjp(xunet_handle* h, const float* params, const xunet_batch* batch, const float* d_eps,
                                  const unsigned long long* seed_dev, void* workspace, float* grads, int accumulate, float* dx,
                                  float* dz, void* stream) {
  xunet_input_grads in{};
  in.dx = dx;
  in.dz = dz;
  return backward_entry("xunet_backward_vjp", h, params, batch, nullptr, d_eps, seed_dev, workspace, grads, nullptr, accumulate,
                        0, nullptr, &in, stream);
}

extern "C" int xunet_backward_vjp_inputs(xunet_handle* h, const float* params, const xunet_batch* batch, const float* d_eps,
                                         const unsigned long long* seed_dev, void* workspace, float* grads, int accumulate,
                                         const xunet_input_grads* out, void* stream) {
  const xunet_input_grads none{};
  return backward_entry("xunet_backward_vjp_inputs", h, params, batch, nullptr, d_eps, seed_dev, workspace, grads, nullptr,
                        accumulate, 0, nullptr, out ? out : &none, stream);
}

static int count_kernel_nodes(cudaGraph_t g) {
  size_t n = 0;
  cudaGraphGetNodes(g, nullptr, &n);
  std::vector<cudaGraphNode_t> nodes(n);
  if (n) cudaGraphGetNodes(g, nodes.data(), &n);
  int k = 0;
  for (size_t i = 0; i < n; ++i) {
    cudaGraphNodeType t;
    if (cudaGraphNodeGetType(nodes[i], &t) == cudaSuccess && t == cudaGraphNodeTypeKernel) ++k;
  }
  return k;
}

extern "C" int xunet_count_kernels(xunet_handle* h, const float* params, const xunet_batch* batch, const float* noise,
                                   const unsigned long long* seed_dev, void* workspace, float* grads, float* loss_out,
                                   int* n_forward, int* n_backward) {
  if (!h || !params || !batch || !workspace || !n_forward) return xu_fail("xunet_count_kernels: null argument");
  cudaStream_t s;
  if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) return xu_fail("count_kernels: stream");
  xu_set_kernel_error("");
  int rc = 0;
  XuDetBind bind(h->det);
  const xunet_bucket_fn saved_fn = h->bucket_fn;   // nothing executes here: the data-parallel hook must not fire
  h->bucket_fn = nullptr;
  for (int pass = 0; pass < 2 && rc == 0; ++pass) {
    if (pass == 1 && (!n_backward || !h->training || !noise || !grads || !loss_out)) break;
    cudaGraph_t g = nullptr;
    if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { rc = xu_fail("count_kernels: begin capture"); break; }
    Ctx c{h, params, grads, (char*)workspace, batch, seed_dev, h->training ? 1 : 0, s};
    int r = pass == 0 ? forward_impl(c, nullptr) : backward_impl(c, noise, loss_out);
    cudaError_t e = cudaStreamEndCapture(s, &g);
    if (r != 0 || e != cudaSuccess || !g) { rc = r ? r : xu_fail("count_kernels: end capture: %s", cudaGetErrorString(e)); if (g) cudaGraphDestroy(g); break; }
    (pass == 0 ? *n_forward : *n_backward) = count_kernel_nodes(g);
    cudaGraphDestroy(g);
  }
  cudaStreamDestroy(s);
  h->bucket_fn = saved_fn;
  return rc;
}

// ---- operator-level entry points ----------------------------------------------------------------------
// fp64 reduction scratch of one operator-level call (kernels.h): stream-ordered allocations, released on the call's stream
struct OpScratch {
  XuDetScratch* d = xu_det_create(true);
  XuDetBind bind{d};
  ~OpScratch() { xu_det_destroy(d); }
};

static int op_done(const char* what) {
  if (int rc = xu_launched(what)) return rc;
  if (xu_kernel_error()[0]) return xu_fail("%s: %s", what, xu_kernel_error());
  return 0;
}

// the public impl of the operator-level conv entries (0 SIMT, 1 tensor cores, 2 a direct 3-channel kernel) -> the kernel to run:
// for 1 and 2, the engine's choice for the shape, which must be of that kind
static int op_conv_kernel(int impl, ConvKernel engine, const char* what, ConvKernel& k) {
  if (impl == 1 && engine != CONV_TC) return xu_fail("%s: shape not supported by the tensor-core kernel", what);
  if (impl == 2 && engine != CONV_CIN3 && engine != CONV_COUT3) return xu_fail("%s: no direct 3-channel kernel takes this shape", what);
  k = impl == 1 || impl == 2 ? engine : CONV_SIMT;
  return 0;
}

// operator-level (test / micro-benchmark) path: the bf16 shadow of a tensor-core conv lives in a process-wide scratch buffer (the
// engine keeps its shadows in the workspace instead).  With XUNET_OP_CACHE_SHADOW=1 the cast/transposition is skipped when the
// same weight pointer and shape are used again (benchmarks time the conv kernel alone; weights must not change in between).
static int op_dispatch_conv(int dtype, ConvKernel k, const ConvShape& cs, const ConvArgs& a, cudaStream_t s, const char* what) {
  static uint8_t* scratch = nullptr;
  static size_t scratch_bytes = 0;
  static const float* last_w = nullptr;
  static long long last_key[4] = {0, 0, 0, 0};
  const long long n = (long long)cs.ks * cs.ks * cs.Ci * cs.Co;
  const long long offC = (n * 2 + 255) / 256 * 256;
  if (k == CONV_TC) {
    const size_t need = (size_t)n * 2 * 2 + 1024;
    if (need > scratch_bytes) {
      cudaDeviceSynchronize();
      if (scratch) cudaFree(scratch);
      if (cudaMalloc(&scratch, need) != cudaSuccess) { scratch = nullptr; scratch_bytes = 0; return xu_fail("%s: cudaMalloc", what); }
      scratch_bytes = need;
      last_w = nullptr;
    }
    const char* e = getenv("XUNET_OP_CACHE_SHADOW");
    const bool cache = e && e[0] == '1';
    const long long key[4] = {cs.ks * cs.ks, cs.Ci, cs.Co, cs.nseg};
    if (!(cache && last_w == a.w && memcmp(key, last_key, sizeof(key)) == 0)) {
      WeightPrepTable tab{};
      prep_entry(tab, cs, 0, 0, offC);
      launch_weight_prep(tab, a.w, scratch, s);
      last_w = a.w;
      memcpy(last_key, key, sizeof(key));
    }
  }
  dispatch_conv(dtype, k, a, k == CONV_TC ? scratch + (a.mode == 0 ? 0 : offC) : nullptr, s);
  return 0;
}

// forward of xunet_op_conv; cstats != nullptr: also add the GroupNorm input statistics of the stored output to cstats, emitted by
// the epilogue where the engine's plan lets it (conv_emits_stats), else by launch_gn_cstats after the conv
static int op_conv_fwd(int dtype, int impl, const void* x, const float* w, const float* bias, const void* res, void* y, float* cstats,
                       int N, int Hi, int Wi, int Ci, int Co, int ksize, int stride, int nseg, float alpha, cudaStream_t s,
                       const char* what) {
  if (ksize != 1 && ksize != 3) return xu_fail("%s: ksize must be 1 or 3", what);
  const ConvShape cs = conv_shape(N, Hi, Wi, Ci, Co, ksize, stride, nseg);
  ConvKernel k;
  if (op_conv_kernel(impl, conv_kernels(dtype, cs, res != nullptr).fwd, what, k)) return 1;
  ConvArgs a = conv_fwd_args(cs, x, w, bias, res, y, alpha);
  const bool fused = cstats != nullptr && conv_emits_stats(k, cs);
  if (fused) a.cstats = cstats;
  if (op_dispatch_conv(dtype, k, cs, a, s, what)) return 1;
  if (cstats != nullptr && !fused) launch_gn_cstats(dtype, y, cstats, N, cs.Ho, cs.Wo, Co, s);
  return op_done(what);
}

extern "C" int xunet_op_conv(int dtype, int impl, const void* x, const float* w, const float* bias, const void* res, void* y,
                             int N, int Hi, int Wi, int Ci, int Co, int ksize, int stride, int nseg, float alpha,
                             void* stream) {
  xu_set_kernel_error("");
  OpScratch scratch;
  return op_conv_fwd(dtype, impl, x, w, bias, res, y, nullptr, N, Hi, Wi, Ci, Co, ksize, stride, nseg, alpha, (cudaStream_t)stream,
                     "xunet_op_conv");
}

extern "C" int xunet_op_conv_dgrad(int dtype, int impl, const void* dy, const float* w, void* dx, int N, int Hi, int Wi,
                                   int Ci, int Co, int ksize, int stride, int nseg, float alpha, int accumulate,
                                   void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_conv_dgrad";
  OpScratch scratch;
  const ConvShape cs = conv_shape(N, Hi, Wi, Ci, Co, ksize, stride, nseg);
  ConvKernel k;
  if (op_conv_kernel(impl, conv_kernels(dtype, cs, false).dgrad, what, k)) return 1;
  return op_dispatch_conv(dtype, k, cs, conv_dgrad_args(cs, dy, w, dx, alpha, accumulate), (cudaStream_t)stream, what) ? 1 : op_done(what);
}

extern "C" int xunet_op_conv_wgrad(int dtype, int impl, const void* x, const void* dy, float* dw, float* dbias, int N,
                                   int Hi, int Wi, int Ci, int Co, int ksize, int stride, int nseg, float alpha,
                                   void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_conv_wgrad";
  OpScratch scratch;
  const ConvShape cs = conv_shape(N, Hi, Wi, Ci, Co, ksize, stride, nseg);
  ConvKernel k;
  if (op_conv_kernel(impl, conv_kernels(dtype, cs, false).wgrad, what, k)) return 1;
  dispatch_wgrad(dtype, k, conv_wgrad_args(cs, x, dy, dw, dbias, alpha), (cudaStream_t)stream);
  return op_done(what);
}

extern "C" int xunet_op_attention(int dtype, int impl, const void* qkv, const void* res, void* out, float* lse, int N,
                                  int L, int C, int heads, int cross, void* stream) {
  xu_set_kernel_error("");
  OpScratch scratch;
  if (impl == 1 && !attn_tc_supported(dtype, L, C, heads)) return xu_fail("xunet_op_attention: shape not supported by the tensor-core kernel");
  dispatch_attn_fwd(dtype, impl, attn_args(qkv, res, out, lse, N, L, C, heads, cross), (cudaStream_t)stream);
  return op_done("op_attention");
}

extern "C" int xunet_op_attention_bwd(int dtype, int impl, const void* qkv, const void* res, const void* out,
                                      const void* dout, const float* lse, float* dscratch, void* dqkv, int N, int L, int C,
                                      int heads, int cross, void* stream) {
  xu_set_kernel_error("");
  OpScratch scratch;
  if (impl == 1 && !attn_tc_supported(dtype, L, C, heads)) return xu_fail("xunet_op_attention_bwd: shape not supported by the tensor-core kernel");
  AttnArgs a = attn_args(qkv, res, const_cast<void*>(out), const_cast<float*>(lse), N, L, C, heads, cross);
  a.dout = dout; a.dscratch = dscratch; a.dqkv = dqkv;
  // XUNET_OP_ATTN_FOLD=1: the caller passes an all-zero dscratch and gets it back all-zero (the D rows are cleared after use)
  a.scratch_zeroed = getenv("XUNET_OP_ATTN_FOLD") != nullptr ? 1 : 0;
  dispatch_attn_bwd(dtype, impl, a, (cudaStream_t)stream);
  return op_done("op_attention_bwd");
}

// ---- operator-level entry points of the GroupNorm path ----------------------------------------------------------------
static_assert(XUNET_GN_PLAIN == GN_PLAIN && XUNET_GN_SWISH == GN_SWISH && XUNET_GN_FILM == GN_FILM, "GroupNorm modes");
static_assert(XUNET_RS_NONE == RS_NONE && XUNET_RS_DOWN == RS_DOWN && XUNET_RS_UP == RS_UP, "GroupNorm resampling");

// the checks every GroupNorm-path entry shares: GroupNorm(32) over both frames of each sample
static int gn_check_shape(const char* what, int dtype, int N, int H, int W, int C) {
  if (dtype != XUNET_DTYPE_F32 && dtype != XUNET_DTYPE_BF16) return xu_fail("%s: bad dtype %d", what, dtype);
  if (N < 2 || N % 2 != 0) return xu_fail("%s: N = %d, need an even N >= 2 (two frames per sample)", what, N);
  if (H < 1 || W < 1) return xu_fail("%s: H = %d, W = %d, need both >= 1", what, H, W);
  if (C < 32 || C % 32 != 0) return xu_fail("%s: C = %d is not a positive multiple of the 32 groups", what, C);
  return 0;
}

static int gn_check_mode(const char* what, int mode, int rs, int H, int W, float drop_rate) {
  if (mode != XUNET_GN_PLAIN && mode != XUNET_GN_SWISH && mode != XUNET_GN_FILM) return xu_fail("%s: bad mode %d", what, mode);
  if (rs != XUNET_RS_NONE && rs != XUNET_RS_DOWN && rs != XUNET_RS_UP) return xu_fail("%s: bad resample %d", what, rs);
  if (rs != XUNET_RS_NONE && mode == XUNET_GN_FILM) return xu_fail("%s: a resampling norm has no FiLM", what);
  if (rs == XUNET_RS_DOWN && (H % 2 != 0 || W % 2 != 0)) return xu_fail("%s: RS_DOWN needs even H, W (got %d x %d)", what, H, W);
  if (!(drop_rate >= 0.f && drop_rate < 1.f)) return xu_fail("%s: drop_rate %g outside [0, 1)", what, drop_rate);
  return 0;
}

extern "C" int xunet_op_conv_stats(int dtype, int impl, const void* x, const float* w, const float* bias, const void* res, void* y,
                                   float* cstats, int N, int H, int W, int Ci, int Co, int ksize, float alpha, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_conv_stats";
  if (!x || !w || !y || !cstats) return xu_fail("%s: NULL pointer argument", what);
  if (gn_check_shape(what, dtype, N, H, W, Co)) return 1;
  OpScratch scratch;
  return op_conv_fwd(dtype, impl, x, w, bias, res, y, cstats, N, H, W, Ci, Co, ksize, 1, 1, alpha, (cudaStream_t)stream, what);
}

extern "C" int xunet_op_attention_stats(int dtype, int impl, const void* qkv, const void* res, void* out, float* lse, float* cstats,
                                        int N, int L, int C, int heads, int cross, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_attention_stats";
  if (!qkv || !res || !out || !lse || !cstats) return xu_fail("%s: NULL pointer argument", what);
  if (gn_check_shape(what, dtype, N, L, 1, C)) return 1;
  if (heads < 1 || C % heads != 0) return xu_fail("%s: C = %d is not a multiple of heads = %d", what, C, heads);
  if (impl == 1 && !attn_tc_supported(dtype, L, C, heads)) return xu_fail("%s: shape not supported by the tensor-core kernel", what);
  OpScratch scratch;
  AttnArgs a = attn_args(qkv, res, out, lse, N, L, C, heads, cross);
  const bool fused = attn_emits_stats(impl);
  if (fused) a.cstats = cstats;
  dispatch_attn_fwd(dtype, impl, a, (cudaStream_t)stream);
  if (!fused) launch_gn_cstats(dtype, out, cstats, N, L, 1, C, (cudaStream_t)stream);
  return op_done(what);
}

extern "C" int xunet_op_groupnorm(int dtype, const void* x, const float* cstats_a, const float* cstats_b, int ca, const float* gamma,
                                  const float* beta, const void* e, void* y, float* stats, float* params_out, int N, int H, int W,
                                  int C, int mode, int resample, float drop_rate, int op_index,
                                  const unsigned long long* seed_dev, int train, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_groupnorm";
  if (!x || !cstats_a || !gamma || !beta || !y || !stats) return xu_fail("%s: NULL pointer argument", what);
  if (gn_check_shape(what, dtype, N, H, W, C) || gn_check_mode(what, mode, resample, H, W, drop_rate)) return 1;
  if (ca < 1 || ca > C) return xu_fail("%s: ca = %d outside [1, C = %d]", what, ca, C);
  if (ca < C && !cstats_b) return xu_fail("%s: ca = %d < C needs cstats_b", what, ca);
  if (mode == XUNET_GN_FILM && !e) return xu_fail("%s: a FiLM norm needs e", what);
  if (mode == XUNET_GN_FILM && train && drop_rate > 0.f && !seed_dev) return xu_fail("%s: dropout in training needs seed_dev", what);
  if (resample != XUNET_RS_NONE && params_out) return xu_fail("%s: a resampling norm has no fused backward (params_out)", what);
  OpScratch scratch;
  GnArgs a = gn_fill(x, y, mode == XUNET_GN_FILM ? e : nullptr, gamma, beta, stats, N, H, W, C, mode, resample, drop_rate, op_index,
                     seed_dev, train ? 1 : 0);
  a.cstatsA = cstats_a; a.csA = ca;
  a.cstatsB = ca < C ? cstats_b : nullptr;
  a.params_out = params_out;
  launch_gn_apply(dtype, a, (cudaStream_t)stream);
  return op_done(what);
}

extern "C" int xunet_op_conv_dgrad_groupnorm(int dtype, const void* dy, const float* w, const void* gn_x, const float* gn_params,
                                             int mode, const void* e, void* de, float drop_rate, int op_index,
                                             const unsigned long long* seed_dev, int train, void* dyh, float* bcs, int N, int H,
                                             int W, int C, int Co, int ksize, int nseg, float alpha, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_conv_dgrad_groupnorm";
  if (!dy || !w || !gn_x || !gn_params || !dyh || !bcs) return xu_fail("%s: NULL pointer argument", what);
  if (gn_check_shape(what, dtype, N, H, W, C) || gn_check_mode(what, mode, XUNET_RS_NONE, H, W, drop_rate)) return 1;
  if ((mode == XUNET_GN_FILM) != (e != nullptr)) return xu_fail("%s: e is given exactly for a FiLM norm", what);
  if (mode == XUNET_GN_FILM && !de) return xu_fail("%s: a FiLM norm needs de", what);
  if (mode == XUNET_GN_FILM && train && drop_rate > 0.f && !seed_dev) return xu_fail("%s: dropout in training needs seed_dev", what);
  if (ksize != 1 && ksize != 3) return xu_fail("%s: ksize must be 1 or 3", what);
  if (nseg < 1 || Co % nseg != 0) return xu_fail("%s: Co = %d is not a multiple of nseg = %d", what, Co, nseg);
  const ConvShape cs = conv_shape(N, H, W, C, Co, ksize, 1, nseg);
  const ConvKernel k = conv_kernels(dtype, cs, false).dgrad;
  if (!dgrad_fuses_gn_bwd(k, cs)) return xu_fail("%s: shape not supported by the fused tensor-core data gradient", what);
  OpScratch scratch;
  ConvArgs a = conv_dgrad_args(cs, dy, w, dyh, alpha, 0);
  set_gn_bwd_epilogue(a, gn_x, gn_params, mode, e, de, bcs, drop_rate, op_index, seed_dev, train ? 1 : 0);
  return op_dispatch_conv(dtype, k, cs, a, (cudaStream_t)stream, what) ? 1 : op_done(what);
}

extern "C" int xunet_op_groupnorm_bwd(int dtype, const void* x, const void* e, const void* dy, void* dx, void* de, const float* gamma,
                                      const float* beta, float* dgamma, float* dbeta, const float* stats, float* bstats,
                                      const float* bcs, const void* extra, float extra_alpha, int N, int H, int W, int C, int mode,
                                      int resample, float drop_rate, int op_index, const unsigned long long* seed_dev, int train,
                                      int accumulate, int de_accumulate, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_groupnorm_bwd";
  if (!x || !dy || !dx || !gamma || !beta || !dgamma || !dbeta || !stats) return xu_fail("%s: NULL pointer argument", what);
  if (gn_check_shape(what, dtype, N, H, W, C) || gn_check_mode(what, mode, resample, H, W, drop_rate)) return 1;
  if (bcs && resample != XUNET_RS_NONE) return xu_fail("%s: the fused backward (bcs) has no resampling", what);
  if (!bcs && !bstats) return xu_fail("%s: the two-kernel backward needs bstats", what);
  if (!bcs && mode == XUNET_GN_FILM && (!e || !de)) return xu_fail("%s: a FiLM norm needs e and de", what);
  if (!bcs && mode == XUNET_GN_FILM && train && drop_rate > 0.f && !seed_dev)
    return xu_fail("%s: dropout in training needs seed_dev", what);
  OpScratch scratch;
  GnArgs a = gn_fill(x, dx, mode == XUNET_GN_FILM ? e : nullptr, gamma, beta, const_cast<float*>(stats), N, H, W, C, mode, resample,
                     drop_rate, op_index, seed_dev, train ? 1 : 0);
  a.dy = dy;
  a.de = mode == XUNET_GN_FILM ? de : nullptr;
  a.dgamma = dgamma; a.dbeta = dbeta;
  a.bstats = bstats;
  a.accumulate = accumulate ? 1 : 0; a.de_accumulate = de_accumulate ? 1 : 0;
  a.extra = extra; a.extra_alpha = extra_alpha;
  if (bcs) {
    a.bcs = bcs;
    launch_gn_bwd_apply_pre(dtype, a, (cudaStream_t)stream);
  } else {
    a.skip_zero = 0;      // bstats is an output here: the reduction zeroes it first (the engine zeroes all of them at once)
    launch_gn_bwd_reduce(dtype, a, (cudaStream_t)stream);
    launch_gn_bwd_apply(dtype, a, (cudaStream_t)stream);
  }
  return op_done(what);
}

// ---- operator-level entry points of the conditioning, resampling, concat and loss launches -----------------------------
static int dtype_ok(const char* what, int dtype) {
  return dtype == XUNET_DTYPE_F32 || dtype == XUNET_DTYPE_BF16 ? 0 : xu_fail("%s: bad dtype %d", what, dtype);
}
// 4-wide vector accesses: 16-byte (fp32) / 8-byte (bf16) aligned pointers
static int vec_aligned(const char* what, int dtype, const void* p) {
  const size_t a = dtype == XUNET_DTYPE_F32 ? 16 : 8;
  return (reinterpret_cast<uintptr_t>(p) % a) == 0 ? 0 : xu_fail("%s: pointer %p is not %zu-byte aligned", what, p, a);
}
static int emb_check(const char* what, int B, int E) {
  if (B < 1) return xu_fail("%s: B = %d, need B >= 1", what, B);
  if (E < 4 || E % 4 != 0) return xu_fail("%s: E = %d, need a positive multiple of 4", what, E);
  return 0;
}

extern "C" int xunet_op_logsnr_emb(const float* logsnr, const float* w0, const float* b0, const float* w1, const float* b1, float* pe,
                                   float* h1, float* lemb, int B, int E, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_logsnr_emb";
  if (!logsnr || !w0 || !b0 || !w1 || !b1 || !pe || !h1 || !lemb) return xu_fail("%s: NULL pointer argument", what);
  if (emb_check(what, B, E)) return 1;
  OpScratch scratch;
  launch_logsnr_emb(logsnr, w0, b0, w1, b1, pe, h1, lemb, B, E, (cudaStream_t)stream);
  return op_done(what);
}

extern "C" int xunet_op_logsnr_emb_bwd(const float* dlemb, const float* w1, const float* pe, const float* h1, float* dh1, float* dw0,
                                       float* db0, float* dw1, float* db1, int B, int E, int accumulate, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_logsnr_emb_bwd";
  if (!dlemb || !w1 || !pe || !h1 || !dh1 || !dw0 || !db0 || !dw1 || !db1) return xu_fail("%s: NULL pointer argument", what);
  if (emb_check(what, B, E)) return 1;
  OpScratch scratch;
  launch_logsnr_emb_bwd(dlemb, w1, pe, h1, dh1, dw0, db0, dw1, db1, B, E, accumulate ? 1 : 0, (cudaStream_t)stream);
  return op_done(what);
}

extern "C" int xunet_op_pose_emb(int dtype, const float* R1, const float* t1, const float* R2, const float* t2, const float* K,
                                 const float* cond_mask, const float* pos_emb, const float* ref_first, const float* ref_other,
                                 float* kinv, void* out, int B, int S, int convention, const float* rays, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_pose_emb";
  if (dtype_ok(what, dtype)) return 1;
  if (!cond_mask || !out) return xu_fail("%s: NULL pointer argument", what);
  if (!rays && (!R1 || !t1 || !R2 || !t2 || !K || !kinv)) return xu_fail("%s: generated rays need R1, t1, R2, t2, K and kinv", what);
  if (!ref_first != !ref_other) return xu_fail("%s: ref_first and ref_other are given together", what);
  if (B < 1 || S < 1) return xu_fail("%s: B = %d, S = %d, need both >= 1", what, B, S);
  if (convention != XUNET_RAYS_V3D130_IJ && convention != XUNET_RAYS_OPENCV_UV) return xu_fail("%s: bad ray convention %d", what, convention);
  OpScratch scratch;
  launch_pose_emb(dtype, R1, t1, R2, t2, K, cond_mask, pos_emb, ref_first, ref_other, kinv, out, B, S, convention, rays,
                  (cudaStream_t)stream);
  return op_done(what);
}

extern "C" int xunet_op_pose_emb_bwd(int dtype, const void* dpose, float* dpos_emb, float* dref_first, float* dref_other, int B, int S,
                                     int accumulate, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_pose_emb_bwd";
  if (dtype_ok(what, dtype)) return 1;
  if (!dpose) return xu_fail("%s: NULL pointer argument", what);
  if (!dref_first != !dref_other) return xu_fail("%s: dref_first and dref_other are given together", what);
  if (B < 1 || S < 1) return xu_fail("%s: B = %d, S = %d, need both >= 1", what, B, S);
  OpScratch scratch;
  launch_pose_emb_bwd(dtype, dpose, dpos_emb, dref_first, dref_other, B, S, accumulate ? 1 : 0, (cudaStream_t)stream);
  return op_done(what);
}

static int film_emb_check(const char* what, int dtype, int N, int HW, int E) {
  if (dtype_ok(what, dtype)) return 1;
  if (N < 2 || N % 2 != 0) return xu_fail("%s: N = %d, need an even N >= 2 (two frames per sample)", what, N);
  if (HW < 1) return xu_fail("%s: HW = %d, need HW >= 1", what, HW);
  return emb_check(what, N / 2, E);
}

extern "C" int xunet_op_film_emb(int dtype, const float* lemb, const void* pe, void* semb, int N, int HW, int E, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_film_emb";
  if (!lemb || !pe || !semb) return xu_fail("%s: NULL pointer argument", what);
  if (film_emb_check(what, dtype, N, HW, E) || vec_aligned(what, dtype, pe) || vec_aligned(what, dtype, semb)) return 1;
  OpScratch scratch;
  launch_emb_fwd(dtype, lemb, pe, semb, N, HW, E, (cudaStream_t)stream);
  return op_done(what);
}

extern "C" int xunet_op_film_emb_bwd(int dtype, const float* lemb, const void* pe, const void* dsemb, void* dpe, float* dlemb, int N,
                                     int HW, int E, int write_dpe, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_film_emb_bwd";
  if (!lemb || !pe || !dsemb || !dlemb || (write_dpe && !dpe)) return xu_fail("%s: NULL pointer argument", what);
  if (film_emb_check(what, dtype, N, HW, E) || vec_aligned(what, dtype, pe) || vec_aligned(what, dtype, dsemb) ||
      (write_dpe && vec_aligned(what, dtype, dpe)))
    return 1;
  OpScratch scratch;
  launch_emb_bwd(dtype, lemb, pe, dsemb, write_dpe ? dpe : nullptr, dlemb, N, HW, E, write_dpe ? 1 : 0, (cudaStream_t)stream);
  return op_done(what);
}

extern "C" int xunet_op_resample(int dtype, const void* x, void* y, int N, int H, int W, int C, int pool, float scale, int accumulate,
                                 void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_resample";
  if (!x || !y) return xu_fail("%s: NULL pointer argument", what);
  if (dtype_ok(what, dtype) || vec_aligned(what, dtype, x) || vec_aligned(what, dtype, y)) return 1;
  if (N < 1 || H < 1 || W < 1) return xu_fail("%s: N = %d, H = %d, W = %d, need all >= 1", what, N, H, W);
  if (C < 4 || C % 4 != 0) return xu_fail("%s: C = %d, need a positive multiple of 4", what, C);
  if (pool && (H % 2 != 0 || W % 2 != 0)) return xu_fail("%s: pooling needs even H, W (got %d x %d)", what, H, W);
  OpScratch scratch;
  launch_resample(dtype, x, y, N, H, W, C, pool ? 1 : 0, scale, accumulate ? 1 : 0, (cudaStream_t)stream);
  return op_done(what);
}

extern "C" int xunet_op_copy_channels(int dtype, const void* src, void* dst, long long npix, int Cs, int Cd, int src_off, int dst_off,
                                      int Cc, int accumulate, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_copy_channels";
  if (!src || !dst) return xu_fail("%s: NULL pointer argument", what);
  if (dtype_ok(what, dtype) || vec_aligned(what, dtype, src) || vec_aligned(what, dtype, dst)) return 1;
  if (npix < 1) return xu_fail("%s: npix = %lld, need npix >= 1", what, npix);
  if (Cc < 4 || Cs % 4 || Cd % 4 || src_off % 4 || dst_off % 4 || Cc % 4)
    return xu_fail("%s: Cs = %d, Cd = %d, src_off = %d, dst_off = %d, Cc = %d, need multiples of 4 and Cc >= 4", what, Cs, Cd, src_off,
                   dst_off, Cc);
  if (src_off < 0 || dst_off < 0 || src_off + Cc > Cs || dst_off + Cc > Cd)
    return xu_fail("%s: channels [%d, %d) of %d to [%d, %d) of %d out of range", what, src_off, src_off + Cc, Cs, dst_off, dst_off + Cc, Cd);
  OpScratch scratch;
  launch_copy_channels(dtype, src, dst, npix, Cs, Cd, src_off, dst_off, Cc, accumulate ? 1 : 0, (cudaStream_t)stream);
  return op_done(what);
}

extern "C" int xunet_op_scale_add(int dtype, const void* src, void* dst, long long n, float alpha, int accumulate, void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_scale_add";
  if (!src || !dst) return xu_fail("%s: NULL pointer argument", what);
  if (dtype_ok(what, dtype) || vec_aligned(what, dtype, src) || vec_aligned(what, dtype, dst)) return 1;
  if (n < 4 || n % 4 != 0) return xu_fail("%s: n = %lld, need a positive multiple of 4", what, n);
  OpScratch scratch;
  launch_scale_add(dtype, src, dst, n, alpha, accumulate ? 1 : 0, (cudaStream_t)stream);
  return op_done(what);
}

extern "C" int xunet_op_loss(int dtype, const float* eps, const float* noise, float* sumsq, float* loss, void* dO, int B, int S,
                             void* stream) {
  xu_set_kernel_error("");
  const char* what = "xunet_op_loss";
  if (!eps || !noise || !sumsq || !loss || !dO) return xu_fail("%s: NULL pointer argument", what);
  if (dtype_ok(what, dtype)) return 1;
  if (B < 1 || S < 1) return xu_fail("%s: B = %d, S = %d, need both >= 1", what, B, S);
  OpScratch scratch;
  launch_loss(dtype, eps, noise, sumsq, loss, dO, B, S, (cudaStream_t)stream);
  return op_done(what);
}
