/* xunet_b200.h -- C-ABI of libxunet_b200.so: the H100 (sm_90a) X-UNet hot path.
 *
 * The reference (shiveshkhaitan/novel_view_synthesis_3d) has no FFI/plugin layer: its boundary is the
 * Flax functional API used by train.py / sampling.py.  Each entry point below names the reference
 * call it stands in for (file:line relative to the reference tree).  Conventions:
 *   - every pointer argument documented "device" is a CUDA device pointer owned by the caller
 *     (the PyTorch host allocates; the library allocates nothing after xunet_create);
 *   - `stream` is a cudaStream_t passed as void*; all launches are asynchronous on it and
 *     graph-capturable (no syncs, no allocations inside forward/backward/adam/sampler calls);
 *   - return 0 on success, non-zero on error; xunet_last_error() gives the message; nothing throws;
 *   - a handle is bound to the device current at creation and is NOT thread-safe.
 *   - inputs are float32 (JAX down-casts the float64 numpy batch with x64 off, train.py:132-140).
 */
#ifndef XUNET_B200_H
#define XUNET_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define XUNET_MAX_LEVELS 8
#define XUNET_DTYPE_F32 0   /* fp32 activations, fp32 SIMT math: the <=1e-3 parity ("verify") mode      */
#define XUNET_DTYPE_BF16 1  /* bf16 activations, fp32 accumulate / statistics / master weights           */

#define XUNET_RAYS_V3D130_IJ 0  /* visu3d<=1.3: K^-1 applied to (row+.5, col+.5)  (requirements.txt:17) */
#define XUNET_RAYS_OPENCV_UV 1  /* visu3d>=1.4: K^-1 applied to (col+.5, row+.5)                        */

/* XUNet module attributes, model/xunet.py:205-215 (ch_mult / attn_resolutions are class attributes there). */
typedef struct xunet_config {
  int ch;
  int n_levels;
  int ch_mult[XUNET_MAX_LEVELS];
  int emb_ch;
  int num_res_blocks;
  int n_attn_resolutions;
  int attn_resolutions[XUNET_MAX_LEVELS];
  int attn_heads;
  float dropout;
  int use_pos_emb;
  int use_ref_pose_emb;
  int ray_convention;
} xunet_config;

typedef struct xunet_handle xunet_handle;

/* Device pointers of one batch: the dict train.py:53-60 / sampling.py:156-165 builds.
 * x, z: (B,S,S,3); logsnr: (B); R1,R2,K: (B,3,3) row-major; t1,t2: (B,3); cond_mask: (B) 0/1 floats
 * (model/xunet.py:176-179).  R,t are cam->world (dataset/data_loader.py:105-108). */
typedef struct xunet_batch {
  const float* x;
  const float* z;
  const float* logsnr;
  const float* R1;
  const float* t1;
  const float* R2;
  const float* t2;
  const float* K;
  const float* cond_mask;
  /* OPTIONAL (NULL = compute rays from R,t,K with cfg.ray_convention): precomputed camera rays of both cameras,
   * (B, 2, S, S, 6) fp32 = [pos xyz | dir xyz] per pixel, camera 0 = (R1,t1), camera 1 = (R2,t2) -- exactly what
   * v3d.Camera(spec, world_from_cam).rays() returns at model/xunet.py:159-161,166-168 (.pos, .dir).  With this set the
   * network never depends on the library's restatement of visu3d's pixel convention; R,t,K are then unused. */
  const float* rays;
} xunet_batch;

const char* xunet_last_error(void);
int xunet_version(void);

/* XUNet() + shape inference of .init (train.py:39-43): builds the static execution plan for
 * (config, batch, side, dtype).  training!=0 reserves gradient storage in the workspace. */
int xunet_create(const xunet_config* cfg, int batch, int side, int dtype, int training, xunet_handle** out);
void xunet_destroy(xunet_handle* h);

/* Parameter tree (SURVEY Appendix A): leaves in Flax naming ("XUNetBlock_3/ResnetBlock_0/Conv_0/kernel"),
 * Flax shapes and C-order element layout, concatenated into ONE flat fp32 buffer at `offset` (elements). */
long long xunet_param_count(const xunet_handle* h);
int xunet_param_leaves(const xunet_handle* h);
int xunet_param_leaf(const xunet_handle* h, int i, const char** name, int* ndim, long long shape[5],
                     long long* offset);

long long xunet_workspace_bytes(const xunet_handle* h);

/* Named activations kept in the workspace after a forward (for parity tests): dims = (N=2B, H, W, C),
 * offset in bytes; *is_f32 != 0 -> fp32 elements, else elements of the handle dtype.  After a backward,
 * *grad_byte_offset (>=0) locates the gradient of the same tensor (-1 if it has none). */
int xunet_tap_count(const xunet_handle* h);
int xunet_tap(const xunet_handle* h, int i, const char** name, int dims[4], long long* byte_offset, int* is_f32,
              long long* grad_byte_offset);

/* The plan's convolution and attention launches, in op order (read-only; needs no GPU), so that tests can run each one through
 * the operator-level entry points at exactly the plan's shape and arguments.  kernel: what runs a direction of a conv. */
#define XUNET_LAUNCH_CONV 0
#define XUNET_LAUNCH_ATTN 1
#define XUNET_KERNEL_NONE -1     /* that direction is not run: no backward (training=0), or the input needs no gradient */
#define XUNET_KERNEL_SIMT 0
#define XUNET_KERNEL_TC 1        /* tensor cores: xunet_op_conv* impl 1 */
#define XUNET_KERNEL_CIN3 2      /* direct 3-channel input kernel: impl 2 */
#define XUNET_KERNEL_COUT3 3     /* direct 3-channel output kernel: impl 2 */
typedef struct xunet_launch_info {
  int kind;                /* XUNET_LAUNCH_* */
  /* conv: y = alpha * (conv(x, W; ksize, stride, SAME) + bias (+ residual)), Co in nseg weight segments */
  int leaf;                /* index of the kernel leaf (xunet_param_leaf numbering); -1 for attention */
  int N, Hi, Wi, Ci, Ho, Wo, Co, ksize, stride, nseg;
  int residual;
  float alpha;
  int fwd, dgrad, wgrad;   /* XUNET_KERNEL_* of the forward, data gradient and weight gradient */
  int emits_stats;         /* conv / attention: the forward emits the GroupNorm statistics of its output */
  float bwd_alpha;         /* alpha of the data and weight gradients (alpha times the scale of an aliased output gradient) */
  int accumulate;          /* the data gradient adds into its destination */
  int gn_mode;             /* the data gradient carries the backward of the GroupNorm before it: XUNET_GN_*; -1 none */
  /* attention: qkv (N, L, 3C), heads, cross = keys and values of the other frame of the sample; impl 1 tensor cores, 0 SIMT */
  int L, C, heads, cross, impl;
} xunet_launch_info;
int xunet_plan_launch_count(const xunet_handle* h);
int xunet_plan_launch(const xunet_handle* h, int i, xunet_launch_info* out);

/* The plan's other launches, in op order (read-only; needs no GPU): what each op's forward and backward launchers receive, so
 * that tests can run them through the operator-level entry points below at the plan's arguments. */
#define XUNET_PLAN_OP_LOGSNR 0          /* the log-SNR MLP: xunet_op_logsnr_emb / _bwd at (B, E) */
#define XUNET_PLAN_OP_POSE 1            /* rays + NeRF posenc: xunet_op_pose_emb / _bwd at (B, S) */
#define XUNET_PLAN_OP_EMB 2             /* swish(logsnr_emb + pose-embedding level): xunet_op_film_emb / _bwd */
#define XUNET_PLAN_OP_RESAMPLE 3        /* the residual path of a resampling ResnetBlock: xunet_op_resample */
#define XUNET_PLAN_OP_CONCAT 4          /* a skip-connection concat: xunet_op_copy_channels, two per direction */
#define XUNET_PLAN_OP_ATTN_RESIDUAL 5   /* the residual gradient of an attention block: xunet_op_scale_add */
#define XUNET_PLAN_OP_LOSS 6            /* the frame-1 output and the ||eps_hat - eps|| loss: xunet_op_loss */
typedef struct xunet_op_info {
  int kind;                /* XUNET_PLAN_OP_* */
  int B, S, E;             /* the plan's samples, image side and emb_ch */
  int N, H, W, C;          /* the op's input (N, H, W, C): EMB the pose-embedding level; RESAMPLE x; CONCAT its first input a;
                              ATTN_RESIDUAL the block output; else N = 2B, H = W = S and C = E (LOGSNR), 144 (POSE), 3 (LOSS) */
  int C2;                  /* CONCAT: channels of the second input b */
  int copies[4][5];        /* CONCAT: (Cs, Cd, src_off, dst_off, Cc) of the forward copies of a and b into y, then of the
                              backward copies of grad(y) into grad(a) and grad(b) */
  int rs;                  /* RESAMPLE: XUNET_RS_DOWN or XUNET_RS_UP */
  int fwd_pool;            /* RESAMPLE: xunet_op_resample's pool and scale in the forward */
  float fwd_scale;
  float gscale;            /* RESAMPLE: scale of the output's aliased gradient (1: not aliased) */
  int bwd_pool;            /* RESAMPLE: pool and scale of the backward (the adjoint, on the output's gradient) */
  float bwd_scale;
  float alpha;             /* ATTN_RESIDUAL: grad(residual) = alpha grad(output) (+ the prior when acc_r) */
  int acc_x, acc_r;        /* the backward adds into grad(x) / grad(second input) instead of storing */
  int need_grad;           /* the backward runs (POSE: the parameter gradients; CONCAT: grad(a) is written) */
  int need_grad_r;         /* CONCAT: grad(b) is written */
  int write_dpe;           /* EMB: the backward writes the gradient of the pose-embedding level */
  int pos_emb, ref_pose_emb, ray_convention;   /* POSE: the pos_emb / ref_pose_emb leaves exist; XUNET_RAYS_* */
} xunet_op_info;
int xunet_plan_op_count(const xunet_handle* h);
int xunet_plan_op(const xunet_handle* h, int i, xunet_op_info* out);

/* XUNet.apply({'params': p}, batch, cond_mask=, train=, rngs=)  (train.py:63-66, sampling.py:131-132).
 * params: device, flat fp32.  seed_dev: device pointer to ONE uint64 dropout seed (read at execution
 * time, so a captured graph sees updates); may be NULL when train==0.  eps_out: device (B,S,S,3) fp32. */
int xunet_forward(xunet_handle* h, const float* params, const xunet_batch* batch, int train,
                  const unsigned long long* seed_dev, void* workspace, float* eps_out, void* stream);

/* Sampler fast path: after one xunet_forward, declare poses / K / cond_mask / params unchanged; subsequent forwards skip the
 * ray + posenc kernel, the pose-embedding convs and the bf16 weight-shadow conversion (the reference recomputes all of it
 * 2000 times per view, sampling.py:131-132).  on=0 restores the full forward. */
int xunet_set_static_conditioning(xunet_handle* h, int on);

/* Sampler feature cache (DeepCache, Ma et al. 2024): level = 0 (the default) restores the full forward; level = L in
 * [1, n_levels - 1] makes the following xunet_forward calls cheap forwards.  A cheap forward reads the output of the up
 * ResnetBlock that leaves level L (the input of up-level L - 1) as the last full forward left it in the workspace, and runs
 * only the ops the output needs given that tensor: the conditioning, the input conv, the down and up blocks of the levels
 * below L and the head.  The deep blocks, the down ResnetBlock into level L, their FiLM Denses and the pose-embedding convs of
 * levels >= L are skipped, so the deep feature keeps the log-SNR and inputs of the step that computed it.  Static
 * conditioning applies to the kept ops as usual, and xunet_count_kernels counts the forward at the current level.
 * Fails on a training handle (a backward needs every activation) and for a level outside [0, n_levels - 1].  A cheap
 * forward at L fails unless a full forward has completed on the handle, and no cheap forward at a deeper level (which
 * recomputes the level-L tensor) has run since. */
int xunet_set_feature_cache(xunet_handle* h, int level);

/* The value_and_grad half of apply_model (train.py:62-71): must follow xunet_forward on the same
 * workspace.  loss = ||eps_hat - noise||_F (train.py:67).  grads: device flat fp32 (param layout),
 * overwritten.  loss_out: device, 1 float. */
int xunet_backward(xunet_handle* h, const float* params, const xunet_batch* batch, const float* noise,
                   const unsigned long long* seed_dev, void* workspace, float* grads, float* loss_out,
                   void* stream);

/* xunet_backward that ADDS the parameter gradient into `grads` instead of overwriting it (gradient accumulation over
 * micro-batches, optax.MultiSteps): each leaf becomes grads + g in fp32, one rounding per element, where g is exactly what
 * xunet_backward would have written.  Same arguments, ordering guarantees, bucket hook and graph-capture behaviour. */
int xunet_backward_accumulate(xunet_handle* h, const float* params, const xunet_batch* batch, const float* noise,
                              const unsigned long long* seed_dev, void* workspace, float* grads, float* loss_out,
                              void* stream);

/* xunet_backward with the mean-squared epsilon loss (L_simple of DDPM / 3DiM) instead of the Frobenius norm, optionally weighted
 * per sample (e.g. min-SNR-gamma):
 *     loss = (1/B) sum_b w_b * (1/P) sum_i (eps_hat - noise)_bi^2        (P = S*S*3; residual in fp32)
 * The sums of squares are reduced in fp64 in an order fixed by (B, P) alone, without atomics, and rounded to fp32 once
 * into loss_out.  The output gradient is fl32(2 w_b / (B P)) * (eps_hat - noise), rounded to the activation dtype.
 * loss_weight: device (B) fp32, or NULL (all 1).  accumulate != 0 adds into grads exactly as xunet_backward_accumulate
 * does.  Same ordering, bucket hook and graph-capture behaviour as xunet_backward. */
int xunet_backward_mse(xunet_handle* h, const float* params, const xunet_batch* batch, const float* noise,
                       const float* loss_weight, const unsigned long long* seed_dev, void* workspace, float* grads,
                       float* loss_out, int accumulate, void* stream);

/* Vector-Jacobian product of the forward (jax.vjp / jax.grad over XUNet.apply): the backward seeded with the caller's
 * d_eps = dL/d(eps_hat) instead of a built-in loss, so any loss on eps_hat is host code.  Must follow xunet_forward on the same
 * handle, workspace, batch, params and seed_dev; that forward's train flag decides the dropout masks, as in xunet_backward.
 *   d_eps: device (B,S,S,3) fp32, the gradient of the tensor xunet_forward wrote to eps_out.  The output gradient of the
 *          network is d_eps rounded once to the activation dtype for the target frame, and zero for the conditioning frame.
 *   grads: device flat fp32 (param layout), overwritten; accumulate != 0 adds into it exactly as xunet_backward_accumulate does.
 *   dx, dz: device (B,S,S,3) fp32, or NULL (that input's gradient is not computed): dL/dx and dL/dz of the two input views,
 *          overwritten.  In bf16 mode the rounding of x and z into the bf16 input tensor counts as identity (straight-through),
 *          and dx / dz come straight from fp32 accumulators, not rounded to bf16.
 * Fixed reduction order and no atomics: repeated calls give the same bits.  Errors as xunet_backward: a NULL required pointer,
 * a handle created with training=0, no xunet_forward yet.  Same bucket hook and graph-capture behaviour as xunet_backward. */
int xunet_backward_vjp(xunet_handle* h, const float* params, const xunet_batch* batch, const float* d_eps,
                       const unsigned long long* seed_dev, void* workspace, float* grads, int accumulate, float* dx, float* dz,
                       void* stream);

/* Input gradients of xunet_backward_vjp_inputs: every pointer is a device fp32 buffer the caller owns, or NULL (not computed).
 *   dx, dz: (B,S,S,3), as in xunet_backward_vjp.
 *   d_rays: (B,2,S,S,6), the layout of xunet_batch.rays: dL/d[pos xyz | dir xyz] of every pixel's ray, camera 0 then camera 1,
 *           whether the rays were given (batch->rays) or generated from R, t, K.  Samples with cond_mask = 0 get exact zeros
 *           (their pose embedding is zeroed in the forward).  Required when any camera output below is set.
 *   dR1, dt1, dR2, dt2, dK: (B,3,3) / (B,3) / (B,3,3): dL/dR, dL/dt of the cameras (R a free 3x3 matrix: projecting onto SO(3) is
 *           the caller's job) and dL/dK of the intrinsics shared by both cameras.  Generated rays only (batch->rays == NULL).
 * The log-SNR gets no gradient. */
typedef struct xunet_input_grads {
  float* dx;
  float* dz;
  float* d_rays;
  float* dR1;
  float* dt1;
  float* dR2;
  float* dt2;
  float* dK;
} xunet_input_grads;

/* xunet_backward_vjp that also returns the gradients of the cameras / rays (out may be NULL: parameter gradient only).  The
 * parameter gradient, dx and dz are bit for bit those of xunet_backward_vjp, with or without camera outputs.  The ray gradient is
 * the data gradient of the pose-embedding convolutions (tensor cores in bf16 mode, weights as the forward's bf16 shadows) with
 * the posenc Jacobian applied per pixel; the camera gradients are reduced from it in fp64 in a fixed order.  Fixed bits, no
 * atomics, no allocation, graph-capturable.  Errors: those of xunet_backward_vjp, a camera output without d_rays, a camera
 * output with batch->rays set. */
int xunet_backward_vjp_inputs(xunet_handle* h, const float* params, const xunet_batch* batch, const float* d_eps,
                              const unsigned long long* seed_dev, void* workspace, float* grads, int accumulate,
                              const xunet_input_grads* out, void* stream);

/* Data-parallel hook (north_star: "one NCCL allreduce of the gradient bucket"; the reference's pmap step would place
 * lax.pmean between value_and_grad and apply_gradients, train.py:70-76).  With a callback installed, xunet_backward calls
 *     fn(user, elem_offset, n_elems)
 * on the HOST, in descending offset order, each time grads[elem_offset, elem_offset+n_elems) is final: every kernel that
 * writes it has been enqueued and ordered before the current point of `stream` (the library's internal side stream is
 * joined first).  The callback typically enqueues an all-reduce of that range on a communication stream ordered after
 * `stream`, so NVLink traffic overlaps the rest of the backward.  The ranges partition the whole flat buffer; buckets
 * are cut at residual-block boundaries once they reach min_bucket_bytes (the last one, offset 0, takes the remainder).
 * fn == NULL removes the hook.  Graph capture: the callback runs at capture time, so what it enqueues is captured too. */
typedef void (*xunet_bucket_fn)(void* user, long long elem_offset, long long n_elems);
int xunet_set_grad_bucket_callback(xunet_handle* h, xunet_bucket_fn fn, void* user, long long min_bucket_bytes);
int xunet_grad_bucket_count(const xunet_handle* h);

/* Number of kernel launches (graph kernel nodes) one xunet_forward / xunet_backward issues for this plan; counted by
 * capturing the call into a throw-away CUDA graph (nothing executes).  Arguments as for forward/backward. */
int xunet_count_kernels(xunet_handle* h, const float* params, const xunet_batch* batch, const float* noise,
                        const unsigned long long* seed_dev, void* workspace, float* grads, float* loss_out,
                        int* n_forward, int* n_backward);

/* update_model / TrainState.apply_gradients with optax.adam (train.py:45,74-76).  `step` is the 1-based
 * step count after increment; if step_dev != NULL the kernel reads *step_dev (device int64) instead.
 * grad_scale multiplies the gradient first (1/world_size after the all-reduce). */
int xunet_adam_step(float* params, const float* grads, float* m, float* v, long long n, long long step,
                    const long long* step_dev, double lr, double b1, double b2, double eps, double grad_scale,
                    void* stream);

/* xunet_adam_step followed by the exponential moving average of the weights DDPM-family models are sampled from:
 *     ema <- d * ema + (1 - d) * params_new        (d = ema_decay, e.g. 0.9999)
 * fused into the same pass (params_new never leaves registers).  ema: device, n floats, updated in place.  Each product and
 * the sum are rounded separately in fp32 (no FMA), so a float32 host restatement reproduces ema bit for bit.  params / m / v
 * come out bit-identical to xunet_adam_step.  ema == NULL or ema_decay outside [0, 1] is an error.  Graph-capturable. */
int xunet_adam_ema_step(float* params, const float* grads, float* m, float* v, float* ema, long long n, long long step,
                        const long long* step_dev, double lr, double b1, double b2, double eps, double grad_scale,
                        double ema_decay, void* stream);

/* Global L2 norm of the (scaled) flat gradient, the reduction of optax.clip_by_global_norm:
 *     *norm_out = (float) sqrt( sum_i fp32(grads[i] * grad_scale)^2 )
 * Every square is accumulated in fp64, in an order fixed by n alone (no atomics, no dependence on the SM count), so the same
 * buffer gives the same bits on every run and every GPU.  scratch: device, XUNET_GRAD_NORM_SCRATCH doubles, contents
 * irrelevant on entry; on completion scratch[0] holds the fp64 sum of squares.  norm_out: device, 1 float.  Two kernels,
 * no host sync, graph-capturable. */
#define XUNET_GRAD_NORM_SCRATCH 1024
int xunet_grad_global_norm(const float* grads, long long n, double grad_scale, double* scratch, float* norm_out,
                           void* stream);

/* xunet_adam_step (ema == NULL) or xunet_adam_ema_step (ema != NULL) with a linear learning-rate warm-up and clipping by a
 * global gradient norm read from the device: optax.chain(optax.clip_by_global_norm(max_norm),
 * optax.adam(optax.linear_schedule(0, lr, warmup_steps))).  With the Adam count `step` (after increment, or *step_dev):
 *   - learning rate: lr_t = lr * min(step - 1, W) / W in double, rounded to fp32 once (W = warmup_steps; the first update
 *     uses lr_t = 0, as the schedule's own count starts at 0); W == 0: the constant lr;
 *   - clipping (norm_dev != NULL, *norm_dev = the norm of grads * grad_scale, e.g. from xunet_grad_global_norm): the scaled
 *     gradient g is used as is if *norm_dev < max_norm, else as fl(fl(g / norm) * max_norm) (each operation rounded once);
 *   - non-finite *norm_dev: the step is skipped -- params / m / v / ema are not touched -- and *skipped_dev (device int64)
 *     is incremented.  The caller's step counter still advances, unlike optax.apply_if_finite, which holds the inner count.
 * norm_dev == NULL: no clipping and no guard (max_norm and skipped_dev are then ignored).  With *norm_dev < max_norm and
 * W == 0 the result is bit-identical to xunet_adam_step / xunet_adam_ema_step.  Errors: max_norm <= 0 or NaN,
 * warmup_steps < 0, skipped_dev == NULL with norm_dev given, ema_decay outside [0, 1] with ema given.  Graph-capturable. */
int xunet_adam_clip_step(float* params, const float* grads, float* m, float* v, float* ema, long long n, long long step,
                         const long long* step_dev, double lr, double b1, double b2, double eps, double grad_scale,
                         double ema_decay, const float* norm_dev, double max_norm, long long warmup_steps,
                         long long* skipped_dev, void* stream);

/* xunet_adam_clip_step keeping two power-function averages of the weights instead of an EMA (post-hoc EMA, Karras et al.
 * 2024, EDM2 §3): with the Adam count t (`step`, or *step_dev) and k in {a, b}
 *     beta_k = (1 - 1/t)^(gamma_k + 1)            in double, beta_k and 1 - beta_k each rounded to fp32 once
 *     ema_k <- beta_k * ema_k + (1 - beta_k) * params_new
 * fused into the same pass, each product and the sum rounded separately in fp32 (no FMA) as in xunet_adam_ema_step.  Weight
 * of the parameters after update tau in ema_k at count t: (tau^(g+1) - (tau-1)^(g+1)) / t^(g+1), g = gamma_k; beta_1 = 0, so
 * the first update overwrites both averages.  Warm-up, clipping and the skip of a non-finite norm are xunet_adam_clip_step's;
 * a skipped update touches neither average.  params / m / v come out bit-identical to xunet_adam_clip_step.  ema_a, ema_b:
 * device, n floats each, updated in place.  Errors: a NULL average, ema_a == ema_b, a gamma that is not finite or is <= -1,
 * step < 1 without step_dev, and xunet_adam_clip_step's clip / warm-up argument errors.  Graph-capturable. */
int xunet_adam_posthoc_step(float* params, const float* grads, float* m, float* v, float* ema_a, float* ema_b, long long n,
                            long long step, const long long* step_dev, double lr, double b1, double b2, double eps,
                            double grad_scale, double gamma_a, double gamma_b, const float* norm_dev, double max_norm,
                            long long warmup_steps, long long* skipped_dev, void* stream);

/* One ancestral update of sampling.py:128-151 with the schedule on the device, for a per-step CUDA graph (forward + this call
 * + counter increment) that is replayed with no host arithmetic in between (the reference does the schedule math in numpy
 * between two un-jitted model calls, sampling.py:133-151).  Given the 2B-batched model output eps2 =
 * [out_cond (B,S,S,3); out_uncond (B,S,S,3)] and the coefficients of row k = *pos_dev of the table:
 *     out = (1+w) out_c - w out_u;  x0 = clip(c_recip z - c_recipm1 out, -1, 1);  z' = c1 x0 + c2 z + sigma * noise_k.
 * The step is linear in the network output, so the table decides what that output is: an eps-prediction table has
 * c_recip = sqrt_recip_alphas_cumprod = 1/sqrt(abar), c_recipm1 = sqrt_recipm1_alphas_cumprod = sqrt(1/abar - 1); a
 * v-prediction table (v = sqrt(abar) eps - sqrt(1 - abar) x0, so x0 = sqrt(abar) z - sqrt(1 - abar) v) has c_recip = sqrt(abar),
 * c_recipm1 = sqrt(1 - abar).  This holds for every step entry below.
 * table: device (steps, 8) floats, row k (k = 0: first executed step = highest t) = {c_recip, c_recipm1,
 * c1 = posterior_mean_coef1, c2 = posterior_mean_coef2, sigma (0 at t=0), log-SNR fed to the NEXT forward (sampling.py:151),
 * 0, 0} (a DDIM table puts its c_x0, c_z, sigma in columns 2-4); pos_dev: device int32 loop position (the caller increments
 * it after the call, in stream order).  z (n = B*S*S*3) is updated in place; the new z is also written to both halves of the next
 * forward's [cond ; uncond] input next_z2 (2n) and next_logsnr2 (batch2 = 2B entries).
 * Noise: noise != NULL: device (steps, n) floats, step k reads noise[k*n .. k*n+n).  noise == NULL: the device hash normal
 * of (*seed_dev - k), i.e. the caller stores seed(first step) and the per-step seeds count down like the timestep index;
 * seed_dev (required either way) is a device uint64 so a captured graph can be re-seeded. */
int xunet_sampler_step_table(const float* eps2, float* z, const float* noise, long long n, float w, const float* table,
                             const int* pos_dev, const unsigned long long* seed_dev, float* next_z2, float* next_logsnr2,
                             int batch2, void* stream);

/* The multistep form of xunet_sampler_step_table (same arguments, same contract) for second-order solvers such as
 * DPM-Solver++(2M): row k = *pos_dev of the table is {c_recip, c_recipm1, c_x0, c_z, sigma, log-SNR of the next forward,
 * c_prev, 0}, and x0_hist (device, n floats, required) carries the previous step's clipped x0 between calls:
 *     x0 = clip(c_recip z - c_recipm1 out, -1, 1)  as above;
 *     z' = fma(sigma, noise_k, fma(c_prev, x0_hist[i], fma(c_x0, x0, c_z * z)))   (fp32, one rounding per fma);
 *     x0_hist[i] = x0.
 * A row with c_prev == 0 skips the c_prev term and never reads x0_hist, so the first step of a chain needs no initialised
 * history.  Graph-capturable. */
int xunet_sampler_step_multistep(const float* eps2, float* z, const float* noise, long long n, float w, const float* table,
                                 const int* pos_dev, const unsigned long long* seed_dev, float* x0_hist, float* next_z2,
                                 float* next_logsnr2, int batch2, void* stream);

/* The sampler step with DYNAMIC THRESHOLDING of x0 (Saharia et al. 2022, Imagen section 2.3) in place of the fixed clip:
 * the same table row, noise, next_z2 / next_logsnr2 writes and (x0_hist != NULL) multistep term as
 * xunet_sampler_step_table (x0_hist == NULL) and xunet_sampler_step_multistep (x0_hist != NULL), with
 *     x0 = c_recip z - c_recipm1 out  (unclipped, out the guided network output as above);  s_b = max(1, quantile_p(|x0|) over the per = n / batch values of view b);
 *     x0 <- clip(x0, -s_b, s_b) / s_b   (fp32 division, round to nearest),
 * and this x0 feeds the update and x0_hist.  quantile_p is numpy's np.quantile(a, p) (method 'linear') in fp64 on the fp32
 * values a = |x0| sorted ascending: idx = (per - 1) p, lo = floor(idx), hi = min(lo + 1, per - 1), g = idx - lo,
 * d = a[hi] - a[lo], q = g < 0.5 ? a[lo] + d g : a[hi] - d (1 - g), each operation rounded once (no fma); s_b = max(fp32(q), 1).
 * A view with s_b = 1 gets exactly the bits of the static step.  s_b is found by an integer radix select, so it depends on the
 * view's values alone (not on batch or on the view's position).  scale_out (device, batch floats) receives s_b when given.
 * Errors: a NULL required pointer, n <= 0, batch2 <= 0, batch < 1, n % batch != 0, per > XUNET_SAMPLER_DYN_MAX_PER (the
 * shared-memory slices are sized for it), percentile NaN or outside (0, 1].  One launch; no allocation, no host sync,
 * graph-capturable. */
#define XUNET_SAMPLER_DYN_MAX_PER (256 * 256 * 3)
int xunet_sampler_step_dynamic(const float* eps2, float* z, const float* noise, long long n, float w, const float* table,
                               const int* pos_dev, const unsigned long long* seed_dev, float* x0_hist, int batch,
                               double percentile, float* scale_out, float* next_z2, float* next_logsnr2, int batch2,
                               void* stream);

/* The UNGUIDED sampler step, for a model whose guidance is in its weights (a distilled student): one B-batch conditional
 * forward per step instead of the [cond ; uncond] 2B batch.  out (device, n = B*S*S*3 floats) is that forward's output, used
 * as is in place of the guided (1+w) out_c - w out_u; everything else is the guided step's:
 *   percentile == 0, x0_hist == NULL: xunet_sampler_step_table;   percentile == 0, x0_hist != NULL: xunet_sampler_step_multistep;
 *   percentile in (0, 1]: xunet_sampler_step_dynamic (x0_hist NULL or set as there), scale_out optional as there.
 * The new z goes to z and to next_z (n floats: the next forward's z input), and the row's log-SNR to next_logsnr (batch
 * floats).  Each instance is the guided kernel with the guidance expression replaced by out, so the result equals the
 * guided step run at w = 0 with out in both halves, bit for bit (but for the sign of an exactly zero output).
 * Errors: a NULL required pointer, n <= 0, batch < 1, n % batch != 0; with percentile != 0 also per > XUNET_SAMPLER_DYN_MAX_PER
 * or percentile NaN or outside (0, 1].  One launch; graph-capturable. */
int xunet_sampler_step_cond(const float* out, float* z, const float* noise, long long n, const float* table, const int* pos_dev,
                            const unsigned long long* seed_dev, float* x0_hist, int batch, double percentile, float* scale_out,
                            float* next_z, float* next_logsnr, void* stream);

/* The AUTOGUIDED sampler step (Karras et al. 2024, "Guiding a diffusion model with a bad version of itself"): the negative
 * of the guidance is the output of a weaker guide model on the same inputs, not the pose-dropped branch of a 2B batch.
 * out_main and out_guide (device, n = B*S*S*3 floats each) are the B-batch outputs of the main and the guide forward, both
 * with cond_mask 1; the step uses
 *     out = (1+w) out_main - w out_guide
 * with the same fp32 operations, in the same order, as the guided steps' (1+w) out_c - w out_u, and is otherwise
 * xunet_sampler_step_cond's:
 *   percentile == 0, x0_hist == NULL: xunet_sampler_step_table;   percentile == 0, x0_hist != NULL: xunet_sampler_step_multistep;
 *   percentile in (0, 1]: xunet_sampler_step_dynamic (x0_hist NULL or set as there), scale_out optional as there.
 * The new z goes to z and to next_z (n floats: the main forward's z input, which the guide forward reads too), and the row's
 * log-SNR to next_logsnr (batch floats).  With w = 0, or with out_guide equal to out_main and w = 1, the result is the bits
 * of xunet_sampler_step_cond on out_main.
 * Errors: a NULL required pointer, n <= 0, batch < 1, n % batch != 0; with percentile != 0 also per > XUNET_SAMPLER_DYN_MAX_PER
 * or percentile NaN or outside (0, 1].  One launch; graph-capturable. */
int xunet_sampler_step_guide(const float* out_main, const float* out_guide, float* z, const float* noise, long long n, float w,
                             const float* table, const int* pos_dev, const unsigned long long* seed_dev, float* x0_hist,
                             int batch, double percentile, float* scale_out, float* next_z, float* next_logsnr, void* stream);

/* Device-side forward diffusion = the per-item work of SceneInstanceDataset.__getitem__ (dataset/data_loader.py:92-110):
 *   t ~ U{0..999};  noise ~ N(0,1);  z = sqrt_ac[t] * x0 + sqrt_1mac[t] * noise;  logsnr = logsnr_schedule_cosine(t/1000);
 *   cond_mask = (u > p_uncond)  (train.py:64).
 * sqrt_ac / sqrt_1mac: device tables of 1000 floats (cosine-beta schedule, data_loader.py:15-25,70-74).  t_in / noise_in may
 * be NULL (drawn on the device from `seed`) or given (parity tests).  All outputs are device buffers; x0 (B, per). */
int xunet_forward_diffusion(const float* x0, const float* noise_in, const int* t_in, unsigned long long seed,
                            const float* sqrt_ac, const float* sqrt_1mac, float p_uncond, float* z, float* noise_out,
                            float* logsnr_out, int* t_out, float* cond_mask_out, int B, long long per, void* stream);

/* xunet_forward_diffusion for v-prediction (Salimans & Ho 2022): the same draws, z, logsnr, t and cond_mask, plus the v target
 *   v = __fsub_rn(__fmul_rn(sqrt_ac[t], noise), __fmul_rn(sqrt_1mac[t], x0))      (each fp32 operation rounded once)
 * stored to v_out (device, B * per floats, required) in the same pass.  noise_out may be NULL (the noise is then not stored).
 * One launch. */
int xunet_forward_diffusion_v(const float* x0, const float* noise_in, const int* t_in, unsigned long long seed,
                              const float* sqrt_ac, const float* sqrt_1mac, float p_uncond, float* z, float* noise_out,
                              float* v_out, float* logsnr_out, int* t_out, float* cond_mask_out, int B, long long per,
                              void* stream);

/* A set of SRN views held in device memory (srn_data.DeviceScenes): item i = view v of instance inst, items of one instance
 * contiguous, instance after instance.  All pointers are device memory.
 *   pixels     (n_items, S, S, 3): uint8 (pixel_kind XUNET_PIXELS_U8: the view's 8-bit RGB centre crop, read as
 *              ((u / 255) - 0.5) * 2 with each fp32 operation rounded once) or fp32 (XUNET_PIXELS_F32: values in [-1, 1]);
 *   R (n_items, 3, 3), t (n_items, 3): cam->world pose of each item;  K (n_instances, 3, 3): intrinsics rescaled to S;
 *   first, count (n_instances) int32: first item and number of views of each instance;  item_inst (n_items) int32. */
#define XUNET_PIXELS_U8 0
#define XUNET_PIXELS_F32 1
typedef struct xunet_srn_store {
  const void* pixels;
  int pixel_kind;
  int S;
  long long n_items;
  int n_instances;
  const float* R;
  const float* t;
  const float* K;
  const int* first;
  const int* count;
  const int* item_inst;
} xunet_srn_store;

/* One training micro-batch drawn, gathered and noised on the device: the host loader + xunet_forward_diffusion in one kernel.
 * step_dev: device int64 holding the 1-based number of the update being run (TrainStep's step counter after its increment);
 * c = *step_dev - 1 is the Adam count before it.  Sample b of micro-batch j of k, on rank `rank` of `world`, has the draw index
 *   g = ((c k + j) world + rank) B + b           (the ranks and micro-batches of one update partition [c k world B, (c+1) k world B))
 * and draws:  epoch = g / N, item = P_{seed,epoch}(g mod N) (a keyed 4-round Feistel bijection of [0, N) with cycle-walking,
 * so every item is the source once per N draws), (inst, v) = the item's instance and view, v2 = mix(seed, g) mod count[inst]
 * (uniform over the instance's views, may equal v).  The micro-batch's diffusion seed is s = mix(seed, c k + j, rank).  Then
 *   out->x[b] = view v, out->R1/t1[b] its pose, out->R2/t2[b] the pose of view v2, out->K[b] = K[inst],
 *   out->z, noise, out->logsnr, out->cond_mask = exactly xunet_forward_diffusion(view v2 of every sample, seed = s, p_uncond)
 * and, when given, loss_weight[b] = snr_weight[t_b] (all 1 when snr_weight is NULL), idx_out (B, 3) int32 = (inst, v, v2),
 * t_out (B) int32 = the drawn timesteps.  The exact mix functions are in csrc/data.cu and restated in numpy by
 * srn_data.draw_indices / diffusion_seed.  out->rays is ignored; out->x .. K, cond_mask, noise are required.
 * Errors: a NULL required pointer, B < 1, k < 1, world < 1, rank outside [0, world), j outside [0, k), an empty store, an
 * unknown pixel_kind.  Deterministic (a function of the store, seed, *step_dev and the integer arguments).  One launch; no
 * atomics, no allocation, no host sync, graph-capturable. */
int xunet_srn_batch(const xunet_srn_store* store, const long long* step_dev, unsigned long long seed, int j, int k, int rank,
                    int world, int B, const float* sqrt_ac, const float* sqrt_1mac, float p_uncond, const float* snr_weight,
                    const xunet_batch* out, float* noise, float* loss_weight, int* idx_out, int* t_out, void* stream);

/* xunet_srn_batch for v-prediction: the same draws and outputs, plus v_out (device, B*S*S*3 floats, required) = the v target of
 * the drawn target views, exactly as xunet_forward_diffusion_v computes it, stored in the same pass.  noise may be NULL (the
 * noise is then not stored), so a training step passes its regression-target buffer as v_out.  Same errors (a NULL v_out
 * in place of a NULL noise); one launch, graph-capturable. */
int xunet_srn_batch_v(const xunet_srn_store* store, const long long* step_dev, unsigned long long seed, int j, int k, int rank,
                      int world, int B, const float* sqrt_ac, const float* sqrt_1mac, float p_uncond, const float* snr_weight,
                      const xunet_batch* out, float* noise, float* v_out, float* loss_weight, int* idx_out, int* t_out,
                      void* stream);

/* xunet_srn_batch for PROGRESSIVE DISTILLATION (Salimans & Ho 2022): the same draws (pairs, poses, K, diffusion seed, noise,
 * z, logsnr of the drawn timestep; z bit for bit as xunet_srn_batch) except
 *   m_b = (the sample hash that xunet_srn_batch draws t from) mod n_grid,   t_b = grid_t[m_b]     (grid_t: device int32, n_grid
 *   entries, the student's timesteps in loop order);   out->cond_mask[b] = 1;   no regression target is stored;
 * and in the same pass the sample's x, z, logsnr, R1, t1, R2, t2, K go to teacher row c*B + b for c < teacher_copies (2: a
 * guided teacher's [cond ; uncond] batch, whose cond_mask the caller sets once; 1: an unguided teacher), m_b to m_out (device,
 * B int32), and idx_out / t_out as in xunet_srn_batch when given.  teacher->cond_mask and ->rays are ignored.  Errors: those of
 * xunet_srn_batch, a NULL grid_t / teacher / m_out / teacher row pointer, n_grid < 1, teacher_copies not 1 or 2.  One launch;
 * no atomics, no allocation, graph-capturable. */
int xunet_srn_batch_distill(const xunet_srn_store* store, const long long* step_dev, unsigned long long seed, int j, int k,
                            int rank, int world, int B, const float* sqrt_ac, const float* sqrt_1mac, const int* grid_t,
                            int n_grid, const xunet_batch* out, const xunet_batch* teacher, int teacher_copies, int* m_out,
                            int* idx_out, int* t_out, void* stream);

/* The teacher's first DDIM step of a distillation sample.  teacher_table: device (2N, 8) floats, the teacher's DDIM (eta = 0)
 * sampler table on its 2N-step grid with log-SNR lag off (sampling.sampler_table); m_dev: device (B) int32 from
 * xunet_srn_batch_distill.  Element i of sample b (per = S*S*3 values each, n = B*per) applies row r = 2 m_b exactly as
 * xunet_sampler_step_table at pos = r does (fp32, as nvcc contracts it, sigma = 0):
 *   out = (1+w) out_c - w out_u (teacher_copies = 2: out_t = [out_c ; out_u], 2n floats) or out_c (teacher_copies = 1, w unused);
 *   x0 = clip(c_recip z - c_recipm1 out, -1, 1);   z' = c_x0 x0 + c_z z,
 * reading z from teacher->z and writing z' to every copy of it, and row r's column 5 (the log-SNR of the next teacher timestep)
 * to every copy of teacher->logsnr.  Errors: a NULL pointer, B < 1, per < 1, teacher_copies not 1 or 2.  One launch. */
int xunet_distill_teacher_step(const float* out_t, float w, int teacher_copies, const float* teacher_table, const int* m_dev,
                               int B, long long per, const xunet_batch* teacher, void* stream);

/* The distillation target: the teacher's second step, row r = 2 m_b + 1, from its second output out_t and teacher_z (z' of
 * xunet_distill_teacher_step, first copy), to z'' as above; then, with target_table (device (N, 4) floats) row m_b =
 * {c_a, c_b, alpha_t, sigma_t}, c_a = 1 / (alpha'' - (sigma''/sigma_t) alpha_t), c_b = (sigma''/sigma_t) c_a (fp64, rounded once):
 *   x~ = __fsub_rn(__fmul_rn(c_a, z''), __fmul_rn(c_b, z_t));   v = __fdiv_rn(__fsub_rn(__fmul_rn(alpha_t, z_t), x~), sigma_t)
 * stored to v_out (device, n floats: the student slot's regression target).  z_t: the student's z input.  A student DDIM step
 * from z_t whose v output is v lands on z''.  Errors: a NULL pointer, B < 1, per < 1, teacher_copies not 1 or 2.  One launch. */
int xunet_distill_target(const float* out_t, float w, int teacher_copies, const float* teacher_table, const float* target_table,
                         const int* m_dev, const float* z_t, const float* teacher_z, int B, long long per, float* v_out,
                         void* stream);

/* The teacher step of CONSISTENCY DISTILLATION (Song et al. 2023, Consistency Models, Alg. 2; guided as in LCM).  The teacher
 * grid G holds N timesteps in loop order; sample b sits at position n = m_b (m_dev: device (B) int32 from
 * xunet_srn_batch_distill with grid_t = G, n_grid = N).  teacher_table: device (N, 8) floats, the teacher's DDIM (eta = 0)
 * sampler table on G with log-SNR lag off (sampling.sampler_table), its last row going to alpha-bar 1.  Element i of sample b
 * (per = S*S*3 values each, n = B*per) applies row r = m_b exactly as xunet_sampler_step_table at pos = r does (fp32, as nvcc
 * contracts it, sigma = 0):
 *   out = (1+w) out_c - w out_u (teacher_copies = 2: out_t = [out_c ; out_u], 2n floats) or out_c (teacher_copies = 1, w unused);
 *   x0 = clip(c_recip z_t - c_recipm1 out, -1, 1);   z^ = c_x0 x0 + c_z z_t,
 * reading z_t (device, n floats: the sample's z) and writing z^ to z_out (device, n floats: the target batch's z, not the
 * teacher's), and row r's column 5 (the log-SNR of t_{r+1}) to logsnr_out[b] (device, B floats).  On the last row z^ is the
 * teacher's clipped x0.  Errors: a NULL pointer, B < 1, per < 1, teacher_copies not 1 or 2.  One launch; graph-capturable. */
int xunet_cd_teacher_step(const float* out_t, float w, int teacher_copies, const float* teacher_table, const int* m_dev, int B,
                          long long per, const float* z_t, float* z_out, float* logsnr_out, void* stream);

/* The consistency-distillation target.  v_minus: device (n floats), the output of the target network (the student's current
 * weights, no dropout, cond_mask 1) at (z^, log-SNR(t_{n+1})); target_table: device (N, 4) floats, row n = {a, b, alpha_n,
 * sigma_n} with a = alpha_{n+1}, b = sigma_{n+1} and (a, b) = (1, 0) on the last row (fp64, rounded once); z_t, z_hat: the
 * sample's z and xunet_cd_teacher_step's z^.  Element i of sample b, with row m_b:
 *   x0- = clip(a z^ - b v-, -1, 1)     (the sampler's x0 expression, as nvcc contracts it: clip(fma(a, z^, -(b v-))))
 *   v*  = __fdiv_rn(__fsub_rn(__fmul_rn(alpha_n, z_t), x0-), sigma_n)
 * stored to v_out (device, n floats: the student slot's regression target).  A student whose v output is v* has the consistency
 * function f(z_t, t_n) = alpha_n z_t - sigma_n v* = x0-; on the last row x0- = z^.  Errors: a NULL pointer, B < 1, per < 1.
 * One launch; graph-capturable. */
int xunet_cd_target(const float* v_minus, const float* target_table, const int* m_dev, const float* z_t, const float* z_hat,
                    int B, long long per, float* v_out, void* stream);

/* The dropout keep-mask the kernels use for residual-block `op_index` (0/1 floats, device), so tests can
 * hand the identical mask to the oracle (nn.Dropout, model/xunet.py:84). */
int xunet_dropout_mask(float* mask_out, long long n, int op_index, unsigned long long seed, float rate,
                       void* stream);

/* Image-quality metrics of generated views against ground truth (3DiM reports PSNR and SSIM on SRN).
 * pred, target: device (B, S, S, 3) fp32 NHWC in [-1, 1] (the sampler's output convention).  Each value is mapped to
 * u = clamp((v + 1) / 2, 0, 1); then, per image b:
 *   mse_out[b]  = mean over the S*S*3 values of (u_pred - u_target)^2;
 *   psnr_out[b] = -10 log10(mse_b)  (data range 1; +inf when mse_b == 0);
 *   ssim_out[b] = SSIM of Wang et al. 2004 with an 11x11 Gaussian window: 1-D weights exp(-i^2 / (2 * 1.5^2)), i = -5..5,
 *                 normalised to sum 1, their outer product in 2-D.  Per channel, at each of the (S-10)^2 pixels whose window
 *                 lies inside the image (no padding), with the window-weighted (population) moments mu_p, mu_t, sp2, st2, spt:
 *                   s = (2 mu_p mu_t + C1)(2 spt + C2) / ((mu_p^2 + mu_t^2 + C1)(sp2 + st2 + C2)),  C1 = 0.01^2, C2 = 0.03^2;
 *                 ssim_b is the mean of s over the 3 channels and those pixels.  This equals skimage's
 *                 structural_similarity(channel_axis=-1, data_range=1, gaussian_weights=True, sigma=1.5,
 *                 use_sample_covariance=False).
 * mse_out, psnr_out, ssim_out: device, B floats each.  Moments and sums are fp64, reduced in an order fixed by S alone (one CTA
 * per image, no atomics), so an image's three values have the same bits alone or at any position of any batch.  One launch; no
 * allocation, no host sync, graph-capturable.  Errors: a NULL pointer, B < 1, S < 11 or S > XUNET_METRICS_MAX_SIDE (the
 * shared-memory ring of filtered rows is sized for it). */
#define XUNET_METRICS_MAX_SIDE 256
int xunet_image_metrics(const float* pred, const float* target, int B, int S, float* mse_out, float* psnr_out,
                        float* ssim_out, void* stream);

/* Radiance grid of the 3D consistency score (3DiM, Watson et al. 2022, section 5: fit a field to some generated views, render
 * it at the poses of the others, score the renders).  The field:
 *   grid  fp32 (G, G, G, 4) channels-last, indexed [ix][iy][iz][c]; c = 0 raw density, c = 1..3 raw colour.  Grid point
 *         (ix, iy, iz) sits at world position -b + 2b (ix, iy, iz) / (G - 1): the cube [-b, b]^3, b = bound.  Inside it the raw
 *         vector is the trilinear interpolation of the 8 surrounding grid points; the activations come after:
 *         sigma = softplus(raw_0 + XUNET_FIELD_DENSITY_SHIFT) (an all-zero grid is nearly transparent), colour =
 *         sigmoid(raw_1..3) in [0, 1].  No view dependence: colour is a function of position only, so the field cannot explain
 *         views that disagree as view-dependent appearance.
 *   rays  pixel (row, col) of view v starts at t_v with direction normalize(R_v K_v^-1 (col + 1/2, row + 1/2, 1)): convention 1
 *         (XUNET_RAYS_OPENCV_UV), SRN's camera model -- whatever ray convention a checkpoint was trained with.  R (V, 3, 3)
 *         camera-to-world, t (V, 3), K (V, 3, 3), row-major.
 *   samples  the ray's segment inside the cube, clipped to t >= near, of length L (empty: the pixel is the background) is cut
 *         into n = ceil(L / step) pieces of length step, the last one shortened so that the lengths d_k sum to L; piece k is
 *         sampled at its midpoint.  No early termination.
 *   compositing  a_k = 1 - exp(-sigma_k d_k), T_0 = 1, T_{k+1} = T_k (1 - a_k); C = sum_k T_k a_k c_k + T_n bg with
 *         bg = (background + 1) / 2; the pixel is 2C - 1 (the sampler's [-1, 1]).
 * Limits: XUNET_FIELD_MIN_GRID <= G <= XUNET_FIELD_MAX_GRID, 0 < bound <= XUNET_FIELD_MAX_BOUND, near >= 0, step > 0 with
 * ceil(2 sqrt(3) bound / step) <= XUNET_FIELD_MAX_SAMPLES samples on the longest chord, V >= 1, S >= 1, V S S < 2^31.
 * Every entry checks its arguments before it launches anything (message starting with the entry's name); no allocation, no
 * host sync, graph-capturable.  kinv: device scratch of V * 9 floats (receives K^-1). */
#define XUNET_FIELD_DENSITY_SHIFT (-6.0f)
#define XUNET_FIELD_MIN_GRID 2
#define XUNET_FIELD_MAX_GRID 256
#define XUNET_FIELD_MAX_BOUND 64.0f
#define XUNET_FIELD_MAX_SAMPLES 4096
#define XUNET_FIELD_MAX_RAYS (1 << 20)
#define XUNET_FIELD_FIXED_ONE 4294967296.0   /* 2^32: one unit of the fixed-point gradient sums */
#define XUNET_FIELD_MAX_GRAD_L1 8388608.0    /* 2^23: the sum of |dC| over the values xunet_field_image_grad scatters */
/* Renders V views: out (V, S, S, 3) in [-1, 1].  Each pixel is composited by one thread on its own, so a view has the same bits
 * alone or anywhere in a batch. */
int xunet_field_render(const float* grid, int G, float bound, const float* R, const float* t, const float* K, float* kinv, int V,
                       int S, float near, float step, float background, float* out, void* stream);
/* One iteration's loss and gradient.  views (V, S, S, 3) in [-1, 1] are the training pixels, u = clamp((view + 1) / 2, 0, 1).
 * With i = *iter_dev (device int64, the Adam count of the update this gradient feeds, 1-based), ray r < rays is pixel
 *     xu_mix64(seed * 0x9E3779B97F4A7C15 + i * 0xD1B54A32D192ED03 + r) mod (V S S)      (index v S S + row S + col)
 * (drawn with replacement), and the loss is (1 / 3N) sum_r sum_ch (C - u)^2 (N = rays) plus the total variation
 *     tv_density / G^3 sum_axes sum (D raw_0)^2 + tv_color / G^3 sum_axes sum_{c=1..3} (D raw_c)^2   (D: forward difference).
 * grad (G, G, G, 4) receives the gradient of that loss w.r.t. the raw grid, and loss_out[i - 1] (when 1 <= i <= loss_len) the
 * data term alone, the mean squared error of the drawn pixels in [0, 1] units.
 * Determinism: each sample's gradient contribution to each corner word is rounded to a multiple of 1 / XUNET_FIELD_FIXED_ONE
 * and the contributions, and each ray's squared error, are summed as int64 with integer atomics in acc (4 G^3 + 1 words, all
 * zero on entry; the call leaves them zero), so grad and loss have the same bits on every run and every GPU.  No overflow:
 * per ray and word, |dL/dC| <= 2 per channel; the colour words add g_ch T_k a_k c(1 - c) w, at most 2 * 1/4 over the ray
 * (sum_k T_k a_k <= 1, w <= 1); the density word adds sum_ch g_ch d_k (T_{k+1} c_k - R_{k+1}) sigmoid(.) w, at most
 * 3 * 2 * L <= 12 sqrt(3) XUNET_FIELD_MAX_BOUND < 1331 (|T_{k+1} c_k - R_{k+1}| <= T_{k+1} <= 1, sum_k d_k = L), plus half a
 * unit of rounding per sample and corner; a ray's squared error is at most 3.  Over XUNET_FIELD_MAX_RAYS = 2^20 rays every
 * sum stays below 1331 * 2^20 + 2^20 * 2^12 * 2^-33 < 2^31 in magnitude, i.e. below 2^63 in fixed point.
 * Three launches: K^-1, the rays, and one finish pass (fixed-point to fp32, the TV stencil, the loss, clearing acc). */
int xunet_field_loss_grad(const float* grid, int G, float bound, const float* views, const float* R, const float* t,
                          const float* K, float* kinv, int V, int S, float near, float step, float background, int rays,
                          const long long* iter_dev, unsigned long long seed, float tv_density, float tv_color, long long* acc,
                          float* grad, float* loss_out, long long loss_len, void* stream);
/* The backward of a given image gradient, over every pixel of V views: with dC (V, S, S, 3) the gradient of some loss w.r.t. the
 * composited colours C (not the pixels 2C - 1) in units of `unit` (the gradient is unit dC), grad (G, G, G, 4) receives
 *     unit d/d(raw grid) [ sum_pixels sum_ch dC_ch C_ch ]  +  the total-variation gradient of xunet_field_loss_grad.
 * A non-finite value of dC is read as 0; a pixel whose three values are 0 is skipped.  The march, the fixed-point scatter, the
 * per-cell register flush and the finish pass are those of xunet_field_loss_grad (one __device__ backward serves both); the
 * finish pass multiplies the sums by unit / XUNET_FIELD_FIXED_ONE.  The unit lets a caller whose gradient is a mean over many
 * values (a few 1e-6 per value) scatter values of order 1, so that a sample's contribution, which can be a few 1e-5 of its
 * value on a nearly empty grid, stays far above the fixed-point quantum 2^-32.
 * No overflow, given sum |dC| <= XUNET_FIELD_MAX_GRAD_L1 = 2^23 over all values (the caller's condition; xunet_lift_grad's
 * output meets it): per ray and word, a colour word adds sum_k dC_ch T_k a_k c(1 - c) w, at most |dC_ch| / 4, and the density
 * word adds sum_ch dC_ch sum_k d_k (T_{k+1} c_k - R_{k+1}) sigmoid(.) w, at most L sum_ch |dC_ch| with L <= 2 sqrt(3)
 * XUNET_FIELD_MAX_BOUND < 222.  Summed over the rays that is below 222 * 2^23 < 1.87e9, plus half a unit of rounding per
 * sample and corner, at most 2^20 rays * 2^12 samples * 2^-33 = 1/2: below 2^31 in magnitude, i.e. below 2^63 in fixed point.
 * acc: 4 G^3 + 1 int64 words, zero on entry and on return (the last word is unused).  Errors: those of xunet_field_render,
 * V S S > XUNET_FIELD_MAX_RAYS, unit not finite or not > 0, tv weights negative or not finite.  Three launches: K^-1, the
 * pixels, and the finish pass. */
int xunet_field_image_grad(const float* grid, int G, float bound, const float* dC, double unit, const float* R, const float* t,
                           const float* K, float* kinv, int V, int S, float near, float step, float background, float tv_density,
                           float tv_color, long long* acc, float* grad, void* stream);

/* Pose estimation by descent on the denoising loss (ID-Pose / iFusion style): given a conditioning view x at a known camera and a
 * target view y (S, S, 3), H pose hypotheses for y's camera are fitted side by side, each seeing P noise draws per iteration.
 * Row b = h P + p of the engine batch (B = H P) is hypothesis h with draw p; n = 3 S^2 values per view.  One iteration is
 *   xunet_pose_draw -> xunet_forward (train = 0) -> xunet_pose_loss -> xunet_backward_vjp_inputs (dR2, dt2)
 *   -> xunet_pose_tangent -> xunet_adam_step on the step buffer -> xunet_pose_retract -> the count + 1.
 * The master poses are fp64 on the device: R (H, 3, 3) cam-to-world, row-major, and t (H, 3).  The tangent coordinates of
 * hypothesis h are (omega, delta): R' = exp([omega]x) R, t' = exp([omega]x) t + delta, a rotation of the camera about the world
 * origin (the object's centre in SRN) plus, with translate != 0, a translation; D = 3 (translate = 0) or 6 values per
 * hypothesis.  i = *iter_dev is the 1-based Adam count (device int64), read at execution time so a replayed graph draws afresh.
 * Every entry checks its arguments before it launches anything (message starting with the entry's name); no allocation, no
 * atomics, no host sync, graph-capturable; the results are functions of the inputs alone (fixed bits). */
#define XUNET_POSE_MAX_T 999                /* timesteps index the 1000-entry cosine-beta tables */
#define XUNET_POSE_LOSS_CHUNK 4096          /* values per partial sum of xunet_pose_loss */
#define XUNET_POSE_SMALL_ANGLE2 1e-6        /* |omega|^2 below which xunet_pose_retract uses the Taylor series */
/* The draws of iteration i: draw p has the hash h_p = xu_mix64(seed * 0x9E3779B97F4A7C15 + i * 0xD1B54A32D192ED03 + p) and
 *   t_p = t_min + h_p mod (t_max - t_min + 1)                                   (strata == 0: uniform)
 *   t_p = t_min + floor((2g + 1)(t_max - t_min + 1) / (2 strata)),  g = ((i - 1) P + p) mod strata     (strata > 0: stratified)
 *   eps_p[k] = the device hash normal of draw k of seed h_p (the sampler's noise, csrc/common.cuh xu_hash_normal).
 * Every hypothesis shares draw p (common random numbers).  Written: z rows (B, S, S, 3), z_b[k] = fma(sa, y[k], fl(sb eps_p[k]))
 * with sa = sqrt_ac[t_p], sb = sqrt_1mac[t_p] (xunet_forward_diffusion's rounding); logsnr (B) = logsnr_schedule_cosine(t_p / 1000)
 * as xunet_forward_diffusion; target (P, S, S, 3) = eps_p (prediction 0) or the v target fl(fl(sa eps) - fl(sb y)) (prediction 1,
 * xunet_forward_diffusion_v's rounding); t_out (P) int32 when not NULL.  Errors: a NULL required pointer, H < 1, P < 1, S < 1,
 * H P S^2 >= 2^31 / 3, 0 <= t_min <= t_max <= XUNET_POSE_MAX_T violated, strata < 0, prediction not 0 / 1.  One launch. */
int xunet_pose_draw(const float* y, int H, int P, int S, int t_min, int t_max, int strata, const long long* iter_dev,
                    unsigned long long seed, const float* sqrt_ac, const float* sqrt_1mac, int prediction, float* z, float* logsnr,
                    float* target, int* t_out, void* stream);
/* The loss of each hypothesis and its seed: with r = fl(out_b - target_p) (out: the forward's output, B rows; target: P rows),
 *   L_h = (1 / (P n)) sum_p sum_k r^2,  d_out_b = fl(fl32(2 / (P n)) r)   (d_out: B rows, the d_eps of the VJP).
 * The squares are summed in fp64: per row, chunks of XUNET_POSE_LOSS_CHUNK values (256 thread sums, a fixed shuffle tree, the 8
 * warp sums in order) into partial (B ceil(n / XUNET_POSE_LOSS_CHUNK) doubles, scratch), then per hypothesis over p and the
 * chunks in order, divided by P n in fp64 and rounded once to fp32 into loss_out[(i - 1) H + h] when 1 <= i <= loss_len.
 * Errors: a NULL pointer, H < 1, P < 1, S < 1, H P S^2 >= 2^31 / 3, loss_len < 0.  Two launches. */
int xunet_pose_loss(const float* out, const float* target, int H, int P, int S, const long long* iter_dev, double* partial,
                    float* d_out, float* loss_out, long long loss_len, void* stream);
/* The gradient in tangent coordinates.  dR (B, 3, 3), dt (B, 3): dL/dR2, dL/dt2 of the rows (xunet_backward_vjp_inputs).  In fp64,
 * G_R = sum_p dR_b and g_t = sum_p dt_b (p ascending), N = G_R R_h^T + g_t t_h^T, and
 *   g_omega = (N32 - N23, N13 - N31, N21 - N12)   (1-based indices),   g_delta = g_t,
 * the derivative of L(exp([omega]x) R_h, exp([omega]x) t_h + delta) at 0.  grad (H, D) receives them rounded to fp32, omega first.
 * Errors: a NULL pointer, H < 1, P < 1, translate not 0 / 1.  One launch. */
int xunet_pose_tangent(const float* dR, const float* dt, int H, int P, const double* R, const double* t, int translate, float* grad,
                       void* stream);
/* The retraction.  step (H, D) fp32 (Adam's update of a zero buffer, i.e. -lr m_hat / (sqrt(v_hat) + eps)) gives omega and delta;
 * in fp64, theta^2 = |omega|^2, A = sin(theta) / theta and B = 2 sin^2(theta / 2) / theta^2 (theta^2 < XUNET_POSE_SMALL_ANGLE2:
 * A = 1 - theta^2 / 6 + theta^4 / 120, B = 1/2 - theta^2 / 24 + theta^4 / 720), E = I + A [omega]x + B (omega omega^T - theta^2 I),
 * R_h <- E R_h, t_h <- E t_h + delta (delta = 0 when translate = 0).  Then R_rows (B, 3, 3) and t_rows (B, 3) of the P rows of
 * hypothesis h receive fp32(R_h), fp32(t_h), and step is zeroed.  A zero step leaves R and t as they are and only writes the rows.
 * Errors: a NULL pointer, H < 1, P < 1, translate not 0 / 1.  One launch. */
int xunet_pose_retract(float* step, int H, int P, int translate, double* R, double* t, float* R_rows, float* t_rows, void* stream);

/* Lifting one view to a radiance grid by score distillation (DreamFusion's SDS, Poole et al. 2022, on a view-conditioned model as
 * in Zero-1-to-3 + SJC and Magic123).  A source view x (S, S, 3) at camera (R1, t1, K) conditions the guided X-UNet; each iteration
 * renders the grid from P drawn cameras around the origin plus the source camera (view P), noises the P renders, runs one forward
 * of the guided batch of 2P rows [cond ; uncond] (row p and row P + p share draw p) and pushes the weighted residual back through
 * the renderer.  n = 3 S^2 values per view; i = *iter_dev is the 1-based Adam count (device int64), read at execution time so a
 * replayed graph draws afresh.  One iteration is
 *   xunet_lift_draw -> xunet_field_render (P + 1 views) -> xunet_lift_noise -> xunet_forward (train = 0, cond_mask [1]*P + [0]*P)
 *   -> xunet_lift_grad -> xunet_field_image_grad (P + 1 views) -> xunet_adam_step on the grid -> the count + 1.
 * Draw p has the hash h_p = xu_mix64((seed ^ XUNET_LIFT_SEED_DOMAIN) 0x9E3779B97F4A7C15 + i 0xD1B54A32D192ED03 + p): the hash of
 * xunet_pose_draw in a seed domain of its own, so a lift and a pose estimate with the same seed draw independently.
 * Every entry checks its arguments before it launches anything (message starting with the entry's name); no allocation, no
 * atomics, no host sync, graph-capturable; the results are functions of the inputs alone (fixed bits). */
#define XUNET_LIFT_SEED_DOMAIN 0x6C6966745F736473ULL   /* "lift_sds" */
#define XUNET_LIFT_MAX_RESIDUAL 16.0f                 /* |eps_hat - eps| per value, clamped */
/* The cameras and timesteps of iteration i, one thread per draw, in fp64 and rounded once to fp32:
 *   t_p = t_min + h_p mod (t_max - t_min + 1);
 *   u_1 = (xu_mix64(h_p + 0x5851F42D4C957F2D) >> 11) 2^-53, u_2 = (xu_mix64(h_p + 0x14057B7EF767814F) >> 11) 2^-53 in [0, 1);
 *   s = sin(elev_lo) + (sin(elev_hi) - sin(elev_lo)) u_1 (the sine of the elevation, uniform: a uniform direction on the band),
 *   phi = 2 pi u_2, c = radius (s up + sqrt(1 - s^2) (cos(phi) e_1 + sin(phi) e_2)), with up = (up_x, up_y, up_z) / |.|,
 *   e_1 = normalize(b - (b . up) up), b the first basis vector of least |up_j|, and e_2 = up x e_1;
 *   the look-at camera at c: f = -c / |c|, right = normalize(f x up), down = f x right, R = [right down f] (columns), and when
 *   |f x up| < 1e-6 (f parallel or nearly parallel to up) right = normalize(e_1 - (e_1 . f) f).  With up = (0, 0, 1) this is
 *   synthetic._look_at: e_1 = (1, 0, 0).
 * Written: R2 (2P, 3, 3) and t2 (2P, 3) rows p and P + p, cam_R (P + 1, 3, 3) and cam_t (P + 1, 3) view p (view P, the source
 * camera, is the caller's), t_out (P) int32.  Errors: a NULL pointer, P < 1, 0 <= t_min <= t_max <= XUNET_POSE_MAX_T violated,
 * up zero or not finite, -pi/2 <= elev_lo <= elev_hi <= pi/2 violated, radius not finite and > 0.  One launch. */
int xunet_lift_draw(int P, int t_min, int t_max, const long long* iter_dev, unsigned long long seed, double up_x, double up_y,
                    double up_z, double elev_lo, double elev_hi, double radius, float* R2, float* t2, float* cam_R, float* cam_t,
                    int* t_out, void* stream);
/* The noise of iteration i, one thread per value of the P drawn views: eps_p[k] = xu_hash_normal(h_p, k), and with
 * sa = sqrt_ac[t_p], sb = sqrt_1mac[t_p] and render (P + 1, S, S, 3) the renders in [-1, 1] (view P is not read),
 *   z rows p and P + p (2P, S, S, 3) = fma(sa, render_p[k], fl(sb eps_p[k]))   (xunet_pose_draw's rounding),
 *   logsnr rows p and P + p = logsnr_schedule_cosine(t_p / 1000), eps (P, S, S, 3) = eps_p.
 * Errors: a NULL pointer, P < 1, S < 1, (P + 1) S^2 > XUNET_FIELD_MAX_RAYS.  One launch. */
int xunet_lift_noise(const float* render, const int* t_draw, int P, int S, const long long* iter_dev, unsigned long long seed,
                     const float* sqrt_ac, const float* sqrt_1mac, float* z, float* logsnr, float* eps, void* stream);
/* The image gradient and the diagnostics.  out (2P, S, S, 3) is the forward's output, z its noisy input rows, eps the noise of
 * xunet_lift_noise, render (P + 1, S, S, 3) the renders (pixel = 2C - 1) and x (S, S, 3) the source view.  Per value k of drawn
 * view p, with sa, sb of t_p:
 *   o_g = (1 + w) out_p - w out_{P+p};  eps_hat = o_g (prediction 0), = sb z_p + sa o_g (prediction 1, v);
 *   r = eps_hat - eps_p, 0 if not finite, clamped to +-XUNET_LIFT_MAX_RESIDUAL;
 *   dC_p[k] = fl32(2 sds_weight omega_t / (3 S^2 P unit)) r,  omega_t = 1 - abar_t = sb^2 in fp64  (the pixel is 2C - 1);
 * and per value of the source view, with C = (render_P + 1) / 2 and u = clamp((x + 1) / 2, 0, 1):
 *   dC_P[k] = fl32(2 recon_weight / (3 S^2 unit)) (C - u),
 * i.e. the gradient w.r.t. C of the loss in units of `unit`, for xunet_field_image_grad with the same unit.  Since |r| <= 16,
 * omega <= 1 and |C - u| <= 1, sum |dC| <= (32 sds_weight + 2 recon_weight) / unit, and the entry refuses a unit that lets this
 * exceed XUNET_FIELD_MAX_GRAD_L1.  lift.grad_unit picks the smallest power of two that meets it, so the values are of order 1
 * (a few 1e-6 before the division at S = 128).  Diagnostics: the squares r^2 and
 (C - u)^2 are summed in fp64 in chunks of XUNET_POSE_LOSS_CHUNK values (256 thread sums, a fixed shuffle tree, the 8 warp sums in
 * order) into partial ((P + 1) ceil(n / XUNET_POSE_LOSS_CHUNK) doubles, scratch), then in order, so that when 1 <= i <= loss_len
 *   sds_out[i - 1] = fp32((1 / (P n)) sum_p sum_k r^2),  loss_out[i - 1] = fp32((1 / n) sum_k (C - u)^2).
 * Errors: a NULL pointer, P < 1, S < 1, (P + 1) S^2 > XUNET_FIELD_MAX_RAYS, w < 0 or not finite, prediction not 0 / 1, weights
 * negative or not finite, unit not finite or not > 0, (32 sds_weight + 2 recon_weight) / unit > XUNET_FIELD_MAX_GRAD_L1,
 * loss_len < 0.  Two launches. */
int xunet_lift_grad(const float* out, const float* z, const float* eps, const float* render, const float* x, const int* t_draw, int P,
                    int S, float w, int prediction, float sds_weight, float recon_weight, double unit, const float* sqrt_ac,
                    const float* sqrt_1mac,
                    const long long* iter_dev, double* partial, float* dC, float* sds_out, float* loss_out, long long loss_len,
                    void* stream);

/* ---- operator-level entry points (parity tests / micro-benchmarks of single kernels) ----
 * dtype as above; tensors channels-last (N,H,W,C). */
int xunet_op_conv(int dtype, int impl, const void* x, const float* w, const float* bias, const void* res, void* y,
                  int N, int Hi, int Wi, int Ci, int Co, int ksize, int stride, int nseg, float alpha, void* stream);
int xunet_op_conv_dgrad(int dtype, int impl, const void* dy, const float* w, void* dx, int N, int Hi, int Wi, int Ci,
                        int Co, int ksize, int stride, int nseg, float alpha, int accumulate, void* stream);
int xunet_op_conv_wgrad(int dtype, int impl, const void* x, const void* dy, float* dw, float* dbias, int N, int Hi, int Wi,
                        int Ci, int Co, int ksize, int stride, int nseg, float alpha, void* stream);
/* qkv: (N, L, 3C) [q | k | v], heads x hd; res/out: (N, L, C); lse: (N, heads, L) fp32. out=(attn+res)/sqrt2 */
int xunet_op_attention(int dtype, int impl, const void* qkv, const void* res, void* out, float* lse, int N, int L, int C,
                       int heads, int cross, void* stream);
/* dscratch: at least N*heads*L floats of scratch, the row dots D = rowsum(dO * O) laid out (N, heads, L); nothing past them
 * is written (a buffer of N*L*(heads + C) floats, the size earlier versions needed, still works).  impl=1 needs lse and
 * dscratch 16-byte aligned.  With XUNET_OP_ATTN_FOLD=1 in the environment the caller promises an all-zero dscratch and gets
 * it back all-zero (one extra memset of the D rows). */
int xunet_op_attention_bwd(int dtype, int impl, const void* qkv, const void* res, const void* out, const void* dout,
                           const float* lse, float* dscratch, void* dqkv, int N, int L, int C, int heads, int cross,
                           void* stream);

/* ---- operator-level entry points of the GroupNorm path: each runs the launch the engine runs for that stage ----
 * GroupNorm(32) pools each group over both frames of a sample: samples are frame pairs (2b, 2b+1), so N is even, and the
 * per-sample tables below have N/2 rows.  C (the normalised channels) is a multiple of 32.  cstats / bcs tables are
 * (N/2, C, 2) fp32, stats / bstats (N/2, 32, 2) fp32, params (N/2, C) float4.  Every entry checks its arguments and returns
 * non-zero (xunet_last_error()) before launching anything. */
#define XUNET_GN_PLAIN 0   /* y = yhat                                   (yhat = (x - mean) * rstd * gamma + beta) */
#define XUNET_GN_SWISH 1   /* y = swish(yhat)                                                                       */
#define XUNET_GN_FILM 2    /* y = dropout(swish(yhat * (1 + scale) + shift)), e = [scale | shift] (N,H,W,2C)       */
#define XUNET_RS_NONE 0
#define XUNET_RS_DOWN 1    /* the activation averaged over 2x2 pixels: output (N, H/2, W/2, C); H, W even          */
#define XUNET_RS_UP 2      /* the activation repeated 2x2 (nearest): output (N, 2H, 2W, C)                          */
/* xunet_op_conv (stride 1, nseg 1) that also ADDS the per-(sample, channel) [sum y, sum y^2] of the stored output y to cstats
 * (N/2, Co, 2): emitted by the tensor-core epilogue where the engine's plan does (impl 1 and every 32-row epilogue slice
 * inside one sample), else by a statistics kernel after the conv. */
int xunet_op_conv_stats(int dtype, int impl, const void* x, const float* w, const float* bias, const void* res, void* y,
                        float* cstats, int N, int H, int W, int Ci, int Co, int ksize, float alpha, void* stream);
/* xunet_op_attention that also ADDS the statistics of out to cstats (N/2, C, 2): the tensor-core forward (impl 1) emits them,
 * the SIMT path runs the statistics kernel after it. */
int xunet_op_attention_stats(int dtype, int impl, const void* qkv, const void* res, void* out, float* lse, float* cstats, int N,
                             int L, int C, int heads, int cross, void* stream);
/* GroupNorm forward from producer-emitted channel statistics: channels [0, ca) of x come with cstats_a (N/2, ca, 2), channels
 * [ca, C) with cstats_b (N/2, C - ca, 2) (a channel concat; cstats_b may be NULL when ca == C).  Writes y, the group sums to
 * stats, and, if params_out is not NULL, the fused backward's table {rstd, -mean*rstd, gamma, beta} (no resampling only).
 * FiLM: e (N,H,W,2C); dropout with keep probability 1 - drop_rate and keep scale 1 / (1 - drop_rate) when train and
 * drop_rate > 0, its mask hashed from (*seed_dev, op_index, element index in (N,H,W,C)) as xunet_dropout_mask does. */
int xunet_op_groupnorm(int dtype, const void* x, const float* cstats_a, const float* cstats_b, int ca, const float* gamma,
                       const float* beta, const void* e, void* y, float* stats, float* params_out, int N, int H, int W, int C,
                       int mode, int resample, float drop_rate, int op_index, const unsigned long long* seed_dev, int train,
                       void* stream);
/* bf16 tensor-core data gradient of a conv (stride 1) whose input is the output of a GroupNorm without resampling, fused with
 * the norm's first backward pass.  dy (N,H,W,Co), w the conv's Flax kernel (ksize^2, C, Co) in nseg segments as in
 * xunet_op_conv; gn_x (N,H,W,C) the norm's input, gn_params its params_out table.  Stores dyh (N,H,W,C), the gradient w.r.t.
 * yhat: alpha * (W^T dy) times swish'(yhat) (SWISH), or through FiLM, dropout and swish (FILM: e, and de (N,H,W,2C) receives
 * [du * yhat | du], du the gradient w.r.t. the swish input), and ADDS [sum dyh * xhat, sum dyh] per (sample, channel) to bcs
 * (N/2, C, 2).  The shape must be one whose 32-row epilogue slices stay inside one sample. */
int xunet_op_conv_dgrad_groupnorm(int dtype, const void* dy, const float* w, const void* gn_x, const float* gn_params, int mode,
                                  const void* e, void* de, float drop_rate, int op_index, const unsigned long long* seed_dev,
                                  int train, void* dyh, float* bcs, int N, int H, int W, int C, int Co, int ksize, int nseg,
                                  float alpha, void* stream);
/* GroupNorm backward.  x, e, gamma, beta, stats as in the forward; dx = rstd (gamma dyh - S1/cnt - xhat S2/cnt) with
 * S1 = sum_group gamma dyh, S2 = sum_group gamma dyh xhat, cnt = 2 H W C/32, plus extra_alpha * extra (N,H,W,C) when extra is
 * not NULL; accumulate: dx += instead of =.  dgamma += sum dyh xhat, dbeta += sum dyh.
 * bcs != NULL (no resampling): the fused second pass after xunet_op_conv_dgrad_groupnorm, dy holds dyh and bcs its sums.
 * bcs == NULL: the two-kernel backward from dy, the gradient of the norm's output (N,Ho,Wo,C); bstats receives the group sums
 * [S1, S2], and a FiLM norm writes (de_accumulate: adds) its gradient to de. */
int xunet_op_groupnorm_bwd(int dtype, const void* x, const void* e, const void* dy, void* dx, void* de, const float* gamma,
                           const float* beta, float* dgamma, float* dbeta, const float* stats, float* bstats, const float* bcs,
                           const void* extra, float extra_alpha, int N, int H, int W, int C, int mode, int resample,
                           float drop_rate, int op_index, const unsigned long long* seed_dev, int train, int accumulate,
                           int de_accumulate, void* stream);

/* ---- operator-level entry points of the conditioning, resampling, concat and loss launches: each runs the launches the
 * engine runs for that op and nothing else, and checks its arguments before launching anything.  fp32 unless dtype says. */
/* log-SNR MLP (B samples, E = emb_ch): pe = posenc_ddpm(1000 * 2 atan(exp(-clip(logsnr, +-20) / 2)) / pi) (B, E),
 * h1 = pe w0 + b0, lemb = swish(h1) w1 + b1; w (E, E) row-major (Flax Dense kernel), b (E). */
int xunet_op_logsnr_emb(const float* logsnr, const float* w0, const float* b0, const float* w1, const float* b1, float* pe, float* h1,
                        float* lemb, int B, int E, void* stream);
/* its backward from dlemb: dh1 = swish'(h1) (dlemb w1^T); dw1 = swish(h1)^T dlemb, db1 = sum_b dlemb, dw0 = pe^T dh1,
 * db0 = sum_b dh1, stored (accumulate: added). */
int xunet_op_logsnr_emb_bwd(const float* dlemb, const float* w1, const float* pe, const float* h1, float* dh1, float* dw0, float* db0,
                            float* dw1, float* db1, int B, int E, int accumulate, void* stream);
/* pose embedding out (2B, S, S, 144) of dtype: per frame [posenc_nerf(ray origin, 15) | posenc_nerf(ray direction, 8)],
 * zero where cond_mask[b] == 0, plus pos_emb (S, S, 144) and ref_first / ref_other (144) when given.  Generated rays
 * (rays == NULL): kinv (B, 9) receives K^-1 and the directions are normalize(R K^-1 p), p per convention (XUNET_RAYS_*);
 * else rays (B, 2, S, S, 6) as in xunet_batch. */
int xunet_op_pose_emb(int dtype, const float* R1, const float* t1, const float* R2, const float* t2, const float* K,
                      const float* cond_mask, const float* pos_emb, const float* ref_first, const float* ref_other, float* kinv,
                      void* out, int B, int S, int convention, const float* rays, void* stream);
/* its parameter gradients from dpose (2B, S, S, 144): dpos_emb = sum over both frames of every sample (stored; accumulate:
 * added; may be NULL), dref_first / dref_other += the sums over frames 0 / 1 (both NULL or both given). */
int xunet_op_pose_emb_bwd(int dtype, const void* dpose, float* dpos_emb, float* dref_first, float* dref_other, int B, int S,
                          int accumulate, void* stream);
/* semb = swish(lemb[n / 2] + pe) over pe (N, HW, E) of dtype, N = 2B. */
int xunet_op_film_emb(int dtype, const float* lemb, const void* pe, void* semb, int N, int HW, int E, void* stream);
/* its backward: dz = dsemb swish'(lemb + pe); dpe = dz when write_dpe; dlemb (B, E) += the sum of dz over both frames. */
int xunet_op_film_emb_bwd(int dtype, const float* lemb, const void* pe, const void* dsemb, void* dpe, float* dlemb, int N, int HW,
                          int E, int write_dpe, void* stream);
/* y = scale * (pool ? the 2x2 sum of x : x repeated 2x2) (+ y when accumulate), x (N, H, W, C) of dtype, C a multiple of 4. */
int xunet_op_resample(int dtype, const void* x, void* y, int N, int H, int W, int C, int pool, float scale, int accumulate,
                      void* stream);
/* dst[p, dst_off + c] = src[p, src_off + c] (+ dst when accumulate) for c < Cc, p < npix; src rows of Cs, dst rows of Cd channels.
 * Every channel count and offset a multiple of 4. */
int xunet_op_copy_channels(int dtype, const void* src, void* dst, long long npix, int Cs, int Cd, int src_off, int dst_off, int Cc,
                           int accumulate, void* stream);
/* dst = alpha src (+ dst when accumulate) over n elements of dtype, n a multiple of 4. */
int xunet_op_scale_add(int dtype, const void* src, void* dst, long long n, float alpha, int accumulate, void* stream);
/* loss = ||eps - noise|| over (B, S, S, 3) fp32; sumsq (1 float) receives the sum of squares, loss (1 float) the loss, and
 * dO (2B, S, S, 3) of dtype the output gradient: frame 1 of sample b = (eps[b] - noise[b]) / loss (0 when loss == 0), frame 0 = 0. */
int xunet_op_loss(int dtype, const float* eps, const float* noise, float* sumsq, float* loss, void* dO, int B, int S, void* stream);

#ifdef __cplusplus
}
#endif
#endif
