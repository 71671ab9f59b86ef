// common.cuh -- shared device helpers for the X-UNet sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdlib.h>

#define XU_RSQRT2 0.70710678118654752440f
#define XU_SQRT2 1.41421356237309504880f
#define XU_GN_EPS 1e-6f
#define XU_GROUPS 32
#define XU_POSE_DIM 144

typedef __nv_bfloat16 bf16;

template <typename T> __device__ __forceinline__ float ldf(const T* p);
template <> __device__ __forceinline__ float ldf<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ldf<bf16>(const bf16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void stf(T* p, float v);
template <> __device__ __forceinline__ void stf<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void stf<bf16>(bf16* p, float v) { *p = __float2bfloat16_rn(v); }

// 4-wide vector load/store (16 B for fp32, 8 B for bf16); pointers must be aligned accordingly.
template <typename T> struct Vec4;
template <> struct Vec4<float> {
  static __device__ __forceinline__ void ld(const float* p, float (&v)[4]) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
  static __device__ __forceinline__ void st(float* p, const float (&v)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
  // read-only (non-coherent) path: lets the compiler hoist the load above unrelated stores -> loads of several
  // pixels in flight per thread
  static __device__ __forceinline__ void ldg(const float* p, float (&v)[4]) {
    float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
  // split load / unpack so that a thread can put several loads in flight before touching any result
  typedef float4 raw;
  static __device__ __forceinline__ raw ldg_raw(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
  static __device__ __forceinline__ void unpack(const raw& t, float (&v)[4]) { v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
};
template <> struct Vec4<bf16> {
  static __device__ __forceinline__ void ld(const bf16* p, float (&v)[4]) {
    uint2 t = *reinterpret_cast<const uint2*>(p);
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&t.x);
    __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&t.y);
    v[0] = __low2float(a); v[1] = __high2float(a); v[2] = __low2float(b); v[3] = __high2float(b);
  }
  static __device__ __forceinline__ void ldg(const bf16* p, float (&v)[4]) {
    uint2 t = __ldg(reinterpret_cast<const uint2*>(p));
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&t.x);
    __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&t.y);
    v[0] = __low2float(a); v[1] = __high2float(a); v[2] = __low2float(b); v[3] = __high2float(b);
  }
  typedef uint2 raw;
  static __device__ __forceinline__ raw ldg_raw(const bf16* p) { return __ldg(reinterpret_cast<const uint2*>(p)); }
  static __device__ __forceinline__ void unpack(const raw& t, float (&v)[4]) {
    v[0] = __uint_as_float(t.x << 16); v[1] = __uint_as_float(t.x & 0xFFFF0000u);
    v[2] = __uint_as_float(t.y << 16); v[3] = __uint_as_float(t.y & 0xFFFF0000u);
  }
  static __device__ __forceinline__ void st(bf16* p, const float (&v)[4]) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]);
    __nv_bfloat162 b = __floats2bfloat162_rn(v[2], v[3]);
    uint2 t;
    t.x = *reinterpret_cast<uint32_t*>(&a);
    t.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = t;
  }
};

// VW-wide vectors with 16-byte accesses for both dtypes: VecW<float> = 4 floats, VecW<bf16> = 8 bf16 (128-bit loads / stores)
template <typename T> struct VecW;
template <> struct VecW<float> {
  static constexpr int W = 4;
  typedef float4 raw;
  static __device__ __forceinline__ raw ldg(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
  static __device__ __forceinline__ raw ld(const float* p) { return *reinterpret_cast<const float4*>(p); }
  static __device__ __forceinline__ void unpack(const raw& t, float (&v)[4]) { v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
  static __device__ __forceinline__ void st(float* p, const float (&v)[4]) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
};
template <> struct VecW<bf16> {
  static constexpr int W = 8;
  typedef uint4 raw;
  static __device__ __forceinline__ raw ldg(const bf16* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
  static __device__ __forceinline__ raw ld(const bf16* p) { return *reinterpret_cast<const uint4*>(p); }
  static __device__ __forceinline__ void unpack(const raw& t, float (&v)[8]) {
    v[0] = __uint_as_float(t.x << 16); v[1] = __uint_as_float(t.x & 0xFFFF0000u);
    v[2] = __uint_as_float(t.y << 16); v[3] = __uint_as_float(t.y & 0xFFFF0000u);
    v[4] = __uint_as_float(t.z << 16); v[5] = __uint_as_float(t.z & 0xFFFF0000u);
    v[6] = __uint_as_float(t.w << 16); v[7] = __uint_as_float(t.w & 0xFFFF0000u);
  }
  static __device__ __forceinline__ void st(bf16* p, const float (&v)[8]) {
    uint4 t;
    __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
    __nv_bfloat162 c = __floats2bfloat162_rn(v[4], v[5]), d = __floats2bfloat162_rn(v[6], v[7]);
    t.x = *reinterpret_cast<uint32_t*>(&a); t.y = *reinterpret_cast<uint32_t*>(&b);
    t.z = *reinterpret_cast<uint32_t*>(&c); t.w = *reinterpret_cast<uint32_t*>(&d);
    *reinterpret_cast<uint4*>(p) = t;
  }
};

__device__ __forceinline__ float sigmoidf_(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }   // 2-ulp fast divide
__device__ __forceinline__ float swishf_(float x) { return x * sigmoidf_(x); }
// d/dx [x sigmoid(x)]
__device__ __forceinline__ float swish_gradf_(float x) {
  float s = sigmoidf_(x);
  return s * (1.f + x * (1.f - s));
}

// Dropout keep decision shared by forward, backward and xunet_dropout_mask (tests replicate it in numpy).
__host__ __device__ __forceinline__ uint64_t xu_mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
// Standard normal draw i of `seed`: Box-Muller on two hashed 24-bit uniforms (the device noise of the sampler and of the
// forward diffusion).
__device__ __forceinline__ float xu_hash_normal(uint64_t seed, uint64_t i) {
  const uint64_t h1 = xu_mix64(seed * 0x9E3779B97F4A7C15ULL + 2ULL * i + 1ULL);
  const uint64_t h2 = xu_mix64(h1 + 0xD1B54A32D192ED03ULL);
  const float u1 = ((float)(h1 >> 40) + 1.f) * (1.0f / 16777216.0f);
  const float u2 = (float)(h2 >> 40) * (1.0f / 16777216.0f);
  return sqrtf(-2.f * logf(u1)) * cosf(6.28318530717958647692f * u2);
}
// ---- forward diffusion (dataset/data_loader.py:92-110), shared by xunet_forward_diffusion and xunet_srn_batch ----------
// Per-sample hash of sample b under `seed`: it draws the timestep and the cond_mask uniform.
__device__ __forceinline__ uint64_t xu_fd_sample_hash(uint64_t seed, int b) {
  return xu_mix64(seed * 0x9E3779B97F4A7C15ULL + 0xABCDEF0123ULL + (uint64_t)b);
}
__device__ __forceinline__ int xu_fd_timestep(uint64_t hb) { return (int)(hb % 1000ULL); }
// logsnr_schedule_cosine(t/1000), logsnr_min=-20, logsnr_max=20 (data_loader.py:94-97), in double like the reference
__device__ __forceinline__ float xu_fd_logsnr(int t) {
  const double bb = atan(exp(-10.0)), aa = atan(exp(10.0)) - bb;
  return (float)(-2.0 * log(tan(aa * ((double)t / 1000.0) + bb)));
}
__device__ __forceinline__ float xu_fd_cond_mask(uint64_t hb, float p_uncond) {
  const float u = (float)(xu_mix64(hb + 0x51ED27ULL) >> 40) * (1.0f / 16777216.0f);
  return u > p_uncond ? 1.f : 0.f;
}
// z of one element: sqrt(abar_t) x0 + sqrt(1 - abar_t) noise
__device__ __forceinline__ float xu_fd_z(float sa, float x0, float sb, float nz) { return sa * x0 + sb * nz; }
// xu_fd_z with its rounding spelled out, for the v-target kernels, whose z must equal the eps kernels' bit for bit: nvcc
// contracts the plain expression to fma(sa, x0, fl(sb noise)) in forward_diffusion_kernel and in the vector path of
// srn_batch_kernel (xu_fd_z_rn), and to fma(sb, noise, fl(sa x0)) in its scalar path (xu_fd_z_rn_scalar)
__device__ __forceinline__ float xu_fd_z_rn(float sa, float x0, float sb, float nz) { return __fmaf_rn(sa, x0, __fmul_rn(sb, nz)); }
__device__ __forceinline__ float xu_fd_z_rn_scalar(float sa, float x0, float sb, float nz) {
  return __fmaf_rn(sb, nz, __fmul_rn(sa, x0));
}
// v target of one element (Salimans & Ho 2022): sqrt(abar_t) noise - sqrt(1 - abar_t) x0, each product and the difference
// rounded once (no contraction), so fp32 numpy restates it bit for bit (diffusion.v_target)
__device__ __forceinline__ float xu_fd_v(float sa, float nz, float sb, float x0) {
  return __fsub_rn(__fmul_rn(sa, nz), __fmul_rn(sb, x0));
}
// what a forward-diffusion producer writes as the regression target: the noise itself, or v in its place / beside it.
// XU_TARGET_DISTILL writes no target: the timestep comes from a distillation grid and the target is made later from the
// teacher's two steps (distill.cu)
enum xu_target { XU_TARGET_EPS = 0, XU_TARGET_V = 1, XU_TARGET_DISTILL = 2 };

// ---- one element of the fixed-clip table step (sampler_step_table_kernel, and the teacher steps of distill.cu) ----------
// The plain expressions, as nvcc contracts them: out = fma(1 + w, out_c, -(w out_u)) for a guided step (out_c alone for an
// unguided one), x0 = clip(fma(c_recip, z, -(c_recipm1 out)), -1, 1), and z' = fma(sigma, noise, fma(c_x0, x0, c_z z)).
// tab is the step's table row {c_recip, c_recipm1, c_x0, c_z, sigma, ...}.
__device__ __forceinline__ float xu_step_guided(float w, float oc, float ou) { return (1.f + w) * oc - w * ou; }
__device__ __forceinline__ float xu_step_x0(const float* tab, float zi, float e) {
  const float x0 = tab[0] * zi - tab[1] * e;
  return fminf(fmaxf(x0, -1.f), 1.f);
}
__device__ __forceinline__ float xu_step_z(const float* tab, float x0, float zi, float nz) {
  return tab[2] * x0 + tab[3] * zi + tab[4] * nz;
}

// one 64-bit hash serves the 4 consecutive elements idx4*4 .. idx4*4+3 (16-bit uniforms): bit j of the result = keep
__host__ __device__ __forceinline__ uint32_t xu_keep4(uint64_t seed, int op_index, uint64_t idx4, float rate) {
  const uint64_t z = xu_mix64(seed * 0x9E3779B97F4A7C15ULL + (uint64_t)(op_index + 1) * 0xD1B54A32D192ED03ULL + idx4);
  const uint32_t thr = (uint32_t)(rate * 65536.0f);
  uint32_t m = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) m |= (((uint32_t)(z >> (16 * j)) & 0xFFFFu) >= thr ? 1u : 0u) << j;
  return m;
}
__host__ __device__ __forceinline__ bool xu_keep(uint64_t seed, int op_index, uint64_t idx, float rate) {
  return (xu_keep4(seed, op_index, idx >> 2, rate) >> (idx & 3)) & 1u;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Ray direction of pixel (row, col) of a camera (model/xunet.py:159-161): normalize(R K^-1 p) with p = (row+.5, col+.5, 1)
// (convention 0, visu3d 1.3) or (col+.5, row+.5, 1) (convention 1).  ki = K^-1 and R row-major, fp32 throughout; the pose
// embedding and its gradient share it, so the gradient sees the forward's directions bit for bit.
__device__ __forceinline__ void xu_ray_dir(const float* ki, const float* R, int row, int col, int convention, float (&d)[3]) {
  const float p0 = (convention == 0 ? (float)row : (float)col) + 0.5f;
  const float p1 = (convention == 0 ? (float)col : (float)row) + 0.5f;
  float cx = ki[0] * p0 + ki[1] * p1 + ki[2];
  float cy = ki[3] * p0 + ki[4] * p1 + ki[5];
  float cz = ki[6] * p0 + ki[7] * p1 + ki[8];
  float wx = R[0] * cx + R[1] * cy + R[2] * cz;
  float wy = R[3] * cx + R[4] * cy + R[5] * cz;
  float wz = R[6] * cx + R[7] * cy + R[8] * cz;
  float inv = 1.f / sqrtf(wx * wx + wy * wy + wz * wz);
  d[0] = wx * inv; d[1] = wy * inv; d[2] = wz * inv;
}

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// SM count of the current device (132 on an H100 SXM), queried once
static inline int xu_device_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) n = v;
    else n = 132;
  }
  return n;
}
// SMs the persistent / wave-sized grids may fill.  Data parallel: NCCL's reduction CTAs need SMs of their own while the
// persistent one-CTA-per-SM kernels run; with XUNET_SM_RESERVE=k those grids leave k SMs free (a persistent grid that does not
// fit runs a second wave).  How a reduction is split into fp32 partial sums never follows the reserve to longer sums: the
// split-K and pixels-per-block choices take xu_device_sms(), or at least its split, so each CTA or thread sums no more terms
// than on the whole device, which the fp64 launch checks bound.
static inline int xu_num_sms() {
  static int n = 0;
  if (n == 0) {
    n = xu_device_sms();
    const char* e = getenv("XUNET_SM_RESERVE");
    if (e && atoi(e) > 0 && atoi(e) < n) n -= atoi(e);
  }
  return n;
}

// ---- programmatic dependent launch (PDL) --------------------------------------------------------------------------
// Every kernel of the library starts with xu_grid_dep_sync(): it blocks until the previous kernel in the stream has
// completed and flushed (so nothing below it can see stale data), then lets the NEXT kernel's CTAs be scheduled as
// SMs drain -- they park on their own griddepcontrol.wait. With ~430 short kernels per training step this hides the
// launch latency between dependent kernels. Both instructions are no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void xu_grid_dep_sync() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
static inline bool xu_pdl_enabled() {
  static const bool on = (getenv("XUNET_NO_PDL") == nullptr);
  return on;
}
// <<<grid, block, smem, stream>>> with the programmatic-stream-serialization attribute (captured into CUDA graphs as
// programmatic dependency edges)
template <typename... KArgs, typename... Args>
static inline void xu_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = xu_pdl_enabled() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
