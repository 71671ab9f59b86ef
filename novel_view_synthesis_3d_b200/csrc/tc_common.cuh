// tc_common.cuh -- PTX wrappers shared by the tensor-core kernels (mbarrier, TMA, GMMA descriptors; wgmma.cuh has the MMAs).
#pragma once
#include "common.cuh"
#include <cuda.h>
#include "wgmma.cuh"

// ---------------------------------------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// TMA store of a 4-D box from shared memory (bulk async-group completion)
__device__ __forceinline__ void tma_store_4d(const void* src, const CUtensorMap* map, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(map), "r"(smem_u32(src)),
               "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// TMA reduce-add of a 4-D box from shared memory into global memory (element type from the tensor map: bf16 add performed at L2):
// the accumulate flavour of the staged epilogue -- no read-modify-write of the destination by the SM
__device__ __forceinline__ void tma_reduce_add_4d(const void* src, const CUtensorMap* map, int c0, int c1, int c2, int c3) {
  asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(map),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// 1-D bulk copy global -> shared (bytes a multiple of 16, both addresses 16-byte aligned), completing on an mbarrier
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_group() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// GMMA shared-memory matrix descriptor (sm_90a wgmma): start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout [62,64)
// (1 = 128B, 2 = 64B, 3 = 32B swizzle).  K-major operand whose rows are exactly one swizzle span wide (BK * 2 bytes), as a
// TMA box {BK, rows} lands; SBO = the 8-row core-matrix group stride.  Tiles start on a swizzle-atom boundary, so a K step
// inside the span is a plain start-address offset (k * 32 bytes per 16 elements).
template <int BK>
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t smem_addr) {
  constexpr uint32_t row_bytes = BK * 2;                    // 128 / 64 / 32
  constexpr uint64_t layout = row_bytes == 128 ? 1ull : (row_bytes == 64 ? 2ull : 3ull);
  constexpr uint64_t sbo = (8 * row_bytes) >> 4;
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | (1ull << 16) | (sbo << 32) | (layout << 62);
}

// MN-major operand (the M/N index is the contiguous one), tile stored as [K rows][W elements] with row pitch = one swizzle
// span (W*2 = 128/64/32 bytes) exactly as a TMA box {W, K} lands; wider M/N extents are further [K rows][W] blocks LBO
// bytes apart (canonical GMMA Major-MN layout: SBO = stride between 8-row K groups, LBO = stride between MN blocks).
template <int W>
__device__ __forceinline__ uint64_t make_mnmajor_desc(uint32_t smem_addr, uint32_t lbo_bytes) {
  constexpr uint32_t row_bytes = W * 2;
  constexpr uint64_t layout = row_bytes == 128 ? 1ull : (row_bytes == 64 ? 2ull : 3ull);
  constexpr uint64_t sbo = (8 * row_bytes) >> 4;
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | (sbo << 32) | (layout << 62);
}
// explicit shared-space accesses: through a generic pointer derived from the dynamic shared-memory base the compiler emits LD.E /
// ST.E (generic address translation on every access) instead of LDS / STS
__device__ __forceinline__ void sts128(void* smem_ptr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(smem_u32(smem_ptr)), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ float lds_f32(const void* smem_ptr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(smem_u32(smem_ptr)) : "memory");
  return v;
}
__device__ __forceinline__ float2 lds_f32x2(const void* smem_ptr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(smem_u32(smem_ptr)) : "memory");
  return v;
}
__device__ __forceinline__ void sts_f32(void* smem_ptr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(smem_u32(smem_ptr)), "f"(v) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// 2^x on the MUFU pipe, flush-to-zero (one instruction; exp2f() adds denormal-range fix-ups the softmax does not need)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Transposing warp reduction: every lane holds x[0..31]; on return lane l holds  sum over the 32 lanes of x[l]  (31 shuffles
// instead of the 160 of 32 independent butterfly reductions).  Step s keeps, on the lanes whose bit s is set, the upper half
// of the still-live values and hands the other half to the partner lane.
template <int S>
__device__ __forceinline__ void xu_wtr_step(float (&x)[32], int lane) {
  const bool up = (lane & S) != 0;
#pragma unroll
  for (int i = 0; i < S; ++i) {
    const float send = up ? x[i] : x[i + S];
    const float keep = up ? x[i + S] : x[i];
    x[i] = keep + __shfl_xor_sync(0xffffffffu, send, S);
  }
}
__device__ __forceinline__ float warp_transpose_reduce32(float (&x)[32], int lane) {
  xu_wtr_step<16>(x, lane);
  xu_wtr_step<8>(x, lane);
  xu_wtr_step<4>(x, lane);
  xu_wtr_step<2>(x, lane);
  xu_wtr_step<1>(x, lane);
  return x[0];
}
// GroupNorm input statistics emitted by the PRODUCER of a tensor (conv / attention epilogues): x[0..15] = 16 consecutive
// channels of this lane's pixel (already rounded to the stored dtype), x[16..31] = their squares.  After the transposing
// reduction lane l < 16 holds sum over the warp's 32 pixels of channel l and lane l >= 16 the sum of squares of channel l-16;
// one scalar red per lane lands on the interleaved [channel][sum, sumsq] row of the sample: 128 contiguous bytes per warp.
// cs_row is an fp64 accumulator (xu_det_scratch) folded into the fp32 statistics after the kernel.
__device__ __forceinline__ void xu_cstats_emit16(float (&x)[32], int lane, double* cs_row /* &cstats[(b*C + c0) * 2] */) {
  const float v = warp_transpose_reduce32(x, lane);
  atomicAdd(cs_row + ((lane & 15) << 1) + (lane >> 4), (double)v);
}

// host: encode a bf16 tiled tensor map (rank <= 5; dims/box innermost first; strides in bytes for dims 1..rank-1;
// swizzle chosen from the inner box width: 64 elements -> 128B, 32 -> 64B, 16 -> 32B).  false + kernel error on failure.
// elem_strides (optional, per dim): TMA traversal strides -- a box of extent box[i] then delivers box[i]/elem_strides[i] elements.
bool xu_encode_bf16_map(CUtensorMap* m, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                        const uint32_t* box, int inner_elems, const uint32_t* elem_strides = nullptr);
