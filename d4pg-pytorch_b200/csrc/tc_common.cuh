// Hopper (sm_90a) tensor-core primitives used by the MLP kernels: wgmma with register accumulators,
// the wgmma shared-memory descriptor, mbarrier, TMA.  Thin inline-PTX wrappers; bit layouts follow the
// PTX ISA "warpgroup-level matrix shared memory layout / matrix descriptor" sections.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace d4pg { namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }

// ---- mbarrier ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}

// generic-proxy smem writes -> visible to the async proxy (tensor core / TMA)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- TMA ---------------------------------------------------------------------------------------
// 2-D tiled bulk tensor load global -> shared (SWIZZLE_128B encoded in the tensor map), completion
// signalled on an mbarrier by byte count.  c0 = inner (contiguous) coordinate, c1 = row coordinate.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

// ---- wgmma ----------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (64-bit) of a K-major SWIZZLE_128B operand (the only layout the kernels use):
//   [0,14)  start address >> 4      [16,30) leading-dim byte offset >> 4 (unused by swizzled K-major: 1)
//   [32,46) stride-dim byte offset >> 4 = 1024 B between 8-row groups      [49,52) base offset = 0 (tiles are
//   1024-B aligned)      [62,64) layout type: 1 = SWIZZLE_128B
// A 128-B row holds 32 tf32 (or 64 bf16) along K; the k8 (bf16: k16) step of one wgmma advances the start address by 32 B.
constexpr uint32_t WG_DESC_HI = (1024u >> 4) | (1u << 30);
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
  return uint64_t(((saddr >> 4) & 0x3FFFu) | (1u << 16)) | (uint64_t(WG_DESC_HI) << 32);
}
// all 128 threads of the warpgroup execute these (.sync.aligned)
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across wgmma fences and waits
template <int N>
__device__ __forceinline__ void wg_fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x N] += A[64 x 8] . B[N x 8]^T, tf32 operands from shared memory, fp32 accumulators in registers.
// Thread t of the warpgroup holds d[i] = D[16 (t / 32) + (t % 32) / 4 + 8 ((i >> 1) & 1)][8 (i >> 2) + 2 (t % 4) + (i & 1)].
__device__ __forceinline__ void wg_mma_n32(float (&d)[16], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b) : "memory");
}
__device__ __forceinline__ void wg_mma_n64(float (&d)[32], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b) : "memory");
}
// D[64 x 32] += A[64 x 16] . B[32 x 16]^T, bf16 operands (both K-major: transpose flags 0) from shared memory, fp32
// accumulators in registers with the same d[] layout as wg_mma_n32.  A 128-B row holds 64 bf16, so the k16 step also
// advances the descriptor's start address by 32 B.
__device__ __forceinline__ void wg_mma_n32_bf16(float (&d)[16], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b) : "memory");
}

// ---- SWIZZLE_128B addressing (generic-proxy staging into the canonical wgmma layouts) ------------
// K-major tile: element (r, k32) of a [rows x 32 fp32] block (128 B per row, 8-row groups 1024 B)
__device__ __forceinline__ uint32_t sw128_kmajor_off(int r, int k) {
  return uint32_t((r >> 3) * 1024 + (r & 7) * 128 + ((((k >> 2) ^ (r & 7)) & 7) << 4) + ((k & 3) << 2));
}
// the same layout for 2-byte elements: element (r, k64) of a [rows x 64 bf16] block, 8 elements per 16-B chunk
__device__ __forceinline__ uint32_t sw128_kmajor_off_b16(int r, int k) {
  return uint32_t((r >> 3) * 1024 + (r & 7) * 128 + ((((k >> 3) ^ (r & 7)) & 7) << 4) + ((k & 7) << 1));
}
// two fp32 -> one bf16x2 word, each rounded to nearest even; `lo` lands in the low half (the lower k / address)
__device__ __forceinline__ uint32_t bf16x2_rn(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// tf32 split: hi = x with the low 13 mantissa bits cleared (exactly representable in tf32),
// lo = tf32(x - hi).  x ~= hi + lo to 2^-22 relative; A*B ~= Ah*Bh + Ah*Bl + Al*Bh.
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }
__device__ __forceinline__ float tf32_lo(float x, float hi) { return __uint_as_float(__float_as_uint(x - hi) & 0xFFFFE000u); }

}}  // namespace d4pg::tc
