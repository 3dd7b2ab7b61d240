// Tensor-core grouped GEMM for the actor/critic MLP layers (precision modes 1 = 3xTF32, 2 = 1xTF32).
//
// Same problem descriptors and epilogues as gemm_ffma.cu (models.py:33-40,77-83 forward, autograd
// backward of ddpg.py:230,242), but the contraction runs on the Hopper tensor cores (wgmma):
//   * one CTA = one warpgroup = one 128 x 32 output tile: two m64n32k8 accumulators in registers,
//   * operands staged per 32-deep K chunk into the canonical K-major SWIZZLE_128B layout (wgmma takes
//     tf32 operands K-major only: sources that are contiguous along the tile dim are transposed while
//     staged),
//   * 3xTF32: every fp32 operand is split into hi = tf32(x) and lo = tf32(x - hi) while it is
//     staged; D += Ah*Bh + Ah*Bl + Al*Bh gives ~2^-21 relative accuracy, enough for the 1e-5
//     parity bar of config 2 (a single-pass TF32 or BF16 product is not),
//   * operands whose rows are 16-B aligned and K-contiguous (activations, 256-wide weights) are
//     fetched by TMA (cp.async.bulk.tensor, SWIZZLE_128B tensor maps, mbarrier complete_tx) one
//     chunk ahead of the MMAs and split hi/lo in place; ragged operands (|s|=17, the 262-wide
//     critic fc2 rows, transposed uses) are staged by the threads,
//   * 2-stage ring: the TMA of chunk c+1 and the staging of chunk c overlap the wgmmas of chunk c-1,
//   * split-K for dW over a large batch (slices accumulate into the pre-zeroed C with fp32 atomics),
//   * epilogue straight from the accumulator registers: bias / ReLU / tanh / activation-derivative
//     masks fused.
#include "gemm_tc_epi.cuh"
#include "tc_common.cuh"
#include <stdlib.h>

namespace d4pg {

using namespace tc;

constexpr int TC_BM = 128, TC_BN = 32, TC_KC = 32;
constexpr int TC_THREADS = 128;                    // one warpgroup
constexpr uint32_t A_BYTES = TC_BM * 128;          // one K-chunk of A (hi or lo): 128 rows x 128 B
constexpr uint32_t B_BYTES = TC_BN * 128;          // one K-chunk of B: 32 rows x 128 B
constexpr uint32_t STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;   // hi + lo for both operands
constexpr int TC_STAGES = 2;
constexpr uint32_t TC_SMEM = TC_STAGES * STAGE_BYTES + 1024 /*alignment slack*/;

// ---- staging into SWIZZLE_128B layouts with the hi/lo split ---------------------------------------
__device__ __forceinline__ void put_split(uint8_t* hi_base, uint8_t* lo_base, uint32_t off, float x) {
  const float h = tf32_hi(x);
  *reinterpret_cast<float*>(hi_base + off) = h;
  *reinterpret_cast<float*>(lo_base + off) = tf32_lo(x, h);
}
__device__ __forceinline__ void put_split4(uint8_t* hi_base, uint8_t* lo_base, uint32_t off, float4 v) {
  float4 h = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
  float4 l = make_float4(tf32_lo(v.x, h.x), tf32_lo(v.y, h.y), tf32_lo(v.z, h.z), tf32_lo(v.w, h.w));
  *reinterpret_cast<float4*>(hi_base + off) = h;
  *reinterpret_cast<float4*>(lo_base + off) = l;
}

// K-major block: rows = M/N index, 32 k per row.  src(row, k) = src[row*ld + k].
template <int ROWS>
__device__ __forceinline__ void stage_kmajor(uint8_t* hi, uint8_t* lo, const float* __restrict__ src, int ld, bool vec,
                                             int row0, int nrows, int k0, int K, int tid) {
  if (vec) {
    // 8 float4 per row; a 16-B chunk keeps its position inside the 128-B row up to the XOR swizzle
#pragma unroll 4
    for (int e = tid; e < ROWS * 8; e += TC_THREADS) {
      const int r = e >> 3, q = e & 7, k = k0 + (q << 2);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row0 + r < nrows && k < K) v = __ldg(reinterpret_cast<const float4*>(src + size_t(row0 + r) * ld + k));
      put_split4(hi, lo, sw128_kmajor_off(r, q << 2), v);
    }
  } else {
#pragma unroll 4
    for (int e = tid; e < ROWS * 32; e += TC_THREADS) {
      const int r = e >> 5, kk = e & 31, k = k0 + kk;
      const float x = (row0 + r < nrows && k < K) ? __ldg(src + size_t(row0 + r) * ld + k) : 0.f;
      put_split(hi, lo, sw128_kmajor_off(r, kk), x);
    }
  }
}
// Transposing stage: the source is contiguous along the tile dim (src(k, col) = src[k*ld + col], as in
// dX's W[nout, kin] and dW's dZ[b, nout] / X[b, kin]); it is read coalesced along `col` and written
// into the SAME K-major layout with (row = col, k): wgmma reads tf32 operands K-major only.
template <int COLS>
__device__ __forceinline__ void stage_transposed(uint8_t* hi, uint8_t* lo, const float* __restrict__ src, int ld, bool vec,
                                                 int col0, int ncols, int k0, int K, int tid) {
  if (vec) {
#pragma unroll 4
    for (int e = tid; e < 32 * (COLS / 4); e += TC_THREADS) {
      const int kk = e / (COLS / 4), col = (e % (COLS / 4)) << 2;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k0 + kk < K && col0 + col < ncols) v = __ldg(reinterpret_cast<const float4*>(src + size_t(k0 + kk) * ld + col0 + col));
      put_split(hi, lo, sw128_kmajor_off(col, kk), v.x);
      put_split(hi, lo, sw128_kmajor_off(col + 1, kk), v.y);
      put_split(hi, lo, sw128_kmajor_off(col + 2, kk), v.z);
      put_split(hi, lo, sw128_kmajor_off(col + 3, kk), v.w);
    }
  } else {
#pragma unroll 4
    for (int e = tid; e < 32 * COLS; e += TC_THREADS) {
      const int kk = e / COLS, col = e % COLS;
      const float x = (k0 + kk < K && col0 + col < ncols) ? __ldg(src + size_t(k0 + kk) * ld + col0 + col) : 0.f;
      put_split(hi, lo, sw128_kmajor_off(col, kk), x);
    }
  }
}

// TMA landed raw fp32 in `hi`; rewrite it as hi and emit lo at the same (already swizzled) offsets
template <int BYTES>
__device__ __forceinline__ void split_in_place(uint8_t* hi, uint8_t* lo, int tid) {
#pragma unroll 4
  for (int e = tid; e < BYTES / 16; e += TC_THREADS) {
    const float4 v = *reinterpret_cast<const float4*>(hi + e * 16);
    put_split4(hi, lo, uint32_t(e) * 16u, v);
  }
}

template <int MODE>
__device__ __forceinline__ void tc_tile(const GemmProblem& P, const CUtensorMap* tmA, const CUtensorMap* tmB,
                                        uint8_t* smem, uint64_t* full, int m0, int n0, int tn, int kbeg, int kend,
                                        int passes) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr bool A_T = (MODE == GEMM_DW);       // source contiguous along the tile dim -> transposing stage
  constexpr bool B_T = (MODE != GEMM_FWD);
  const bool avec = (P.flags & GEMM_A_VEC) != 0, bvec = (P.flags & GEMM_B_VEC) != 0;
  const bool a_tma = (P.flags & GEMM_A_TMA) != 0, b_tma = (P.flags & GEMM_B_TMA) != 0;
  const int nchunks = (kend - kbeg + TC_KC - 1) / TC_KC;
  const bool split = P.ksplit > 1;

  // TMA for chunk c (thread 0): A from the main source only (the concat tail is staged by threads)
  auto issue_tma = [&](int c) {
    const int st = c % TC_STAGES, k0 = kbeg + c * TC_KC;
    uint8_t* Ahi = smem + st * STAGE_BYTES;
    uint8_t* Bhi = Ahi + 2 * A_BYTES;
    const bool a_now = a_tma && k0 < P.K1, b_now = b_tma;
    if (!(a_now || b_now)) return;
    mbar_expect_tx(&full[st], (a_now ? A_BYTES : 0u) + (b_now ? B_BYTES : 0u));
    if (a_now) tma_load_2d(Ahi, tmA, &full[st], k0, m0);
    if (b_now) tma_load_2d(Bhi, tmB, &full[st], k0, n0);
  };
  if (tid == 0 && (a_tma || b_tma)) issue_tma(0);
  uint32_t full_parity[TC_STAGES] = {0u, 0u};      // per-stage phase of the TMA barrier (not every chunk uses it)

  float acc[2][16];                                // rows [0, 64) and [64, 128) of the tile
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[h][i] = 0.f;

  for (int c = 0; c < nchunks; ++c) {
    const int st = c % TC_STAGES;
    uint8_t* Ahi = smem + st * STAGE_BYTES;
    uint8_t* Alo = Ahi + A_BYTES;
    uint8_t* Bhi = Alo + A_BYTES;
    uint8_t* Blo = Bhi + B_BYTES;
    const int k0 = kbeg + c * TC_KC;
    // the other stage is reused by chunk c+1: the wgmmas of chunk c-1 must have drained it before its TMA flies.
    // wgmma completion is tracked per warpgroup, but the barrier makes every warp's wait precede thread 0's TMA
    // explicitly (it also orders this chunk's staging writes after all reads of the stage).
    wg_wait<0>();
    __syncthreads();
    if (c + 1 < nchunks && tid == 0 && (a_tma || b_tma)) issue_tma(c + 1);
    const bool a_now = a_tma && k0 < P.K1;
    // ---- thread-staged operands -----------------------------------------------------------------
    if (!a_now) {
      if (A_T) stage_transposed<TC_BM>(Ahi, Alo, P.A, P.lda, avec, m0, P.M, k0, kend, tid);             // dZ[k*lda + m]
      else if (k0 >= P.K1) stage_kmajor<TC_BM>(Ahi, Alo, P.A2, P.lda2, false, m0, P.M, k0 - P.K1, P.K - P.K1, tid);
      else stage_kmajor<TC_BM>(Ahi, Alo, P.A, P.lda, avec, m0, P.M, k0, P.K1, tid);
    }
    if (!b_tma) {
      if (B_T) stage_transposed<TC_BN>(Bhi, Blo, P.Bm, P.ldb, bvec, n0, P.N, k0, kend, tid);            // B[k*ldb + n]
      else stage_kmajor<TC_BN>(Bhi, Blo, P.Bm, P.ldb, bvec, n0, P.N, k0, P.K, tid);                     // W[n*ldb + k]
    }
    // ---- TMA-fed operands: wait for the bytes, split hi/lo in place --------------------------------
    if (a_now || b_tma) {
      mbar_wait(&full[st], full_parity[st]);
      full_parity[st] ^= 1u;
      if (passes > 1) {
        if (a_now) split_in_place<A_BYTES>(Ahi, Alo, tid);
        if (b_tma) split_in_place<B_BYTES>(Bhi, Blo, tid);
      }
    }
    fence_proxy_async();                           // generic-proxy staging -> the tensor core's async-proxy reads
    __syncthreads();
    wg_fence_regs(acc[0]); wg_fence_regs(acc[1]);
    wg_fence();
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      if (p >= passes) break;
      const uint8_t* Ap = (p == 2) ? Alo : Ahi;
      const uint8_t* Bp = (p == 1) ? Blo : Bhi;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t bd = wg_desc(smem_u32(Bp + ks * 32));
        wg_mma_n32(acc[0], wg_desc(smem_u32(Ap + ks * 32)), bd);
        wg_mma_n32(acc[1], wg_desc(smem_u32(Ap + 64 * 128 + ks * 32)), bd);
      }
    }
    wg_commit();
  }
  wg_wait<0>();
  wg_fence_regs(acc[0]); wg_fence_regs(acc[1]);

  tc_epilogue(P, acc, m0, n0, split, warp, lane);
  if (MODE == GEMM_DW && P.bias_grad != nullptr && tn == 0) tc_bias_grad(P, m0, kbeg, kend, split);
}

__global__ void __launch_bounds__(TC_THREADS) gemm_tc_kernel(const __grid_constant__ GemmBatch batch, int passes) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t full[TC_STAGES];

  int pi = 0;
#pragma unroll
  for (int i = 1; i < GEMM_MAX_PROBLEMS; ++i)
    if (i < batch.n && int(blockIdx.x) >= batch.p[i].tile_begin) pi = i;
  const GemmProblem P = batch.p[pi];
  const int tile = blockIdx.x - P.tile_begin;
  const int per_slice = P.tiles_m * P.tiles_n;
  const int kslice_id = tile / per_slice, tile2 = tile - kslice_id * per_slice;
  const int tm = tile2 / P.tiles_n, tn = tile2 - tm * P.tiles_n;
  // split-K (dW over a large batch): this CTA contracts K rows [kbeg, kend)
  const int kbeg = kslice_id * P.kslice, kend = min(P.K, kbeg + P.kslice);

  if (threadIdx.x == 0) {
    for (int i = 0; i < TC_STAGES; ++i) mbar_init(&full[i], 1);
    mbar_fence_init();
  }
  pdl_trigger(batch.pdl);
  __syncthreads();
  pdl_wait();                                   // prologue above overlapped the previous kernel's tail

  const CUtensorMap* tmA = &batch.tmap_a[pi];
  const CUtensorMap* tmB = &batch.tmap_b[pi];
  if (P.mode == GEMM_FWD) tc_tile<GEMM_FWD>(P, tmA, tmB, smem, full, tm * TC_BM, tn * TC_BN, tn, kbeg, kend, passes);
  else if (P.mode == GEMM_DX) tc_tile<GEMM_DX>(P, tmA, tmB, smem, full, tm * TC_BM, tn * TC_BN, tn, kbeg, kend, passes);
  else tc_tile<GEMM_DW>(P, tmA, tmB, smem, full, tm * TC_BM, tn * TC_BN, tn, kbeg, kend, passes);
  pdl_trigger_end(batch.pdl);
}

// ---- host: TMA descriptors -------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encoder() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}
// [rows x inner] fp32, row pitch ld floats, box = 32 x box_rows, 128-B swizzle, zero fill out of bounds
static bool encode_kmajor(CUtensorMap* tm, const float* base, int inner, int rows, int ld, int box_rows) {
  EncodeTiledFn enc = get_encoder();
  if (!enc) return false;
  cuuint64_t dims[2] = {cuuint64_t(inner), cuuint64_t(rows)};
  cuuint64_t strides[1] = {cuuint64_t(ld) * 4};
  cuuint32_t box[2] = {32, cuuint32_t(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
static bool tma_ok(const float* p, int ld) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0 && ld % 4 == 0; }

// Decide per operand whether TMA may fetch it (K-contiguous source, 16-B aligned rows) and encode the maps.
static unsigned long long* g_trace = nullptr;
unsigned long long* debug_trace_buffer() {
  static const bool tracing = getenv("D4PG_TC_TRACE") != nullptr;
  if (tracing && !g_trace) { cudaMalloc(&g_trace, 512 * sizeof(unsigned long long)); cudaMemset(g_trace, 0, 512 * 8); }
  return tracing ? g_trace : nullptr;
}
void gemm_tc_prepare(GemmBatch& b) {
  b.trace = debug_trace_buffer();
  gemm_batch_retile(b, TC_BM, TC_BN);
  for (int i = 0; i < b.n; ++i) {
    GemmProblem& p = b.p[i];
    p.flags &= ~(GEMM_A_TMA | GEMM_B_TMA);
    if (p.mode != GEMM_DW && tma_ok(p.A, p.lda) && encode_kmajor(&b.tmap_a[i], p.A, p.K1, p.M, p.lda, TC_BM))
      p.flags |= GEMM_A_TMA;
    if (p.mode == GEMM_FWD && tma_ok(p.Bm, p.ldb) && encode_kmajor(&b.tmap_b[i], p.Bm, p.K, p.N, p.ldb, TC_BN))
      p.flags |= GEMM_B_TMA;
  }
}

int gemm_tc_batch_launch(const GemmBatch& b, int passes, cudaStream_t st) {
  D4PG_REQUIRE(b.n > 0 && b.n <= GEMM_MAX_PROBLEMS, D4PG_EINVAL, "gemm_tc_batch_launch: %d problems", b.n);
  for (int i = 0; i < b.n; ++i) {
    D4PG_REQUIRE(b.p[i].mode != GEMM_FWD || b.p[i].K1 == b.p[i].K || b.p[i].K1 % TC_KC == 0, D4PG_ENOTSUP,
                 "gemm_tc_batch_launch: concat split K1=%d must be a multiple of %d", b.p[i].K1, TC_KC);
    D4PG_REQUIRE(b.p[i].ksplit == 1 || b.p[i].kslice % TC_KC == 0, D4PG_ENOTSUP,
                 "gemm_tc_batch_launch: split-K slice %d must be a multiple of %d", b.p[i].kslice, TC_KC);
  }
  static bool attr_set = false;
  if (!attr_set) {
    D4PG_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(TC_SMEM)));
    D4PG_MAX_CARVEOUT(gemm_tc_kernel);
    attr_set = true;
  }
  const_cast<GemmBatch&>(b).pdl = pdl_mode();
  D4PG_CUDA_OK(launch_pdl(gemm_tc_kernel, dim3(b.total_tiles), dim3(TC_THREADS), TC_SMEM, st, b, passes));
  return D4PG_OK;
}

}  // namespace d4pg

// debug: %globaltimer (ns) phase stamps written by the step kernels (D4PG_TC_TRACE=1)
extern "C" int32_t d4pg_debug_trace_read(unsigned long long* out, int32_t n) {
  if (!d4pg::g_trace || !out || n < 1 || n > 512) return D4PG_ESTATE;
  D4PG_CUDA_OK(cudaMemcpy(out, d4pg::g_trace, size_t(n) * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  return D4PG_OK;
}
extern "C" int32_t d4pg_debug_tc_trace(unsigned long long* out16) {
  if (!d4pg::g_trace || !out16) return D4PG_ESTATE;
  D4PG_CUDA_OK(cudaMemcpy(out16, d4pg::g_trace, 32 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  return D4PG_OK;
}
