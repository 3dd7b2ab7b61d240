// bf16 tensor-core grouped GEMM for the actor/critic MLP layers (precision mode 3).
//
// Same problem descriptors, modes, epilogues, split-K and PDL launch as gemm_tc.cu; the contraction is ONE wgmma pass
// on bf16 operands:
//   * arithmetic: every operand element is rounded fp32 -> bf16 (round to nearest even, cvt.rn.bf16x2.f32) while it is
//     staged -- X and W in the forward pass, dZ and W for dX, dZ and X for dW -- and the products accumulate in fp32
//     registers (wgmma ... k16.f32.bf16.bf16).  Everything else stays fp32: the stored activations and deltas, the bias
//     adds, the bias gradients (column sums of the unrounded dZ, tc_bias_grad), and no bf16 copy is kept anywhere;
//   * one CTA = one warpgroup = one 128 x 32 output tile (the tiling of gemm_tc.cu: two m64n32k16 accumulators, the
//     shared tc_epilogue), 64-deep K chunks: one 128-B SWIZZLE_128B row holds 64 bf16, so a k16 step advances the
//     descriptor by 32 B exactly as the tf32 k8 step does;
//   * layout: every operand is staged K-major.  Sources that are contiguous along the tile dim (dX's W, both dW
//     operands) are transposed while staged, as gemm_tc.cu does, rather than handed to wgmma's MN-major form: the
//     threads convert every element anyway, so the transpose costs only the store pattern; one layout and one
//     descriptor serve all operands; and the 32-wide N tile (64 B of bf16) would need a second swizzle mode in
//     MN-major form.  A transposing thread pairs the source rows k, k+1 so every shared store is a whole bf16x2 word;
//   * staging by the threads (TMA cannot convert fp32 to bf16): float4 loads where rows are 16-B aligned, scalar loads
//     for ragged rows (|s| = 17 inputs of the forward entry points, the critic fc2 concatenation tail);
//   * 2-stage ring: the staging of chunk c overlaps the wgmmas of chunk c-1.
#include "gemm_tc_epi.cuh"
#include "tc_common.cuh"

namespace d4pg {

using namespace tc;

constexpr int BF_BM = 128, BF_BN = 32, BF_KC = 64;
constexpr int BF_THREADS = 128;                          // one warpgroup
constexpr uint32_t BF_A_BYTES = BF_BM * 128;             // one K chunk of A: 128 rows x 64 bf16
constexpr uint32_t BF_B_BYTES = BF_BN * 128;             // one K chunk of B: 32 rows x 64 bf16
constexpr uint32_t BF_STAGE_BYTES = BF_A_BYTES + BF_B_BYTES;
constexpr int BF_STAGES = 2;

// K-major source: src(row, k) = src[row*ld + k], rows [row0, row0 + ROWS) of an [nrows x K] operand, k in [k0, k0 + 64)
template <int ROWS>
__device__ __forceinline__ void stage_kmajor_bf16(uint8_t* dst, const float* __restrict__ src, int ld, bool vec,
                                                  int row0, int nrows, int k0, int K, int tid) {
  if (vec) {
    // 8 consecutive k of one row (two float4) -> one 16-B chunk of the swizzled row; K % 4 == 0
#pragma unroll 4
    for (int e = tid; e < ROWS * 8; e += BF_THREADS) {
      const int r = e >> 3, q = (e & 7) << 3, k = k0 + q;
      float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
      if (row0 + r < nrows) {
        const float* p = src + size_t(row0 + r) * ld + k;
        if (k < K) v0 = __ldg(reinterpret_cast<const float4*>(p));
        if (k + 4 < K) v1 = __ldg(reinterpret_cast<const float4*>(p + 4));
      }
      *reinterpret_cast<uint4*>(dst + sw128_kmajor_off_b16(r, q)) =
          make_uint4(bf16x2_rn(v0.x, v0.y), bf16x2_rn(v0.z, v0.w), bf16x2_rn(v1.x, v1.y), bf16x2_rn(v1.z, v1.w));
    }
  } else {
    // 2 consecutive k of one row -> one bf16x2 word
#pragma unroll 4
    for (int e = tid; e < ROWS * 32; e += BF_THREADS) {
      const int r = e >> 5, q = (e & 31) << 1, k = k0 + q;
      float x0 = 0.f, x1 = 0.f;
      if (row0 + r < nrows) {
        const float* p = src + size_t(row0 + r) * ld + k;
        if (k < K) x0 = __ldg(p);
        if (k + 1 < K) x1 = __ldg(p + 1);
      }
      *reinterpret_cast<uint32_t*>(dst + sw128_kmajor_off_b16(r, q)) = bf16x2_rn(x0, x1);
    }
  }
}

// Transposing stage: src(k, col) = src[k*ld + col] (dX's W[nout, kin], dW's dZ[b, nout] and X[b, kin]), written into
// the same K-major layout as (row = col, k).  A thread converts the k pair (k, k+1) of 4 columns (vec) or 1 column.
// Vec mapping: a warp covers 8 k pairs x 4 column quads, i.e. 64 contiguous bytes of 16 source rows (whole sectors)
// and 16 distinct banks per store.
template <int COLS>
__device__ __forceinline__ void stage_transposed_bf16(uint8_t* dst, const float* __restrict__ src, int ld, bool vec,
                                                      int col0, int ncols, int k0, int K, int tid) {
  if (vec) {
#pragma unroll 4
    for (int e = tid; e < 32 * (COLS / 4); e += BF_THREADS) {
      const int rest = e >> 3;
      const int kk = ((e & 7) + 8 * (rest / (COLS / 4))) << 1, col = (rest % (COLS / 4)) << 2, k = k0 + kk;
      float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
      if (col0 + col < ncols) {                            // ncols % 4 == 0
        const float* p = src + size_t(k) * ld + col0 + col;
        if (k < K) v0 = __ldg(reinterpret_cast<const float4*>(p));
        if (k + 1 < K) v1 = __ldg(reinterpret_cast<const float4*>(p + ld));
      }
      *reinterpret_cast<uint32_t*>(dst + sw128_kmajor_off_b16(col, kk)) = bf16x2_rn(v0.x, v1.x);
      *reinterpret_cast<uint32_t*>(dst + sw128_kmajor_off_b16(col + 1, kk)) = bf16x2_rn(v0.y, v1.y);
      *reinterpret_cast<uint32_t*>(dst + sw128_kmajor_off_b16(col + 2, kk)) = bf16x2_rn(v0.z, v1.z);
      *reinterpret_cast<uint32_t*>(dst + sw128_kmajor_off_b16(col + 3, kk)) = bf16x2_rn(v0.w, v1.w);
    }
  } else {
#pragma unroll 4
    for (int e = tid; e < 32 * COLS; e += BF_THREADS) {
      const int kk = (e & 31) << 1, col = e >> 5, k = k0 + kk;
      float x0 = 0.f, x1 = 0.f;
      if (col0 + col < ncols) {
        const float* p = src + size_t(k) * ld + col0 + col;
        if (k < K) x0 = __ldg(p);
        if (k + 1 < K) x1 = __ldg(p + ld);
      }
      *reinterpret_cast<uint32_t*>(dst + sw128_kmajor_off_b16(col, kk)) = bf16x2_rn(x0, x1);
    }
  }
}

template <int MODE>
__device__ __forceinline__ void bf16_tile(const GemmProblem& P, uint8_t* smem, int m0, int n0, int tn, int kbeg, int kend) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const bool avec = (P.flags & GEMM_A_VEC) != 0, bvec = (P.flags & GEMM_B_VEC) != 0;
  const int nchunks = (kend - kbeg + BF_KC - 1) / BF_KC;
  const bool split = P.ksplit > 1;

  float acc[2][16];                                      // rows [0, 64) and [64, 128) of the tile
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[h][i] = 0.f;
  // the zero fill is pinned here: a register fence inside the loop would count as a non-wgmma definition of the
  // accumulators and make ptxas serialize the wgmmas
  wg_fence_regs(acc[0]); wg_fence_regs(acc[1]);

  for (int c = 0; c < nchunks; ++c) {
    uint8_t* As = smem + (c % BF_STAGES) * BF_STAGE_BYTES;
    uint8_t* Bs = As + BF_A_BYTES;
    const int k0 = kbeg + c * BF_KC;
    // this stage was last read by the wgmmas of chunk c-2, which completed before chunk c-1 was issued (wait and
    // barrier below); chunk c-1's wgmmas on the other stage run while this chunk is staged
    if (MODE == GEMM_DW) stage_transposed_bf16<BF_BM>(As, P.A, P.lda, avec, m0, P.M, k0, kend, tid);             // dZ[k*lda + m]
    else if (k0 >= P.K1) stage_kmajor_bf16<BF_BM>(As, P.A2, P.lda2, false, m0, P.M, k0 - P.K1, P.K - P.K1, tid); // concat tail
    else stage_kmajor_bf16<BF_BM>(As, P.A, P.lda, avec, m0, P.M, k0, P.K1, tid);
    if (MODE == GEMM_FWD) stage_kmajor_bf16<BF_BN>(Bs, P.Bm, P.ldb, bvec, n0, P.N, k0, P.K, tid);                // W[n*ldb + k]
    else stage_transposed_bf16<BF_BN>(Bs, P.Bm, P.ldb, bvec, n0, P.N, k0, kend, tid);                            // B[k*ldb + n]
    fence_proxy_async();                                 // generic-proxy staging -> the tensor core's async-proxy reads
    // chunk c-1 done before chunk c is issued: no wgmma is in flight across the loop's back edge (ptxas would
    // otherwise serialize the wgmma pipeline).  The barrier orders every warp's wait before the next staging writes.
    wg_wait<0>();
    __syncthreads();
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t bd = wg_desc(smem_u32(Bs + ks * 32));
      wg_mma_n32_bf16(acc[0], wg_desc(smem_u32(As + ks * 32)), bd);
      wg_mma_n32_bf16(acc[1], wg_desc(smem_u32(As + 64 * 128 + ks * 32)), bd);
    }
    wg_commit();
  }
  wg_wait<0>();
  wg_fence_regs(acc[0]); wg_fence_regs(acc[1]);

  tc_epilogue(P, acc, m0, n0, split, warp, lane);
  if (MODE == GEMM_DW && P.bias_grad != nullptr && tn == 0) tc_bias_grad(P, m0, kbeg, kend, split);
}

__global__ void __launch_bounds__(BF_THREADS) gemm_bf16_kernel(const __grid_constant__ GemmBatch batch) {
  __shared__ __align__(1024) uint8_t smem[BF_STAGES * BF_STAGE_BYTES];    // SWIZZLE_128B atoms are 1024-B aligned
  pdl_trigger(batch.pdl);
  pdl_wait();
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
  if (P.mode == GEMM_FWD) bf16_tile<GEMM_FWD>(P, smem, tm * BF_BM, tn * BF_BN, tn, kbeg, kend);
  else if (P.mode == GEMM_DX) bf16_tile<GEMM_DX>(P, smem, tm * BF_BM, tn * BF_BN, tn, kbeg, kend);
  else bf16_tile<GEMM_DW>(P, smem, tm * BF_BM, tn * BF_BN, tn, kbeg, kend);
  pdl_trigger_end(batch.pdl);
}

int gemm_bf16_batch_launch(GemmBatch& b, cudaStream_t st) {
  D4PG_REQUIRE(b.n > 0 && b.n <= GEMM_MAX_PROBLEMS, D4PG_EINVAL, "gemm_bf16_batch_launch: %d problems", b.n);
  for (int i = 0; i < b.n; ++i) {
    D4PG_REQUIRE(b.p[i].mode != GEMM_FWD || b.p[i].K1 == b.p[i].K || b.p[i].K1 % BF_KC == 0, D4PG_ENOTSUP,
                 "gemm_bf16_batch_launch: concat split K1=%d must be a multiple of %d", b.p[i].K1, BF_KC);
    D4PG_REQUIRE(b.p[i].ksplit == 1 || b.p[i].kslice % BF_KC == 0, D4PG_ENOTSUP,
                 "gemm_bf16_batch_launch: split-K slice %d must be a multiple of %d", b.p[i].kslice, BF_KC);
  }
  gemm_batch_retile(b, BF_BM, BF_BN);
  D4PG_MAX_CARVEOUT(gemm_bf16_kernel);
  b.pdl = pdl_mode();
  D4PG_CUDA_OK(launch_pdl(gemm_bf16_kernel, dim3(b.total_tiles), dim3(BF_THREADS), 0, st, b));
  return D4PG_OK;
}

}  // namespace d4pg
