// Device code of the exact-fp32 grouped GEMM.
#pragma once
#include "gemm_ffma.cuh"

namespace d4pg {

constexpr int BM = 32, BN = 32, KC = 64;
constexpr int LDS_A = BM;       // dense rows; bank conflicts of the transposed stores are handled by swz()
constexpr int LDS_B = BN;
constexpr int GEMM_THREADS = 256;
constexpr int GEMM_WARPS = GEMM_THREADS / 32;
constexpr int KW = KC / GEMM_WARPS;                  // k values per warp per chunk (intra-CTA split-K)
constexpr int PER_THREAD = BM * KC / GEMM_THREADS;   // 8 staged elements per thread per operand per chunk

// smem tiles are k-major [kk][32]; the 8 float4 columns of a row are XOR-permuted by (kk>>3)&7 so that
// the transposed stores of a K-contiguous source (a warp writes one column at 16 different kk) spread
// over the banks (8-way conflict without it) while float4 reads along a row stay aligned.
__device__ __forceinline__ int swz(int kk, int idx) { return ((((idx >> 2) ^ (kk >> 3)) & 7) << 2) | (idx & 3); }

// ---- asynchronous copies (LDGSTS, L2-only so planes written by other SMs are read coherently) -------
__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gsrc) {
  const unsigned d = unsigned(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---- operand staging ---------------------------------------------------------------------------
// Two source shapes, each with a 128-bit fast path (scalar staging spends most of its instructions on address
// arithmetic, predicates and constant-bank loads):
//   K-contiguous  src[row*ld + k]  (rows = tile dim): thread reads 2 float4 along k
//   row-contiguous src[k*ld + col] (cols = tile dim): thread reads 2 float4 along the tile dim
// Everything is read into registers first (all loads of a chunk in flight together), then
// written to the k-major smem tiles As[kk][i] / Bs[kk][j].
template <bool VEC>
__device__ __forceinline__ void load_kcontig(const float* __restrict__ src, int ld, int row0, int nrows, int k0, int K,
                                             int tid, float (&r)[PER_THREAD]) {
  if (VEC) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int e = tid + q * GEMM_THREADS, row = e >> 4, k = k0 + ((e & 15) << 2);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row0 + row < nrows && k < K) v = __ldg(reinterpret_cast<const float4*>(src + size_t(row0 + row) * ld + k));
      r[4 * q] = v.x; r[4 * q + 1] = v.y; r[4 * q + 2] = v.z; r[4 * q + 3] = v.w;
    }
  } else {
#pragma unroll
    for (int q = 0; q < PER_THREAD; ++q) {
      const int e = tid + q * GEMM_THREADS, row = e >> 6, k = k0 + (e & 63);
      r[q] = (row0 + row < nrows && k < K) ? __ldg(src + size_t(row0 + row) * ld + k) : 0.f;
    }
  }
}
template <bool VEC>
__device__ __forceinline__ void store_kcontig(float* __restrict__ dst, int lds, int tid, const float (&r)[PER_THREAD]) {
  if (VEC) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int e = tid + q * GEMM_THREADS, row = e >> 4, kk = (e & 15) << 2;
#pragma unroll
      for (int c = 0; c < 4; ++c) dst[(kk + c) * lds + swz(kk + c, row)] = r[4 * q + c];
    }
  } else {
#pragma unroll
    for (int q = 0; q < PER_THREAD; ++q) {
      const int e = tid + q * GEMM_THREADS;
      dst[(e & 63) * lds + swz(e & 63, e >> 6)] = r[q];
    }
  }
}
template <bool VEC>
__device__ __forceinline__ void load_rowcontig(const float* __restrict__ src, int ld, int col0, int ncols, int k0, int K,
                                               int tid, float (&r)[PER_THREAD]) {
  if (VEC) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int e = tid + q * GEMM_THREADS, kk = e >> 3, col = col0 + ((e & 7) << 2);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k0 + kk < K && col < ncols) v = __ldg(reinterpret_cast<const float4*>(src + size_t(k0 + kk) * ld + col));
      r[4 * q] = v.x; r[4 * q + 1] = v.y; r[4 * q + 2] = v.z; r[4 * q + 3] = v.w;
    }
  } else {
#pragma unroll
    for (int q = 0; q < PER_THREAD; ++q) {
      const int e = tid + q * GEMM_THREADS, kk = e >> 5, col = col0 + (e & 31);
      r[q] = (k0 + kk < K && col < ncols) ? __ldg(src + size_t(k0 + kk) * ld + col) : 0.f;
    }
  }
}
template <bool VEC>
__device__ __forceinline__ void store_rowcontig(float* __restrict__ dst, int lds, int tid, const float (&r)[PER_THREAD]) {
  if (VEC) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int e = tid + q * GEMM_THREADS, kk = e >> 3, col = (e & 7) << 2;
      *reinterpret_cast<float4*>(&dst[kk * lds + swz(kk, col)]) = make_float4(r[4 * q], r[4 * q + 1], r[4 * q + 2], r[4 * q + 3]);
    }
  } else {
#pragma unroll
    for (int q = 0; q < PER_THREAD; ++q) {
      const int e = tid + q * GEMM_THREADS;
      dst[(e >> 5) * lds + swz(e >> 5, e & 31)] = r[q];
    }
  }
}

struct Operand { const float* p; int ld; bool vec; };

// A-operand source for chunk k0: FWD may switch to the concatenated second source (k >= K1)
template <int MODE>
__device__ __forceinline__ void load_A(const GemmProblem& P, int m0, int k0, int kend, int tid, float (&ra)[PER_THREAD], bool& vec) {
  if (MODE == GEMM_DW) {               // A(i,k) = dZ[k*lda + i]
    vec = (P.flags & GEMM_A_VEC) != 0;
    if (vec) load_rowcontig<true>(P.A, P.lda, m0, P.M, k0, kend, tid, ra);
    else load_rowcontig<false>(P.A, P.lda, m0, P.M, k0, kend, tid, ra);
  } else if (k0 >= P.K1) {             // concatenated tail (critic fc2's action columns): scalar
    vec = false;
    load_kcontig<false>(P.A2, P.lda2, m0, P.M, k0 - P.K1, P.K - P.K1, tid, ra);
  } else {
    vec = (P.flags & GEMM_A_VEC) != 0;
    if (vec) load_kcontig<true>(P.A, P.lda, m0, P.M, k0, P.K1, tid, ra);
    else load_kcontig<false>(P.A, P.lda, m0, P.M, k0, P.K1, tid, ra);
  }
}
template <int MODE>
__device__ __forceinline__ void store_A(float* As, int tid, const float (&ra)[PER_THREAD], bool vec) {
  if (MODE == GEMM_DW) { if (vec) store_rowcontig<true>(As, LDS_A, tid, ra); else store_rowcontig<false>(As, LDS_A, tid, ra); }
  else { if (vec) store_kcontig<true>(As, LDS_A, tid, ra); else store_kcontig<false>(As, LDS_A, tid, ra); }
}
template <int MODE>
__device__ __forceinline__ void load_B(const GemmProblem& P, int n0, int k0, int kend, int tid, float (&rb)[PER_THREAD]) {
  const bool vec = (P.flags & GEMM_B_VEC) != 0;
  if (MODE == GEMM_FWD) {              // B(k,j) = W[j*ldb + k]
    if (vec) load_kcontig<true>(P.Bm, P.ldb, n0, P.N, k0, kend, tid, rb);
    else load_kcontig<false>(P.Bm, P.ldb, n0, P.N, k0, kend, tid, rb);
  } else {                             // B(k,j) = B[k*ldb + j]
    if (vec) load_rowcontig<true>(P.Bm, P.ldb, n0, P.N, k0, kend, tid, rb);
    else load_rowcontig<false>(P.Bm, P.ldb, n0, P.N, k0, kend, tid, rb);
  }
}
template <int MODE>
__device__ __forceinline__ void store_B(const GemmProblem& P, float* Bs, int tid, const float (&rb)[PER_THREAD]) {
  const bool vec = (P.flags & GEMM_B_VEC) != 0;
  if (MODE == GEMM_FWD) { if (vec) store_kcontig<true>(Bs, LDS_B, tid, rb); else store_kcontig<false>(Bs, LDS_B, tid, rb); }
  else { if (vec) store_rowcontig<true>(Bs, LDS_B, tid, rb); else store_rowcontig<false>(Bs, LDS_B, tid, rb); }
}

// One 32x32 output tile.  The 8 warps split K inside the CTA: each warp owns the whole tile for
// 1/8 of every K-chunk with an 8x4 register tile per lane (32 independent FFMAs per 3 LDS.128);
// the 8 partial tiles are summed through shared memory in fixed warp order (deterministic).
template <int MODE, bool SPLIT>
__device__ __forceinline__ void gemm_tile(const GemmProblem& P, float* smem, int m0, int n0, int tn, int kbeg_in, int kend_in) {
  // the common (non-split) instantiation keeps kbeg = 0 / kend = K as it was before split-K existed
  const int kbeg = SPLIT ? kbeg_in : 0, kend = SPLIT ? kend_in : P.K;
  float* As0 = smem;                      // [2][KC*LDS_A]
  float* Bs0 = smem + 2 * KC * LDS_A;     // [2][KC*LDS_B]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r0 = (lane >> 3) * 8, c0 = (lane & 7) * 4;      // lane's 8x4 sub-tile

  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float colsum = 0.f;                       // DW: bias gradient, threads < BM of the tn==0 tiles
  const bool want_bias_grad = (MODE == GEMM_DW) && (P.bias_grad != nullptr) && (tn == 0);

  float ra[PER_THREAD], rb[PER_THREAD];
  bool avec;
  const int nchunks = (kend - kbeg + KC - 1) / KC;
  load_A<MODE>(P, m0, kbeg, kend, tid, ra, avec);
  load_B<MODE>(P, n0, kbeg, kend, tid, rb);
  store_A<MODE>(As0, tid, ra, avec);
  store_B<MODE>(P, Bs0, tid, rb);
  __syncthreads();
  for (int c = 0; c < nchunks; ++c) {
    const int cur = c & 1;
    if (c + 1 < nchunks) {                                                      // in flight during the FMAs
      load_A<MODE>(P, m0, kbeg + (c + 1) * KC, kend, tid, ra, avec);
      load_B<MODE>(P, n0, kbeg + (c + 1) * KC, kend, tid, rb);
    }
    const float* __restrict__ as = As0 + cur * KC * LDS_A;
    const float* __restrict__ bs = Bs0 + cur * KC * LDS_B;
#pragma unroll
    for (int k = 0; k < KW; ++k) {                                              // zero-padded past K
      const int kk = warp * KW + k;
      const float4 a0 = *reinterpret_cast<const float4*>(&as[kk * LDS_A + swz(kk, r0)]);
      const float4 a1 = *reinterpret_cast<const float4*>(&as[kk * LDS_A + swz(kk, r0 + 4)]);
      const float4 b = *reinterpret_cast<const float4*>(&bs[kk * LDS_B + swz(kk, c0)]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (want_bias_grad && tid < BM) {
#pragma unroll 8
      for (int kk = 0; kk < KC; ++kk) colsum += as[kk * LDS_A + swz(kk, tid)];
    }
    if (c + 1 < nchunks) {
      store_A<MODE>(As0 + (cur ^ 1) * KC * LDS_A, tid, ra, avec);
      store_B<MODE>(P, Bs0 + (cur ^ 1) * KC * LDS_B, tid, rb);
    }
    __syncthreads();
  }

  // ---- cross-warp reduction of the 8 partial tiles (fixed order w = 0..7) ---------------------
  float* red = smem;                        // [GEMM_WARPS][BM][BN]
#pragma unroll
  for (int i = 0; i < 8; ++i)
    *reinterpret_cast<float4*>(&red[(warp * BM + r0 + i) * BN + c0]) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
  __syncthreads();
  const int orow = tid >> 3, ocol = (tid & 7) * 4;          // thread's 4 outputs
  float4 sum = *reinterpret_cast<const float4*>(&red[orow * BN + ocol]);
#pragma unroll
  for (int w = 1; w < GEMM_WARPS; ++w) {
    const float4 t = *reinterpret_cast<const float4*>(&red[(w * BM + orow) * BN + ocol]);
    sum.x += t.x; sum.y += t.y; sum.z += t.z; sum.w += t.w;
  }

  // ---- epilogue ------------------------------------------------------------------------------
  const int gi = m0 + orow;
  if (gi < P.M) {
    const float v[4] = {sum.x, sum.y, sum.z, sum.w};
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const int gj = n0 + ocol + cc;
      if (gj >= P.N) continue;
      float x = v[cc];
      switch (P.epi) {
        case EPI_BIAS: x += __ldg(P.bias + gj); break;
        case EPI_BIAS_RELU: x = fmaxf(x + __ldg(P.bias + gj), 0.f); break;
        case EPI_BIAS_TANH: x = tanhf(x + __ldg(P.bias + gj)); break;
        case EPI_RELU_MASK: x = (__ldg(P.aux + size_t(gi) * P.ldaux + gj) > 0.f) ? x : 0.f; break;
        case EPI_TANH_MASK: { const float t = __ldg(P.aux + size_t(gi) * P.ldaux + gj); x *= (1.f - t * t); } break;
        default: break;
      }
      if (SPLIT) atomicAdd(&P.C[size_t(gi) * P.ldc + gj], x);            // split-K slice (C pre-zeroed)
      else P.C[size_t(gi) * P.ldc + gj] = x;
    }
  }
  if (want_bias_grad && tid < BM && m0 + tid < P.M) {
    if (SPLIT) atomicAdd(&P.bias_grad[m0 + tid], colsum);
    else P.bias_grad[m0 + tid] = colsum;
  }
}


// dW tile with both operands fetched asynchronously, up to 256 batch rows (the whole contraction at
// batch 256) in flight at once: the chunk-by-chunk register staging of gemm_tile pays one L2 round
// trip per 64 rows, which is what a 256-row dW costs almost entirely.  Same order of additions as
// gemm_tile<GEMM_DW>.  Needs 16-B aligned operands with 16-B row pitches (GEMM_ASYNC_OK).
constexpr int DW_STAGE = 256;
constexpr int DW_SMEM_FLOATS = 2 * DW_STAGE * BM;
template <bool SPLIT>
__device__ __forceinline__ void gemm_dw_tile_async(const GemmProblem& P, float* smem, int m0, int n0, int tn, int kbeg, int kend) {
  float* As = smem;                       // [DW_STAGE][32]  dZ[k][m0+i]
  float* Bs = smem + DW_STAGE * BM;       // [DW_STAGE][32]  X[k][n0+j]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r0 = (lane >> 3) * 8, c0 = (lane & 7) * 4;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float colsum = 0.f;
  const bool want_bias_grad = (P.bias_grad != nullptr) && (tn == 0);
  const float* __restrict__ A = P.A; const float* __restrict__ Bm = P.Bm;
  const int lda = P.lda, ldb = P.ldb;

  for (int s0 = kbeg; s0 < kend; s0 += DW_STAGE) {
    const int kn = min(DW_STAGE, kend - s0);
    for (int e = tid; e < kn * 8; e += GEMM_THREADS) {
      const int k = e >> 3, c4 = (e & 7) << 2;
      if (m0 + c4 < lda) cp_async16(As + k * BM + c4, A + size_t(s0 + k) * lda + m0 + c4);
      if (n0 + c4 < ldb) cp_async16(Bs + k * BN + c4, Bm + size_t(s0 + k) * ldb + n0 + c4);
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    for (int kb = warp * KW; kb < kn; kb += KC) {
#pragma unroll
      for (int k = 0; k < KW; ++k) {
        const int kk = kb + k;
        if (kk >= kn) break;
        const float4 a0 = *reinterpret_cast<const float4*>(&As[kk * BM + r0]);
        const float4 a1 = *reinterpret_cast<const float4*>(&As[kk * BM + r0 + 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Bs[kk * BN + c0]);
        const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
    }
    if (want_bias_grad && tid < BM && m0 + tid < P.M) {
#pragma unroll 8
      for (int kk = 0; kk < kn; ++kk) colsum += As[kk * BM + tid];
    }
    __syncthreads();
  }

  float* red = smem;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    *reinterpret_cast<float4*>(&red[(warp * BM + r0 + i) * BN + c0]) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
  __syncthreads();
  const int orow = tid >> 3, ocol = (tid & 7) * 4;
  float4 sum = *reinterpret_cast<const float4*>(&red[orow * BN + ocol]);
#pragma unroll
  for (int w = 1; w < GEMM_WARPS; ++w) {
    const float4 t = *reinterpret_cast<const float4*>(&red[(w * BM + orow) * BN + ocol]);
    sum.x += t.x; sum.y += t.y; sum.z += t.z; sum.w += t.w;
  }
  const int gi = m0 + orow;
  if (gi < P.M) {
    const float v[4] = {sum.x, sum.y, sum.z, sum.w};
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const int gj = n0 + ocol + cc;
      if (gj >= P.N) continue;
      if (SPLIT) atomicAdd(&P.C[size_t(gi) * P.ldc + gj], v[cc]);
      else P.C[size_t(gi) * P.ldc + gj] = v[cc];
    }
  }
  if (want_bias_grad && tid < BM && m0 + tid < P.M) {
    if (SPLIT) atomicAdd(&P.bias_grad[m0 + tid], colsum);
    else P.bias_grad[m0 + tid] = colsum;
  }
}

// dispatch one 32x32 tile of problem P (block-uniform mode switch)
template <bool ALLOW_SPLIT, bool ASYNC_DW = false>
__device__ __forceinline__ void gemm_tile_dispatch(const GemmProblem& P, float* smem, int tile) {
  if (ALLOW_SPLIT && P.ksplit > 1) {        // dW over a large batch (only compiled into the split-K kernel)
    const int per_slice = P.tiles_m * P.tiles_n;
    const int ks = tile / per_slice, t2 = tile - ks * per_slice;
    const int tm = t2 / P.tiles_n, tn = t2 - tm * P.tiles_n;
    const int kbeg = ks * P.kslice;
    if (ASYNC_DW && (P.flags & GEMM_ASYNC_OK)) gemm_dw_tile_async<true>(P, smem, tm * BM, tn * BN, tn, kbeg, min(P.K, kbeg + P.kslice));
    else gemm_tile<GEMM_DW, true>(P, smem, tm * BM, tn * BN, tn, kbeg, min(P.K, kbeg + P.kslice));
    return;
  }
  const int tm = tile / P.tiles_n, tn = tile - tm * P.tiles_n;
  if (ASYNC_DW && P.mode == GEMM_DW && (P.flags & GEMM_ASYNC_OK)) { gemm_dw_tile_async<false>(P, smem, tm * BM, tn * BN, tn, 0, P.K); return; }
  if (P.mode == GEMM_FWD) gemm_tile<GEMM_FWD, false>(P, smem, tm * BM, tn * BN, tn, 0, 0);
  else if (P.mode == GEMM_DX) gemm_tile<GEMM_DX, false>(P, smem, tm * BM, tn * BN, tn, 0, 0);
  else gemm_tile<GEMM_DW, false>(P, smem, tm * BM, tn * BN, tn, 0, 0);
}
constexpr int GEMM_SMEM_FLOATS = 2 * KC * LDS_A + 2 * KC * LDS_B;

}  // namespace d4pg
