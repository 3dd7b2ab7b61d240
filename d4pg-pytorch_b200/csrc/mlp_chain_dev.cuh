// Device-side building blocks of the fp32 cluster chain (mlp_chain_kernel in mlp_chain.cu, act_chain_kernel in act.cu):
// cluster barriers, the A-plane fills, the weight-slice fetch and the exact FFMA tile.
#pragma once
#include "gemm_ffma_dev.cuh"
#include "mlp_chain.cuh"

namespace d4pg {

__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ unsigned long long chain_gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// optional phase stamps of CTA 0 (D4PG_TC_TRACE): 6 per slot
#define CTRACE(i) do { if (tr) tr[(i)] = chain_gtime(); } while (0)
__device__ __forceinline__ unsigned cluster_ctarank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

// Shared-memory layouts (no swizzle needed: every access below is conflict-free as is)
//   A plane   As[k][32 rows]          lane reads 8 rows of one k: 2 LDS.128, broadcast over 8 lanes
//   W (FWD)   Ws[j][P], P = 4 mod 32  W[j][k] rows as they lie in memory; lane owns columns
//                                     j = (lane&7) + 8*jj and reads 4 consecutive k of one j per LDS.128
//   W (DX)    Ws[k][32 cols]          W[k][n0+j]; lane reads 4 consecutive columns of one k
__host__ __device__ static inline int chain_wpitch(int K) { return ((((K + 3) & ~3) + 31) & ~31) + 4; }

// A rows [kbase, kbase+kn) from a row-major global array (transposing, through registers)
// Tensor-core path: the 32 rows (columns) of k-row k are XOR-permuted in groups of 8 by (k & 3) so that the MMA
// fragment loads -- 4 consecutive k for 8 rows -- hit 32 different banks with the dense 32-float pitch.
__device__ __forceinline__ int mma_swz(int k) { return (k & 3) << 3; }
template <bool SWZ>
__device__ __forceinline__ void fill_from_rows(float* As, int kbase, const float* __restrict__ src, int ld, int m0, int B,
                                               int kn, int tid) {
  const int nq = (kn + 3) >> 2;
  for (int e = tid; e < nq * CHAIN_ROWS; e += GEMM_THREADS) {
    const int row = e & 31, k = (e >> 5) << 2;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m0 + row < B) v = __ldg(reinterpret_cast<const float4*>(src + size_t(m0 + row) * ld + k));
    const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (k + c < kn) { const int kk = kbase + k + c; As[kk * CHAIN_ROWS + (SWZ ? (row ^ mma_swz(kk)) : row)] = x[c]; }
  }
}
// A rows [kbase, kbase+kn) from a k-major exchange plane written earlier in this launch by the cluster
template <bool SWZ>
__device__ __forceinline__ void fill_from_plane(float* As, int kbase, const float* plane, int kn, int tid) {
  for (int e = tid; e < kn * 8; e += GEMM_THREADS) {
    const int kk = kbase + (e >> 3), c4 = (e & 7) * 4;
    cp_async16(As + kk * CHAIN_ROWS + (SWZ ? (c4 ^ mma_swz(kk)) : c4), plane + e * 4);
  }
}
// the CTA's 32-column weight slice of one slot, all of K at once
template <bool SWZ>
__device__ __forceinline__ void fetch_weights(float* Ws, const float* __restrict__ W, int ldw, int N, int K, int mode, int n0, int tid);
template <bool SWZ>
__device__ __forceinline__ void fetch_weights(float* Ws, const ChainSlot& S, int n0, int tid) {
  fetch_weights<SWZ>(Ws, S.W, S.ldw, S.N, S.K, S.mode, n0, tid);
}
template <bool SWZ>
__device__ __forceinline__ void fetch_weights(float* Ws, const float* __restrict__ W, int ldw, int N, int K, int mode, int n0, int tid) {
  if (mode == GEMM_FWD) {                      // rows j = n0..n0+31 of W[N][ldw], K floats each
    const int kq = (K + 3) >> 2, P = chain_wpitch(K);
    const int j = tid >> 3;                      // 8 threads per weight row
    if (n0 + j < N) {
      float* dst = Ws + j * P;
      const float* __restrict__ src = W + size_t(n0 + j) * ldw;
      for (int q = tid & 7; q < kq; q += 8) cp_async16(dst + q * 4, src + q * 4);
    }
  } else {                                       // rows k = 0..K-1 of W[K][ldw], columns n0..n0+31
    for (int e = tid; e < K * 8; e += GEMM_THREADS) {
      const int k = e >> 3, c4 = (e & 7) << 2;
      if (n0 + c4 < N) cp_async16(Ws + k * BN + (SWZ ? (c4 ^ mma_swz(k)) : c4), W + size_t(k) * ldw + n0 + c4);
    }
  }
}

struct TileDesc { int N, K, epi; float* C; int ldc; };
__device__ __forceinline__ TileDesc tile_of(const ChainSlot& S) { return TileDesc{S.N, S.K, S.epi, S.C, S.ldc}; }

// As: the A operand (k-major, 32 rows); red: the 8-warp reduce buffer (aliases the slot's A plane, which is dead by then);
// sout: optional shared-memory k-major copy of the output (pre-layers)
template <int MODE>
__device__ __forceinline__ void chain_tile(const TileDesc& S, const float* As, float* red, const float* Ws, int m0, int n0, int B,
                                           float* xout, float* sout, const float (&eop)[4], unsigned long long* tr) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r0 = (lane >> 3) * 8, c0 = (lane & 7) * 4, l7 = lane & 7;
  const int N = S.N, K = S.K;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int P = chain_wpitch(K);
  for (int kb = warp * KW; kb < K; kb += KC) {
    if (MODE == GEMM_FWD) {
#pragma unroll
      for (int g = 0; g < KW; g += 4) {
        const int k4 = kb + g;
        if (k4 >= K) break;
        float bq[4][4];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const float4 t = *reinterpret_cast<const float4*>(&Ws[(l7 + 8 * jj) * P + k4]);
          bq[jj][0] = t.x; bq[jj][1] = t.y; bq[jj][2] = t.z; bq[jj][3] = t.w;
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int kk = k4 + t;
          if (kk < K) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[kk * CHAIN_ROWS + r0]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[kk * CHAIN_ROWS + r0 + 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
              for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bq[j][t], acc[i][j]);
          }
        }
      }
    } else {
#pragma unroll
      for (int k = 0; k < KW; ++k) {
        const int kk = kb + k;
        if (kk >= K) break;
        const float4 a0 = *reinterpret_cast<const float4*>(&As[kk * CHAIN_ROWS + r0]);
        const float4 a1 = *reinterpret_cast<const float4*>(&As[kk * CHAIN_ROWS + r0 + 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Ws[kk * BN + c0]);
        const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
    }
  }
  __syncthreads();                                   // every warp is done with the A plane: reuse it
  CTRACE(3);

  // cross-warp reduction in fixed order.  Buffer column c' = 4*(lane&7) + jj holds output column
  // (FWD) (lane&7) + 8*jj / (DX) c' itself.
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
  const float v[4] = {sum.x, sum.y, sum.z, sum.w};
  const int epi = S.epi;
  float* __restrict__ C = S.C; const int ldc = S.ldc;
#pragma unroll
  for (int cc = 0; cc < 4; ++cc) {
    const int gj = n0 + (MODE == GEMM_FWD ? (tid & 7) + 8 * cc : ocol + cc);
    if (gj >= N) continue;
    float x = v[cc];
    if (gi < B) {
      const float e = eop[cc];                        // bias / forward activation, fetched before the FMA loop
      switch (epi) {
        case EPI_BIAS: x += e; break;
        case EPI_BIAS_RELU: x = fmaxf(x + e, 0.f); break;
        case EPI_BIAS_TANH: x = tanhf(x + e); break;
        case EPI_RELU_MASK: x = (e > 0.f) ? x : 0.f; break;
        case EPI_TANH_MASK: x *= (1.f - e * e); break;
        default: break;
      }
      if (C) C[size_t(gi) * ldc + gj] = x;
    } else x = 0.f;                                   // rows past the batch stay finite in the planes
    if (xout) xout[gj * CHAIN_ROWS + orow] = x;
    if (sout) sout[gj * CHAIN_ROWS + orow] = x;
  }
}

}  // namespace d4pg
