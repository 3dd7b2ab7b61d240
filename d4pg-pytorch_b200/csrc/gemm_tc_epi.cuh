// Epilogue of the wgmma level GEMMs (gemm_tc.cu: 3xTF32 / TF32, gemm_bf16.cu: bf16).  One warpgroup owns a 128 x 32
// output tile held as two m64n32 fp32 accumulators (rows [0, 64) and [64, 128)); the accumulator layout depends on the
// tile shape only, not on the operand type, so both kernels share this code.
#pragma once
#include "gemm_ffma.cuh"

namespace d4pg {

// straight from the accumulator registers: 2 x 2 rows x 8 column pairs per thread; bias / ReLU / tanh /
// activation-derivative masks fused; split-K slices add into the pre-zeroed C with fp32 atomics
// (warp / lane come from the caller: computed there, ahead of the K loop, ptxas keeps the wgmma pipeline unserialized)
__device__ __forceinline__ void tc_epilogue(const GemmProblem& P, const float (&acc)[2][16], int m0, int n0, bool split, int warp, int lane) {
  const float* bias = (P.epi == EPI_BIAS || P.epi == EPI_BIAS_RELU || P.epi == EPI_BIAS_TANH) ? P.bias : nullptr;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int gi = m0 + 64 * h + 16 * warp + (lane >> 2) + 8 * rr;
      if (gi >= P.M) continue;
      float* crow = P.C + size_t(gi) * P.ldc;
      const float* arow = P.aux ? P.aux + size_t(gi) * P.ldaux : nullptr;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int gj = n0 + 8 * (i >> 1) + 2 * (lane & 3) + (i & 1);
        if (gj >= P.N) continue;
        float x = acc[h][(i >> 1) * 4 + rr * 2 + (i & 1)];
        switch (P.epi) {
          case EPI_BIAS: x += __ldg(bias + gj); break;
          case EPI_BIAS_RELU: x = fmaxf(x + __ldg(bias + gj), 0.f); break;
          case EPI_BIAS_TANH: x = tanhf(x + __ldg(bias + gj)); break;
          case EPI_RELU_MASK: x = (__ldg(arow + gj) > 0.f) ? x : 0.f; break;
          case EPI_TANH_MASK: { const float t = __ldg(arow + gj); x *= (1.f - t * t); } break;
          default: break;
        }
        if (split) atomicAdd(crow + gj, x);        // C pre-zeroed
        else crow[gj] = x;
      }
    }
  }
}

// dW: bias gradient = column sums of dZ (rows of A) over K rows [kbeg, kend), exact fp32 from the unrounded source;
// 128 threads <-> the tile's 128 A rows.  Called by the tn == 0 tiles only.
__device__ __forceinline__ void tc_bias_grad(const GemmProblem& P, int m0, int kbeg, int kend, bool split) {
  const int m = m0 + threadIdx.x;
  if (m < P.M) {
    float s = 0.f;
    for (int k = kbeg; k < kend; ++k) s += __ldg(P.A + size_t(k) * P.lda + m);    // coalesced across threads
    if (split) atomicAdd(P.bias_grad + m, s);
    else P.bias_grad[m] = s;
  }
}

}  // namespace d4pg
