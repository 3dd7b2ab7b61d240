// Running per-feature observation normalizer (DESIGN §3 "Observation normalization").
//   stats  f64 [1 + 2S] = {n, mean[S], M2[S]}      affine f32 [2S] = {shift[S], scale[S]}
// Update: Welford, one row at a time in insertion order, every operation rounded and not contracted.
// Affine: n == 0 -> (0, 1); else shift = f32(mean), scale = f32(1 / sqrt(M2 / n + eps)) (fp64, one cast at the end).
// Apply:  y = min(max((x - shift) * scale, -clip), clip) in fp32.
#pragma once
#include "common.cuh"

namespace d4pg {

__device__ __forceinline__ float obs_norm_pre(float x, float shift, float scale) {
  return __fmul_rn(__fsub_rn(x, shift), scale);
}
__device__ __forceinline__ float obs_norm_apply(float x, float shift, float scale, float clip) {
  return fminf(fmaxf(obs_norm_pre(x, shift, scale), -clip), clip);
}

// fold rows [n, ld] into stats and rewrite the affine (n == 0: the affine alone, from the stats as they are)
int launch_obs_stats(double* stats, float* affine, int obs_dim, const float* rows, int64_t n, int64_t ld, double eps,
                     cudaStream_t st);
// stats = 0 (n = 0), affine = identity
int launch_obs_norm_reset(double* stats, float* affine, int obs_dim, cudaStream_t st);

}  // namespace d4pg
