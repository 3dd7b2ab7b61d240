// Running per-feature observation normalizer: the statistics fold run at every replay insert, and the apply used by
// the actor / critic modules.  The learner's batch is normalized inside the replay sampler (replay_dev.cuh).
#include "obs_norm.cuh"
#include <algorithm>
#include <cmath>

namespace d4pg {

constexpr int OBS_STATS_MAX_THREADS = 1024;

// One CTA; thread j owns feature j (and j + blockDim, ...) and walks the n rows in order, so a warp reads consecutive
// features of one row.  No atomics: the result depends only on the sequence of rows, not on the launch configuration.
__global__ void __launch_bounds__(OBS_STATS_MAX_THREADS) obs_stats_kernel(double* stats, float* affine, int S,
                                                                          const float* __restrict__ rows, int64_t n,
                                                                          int64_t ld, double eps) {
  const double n0 = stats[0];
  __syncthreads();                                   // every thread has read n before thread 0 rewrites it
  for (int j = threadIdx.x; j < S; j += blockDim.x) {
    double cnt = n0, mean = stats[1 + j], m2 = stats[1 + S + j];
#pragma unroll 4
    for (int64_t i = 0; i < n; ++i) {
      const double x = double(__ldg(rows + i * ld + j));
      cnt = __dadd_rn(cnt, 1.0);
      const double d = __dsub_rn(x, mean);
      mean = __dadd_rn(mean, __ddiv_rn(d, cnt));
      m2 = __dadd_rn(m2, __dmul_rn(d, __dsub_rn(x, mean)));
    }
    stats[1 + j] = mean;
    stats[1 + S + j] = m2;
    float shift = 0.f, scale = 1.f;
    if (cnt > 0.0) {
      const double var = __ddiv_rn(m2, cnt);
      shift = __double2float_rn(mean);
      scale = __double2float_rn(__ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(var, eps))));
    }
    affine[j] = shift;
    affine[S + j] = scale;
  }
  if (threadIdx.x == 0) stats[0] = __dadd_rn(n0, double(n));
}

__global__ void obs_norm_reset_kernel(double* stats, float* affine, int S) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < 1 + 2 * S; j += gridDim.x * blockDim.x) {
    stats[j] = 0.0;
    if (j < 2 * S) affine[j] = j < S ? 0.f : 1.f;
  }
}

// y = apply(x) over [n, S] rows; dydx (optional) = scale where the pre-clip value lies in [-clip, clip], else 0
__global__ void obs_normalize_kernel(const float* __restrict__ affine, int S, float clip, const float* __restrict__ x,
                                     int64_t total, float* __restrict__ y, float* __restrict__ dydx) {
  for (int64_t e = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; e < total; e += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(e % S);
    const float sh = __ldg(affine + c), sc = __ldg(affine + S + c);
    const float v = obs_norm_pre(__ldg(x + e), sh, sc);
    y[e] = fminf(fmaxf(v, -clip), clip);
    if (dydx) dydx[e] = (v >= -clip && v <= clip) ? sc : 0.f;
  }
}

int launch_obs_stats(double* stats, float* affine, int obs_dim, const float* rows, int64_t n, int64_t ld, double eps,
                     cudaStream_t st) {
  const int threads = std::min(OBS_STATS_MAX_THREADS, (obs_dim + 31) / 32 * 32);
  obs_stats_kernel<<<1, threads, 0, st>>>(stats, affine, obs_dim, rows, n, ld, eps);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

int launch_obs_norm_reset(double* stats, float* affine, int obs_dim, cudaStream_t st) {
  obs_norm_reset_kernel<<<cdiv(1 + 2 * obs_dim, 256), 256, 0, st>>>(stats, affine, obs_dim);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

}  // namespace d4pg

using namespace d4pg;

static bool obs_norm_param_ok(double v) { return std::isfinite(v) && v > 0.0; }

extern "C" int32_t d4pg_obs_norm_update(double* stats, float* affine, int32_t obs_dim, const float* rows, int64_t n,
                                        int64_t ld, double eps, d4pg_stream_t stream) {
  D4PG_REQUIRE(stats && affine && obs_dim > 0 && n >= 0 && (n == 0 || (rows && ld >= obs_dim)), D4PG_EINVAL,
               "d4pg_obs_norm_update: bad arguments");
  D4PG_REQUIRE(obs_norm_param_ok(eps), D4PG_EINVAL, "d4pg_obs_norm_update: eps must be finite and > 0 (got %g)", eps);
  return launch_obs_stats(stats, affine, obs_dim, rows, n, ld, eps, as_stream(stream));
}

extern "C" int32_t d4pg_obs_normalize(const float* affine, int32_t obs_dim, double clip, const float* x, int64_t n,
                                      float* y, float* dydx, d4pg_stream_t stream) {
  D4PG_REQUIRE(affine && obs_dim > 0 && n > 0 && x && y, D4PG_EINVAL, "d4pg_obs_normalize: bad arguments");
  D4PG_REQUIRE(obs_norm_param_ok(clip), D4PG_EINVAL, "d4pg_obs_normalize: clip must be finite and > 0 (got %g)", clip);
  const int64_t total = n * obs_dim;
  const int blocks = int(std::min<int64_t>(4 * device_sm_count(), (total + 255) / 256));
  obs_normalize_kernel<<<blocks, 256, 0, as_stream(stream)>>>(affine, obs_dim, float(clip), x, total, y, dydx);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}
