// Adaptive parameter-space exploration noise (Plappert et al. 2018; baselines' AdaptiveParamNoiseSpec): the actor
// perturbation kernel and the policy-distance adaptation kernel, with their C ABI d4pg_actor_perturb and
// d4pg_param_noise_adapt.  The semantics are DESIGN §3 "Parameter-space noise".
#include "common.cuh"
#include <cmath>

namespace d4pg {

constexpr int PERTURB_THREADS = 256;
constexpr int ADAPT_THREADS = 256;                // fixed: the summation order belongs to the build, not the device
constexpr double PN_TWO_PI = 2.0 * 3.14159265358979323846;     // == 2 * numpy.pi

// The 8 tensors of the actor's flat buffer (fc1.weight, fc1.bias, ..., fc3.bias) in d4pg_actor_layout order: where each
// starts in the padded buffer, where its first element sits in the logical (unpadded) concatenation, its row pitch (1 for
// a bias), its logical row width and its row count.
struct PerturbArgs {
  int64_t off[8], base[8];
  int pitch[8], width[8], rows[8];
  int64_t groups;                 // padded floats / 4
  const float* src;
  float* dst;
  const double* state;            // {sigma, last distance}
  uint64_t seed, counter;
};

// z = sqrt(-2 log(1 - u1)) cos(2 pi u2) of logical element i, u1 / u2 = uniform53(seed, counter, 2i / 2i + 1): the
// construction of act_chain_kernel's noise, every fp64 operation rounded on its own
__device__ __forceinline__ double perturb_normal(uint64_t seed, uint64_t counter, uint32_t i) {
  const double u1 = Philox::uniform53(seed, counter, 2u * i);
  const double u2 = Philox::uniform53(seed, counter, 2u * i + 1u);
  return __dmul_rn(__dsqrt_rn(__dmul_rn(-2.0, log(__dsub_rn(1.0, u1)))), cos(__dmul_rn(PN_TWO_PI, u2)));
}

// Grid-stride over the padded buffer in 4-float groups.  Every tensor starts 4-float aligned and every weight row pitch
// is a multiple of 4, so a group never straddles two tensors or two rows: the group finds its tensor and row once, and
// each of its floats is either a logical element (p' = f32(f64(p) + sigma * z)) or padding (written as 0).
__global__ void __launch_bounds__(PERTURB_THREADS) actor_perturb_kernel(const __grid_constant__ PerturbArgs a) {
  const double sigma = a.state[0];
  for (int64_t g = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; g < a.groups; g += int64_t(gridDim.x) * blockDim.x) {
    const int64_t p = 4 * g;
    int t = 0;
#pragma unroll
    for (int k = 1; k < 8; ++k)
      if (p >= a.off[k]) t = k;
    const int64_t r = p - a.off[t];
    const int64_t row = r / a.pitch[t];
    const int col = int(r - row * a.pitch[t]);
    const float4 v = __ldg(reinterpret_cast<const float4*>(a.src) + g);
    const float x[4] = {v.x, v.y, v.z, v.w};
    float y[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if (row < a.rows[t] && col + c < a.width[t]) {
        const int64_t i = a.base[t] + row * a.width[t] + col + c;
        y[c] = __double2float_rn(__dadd_rn(double(x[c]), __dmul_rn(sigma, perturb_normal(a.seed, a.counter, uint32_t(i)))));
      } else {
        y[c] = 0.f;
      }
    }
    reinterpret_cast<float4*>(a.dst)[g] = make_float4(y[0], y[1], y[2], y[3]);
  }
}

// One CTA.  d = sqrt(sum_i (f64(ap_i) - f64(a_i))^2 / n): thread t sums i = t, t + T, ... in index order, then a fixed
// shared-memory tree; thread 0 applies baselines' rule sigma = d > desired ? sigma / coef : sigma * coef and stores
// {sigma, d}.  No atomics, so the bits depend on the inputs alone.
__global__ void __launch_bounds__(ADAPT_THREADS) param_noise_adapt_kernel(const float* __restrict__ a, const float* __restrict__ ap,
                                                                          int64_t n, double desired, double coef, double* state) {
  __shared__ double part[ADAPT_THREADS];
  const int t = threadIdx.x;
  double s = 0.0;
  for (int64_t i = t; i < n; i += ADAPT_THREADS) {
    const double d = __dsub_rn(double(__ldg(ap + i)), double(__ldg(a + i)));
    s = __dadd_rn(s, __dmul_rn(d, d));
  }
  part[t] = s;
  __syncthreads();
#pragma unroll
  for (int w = ADAPT_THREADS / 2; w > 0; w >>= 1) {
    if (t < w) part[t] = __dadd_rn(part[t], part[t + w]);
    __syncthreads();
  }
  if (t == 0) {
    const double d = __dsqrt_rn(__ddiv_rn(part[0], double(n)));
    const double sigma = state[0];
    state[0] = d > desired ? __ddiv_rn(sigma, coef) : __dmul_rn(sigma, coef);
    state[1] = d;
  }
}

}  // namespace d4pg

using namespace d4pg;

static bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

extern "C" int32_t d4pg_actor_perturb(const float* params, int32_t obs_dim, int32_t act_dim, const double* noise_state,
                                      uint64_t seed, uint64_t counter, float* out, d4pg_stream_t stream) {
  D4PG_REQUIRE(params && noise_state && out, D4PG_EINVAL, "d4pg_actor_perturb: null argument");
  D4PG_REQUIRE(aligned(params, 16) && aligned(out, 16) && aligned(noise_state, 8), D4PG_EINVAL,
               "d4pg_actor_perturb: params and out must be 16-B aligned, noise_state 8-B aligned");
  D4PG_REQUIRE(obs_dim > 0 && act_dim > 0, D4PG_EINVAL, "d4pg_actor_perturb: obs_dim %d / act_dim %d", obs_dim, act_dim);
  const NetDims d = actor_dims(obs_dim, act_dim);
  PerturbArgs a{};
  int64_t count = 0;
  for (int l = 0; l < 4; ++l) {
    a.off[2 * l] = d.w_off[l]; a.base[2 * l] = count; a.pitch[2 * l] = d.ld[l];
    a.width[2 * l] = d.in[l]; a.rows[2 * l] = d.out[l];
    count += int64_t(d.in[l]) * d.out[l];
    a.off[2 * l + 1] = d.b_off[l]; a.base[2 * l + 1] = count; a.pitch[2 * l + 1] = 1 << 30;   // one "row"
    a.width[2 * l + 1] = d.out[l]; a.rows[2 * l + 1] = 1;
    count += d.out[l];
  }
  D4PG_REQUIRE(2 * count < (int64_t(1) << 32), D4PG_EINVAL,
               "d4pg_actor_perturb: %lld parameters (the draw index needs 2 * count < 2^32)", (long long)count);
  a.groups = d.total / 4;
  a.src = params; a.dst = out; a.state = noise_state;
  a.seed = seed; a.counter = counter;
  const int64_t want = (a.groups + PERTURB_THREADS - 1) / PERTURB_THREADS;
  const int grid = int(want < int64_t(8) * device_sm_count() ? want : int64_t(8) * device_sm_count());
  actor_perturb_kernel<<<grid, PERTURB_THREADS, 0, as_stream(stream)>>>(a);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

extern "C" int32_t d4pg_param_noise_adapt(const float* a, const float* a_perturbed, int64_t n, double desired_stddev,
                                          double coefficient, double* noise_state, d4pg_stream_t stream) {
  D4PG_REQUIRE(a && a_perturbed && noise_state, D4PG_EINVAL, "d4pg_param_noise_adapt: null argument");
  D4PG_REQUIRE(aligned(a, 4) && aligned(a_perturbed, 4) && aligned(noise_state, 8), D4PG_EINVAL,
               "d4pg_param_noise_adapt: misaligned pointer");
  D4PG_REQUIRE(n >= 1, D4PG_EINVAL, "d4pg_param_noise_adapt: n = %lld (need n >= 1)", (long long)n);
  D4PG_REQUIRE(std::isfinite(desired_stddev) && desired_stddev > 0.0, D4PG_EINVAL,
               "d4pg_param_noise_adapt: desired_stddev must be finite and > 0 (got %g)", desired_stddev);
  D4PG_REQUIRE(std::isfinite(coefficient) && coefficient > 1.0, D4PG_EINVAL,
               "d4pg_param_noise_adapt: coefficient must be finite and > 1 (got %g)", coefficient);
  param_noise_adapt_kernel<<<1, ADAPT_THREADS, 0, as_stream(stream)>>>(a, a_perturbed, n, desired_stddev, coefficient,
                                                                        noise_state);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}
