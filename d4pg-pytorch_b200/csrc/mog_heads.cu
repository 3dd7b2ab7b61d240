// Mixture-of-Gaussians critic head (critic_dist_info['type'] == 'mixture_of_gaussian', K components): the fused
// loss / TD / priority / raw-head-gradient row kernel of the learner step, plus the two small kernels of the standalone
// critic module (raw head -> (w, mu, sigma), and (g_w, g_mu, g_sigma) -> d raw head).
//
// DERIVED semantics (the reference stubs this branch with `TODO: pass`, ddpg.py:48-50, models.py:63-65):
//   raw row o [3K]:  w = softmax(o[0:K]),  mu = o[K:2K],  sigma = softplus(o[2K:3K]) + 1e-3  (torch softplus: x for x > 20)
//   target mixture of row i: weights w'_k, means r_i + c mu'_k, std devs c sigma'_k, c = discount * (1 - done_i)
//   critic loss row: the cross-entropy of the online mixture under the target mixture, integrated with Q = 8
//   Gauss-Hermite nodes per target component:  L_i = -sum_{k,q} omega_kq log p(y_kq),
//   y_kq = r_i + c (mu'_k + sqrt(2) sigma'_k x_q),  omega_kq = w'_k h_q / sqrt(pi)
//   td_i = sum_j w_j mu_j - (r_i + c sum_k w'_k mu'_k),  priority = |td_i| + eps
//   policy loss row: -sum_j w_j mu_j on critic(s, actor(s))
// One warp per row, one lane per online component (K <= 32), the quadrature points spread over the lanes; the whole row is evaluated in fp64 from the fp32 raw head (the
// log-densities of far-away nodes reach 1e9 when sigma sits at its 1e-3 floor) and the results are rounded to fp32.
#include "internal.cuh"

namespace d4pg {

constexpr int MOG_WARPS = 4;
constexpr int MOG_Q = 8;

// numpy.polynomial.hermite.hermgauss(8): nodes x_q and weights h_q (sum h_q = sqrt(pi))
#define D4PG_GH_X {-2.930637420257244, -1.981656756695843, -1.1571937124467802, -0.3811869902073221, \
                   0.3811869902073221, 1.1571937124467802, 1.981656756695843, 2.930637420257244}
#define D4PG_GH_H {0.00019960407221136783, 0.017077983007413467, 0.20780232581489183, 0.6611470125582415, \
                   0.6611470125582415, 0.20780232581489183, 0.017077983007413467, 0.00019960407221136783}
static const double h_gh_x[MOG_Q] = D4PG_GH_X, h_gh_h[MOG_Q] = D4PG_GH_H;
__constant__ double c_gh_x[MOG_Q] = D4PG_GH_X;
__constant__ double c_gh_h[MOG_Q] = D4PG_GH_H;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// component `lane` of one raw row (lanes >= K: weight 0, log-weight -inf)
struct MogComp { double logw, w, mu, sigma, dsigma; };   // dsigma = d sigma / d raw (softplus')
__device__ __forceinline__ MogComp mog_comp(const float* __restrict__ raw, int K, int lane) {
  MogComp c;
  const bool on = lane < K;
  const double a = on ? double(raw[lane]) : -INFINITY;
  const double mx = warp_max_d(a);
  const double e = on ? exp(a - mx) : 0.0;
  const double s = warp_sum_d(e);
  c.logw = on ? (a - mx) - log(s) : -INFINITY;
  c.w = e / s;
  c.mu = on ? double(raw[K + lane]) : 0.0;
  const double x = on ? double(raw[2 * K + lane]) : 0.0;
  const double z = exp(x);
  c.sigma = (x > 20.0 ? x : log1p(z)) + 1e-3;
  c.dsigma = x > 20.0 ? 1.0 : z / (z + 1.0);                 // torch's softplus backward
  return c;
}

// critic part of one row: loss row, td, priority, d loss / d raw online head.
// Lane j holds online component j; the 8K quadrature points are spread over the lanes (point p = 8k + q on lane p % 32,
// NT = ceil(8K / 32) per lane), so the per-point logsumexp over the components runs in registers and only the K
// per-component gradient sums need warp reductions.
template <int NT, bool HZ>
__device__ __forceinline__ void mog_critic_row(const MogArgs& a, int row, int lane) {
  const int K = a.K;
  const size_t ro = size_t(row) * a.h.ld;
  const bool on = lane < K;
  const MogComp t = mog_comp(a.h.target + ro, K, lane);
  const MogComp q = mog_comp(a.h.q + ro, K, lane);
  const double r = a.h.rewards[row];
  const double c = a.h.dones[row] ? 0.0 : (HZ ? head_discount(a.h, row) : a.h.discount);
  const float isw = a.h.is_weights ? __ldg(a.h.is_weights + row) : 1.f;
  const double LOG_2PI = 1.8378770664093453, SQRT2 = 1.4142135623730951, INV_SQRTPI = 0.5641895835477563;
  const double inv_sig = 1.0 / q.sigma;
  const double lc = on ? q.logw - log(q.sigma) - 0.5 * LOG_2PI : -INFINITY;
  // this lane's points: y = r + c (mu'_k + sqrt(2) sigma'_k x_q), omega = w'_k h_q / sqrt(pi)  (0 past the last point)
  double y[NT], om[NT], lse[NT];
#pragma unroll
  for (int u = 0; u < NT; ++u) {
    const int p = lane + 32 * u, k = min(p / MOG_Q, K - 1), qn = p % MOG_Q;
    const double wk = __shfl_sync(0xffffffffu, t.w, k);
    const double mk = __shfl_sync(0xffffffffu, t.mu, k);
    const double sk = __shfl_sync(0xffffffffu, t.sigma, k);
    y[u] = r + c * (mk + SQRT2 * sk * c_gh_x[qn]);
    om[u] = p < MOG_Q * K ? wk * c_gh_h[qn] * INV_SQRTPI : 0.0;
  }
  // log p(y) = logsumexp_j (lc_j - z_j^2 / 2): max pass, then the sum of exponentials
  double mx[NT], sm[NT];
#pragma unroll
  for (int u = 0; u < NT; ++u) { mx[u] = -INFINITY; sm[u] = 0.0; }
  for (int j = 0; j < K; ++j) {
    const double lj = __shfl_sync(0xffffffffu, lc, j), mj = __shfl_sync(0xffffffffu, q.mu, j);
    const double ij = __shfl_sync(0xffffffffu, inv_sig, j);
#pragma unroll
    for (int u = 0; u < NT; ++u) { const double z = (y[u] - mj) * ij; mx[u] = fmax(mx[u], lj - 0.5 * z * z); }
  }
  for (int j = 0; j < K; ++j) {
    const double lj = __shfl_sync(0xffffffffu, lc, j), mj = __shfl_sync(0xffffffffu, q.mu, j);
    const double ij = __shfl_sync(0xffffffffu, inv_sig, j);
#pragma unroll
    for (int u = 0; u < NT; ++u) { const double z = (y[u] - mj) * ij; sm[u] += exp(lj - 0.5 * z * z - mx[u]); }
  }
  double loss = 0.0;
#pragma unroll
  for (int u = 0; u < NT; ++u) { lse[u] = mx[u] + log(sm[u]); loss -= om[u] * lse[u]; }
  loss = warp_sum_d(loss);
  // per component j: sum over points of omega * responsibility_j * (1, z, z^2 - 1)
  double gl = 0.0, gm = 0.0, gs = 0.0;
  for (int j = 0; j < K; ++j) {
    const double lj = __shfl_sync(0xffffffffu, lc, j), mj = __shfl_sync(0xffffffffu, q.mu, j);
    const double ij = __shfl_sync(0xffffffffu, inv_sig, j);
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
#pragma unroll
    for (int u = 0; u < NT; ++u) {
      const double z = (y[u] - mj) * ij;
      const double g = om[u] * exp(lj - 0.5 * z * z - lse[u]);
      s0 += g; s1 += g * z; s2 += g * (z * z - 1.0);
    }
    s0 = warp_sum_d(s0); s1 = warp_sum_d(s1); s2 = warp_sum_d(s2);
    if (lane == j) { gl = -s0; gm = -s1 * ij; gs = -s2 * ij; }
  }
  const double sum_gl = warp_sum_d(gl);
  const double ev = warp_sum_d(q.w * q.mu), evt = warp_sum_d(t.w * t.mu);
  const double gscale = double(a.h.grad_scale) * double(isw);
  if (on && a.h.dq) {
    a.h.dq[ro + lane] = float((gl - q.w * sum_gl) * gscale);       // softmax Jacobian
    a.h.dq[ro + K + lane] = float(gm * gscale);
    a.h.dq[ro + 2 * K + lane] = float(gs * q.dsigma * gscale);     // softplus'
  }
  if (lane == 0) {
    const float tdv = float(ev - (r + c * evt));
    if (a.h.loss_rows) a.h.loss_rows[row] = float(loss * double(isw));
    if (a.h.td) a.h.td[row] = tdv;
    if (a.h.prio) a.h.prio[row] = fabsf(tdv) + float(a.h.prio_eps);
  }
}

// policy part of one row: -E[Q] and its raw-head gradient (sigma does not enter)
__device__ __forceinline__ void mog_policy_row(const MogArgs& a, int row, int lane) {
  const int K = a.K;
  const size_t ro = size_t(row) * a.h.ld;
  const MogComp p = mog_comp(a.h.pi + ro, K, lane);
  const double ev = warp_sum_d(p.w * p.mu);
  const double gsc = double(a.h.grad_scale);
  if (lane < K && a.h.dpi) {
    a.h.dpi[ro + lane] = float(-gsc * p.w * (p.mu - ev));
    a.h.dpi[ro + K + lane] = float(-gsc * p.w);
    a.h.dpi[ro + 2 * K + lane] = 0.f;
  }
  if (lane == 0 && a.h.pi_rows) a.h.pi_rows[row] = float(-ev);
}

// warps [0, B): critic part of row g; [B, 2B): policy part of row g - B (only_policy: warps [0, B) run the policy part).
// The post-update plan's first launch has no policy head (pi null): its grid covers B warps only, rounded up to whole
// blocks, and the warps past B must not run a policy row.
// Also does what heads_kernel does for the step besides the maths: PDL wait / trigger, the step stamps and the
// sampler-clock advance of the prefetch / host pipelines.
// __maxnreg__(255): without it ptxas aims at 64-96 registers and spills the per-point arrays (blocks are 128 threads).
// HZ: the batch carries per-row horizons (episode tails); a separate instantiation, so the plain one keeps its registers
template <int NT, bool HZ>
__global__ void __maxnreg__(255) mog_heads_kernel(const MogArgs a) {
  pdl_trigger(a.h.pdl);
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x * MOG_WARPS + warp;
  step_stamp(a.h.trace, 2);
  if (a.h.only_policy) { if (g < a.h.B) mog_policy_row(a, g, lane); }
  else if (g < a.h.B) mog_critic_row<NT, HZ>(a, g, lane);
  else if (a.h.pi && g < 2 * a.h.B) mog_policy_row(a, g - a.h.B, lane);
  step_stamp(a.h.trace, 2 + 16);
  if (a.h.sampler_clock && blockIdx.x == 0 && threadIdx.x == 0) {
    a.h.sampler_clock->s_adam_step += 1; a.h.sampler_clock->s_beta_t += 1; a.h.sampler_clock->s_steps_done += 1;
  }
  pdl_trigger_end(a.h.pdl);
}

template <bool HZ>
static int launch_mog_heads_nt(const MogArgs& a, dim3 grid, dim3 block, cudaStream_t st) {
  D4PG_MAX_CARVEOUT((mog_heads_kernel<1, HZ>)); D4PG_MAX_CARVEOUT((mog_heads_kernel<2, HZ>));
  D4PG_MAX_CARVEOUT((mog_heads_kernel<4, HZ>)); D4PG_MAX_CARVEOUT((mog_heads_kernel<8, HZ>));
  // NT = quadrature points per lane: 8K points over 32 lanes
  if (a.K <= 4) D4PG_CUDA_OK(launch_pdl(mog_heads_kernel<1, HZ>, grid, block, 0, st, a));
  else if (a.K <= 8) D4PG_CUDA_OK(launch_pdl(mog_heads_kernel<2, HZ>, grid, block, 0, st, a));
  else if (a.K <= 16) D4PG_CUDA_OK(launch_pdl(mog_heads_kernel<4, HZ>, grid, block, 0, st, a));
  else D4PG_CUDA_OK(launch_pdl(mog_heads_kernel<8, HZ>, grid, block, 0, st, a));
  return D4PG_OK;
}

int launch_mog_heads(const MogArgs& a_in, cudaStream_t st) {
  MogArgs a = a_in;
  a.h.pdl = pdl_mode();
  a.h.trace = (a.h.sampler_clock && debug_trace_buffer()) ? debug_trace_buffer() + STEP_TRACE_BASE : nullptr;
  dim3 grid(cdiv(((a.h.pi && !a.h.only_policy) ? 2 : 1) * a.h.B, MOG_WARPS)), block(MOG_WARPS * 32);
  if (a.h.horizon) return launch_mog_heads_nt<true>(a, grid, block, st);
  return launch_mog_heads_nt<false>(a, grid, block, st);
}

// raw head [B, ldr] -> w, mu, sigma [B, K] (dense), one warp per row
__global__ void mog_transform_kernel(const float* __restrict__ raw, int ldr, int B, int K, float* __restrict__ w,
                                     float* __restrict__ mu, float* __restrict__ sigma) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= B) return;
  const MogComp c = mog_comp(raw + size_t(row) * ldr, K, lane);
  if (lane < K) {
    const size_t o = size_t(row) * K + lane;
    w[o] = float(c.w); mu[o] = float(c.mu); sigma[o] = float(c.sigma);
  }
}

// (g_w, g_mu, g_sigma) [B, K] (a NULL term counts as zero) -> dZ of the raw head [B, ldz] (pad columns written as zero):
//   dz_w = w (g_w - sum_j g_w,j w_j),  dz_mu = g_mu,  dz_sigma = g_sigma softplus'(raw)
__global__ void mog_head_backward_kernel(const float* __restrict__ raw, int ldr, const float* __restrict__ gw,
                                         const float* __restrict__ gmu, const float* __restrict__ gsig, int B, int K,
                                         float* __restrict__ dz, int ldz) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= B) return;
  const MogComp c = mog_comp(raw + size_t(row) * ldr, K, lane);
  const bool on = lane < K;
  const size_t o = size_t(row) * K + lane;
  const double g_w = (on && gw) ? double(gw[o]) : 0.0;
  const double dot = warp_sum_d(g_w * c.w);
  float* out = dz + size_t(row) * ldz;
  if (on) {
    out[lane] = float(c.w * (g_w - dot));
    out[K + lane] = gmu ? gmu[o] : 0.f;
    out[2 * K + lane] = gsig ? float(double(gsig[o]) * c.dsigma) : 0.f;
  }
  for (int k = 3 * K + lane; k < ldz; k += 32) out[k] = 0.f;
}

int launch_mog_transform(const float* raw, int ldr, int B, int K, float* w, float* mu, float* sigma, cudaStream_t st) {
  mog_transform_kernel<<<cdiv(B * 32, 256), 256, 0, st>>>(raw, ldr, B, K, w, mu, sigma);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}
int launch_mog_head_backward(const float* raw, int ldr, const float* gw, const float* gmu, const float* gsig, int B, int K,
                             float* dz, int ldz, cudaStream_t st) {
  mog_head_backward_kernel<<<cdiv(B * 32, 256), 256, 0, st>>>(raw, ldr, gw, gmu, gsig, B, K, dz, ldz);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

}  // namespace d4pg

extern "C" int32_t d4pg_mog_quadrature(double* x, double* h) {
  using namespace d4pg;
  D4PG_REQUIRE(x && h, D4PG_EINVAL, "d4pg_mog_quadrature: null argument");
  for (int q = 0; q < MOG_Q; ++q) { x[q] = h_gh_x[q]; h[q] = h_gh_h[q]; }
  return D4PG_OK;
}

extern "C" int32_t d4pg_mog_loss(const float* target_raw, const float* q_raw, const float* pi_raw,
                                 const double* rewards, const uint8_t* dones, int32_t B, int32_t K,
                                 double discount, double prio_eps, float grad_scale,
                                 float* loss_rows, float* td, float* prio, float* dq_raw,
                                 float* pi_rows, float* dpi_raw, d4pg_stream_t stream) {
  using namespace d4pg;
  D4PG_REQUIRE(target_raw && q_raw && rewards && dones, D4PG_EINVAL, "d4pg_mog_loss: null input");
  D4PG_REQUIRE(B > 0 && K >= 1 && K <= D4PG_MAX_COMPONENTS, D4PG_EINVAL,
               "d4pg_mog_loss: need B>0, 1<=K<=%d (got B=%d K=%d)", D4PG_MAX_COMPONENTS, B, K);
  MogArgs a{};
  a.h.target = target_raw; a.h.q = q_raw; a.h.pi = pi_raw;
  a.h.rewards = rewards; a.h.dones = dones; a.h.B = B; a.K = K; a.h.ld = 3 * K;
  a.h.discount = discount; a.h.prio_eps = prio_eps; a.h.grad_scale = grad_scale;
  a.h.loss_rows = loss_rows; a.h.td = td; a.h.prio = prio; a.h.dq = dq_raw; a.h.pi_rows = pi_rows; a.h.dpi = dpi_raw;
  return launch_mog_heads(a, as_stream(stream));
}

// critic.forward of a mixture critic: the categorical critic's MLP with a 3K-wide fc3, then the head transform
extern "C" int32_t d4pg_critic_forward_mog(const float* params, int32_t obs_dim, int32_t act_dim, int32_t K,
                                           const float* s, const float* a, int32_t B, float* w, float* mu, float* sigma,
                                           float* raw, float* workspace, int32_t precision, d4pg_stream_t stream) {
  using namespace d4pg;
  D4PG_REQUIRE(w && mu && sigma && workspace && B > 0, D4PG_EINVAL, "d4pg_critic_forward_mog: null/empty argument");
  D4PG_REQUIRE(K >= 1 && K <= D4PG_MAX_COMPONENTS, D4PG_EINVAL, "d4pg_critic_forward_mog: K=%d outside [1,%d]", K, D4PG_MAX_COMPONENTS);
  float* z = raw ? raw : workspace;                    // h1 is dead after fc2 (as in d4pg_critic_forward)
  const int rc = d4pg_critic_forward(params, obs_dim, act_dim, 3 * K, s, a, B, nullptr, z, workspace, precision, stream);
  if (rc) return rc;
  return launch_mog_transform(z, 3 * K, B, K, w, mu, sigma, as_stream(stream));
}
