// Quantile-regression critic head (critic_dist_info['type'] == 'quantile', N quantiles): the fused quantile-Huber loss /
// TD / priority / quantile-gradient row kernel of the learner step.  The critic module needs no kernel of its own: its
// output is the raw fc3 row (d4pg_critic_forward without the softmax) and its head backward passes the gradient through.
//
// DERIVED semantics (QR-DQN, Dabney et al. 2018; the reference has no quantile code):
//   theta_k = fc3 row, tau_k = (2k+1) / (2N);  c = discount * (1 - done_i);  y_j = r_i + c theta'_j;  u_jk = y_j - theta_k
//   H(u) = u^2/2 for |u| <= kappa, kappa (|u| - kappa/2) otherwise;  rho_jk = |tau_k - 1{u_jk < 0}| H(u_jk) / kappa
//   loss row L_i = (1/N) sum_j sum_k rho_jk;  dL_i/dtheta_k = -(1/N) sum_j |tau_k - 1{u_jk < 0}| clamp(u_jk, -kappa, kappa) / kappa
//   td_i = mean_k theta_k - (r_i + c mean_j theta'_j);  priority |td_i| + eps, or L_i + eps (ce_priority)
//   policy row: -mean_k theta_k on critic(s, actor(s)), gradient -1/N per quantile
// One warp per row.  Lane owns quantiles k = lane + 32 t (t < NT = ceil(N/32)); the row's N targets are staged once per
// warp in shared memory and each lane walks all of them for its own quantiles, so the per-quantile gradient sums need no
// cross-lane reduction (only the loss row and the two means of td are warp sums).  The N^2 pair terms are evaluated in
// fp64 from the fp32 rows (u = y - theta keeps full precision whatever the reward's magnitude) and rounded to fp32 at the
// end.  No atomics: results are run-to-run identical.
#include "internal.cuh"

namespace d4pg {

constexpr int QR_WARPS = 4;

__device__ __forceinline__ double qr_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// critic part of one row: loss row, td, priority, d loss / d theta.  `ys` = this warp's staging row of N targets.
template <int NT>
__device__ __forceinline__ void qr_critic_row(const QrArgs& a, int row, int lane, double* ys) {
  const int N = a.N;
  const size_t ro = size_t(row) * a.h.ld;
  const double r = a.h.rewards[row];
  const double c = a.h.dones[row] ? 0.0 : head_discount(a.h, row);
  const float isw = a.h.is_weights ? __ldg(a.h.is_weights + row) : 1.f;
  const double kap = a.kappa;
  double th[NT], tau[NT], g[NT], ls[NT];
  double sum_t = 0.0, sum_q = 0.0;
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    const int k = lane + 32 * t;
    const bool on = k < N;
    const double tp = on ? double(__ldg(a.h.target + ro + k)) : 0.0;
    if (on) ys[k] = r + c * tp;
    sum_t += tp;
    th[t] = on ? double(__ldg(a.h.q + ro + k)) : 0.0;
    sum_q += th[t];
    tau[t] = double(2 * k + 1) / double(2 * N);
    g[t] = 0.0; ls[t] = 0.0;
  }
  __syncwarp();
  // sum_j w c and sum_j w c (u - c/2) = sum_j w H(u), with c = clamp(u, -kappa, kappa) and w = tau or 1 - tau
  for (int j = 0; j < N; ++j) {
    const double y = ys[j];
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const double u = y - th[t];
      const double cu = fmin(fmax(u, -kap), kap);
      const double wc = (u < 0.0 ? 1.0 - tau[t] : tau[t]) * cu;
      g[t] += wc;
      ls[t] = fma(wc, fma(-0.5, cu, u), ls[t]);
    }
  }
  __syncwarp();                                     // ys is reused by the warp's next row
  double loss = 0.0;
#pragma unroll
  for (int t = 0; t < NT; ++t) loss += (lane + 32 * t < N) ? ls[t] : 0.0;
  const double invN = 1.0 / double(N);
  loss = qr_warp_sum(loss) * invN / kap;
  const double gscale = double(a.h.grad_scale) * double(isw);
  if (a.h.dq) {
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const int k = lane + 32 * t;
      if (k < N) a.h.dq[ro + k] = float(-g[t] * invN / kap * gscale);
    }
  }
  sum_t = qr_warp_sum(sum_t); sum_q = qr_warp_sum(sum_q);
  if (lane == 0) {
    const float tdv = float(sum_q * invN - (r + c * (sum_t * invN)));
    if (a.h.loss_rows) a.h.loss_rows[row] = float(loss * double(isw));
    if (a.h.td) a.h.td[row] = tdv;
    if (a.h.prio) a.h.prio[row] = (a.ce_priority ? float(loss) : fabsf(tdv)) + float(a.h.prio_eps);
  }
}

// policy part of one row: -mean_k theta_k and its gradient -grad_scale / N
template <int NT>
__device__ __forceinline__ void qr_policy_row(const QrArgs& a, int row, int lane) {
  const int N = a.N;
  const size_t ro = size_t(row) * a.h.ld;
  double s = 0.0;
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    const int k = lane + 32 * t;
    if (k < N) s += double(__ldg(a.h.pi + ro + k));
  }
  s = qr_warp_sum(s);
  if (a.h.dpi) {
    const float gk = float(-double(a.h.grad_scale) / double(N));
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const int k = lane + 32 * t;
      if (k < N) a.h.dpi[ro + k] = gk;
    }
  }
  if (lane == 0 && a.h.pi_rows) a.h.pi_rows[row] = float(-s / double(N));
}

// warps [0, B): critic part of row g; [B, 2B): policy part of row g - B (only_policy: warps [0, B) run the policy part).
// The post-update plan's first launch has no policy head (pi null): its grid covers B warps only, rounded up to whole
// blocks, and the warps past B must not run a policy row.
// Also does what heads_kernel does for the step besides the maths: PDL wait / trigger, the step stamps and the
// sampler-clock advance of the prefetch / host pipelines.
template <int NT>
__global__ void __launch_bounds__(QR_WARPS * 32) qr_heads_kernel(const QrArgs a) {
  __shared__ double ys[QR_WARPS][32 * NT];
  pdl_trigger(a.h.pdl);
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x * QR_WARPS + warp;
  step_stamp(a.h.trace, 2);
  if (a.h.only_policy) { if (g < a.h.B) qr_policy_row<NT>(a, g, lane); }
  else if (g < a.h.B) qr_critic_row<NT>(a, g, lane, ys[warp]);
  else if (a.h.pi && g < 2 * a.h.B) qr_policy_row<NT>(a, g - a.h.B, lane);
  step_stamp(a.h.trace, 2 + 16);
  if (a.h.sampler_clock && blockIdx.x == 0 && threadIdx.x == 0) {
    a.h.sampler_clock->s_adam_step += 1; a.h.sampler_clock->s_beta_t += 1; a.h.sampler_clock->s_steps_done += 1;
  }
  pdl_trigger_end(a.h.pdl);
}

int launch_qr_heads(const QrArgs& a_in, cudaStream_t st) {
  QrArgs a = a_in;
  a.h.pdl = pdl_mode();
  a.h.trace = (a.h.sampler_clock && debug_trace_buffer()) ? debug_trace_buffer() + STEP_TRACE_BASE : nullptr;
  dim3 grid(cdiv(((a.h.pi && !a.h.only_policy) ? 2 : 1) * a.h.B, QR_WARPS)), block(QR_WARPS * 32);
  D4PG_MAX_CARVEOUT(qr_heads_kernel<1>); D4PG_MAX_CARVEOUT(qr_heads_kernel<2>);
  D4PG_MAX_CARVEOUT(qr_heads_kernel<3>); D4PG_MAX_CARVEOUT(qr_heads_kernel<4>);
  // NT = quantiles per lane
  if (a.N <= 32) D4PG_CUDA_OK(launch_pdl(qr_heads_kernel<1>, grid, block, 0, st, a));
  else if (a.N <= 64) D4PG_CUDA_OK(launch_pdl(qr_heads_kernel<2>, grid, block, 0, st, a));
  else if (a.N <= 96) D4PG_CUDA_OK(launch_pdl(qr_heads_kernel<3>, grid, block, 0, st, a));
  else D4PG_CUDA_OK(launch_pdl(qr_heads_kernel<4>, grid, block, 0, st, a));
  return D4PG_OK;
}

}  // namespace d4pg

extern "C" int32_t d4pg_qr_loss(const float* target_q, const float* q, const float* pi_q,
                                const double* rewards, const uint8_t* dones, int32_t B, int32_t N,
                                double discount, double kappa, double prio_eps, float grad_scale, int32_t ce_priority,
                                float* loss_rows, float* td, float* prio, float* dq,
                                float* pi_rows, float* dpi, d4pg_stream_t stream) {
  using namespace d4pg;
  D4PG_REQUIRE(target_q && q && rewards && dones, D4PG_EINVAL, "d4pg_qr_loss: null input");
  D4PG_REQUIRE(B > 0 && N >= 2 && N <= D4PG_MAX_ATOMS, D4PG_EINVAL,
               "d4pg_qr_loss: need B>0, 2<=N<=%d (got B=%d N=%d)", D4PG_MAX_ATOMS, B, N);
  D4PG_REQUIRE(std::isfinite(kappa) && kappa > 0.0, D4PG_EINVAL, "d4pg_qr_loss: kappa must be finite and > 0 (got %g)", kappa);
  QrArgs a{};
  a.h.target = target_q; a.h.q = q; a.h.pi = pi_q;
  a.h.rewards = rewards; a.h.dones = dones; a.h.B = B; a.N = N; a.h.ld = N;
  a.h.discount = discount; a.kappa = kappa; a.h.prio_eps = prio_eps; a.h.grad_scale = grad_scale;
  a.ce_priority = ce_priority ? 1 : 0;
  a.h.loss_rows = loss_rows; a.h.td = td; a.h.prio = prio; a.h.dq = dq; a.h.pi_rows = pi_rows; a.h.dpi = dpi;
  return launch_qr_heads(a, as_stream(stream));
}
