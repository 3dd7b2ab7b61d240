// Fused Adam (beta=(0.9,0.9) by default) + Polyak soft target update over flat fp32 buffers.
//
// Replaces (reference, relative to its repository root):
//   shared_adam.py:3-17 + torch.optim.Adam.step as called at ddpg.py:232,244.  Arithmetic follows
//     torch 2.11 `_single_tensor_adam` (the form the reference executes in this image):
//       m <- lerp(m, g, 1-b1); v <- v*b2 + (1-b2)*g*g;
//       p <- p - (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps),  bc = 1 - b^step
//   ddpg.py:118-120 sync_local_global: identity (local and global share storage)
//   ddpg.py:110-116 update_target_parameters: t <- (1-tau)*t + tau*p   (p = post-step value)
// Pure streaming kernel: 4 reads + 4 writes of P floats -> HBM/L2 bound, float4 vectorised.
#include "adam_dev.cuh"
#include <math.h>
#include <cmath>
#include <algorithm>

namespace d4pg {

__global__ void __launch_bounds__(256) adam_polyak_kernel(const AdamArgs a) {
  __shared__ float red[2][8];
  pdl_trigger(a.pdl);
  pdl_wait();
  if (int(blockIdx.y) == a.nseg) {
    if (blockIdx.x == 0) adam_tail(a, red);
    return;
  }
  step_stamp(a.trace, 7);
  adam_segment<false>(a, blockIdx.y, blockIdx.x, gridDim.x);
  step_stamp(a.trace, 7 + 16);
  pdl_trigger_end(a.pdl);
}

// the same update on the effective gradient coef * g + wd * p: global-norm clipping and / or weight decay
__global__ void __launch_bounds__(256) adam_polyak_clip_kernel(const AdamArgs a) {
  __shared__ float red[2][8];
  __shared__ double bcast;
  pdl_trigger(a.pdl);
  pdl_wait();
  if (int(blockIdx.y) == a.nseg) {
    if (blockIdx.x == 0) adam_tail(a, red);
    return;
  }
  step_stamp(a.trace, 7);
  adam_segment<true>(a, blockIdx.y, blockIdx.x, gridDim.x, &bcast);
  step_stamp(a.trace, 7 + 16);
  pdl_trigger_end(a.pdl);
}

static_assert(GRAD_NORM_CTAS == 64, "clip_coef sums the partials as one warp, two per lane");
__global__ void __launch_bounds__(256) grad_sqnorm_kernel(const GradNormArgs a) {
  __shared__ double red[8];
  pdl_trigger(a.pdl);
  pdl_wait();                                                   // the gradient is the previous launches' output
  const int sg = blockIdx.y;                                    // (selects, not indexing: the arguments stay in constant memory)
  const float4* g4 = reinterpret_cast<const float4*>(sg ? a.g[1] : a.g[0]);
  const int64_t n4 = (sg ? a.n[1] : a.n[0]) >> 2;
  double acc = 0.0;
  for (int64_t i = blockIdx.x * int64_t(256) + threadIdx.x; i < n4; i += int64_t(GRAD_NORM_CTAS) * 256) {
    const float4 g = g4[i];
    const double x = g.x, y = g.y, z = g.z, w = g.w;
    acc += (x * x + y * y) + (z * z + w * w);
  }
  acc = warp_sum_f64(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += red[w];
    (sg ? a.partials[1] : a.partials[0])[blockIdx.x] = s;
  }
  pdl_trigger_end(a.pdl);
}

int launch_grad_sqnorm(const AdamArgs& a, cudaStream_t st) {
  GradNormArgs n{};
  for (int i = 0; i < a.nseg; ++i)
    if (a.seg[i].sq_partials) {
      n.g[n.nseg] = a.seg[i].g; n.partials[n.nseg] = const_cast<double*>(a.seg[i].sq_partials); n.n[n.nseg] = a.seg[i].n;
      ++n.nseg;
    }
  D4PG_REQUIRE(n.nseg > 0, D4PG_EINVAL, "launch_grad_sqnorm: no segment clips");
  n.pdl = pdl_mode();
  D4PG_MAX_CARVEOUT(grad_sqnorm_kernel);
  D4PG_CUDA_OK(launch_pdl(grad_sqnorm_kernel, dim3(GRAD_NORM_CTAS, n.nseg), dim3(256), 0, st, n));
  return D4PG_OK;
}


int launch_adam(const AdamArgs& a_in, cudaStream_t st) {
  AdamArgs a = a_in;
  a.pdl = pdl_mode();
  a.trace = (a.clock && debug_trace_buffer()) ? debug_trace_buffer() + STEP_TRACE_BASE : nullptr;
  int64_t nmax = 0;
  for (int i = 0; i < a.nseg; ++i) nmax = a.seg[i].n > nmax ? a.seg[i].n : nmax;
  int blocks = int((nmax / 4 + 255) / 256);
  if (blocks > 4 * device_sm_count()) blocks = 4 * device_sm_count();     // grid-stride: 4 CTAs per SM
  if (blocks < 1) blocks = 1;
  const int tail = ((a.clock || a.loss_out) && !a.skip_tail) ? 1 : 0;
  bool ex = adam_clips(a);
  for (int i = 0; i < a.nseg; ++i) ex = ex || a.seg[i].wd != 0.f;
  if (ex) {
    D4PG_MAX_CARVEOUT(adam_polyak_clip_kernel);
    D4PG_CUDA_OK(launch_pdl(adam_polyak_clip_kernel, dim3(blocks, a.nseg + tail), dim3(256), 0, st, a));
    return D4PG_OK;
  }
  D4PG_MAX_CARVEOUT(adam_polyak_kernel);
  D4PG_CUDA_OK(launch_pdl(adam_polyak_kernel, dim3(blocks, a.nseg + tail), dim3(256), 0, st, a));
  return D4PG_OK;
}

}  // namespace d4pg

using namespace d4pg;

extern "C" int32_t d4pg_adam_polyak_ex(float* p, const float* g, float* m, float* v, float* target, int64_t n,
                                       double lr, double beta1, double beta2, double eps, int64_t step,
                                       double tau, float grad_scale, d4pg_stream_t stream,
                                       double weight_decay, double max_grad_norm, double* partials, float* norm_out) {
  D4PG_REQUIRE(p && g && m && v, D4PG_EINVAL, "d4pg_adam_polyak: null buffer");
  D4PG_REQUIRE(n > 0 && n % 4 == 0, D4PG_EINVAL, "d4pg_adam_polyak: n must be a positive multiple of 4 (flat layout is 4-aligned)");
  D4PG_REQUIRE(step >= 1, D4PG_EINVAL, "d4pg_adam_polyak: step is the post-increment count (>= 1)");
  D4PG_REQUIRE(std::isfinite(weight_decay) && weight_decay >= 0.0, D4PG_EINVAL,
               "d4pg_adam_polyak_ex: weight_decay must be finite and >= 0 (got %g)", weight_decay);
  D4PG_REQUIRE(max_grad_norm == 0.0 || max_grad_norm > 0.0, D4PG_EINVAL,
               "d4pg_adam_polyak_ex: max_grad_norm must be 0 (off), +inf (report only) or > 0 (got %g)", max_grad_norm);
  D4PG_REQUIRE(max_grad_norm == 0.0 || partials, D4PG_EINVAL,
               "d4pg_adam_polyak_ex: clipping needs a device workspace of %d doubles", GRAD_NORM_CTAS);
  AdamArgs a{};
  const double bc1 = 1.0 - pow(beta1, double(step));
  const double bc2 = 1.0 - pow(beta2, double(step));
  a.seg[0] = AdamSeg{p, g, m, v, target, n, nullptr, 0, float(-(lr / bc1)), -1};
  a.seg[0].wd = float(weight_decay);
  if (max_grad_norm > 0.0) { a.seg[0].sq_partials = partials; a.seg[0].max_norm = max_grad_norm; a.seg[0].norm_out = norm_out; }
  a.nseg = 1;
  a.w1 = float(1.0 - beta1); a.w2 = float(1.0 - beta2); a.beta2 = float(beta2); a.eps = float(eps);
  a.bc2_sqrt = float(sqrt(bc2)); a.tau = float(tau); a.one_minus_tau = float(1.0 - tau);
  a.grad_scale = grad_scale; a.pipe_slot = -1;
  if (adam_clips(a))
    if (int rc = launch_grad_sqnorm(a, as_stream(stream))) return rc;
  return launch_adam(a, as_stream(stream));
}

extern "C" int32_t d4pg_adam_polyak(float* p, const float* g, float* m, float* v, float* target, int64_t n,
                                    double lr, double beta1, double beta2, double eps, int64_t step,
                                    double tau, float grad_scale, d4pg_stream_t stream) {
  return d4pg_adam_polyak_ex(p, g, m, v, target, n, lr, beta1, beta2, eps, step, tau, grad_scale, stream, 0.0, 0.0, nullptr, nullptr);
}

namespace d4pg {
__global__ void polyak_kernel(float* t, const float* s, int64_t n, float tau, float omt) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
    t[i] = __fadd_rn(__fmul_rn(omt, t[i]), __fmul_rn(tau, s[i]));
}
}  // namespace d4pg

extern "C" int32_t d4pg_polyak(float* target, const float* src, int64_t n, double tau, d4pg_stream_t stream) {
  D4PG_REQUIRE(target && src && n > 0, D4PG_EINVAL, "d4pg_polyak: bad arguments");
  int blocks = int(std::min<int64_t>(4 * d4pg::device_sm_count(), (n + 255) / 256));   // grid-stride
  polyak_kernel<<<blocks, 256, 0, as_stream(stream)>>>(target, src, n, float(tau), float(1.0 - tau));
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

extern "C" int32_t d4pg_copy_f32(float* dst, const float* src, int64_t n, d4pg_stream_t stream) {
  D4PG_REQUIRE(dst && src && n >= 0, D4PG_EINVAL, "d4pg_copy_f32: bad arguments");
  D4PG_CUDA_OK(cudaMemcpyAsync(dst, src, size_t(n) * sizeof(float), cudaMemcpyDeviceToDevice, as_stream(stream)));
  return D4PG_OK;
}
