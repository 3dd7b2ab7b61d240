// Standalone backward of the actor / critic forward entry points (abi.cu): the autograd backward of
// models.py:32-41 / 76-88 for callers that own the loss (the reference's learner body ddpg.py:229-244
// written against the modules, other losses, gradient checks).
//
// One small kernel turns the upstream gradient of the network's output into the output layer's dZ (tanh'
// for the actor, the softmax Jacobian for the critic); everything else runs on the level GEMMs the learner's
// PLAN_LEVELS backward uses (gemm_ffma / gemm_tc / gemm_bf16 through gemm_launch), one grouped launch per
// layer: dX of layer l (activation mask fused into its epilogue) and dW of layer l (bias gradient fused)
// share the launch.  So every precision computes exactly the arithmetic of the learner's levels.
#include "common.cuh"
#include "gemm_ffma.cuh"

namespace d4pg {

// dZ of the output layer, one warp per row, into a plane of row pitch ldz (pad columns written as zero).
//   tanh head (softmax == 0):  dz = gy * (1 - y^2)                          y = the saved tanh output
//   softmax head (softmax == 1): dz = gz + y * (gy - sum_j gy_j y_j)          y = the saved probabilities
// gy / gz are [B, N] dense; a NULL term counts as zero.
__global__ void head_backward_kernel(const float* __restrict__ y, const float* __restrict__ gy,
                                     const float* __restrict__ gz, float* __restrict__ dz, int B, int N, int ldz,
                                     int softmax) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B) return;
  const size_t row = size_t(warp) * N;
  float* out = dz + size_t(warp) * ldz;
  if (!softmax) {
    for (int k = lane; k < ldz; k += 32) {
      float v = 0.f;
      if (k < N) { const float t = y[row + k]; v = gy[row + k] * (1.f - t * t); }
      out[k] = v;
    }
    return;
  }
  float dot = 0.f;
  if (gy) {
    for (int k = lane; k < N; k += 32) dot += gy[row + k] * y[row + k];
    dot = warp_sum(dot);
  }
  for (int k = lane; k < ldz; k += 32) {
    float v = 0.f;
    if (k < N) {
      if (gy) v = y[row + k] * (gy[row + k] - dot);
      if (gz) v += gz[row + k];
    }
    out[k] = v;
  }
}

int launch_mog_head_backward(const float* raw, int ldr, const float* gw, const float* gmu, const float* gsig, int B, int K,
                             float* dz, int ldz, cudaStream_t st);      // mog_heads.cu

// The levels fc3 -> fc2_2 -> fc2 -> fc1 of a network from the output layer's dZ plane `dz` [B, pitch4(out[3])], held in
// scratch behind the two [B, H] delta planes p0 / p1, which the levels use in turn.  Level l is one grouped launch: the
// dX of layer l (masked by dx_mask) and the dW of layer l with its bias gradient.  The critic's fc2 (a != NULL) adds its
// action columns W2[:, H:]: dX = grad_a, dW without bias.  grad_params is cleared first (pads stay zero; split-K dW
// adds); a NULL gradient drops the problems that only it needs.  The caller checked the arguments.
static int net_backward(const NetDims& d, const float* params, const float* s, const float* a, int B,
                        const float* workspace, const float* dz, float* grad_params, float* grad_s, float* grad_a,
                        float* scratch, int precision, cudaStream_t st) {
  const int H = D4PG_HIDDEN, A = a ? d.in[1] - H : 0;
  const float* h[3] = {workspace, workspace + size_t(B) * H, workspace + size_t(B) * 2 * H};
  float* p[2] = {scratch, scratch + size_t(B) * H};
  const float* W = params; float* G = grad_params;
  if (G) D4PG_CUDA_OK(cudaMemsetAsync(G, 0, size_t(d.total) * sizeof(float), st));
  for (int l = 3; l >= 0; --l) {
    // level l reads the dZ level l+1 wrote (p0 from fc3, p1 from fc2_2, p0 from fc2) and writes the other plane
    const float* Z = l == 3 ? dz : p[l % 2];
    const int ldz = l == 3 ? pitch4(d.out[3]) : H;
    const float* X = l ? h[l - 1] : s;
    const int n_in = l ? H : d.in[0], mask = dx_mask(d, l);
    float* dX = l ? p[(l + 1) % 2] : grad_s;
    GemmBatch g; gemm_batch_begin(g);
    if (dX && (l != 1 || G || grad_s))     // fc2's dX (fc1's dZ) feeds only dW1 and grad_s
      gemm_batch_add(g, gemm_dx(Z, ldz, W + d.w_off[l], d.ld[l], dX, n_in, B, n_in, d.out[l], mask,
                                mask == EPI_NONE ? nullptr : X, mask == EPI_NONE ? 0 : n_in));
    if (l == 1 && grad_a)
      gemm_batch_add(g, gemm_dx(Z, ldz, W + d.w_off[1] + H, d.ld[1], grad_a, A, B, A, H, EPI_NONE, nullptr, 0));
    if (G) gemm_batch_add(g, gemm_dw(Z, ldz, X, n_in, G + d.w_off[l], d.ld[l], G + d.b_off[l], d.out[l], n_in, B));
    if (l == 1 && G && a) gemm_batch_add(g, gemm_dw(Z, ldz, a, A, G + d.w_off[1] + H, d.ld[1], nullptr, H, A, B));
    if (g.n) {
      const int rc = gemm_launch(g, precision, st);
      if (rc) return rc;
    }
  }
  return D4PG_OK;
}

}  // namespace d4pg

using namespace d4pg;

// actor: tanh' into the fc3 dZ plane, then the levels
extern "C" int32_t d4pg_actor_backward(const float* params, int32_t obs_dim, int32_t act_dim, const float* s, int32_t B,
                                       const float* action, const float* workspace, const float* grad_action,
                                       float* grad_params, float* grad_s, float* scratch, int32_t precision,
                                       d4pg_stream_t stream) {
  D4PG_REQUIRE(params && s && action && workspace && grad_action && scratch && B > 0 && obs_dim > 0 && act_dim > 0,
               D4PG_EINVAL, "d4pg_actor_backward: null/empty argument");
  D4PG_REQUIRE(precision >= 0 && precision <= 3, D4PG_ENOTSUP, "d4pg_actor_backward: unknown precision %d", precision);
  if (!grad_params && !grad_s) return D4PG_OK;
  // scratch holds B*(2H + max(H, Ap)) floats: the fc3 dZ plane [B, Ap] may be wider than H
  float* dz = scratch + size_t(B) * 2 * D4PG_HIDDEN;
  cudaStream_t st = as_stream(stream);
  head_backward_kernel<<<cdiv(B * 32, 256), 256, 0, st>>>(action, grad_action, nullptr, dz, B, act_dim, pitch4(act_dim), 0);
  D4PG_LAUNCH_OK();
  return net_backward(actor_dims(obs_dim, act_dim), params, s, nullptr, B, workspace, dz, grad_params, grad_s, nullptr,
                      scratch, precision, st);
}

// critic: the softmax Jacobian (or the logits' own gradient) into the fc3 dZ plane, then the levels
extern "C" int32_t d4pg_critic_backward(const float* params, int32_t obs_dim, int32_t act_dim, int32_t n_atoms,
                                        const float* s, const float* a, int32_t B, const float* probs,
                                        const float* workspace, const float* grad_probs, const float* grad_logits,
                                        float* grad_params, float* grad_s, float* grad_a, float* scratch,
                                        int32_t precision, d4pg_stream_t stream) {
  D4PG_REQUIRE(params && s && a && workspace && scratch && B > 0 && obs_dim > 0 && act_dim > 0, D4PG_EINVAL,
               "d4pg_critic_backward: null/empty argument");
  D4PG_REQUIRE(grad_probs || grad_logits, D4PG_EINVAL, "d4pg_critic_backward: grad_probs and grad_logits are both NULL");
  D4PG_REQUIRE(probs || !grad_probs, D4PG_EINVAL, "d4pg_critic_backward: grad_probs needs probs");
  D4PG_REQUIRE(n_atoms >= 2 && n_atoms <= D4PG_MAX_ATOMS, D4PG_EINVAL, "d4pg_critic_backward: n_atoms out of range");
  D4PG_REQUIRE(precision >= 0 && precision <= 3, D4PG_ENOTSUP, "d4pg_critic_backward: unknown precision %d", precision);
  const int Np = pitch4(n_atoms);
  float* dz = scratch + size_t(B) * 2 * D4PG_HIDDEN;
  if (!grad_params && !grad_s && !grad_a) return D4PG_OK;
  head_backward_kernel<<<cdiv(B * 32, 256), 256, 0, as_stream(stream)>>>(probs, grad_probs, grad_logits, dz, B, n_atoms, Np, 1);
  D4PG_LAUNCH_OK();
  return net_backward(critic_dims(obs_dim, act_dim, n_atoms), params, s, a, B, workspace, dz, grad_params, grad_s, grad_a,
                      scratch, precision, as_stream(stream));
}

// mixture-of-Gaussians critic (mog_heads.cu): the raw head's dZ from (g_w, g_mu, g_sigma), then the same levels
extern "C" int32_t d4pg_critic_backward_mog(const float* params, int32_t obs_dim, int32_t act_dim, int32_t K,
                                            const float* s, const float* a, int32_t B, const float* raw,
                                            const float* workspace, const float* grad_w, const float* grad_mu,
                                            const float* grad_sigma, float* grad_params, float* grad_s, float* grad_a,
                                            float* scratch, int32_t precision, d4pg_stream_t stream) {
  D4PG_REQUIRE(params && s && a && raw && workspace && scratch && B > 0 && obs_dim > 0 && act_dim > 0, D4PG_EINVAL,
               "d4pg_critic_backward_mog: null/empty argument");
  D4PG_REQUIRE(grad_w || grad_mu || grad_sigma, D4PG_EINVAL, "d4pg_critic_backward_mog: grad_w, grad_mu and grad_sigma are all NULL");
  D4PG_REQUIRE(K >= 1 && K <= D4PG_MAX_COMPONENTS, D4PG_EINVAL, "d4pg_critic_backward_mog: K=%d outside [1,%d]", K, D4PG_MAX_COMPONENTS);
  D4PG_REQUIRE(precision >= 0 && precision <= 3, D4PG_ENOTSUP, "d4pg_critic_backward_mog: unknown precision %d", precision);
  if (!grad_params && !grad_s && !grad_a) return D4PG_OK;
  const int N = 3 * K;
  float* dz = scratch + size_t(B) * 2 * D4PG_HIDDEN;
  const int rc = launch_mog_head_backward(raw, N, grad_w, grad_mu, grad_sigma, B, K, dz, pitch4(N), as_stream(stream));
  if (rc) return rc;
  return net_backward(critic_dims(obs_dim, act_dim, N), params, s, a, B, workspace, dz, grad_params, grad_s, grad_a,
                      scratch, precision, as_stream(stream));
}
