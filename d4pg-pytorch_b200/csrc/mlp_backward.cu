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

static int launch_level(GemmBatch& b, int precision, cudaStream_t st) {
  return b.n ? gemm_launch(b, precision, st) : D4PG_OK;
}

}  // namespace d4pg

using namespace d4pg;

#define RUN_LEVEL(b)                                       \
  do {                                                     \
    const int _rc = launch_level(b, precision, st);        \
    if (_rc) return _rc;                                   \
  } while (0)

// actor: fc1 -> relu -> fc2 -> fc2_2 -> relu -> fc3 -> tanh (no relu after fc2, H9).  Levels fc3 -> fc2_2 -> fc2 -> fc1.
extern "C" int32_t d4pg_actor_backward(const float* params, int32_t obs_dim, int32_t act_dim, const float* s, int32_t B,
                                       const float* action, const float* workspace, const float* grad_action,
                                       float* grad_params, float* grad_s, float* scratch, int32_t precision,
                                       d4pg_stream_t stream) {
  D4PG_REQUIRE(params && s && action && workspace && grad_action && scratch && B > 0 && obs_dim > 0 && act_dim > 0,
               D4PG_EINVAL, "d4pg_actor_backward: null/empty argument");
  D4PG_REQUIRE(precision >= 0 && precision <= 3, D4PG_ENOTSUP, "d4pg_actor_backward: unknown precision %d", precision);
  const NetDims d = actor_dims(obs_dim, act_dim);
  const int H = D4PG_HIDDEN, S = obs_dim, A = act_dim, Ap = pitch4(act_dim);
  const float* h1 = workspace; const float* h2 = h1 + size_t(B) * H; const float* h3 = h2 + size_t(B) * H;
  // two delta planes + the head plane [B, Ap] (scratch holds B*(2H + max(H, Ap)) floats: act_dim may exceed H)
  float* p0 = scratch; float* p1 = p0 + size_t(B) * H; float* dz3 = p1 + size_t(B) * H;
  const float* W = params; float* G = grad_params;
  cudaStream_t st = as_stream(stream);
  if (!G && !grad_s) return D4PG_OK;
  if (G) D4PG_CUDA_OK(cudaMemsetAsync(G, 0, size_t(d.total) * sizeof(float), st));   // pads stay zero; split-K dW adds

  head_backward_kernel<<<cdiv(B * 32, 256), 256, 0, st>>>(action, grad_action, nullptr, dz3, B, A, Ap, 0);
  D4PG_LAUNCH_OK();
  GemmBatch g;
  // fc3: dz22 = (dz3 W3) * (h3 > 0);  dW3 = dz3^T h3
  gemm_batch_begin(g);
  gemm_batch_add(g, gemm_dx(dz3, Ap, W + d.w_off[3], d.ld[3], p0, H, B, H, A, EPI_RELU_MASK, h3, H));
  if (G) gemm_batch_add(g, gemm_dw(dz3, Ap, h3, H, G + d.w_off[3], d.ld[3], G + d.b_off[3], A, H, B));
  RUN_LEVEL(g);
  // fc2_2: its input h2 has no activation -> plain dX
  gemm_batch_begin(g);
  gemm_batch_add(g, gemm_dx(p0, H, W + d.w_off[2], d.ld[2], p1, H, B, H, H, EPI_NONE, nullptr, 0));
  if (G) gemm_batch_add(g, gemm_dw(p0, H, h2, H, G + d.w_off[2], d.ld[2], G + d.b_off[2], H, H, B));
  RUN_LEVEL(g);
  // fc2
  gemm_batch_begin(g);
  gemm_batch_add(g, gemm_dx(p1, H, W + d.w_off[1], d.ld[1], p0, H, B, H, H, EPI_RELU_MASK, h1, H));
  if (G) gemm_batch_add(g, gemm_dw(p1, H, h1, H, G + d.w_off[1], d.ld[1], G + d.b_off[1], H, H, B));
  RUN_LEVEL(g);
  // fc1: d state, dW1 = dz1^T s
  gemm_batch_begin(g);
  if (grad_s) gemm_batch_add(g, gemm_dx(p0, H, W + d.w_off[0], d.ld[0], grad_s, S, B, S, H, EPI_NONE, nullptr, 0));
  if (G) gemm_batch_add(g, gemm_dw(p0, H, s, S, G + d.w_off[0], d.ld[0], G + d.b_off[0], H, S, B));
  RUN_LEVEL(g);
  return D4PG_OK;
}

// the critic's levels fc3 -> fc2_2 -> fc2 -> fc1 from the output layer's dZ plane `dz` [B, pitch4(N)] (held in scratch
// behind the two delta planes); the caller checked the arguments
static int critic_levels(const float* params, int obs_dim, int act_dim, int n_atoms, const float* s, const float* a, int B,
                         const float* workspace, const float* dz, float* grad_params, float* grad_s, float* grad_a,
                         float* scratch, int precision, cudaStream_t st) {
  const NetDims d = critic_dims(obs_dim, act_dim, n_atoms);
  const int H = D4PG_HIDDEN, S = obs_dim, A = act_dim, N = n_atoms, Np = pitch4(n_atoms);
  const float* h1 = workspace; const float* h2 = h1 + size_t(B) * H; const float* h3 = h2 + size_t(B) * H;
  float* p0 = scratch; float* p1 = p0 + size_t(B) * H;
  const float* W = params; float* G = grad_params;
  if (!G && !grad_s && !grad_a) return D4PG_OK;
  if (G) D4PG_CUDA_OK(cudaMemsetAsync(G, 0, size_t(d.total) * sizeof(float), st));
  const bool need_dz1 = G || grad_s;

  GemmBatch g;
  // fc3
  gemm_batch_begin(g);
  gemm_batch_add(g, gemm_dx(dz, Np, W + d.w_off[3], d.ld[3], p0, H, B, H, N, EPI_RELU_MASK, h3, H));
  if (G) gemm_batch_add(g, gemm_dw(dz, Np, h3, H, G + d.w_off[3], d.ld[3], G + d.b_off[3], N, H, B));
  RUN_LEVEL(g);
  // fc2_2
  gemm_batch_begin(g);
  gemm_batch_add(g, gemm_dx(p0, H, W + d.w_off[2], d.ld[2], p1, H, B, H, H, EPI_RELU_MASK, h2, H));
  if (G) gemm_batch_add(g, gemm_dw(p0, H, h2, H, G + d.w_off[2], d.ld[2], G + d.b_off[2], H, H, B));
  RUN_LEVEL(g);
  // fc2: dh1 (masked), d action, dW2 = [dz2^T h1 | dz2^T a]
  gemm_batch_begin(g);
  if (need_dz1) gemm_batch_add(g, gemm_dx(p1, H, W + d.w_off[1], d.ld[1], p0, H, B, H, H, EPI_RELU_MASK, h1, H));
  if (grad_a) gemm_batch_add(g, gemm_dx(p1, H, W + d.w_off[1] + H, d.ld[1], grad_a, A, B, A, H, EPI_NONE, nullptr, 0));
  if (G) gemm_batch_add(g, gemm_dw(p1, H, h1, H, G + d.w_off[1], d.ld[1], G + d.b_off[1], H, H, B));
  if (G) gemm_batch_add(g, gemm_dw(p1, H, a, A, G + d.w_off[1] + H, d.ld[1], nullptr, H, A, B));
  RUN_LEVEL(g);
  // fc1
  if (need_dz1) {
    gemm_batch_begin(g);
    if (grad_s) gemm_batch_add(g, gemm_dx(p0, H, W + d.w_off[0], d.ld[0], grad_s, S, B, S, H, EPI_NONE, nullptr, 0));
    if (G) gemm_batch_add(g, gemm_dw(p0, H, s, S, G + d.w_off[0], d.ld[0], G + d.b_off[0], H, S, B));
    RUN_LEVEL(g);
  }
  return D4PG_OK;
}

// critic: fc1 -> relu -> cat(., a) -> fc2 -> relu -> fc2_2 -> relu -> fc3 -> softmax.  Levels fc3 -> fc2_2 -> fc2 -> fc1;
// fc2 splits into its h1 columns (dX masked by h1 > 0, dW with the bias gradient) and its action columns W2[:, H:]
// (dX = d action, dW without bias).
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
  return critic_levels(params, obs_dim, act_dim, n_atoms, s, a, B, workspace, dz, grad_params, grad_s, grad_a, scratch,
                       precision, as_stream(stream));
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
  return critic_levels(params, obs_dim, act_dim, N, s, a, B, workspace, dz, grad_params, grad_s, grad_a, scratch,
                       precision, as_stream(stream));
}
