// C-ABI plumbing: error channel, version, network layouts, standalone actor/critic forward.
#include "common.cuh"
#include "gemm_ffma.cuh"
#include <string.h>
#include <stdlib.h>

namespace d4pg {

static thread_local char g_err[512] = "";

int pdl_mode() {
  static const int m = getenv("D4PG_PDL") ? atoi(getenv("D4PG_PDL")) : 0;
  return m;
}
bool pdl_enabled() {
  // opt-in: D4PG_PDL=1 enables it (tools/ab_pdl.sh compares the modes).
  static const bool on = getenv("D4PG_PDL") != nullptr;
  return on;
}

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static NetDims make_dims(const int* in, const int* out, const int* epi) {
  NetDims d{};
  int64_t off = 0;
  for (int l = 0; l < 4; ++l) {
    d.in[l] = in[l]; d.out[l] = out[l]; d.ld[l] = pitch4(in[l]); d.epi[l] = epi[l];
    d.w_off[l] = off; off = align4(off + int64_t(d.ld[l]) * out[l]);
    d.b_off[l] = off; off = align4(off + out[l]);
  }
  d.total = off;
  return d;
}
// models.py:33-40: fc1 -> relu -> fc2 -> fc2_2 -> relu -> fc3 -> tanh (no relu after fc2, SURVEY.md H9)
NetDims actor_dims(int obs_dim, int act_dim) {
  const int in[4] = {obs_dim, D4PG_HIDDEN, D4PG_HIDDEN, D4PG_HIDDEN};
  const int out[4] = {D4PG_HIDDEN, D4PG_HIDDEN, D4PG_HIDDEN, act_dim};
  const int epi[4] = {EPI_BIAS_RELU, EPI_BIAS, EPI_BIAS_RELU, EPI_BIAS_TANH};
  return make_dims(in, out, epi);
}
// models.py:77-83: fc1 -> relu -> cat(., a) -> fc2 -> relu -> fc2_2 -> relu -> fc3, the raw head (fc2 contracts
// cat(h1, a): in[1] = H + |a|, the action columns from column H on)
NetDims critic_dims(int obs_dim, int act_dim, int n_atoms) {
  const int in[4] = {obs_dim, D4PG_HIDDEN + act_dim, D4PG_HIDDEN, D4PG_HIDDEN};
  const int out[4] = {D4PG_HIDDEN, D4PG_HIDDEN, D4PG_HIDDEN, n_atoms};
  const int epi[4] = {EPI_BIAS_RELU, EPI_BIAS_RELU, EPI_BIAS_RELU, EPI_BIAS};
  return make_dims(in, out, epi);
}

static void fill_layout(const NetDims& d, d4pg_net_layout_t* out) {
  for (int l = 0; l < 4; ++l) {
    out->offsets[2 * l] = d.w_off[l]; out->sizes[2 * l] = int64_t(d.ld[l]) * d.out[l]; out->pitch[l] = d.ld[l];
    out->offsets[2 * l + 1] = d.b_off[l]; out->sizes[2 * l + 1] = d.out[l];
  }
  out->total = d.total;
}

__global__ void softmax_rows_kernel(const float* logits, float* probs, int B, int N) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B) return;
  const float* x = logits + size_t(warp) * N;
  float mx = -INFINITY;
  for (int k = lane; k < N; k += 32) mx = fmaxf(mx, x[k]);
  mx = warp_max(mx);
  float s = 0.f;
  for (int k = lane; k < N; k += 32) s += expf(x[k] - mx);
  s = warp_sum(s);
  for (int k = lane; k < N; k += 32) probs[size_t(warp) * N + k] = expf(x[k] - mx) / s;
}

// The four forward levels of a network, one grouped launch each.  fc1 reads s [B, in[0]]; the critic's fc2 (a != NULL)
// also reads the action rows a [B, |a|] as its columns H.. (as learner.cu level_fwd does).  fc1..fc2_2 write the [B, H]
// planes h1..h3 of `workspace`, fc3 writes y [B, out[3]].
static int net_forward(const NetDims& d, const float* params, const float* s, const float* a, int B, float* workspace,
                       float* y, int precision, cudaStream_t st) {
  const int H = D4PG_HIDDEN, A = a ? d.in[1] - H : 0;
  float* h[3] = {workspace, workspace + size_t(B) * H, workspace + size_t(B) * 2 * H};
  for (int l = 0; l < 4; ++l) {
    const float* X2 = l == 1 ? a : nullptr;
    GemmBatch b; gemm_batch_begin(b);
    gemm_batch_add(b, gemm_fwd(l ? h[l - 1] : s, d.in[l] - (X2 ? A : 0), X2, X2 ? A : 0, X2 ? H : 0,
                               params + d.w_off[l], d.ld[l], params + d.b_off[l], l < 3 ? h[l] : y, d.out[l], B,
                               d.out[l], d.in[l], d.epi[l]));
    const int rc = gemm_launch(b, precision, st);
    if (rc) return rc;
  }
  return D4PG_OK;
}

}  // namespace d4pg

using namespace d4pg;

extern "C" const char* d4pg_last_error(void) { return g_err; }
extern "C" int32_t d4pg_version(void) { return 1200; }   /* 0.12.0 */
/* sizeof of the structs that cross the ABI by pointer: a binding whose mirror has another size is out of date */
extern "C" int32_t d4pg_struct_size(int32_t which) {
  switch (which) {
    case 0: return int32_t(sizeof(d4pg_learner_config_t));
    case 1: return int32_t(sizeof(d4pg_learner_buffers_t));
    case 2: return int32_t(sizeof(d4pg_net_layout_t));
    default: return -1;
  }
}

extern "C" int32_t d4pg_device_sm(void) {
  int dev = 0, major = 0, minor = 0;
  D4PG_CUDA_OK(cudaGetDevice(&dev));
  D4PG_CUDA_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  D4PG_CUDA_OK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  return major * 10 + minor;
}
namespace d4pg {
int device_sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return 1;
  return n > 0 ? n : 1;
}
}  // namespace d4pg

extern "C" int32_t d4pg_actor_layout(int32_t obs_dim, int32_t act_dim, d4pg_net_layout_t* out) {
  D4PG_REQUIRE(out && obs_dim > 0 && act_dim > 0, D4PG_EINVAL, "d4pg_actor_layout: bad arguments");
  fill_layout(actor_dims(obs_dim, act_dim), out);
  return D4PG_OK;
}
extern "C" int32_t d4pg_critic_layout(int32_t obs_dim, int32_t act_dim, int32_t n_atoms, d4pg_net_layout_t* out) {
  D4PG_REQUIRE(out && obs_dim > 0 && act_dim > 0 && n_atoms >= 2 && n_atoms <= D4PG_MAX_ATOMS, D4PG_EINVAL,
               "d4pg_critic_layout: bad arguments");
  fill_layout(critic_dims(obs_dim, act_dim, n_atoms), out);
  return D4PG_OK;
}

// actor.forward, models.py:32-41
extern "C" int32_t d4pg_actor_forward(const float* params, int32_t obs_dim, int32_t act_dim,
                                      const float* s, int32_t B, float* action, float* workspace,
                                      int32_t precision, d4pg_stream_t stream) {
  D4PG_REQUIRE(params && s && action && workspace && B > 0, D4PG_EINVAL, "d4pg_actor_forward: null/empty argument");
  D4PG_REQUIRE(precision >= 0 && precision <= 3, D4PG_ENOTSUP, "d4pg_actor_forward: unknown precision %d", precision);
  return net_forward(actor_dims(obs_dim, act_dim), params, s, nullptr, B, workspace, action, precision, as_stream(stream));
}

// critic.forward, models.py:76-88: the raw head, then softmax
extern "C" int32_t d4pg_critic_forward(const float* params, int32_t obs_dim, int32_t act_dim, int32_t n_atoms,
                                       const float* s, const float* a, int32_t B, float* probs, float* logits,
                                       float* workspace, int32_t precision, d4pg_stream_t stream) {
  D4PG_REQUIRE(params && s && a && workspace && B > 0 && (probs || logits), D4PG_EINVAL, "d4pg_critic_forward: null/empty argument");
  D4PG_REQUIRE(precision >= 0 && precision <= 3, D4PG_ENOTSUP, "d4pg_critic_forward: unknown precision %d", precision);
  D4PG_REQUIRE(n_atoms >= 2 && n_atoms <= D4PG_MAX_ATOMS, D4PG_EINVAL, "d4pg_critic_forward: n_atoms out of range");
  // the logits go to h1 when the caller only wants probabilities: h1 is dead after fc2
  float* z = logits ? logits : workspace;
  cudaStream_t st = as_stream(stream);
  const int rc = net_forward(critic_dims(obs_dim, act_dim, n_atoms), params, s, a, B, workspace, z, precision, st);
  if (rc) return rc;
  if (probs) {
    softmax_rows_kernel<<<cdiv(B * 32, 256), 256, 0, st>>>(z, probs, B, n_atoms);
    D4PG_LAUNCH_OK();
  }
  return D4PG_OK;
}
