// Cross-translation-unit internals of libd4pg_sm90.so (not part of the C ABI).
#pragma once
#include "common.cuh"
#include "adam.cuh"

struct d4pg_replay;
struct d4pg_comm;

namespace d4pg {

// What the three loss heads of the learner step share.  `target`, `q`, `pi` are the raw fc3 rows of critic_target(s', .),
// critic(s, a) and critic(s, actor(s)) (logits, raw mixture heads or quantiles); every such plane has row pitch `ld`.
struct HeadCommon {
  const float* target; const float* q; const float* pi;
  const double* rewards; const uint8_t* dones;
  int B, ld;
  double discount, prio_eps;
  float grad_scale;
  float* loss_rows; float* td; float* prio; float* dq; float* pi_rows; float* dpi;
  const float* is_weights;       // non-null: critic loss row i is scaled by the PER importance weight w_i (SURVEY.md section 8f.4, H3)
  int pdl;                       // programmatic-dependent-launch trigger position (0/1/2)
  unsigned long long* trace;
  int only_policy;               // 1: only the policy head (pi_rows, dpi) -- the second loss launch of the post-update-critic plan
  LearnerClock* sampler_clock;   // prefetch pipeline: thread 0 advances the sampler's counters (after sample(k), before sample(k+1))
  // episode tails (DESIGN.md §3 "Episode tails"): the batch's per-row horizon k (0 = `discount`) and gtab[k] = gamma^k;
  // both null without them.  Read from the batch, never from the ring, which a later add may already overwrite
  const uint8_t* horizon; const double* gtab;
};

// bootstrap discount of batch row `row` that is not done: gamma^k of its horizon, `discount` for a full row
__device__ __forceinline__ double head_discount(const HeadCommon& h, int row) {
  const int k = h.horizon ? int(h.horizon[row]) : 0;
  return k ? h.gtab[k] : h.discount;
}

// categorical head (proj_loss.cu): N atoms on [v_min, v_max]
struct HeadsArgs {
  HeadCommon h;
  int N; int flags;
  double v_min, v_max, delta;     // v_max: the top of the return clip, proj_clip_top(v_min, v_max, N, delta)
  float* m; int32_t* bins_l; int32_t* bins_u; float* target_probs; float* q_probs;
  int ce_priority;               // 1: priority = CE_i + eps instead of |sum_j m_ij q_ij| + eps (the reference does not, H4)
};
int launch_heads(const HeadsArgs& a, int mode, cudaStream_t st);
double proj_clip_top(double v_min, double v_max, int N, double delta);

// mixture-of-Gaussians head (mog_heads.cu): K components, raw planes of 3K columns
struct MogArgs {
  HeadCommon h;
  int K;
};
int launch_mog_heads(const MogArgs& a, cudaStream_t st);
int launch_mog_transform(const float* raw, int ldr, int B, int K, float* w, float* mu, float* sigma, cudaStream_t st);
int launch_mog_head_backward(const float* raw, int ldr, const float* gw, const float* gmu, const float* gsig, int B, int K,
                             float* dz, int ldz, cudaStream_t st);

// quantile-regression head (qr_heads.cu): N quantiles
struct QrArgs {
  HeadCommon h;
  int N;
  double kappa;
  int ce_priority;               // 1: priority = L_i + eps (unweighted) instead of |td_i| + eps
};
int launch_qr_heads(const QrArgs& a, cudaStream_t st);

constexpr int SAMPLE_ROWS = 32;      // batch rows per CTA of the sample + gather kernel (replay_dev.cuh)

// sample for the learner: per-step scalars come from device memory (graph replay safe)
int learner_sample(d4pg_replay* h, int B, int prioritized, const double* uniforms, const int32_t* positions,
                   uint64_t seed, LearnerClock* clock, const ClockParams& cp,
                   int32_t* idx, float* weights, float* s, float* a, double* r, float* s2, uint8_t* d, uint8_t* hz,
                   int ld_obs, int ld_act, const float* norm, float norm_clip, int pipe_slot, cudaStream_t st,
                   bool dependent = false, unsigned long long* done_epoch = nullptr);
// gate != nullptr: *gate is bumped (release) once the trees are complete -- by the update kernel itself when it can
int launch_tree_update(d4pg_replay* h, int B, const int32_t* idx, const float* prio, cudaStream_t st, unsigned long long* gate = nullptr);
int64_t replay_generation(const d4pg_replay* h);
// the replay's observation normalizer: its affine (nullptr when none is registered) and clip
const float* replay_obs_norm(const d4pg_replay* h, double* clip);
// the replay's per-row horizon column (d4pg_replay_set_horizons; nullptr when none is registered)
const uint8_t* replay_horizons(const d4pg_replay* h);
// ingest gate (host pipeline): every gated learner step bumps the buffer's flag once (launch_gate_signal) and arms the
// gate after its launch; the next add / presample on the ingest stream first waits for flag >= number of armed steps
unsigned long long* replay_gate_flag(d4pg_replay* h);
void replay_arm_gate(d4pg_replay* h);
int replay_gate_consume(d4pg_replay* h, cudaStream_t st);
int launch_gate_signal(unsigned long long* flag, cudaStream_t st);
void trace_set_side_stream(cudaStream_t s);     // changes whenever the caller mutates the buffer
int comm_allreduce(d4pg_comm* c, float* buf, int64_t n, cudaStream_t st);
// fused all-reduce over IPC-mapped peer memory (comm.cu): x[r] = rank r's [2][n] gradient halves
bool comm_peer_info(d4pg_comm* c, PeerInfo* out);
PeerSignal comm_peer_signal(const PeerInfo& info, int kind);    // kind 0: gradient half complete, 1: reduced slice pushed
int comm_peer_barrier(d4pg_comm* c, cudaStream_t st);
// reduce-scatter + all-gather of the step's gradient over peer memory: this rank sums ITS slice of every rank's half
// `parity` (rank order) and pushes the result into every rank's reduced buffer; publishes flag2 when done
int comm_peer_reduce_scatter(d4pg_comm* c, int parity, cudaStream_t st);
// two-phase in-switch form: multimem.ld_reduce of this rank's slice, multimem.st into every rank's reduced buffer
// (mc_uc + 2n on each rank), then flag2
int comm_mc_reduce_bcast(d4pg_comm* c, int parity, cudaStream_t st);

}  // namespace d4pg
