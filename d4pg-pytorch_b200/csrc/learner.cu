// The learner: one DDPG.train() body (ddpg.py:200-255) as a fixed sequence of launches,
// captured once into a CUDA graph and replayed.  No host synchronisation inside a step; every
// per-step scalar (Adam bias corrections, PER beta, Philox counter) lives in device memory and
// is advanced by a one-thread clock kernel so the captured graph never needs patching.
//
// Step order (reference line -> phase function of enqueue_step: launch):
//   ddpg.py:202  sample                       -> sample_batch: sample_gather_kernel (tree descent + row gather)
//   ddpg.py:205-208 target/online forwards    -> forward_levels: 7 grouped-GEMM levels (actor_target, critic_target,
//                                                critic, actor and critic(s, actor(s)) in lock-step);
//                                                forward_chain / forward_tc_chain: the same layers as three cluster chains
//   ddpg.py:214-222 projection, CE loss, td   -> launch_step_heads: heads_kernel (also the policy head of ddpg.py:236-238)
//   ddpg.py:252-255 update_priorities         -> side_branch: tree_write_kernel<TREE_UPDATE>, beside the backward pass
//   ddpg.py:229-231 critic backward           -> backward_levels: grouped dX / dW levels (shared with the policy pass);
//                                                backward_chain / backward_tc_chain: two dX chains, then dw_wide
//   ddpg.py:236-243 policy backward           -> uses the PRE-update critic weights (SURVEY.md H7):
//                                                both backward passes run before any Adam update
//   ddpg.py:232,244,247,250 Adam x2, sync, Polyak -> exchange_gradients, then one fused adam_polyak_kernel (2 segments)
//   (no reference line) max_grad_norm        -> launch_update: grad_sqnorm_kernel before each Adam launch, only when configured
#include "common.cuh"
#include "gemm_ffma.cuh"
#include "adam.cuh"
#include <string.h>
#include <stdlib.h>
#include <initializer_list>
#include <new>
#include <string>
#include <vector>

#include "internal.cuh"
#include "mlp_chain.cuh"
#include "mlp_tc_chain.cuh"

namespace d4pg {

// One half of the double-buffered batch: the rows the sample kernel gathers, the indices and IS weights it draws
struct Batch { float *s, *a, *s2; double* r; uint8_t* done; int32_t* idx; float* wts; uint8_t* hz; };   // hz: nstep_tails only

struct Workspace {
  // batch[1] exists under the prefetch / host pipelines only; without them batch[0].idx / .wts are the caller's
  // buffers (d4pg_learner_create), with them the sampler's own
  Batch batch[2];
  // activations: [0]=actor_target [1]=critic_target [2]=critic [3]=actor [4]=critic on policy action
  float *h1[5], *h2[5], *h3[5], *out[5];
  // heads
  float *m, *q_probs, *target_probs, *dlogits_q, *dlogits_pi, *loss_rows, *pi_rows;
  // backward
  float *c_dz22, *c_dz2, *c_dz1, *p_dz22, *p_dz2, *a_dz3, *a_dz22, *a_dh2, *a_dz1;
  LearnerClock* clock;
  float* xchg;                     // exchange planes of the cluster-fused chain kernels (chain mode)
  unsigned long long* pipe_epoch;  // host pipeline: per-CTA completion epochs of the presample kernel (polled by the forward chains)
  double* sq_partials;             // [2][GRAD_NORM_CTAS] partial sums of g^2 (actor, critic); only when a network clips
  int64_t total;
};

// The step plan, decided once from the config:
//   PLAN_LEVELS    one grouped launch per dependency level (the only plan of precision 3, bf16);
//   PLAN_CHAIN     cluster-fused chains of mlp_chain.cu: exact FFMA tiles at fp32, mma.sync 3xTF32 / TF32 tiles otherwise;
//   PLAN_TC_CHAIN  cluster-fused wgmma chains of mlp_tc_chain.cu, with pre-packed hi/lo weight images.
// The chain plans pay off while the batch fits one wave of clusters (a 64-row cluster chain is a latency design; 128-row
// level tiles suit larger batches), so batches above CHAIN_MAX_BATCH rows always run the level plan.  PLAN_CHAIN also
// needs every slot of its forward and dX launches to fit one chain CTA (chain_plan_fits): a wide observation or action
// runs the level plan.
enum StepPlan { PLAN_LEVELS, PLAN_CHAIN, PLAN_TC_CHAIN };
constexpr int CHAIN_MAX_BATCH = 512;
// pre-layers (a narrow layer computed inside the slot that consumes it): fp32 tile, |a| <= 8
static bool chain_pre_ok(const d4pg_learner_config_t& c) { return c.precision == 0 && c.act_dim <= 8; }
// chain_fits (mlp_chain.cu) of the PLAN_CHAIN launches, on slots of the shapes chain_build_actor_critic, forward_chain
// and backward_chain add: fc1 is |s| deep, critic fc2 H + |a|, actor fc3 and the d-action layer |a| wide, critic fc3
// as wide as the head.  Sizes only: no launch is built from these slots.
static bool chain_plan_fits(const d4pg_learner_config_t& c) {
  const int H = D4PG_HIDDEN, S = c.obs_dim, A = c.act_dim, N = c.n_atoms;
  ChainArgs f, b;
  chain_args_begin(f, c.batch, nullptr, c.precision);
  chain_add(f, 0, chain_fwd(nullptr, 0, nullptr, H, S, EPI_BIAS_RELU, nullptr, 0, 1));             // fc1
  chain_add(f, 0, chain_fwd(nullptr, 0, nullptr, H, H, EPI_BIAS_RELU, nullptr, 0, 1));             // actor fc2, fc2_2
  ChainSlot fc2 = chain_fwd(nullptr, 0, nullptr, H, H + A, EPI_BIAS_RELU, nullptr, 0, 1);           // critic fc2
  if (chain_pre_ok(c)) chain_pre_layer(fc2, nullptr, 0, nullptr, nullptr, 0, A, H, EPI_BIAS_TANH, nullptr, 0, 0, H, false);
  else chain_add(f, 0, chain_fwd(nullptr, 0, nullptr, A, H, EPI_BIAS_TANH, nullptr, 0, 1));       // actor fc3
  chain_add(f, 0, fc2);
  chain_add(f, 0, chain_fwd(nullptr, 0, nullptr, N, H, EPI_BIAS, nullptr, 0, 0));                  // critic fc3
  chain_args_begin(b, c.batch, nullptr, c.precision);
  chain_add(b, 0, chain_dx(nullptr, 0, H, N, EPI_RELU_MASK, nullptr, 0, nullptr, 0, 1));           // critic fc3
  chain_add(b, 0, chain_dx(nullptr, 0, H, H, EPI_RELU_MASK, nullptr, 0, nullptr, 0, 1));           // the H x H layers
  ChainSlot fc3 = chain_dx(nullptr, 0, H, A, EPI_RELU_MASK, nullptr, 0, nullptr, 0, 1);             // actor fc3
  if (chain_pre_ok(c)) chain_pre_layer(fc3, nullptr, 0, nullptr, nullptr, 0, A, H, EPI_TANH_MASK, nullptr, 0, 0, H, true);
  else chain_add(b, 0, chain_dx(nullptr, 0, A, H, EPI_TANH_MASK, nullptr, 0, nullptr, 0, 1));      // d action
  chain_add(b, 0, fc3);
  return chain_fits(f) && chain_fits(b);
}
static StepPlan step_plan(const d4pg_learner_config_t& c) {
  if (c.batch > CHAIN_MAX_BATCH || c.chain != 1) return PLAN_LEVELS;
  if (c.precision == 3) return PLAN_LEVELS;             // bf16: the level kernel only (no bf16 chain tiles)
  // the wgmma chains need |s| <= 32 (one resident input chunk), |a| <= 32 (one K-tail chunk) and <= 256 atoms
  if (c.precision >= 1 && c.obs_dim <= 32 && c.act_dim <= 32 && c.n_atoms <= 256) return PLAN_TC_CHAIN;
  return chain_plan_fits(c) ? PLAN_CHAIN : PLAN_LEVELS;
}
// The mixture-of-Gaussians critic (dist_type 1) has a raw head of 3K columns: it takes the place of n_atoms wherever a
// plane or a layer is sized (carve, critic_dims, step_plan, tcc_setup), so the learner keeps the config with n_atoms = 3K
static d4pg_learner_config_t with_head_width(const d4pg_learner_config_t& c) {
  d4pg_learner_config_t e = c;
  if (c.dist_type == 1) e.n_atoms = 3 * c.n_components;
  return e;
}
// The warm host-pipeline graph of the wgmma plan waits for the sampler by polling its per-CTA epochs from the forward
// chains' threads (one epoch per thread)
static_assert((CHAIN_MAX_BATCH + SAMPLE_ROWS - 1) / SAMPLE_ROWS <= TCC_THREADS, "sampler epochs exceed the chain CTA's threads");

// Every 2-D plane has a row pitch that is a multiple of 4 floats (16-B rows): |s|=17 -> 20,
// |a|=6 -> 8, N=51 -> 52.  That makes every GEMM operand TMA- and float4-addressable.
static Workspace carve(float* base, int B, int S, int A, int N, StepPlan plan, bool prefetch, bool clip, bool tails) {
  Workspace w{};
  int64_t off = 0;
  auto take = [&](int64_t n) { float* p = base ? base + off : nullptr; off += align4(n); return p; };
  const int H = D4PG_HIDDEN, Sp = pitch4(S), Ap = pitch4(A), Np = pitch4(N);
  auto take_rows = [&](Batch& h) {
    h.s = take(int64_t(B) * Sp); h.a = take(int64_t(B) * Ap); h.s2 = take(int64_t(B) * Sp);
    h.r = reinterpret_cast<double*>(take(int64_t(B) * 2));
    h.done = reinterpret_cast<uint8_t*>(take((B + 3) / 4));
  };
  take_rows(w.batch[0]);
  for (int k = 0; k < 5; ++k) {
    if (k != 4) w.h1[k] = take(int64_t(B) * H);
    w.h2[k] = take(int64_t(B) * H); w.h3[k] = take(int64_t(B) * H);
  }
  w.out[0] = take(int64_t(B) * Ap); w.out[3] = take(int64_t(B) * Ap);
  w.out[1] = take(int64_t(B) * Np); w.out[2] = take(int64_t(B) * Np); w.out[4] = take(int64_t(B) * Np);
  w.m = take(int64_t(B) * Np); w.q_probs = take(int64_t(B) * Np); w.target_probs = take(int64_t(B) * Np);
  w.dlogits_q = take(int64_t(B) * Np); w.dlogits_pi = take(int64_t(B) * Np);
  w.loss_rows = take(B); w.pi_rows = take(B);
  w.c_dz22 = take(int64_t(B) * H); w.c_dz2 = take(int64_t(B) * H); w.c_dz1 = take(int64_t(B) * H);
  w.p_dz22 = take(int64_t(B) * H); w.p_dz2 = take(int64_t(B) * H);
  w.a_dz3 = take(int64_t(B) * Ap); w.a_dz22 = take(int64_t(B) * H); w.a_dh2 = take(int64_t(B) * H);
  w.a_dz1 = take(int64_t(B) * H);
  w.clock = reinterpret_cast<LearnerClock*>(take(sizeof(LearnerClock) / 4 + 4));
  w.xchg = plan != PLAN_LEVELS ? take(std::max(chain_xchg_floats(B), tcc_xchg_floats(B))) : nullptr;
  w.pipe_epoch = reinterpret_cast<unsigned long long*>(take(2 * int64_t((B + SAMPLE_ROWS - 1) / SAMPLE_ROWS)));
  if (prefetch) {
    take_rows(w.batch[1]);
    for (int k = 0; k < 2; ++k) { w.batch[k].idx = reinterpret_cast<int32_t*>(take(B)); w.batch[k].wts = take(B); }
  }
  if (clip) w.sq_partials = reinterpret_cast<double*>(take(2 * GRAD_NORM_CTAS * 2));
  // the batch's horizons (nstep_tails), last so that every other plane keeps its offset
  if (tails)
    for (int k = 0; k < (prefetch ? 2 : 1); ++k) w.batch[k].hz = reinterpret_cast<uint8_t*>(take((B + 3) / 4));
  w.total = off;
  return w;
}
}  // namespace d4pg

using namespace d4pg;

struct d4pg_learner {
  d4pg_learner_config_t cfg;
  d4pg_learner_buffers_t buf;
  d4pg_replay* replay;
  d4pg_comm* comm;
  StepPlan plan;
  Workspace ws;
  NetDims da, dc;
  ClockParams clock_params;        // what the sample kernel derives the step's device-side scalars from
  cudaGraphExec_t graph_exec[4];   // [batch parity * 2 + cold]; only [0] without the prefetch pipeline
  bool graph_ready[4];
  cudaGraphExec_t multi_exec[2];   // RUN_UNROLL warm steps in one graph, by starting batch parity (d4pg_learner_run)
  bool multi_ready[2];
  int pipe_par;                    // half of the double-buffered batch the NEXT step trains on
  int last_par;                    // ... the last step trained on
  bool prefetch_valid;             // that half already holds the next step's batch
  int64_t seen_gen;                // replay generation when it was sampled
  int64_t steps_done;
  int kernels_per_step;
  // profiling (d4pg_learner_profile_step): CUDA-event pair around every launch of an eager step
  cudaStream_t side; cudaEvent_t ev_fork, ev_join;
  ChainArgs chain_fwd_args, chain_bwd_args;
  // wgmma chains (PLAN_TC_CHAIN): library-owned weight images + the per-step pack / chain descriptors
  // weight images: forward ones (packed at the start of a graph launch, then kept current by the Adam kernel) and the
  // transposed ones of the dX chains (packed every step on the side branch, off the critical path)
  uint8_t* tcc_images; TccPackArgs tcc_pack_fwd, tcc_pack_dx; TccImage tcc_img[32];
  cudaEvent_t ev_fork2, ev_join2;
  TccArgs tcc_fwd_args, tcc_bwd_args;
  GemmWideBatch dw_batch;
  // host-facing step: library-owned pinned staging, double-buffered by step parity (a buffer is rewritten only after
  // the H2D copy out of it, two steps earlier, has completed)
  double* host_u[4]; int32_t* host_pos[4]; float* host_losses; cudaEvent_t ev_in, ev_out, ev_h2d[4];
  int64_t host_steps;
  // results of the host-facing steps: {critic loss, actor loss, -, -} of step k land in ring slot k & 1 (async D2H queued
  // by the step itself), so a caller can read step k-1 while step k runs
  float* loss_ring[2]; cudaEvent_t ev_loss[2]; int64_t loss_steps;
  // host pipeline: library-owned ingest stream (adds + the presample of the next batch), the gate flag the step's
  // priority write-back bumps, how many gated steps were launched
  cudaStream_t ing; cudaEvent_t ev_ing; unsigned long long* gate_flag;
  bool images_dirty;               // parameters were written outside the library since the forward weight images were last current
  // cfg.obs_norm: the replay's observation normalizer, applied to s / s2 by every sample launch of the step
  const float* norm_affine; float norm_clip;
  double* gtab;                    // cfg.nstep_tails: gamma^k for k < D4PG_STEPS_MAX_N (device), the tail rows' discounts
  bool profiling;
  std::vector<cudaEvent_t> ev;
  std::vector<std::string> ev_name;
  std::vector<int> ev_reps;        // how many times the launch between the event pair was repeated
};

// prefetch pipeline: batch t+1 is sampled on a side branch of step t (device-side sampling only)
static bool prefetching(const d4pg_learner_config_t& c) { return c.prefetch != 0 && c.sample_mode == 1; }
// host pipeline (host-drawn uniforms / positions, cfg.prefetch): the host-facing step samples batch k on the library's
// ingest stream -- behind the caller's add(k), gated on step k-1's priority write-back -- while step k-1's backward
// pass, dW and Adam still run on the learner stream; the step graph then starts from the sampled batch.  Same double
// buffers and clock slots as the device prefetch pipeline; the order of tree operations is the reference's
// (update_priorities(k-1) -> add(k) -> sample(k), main.py / ddpg.py:200-255).
static bool host_pipe(const d4pg_learner_config_t& c) { return c.prefetch != 0 && c.sample_mode == 0 && c.use_graph != 0; }
static bool piped(const d4pg_learner_config_t& c) { return prefetching(c) || host_pipe(c); }
// some network's gradient is clipped to (or measured against) a global norm: the step has a norm launch before each Adam
static bool clipping(const d4pg_learner_config_t& c) { return c.max_grad_norm_actor != 0.0 || c.max_grad_norm_critic != 0.0; }

// ---- the layers ---------------------------------------------------------------------------------------------------
enum Net { ACTOR, ACTOR_TARGET, CRITIC, CRITIC_TARGET };
// Layer l (fc1, fc2, fc2_2, fc3) of a network as every plan's forward pass consumes it
struct Layer { const float* W; int ldw; const float* bias; int n_out, k_in, epi; };
static Layer layer(const d4pg_learner* L, Net net, int l) {
  const bool critic = net >= CRITIC;
  const NetDims& d = critic ? L->dc : L->da;
  const float* P[4] = {L->buf.actor, L->buf.actor_target, L->buf.critic, L->buf.critic_target};
  return Layer{P[net] + d.w_off[l], d.ld[l], P[net] + d.b_off[l], d.out[l], d.in[l], d.epi[l]};
}
// critic fc2's action columns start H floats into each row of its weight (and weight-gradient) matrix
static int64_t critic_fc2_action_off(const d4pg_learner* L) { return L->dc.w_off[1] + D4PG_HIDDEN; }
// The same layer as the dX pass of the online nets consumes it: dX[., n_in] = dZ[., k_out] . W.  Critic fc2 is its h1
// columns here; its action columns are a problem of their own
struct LayerDx { const float* W; int ldw, n_in, k_out; };
static LayerDx layer_dx(const d4pg_learner* L, Net net, int l) {
  const Layer y = layer(L, net, l);
  return LayerDx{y.W, y.ldw, (net == CRITIC && l == 1) ? D4PG_HIDDEN : y.k_in, y.n_out};
}
static LayerDx critic_fc2_action_dx(const d4pg_learner* L) {
  return LayerDx{L->buf.critic + critic_fc2_action_off(L), L->dc.ld[1], L->cfg.act_dim, D4PG_HIDDEN};
}

// weight matrices as the tensor-core chains consume them (F = forward image, D = transposed image for dX)
enum { U_A_F1, U_A_F2, U_A_F22, U_A_F3, U_A_D3, U_A_D22, U_A_D2, U_AT_F1, U_AT_F2, U_AT_F22, U_AT_F3,
       U_C_F1, U_C_F2, U_C_F22, U_C_F3, U_C_D3, U_C_D22, U_C_D2H, U_C_D2A, U_CT_F1, U_CT_F2, U_CT_F22, U_CT_F3, U_COUNT };
static int fwd_image(Net net, int l) {
  const int fc1[4] = {U_A_F1, U_AT_F1, U_C_F1, U_CT_F1};
  return fc1[net] + l;
}

// the weight images of the wgmma chains (PLAN_TC_CHAIN only)
static int tcc_setup(d4pg_learner* L) {
  TccPackArgs& pf = L->tcc_pack_fwd; TccPackArgs& pd = L->tcc_pack_dx;
  tcc_pack_begin(pf, nullptr); tcc_pack_begin(pd, nullptr);
  int use_of[U_COUNT]; bool is_dx[U_COUNT];
  auto add_dx = [&](int id, const LayerDx& d) {
    is_dx[id] = true;
    use_of[id] = tcc_pack_add(pd, d.W, d.ldw, GEMM_DX, d.n_in, d.k_out);
  };
  for (int net = ACTOR; net <= CRITIC_TARGET; ++net)
    for (int l = 0; l < 4; ++l) {                  // critic fc2: K = [h1 (256) | action]: 8 chunks + a tail chunk
      const Layer y = layer(L, Net(net), l);
      const int id = fwd_image(Net(net), l);
      is_dx[id] = false;
      use_of[id] = tcc_pack_add(pf, y.W, y.ldw, GEMM_FWD, y.n_out, y.k_in);
    }
  add_dx(U_A_D3, layer_dx(L, ACTOR, 3));
  add_dx(U_A_D22, layer_dx(L, ACTOR, 2));
  add_dx(U_A_D2, layer_dx(L, ACTOR, 1));
  add_dx(U_C_D3, layer_dx(L, CRITIC, 3));
  add_dx(U_C_D22, layer_dx(L, CRITIC, 2));
  add_dx(U_C_D2H, layer_dx(L, CRITIC, 1));
  add_dx(U_C_D2A, critic_fc2_action_dx(L));
  for (int i = 0; i < U_COUNT; ++i) D4PG_REQUIRE(use_of[i] >= 0, D4PG_ENOTSUP, "tcc_setup: too many weight images");
  const long long fwd_bytes = tcc_pack_bytes(pf), all_bytes = fwd_bytes + tcc_pack_bytes(pd);
  D4PG_CUDA_OK(cudaMalloc(&L->tcc_images, size_t(all_bytes)));
  D4PG_CUDA_OK(cudaMemset(L->tcc_images, 0, size_t(all_bytes)));
  tcc_pack_set_base(pf, L->tcc_images, 0);
  tcc_pack_set_base(pd, L->tcc_images, fwd_bytes);
  for (int i = 0; i < U_COUNT; ++i) L->tcc_img[i] = tcc_image(is_dx[i] ? pd : pf, use_of[i]);
  (void)tcc_watchdog_device();                         // allocate outside of any stream capture
  return D4PG_OK;
}

// ---- one step -----------------------------------------------------------------------------------------------------
// Exchange shapes of the data-parallel gradient (D4PG_COMM_MODE=mc|mc2|pull|rs; default: "mc" from D4PG_COMM_MC_FROM =
// 3 ranks up when the communicator set up a multicast object, else "pull").  These defaults were chosen on another GPU
// generation and have NOT been validated on Hopper (no multi-GPU H100 measurement exists yet; tools/ab_mc8.sh compares
// the modes):
//   XCHG_ALLREDUCE  no IPC-mapped peers: the communicator's all-reduce over the flat [P_a + P_c] buffer;
//   XCHG_PULL  one hop, every rank sums all N halves inside Adam (N x 1.15 MB inbound over NVLink);
//   XCHG_MC    in-switch reduction: ONE hop and 1.15 MB inbound per rank -- the Adam kernel's multimem.ld_reduce over an NVLS
//              multicast object returns the sum over all ranks, added by the NVSwitch;
//   XCHG_MC2   its two-phase form: every rank ld_reduces its 1/N slice and multimem.st's it to everyone (2 x 1.15 MB per
//              GPU whatever N), then a second flag hop;
//   XCHG_RS    reduce-scatter + all-gather over peer memory: TWO hops of 16-B remote accesses.
enum Exchange { XCHG_NONE, XCHG_ALLREDUCE, XCHG_PULL, XCHG_MC, XCHG_MC2, XCHG_RS };
static Exchange exchange_mode(d4pg_learner* L, PeerInfo* peers) {
  if (L->cfg.world_size <= 1) return XCHG_NONE;
  if (!comm_peer_info(L->comm, peers)) return XCHG_ALLREDUCE;
  static const int comm_mode = [] { const char* e = getenv("D4PG_COMM_MODE");
                                    return !e ? 0 : (e[0] == 'p' ? 1 : (e[0] == 'r' ? 2 : (e[0] == 'm' && e[1] == 'c' && e[2] == '2' ? 4 : 3))); }();
  static const int mc_from = [] { const char* e = getenv("D4PG_COMM_MC_FROM"); return e ? atoi(e) : 3; }();
  static const int mc2_from = [] { const char* e = getenv("D4PG_COMM_MC2_FROM"); return e ? atoi(e) : 1000; }();
  const bool mc_avail = peers->mc != nullptr && L->plan != PLAN_LEVELS;
  if (mc_avail && (comm_mode == 4 || (comm_mode == 0 && peers->world >= mc2_from))) return XCHG_MC2;
  if (mc_avail && (comm_mode == 3 || (comm_mode == 0 && peers->world >= mc_from))) return XCHG_MC;
  return comm_mode == 2 ? XCHG_RS : XCHG_PULL;
}

// What the phases of one step share
struct Step {
  d4pg_learner* L; cudaStream_t st;
  const d4pg_learner_config_t& c; const d4pg_learner_buffers_t& b; const Workspace& w;
  Batch bt;                          // the half of the double-buffered batch this step trains on
  int par; bool cold;                // that half's index; sample it first (no valid prefetch)
  bool pf;                           // prefetch or host pipeline
  // corrected-semantics switch (SURVEY.md H7, loss_flags & 4): the actor gradient goes through the critic AFTER this
  // step's critic update (the reference uses the stale local copy, ddpg.py:229-247).  Two half steps: critic forward /
  // loss / backward / Adam, then the policy pass through the updated critic, actor backward / Adam.
  bool h7;                           // PLAN_TC_CHAIN on one GPU (checked at create)
  int B, S, A, N, Sp, Ap, Np;        // Sp, Ap, Np: activation row pitches
  Exchange xm; PeerInfo peers; int gpar;   // gradient exchange: its shape, the peers, which half of the exchange buffer
  float *Ga, *Gc;                    // where this step's gradients go
  int nk;                            // launches so far
};
static bool peer_exchange(const Step& x) { return x.xm >= XCHG_PULL; }

// idempotent launches (pure functions of their inputs) are repeated in profile mode
constexpr int PROFILE_REPS = 16;
// One launch of the step, counted, under the name d4pg_learner_profile_step reports it by.  Profile mode puts a
// CUDA-event pair around it on the step's stream and repeats it when the call site says it is repeatable.
template <class F>
static int run_launch(Step& x, const char* name, bool repeatable, F launch) {
  d4pg_learner* L = x.L;
  int rc;
  if (L->profiling) {
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0, x.st); rc = launch();
    for (int r = 1; repeatable && r < PROFILE_REPS && rc == 0; ++r) rc = launch();
    cudaEventRecord(e1, x.st);
    L->ev.push_back(e0); L->ev.push_back(e1); L->ev_reps.push_back(repeatable ? PROFILE_REPS : 1);
    L->ev_name.push_back(name);
  } else rc = launch();
  if (rc == 0) ++x.nk;
  return rc;
}
#define RUN(name, repeatable, call) \
  do { if (int rc_ = run_launch(x, name, repeatable, [&] { return (call); })) return rc_; } while (0)
// One dependency level of the level plan: its GEMMs as one grouped launch
static int run_level(Step& x, std::initializer_list<GemmProblem> problems) {
  GemmBatch g;
  gemm_batch_begin(g);
  for (const GemmProblem& p : problems) gemm_batch_add(g, p);
  // a split-K dW level adds into the step's zeroed gradient buffer, so a repeat would multiply the gradient
  RUN("gemm_launch", !gemm_batch_has_splitk(g), gemm_launch(g, x.c.precision, x.st));
  return D4PG_OK;
}

// 1. sample + gather (ddpg.py:187-197).  The same kernel derives this step's device-side
//    scalars (Adam bias corrections, PER beta, Philox counter) from the learner clock.
static int sample_batch(Step& x) {
  const d4pg_learner_config_t& c = x.c;
  RUN("learner_sample", false,
      learner_sample(x.L->replay, x.B, c.prioritized, c.sample_mode == 0 ? x.b.uniforms : nullptr,
                     (c.sample_mode == 0 && !c.prioritized) ? x.b.positions : nullptr,
                     c.philox_seed, x.w.clock, x.L->clock_params,
                     x.bt.idx, x.bt.wts, x.bt.s, x.bt.a, x.bt.r, x.bt.s2, x.bt.done, x.bt.hz, x.Sp, x.Ap, x.L->norm_affine,
                     x.L->norm_clip, x.pf ? x.par : -1, x.st));
  return D4PG_OK;
}

// ---- forward, PLAN_TC_CHAIN (mlp_tc_chain.cu): clusters of 8 CTAs own 64 rows, every layer a wgmma tile ---------------
static void tcc_begin(const Step& x, TccArgs& a, int step_slot) {
  tcc_args_begin(a, x.B, reinterpret_cast<uint8_t*>(x.w.xchg), x.c.precision == 1 ? 3 : 1);
  a.step_slot = step_slot;
}
// output group of layer l of `net` in slot `sl` of chain `ci`
static int tcc_fwd_group(TccArgs& fa, int ci, int sl, const Step& x, Net net, int l, float* C, int ldc, int publish) {
  const Layer y = layer(x.L, net, l);
  return tcc_slot_group(fa, ci, sl, x.L->tcc_img[fwd_image(net, l)], y.epi, y.bias, nullptr, 0, C, ldc, publish);
}
// Actor `an` on `s`, then critic `cn` on (s, that action); fc1 of both networks share the resident chunk of s:
//   T: actor_target(s') -> critic_target(s', .)                                                          ddpg.py:205-206
//   P: actor(s) -> critic(s, actor(s))                                                                   ddpg.py:236-238
// keep: the hidden activations are also stored row-major (sets ka / kc), for the backward pass of the online nets.
// actor_only: the post-update plan's chain 1; its critic pass follows the critic's Adam
static void tcc_build_actor_critic(TccArgs& fa, int ci, const Step& x, Net an, Net cn, const float* s, int ka, int kc,
                                   bool keep, bool actor_only = false) {
  const Workspace& w = x.w;
  const int H = D4PG_HIDDEN;
  int l, p1, p2 = -1;
  tcc_chain_x0(fa, ci, s, x.Sp, x.S);
  l = tcc_slot_begin(fa, ci); tcc_slot_src_x(fa, ci, l);
  p1 = tcc_fwd_group(fa, ci, l, x, an, 0, keep ? w.h1[ka] : nullptr, H, 1);
  if (!actor_only) p2 = tcc_fwd_group(fa, ci, l, x, cn, 0, nullptr, H, 1);   // (P: same values as chain Q's h1)
  l = tcc_slot_begin(fa, ci); tcc_slot_src_plane(fa, ci, l, p1, 8);
  p1 = tcc_fwd_group(fa, ci, l, x, an, 1, keep ? w.h2[ka] : nullptr, H, 1);
  l = tcc_slot_begin(fa, ci); tcc_slot_src_plane(fa, ci, l, p1, 8);
  p1 = tcc_fwd_group(fa, ci, l, x, an, 2, keep ? w.h3[ka] : nullptr, H, 1);
  l = tcc_slot_begin(fa, ci); tcc_slot_src_plane(fa, ci, l, p1, 8);
  const int pa = tcc_fwd_group(fa, ci, l, x, an, 3, w.out[ka], x.Ap, 1);
  if (actor_only) return;
  l = tcc_slot_begin(fa, ci); tcc_slot_src_plane(fa, ci, l, p2, 8); tcc_slot_src_plane(fa, ci, l, pa, 1);
  p1 = tcc_fwd_group(fa, ci, l, x, cn, 1, keep ? w.h2[kc] : nullptr, H, 1);
  l = tcc_slot_begin(fa, ci); tcc_slot_src_plane(fa, ci, l, p1, 8);
  p1 = tcc_fwd_group(fa, ci, l, x, cn, 2, keep ? w.h3[kc] : nullptr, H, 1);
  l = tcc_slot_begin(fa, ci); tcc_slot_src_plane(fa, ci, l, p1, 8);
  tcc_fwd_group(fa, ci, l, x, cn, 3, w.out[kc], x.Np, 0);
}
// critic(s, `act`): the resident chunk holds s for fc1, then the action rows (fc2's K tail)                ddpg.py:208
static void tcc_build_Q(TccArgs& fa, int ci, const Step& x, const float* act, float* h1, float* h2, float* h3, float* logits) {
  const int H = D4PG_HIDDEN;
  int l, p1;
  tcc_chain_x0(fa, ci, x.bt.s, x.Sp, x.S);
  l = tcc_slot_begin(fa, ci); tcc_slot_src_x(fa, ci, l); tcc_slot_reconvert_x(fa, ci, l, act, x.Ap, x.A);
  p1 = tcc_fwd_group(fa, ci, l, x, CRITIC, 0, h1, H, 1);
  l = tcc_slot_begin(fa, ci); tcc_slot_src_plane(fa, ci, l, p1, 8); tcc_slot_src_x(fa, ci, l);
  p1 = tcc_fwd_group(fa, ci, l, x, CRITIC, 1, h2, H, 1);
  l = tcc_slot_begin(fa, ci); tcc_slot_src_plane(fa, ci, l, p1, 8);
  p1 = tcc_fwd_group(fa, ci, l, x, CRITIC, 2, h3, H, 1);
  l = tcc_slot_begin(fa, ci); tcc_slot_src_plane(fa, ci, l, p1, 8);
  tcc_fwd_group(fa, ci, l, x, CRITIC, 3, logits, x.Np, 0);
}
// 2''. the three forward chains on the tensor cores.  pack_fwd: re-pack the hi/lo forward weight images first (the
// caller may have changed the parameters; otherwise the previous step's Adam kernel kept them current)
static int forward_tc_chain(Step& x, bool pack_fwd) {
  d4pg_learner* L = x.L; const Workspace& w = x.w;
  if (pack_fwd) RUN("launch_tcc_pack", false, launch_tcc_pack(L->tcc_pack_fwd, x.st));
  // the transposed images of the dX chains are needed only after the forward chains and heads: packed on the side branch
  D4PG_CUDA_OK(cudaEventRecord(L->ev_fork2, x.st));
  D4PG_CUDA_OK(cudaStreamWaitEvent(L->side, L->ev_fork2, 0));
  RUN("launch_tcc_pack", false, launch_tcc_pack(L->tcc_pack_dx, L->side));
  D4PG_CUDA_OK(cudaEventRecord(L->ev_join2, L->side));
  TccArgs& fa = L->tcc_fwd_args;
  tcc_begin(x, fa, 1);
  tcc_build_actor_critic(fa, 0, x, ACTOR_TARGET, CRITIC_TARGET, x.bt.s2, 0, 1, false);   // chain 0  T
  tcc_build_actor_critic(fa, 1, x, ACTOR, CRITIC, x.bt.s, 3, 4, true, x.h7);             // chain 1  P (post-update plan: the actor alone)
  tcc_build_Q(fa, 2, x, x.bt.a, w.h1[2], w.h2[2], w.h3[2], w.out[2]);   // chain 2  Q: critic(s, a)
  if (host_pipe(x.c) && !x.cold) {
    // warm host-pipeline variant: the batch comes from the ingest stream's sample kernel; instead of a stream event
    // (event + graph start after the sample ends) every CTA polls the epochs that kernel publishes
    fa.wait_epoch = w.pipe_epoch; fa.wait_clock = reinterpret_cast<const long long*>(&w.clock->steps_done);
    fa.wait_n = cdiv(x.B, SAMPLE_ROWS);
  }
  RUN("launch_mlp_tc_chain", true, launch_mlp_tc_chain(fa, x.st));
  return D4PG_OK;
}

// ---- forward, PLAN_CHAIN (mlp_chain.cu) -----------------------------------------------------------------------------
static ChainSlot chain_layer(const Step& x, Net net, int l, float* C, int ldc, int publish) {
  const Layer y = layer(x.L, net, l);
  return chain_fwd(y.W, y.ldw, y.bias, y.n_out, y.k_in, y.epi, C, ldc, publish);
}
// actor `an` on `s`, then critic `cn` on (s, that action), as chain `ci`: T (the targets on s') and P (the online nets on
// s).  ka / kc: the activation sets they write; c_h1: where the critic's h1 goes (nullptr: exchange only)
static void chain_build_actor_critic(const Step& x, ChainArgs& ca, int ci, Net an, Net cn, const float* s, int ka,
                                     float* c_h1, int kc) {
  const Workspace& w = x.w;
  const int H = D4PG_HIDDEN;
  ChainSlot sl; int t, a3 = -1;
  sl = chain_layer(x, an, 0, w.h1[ka], H, 1); chain_src_global(sl, s, x.Sp); t = chain_add(ca, ci, sl);
  sl = chain_layer(x, an, 1, w.h2[ka], H, 1); chain_src_plane(sl, t); t = chain_add(ca, ci, sl);
  sl = chain_layer(x, an, 2, w.h3[ka], H, 1); chain_src_plane(sl, t); const int a22 = chain_add(ca, ci, sl);
  // the 6-wide actor fc3 is a PRE-LAYER of the critic's fc2 slot (every CTA computes it for its 32 rows) instead of
  // a slot of its own, when it fits; otherwise it is a slot that publishes 8 plane rows
  if (!chain_pre_ok(x.c)) { sl = chain_layer(x, an, 3, w.out[ka], x.Ap, 1); chain_src_plane(sl, a22); a3 = chain_add(ca, ci, sl); }
  sl = chain_layer(x, cn, 0, c_h1, H, 1); chain_src_global(sl, s, x.Sp); t = chain_add(ca, ci, sl);
  sl = chain_layer(x, cn, 1, w.h2[kc], H, 1); chain_src_plane(sl, t);
  if (chain_pre_ok(x.c)) {
    const Layer y = layer(x.L, an, 3);
    chain_pre_layer(sl, y.W, y.ldw, y.bias, nullptr, 0, y.n_out, y.k_in, y.epi, w.out[ka], x.Ap, a22, H, false);
  } else chain_src2_plane(sl, H, a3);
  t = chain_add(ca, ci, sl);
  sl = chain_layer(x, cn, 2, w.h3[kc], H, 1); chain_src_plane(sl, t); t = chain_add(ca, ci, sl);
  sl = chain_layer(x, cn, 3, w.out[kc], x.Np, 0); chain_src_plane(sl, t); chain_add(ca, ci, sl);
}
// 2'. the three forward chains of the step as ONE cluster launch:
//   chain 0  T: actor_target(s') -> critic_target(s', .)      ddpg.py:205-206
//   chain 1  P: actor(s) -> critic(s, actor(s))                ddpg.py:236-238 (fc1 of the critic is recomputed: K=|s|)
//   chain 2  Q: critic(s, a)                                   ddpg.py:208
// The block scheduler fills SMs in launch order: the two 8-layer chains come first so that each of their CTAs
// gets an SM of its own, and the short 4-layer chain is the one that doubles up
static int forward_chain(Step& x) {
  const Workspace& w = x.w;
  const int H = D4PG_HIDDEN;
  ChainArgs& ca = x.L->chain_fwd_args;
  chain_args_begin(ca, x.B, w.xchg, x.c.precision);
  chain_build_actor_critic(x, ca, 0, ACTOR_TARGET, CRITIC_TARGET, x.bt.s2, 0, w.h1[1], 1);
  ChainSlot sl; int t;
  sl = chain_layer(x, CRITIC, 0, w.h1[2], H, 1); chain_src_global(sl, x.bt.s, x.Sp); t = chain_add(ca, 2, sl);
  sl = chain_layer(x, CRITIC, 1, w.h2[2], H, 1); chain_src_plane(sl, t); chain_src2_global(sl, H, x.bt.a, x.Ap); t = chain_add(ca, 2, sl);
  sl = chain_layer(x, CRITIC, 2, w.h3[2], H, 1); chain_src_plane(sl, t); t = chain_add(ca, 2, sl);
  sl = chain_layer(x, CRITIC, 3, w.out[2], x.Np, 0); chain_src_plane(sl, t); chain_add(ca, 2, sl);
  chain_build_actor_critic(x, ca, 1, ACTOR, CRITIC, x.bt.s, 3, nullptr, 4);
  RUN("launch_mlp_chain", true, launch_mlp_chain(ca, x.st));
  return D4PG_OK;
}

// ---- forward, PLAN_LEVELS: one grouped launch per dependency level ----------------------------------------------------
static GemmProblem level_fwd(const Step& x, Net net, int l, const float* X, int ldx, float* Y, int ldy,
                             const float* act = nullptr) {     // act: the action rows critic fc2 concatenates to X
  const Layer y = layer(x.L, net, l);
  return gemm_fwd(X, ldx, act, act ? x.Ap : 0, act ? D4PG_HIDDEN : 0, y.W, y.ldw, y.bias, Y, ldy, x.B, y.n_out, y.k_in, y.epi);
}
static int forward_levels(Step& x) {
  const Workspace& w = x.w; const Batch& bt = x.bt;
  const int H = D4PG_HIDDEN, Sp = x.Sp, Ap = x.Ap, Np = x.Np;
  // 2. forward level 1: fc1 of actor_target(s'), critic_target(s'), critic(s), actor(s)
  int rc = run_level(x, {level_fwd(x, ACTOR_TARGET, 0, bt.s2, Sp, w.h1[0], H),
                         level_fwd(x, CRITIC_TARGET, 0, bt.s2, Sp, w.h1[1], H),
                         level_fwd(x, CRITIC, 0, bt.s, Sp, w.h1[2], H),
                         level_fwd(x, ACTOR, 0, bt.s, Sp, w.h1[3], H)});
  // level 2: fc2 (actor: no activation, models.py:36; critic: cat(h1, a) + relu, models.py:80)
  if (!rc) rc = run_level(x, {level_fwd(x, ACTOR_TARGET, 1, w.h1[0], H, w.h2[0], H),
                              level_fwd(x, CRITIC, 1, w.h1[2], H, w.h2[2], H, bt.a),
                              level_fwd(x, ACTOR, 1, w.h1[3], H, w.h2[3], H)});
  // level 3: fc2_2 + relu
  if (!rc) rc = run_level(x, {level_fwd(x, ACTOR_TARGET, 2, w.h2[0], H, w.h3[0], H),
                              level_fwd(x, CRITIC, 2, w.h2[2], H, w.h3[2], H),
                              level_fwd(x, ACTOR, 2, w.h2[3], H, w.h3[3], H)});
  // level 4: fc3 (actor: tanh; critic: logits)
  if (!rc) rc = run_level(x, {level_fwd(x, ACTOR_TARGET, 3, w.h3[0], H, w.out[0], Ap),
                              level_fwd(x, CRITIC, 3, w.h3[2], H, w.out[2], Np),
                              level_fwd(x, ACTOR, 3, w.h3[3], H, w.out[3], Ap)});
  // level 5: critic_target.fc2([h1t, a_t(s')]) and critic.fc2([h1, actor(s)]) (h1 of the critic is reused)
  if (!rc) rc = run_level(x, {level_fwd(x, CRITIC_TARGET, 1, w.h1[1], H, w.h2[1], H, w.out[0]),
                              level_fwd(x, CRITIC, 1, w.h1[2], H, w.h2[4], H, w.out[3])});
  if (!rc) rc = run_level(x, {level_fwd(x, CRITIC_TARGET, 2, w.h2[1], H, w.h3[1], H),
                              level_fwd(x, CRITIC, 2, w.h2[4], H, w.h3[4], H)});
  if (!rc) rc = run_level(x, {level_fwd(x, CRITIC_TARGET, 3, w.h3[1], H, w.out[1], Np),
                              level_fwd(x, CRITIC, 3, w.h3[4], H, w.out[4], Np)});
  return rc;
}

// 3. heads: softmaxes, projection, CE loss, td, priorities, logit gradients (ddpg.py:214-222,236-238); the mixture
//    critic's quadrature cross-entropy (mog_heads.cu) or the quantile critic's quantile-Huber loss (qr_heads.cu) in their
//    place.  only_policy: the second loss launch of the post-update plan, the policy head on the updated critic's output
static HeadCommon head_common(const Step& x, bool only_policy) {
  const d4pg_learner_config_t& c = x.c; const Workspace& w = x.w;
  HeadCommon h{};
  h.target = w.out[1]; h.q = w.out[2]; h.pi = (x.h7 && !only_policy) ? nullptr : w.out[4];
  h.rewards = x.bt.r; h.dones = x.bt.done; h.B = x.B; h.ld = x.Np;
  // live projection discounts with gamma even for n_steps>1 (SURVEY.md H5); mode 1 uses gamma**n (ddpg.py:24)
  h.discount = (c.proj_mode == 1) ? pow(c.gamma, double(c.n_steps)) : c.gamma; h.prio_eps = c.prio_eps;
  h.grad_scale = 1.0f / (float(x.B) * float(c.world_size > 1 ? c.world_size : 1));
  h.loss_rows = w.loss_rows; h.td = x.b.td; h.prio = x.b.prio; h.dq = w.dlogits_q;
  h.pi_rows = w.pi_rows; h.dpi = w.dlogits_pi;
  h.is_weights = ((c.loss_flags & 1) && c.prioritized) ? x.bt.wts : nullptr;
  h.only_policy = only_policy ? 1 : 0;
  h.sampler_clock = (x.pf && !only_policy) ? w.clock : nullptr;    // sample(t) is done, sample(t+1) not yet launched
  h.horizon = x.bt.hz; h.gtab = x.L->gtab;                           // episode tails: this batch's horizons
  return h;
}
static int launch_step_heads(Step& x, bool only_policy) {
  const d4pg_learner_config_t& c = x.c; const Workspace& w = x.w;
  const HeadCommon h = head_common(x, only_policy);
  const int ce_priority = (c.loss_flags & 2) ? 1 : 0;
  // the loss kernel also advances the sampler clock under the pipelines: not idempotent there
  const bool rep = !x.pf;
  if (c.dist_type == 1) {
    MogArgs ma{h, c.n_components};
    RUN("launch_mog_heads", rep, launch_mog_heads(ma, x.st));
  } else if (c.dist_type == 2) {
    QrArgs qa{h, x.N, c.qr_kappa, ce_priority};
    RUN("launch_qr_heads", rep, launch_qr_heads(qa, x.st));
  } else {
    HeadsArgs ha{};
    ha.h = h; ha.N = x.N; ha.ce_priority = ce_priority;
    ha.v_min = c.v_min; ha.delta = (c.v_max - c.v_min) / double(x.N - 1);
    ha.v_max = proj_clip_top(c.v_min, c.v_max, x.N, ha.delta);
    ha.m = w.m; ha.target_probs = w.target_probs; ha.q_probs = w.q_probs;
    RUN("launch_heads", rep, launch_heads(ha, c.proj_mode, x.st));
  }
  return D4PG_OK;
}

// 4. priorities into the trees (ddpg.py:252-255): independent of the backward pass, so it runs
//    on a forked branch (side stream -> parallel graph branch) and joins before the step ends
static int side_branch(Step& x) {
  d4pg_learner* L = x.L; const d4pg_learner_config_t& c = x.c;
  D4PG_CUDA_OK(cudaEventRecord(L->ev_fork, x.st));
  D4PG_CUDA_OK(cudaStreamWaitEvent(L->side, L->ev_fork, 0));
  // host pipeline: the write-back also opens the ingest gate of step k+1 (its tree add / presample wait for this step's
  // loss kernel -- which advanced the sampler clock -- and for the priorities)
  if (c.prioritized)
    RUN("launch_tree_update", false,
        launch_tree_update(L->replay, x.B, x.bt.idx, x.b.prio, L->side, host_pipe(c) ? L->gate_flag : nullptr));
  else if (host_pipe(c)) RUN("launch_gate_signal", false, launch_gate_signal(L->gate_flag, L->side));
  if (prefetching(c)) {
    // 4'. the NEXT step's batch, sampled from the just-updated trees into the other half of the batch buffers
    // while this step's backward pass, dW and Adam run (it needs the trees, not the weights)
    const int q = x.par ^ 1;
    const Batch& o = x.w.batch[q];
    RUN("learner_sample", false,
        learner_sample(L->replay, x.B, c.prioritized, nullptr, nullptr, c.philox_seed, x.w.clock, L->clock_params,
                       o.idx, o.wts, o.s, o.a, o.r, o.s2, o.done, o.hz, x.Sp, x.Ap, L->norm_affine, L->norm_clip, q, L->side));
  }
  if (x.pf) {                           // the caller-visible copies of this step's indices / IS weights (off the
    // path to the next batch: after the write-back and the prefetch)
    D4PG_CUDA_OK(cudaMemcpyAsync(x.b.idx, x.bt.idx, size_t(x.B) * sizeof(int32_t), cudaMemcpyDeviceToDevice, L->side));
    if (x.b.weights && c.prioritized)
      D4PG_CUDA_OK(cudaMemcpyAsync(x.b.weights, x.bt.wts, size_t(x.B) * sizeof(float), cudaMemcpyDeviceToDevice, L->side));
  }
  D4PG_CUDA_OK(cudaEventRecord(L->ev_join, L->side));
  return D4PG_OK;
}

// Where this step's gradients go, and how the ranks will exchange them
static int choose_gradient_buffers(Step& x) {
  const d4pg_learner_buffers_t& b = x.b;
  x.Ga = b.grad_actor; x.Gc = b.grad_critic;
  x.peers = PeerInfo{};
  x.xm = exchange_mode(x.L, &x.peers);
  x.gpar = x.pf ? x.par : int(x.L->steps_done & 1);
  // data parallel with IPC-mapped peers: this step's gradients go straight into this rank's half of the exchange
  // buffer (double-buffered by step parity), the Adam kernel sums all ranks' halves over NVLink: the multicast-bound
  // buffer when the in-switch reduction is set up, else the IPC-mapped one the peers read directly
  if (peer_exchange(x)) {
    const bool use_mc_buf = x.xm == XCHG_MC || x.xm == XCHG_MC2;
    x.Ga = (use_mc_buf ? x.peers.mc_uc : x.peers.x[x.peers.rank]) + int64_t(x.gpar) * x.peers.n;
    x.Gc = x.Ga + x.L->da.total;
  }
  if (x.B >= 1024)                // dW levels run split-K with fp32 atomics: the gradient buffer must start at zero
    D4PG_CUDA_OK(cudaMemsetAsync(x.Ga, 0, size_t(x.L->da.total + x.L->dc.total) * sizeof(float), x.st));
  return D4PG_OK;
}

// ---- backward -----------------------------------------------------------------------------------------------------
// "c_" = critic-loss pass, "p_" = policy pass through the critic, "a_" = actor.
// C: critic loss, dlogits_q -> fc3 -> fc2_2 -> fc2[:, :H]                                                  ddpg.py:230
static void tcc_build_bwd_C(TccArgs& ba, int ci, const Step& x) {
  const TccImage* U = x.L->tcc_img; const Workspace& w = x.w;
  const int H = D4PG_HIDDEN;
  int l, p1;
  tcc_chain_pre(ba, ci, w.dlogits_q, x.Np, x.N);
  l = tcc_slot_begin(ba, ci); tcc_slot_src_pre(ba, ci, l);
  p1 = tcc_slot_group(ba, ci, l, U[U_C_D3], EPI_RELU_MASK, nullptr, w.h3[2], H, w.c_dz22, H, 1);
  l = tcc_slot_begin(ba, ci); tcc_slot_src_plane(ba, ci, l, p1, 8);
  p1 = tcc_slot_group(ba, ci, l, U[U_C_D22], EPI_RELU_MASK, nullptr, w.h2[2], H, w.c_dz2, H, 1);
  l = tcc_slot_begin(ba, ci); tcc_slot_src_plane(ba, ci, l, p1, 8);
  tcc_slot_group(ba, ci, l, U[U_C_D2H], EPI_RELU_MASK, nullptr, w.h1[2], H, w.c_dz1, H, 0);
}
// P: policy loss, dlogits_pi -> critic fc3 -> fc2_2 -> fc2[:, H:] (d action, tanh') -> actor fc3 -> fc2_2 -> fc2   ddpg.py:242
static void tcc_build_bwd_P(TccArgs& ba, int ci, const Step& x) {
  const TccImage* U = x.L->tcc_img; const Workspace& w = x.w;
  const int H = D4PG_HIDDEN;
  int l, p1;
  tcc_chain_pre(ba, ci, w.dlogits_pi, x.Np, x.N);
  l = tcc_slot_begin(ba, ci); tcc_slot_src_pre(ba, ci, l);
  p1 = tcc_slot_group(ba, ci, l, U[U_C_D3], EPI_RELU_MASK, nullptr, w.h3[4], H, nullptr, H, 1);
  l = tcc_slot_begin(ba, ci); tcc_slot_src_plane(ba, ci, l, p1, 8);
  p1 = tcc_slot_group(ba, ci, l, U[U_C_D22], EPI_RELU_MASK, nullptr, w.h2[4], H, nullptr, H, 1);
  l = tcc_slot_begin(ba, ci); tcc_slot_src_plane(ba, ci, l, p1, 8);
  p1 = tcc_slot_group(ba, ci, l, U[U_C_D2A], EPI_TANH_MASK, nullptr, w.out[3], x.Ap, w.a_dz3, x.Ap, 1);
  l = tcc_slot_begin(ba, ci); tcc_slot_src_plane(ba, ci, l, p1, 1);
  p1 = tcc_slot_group(ba, ci, l, U[U_A_D3], EPI_RELU_MASK, nullptr, w.h3[3], H, w.a_dz22, H, 1);
  l = tcc_slot_begin(ba, ci); tcc_slot_src_plane(ba, ci, l, p1, 8);
  p1 = tcc_slot_group(ba, ci, l, U[U_A_D22], EPI_NONE, nullptr, nullptr, 0, w.a_dh2, H, 1);
  l = tcc_slot_begin(ba, ci); tcc_slot_src_plane(ba, ci, l, p1, 8);
  tcc_slot_group(ba, ci, l, U[U_A_D2], EPI_RELU_MASK, nullptr, w.h1[3], H, w.a_dz1, H, 0);
}
// 5''. both dX chains on the tensor cores (transposed weight images; masks applied by the epilogue)
static int backward_tc_chain(Step& x) {
  D4PG_CUDA_OK(cudaStreamWaitEvent(x.st, x.L->ev_join2, 0));     // transposed weight images are packed
  TccArgs& ba = x.L->tcc_bwd_args;
  tcc_begin(x, ba, 5);
  tcc_build_bwd_C(ba, 0, x);                                   // C: critic loss
  if (!x.h7) tcc_build_bwd_P(ba, 1, x);                        // P: policy loss (PRE-update critic weights, SURVEY.md H7)
  RUN("launch_mlp_tc_chain", true, launch_mlp_tc_chain(ba, x.st));
  return D4PG_OK;
}

static ChainSlot chain_layer_dx(const LayerDx& d, int epi, const float* aux, int ldaux, float* C, int ldc, int publish) {
  return chain_dx(d.W, d.ldw, d.n_in, d.k_out, epi, aux, ldaux, C, ldc, publish);
}
// 5'. both dX chains as ONE cluster launch
//   C: critic loss  dlogits_q  -> fc3 -> fc2_2 -> fc2[:, :H]                         ddpg.py:230
//   P: policy loss  dlogits_pi -> fc3 -> fc2_2 -> fc2[:, H:] (d action, tanh') ->
//                   actor fc3 -> fc2_2 -> fc2   (PRE-update critic weights, SURVEY.md H7)  ddpg.py:242
static int backward_chain(Step& x) {
  d4pg_learner* L = x.L; const Workspace& w = x.w;
  const int H = D4PG_HIDDEN, Ap = x.Ap, Np = x.Np;
  ChainArgs& cb = L->chain_bwd_args;
  chain_args_begin(cb, x.B, w.xchg, x.c.precision); cb.trace_base = 6 * CHAIN_MAX_SLOTS;
  ChainSlot sl; int t;
  sl = chain_layer_dx(layer_dx(L, CRITIC, 3), EPI_RELU_MASK, w.h3[2], H, w.c_dz22, H, 1); chain_src_global(sl, w.dlogits_q, Np); t = chain_add(cb, 0, sl);
  sl = chain_layer_dx(layer_dx(L, CRITIC, 2), EPI_RELU_MASK, w.h2[2], H, w.c_dz2, H, 1); chain_src_plane(sl, t); t = chain_add(cb, 0, sl);
  sl = chain_layer_dx(layer_dx(L, CRITIC, 1), EPI_RELU_MASK, w.h1[2], H, w.c_dz1, H, 0); chain_src_plane(sl, t); chain_add(cb, 0, sl);

  sl = chain_layer_dx(layer_dx(L, CRITIC, 3), EPI_RELU_MASK, w.h3[4], H, w.p_dz22, H, 1); chain_src_global(sl, w.dlogits_pi, Np); t = chain_add(cb, 1, sl);
  sl = chain_layer_dx(layer_dx(L, CRITIC, 2), EPI_RELU_MASK, w.h2[4], H, w.p_dz2, H, 1); chain_src_plane(sl, t); t = chain_add(cb, 1, sl);
  const LayerDx da = critic_fc2_action_dx(L);
  if (chain_pre_ok(x.c)) {      // d action (6 wide) as a pre-layer of the step through actor fc3
    sl = chain_layer_dx(layer_dx(L, ACTOR, 3), EPI_RELU_MASK, w.h3[3], H, w.a_dz22, H, 1);
    chain_pre_layer(sl, da.W, da.ldw, nullptr, w.out[3], Ap, da.n_in, da.k_out, EPI_TANH_MASK, w.a_dz3, Ap, t, H, true);
    t = chain_add(cb, 1, sl);
  } else {
    sl = chain_layer_dx(da, EPI_TANH_MASK, w.out[3], Ap, w.a_dz3, Ap, 1); chain_src_plane(sl, t); t = chain_add(cb, 1, sl);
    sl = chain_layer_dx(layer_dx(L, ACTOR, 3), EPI_RELU_MASK, w.h3[3], H, w.a_dz22, H, 1); chain_src_plane(sl, t); t = chain_add(cb, 1, sl);
  }
  sl = chain_layer_dx(layer_dx(L, ACTOR, 2), EPI_NONE, nullptr, 0, w.a_dh2, H, 1); chain_src_plane(sl, t); t = chain_add(cb, 1, sl);
  sl = chain_layer_dx(layer_dx(L, ACTOR, 1), EPI_RELU_MASK, w.h1[3], H, w.a_dz1, H, 0); chain_src_plane(sl, t); chain_add(cb, 1, sl);
  RUN("launch_mlp_chain", true, launch_mlp_chain(cb, x.st));
  return D4PG_OK;
}

// The weight (and bias) gradient of layer l of the critic (from the critic-loss pass) or of the actor
static GemmProblem dw_problem(const Step& x, Net net, int l) {
  const Workspace& w = x.w; const NetDims& da = x.L->da; const NetDims& dc = x.L->dc;
  const int B = x.B, S = x.S, A = x.A, N = x.N, H = D4PG_HIDDEN, Sp = x.Sp, Ap = x.Ap, Np = x.Np;
  const int* la = da.ld; const int* lc = dc.ld;
  float* Ga = x.Ga; float* Gc = x.Gc;
  if (net == CRITIC) switch (l) {
    case 0: return gemm_dw(w.c_dz1, H, x.bt.s, Sp, Gc + dc.w_off[0], lc[0], Gc + dc.b_off[0], H, S, B);
    case 1: return gemm_dw(w.c_dz2, H, w.h1[2], H, Gc + dc.w_off[1], lc[1], Gc + dc.b_off[1], H, H, B);   // the h1 columns
    case 2: return gemm_dw(w.c_dz22, H, w.h2[2], H, Gc + dc.w_off[2], lc[2], Gc + dc.b_off[2], H, H, B);
    default: return gemm_dw(w.dlogits_q, Np, w.h3[2], H, Gc + dc.w_off[3], lc[3], Gc + dc.b_off[3], N, H, B);
  }
  switch (l) {
    case 0: return gemm_dw(w.a_dz1, H, x.bt.s, Sp, Ga + da.w_off[0], la[0], Ga + da.b_off[0], H, S, B);
    case 1: return gemm_dw(w.a_dh2, H, w.h1[3], H, Ga + da.w_off[1], la[1], Ga + da.b_off[1], H, H, B);
    case 2: return gemm_dw(w.a_dz22, H, w.h2[3], H, Ga + da.w_off[2], la[2], Ga + da.b_off[2], H, H, B);
    default: return gemm_dw(w.a_dz3, Ap, w.h3[3], H, Ga + da.w_off[3], la[3], Ga + da.b_off[3], A, H, B);
  }
}
// critic fc2's action columns: dW2 = [dz2^T h1 | dz2^T a]
static GemmProblem dw_critic_fc2_action(const Step& x) {
  return gemm_dw(x.w.c_dz2, D4PG_HIDDEN, x.bt.a, x.Ap, x.Gc + critic_fc2_action_off(x.L), x.L->dc.ld[1], nullptr,
                 D4PG_HIDDEN, x.A, x.B);
}
// chain plans: every dW of the step as ONE grouped launch (the post-update plan: the critic's, later the actor's)
static int dw_wide(Step& x, bool critic, bool actor) {
  GemmWideBatch& gw = x.L->dw_batch;
  PeerSignal sig1{};
  if (peer_exchange(x)) sig1 = comm_peer_signal(x.peers, 0);
  gemm_wide_begin(gw, peer_exchange(x) ? &sig1 : nullptr);         // its last CTA signals the peers
  if (critic) gemm_wide_add(gw, dw_problem(x, CRITIC, 2));
  if (critic) gemm_wide_add(gw, dw_problem(x, CRITIC, 1));
  if (actor) gemm_wide_add(gw, dw_problem(x, ACTOR, 2));
  if (actor) gemm_wide_add(gw, dw_problem(x, ACTOR, 1));
  if (critic) gemm_wide_add(gw, dw_problem(x, CRITIC, 3));
  if (critic) gemm_wide_add(gw, dw_critic_fc2_action(x));
  if (critic) gemm_wide_add(gw, dw_problem(x, CRITIC, 0));
  if (actor) gemm_wide_add(gw, dw_problem(x, ACTOR, 3));
  if (actor) gemm_wide_add(gw, dw_problem(x, ACTOR, 0));
  RUN("gemm_wide_launch", false, gemm_wide_launch(gw, x.st));
  return D4PG_OK;
}

static GemmProblem level_dx(const Step& x, const LayerDx& d, const float* dZ, int lddz, float* dX, int lddx, int epi,
                            const float* aux, int ldaux) {
  return gemm_dx(dZ, lddz, d.W, d.ldw, dX, lddx, x.B, d.n_in, d.k_out, epi, aux, ldaux);
}
// 5. backward of the level plan: dX and dW of a layer share a level
static int backward_levels(Step& x) {
  d4pg_learner* L = x.L; const Workspace& w = x.w;
  const int H = D4PG_HIDDEN, Ap = x.Ap, Np = x.Np;
  // level B1: through critic.fc3
  int rc = run_level(x, {level_dx(x, layer_dx(L, CRITIC, 3), w.dlogits_q, Np, w.c_dz22, H, EPI_RELU_MASK, w.h3[2], H),
                         level_dx(x, layer_dx(L, CRITIC, 3), w.dlogits_pi, Np, w.p_dz22, H, EPI_RELU_MASK, w.h3[4], H),
                         dw_problem(x, CRITIC, 3)});
  // level B2: through critic.fc2_2
  if (!rc) rc = run_level(x, {level_dx(x, layer_dx(L, CRITIC, 2), w.c_dz22, H, w.c_dz2, H, EPI_RELU_MASK, w.h2[2], H),
                              level_dx(x, layer_dx(L, CRITIC, 2), w.p_dz22, H, w.p_dz2, H, EPI_RELU_MASK, w.h2[4], H),
                              dw_problem(x, CRITIC, 2)});
  // level B3: through critic.fc2: dh1 (critic loss), d action (policy, tanh' folded in), dW2 = [dz2^T h1 | dz2^T a]
  if (!rc) rc = run_level(x, {level_dx(x, layer_dx(L, CRITIC, 1), w.c_dz2, H, w.c_dz1, H, EPI_RELU_MASK, w.h1[2], H),
                              level_dx(x, critic_fc2_action_dx(L), w.p_dz2, H, w.a_dz3, Ap, EPI_TANH_MASK, w.out[3], Ap),
                              dw_problem(x, CRITIC, 1),
                              dw_critic_fc2_action(x)});
  // level B4: critic.fc1 weights; actor.fc3
  if (!rc) rc = run_level(x, {dw_problem(x, CRITIC, 0),
                              level_dx(x, layer_dx(L, ACTOR, 3), w.a_dz3, Ap, w.a_dz22, H, EPI_RELU_MASK, w.h3[3], H),
                              dw_problem(x, ACTOR, 3)});
  // level B5: actor.fc2_2 (its input h2 has no activation -> plain dX)
  if (!rc) rc = run_level(x, {level_dx(x, layer_dx(L, ACTOR, 2), w.a_dz22, H, w.a_dh2, H, EPI_NONE, nullptr, 0),
                              dw_problem(x, ACTOR, 2)});
  // level B6: actor.fc2
  if (!rc) rc = run_level(x, {level_dx(x, layer_dx(L, ACTOR, 1), w.a_dh2, H, w.a_dz1, H, EPI_RELU_MASK, w.h1[3], H),
                              dw_problem(x, ACTOR, 1)});
  // level B7: actor.fc1
  if (!rc) rc = run_level(x, {dw_problem(x, ACTOR, 0)});
  return rc;
}

// 6. data-parallel gradient exchange: ONE all-reduce over the flat [P_a + P_c] buffer.
// Every rank's half of this step must be complete before Adam sums them: the chain plans signal from the dW
// kernel and wait inside the Adam kernel; the level plan (several dW launches) uses a small barrier launch
static bool inline_sync(const Step& x) { return peer_exchange(x) && x.L->plan != PLAN_LEVELS; }
static int exchange_gradients(Step& x) {
  d4pg_learner* L = x.L;
  if (peer_exchange(x) && !inline_sync(x)) RUN("comm_peer_barrier", false, comm_peer_barrier(L->comm, x.st));
  // reduce-scatter + all-gather over peer memory: each rank reduces its 1/N slice and pushes it to everyone
  if (x.xm == XCHG_MC2) RUN("comm_mc_reduce_bcast", false, comm_mc_reduce_bcast(L->comm, x.gpar, x.st));
  else if (x.xm == XCHG_RS) RUN("comm_peer_reduce_scatter", false, comm_peer_reduce_scatter(L->comm, x.gpar, x.st));
  else if (x.xm == XCHG_ALLREDUCE)
    RUN("comm_allreduce", false, comm_allreduce(L->comm, x.Ga, L->da.total + L->dc.total, x.st));
  return D4PG_OK;
}

// 7. Adam (actor + critic), sync (identity), Polyak -- one launch, two segments
static AdamArgs adam_args(const Step& x) {
  d4pg_learner* L = x.L; const d4pg_learner_config_t& c = x.c; const d4pg_learner_buffers_t& b = x.b;
  const NetDims& da = L->da; const NetDims& dc = L->dc; const PeerInfo& peers = x.peers;
  AdamArgs aa{};
  aa.seg[0] = AdamSeg{b.actor, x.Ga, b.adam_m_actor, b.adam_v_actor, b.actor_target, da.total, nullptr, 0, 0.f, 0};
  aa.seg[1] = AdamSeg{b.critic, x.Gc, b.adam_m_critic, b.adam_v_critic, b.critic_target, dc.total, nullptr, 0, 0.f, 1};
  if (peer_exchange(x)) {                                       // sum of the ranks' halves, also stored in the caller's buffer
    aa.npeers = peers.world;
    for (int r = 0; r < peers.world; ++r) aa.peer_g[r] = peers.x[r] + int64_t(x.gpar) * peers.n;
    aa.seg[0].g_out = b.grad_actor; aa.seg[0].g_off = 0;
    aa.seg[1].g_out = b.grad_critic; aa.seg[1].g_off = da.total;
    aa.my_flags = inline_sync(x) ? peers.flag[peers.rank] : nullptr; aa.rank = peers.rank;
    if (x.xm == XCHG_MC) aa.mc_g = peers.mc + int64_t(x.gpar) * peers.n;   // NVSwitch reduces; signal 0 (every rank's dW done) is awaited in-kernel
    if (x.xm == XCHG_MC2) {                                     // the reduced gradient was broadcast into the local multicast-bound buffer
      aa.peer_reduced = 1;
      aa.seg[0].g = peers.mc_uc + 2 * peers.n; aa.seg[1].g = peers.mc_uc + 2 * peers.n + da.total;
      aa.my_flags = peers.flag2[peers.rank];
    }
    if (x.xm == XCHG_RS) {                                      // the reduced gradient is local: wait for every rank's "slice pushed", then stream it
      aa.peer_reduced = 1;
      aa.seg[0].g = peers.red[peers.rank]; aa.seg[1].g = peers.red[peers.rank] + da.total;
      aa.my_flags = peers.flag2[peers.rank];
    }
  }
  aa.nseg = 2;
  aa.seg[0].wd = float(c.weight_decay_actor); aa.seg[1].wd = float(c.weight_decay_critic);
  const double max_norm[2] = {c.max_grad_norm_actor, c.max_grad_norm_critic};
  for (int sg = 0; sg < 2; ++sg)
    if (max_norm[sg] != 0.0) {                                  // its norm goes to losses[2] (actor) / losses[3] (critic)
      aa.seg[sg].sq_partials = x.w.sq_partials + sg * GRAD_NORM_CTAS; aa.seg[sg].max_norm = max_norm[sg];
      aa.seg[sg].norm_out = b.losses + 2 + sg;
    }
  if (L->plan == PLAN_TC_CHAIN) {                               // keep the forward weight images of the tensor-core chains current
    const TccImage* U = L->tcc_img;
    const NetDims* nd[2] = {&da, &dc};
    const Net online[2] = {ACTOR, CRITIC}, target[2] = {ACTOR_TARGET, CRITIC_TARGET};
    for (int sg = 0; sg < 2; ++sg) {
      aa.seg[sg].nimg = 4;
      for (int ly = 0; ly < 4; ++ly) {
        AdamImgLayer& I = aa.seg[sg].imgl[ly];
        I.w_off = nd[sg]->w_off[ly]; I.w_end = I.w_off + int64_t(nd[sg]->out[ly]) * nd[sg]->ld[ly];
        I.ld = nd[sg]->ld[ly]; I.nchunks = U[fwd_image(online[sg], ly)].kchunks;
        I.img = const_cast<uint8_t*>(U[fwd_image(online[sg], ly)].ptr);
        I.img_t = const_cast<uint8_t*>(U[fwd_image(target[sg], ly)].ptr);
      }
    }
  }
  aa.w1 = float(1.0 - c.beta1); aa.w2 = float(1.0 - c.beta2); aa.beta2 = float(c.beta2); aa.eps = float(c.adam_eps);
  aa.tau = float(c.tau); aa.one_minus_tau = float(1.0 - c.tau); aa.grad_scale = 1.0f; aa.clock = x.w.clock;
  aa.pipe_slot = x.pf ? x.par : -1;
  // tail slice of the same launch: reported batch-mean losses + advance the device clock
  aa.loss_rows = x.w.loss_rows; aa.pi_rows = x.w.pi_rows; aa.B = x.B; aa.inv_count = 1.0f / float(x.B); aa.loss_out = b.losses;
  return aa;
}
// An Adam launch; when a segment of it clips, the sum of squares of that segment's complete gradient right before it
static int launch_update(Step& x, const AdamArgs& a) {
  if (adam_clips(a)) RUN("launch_grad_sqnorm", true, launch_grad_sqnorm(a, x.st));
  RUN("launch_adam", false, launch_adam(a, x.st));
  return D4PG_OK;
}
// the second half of a post-update-critic step: the critic's Adam, then the policy pass through the updated critic
static int post_update_half(Step& x, const AdamArgs& aa) {
  d4pg_learner* L = x.L; const Workspace& w = x.w;
  AdamArgs ac = aa;                                            // critic update alone (writes the critic's forward images too)
  ac.seg[0] = aa.seg[1]; ac.nseg = 1; ac.skip_tail = 1;
  if (int rc = launch_update(x, ac)) return rc;
  RUN("launch_tcc_pack", false, launch_tcc_pack(L->tcc_pack_dx, x.st));   // transposed images of the UPDATED critic for the policy backward
  TccArgs& fb = L->tcc_fwd_args;
  tcc_begin(x, fb, 1);
  tcc_build_Q(fb, 0, x, w.out[3], nullptr, w.h2[4], w.h3[4], w.out[4]);      // critic(s, actor(s)) with the new critic weights
  RUN("launch_mlp_tc_chain", true, launch_mlp_tc_chain(fb, x.st));
  if (int rc = launch_step_heads(x, true)) return rc;
  TccArgs& bb = L->tcc_bwd_args;
  tcc_begin(x, bb, 5);
  tcc_build_bwd_P(bb, 0, x);
  RUN("launch_mlp_tc_chain", true, launch_mlp_tc_chain(bb, x.st));
  if (int rc = dw_wide(x, false, true)) return rc;
  AdamArgs ab = aa;                                            // actor update + the step's tail (loss means, clock)
  ab.nseg = 1;
  return launch_update(x, ab);
}

// 7'. one launch for both networks, or the two half steps of the post-update plan
static int update(Step& x) {
  const AdamArgs aa = adam_args(x);
  if (x.h7) return post_update_half(x, aa);
  return launch_update(x, aa);
}

// par: half of the double-buffered batch this step trains on; cold: sample it first (no valid prefetch)
// pack_fwd: re-pack the forward weight images first (start of a graph launch / eager step: the caller may have changed
// the parameters); later steps of one multi-step graph rely on the images the previous step's Adam kernel wrote
static int enqueue_step(d4pg_learner* L, cudaStream_t st, int par, bool cold, bool pack_fwd) {
  const d4pg_learner_config_t& c = L->cfg;
  const bool pf = piped(c);
  Step x{L, st, c, L->buf, L->ws, L->ws.batch[par], par, cold, pf, (c.loss_flags & 4) != 0,
         c.batch, c.obs_dim, c.act_dim, c.n_atoms, pitch4(c.obs_dim), pitch4(c.act_dim), pitch4(c.n_atoms)};
  const StepPlan plan = L->plan;
  const bool side = c.prioritized || pf;                         // the step has a side branch
  int rc = (!pf || cold) ? sample_batch(x) : D4PG_OK;
  if (!rc) rc = plan == PLAN_TC_CHAIN ? forward_tc_chain(x, pack_fwd) : plan == PLAN_CHAIN ? forward_chain(x) : forward_levels(x);
  if (!rc) rc = launch_step_heads(x, false);
  if (!rc && side) rc = side_branch(x);
  if (!rc) rc = choose_gradient_buffers(x);
  if (!rc && plan == PLAN_TC_CHAIN) rc = backward_tc_chain(x);
  if (!rc && plan == PLAN_CHAIN) rc = backward_chain(x);
  if (!rc) rc = plan == PLAN_LEVELS ? backward_levels(x) : dw_wide(x, true, !x.h7);
  if (!rc) rc = exchange_gradients(x);
  if (!rc) rc = update(x);
  if (rc) return rc;
  if (side) D4PG_CUDA_OK(cudaStreamWaitEvent(st, L->ev_join, 0));
  L->kernels_per_step = x.nk;
  return D4PG_OK;
}
#undef RUN

extern "C" int64_t d4pg_learner_workspace_floats(const d4pg_learner_config_t* cfg) {
  if (!cfg) return -1;
  const d4pg_learner_config_t ec = with_head_width(*cfg);
  return carve(nullptr, ec.batch, ec.obs_dim, ec.act_dim, ec.n_atoms, step_plan(ec), piped(ec), clipping(ec),
               ec.nstep_tails != 0).total;
}

extern "C" int32_t d4pg_learner_create(const d4pg_learner_config_t* cfg, const d4pg_learner_buffers_t* buf,
                                       d4pg_replay_t* replay, d4pg_comm_t* comm, d4pg_learner_t** out) {
  D4PG_REQUIRE(cfg && buf && replay && out, D4PG_EINVAL, "d4pg_learner_create: null argument");
  D4PG_REQUIRE(cfg->batch > 0 && cfg->obs_dim > 0 && cfg->act_dim > 0, D4PG_EINVAL, "d4pg_learner_create: bad dims");
  D4PG_REQUIRE(cfg->dist_type >= 0 && cfg->dist_type <= 2, D4PG_EINVAL,
               "d4pg_learner_create: dist_type must be 0 (categorical), 1 (mixture of Gaussians) or 2 (quantile regression)");
  if (cfg->dist_type == 2) {
    D4PG_REQUIRE(cfg->n_atoms >= 2 && cfg->n_atoms <= D4PG_MAX_ATOMS, D4PG_EINVAL,
                 "d4pg_learner_create: the quantile critic's n_atoms (its N quantiles) must be in [2,%d]", D4PG_MAX_ATOMS);
    D4PG_REQUIRE(std::isfinite(cfg->qr_kappa) && cfg->qr_kappa > 0.0, D4PG_EINVAL,
                 "d4pg_learner_create: qr_kappa must be finite and > 0 (got %g)", cfg->qr_kappa);
  } else if (cfg->dist_type == 1) {
    D4PG_REQUIRE(cfg->n_components >= 1 && cfg->n_components <= D4PG_MAX_COMPONENTS, D4PG_EINVAL,
                 "d4pg_learner_create: n_components must be in [1,%d]", D4PG_MAX_COMPONENTS);
    D4PG_REQUIRE(!(cfg->loss_flags & 2), D4PG_ENOTSUP,
                 "d4pg_learner_create: loss_flags & 2 (cross-entropy priority) is not supported by the mixture critic: the cross-entropy of a density can be negative");
  } else {
    D4PG_REQUIRE(cfg->n_atoms >= 2 && cfg->n_atoms <= D4PG_MAX_ATOMS, D4PG_EINVAL, "d4pg_learner_create: n_atoms must be in [2,%d]", D4PG_MAX_ATOMS);
    D4PG_REQUIRE(cfg->v_max > cfg->v_min, D4PG_EINVAL, "d4pg_learner_create: v_max <= v_min");
  }
  const d4pg_learner_config_t ec = with_head_width(*cfg);
  D4PG_REQUIRE(cfg->proj_mode == 0 || cfg->proj_mode == 1, D4PG_EINVAL, "d4pg_learner_create: proj_mode must be 0/1");
  D4PG_REQUIRE(cfg->precision >= 0 && cfg->precision <= 3, D4PG_ENOTSUP,
               "d4pg_learner_create: precision %d unknown (0 fp32 FFMA, 1 3xTF32 wgmma, 2 TF32 wgmma, 3 bf16 wgmma)", cfg->precision);
  D4PG_REQUIRE(!clipping(*cfg) || cfg->world_size <= 1, D4PG_EINVAL,
               "d4pg_learner_create: max_grad_norm is not supported with world_size > 1: the ranks' gradients are summed "
               "inside the Adam kernel, so the norm of the summed gradient does not exist before the update");
  D4PG_REQUIRE(cfg->obs_norm == 0 || cfg->obs_norm == 1, D4PG_EINVAL, "d4pg_learner_create: obs_norm must be 0 or 1");
  D4PG_REQUIRE(!cfg->obs_norm || cfg->world_size <= 1, D4PG_EINVAL,
               "d4pg_learner_create: obs_norm is not supported with world_size > 1: each rank would normalize with the "
               "statistics of its own shard");
  double norm_clip = 0.0;
  const float* norm_affine = cfg->obs_norm ? replay_obs_norm(replay, &norm_clip) : nullptr;
  D4PG_REQUIRE(!cfg->obs_norm || norm_affine, D4PG_EINVAL,
               "d4pg_learner_create: obs_norm needs a replay with an observation normalizer (d4pg_replay_set_obs_norm)");
  D4PG_REQUIRE(cfg->nstep_tails == 0 || cfg->nstep_tails == 1, D4PG_EINVAL, "d4pg_learner_create: nstep_tails must be 0 or 1");
  D4PG_REQUIRE(!cfg->nstep_tails || cfg->proj_mode == 1 || cfg->n_steps <= 1, D4PG_EINVAL,
               "d4pg_learner_create: nstep_tails with proj_mode 0 (gamma for every row) and n_steps > 1: a per-row horizon "
               "has no meaning there");
  D4PG_REQUIRE(!cfg->nstep_tails || replay_horizons(replay), D4PG_EINVAL,
               "d4pg_learner_create: nstep_tails needs a replay with a horizon column (d4pg_replay_set_horizons)");
  D4PG_REQUIRE(cfg->world_size <= 1 || comm, D4PG_EINVAL, "d4pg_learner_create: world_size>1 needs a communicator");
  D4PG_REQUIRE(cfg->chain == 0 || cfg->chain == 1, D4PG_EINVAL, "d4pg_learner_create: chain must be 0 or 1");
  for (double mn : {cfg->max_grad_norm_actor, cfg->max_grad_norm_critic})
    D4PG_REQUIRE(mn == 0.0 || mn > 0.0, D4PG_EINVAL,
                 "d4pg_learner_create: max_grad_norm must be 0 (off), +inf (report only) or > 0 (got %g)", mn);
  for (double wd : {cfg->weight_decay_actor, cfg->weight_decay_critic})
    D4PG_REQUIRE(std::isfinite(wd) && wd >= 0.0, D4PG_EINVAL, "d4pg_learner_create: weight_decay must be finite and >= 0 (got %g)", wd);
  D4PG_REQUIRE(!(cfg->loss_flags & 4) || (step_plan(ec) == PLAN_TC_CHAIN && cfg->world_size <= 1), D4PG_ENOTSUP,
               "d4pg_learner_create: loss_flags & 4 (post-update-critic actor gradient) needs the tensor-core chain plan: precision 1 or 2 (not 0 or 3), chain 1, "
               "batch <= 512, obs_dim <= 32, act_dim <= 32, on one GPU");
  D4PG_REQUIRE(buf->actor && buf->actor_target && buf->critic && buf->critic_target && buf->grad_actor && buf->grad_critic &&
               buf->adam_m_actor && buf->adam_v_actor && buf->adam_m_critic && buf->adam_v_critic &&
               buf->idx && buf->prio && buf->td && buf->losses && buf->workspace, D4PG_EINVAL,
               "d4pg_learner_create: null device buffer");
  d4pg_learner* L = new (std::nothrow) d4pg_learner();
  D4PG_REQUIRE(L, D4PG_EINVAL, "d4pg_learner_create: out of host memory");
  L->cfg = ec; L->buf = *buf; L->replay = replay; L->comm = comm; L->plan = step_plan(ec);
  L->da = actor_dims(cfg->obs_dim, cfg->act_dim);
  L->dc = critic_dims(ec.obs_dim, ec.act_dim, ec.n_atoms);
  if (buf->grad_critic != buf->grad_actor + L->da.total) {
    set_error("d4pg_learner_create: grad_critic must equal grad_actor + P_a (one flat gradient buffer)");
    delete L; return D4PG_EINVAL;
  }
  L->ws = carve(buf->workspace, ec.batch, ec.obs_dim, ec.act_dim, ec.n_atoms, L->plan, piped(ec), clipping(ec),
                ec.nstep_tails != 0);
  if (!piped(ec)) { L->ws.batch[0].idx = buf->idx; L->ws.batch[0].wts = buf->weights; }   // sampled straight into the caller's buffers
  L->clock_params = ClockParams{ec.lr_actor, ec.lr_critic, ec.beta1, ec.beta2, ec.per_beta0, ec.per_beta_final,
                                ec.per_beta_iters > 0 ? ec.per_beta_iters : 1};
  for (int i = 0; i < 4; ++i) { L->graph_exec[i] = nullptr; L->graph_ready[i] = false; }
  for (int i = 0; i < 2; ++i) { L->multi_exec[i] = nullptr; L->multi_ready[i] = false; }
  L->pipe_par = 0; L->last_par = 0; L->prefetch_valid = false; L->seen_gen = -1;
  L->steps_done = 0; L->kernels_per_step = 0;
  L->profiling = false;
  (void)debug_trace_buffer();          // allocate outside of any stream capture
  if (L->plan == PLAN_TC_CHAIN)
    if (int rc = tcc_setup(L)) { delete L; return rc; }
  L->host_steps = 0; L->host_losses = nullptr; L->ev_in = nullptr; L->ev_out = nullptr;
  for (int i = 0; i < 4; ++i) { L->host_u[i] = nullptr; L->host_pos[i] = nullptr; L->ev_h2d[i] = nullptr; }
  for (int i = 0; i < 2; ++i) { L->loss_ring[i] = nullptr; L->ev_loss[i] = nullptr; }
  L->loss_steps = 0;
  L->ing = nullptr; L->ev_ing = nullptr; L->gate_flag = nullptr; L->images_dirty = true;
  L->norm_affine = norm_affine; L->norm_clip = float(norm_clip);
  L->gtab = nullptr;
  if (cfg->nstep_tails) {
    // the same pow as head_common's gamma^n_steps; uploaded once, so graph capture never sees the copy
    double g[D4PG_STEPS_MAX_N];
    for (int k = 0; k < D4PG_STEPS_MAX_N; ++k) g[k] = pow(cfg->gamma, double(k));
    if (cudaMalloc(reinterpret_cast<void**>(&L->gtab), sizeof(g)) != cudaSuccess ||
        cudaMemcpy(L->gtab, g, sizeof(g), cudaMemcpyHostToDevice) != cudaSuccess) {
      set_error("d4pg_learner_create: horizon table upload failed"); delete L; return D4PG_ECUDA;
    }
  }
  if (host_pipe(*cfg)) {
    L->gate_flag = replay_gate_flag(replay);
    const bool ok = L->gate_flag && cudaStreamCreateWithFlags(&L->ing, cudaStreamNonBlocking) == cudaSuccess &&
                    cudaEventCreateWithFlags(&L->ev_ing, cudaEventDisableTiming) == cudaSuccess;
    if (!ok) {
      set_error("d4pg_learner_create: ingest stream setup failed"); delete L; return D4PG_ECUDA;
    }
  }
  {
    const size_t nb = size_t(cfg->batch);
    bool ok = cudaEventCreateWithFlags(&L->ev_in, cudaEventDisableTiming) == cudaSuccess &&
              cudaEventCreateWithFlags(&L->ev_out, cudaEventDisableTiming) == cudaSuccess &&
              cudaHostAlloc(reinterpret_cast<void**>(&L->host_losses), 4 * sizeof(float), cudaHostAllocDefault) == cudaSuccess;
    for (int i = 0; i < 2 && ok; ++i)
      ok = cudaEventCreateWithFlags(&L->ev_loss[i], cudaEventDisableTiming) == cudaSuccess &&
           cudaHostAlloc(reinterpret_cast<void**>(&L->loss_ring[i]), 4 * sizeof(float), cudaHostAllocDefault) == cudaSuccess;
    for (int i = 0; i < 4 && ok; ++i)
      ok = cudaEventCreateWithFlags(&L->ev_h2d[i], cudaEventDisableTiming) == cudaSuccess &&
           cudaHostAlloc(reinterpret_cast<void**>(&L->host_u[i]), nb * sizeof(double), cudaHostAllocMapped) == cudaSuccess &&
           cudaHostAlloc(reinterpret_cast<void**>(&L->host_pos[i]), nb * sizeof(int32_t), cudaHostAllocMapped) == cudaSuccess;
    if (!ok) { set_error("d4pg_learner_create: pinned staging allocation failed"); delete L; return D4PG_ECUDA; }
  }
  if (cudaStreamCreateWithFlags(&L->side, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&L->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&L->ev_join, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&L->ev_fork2, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&L->ev_join2, cudaEventDisableTiming) != cudaSuccess) {
    set_error("d4pg_learner_create: stream/event creation failed"); delete L; return D4PG_ECUDA;
  }
  trace_set_side_stream(L->side);
  cudaError_t e = cudaMemset(L->ws.clock, 0, sizeof(LearnerClock));
  if (e == cudaSuccess) e = cudaMemset(L->ws.pipe_epoch, 0, sizeof(unsigned long long) * size_t(cdiv(cfg->batch, SAMPLE_ROWS)));
  if (e != cudaSuccess) { set_error("d4pg_learner_create: %s", cudaGetErrorString(e)); delete L; return D4PG_ECUDA; }
  *out = L;
  return D4PG_OK;
}

extern "C" int32_t d4pg_learner_destroy(d4pg_learner_t* L) {
  if (!L) return D4PG_OK;
  for (int i = 0; i < 4; ++i) if (L->graph_exec[i]) cudaGraphExecDestroy(L->graph_exec[i]);
  for (int i = 0; i < 2; ++i) if (L->multi_exec[i]) cudaGraphExecDestroy(L->multi_exec[i]);
  cudaEventDestroy(L->ev_fork); cudaEventDestroy(L->ev_join); cudaEventDestroy(L->ev_fork2); cudaEventDestroy(L->ev_join2);
  cudaStreamDestroy(L->side);
  if (L->tcc_images) cudaFree(L->tcc_images);
  if (L->gtab) cudaFree(L->gtab);
  if (L->ing) { cudaStreamSynchronize(L->ing); cudaStreamDestroy(L->ing); }
  if (L->ev_ing) cudaEventDestroy(L->ev_ing);
  if (L->ev_in) cudaEventDestroy(L->ev_in);
  if (L->ev_out) cudaEventDestroy(L->ev_out);
  if (L->host_losses) cudaFreeHost(L->host_losses);
  for (int i = 0; i < 2; ++i) {
    if (L->ev_loss[i]) cudaEventDestroy(L->ev_loss[i]);
    if (L->loss_ring[i]) cudaFreeHost(L->loss_ring[i]);
  }
  for (int i = 0; i < 4; ++i) {
    if (L->ev_h2d[i]) cudaEventDestroy(L->ev_h2d[i]);
    if (L->host_u[i]) cudaFreeHost(L->host_u[i]);
    if (L->host_pos[i]) cudaFreeHost(L->host_pos[i]);
  }
  delete L;
  return D4PG_OK;
}

// which half of the batch buffers the next step uses, and whether it has to sample it first
static void next_variant(d4pg_learner* L, int* par, bool* cold) {
  if (!piped(L->cfg)) { *par = 0; *cold = true; return; }
  *par = L->pipe_par;
  // host pipeline: a direct d4pg_learner_step samples in the graph; d4pg_learner_step_host presamples on the ingest stream
  *cold = host_pipe(L->cfg) || !L->prefetch_valid || replay_generation(L->replay) != L->seen_gen;
}
static void commit_variant(d4pg_learner* L, int par) {
  ++L->steps_done;
  if (!piped(L->cfg)) return;
  L->last_par = par; L->pipe_par = par ^ 1; L->prefetch_valid = true; L->seen_gen = replay_generation(L->replay);
}

// adds issued on the ingest stream come before the step
static int wait_for_ingest(d4pg_learner* L, cudaStream_t st) {
  if (!L->ing) return D4PG_OK;
  D4PG_CUDA_OK(cudaEventRecord(L->ev_ing, L->ing));
  D4PG_CUDA_OK(cudaStreamWaitEvent(st, L->ev_ing, 0));
  return D4PG_OK;
}

// capture what `body` enqueues on `st` into an executable graph
template <class F>
static int capture_graph(cudaStream_t st, cudaGraphExec_t* exec, const char* what, F body) {
  D4PG_REQUIRE(st != nullptr, D4PG_EINVAL, "%s: graph capture needs a non-default stream", what);
  cudaGraph_t graph = nullptr;
  D4PG_CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  const int rc = body();
  cudaError_t e = cudaStreamEndCapture(st, &graph);
  if (rc != D4PG_OK) { if (graph) cudaGraphDestroy(graph); return rc; }
  if (e != cudaSuccess) { set_error("%s: end capture: %s", what, cudaGetErrorString(e)); return D4PG_ECUDA; }
  e = cudaGraphInstantiate(exec, graph, 0);
  cudaGraphDestroy(graph);
  if (e != cudaSuccess) { set_error("%s: instantiate: %s", what, cudaGetErrorString(e)); return D4PG_ECUDA; }
  return D4PG_OK;
}

// one step of variant (par, cold) enqueued directly on `st`; arms the ingest gate of the next step
static int step_eager(d4pg_learner* L, cudaStream_t st, int par, bool cold) {
  // warm host-pipeline variants start from a sampled batch AND packed forward images (d4pg_learner_step_host packs
  // eagerly on the learner stream while the ingest stream still samples)
  const int rc = enqueue_step(L, st, par, cold, !(host_pipe(L->cfg) && !cold));
  if (rc == D4PG_OK) { commit_variant(L, par); if (L->ing) replay_arm_gate(L->replay); }
  return rc;
}

// the step graph of variant (par, cold) on `st` (captured on first use); arms the ingest gate of the next step
static int launch_variant(d4pg_learner* L, cudaStream_t st, int par, bool cold) {
  if (!L->cfg.use_graph) return step_eager(L, st, par, cold);
  // without the prefetch pipeline the only per-step variation is the gradient half of the peer exchange
  const int v = piped(L->cfg) ? par * 2 + (cold ? 1 : 0) : int(L->steps_done & 1);
  if (!L->graph_ready[v]) {
    const int rc = capture_graph(st, &L->graph_exec[v], "d4pg_learner_step",
                                 [&] { return enqueue_step(L, st, par, cold, !(host_pipe(L->cfg) && !cold)); });
    if (rc) return rc;
    L->graph_ready[v] = true;
  }
  D4PG_CUDA_OK(cudaGraphLaunch(L->graph_exec[v], st));
  commit_variant(L, par);
  if (L->ing) replay_arm_gate(L->replay);
  return D4PG_OK;
}

extern "C" int32_t d4pg_learner_step(d4pg_learner_t* L, d4pg_stream_t stream) {
  D4PG_REQUIRE(L, D4PG_EINVAL, "d4pg_learner_step: null handle");
  cudaStream_t st = as_stream(stream);
  int par; bool cold;
  next_variant(L, &par, &cold);
  if (int rc = wait_for_ingest(L, st)) return rc;
  return launch_variant(L, st, par, cold);
}

// host pipeline: sample + gather batch `par` from the device copy of this step's uniforms / positions (the launch the
// cold graph variant starts with, issued on the ingest stream instead)
static int presample(d4pg_learner* L, int par, const double* uniforms, const int32_t* positions, cudaStream_t st) {
  const d4pg_learner_config_t& c = L->cfg; const Workspace& w = L->ws; const Batch& o = w.batch[par];
  return learner_sample(L->replay, c.batch, c.prioritized, uniforms, !c.prioritized ? positions : nullptr, c.philox_seed,
                        w.clock, L->clock_params, o.idx, o.wts, o.s, o.a, o.r, o.s2, o.done, o.hz, pitch4(c.obs_dim),
                        pitch4(c.act_dim), L->norm_affine, L->norm_clip, par, st, /*dependent=*/true, w.pipe_epoch);
}

// The host-facing step: stage this step's host inputs in pinned memory, H2D, the step, order the caller after it.
static int step_host_common(d4pg_learner_t* L, const double* uniforms, const uint32_t* mt_words, const int32_t* positions,
                            d4pg_stream_t caller_stream, d4pg_stream_t learner_stream) {
  cudaStream_t cs = as_stream(caller_stream), ls = as_stream(learner_stream);
  const int B = L->cfg.batch;
  D4PG_CUDA_OK(cudaEventRecord(L->ev_in, cs));                 // adds / weight loads issued by the caller
  D4PG_CUDA_OK(cudaStreamWaitEvent(ls, L->ev_in, 0));
  const bool pipe = L->ing != nullptr && (uniforms || mt_words || positions);
  // piped: the sample kernel reads this step's uniforms / positions (2 KB) straight out of the pinned staging slot over
  // PCIe -- no copy node between the caller's add and the sample on the ingest stream -- so the slots form a ring of 4.
  // (The caller's replay operations on caller_stream are NOT waited for before sampling: the host mirror orders them
  // explicitly with d4pg_replay_order_after, see d4pg_learner_ingest_stream in the header.)
  const int par = int(L->host_steps & (pipe ? 3 : 1));
  double* du = L->buf.uniforms;
  int32_t* dpos = L->buf.positions;
  if (uniforms || mt_words || positions) {
    if (L->host_steps >= (pipe ? 4 : 2)) D4PG_CUDA_OK(cudaEventSynchronize(L->ev_h2d[par]));   // the last reader of this slot
    if (uniforms || mt_words) {
      D4PG_REQUIRE(du, D4PG_ESTATE, "d4pg_learner_step_host: no device uniforms buffer");
      double* u = L->host_u[par];
      if (uniforms) memcpy(u, uniforms, size_t(B) * sizeof(double));
      else                                                     // CPython random.random(): (a >> 5, b >> 6) -> (a * 2^26 + b) / 2^53
        for (int i = 0; i < B; ++i)
          u[i] = (double(mt_words[2 * i] >> 5) * 67108864.0 + double(mt_words[2 * i + 1] >> 6)) * (1.0 / 9007199254740992.0);
      if (pipe) D4PG_CUDA_OK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&du), u, 0));
      else D4PG_CUDA_OK(cudaMemcpyAsync(du, u, size_t(B) * sizeof(double), cudaMemcpyHostToDevice, ls));
    }
    if (positions) {
      D4PG_REQUIRE(dpos, D4PG_ESTATE, "d4pg_learner_step_host: no device positions buffer");
      memcpy(L->host_pos[par], positions, size_t(B) * sizeof(int32_t));
      if (pipe) D4PG_CUDA_OK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&dpos), L->host_pos[par], 0));
      else D4PG_CUDA_OK(cudaMemcpyAsync(dpos, L->host_pos[par], size_t(B) * sizeof(int32_t), cudaMemcpyHostToDevice, ls));
    }
    if (!pipe) D4PG_CUDA_OK(cudaEventRecord(L->ev_h2d[par], ls));
    ++L->host_steps;
  }
  int rc;
  if (pipe) {
    // batch k on the ingest stream: behind the caller's add(k) (same stream) and the gate of step k-1, while step k-1's
    // backward pass / dW / Adam still run on the learner stream; the step graph starts from the sampled batch
    const int bpar = L->pipe_par;
    rc = replay_gate_consume(L->replay, L->ing);
    if (rc) return rc;
    rc = presample(L, bpar, du, dpos, L->ing);
    if (rc) return rc;
    D4PG_CUDA_OK(cudaEventRecord(L->ev_h2d[par], L->ing));      // the staging slot has been read
    D4PG_CUDA_OK(cudaEventRecord(L->ev_ing, L->ing));
    // forward weight images: the Adam kernel keeps them current, so they are re-packed only after the caller reported a
    // parameter write of its own (d4pg_learner_weights_changed) -- behind Adam(k-1), beside the ingest stream's tail
    if (L->images_dirty && L->plan == PLAN_TC_CHAIN) {
      rc = launch_tcc_pack(L->tcc_pack_fwd, ls);
      if (rc) return rc;
    }
    L->images_dirty = false;
    // the wgmma forward chains poll the sampler's epochs themselves; the other plans start after its event
    if (L->plan != PLAN_TC_CHAIN) D4PG_CUDA_OK(cudaStreamWaitEvent(ls, L->ev_ing, 0));
    rc = launch_variant(L, ls, bpar, false);
  } else {
    rc = d4pg_learner_step(L, learner_stream);
  }
  if (rc) return rc;
  {                                                            // this step's result, queued for d4pg_learner_fetch_losses
    const int slot = int(L->loss_steps & 1);
    D4PG_CUDA_OK(cudaMemcpyAsync(L->loss_ring[slot], L->buf.losses, 4 * sizeof(float), cudaMemcpyDeviceToHost, ls));
    D4PG_CUDA_OK(cudaEventRecord(L->ev_loss[slot], ls));
    ++L->loss_steps;
  }
  D4PG_CUDA_OK(cudaEventRecord(L->ev_out, ls));
  D4PG_CUDA_OK(cudaStreamWaitEvent(cs, L->ev_out, 0));
  return D4PG_OK;
}

extern "C" int32_t d4pg_learner_fetch_losses(d4pg_learner_t* L, int32_t lag, float* out4) {
  D4PG_REQUIRE(L && out4 && (lag == 0 || lag == 1), D4PG_EINVAL, "d4pg_learner_fetch_losses: lag must be 0 or 1");
  D4PG_REQUIRE(L->loss_steps > lag, D4PG_ESTATE, "d4pg_learner_fetch_losses: no such step yet");
  const int slot = int((L->loss_steps - 1 - lag) & 1);
  D4PG_CUDA_OK(cudaEventSynchronize(L->ev_loss[slot]));
  for (int i = 0; i < 4; ++i) out4[i] = L->loss_ring[slot][i];
  return D4PG_OK;
}

extern "C" int32_t d4pg_learner_step_host(d4pg_learner_t* L, const double* uniforms, const int32_t* positions,
                                          d4pg_stream_t caller_stream, d4pg_stream_t learner_stream) {
  D4PG_REQUIRE(L, D4PG_EINVAL, "d4pg_learner_step_host: null handle");
  return step_host_common(L, uniforms, nullptr, positions, caller_stream, learner_stream);
}

extern "C" int32_t d4pg_learner_step_host_mt(d4pg_learner_t* L, const uint32_t* mt_words,
                                             d4pg_stream_t caller_stream, d4pg_stream_t learner_stream) {
  D4PG_REQUIRE(L && mt_words, D4PG_EINVAL, "d4pg_learner_step_host_mt: null argument");
  return step_host_common(L, nullptr, mt_words, nullptr, caller_stream, learner_stream);
}

extern "C" int32_t d4pg_learner_read_losses(d4pg_learner_t* L, float* out4, d4pg_stream_t learner_stream) {
  D4PG_REQUIRE(L && out4, D4PG_EINVAL, "d4pg_learner_read_losses: null argument");
  cudaStream_t ls = as_stream(learner_stream);
  D4PG_CUDA_OK(cudaMemcpyAsync(L->host_losses, L->buf.losses, 4 * sizeof(float), cudaMemcpyDeviceToHost, ls));
  D4PG_CUDA_OK(cudaStreamSynchronize(ls));
  for (int i = 0; i < 4; ++i) out4[i] = L->host_losses[i];
  return D4PG_OK;
}

// Back-to-back steps with nothing in between: warm prefetch steps are replayed RUN_UNROLL at a time from one graph
// (a graph launch boundary leaves the GPU idle; inside a graph consecutive steps are ordinary dependent nodes).
constexpr int RUN_UNROLL = 8;
extern "C" int32_t d4pg_learner_run(d4pg_learner_t* L, int32_t n_steps, d4pg_stream_t stream) {
  D4PG_REQUIRE(L && n_steps > 0, D4PG_EINVAL, "d4pg_learner_run: bad arguments");
  cudaStream_t st = as_stream(stream);
  int n = n_steps;
  while (n > 0) {
    int par; bool cold;
    next_variant(L, &par, &cold);
    if (L->cfg.use_graph && prefetching(L->cfg) && !cold && n >= RUN_UNROLL && st != nullptr) {
      if (!L->multi_ready[par]) {
        const int rc = capture_graph(st, &L->multi_exec[par], "d4pg_learner_run", [&] {
          int rc = D4PG_OK;
          for (int i = 0; i < RUN_UNROLL && rc == D4PG_OK; ++i) rc = enqueue_step(L, st, par ^ (i & 1), false, i == 0);
          return rc;
        });
        if (rc) return rc;
        L->multi_ready[par] = true;
      }
      D4PG_CUDA_OK(cudaGraphLaunch(L->multi_exec[par], st));
      for (int i = 0; i < RUN_UNROLL; ++i) commit_variant(L, par ^ (i & 1));
      n -= RUN_UNROLL;
      continue;
    }
    int rc = d4pg_learner_step(L, stream);
    if (rc) return rc;
    --n;
  }
  return D4PG_OK;
}

extern "C" int32_t d4pg_learner_profile_step(d4pg_learner_t* L, d4pg_stream_t stream, int32_t max_launches,
                                             float* ms_out, char* names_out, int32_t name_stride, int32_t* n_out) {
  D4PG_REQUIRE(L && ms_out && n_out && max_launches > 0, D4PG_EINVAL, "d4pg_learner_profile_step: bad arguments");
  cudaStream_t st = as_stream(stream);
  int par; bool cold;
  next_variant(L, &par, &cold);
  if (int rc = wait_for_ingest(L, st)) return rc;
  L->profiling = true; L->ev.clear(); L->ev_name.clear(); L->ev_reps.clear();
  const int rc = step_eager(L, st, par, cold);
  L->profiling = false;
  cudaError_t e = cudaStreamSynchronize(st);
  const int n = int(L->ev_name.size());
  *n_out = n < max_launches ? n : max_launches;
  for (int i = 0; i < n; ++i) {
    float ms = 0.f;
    if (e == cudaSuccess) cudaEventElapsedTime(&ms, L->ev[2 * i], L->ev[2 * i + 1]);
    ms /= float(L->ev_reps[i]);
    if (i < max_launches) {
      ms_out[i] = ms;
      if (names_out && name_stride > 1) {
        strncpy(names_out + size_t(i) * name_stride, L->ev_name[i].c_str(), name_stride - 1);
        names_out[size_t(i) * name_stride + name_stride - 1] = 0;
      }
    }
    cudaEventDestroy(L->ev[2 * i]); cudaEventDestroy(L->ev[2 * i + 1]);
  }
  L->ev.clear(); L->ev_name.clear(); L->ev_reps.clear();
  if (e != cudaSuccess) { set_error("d4pg_learner_profile_step: %s", cudaGetErrorString(e)); return D4PG_ECUDA; }
  return rc;
}

extern "C" int32_t d4pg_learner_weights_changed(d4pg_learner_t* L) {
  D4PG_REQUIRE(L, D4PG_EINVAL, "d4pg_learner_weights_changed: null handle");
  L->images_dirty = true;
  return D4PG_OK;
}
extern "C" void* d4pg_learner_ingest_stream(const d4pg_learner_t* L) { return L ? static_cast<void*>(L->ing) : nullptr; }
extern "C" int64_t d4pg_learner_steps_done(const d4pg_learner_t* L) { return L ? L->steps_done : -1; }
extern "C" int32_t d4pg_learner_kernels_per_step(const d4pg_learner_t* L) { return L ? L->kernels_per_step : -1; }

extern "C" int32_t d4pg_learner_set_counters(d4pg_learner_t* L, int64_t adam_step, int64_t beta_t, d4pg_stream_t stream) {
  D4PG_REQUIRE(L && adam_step >= 0 && beta_t >= 0, D4PG_EINVAL, "d4pg_learner_set_counters: bad arguments");
  LearnerClock c{};
  c.adam_step = adam_step; c.beta_t = beta_t; c.steps_done = adam_step;
  c.s_adam_step = adam_step; c.s_beta_t = beta_t; c.s_steps_done = adam_step;
  L->prefetch_valid = false;                          // a prefetched batch was drawn with the old counters
  D4PG_CUDA_OK(cudaMemsetAsync(L->ws.pipe_epoch, 0, sizeof(unsigned long long) * size_t(cdiv(L->cfg.batch, SAMPLE_ROWS)), as_stream(stream)));
  D4PG_CUDA_OK(cudaMemcpyAsync(L->ws.clock, &c, sizeof(c), cudaMemcpyHostToDevice, as_stream(stream)));
  D4PG_CUDA_OK(cudaStreamSynchronize(as_stream(stream)));
  return D4PG_OK;
}

extern "C" int32_t d4pg_learner_tensor(d4pg_learner_t* L, const char* name, void** ptr, int64_t* count, int32_t* ld) {
  D4PG_REQUIRE(L && name && ptr && count && ld, D4PG_EINVAL, "d4pg_learner_tensor: null argument");
  const Workspace& w = L->ws; const Batch& bt = w.batch[L->last_par];     // the half the last step trained on
  const int64_t B = L->cfg.batch;
  const int Sp = pitch4(L->cfg.obs_dim), Ap = pitch4(L->cfg.act_dim), Np = pitch4(L->cfg.n_atoms);
  struct E { const char* n; void* p; int64_t c; int ld; };
  const E table[] = {
      {"s", bt.s, B * Sp, Sp}, {"a", bt.a, B * Ap, Ap}, {"r", bt.r, B, 1}, {"s2", bt.s2, B * Sp, Sp}, {"done", bt.done, B, 1},
      {"h", bt.hz, bt.hz ? B : 0, 1},
      {"target_logits", w.out[1], B * Np, Np}, {"q_logits", w.out[2], B * Np, Np}, {"pi_logits", w.out[4], B * Np, Np},
      {"m", w.m, B * Np, Np}, {"q_probs", w.q_probs, B * Np, Np}, {"target_probs", w.target_probs, B * Np, Np},
      {"dlogits_q", w.dlogits_q, B * Np, Np}, {"dlogits_pi", w.dlogits_pi, B * Np, Np},
      {"actor_out", w.out[3], B * Ap, Ap}, {"actor_target_out", w.out[0], B * Ap, Ap},
      {"loss_rows", w.loss_rows, B, 1}, {"pi_rows", w.pi_rows, B, 1},
      {"h1_c", w.h1[2], B * 256, 256}, {"h2_c", w.h2[2], B * 256, 256}, {"h3_c", w.h3[2], B * 256, 256},
      {"h1_a", w.h1[3], B * 256, 256}, {"h2_a", w.h2[3], B * 256, 256}, {"h3_a", w.h3[3], B * 256, 256},
      {"h2_p", w.h2[4], B * 256, 256}, {"h3_p", w.h3[4], B * 256, 256},
      {"h1_at", w.h1[0], B * 256, 256}, {"h2_at", w.h2[0], B * 256, 256}, {"h3_at", w.h3[0], B * 256, 256},
      {"h1_ct", w.h1[1], B * 256, 256}, {"h2_ct", w.h2[1], B * 256, 256}, {"h3_ct", w.h3[1], B * 256, 256},
      {"p_dz22", w.p_dz22, B * 256, 256}, {"p_dz2", w.p_dz2, B * 256, 256},
      {"c_dz22", w.c_dz22, B * 256, 256}, {"c_dz2", w.c_dz2, B * 256, 256}, {"c_dz1", w.c_dz1, B * 256, 256},
      {"a_dz3", w.a_dz3, B * Ap, Ap}, {"a_dz22", w.a_dz22, B * 256, 256}, {"a_dh2", w.a_dh2, B * 256, 256},
      {"a_dz1", w.a_dz1, B * 256, 256}};
  for (const E& e : table)
    if (e.p && strcmp(e.n, name) == 0) { *ptr = e.p; *count = e.c; *ld = e.ld; return D4PG_OK; }
  set_error("d4pg_learner_tensor: unknown tensor '%s'", name);
  return D4PG_EINVAL;
}
