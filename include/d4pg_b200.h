/*
 * d4pg_b200.h -- C ABI of libd4pg_sm90.so: the H100 (sm_90a) D4PG learner hot path.
 *
 * The reference (ajgupta93/d4pg-pytorch) is pure Python and has no FFI of its own; its
 * boundary for this path is the Python class API (SURVEY.md section 8b).  Each entry point
 * below replaces the *body* of one reference method; the Python classes in
 * `d4pg-pytorch_b200/` keep the reference signatures and bind these symbols with ctypes
 * (INTEGRATION.md shows the stub).  Citations are relative to the reference repository's root.
 *
 * Conventions
 *   - every function returns 0 on success or a negative D4PG_E* code; never throws.
 *     `d4pg_last_error()` returns a thread-local message for the last failure.
 *   - the CALLER owns all device memory (plain pointers + element counts); the library owns
 *     only opaque handles made by *_create and freed by *_destroy.
 *   - all work is asynchronous on the given `cudaStream_t` (passed as void*); no hidden
 *     synchronisation, no allocation after *_create.
 *   - a handle is not thread-safe; distinct handles are.
 *   - no torch types cross this boundary.
 */
#ifndef D4PG_B200_H_
#define D4PG_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define D4PG_OK            0
#define D4PG_EINVAL       -1   /* bad argument */
#define D4PG_ECUDA        -2   /* CUDA runtime error (see d4pg_last_error) */
#define D4PG_ENOTSUP      -3   /* unsupported configuration */
#define D4PG_ENCCL        -4   /* NCCL error / NCCL not loadable */
#define D4PG_ESTATE       -5   /* call out of order */

#define D4PG_HIDDEN      256   /* models.py:18-23,56-62 hard-code 256 hidden units */
#define D4PG_MAX_ATOMS   128
#define D4PG_MAX_COMPONENTS 32  /* mixture-of-Gaussians critic: at most 32 components (one warp lane each) */

typedef void* d4pg_stream_t;   /* cudaStream_t */

const char* d4pg_last_error(void);
int32_t     d4pg_version(void);            /* 10000*major + 100*minor + patch */
/* sizeof of the structs that cross this ABI by pointer (0 d4pg_learner_config_t, 1 d4pg_learner_buffers_t,
 * 2 d4pg_net_layout_t; -1 otherwise): lets a binding verify that its mirror of the struct is current */
int32_t     d4pg_struct_size(int32_t which);
/* compute capability of the current device as 10*major+minor (90 on H100), or <0 */
int32_t     d4pg_device_sm(void);

/* ---------------------------------------------------------------------------------------
 * Parameter layout.  One flat fp32 buffer per network role, tensors in nn.Module order
 * fc1.weight, fc1.bias, fc2.weight, fc2.bias, fc2_2.weight, fc2_2.bias, fc3.weight, fc3.bias
 * (models.py:18-23 actor, models.py:56-62 critic), nn.Linear row-major [out,in] with the row
 * PITCH rounded up to 4 floats (16-B aligned rows: every operand is TMA- and 128-bit addressable;
 * the pad columns are zero and stay zero), every tensor start aligned to 4 floats.
 * `offsets[8]` / `sizes[8]` (allocated floats, = out*pitch for weights) / `pitch[4]` are in floats.
 * ------------------------------------------------------------------------------------- */
typedef struct {
  int64_t offsets[8];
  int64_t sizes[8];
  int64_t pitch[4];
  int64_t total;      /* padded float count of the network */
} d4pg_net_layout_t;

int32_t d4pg_actor_layout(int32_t obs_dim, int32_t act_dim, d4pg_net_layout_t* out);
int32_t d4pg_critic_layout(int32_t obs_dim, int32_t act_dim, int32_t n_atoms, d4pg_net_layout_t* out);

/* ---------------------------------------------------------------------------------------
 * Fused projection + critic loss + TD proxy + priorities + logit gradients.
 * Replaces DDPG.reproject2 (ddpg.py:142-185, proj_mode 0) or DDPG.reproj_categorical_dist
 * (ddpg.py:122-140, proj_mode 1), the loss / td expressions ddpg.py:217,220-222,253 and the
 * policy-loss head ddpg.py:236-238.  One warp per batch row.
 *
 *   target_logits [B,N] f32  critic_target pre-softmax output for (s', actor_target(s'))
 *   q_logits      [B,N] f32  critic pre-softmax output for (s,a)
 *   pi_logits     [B,N] f32  critic pre-softmax output for (s, actor(s)); may be NULL
 *   rewards       [B]   f64, dones [B] u8
 *   discount            gamma (mode 0) or gamma**n_steps (mode 1)
 * outputs (any may be NULL):
 *   m [B,N] f32 projected target; bins_l/bins_u [B,N] i32 (the integer atom bins);
 *   target_probs, q_probs [B,N] f32; loss_rows [B] = -sum_j m log(q+1e-10);
 *   td [B] = -sum_j m q; prio [B] = |td| + prio_eps; dlogits_q [B,N] = d(mean loss)/d q_logits;
 *   pi_rows [B] = -sum_j softmax(pi)_j z_j; dlogits_pi [B,N] = d(mean pi loss)/d pi_logits.
 *   `grad_scale` multiplies both gradients (1/B for the reference's mean; 1/(B*world) under DP).
 *   `flags`: D4PG_PROJ_TARGET_IS_PROBS = target_logits already holds softmax outputs (the
 *   reference's reproject2(target_z_dist, ...) signature); D4PG_PROJ_Q_IS_PROBS likewise for q.
 * ------------------------------------------------------------------------------------- */
#define D4PG_PROJ_TARGET_IS_PROBS 1
#define D4PG_PROJ_Q_IS_PROBS      2
int32_t d4pg_proj_loss(const float* target_logits, const float* q_logits, const float* pi_logits,
                       const double* rewards, const uint8_t* dones,
                       int32_t B, int32_t N, double v_min, double v_max, double discount,
                       int32_t proj_mode, int32_t flags, double prio_eps, float grad_scale,
                       float* m, int32_t* bins_l, int32_t* bins_u,
                       float* target_probs, float* q_probs,
                       float* loss_rows, float* td, float* prio, float* dlogits_q,
                       float* pi_rows, float* dlogits_pi, d4pg_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Mixture-of-Gaussians critic head (critic_dist_info['type'] == 'mixture_of_gaussian', K = n_components in
 * [1, D4PG_MAX_COMPONENTS]).  The reference stubs this branch (ddpg.py:48-50, models.py:63-65); these semantics are
 * the library's own.  A raw head row o has 3K columns:
 *   w = softmax(o[0:K]),  mu = o[K:2K],  sigma = softplus(o[2K:3K]) + 1e-3   (softplus(x) = x for x > 20)
 * Target mixture of row i (from target_raw): weights w'_k, means r_i + c mu'_k, std devs c sigma'_k, with
 * c = discount * (1 - done_i) -- a terminal row is a Dirac at r_i.
 *   loss_rows [B]  L_i = -sum_{k,q} w'_k h_q / sqrt(pi) * log p(r_i + c (mu'_k + sqrt(2) sigma'_k x_q)), the
 *                  cross-entropy of the online mixture p (from q_raw) under the target mixture, integrated with the
 *                  8 Gauss-Hermite nodes (x_q, h_q) of d4pg_mog_quadrature (deterministic: no sampling)
 *   td [B]         sum_j w_j mu_j - (r_i + c sum_k w'_k mu'_k);  prio [B] = |td| + prio_eps
 *   dq_raw [B,3K]  d(mean loss)/d q_raw;  pi_rows [B] = -sum_j w_j mu_j of pi_raw;  dpi_raw [B,3K] its gradient
 * Both gradients are multiplied by `grad_scale`.  Raw planes are dense [B,3K]; every output may be NULL, and so may
 * pi_raw.  The row is evaluated in fp64, one warp per row.
 * d4pg_mog_quadrature writes the 8 nodes x[8] and weights h[8] (numpy.polynomial.hermite.hermgauss(8)); host only.
 * ------------------------------------------------------------------------------------- */
int32_t d4pg_mog_loss(const float* target_raw, const float* q_raw, const float* pi_raw,
                      const double* rewards, const uint8_t* dones, int32_t B, int32_t K,
                      double discount, double prio_eps, float grad_scale,
                      float* loss_rows, float* td, float* prio, float* dq_raw,
                      float* pi_rows, float* dpi_raw, d4pg_stream_t stream);
int32_t d4pg_mog_quadrature(double* x, double* h);

/* ---------------------------------------------------------------------------------------
 * Quantile-regression critic head (critic_dist_info['type'] == 'quantile', N = n_quantiles in [2, D4PG_MAX_ATOMS]):
 * the quantile-Huber loss of QR-DQN (Dabney et al. 2018).  The reference has no quantile code; these semantics are the
 * library's own.  A row theta [N] is the critic's raw fc3 output (no head transform); quantile k sits at the midpoint
 * tau_k = (2k+1) / (2N).  With c = discount * (1 - done_i), targets y_j = r_i + c theta'_j (theta' from target_q; a
 * terminal row's targets are all r_i), u_jk = y_j - theta_k,
 *   H(u) = u^2/2 if |u| <= kappa, else kappa (|u| - kappa/2);   rho_jk = |tau_k - 1{u_jk < 0}| H(u_jk) / kappa
 *   loss_rows [B]  L_i = (1/N) sum_j sum_k rho_jk   (>= 0; no gradient into the target)
 *   dq [B,N]       grad_scale * dL_i/dtheta_k = -grad_scale/N sum_j |tau_k - 1{u_jk < 0}| clamp(u_jk, -kappa, kappa) / kappa
 *   td [B]         mean_k theta_k - (r_i + c mean_j theta'_j);  prio [B] = |td| + prio_eps, or L_i + prio_eps when
 *                  ce_priority != 0
 *   pi_rows [B]    -mean_k theta_k of pi_q;  dpi [B,N] = -grad_scale / N
 * kappa must be finite and > 0.  Planes are dense [B,N]; every output may be NULL, and so may pi_q.  One warp per row,
 * the N^2 pair terms in fp64; no atomics (run-to-run identical).  In the learner (dist_type 2) the loss row is also
 * multiplied by the PER importance weight with loss_flags & 1, and so is dq.
 * The critic module of a quantile critic is d4pg_critic_forward with probs = NULL (logits = theta) and
 * d4pg_critic_backward with probs = grad_probs = NULL (grad_logits = d loss / d theta).
 * ------------------------------------------------------------------------------------- */
int32_t d4pg_qr_loss(const float* target_q, const float* q, const float* pi_q,
                     const double* rewards, const uint8_t* dones, int32_t B, int32_t N,
                     double discount, double kappa, double prio_eps, float grad_scale, int32_t ce_priority,
                     float* loss_rows, float* td, float* prio, float* dq,
                     float* pi_rows, float* dpi, d4pg_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Prioritized replay: GPU-resident sum/min segment trees + SoA transition storage.
 * Replaces SegmentTree / SumSegmentTree / MinSegmentTree (prioritized_replay_memory.py:33-162),
 * ReplayBuffer (:164-222) and PrioritizedReplayBuffer (:224-335).
 * Tree layout as the reference: root at 1, leaves at [cap, 2cap), fp32 nodes
 * (NumPy-2 semantics of the reference, SURVEY.md H11), cap = next pow2 >= size (:243-245).
 *
 * Caller-owned device buffers handed over at create time (sizes in elements):
 *   sum_tree, min_tree  f32 [2*cap]      obs, obs2 f32 [size*obs_dim]   act f32 [size*act_dim]
 *   rew f64 [size]                       done u8 [size]
 *   scratch i32 [cap]  (last-writer resolution for duplicate indices)
 *   state   f32 [8]    (device-resident scalars: max_priority, ...; opaque)
 * ------------------------------------------------------------------------------------- */
typedef struct d4pg_replay d4pg_replay_t;

int32_t d4pg_replay_capacity(int64_t size, int64_t* cap_out);          /* :243-245 */
int32_t d4pg_replay_create(int64_t size, int32_t obs_dim, int32_t act_dim, double alpha,
                           float* sum_tree, float* min_tree,
                           float* obs, float* act, double* rew, float* obs2, uint8_t* done,
                           int32_t* scratch, float* state,
                           d4pg_stream_t stream, d4pg_replay_t** out);
int32_t d4pg_replay_destroy(d4pg_replay_t* h);
int64_t d4pg_replay_len(const d4pg_replay_t* h);                        /* __len__, :177 */
int64_t d4pg_replay_next_idx(const d4pg_replay_t* h);

/* add() for n transitions already resident on the device (row-major [n,dim]); ring insert at
 * _next_idx, leaf = max_priority**alpha in both trees (:180-187,251-256).  `prioritized`=0
 * skips the trees (uniform Replay.add, replay_memory.py:14-19). */
int32_t d4pg_replay_add(d4pg_replay_t* h, int64_t n, const float* obs, const float* act,
                        const double* rew, const float* obs2, const uint8_t* done,
                        int32_t prioritized, d4pg_stream_t stream);

/* Host-side ingest: register a caller-owned PINNED host staging buffer and a device staging buffer
 * of `bytes` each (>= d4pg_replay_staging_bytes(rows)), then add() n <= rows transitions straight from
 * ordinary host arrays: the five arrays are packed into the pinned buffer, moved with ONE async H2D
 * copy and unpacked by the ring-write kernel.  Stream-ordered.  The buffers are used as TWO slots of bytes/2
 * (d4pg_replay_staging_bytes already counts both), alternating per call, so the host can stage add k+1 while
 * add k still waits on the device; a slot is re-used only after the add that read it has completed. */
int64_t d4pg_replay_staging_bytes(const d4pg_replay_t* h, int64_t rows);
int32_t d4pg_replay_set_staging(d4pg_replay_t* h, void* pinned_host, void* device, int64_t bytes);
int32_t d4pg_replay_add_host(d4pg_replay_t* h, int64_t n, const float* obs, const float* act, const double* rew,
                             const float* obs2, const uint8_t* done, int32_t prioritized, d4pg_stream_t stream);
/* Order stream `then` after everything enqueued so far on stream `first` (event record + wait; no-op if equal).  The
 * host mirror uses it to keep buffer operations issued on the caller's stream and on a learner's ingest stream
 * (d4pg_learner_ingest_stream) in program order. */
int32_t d4pg_replay_order_after(d4pg_replay_t* h, d4pg_stream_t first, d4pg_stream_t then);

/* Device-side ingest with n-step return accumulation at insert (replay_memory.py:38-45).  The arrays hold ONE episode
 * of T consecutive steps, resident on the device; transition i = (s_i, a_i, sum_{k<n} gamma^k r_{i+k}, s'_{i+n-1},
 * done_{i+n-1}) for i <= T-n is inserted (nothing when T < n, like the reference before step n-1).  The return is the
 * reference's left-to-right f64 loop, bit for bit.  `rew_scratch` f64 [T] is caller-owned device scratch.
 * d4pg_nstep_returns is the arithmetic alone: out[i], i <= T-n. */
int32_t d4pg_nstep_returns(const double* rew, int64_t T, int32_t n_steps, double gamma, double* out, d4pg_stream_t stream);
int32_t d4pg_replay_add_nstep(d4pg_replay_t* h, int64_t T, const float* obs, const float* act, const double* rew,
                              const float* obs2, const uint8_t* done, int32_t n_steps, double gamma,
                              double* rew_scratch, int32_t prioritized, d4pg_stream_t stream);

/* Streaming n-step insert: one vector step of E environments per call, the n-step windows kept on the device.
 *   obs, obs2 f32 [E, obs_dim]   act f32 [E, act_dim]   rew f64 [E]   terminated u8 [E]   episode_end u8 [E] or NULL
 * Environment e appends (obs_e, act_e, rew_e) to its window.  With f = the steps of e's current episode before this
 * call, e emits when f + 1 >= n: the row (s_{f-n+1}, a_{f-n+1}, R, obs2_e, terminated_e != 0), with
 *   R = sum_{k<n} gamma^k r_{f-n+1+k}, the left-to-right f64 loop of d4pg_nstep_returns, bit for bit.
 * Then the window is cleared when terminated_e != 0 or episode_end_e != 0 (pass truncated, or terminated | truncated;
 * NULL = terminated only).  Windows that never fill are dropped, like replay_memory.py:38 before step n-1.
 * The emitting environments take ring rows next_idx, next_idx + 1, ... in ascending e; the leaves, the normalizer's
 * fold and len / next_idx follow as for d4pg_replay_add of those rows in that order (n_steps = 1 stores what
 * d4pg_replay_add of the E rows stores, except that R = 0.0 + 1.0 * r turns a reward of -0.0 into +0.0).
 *   n_rows: the number of emitting environments, which the caller counts from the episode ends of earlier calls (a
 *           host mirror of the fills, no device read).  The kernel writes no ring row outside [next_idx, next_idx + n_rows).
 *   window: caller-owned device memory of d4pg_replay_steps_window_bytes(E, obs_dim, act_dim, n_steps) bytes (-1 on
 *           bad arguments), zero-filled before the first call.  It holds the per-environment state: a u64 record
 *           {call id, fill before, fill after} [E], rewards f64 [E, 2n] (each stored twice, so the last n are
 *           contiguous), states f32 [E, n, obs_dim] and actions f32 [E, n, act_dim].  Zero-filling it again discards
 *           the pending windows.  E, n_steps and gamma must stay the same between zero-fills.
 * One kernel per call, plus the d4pg_replay_add tail when n_rows > 0 (the normalizer's fold, split at the ring's
 * wrap; the tree add).  Stream-ordered, no allocation.  D4PG_EINVAL: null pointers, E outside (0, size], n_steps
 * outside [1, D4PG_STEPS_MAX_N], n_rows outside [0, E]. */
#define D4PG_STEPS_MAX_N 64
int64_t d4pg_replay_steps_window_bytes(int64_t E, int32_t obs_dim, int32_t act_dim, int32_t n_steps);
int32_t d4pg_replay_add_steps(d4pg_replay_t* h, int64_t E, const float* obs, const float* act, const double* rew,
                              const float* obs2, const uint8_t* terminated, const uint8_t* episode_end,
                              int32_t n_steps, double gamma, void* window, int64_t n_rows, int32_t prioritized,
                              d4pg_stream_t stream);

/* Episode tails of the streaming insert (DESIGN.md §3 "Episode tails").  d4pg_replay_set_horizons registers a
 * caller-owned device column horizon u8 [size] with the replay and zero-fills it on `stream` (NULL unregisters): every
 * row then carries its bootstrap horizon, 0 for a full-horizon row.  Every insert path clears the horizons of the slots
 * it writes (a cudaMemsetAsync on the stream of its ring write), except d4pg_replay_add_steps_ex with tails = 1.
 * d4pg_replay_add_steps_ex with tails = 0 is d4pg_replay_add_steps.  With tails = 1 (needs the column; D4PG_ESTATE
 * otherwise) an episode of L steps that ends at call k -- terminated or truncated -- also yields, at call k+1 and before
 * that call's own step, one tail row per start u in [max(0, L-n+1), L-1]: (s_u, a_u, the f64 n-step return over its
 * k = L-u remaining rewards, obs_next and terminated of step L-1) with horizon k; full rows get horizon 0.  Rows of one
 * call go in ascending environment, then ascending u.  n_rows counts tail rows too: at most E * max(1, n_steps-1) and
 * at most size.  The window of a tails call is d4pg_replay_steps_window_bytes_ex(E, obs_dim, act_dim, n_steps, 1)
 * bytes (it also keeps the ending step's obs_next); a window is used with one tails setting only. */
int32_t d4pg_replay_set_horizons(d4pg_replay_t* h, uint8_t* horizon, d4pg_stream_t stream);
int64_t d4pg_replay_steps_window_bytes_ex(int64_t E, int32_t obs_dim, int32_t act_dim, int32_t n_steps, int32_t tails);
int32_t d4pg_replay_add_steps_ex(d4pg_replay_t* h, int64_t E, const float* obs, const float* act, const double* rew,
                                 const float* obs2, const uint8_t* terminated, const uint8_t* episode_end,
                                 int32_t n_steps, double gamma, void* window, int64_t n_rows, int32_t tails,
                                 int32_t prioritized, d4pg_stream_t stream);

/* Hindsight-experience relabelling on the device (main.py:154-184, "future" strategy) as a gather kernel that produces
 * the rows d4pg_replay_add then inserts.  Episode of T goal-conditioned steps: obs / obs_next f32 [T, obs_dim], goal
 * f64 [T, goal_dim] (desired goal of every step), ag_next f64 [T, goal_dim] (achieved goal of the next state), act f32
 * [T, act_dim], rew f64 [T], done u8 [T].  select u8 [T] / future i32 [T] are the caller's draws
 * (np.random.uniform() < her_ratio; np.random.randint(t, T)), dst_row i32 [T] = exclusive prefix sum of (1 + select).
 * Output rows (state width obs_dim + goal_dim): the original transition of step t, then -- if selected -- its copy with
 * goal' = ag_next[future[t]], reward = -(||ag_next[t] - goal'||_2 > threshold) in f64 (the sparse gym-robotics
 * compute_reward) and done = (reward == 0).  her_action_mode 0 keeps the reference's behaviour of storing the rollout's
 * LAST action with the relabelled copy (main.py:184 uses `action`, not the step's `a`); 1 stores a_t. */
int32_t d4pg_her_relabel(int32_t T, int32_t obs_dim, int32_t goal_dim, int32_t act_dim,
                         const float* obs, const float* obs_next, const double* goal, const double* ag_next,
                         const float* act, const double* rew, const uint8_t* done,
                         const uint8_t* select, const int32_t* future, const int32_t* dst_row,
                         double threshold, int32_t her_action_mode,
                         float* out_s, float* out_a, double* out_r, float* out_s2, uint8_t* out_d,
                         d4pg_stream_t stream);

/* Streaming hindsight relabelling (DESIGN.md §3 "Streaming hindsight relabelling"): one vector step of E
 * goal-conditioned environments per call, each environment's current episode kept in a window on the device.
 *   obs, obs2 f32 [E, obs_dim]   goal, ag2 f64 [E, goal_dim]   act f32 [E, act_dim]   rew f64 [E]
 *   terminated u8 [E]   episode_end u8 [E] or NULL
 * ag2 is the achieved goal after the step.  The replay's obs_dim must be obs_dim + goal_dim; its act_dim is used.
 * Environment e appends (obs, goal, act, rew, obs2, ag2, terminated) as step t of its episode; the episode ends on
 * terminated_e != 0 or episode_end_e != 0.  An episode of L steps that ended at call k is emitted at call k+1 (or by a
 * call with no_step = 1), before that call's step is appended: for every t the original row
 * (obs_t || goal_t, act_t, rew_t, obs2_t || goal_t, terminated_t), directly followed, where the plan selects it, by the
 * copy with goal' = ag2_f (f = future[t], t <= f < L), reward -(||ag2_t - goal'||_2 > threshold) in f64 (the
 * arithmetic of d4pg_her_relabel) and done = (reward == 0); its action is act_{L-1} (her_action_mode 0, main.py:184)
 * or act_t (1).  Rows go in ascending e, then t, and take ring rows next_idx, next_idx + 1, ...; the leaves, the
 * normalizer's fold and len / next_idx follow as for d4pg_replay_add of those rows; their horizons are cleared.
 *   window: caller-owned device memory of d4pg_replay_goal_window_bytes(E, obs_dim, goal_dim, act_dim,
 *           max_episode_steps) bytes (-1 on bad arguments), zero-filled before the first call; zero-filling it again
 *           discards the pending episodes.  E, the dims and max_episode_steps stay the same between zero-fills, and
 *           no episode may grow past max_episode_steps steps (the caller counts them).
 *   plan:   the host's draws, i32, NULL when n_draws = 0: step_off [E] (first draw of e's emitted episode, draws in
 *           ascending e then t), future [n_draws] (-1 = no copy), dst [n_draws] (rank in this call of the original row
 *           of each step; a copy takes the next rank).  n_draws = the summed length of the emitted episodes.
 *   n_rows: n_draws + the selected steps; the kernel writes no ring row outside [next_idx, next_idx + n_rows).
 *   no_step: 1 = emit the ended episodes only (the step inputs may be NULL); running episodes keep their windows.
 * One kernel per call, plus the d4pg_replay_add tail when n_rows > 0.  Stream-ordered, no allocation.  A call with
 * n_rows = 0 leaves the replay's generation unchanged.  D4PG_EINVAL: null pointers, E outside (0, size], a dim
 * mismatch, max_episode_steps outside [1, D4PG_GOAL_MAX_STEPS], a threshold that is negative or not finite, n_draws
 * outside [0, E * max_episode_steps], n_rows outside [0, min(2 * n_draws, size)]. */
#define D4PG_GOAL_MAX_STEPS 65536
int64_t d4pg_replay_goal_window_bytes(int64_t E, int32_t obs_dim, int32_t goal_dim, int32_t act_dim, int32_t max_episode_steps);
int32_t d4pg_replay_add_goal_steps(d4pg_replay_t* h, int64_t E, int32_t obs_dim, int32_t goal_dim,
                                   const float* obs, const double* goal, const float* act, const double* rew,
                                   const float* obs2, const double* ag2, const uint8_t* terminated,
                                   const uint8_t* episode_end, int32_t max_episode_steps, void* window,
                                   const int32_t* plan, int64_t n_draws, int64_t n_rows, double threshold,
                                   int32_t her_action_mode, int32_t no_step, int32_t prioritized, d4pg_stream_t stream);

/* Running per-feature observation normalizer (mean / variance over every stored row, with clipping).
 *   stats  f64 [1 + 2*obs_dim] = {n, mean[S], M2[S]}      affine f32 [2*obs_dim] = {shift[S], scale[S]}
 * Update: every row an insert stores contributes its s once, in insertion order (rows later overwritten by the ring
 * still count), folded in with Welford's step, every fp64 operation rounded and not contracted:
 *   n = n + 1;  d = x - mean;  mean = mean + d / n;  M2 = M2 + d * (x - mean)
 * Affine, recomputed at the end of every update: n == 0 -> shift 0, scale 1; otherwise shift = f32(mean),
 *   scale = f32(1 / sqrt(M2 / n + eps)) (fp64, correctly rounded, one cast at the end).
 * Apply (fp32): y = min(max((x - shift) * scale, -clip), clip).  clip and eps: finite and > 0 (5.0 and 1e-8 are usual).
 *
 * d4pg_replay_set_obs_norm registers caller-owned device buffers with the replay and resets them to n = 0 on `stream`;
 * from then on every insert (add, add_host, add_nstep, add_steps) updates them on its own stream, right after its ring write.
 * stats == NULL detaches.  The stored rows and every sample / gather of this section stay raw; only a learner created
 * with obs_norm = 1 reads the affine.  d4pg_replay_obs_norm_refresh recomputes the affine from the stats after the
 * caller wrote them (a state load).  Both bump the replay's generation, so a learner's prefetched batch is re-sampled.
 * d4pg_obs_norm_update is the same fold + affine on caller rows [n, ld] (n == 0: the affine alone), without a replay;
 * d4pg_obs_normalize applies the affine to x [n, obs_dim] into y and, when dydx is given, writes dy/dx: scale where the
 * pre-clip value lies in [-clip, clip], else 0. */
int32_t d4pg_replay_set_obs_norm(d4pg_replay_t* h, double* stats, float* affine, double clip, double eps, d4pg_stream_t stream);
int32_t d4pg_replay_obs_norm_refresh(d4pg_replay_t* h, d4pg_stream_t stream);
int32_t d4pg_obs_norm_update(double* stats, float* affine, int32_t obs_dim, const float* rows, int64_t n, int64_t ld,
                             double eps, d4pg_stream_t stream);
int32_t d4pg_obs_normalize(const float* affine, int32_t obs_dim, double clip, const float* x, int64_t n,
                           float* y, float* dydx, d4pg_stream_t stream);

/* _sample_proportional + IS weights + _encode_sample (:258-313,189-199).
 *   uniforms [B] f64 in [0,1): the reference's random.random() draws; NULL = device Philox
 *   (seed, counter) stream.  mass = u * sum(0,len-1) with the reference's association and
 *   dtype rules (f64 while the tree is pristine, f32 afterwards).
 *   outputs: idx [B] i32, weights [B] f32 (may be NULL), gathered batch s,a,r,s2,done. */
int32_t d4pg_replay_sample(d4pg_replay_t* h, int32_t B, const double* uniforms,
                           uint64_t philox_seed, uint64_t philox_counter, double beta,
                           int32_t* idx, float* weights,
                           float* s, float* a, double* r, float* s2, uint8_t* done,
                           d4pg_stream_t stream);
/* uniform Replay.sample gather for caller-chosen positions (replay_memory.py:61-80) */
int32_t d4pg_replay_gather(d4pg_replay_t* h, int32_t B, const int32_t* idx,
                           float* s, float* a, double* r, float* s2, uint8_t* done,
                           d4pg_stream_t stream);
/* update_priorities (:315-335): leaf = prio**alpha (fp32 pow semantics), duplicates: last
 * writer wins, max_priority = max(max_priority, prio). */
int32_t d4pg_replay_update_priorities(d4pg_replay_t* h, int32_t B, const int32_t* idx,
                                      const float* prio, d4pg_stream_t stream);
/* SumSegmentTree.sum(start,end) / MinSegmentTree.min(start,end) over leaves [start,end) into
 * out[0], out[1] (device f32[2]) with SegmentTree.reduce's association; end<=0 counts from the
 * capacity as the reference's None/negative `end` does (:61-96,122-124,158-162). */
int32_t d4pg_replay_reduce(d4pg_replay_t* h, int64_t start, int64_t end, float* out, d4pg_stream_t stream);
/* SumSegmentTree.find_prefixsum_idx for n caller-supplied masses (:126-149) */
int32_t d4pg_replay_find_prefixsum(d4pg_replay_t* h, int32_t n, const double* masses, int32_t* idx,
                                   d4pg_stream_t stream);
/* raw leaf write + parent recompute for n (idx, value) pairs: SegmentTree.__setitem__ (:98-108) */
int32_t d4pg_replay_set_leaves(d4pg_replay_t* h, int32_t n, const int32_t* idx, const float* sum_vals,
                               const float* min_vals, d4pg_stream_t stream);
/* host-visible bookkeeping the drop-in needs after a host-side restore (stream-ordered like every other mutator) */
int32_t d4pg_replay_set_len(d4pg_replay_t* h, int64_t len, int64_t next_idx, int32_t pristine, d4pg_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Actor / critic forward (inference entry points).  Replace actor.forward (models.py:32-41)
 * and critic.forward (models.py:76-88).  `params` = flat buffer in d4pg_*_layout order.
 * `workspace` f32 [3*B*256] scratch.  precision: 0 fp32 (FFMA), 1 3xTF32 wgmma (fp32-accurate), 2 one TF32 wgmma pass
 * (operands truncated to TF32, round toward zero), 3 one bf16 wgmma pass (each GEMM operand rounded to bf16, round to nearest even; fp32 accumulate, fp32 bias and
 * activation; inputs, weights and outputs stay fp32).  Any other value fails with D4PG_ENOTSUP.
 * ------------------------------------------------------------------------------------- */
int32_t d4pg_actor_forward(const float* params, int32_t obs_dim, int32_t act_dim,
                           const float* s, int32_t B, float* action, float* workspace,
                           int32_t precision, d4pg_stream_t stream);
int32_t d4pg_critic_forward(const float* params, int32_t obs_dim, int32_t act_dim, int32_t n_atoms,
                            const float* s, const float* a, int32_t B, float* probs, float* logits,
                            float* workspace, int32_t precision, d4pg_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Exploratory action selection (main.py:145-146,216-217,279: np.clip(actor(s) + noise.sample(), -1, 1)) in ONE launch:
 * the actor at precision 0 as a 4-slot cluster chain, with the observation normalizer applied to the rows it reads,
 * and the noise and the clip in fc3's epilogue.
 *   s [E, obs_dim] f32 device rows with pitch lds (a multiple of 4 floats, 16-B aligned base; d4pg_copy_rows_f32
 *     lands other layouts); 1 <= E and 2 * E * act_dim < 2^31;  action [E, act_dim] f32 device
 *   norm_affine  {shift[obs_dim], scale[obs_dim]} of an observation normalizer (NULL = raw rows); then every s is
 *     min(max((s - shift) * scale, -norm_clip), norm_clip) in fp32, as d4pg_obs_normalize computes it
 *   noise  0: none -- action = actor(s), bit-identical to d4pg_actor_forward at precision 0
 *          1: Gaussian, noise_params {eps, mu, var}:               n = eps * (mu + var * z)
 *          2: Ornstein-Uhlenbeck, noise_params {eps, theta, mu, sigma, dt}; ou_state f64 [E, act_dim] device, updated in
 *             place; rows with reset[row] != 0 (u8 [E] device, NULL = none) restart from 0 first:
 *             x = (x + (theta * (mu - x)) * dt) + (sigma * sqrt(dt)) * z,  n = eps * x
 *          with noise: action = f32(min(max(f64(actor(s)) + n, -1), 1)).  noise_params is host memory, read during the call.
 *   z of element i = row * act_dim + j: u1 = Philox4x32-10 uniform53(seed, counter, 2i), u2 = (.., 2i + 1) (the device
 *     sampler's construction), z = sqrt(-2 log(1 - u1)) * cos(2 pi u2); every fp64 operation rounded, none contracted.
 *   workspace  d4pg_act_workspace_floats(E, obs_dim) floats of device scratch (-1: bad arguments)
 * D4PG_ENOTSUP when the actor's fc1 does not fit one chain slot (obs_dim > 576).
 * d4pg_copy_rows_f32: rows x width floats from src (pitch lds) to dst (pitch ldd), host or device, one 2-D copy on
 * `stream` (no kernel).
 * ------------------------------------------------------------------------------------- */
int64_t d4pg_act_workspace_floats(int32_t E, int32_t obs_dim);
int32_t d4pg_act(const float* actor_params, int32_t obs_dim, int32_t act_dim, const float* s, int64_t lds, int32_t E,
                 const float* norm_affine, double norm_clip, int32_t noise, const double* noise_params, uint64_t seed,
                 uint64_t counter, double* ou_state, const uint8_t* reset, float* action, float* workspace,
                 d4pg_stream_t stream);
int32_t d4pg_copy_rows_f32(float* dst, int64_t ldd, const float* src, int64_t lds, int64_t rows, int64_t width,
                           d4pg_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Adaptive parameter-space exploration noise (Plappert et al. 2018, "Parameter Space Noise for Exploration"; the
 * baselines DDPG's AdaptiveParamNoiseSpec).  The reference has none; these semantics are the library's own.
 *   noise_state  f64 [2] device {sigma, last distance}; sigma is read on the device, so both calls can be captured
 *
 * d4pg_actor_perturb: out = the actor `params` (d4pg_actor_layout(obs_dim, act_dim) order) with Gaussian noise of std
 *   dev sigma added to every parameter, in one launch.  Logical element i is the i-th float of the unpadded
 *   concatenation fc1.weight, fc1.bias, ..., fc3.bias (nn.Module parameter order, row-major weights):
 *     u1 = Philox4x32-10 uniform53(seed, counter, 2i), u2 = (.., 2i + 1), z = sqrt(-2 log(1 - u1)) * cos(2 pi u2),
 *     out_i = f32(f64(p_i) + sigma * z), every fp64 operation rounded, none contracted (d4pg_act's construction).
 *   Every padding float of out (row pitch columns, tensor alignment gaps) is written as 0.  params and out: 16-B
 *   aligned, both d4pg_actor_layout().total floats; count = the logical parameter count, 2 * count < 2^32.
 * d4pg_param_noise_adapt: the policy distance of two action planes a, a_perturbed [n] f32 (n >= 1, usually the actor's
 *   and the perturbed actor's d4pg_act outputs on the same states):
 *     d = sqrt(sum_i (f64(a_perturbed_i) - f64(a_i))^2 / n) in fp64 (one CTA, fixed summation order, no atomics),
 *     sigma = d > desired_stddev ? sigma / coefficient : sigma * coefficient;  noise_state = {sigma, d}.
 *   desired_stddev finite and > 0, coefficient finite and > 1.
 * Bad arguments fail with D4PG_EINVAL before any device work.
 * ------------------------------------------------------------------------------------- */
int32_t d4pg_actor_perturb(const float* params, int32_t obs_dim, int32_t act_dim, const double* noise_state,
                           uint64_t seed, uint64_t counter, float* out, d4pg_stream_t stream);
int32_t d4pg_param_noise_adapt(const float* a, const float* a_perturbed, int64_t n, double desired_stddev,
                               double coefficient, double* noise_state, d4pg_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Actor / critic backward: the autograd backward of the two forward calls above, for callers that own
 * the loss (ddpg.py:229-244 written against the modules, other losses, gradient checks).  Runs the same
 * per-layer GEMM kernels as the learner's one-launch-per-level plan at the same `precision` (3 rounds dZ and W
 * for dX, dZ and X for dW to bf16), one launch per layer after a small kernel for the output head.
 *   params, s (, a), B, precision  exactly as given to the forward call;
 *   action / probs      the forward's output (tanh output [B,act_dim]; softmax probabilities [B,n_atoms]);
 *   workspace           h1..h3 exactly as the matching forward call left them.  d4pg_critic_forward reuses h1
 *                       as logits scratch when `logits` is NULL: a critic forward meant for this backward must
 *                       be given a logits buffer;
 *   grad_action         d loss / d action [B,act_dim];
 *   grad_probs, grad_logits  d loss / d probs and d loss / d logits [B,n_atoms]; either may be NULL (counts as
 *                       zero), not both; grad_probs needs probs;
 * outputs (each may be NULL, which skips its launches):
 *   grad_params         flat buffer in d4pg_*_layout order, overwritten (the call clears it first: the dW of a
 *                       batch of 1024 rows or more runs split-K with fp32 atomics); pad columns stay zero;
 *   grad_s [B,obs_dim], grad_a [B,act_dim]  d loss / d input, overwritten;
 *   scratch             f32 [B*(512 + max(256, pitch4(out)))], out = act_dim (actor) or n_atoms (critic), pitch4(x) =
 *                       x rounded up to a multiple of 4: two [B,256] delta planes, then the output head's dZ plane
 *                       [B, pitch4(out)].  For n_atoms <= 128 and act_dim <= 256 that is f32 [3*B*256].
 * Bad arguments fail with D4PG_EINVAL, an unknown precision with D4PG_ENOTSUP.
 * ------------------------------------------------------------------------------------- */
int32_t d4pg_actor_backward(const float* params, int32_t obs_dim, int32_t act_dim, const float* s, int32_t B,
                            const float* action, const float* workspace, const float* grad_action,
                            float* grad_params, float* grad_s, float* scratch, int32_t precision, d4pg_stream_t stream);
int32_t d4pg_critic_backward(const float* params, int32_t obs_dim, int32_t act_dim, int32_t n_atoms,
                             const float* s, const float* a, int32_t B, const float* probs, const float* workspace,
                             const float* grad_probs, const float* grad_logits,
                             float* grad_params, float* grad_s, float* grad_a, float* scratch,
                             int32_t precision, d4pg_stream_t stream);

/* Mixture-of-Gaussians critic (K components, see d4pg_mog_loss): the critic MLP with a 3K-wide fc3 (parameters in
 * d4pg_critic_layout(obs_dim, act_dim, 3K) order), then the head transform.
 *   d4pg_critic_forward_mog   w, mu, sigma [B,K] f32 (required); raw [B,3K] the fc3 output (may be NULL: then h1 of the
 *                             workspace is used as scratch, so a forward meant for the backward below must be given raw)
 *   d4pg_critic_backward_mog  raw = the forward's raw output; grad_w, grad_mu, grad_sigma [B,K] (each may be NULL,
 *                             counting as zero, not all three); everything else as d4pg_critic_backward with
 *                             n_atoms = 3K (scratch f32 [B*(512 + 256)] since 3K <= 96). */
int32_t d4pg_critic_forward_mog(const float* params, int32_t obs_dim, int32_t act_dim, int32_t K,
                                const float* s, const float* a, int32_t B, float* w, float* mu, float* sigma,
                                float* raw, float* workspace, int32_t precision, d4pg_stream_t stream);
int32_t d4pg_critic_backward_mog(const float* params, int32_t obs_dim, int32_t act_dim, int32_t K,
                                 const float* s, const float* a, int32_t B, const float* raw, const float* workspace,
                                 const float* grad_w, const float* grad_mu, const float* grad_sigma,
                                 float* grad_params, float* grad_s, float* grad_a, float* scratch,
                                 int32_t precision, d4pg_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Fused Adam + Polyak.  Replaces SharedAdam / torch.optim.Adam.step (shared_adam.py:3-17,
 * called at ddpg.py:232,244; torch-2.11 single-tensor formula), sync_local_global
 * (ddpg.py:118-120, identity on shared storage) and update_target_parameters (ddpg.py:110-116).
 *   p <- p - (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps);  target <- (1-tau)*target + tau*p
 * `step` is the post-increment step count.  `grad_scale` multiplies g first (DP averaging).
 * ------------------------------------------------------------------------------------- */
int32_t d4pg_adam_polyak(float* p, const float* g, float* m, float* v, float* target, int64_t n,
                         double lr, double beta1, double beta2, double eps, int64_t step,
                         double tau, float grad_scale, d4pg_stream_t stream);
/* The same update on the effective gradient coef * (grad_scale * g) + weight_decay * p (p = the pre-update value):
 *   weight_decay   finite, >= 0; 0 = none
 *   max_grad_norm  0 = no clipping; otherwise coef = min(1, max_grad_norm / (norm + 1e-6)) with norm = |grad_scale| *
 *                  sqrt(sum g^2) in fp64 (+inf: coef = 1, the norm is only reported).  Runs grad_sqnorm_kernel, then the
 *                  update, on `stream`
 *   partials       device workspace of 64 doubles; may be NULL when max_grad_norm == 0
 *   norm_out       optional device float: float32 of norm (written only when max_grad_norm != 0) */
int32_t d4pg_adam_polyak_ex(float* p, const float* g, float* m, float* v, float* target, int64_t n,
                            double lr, double beta1, double beta2, double eps, int64_t step,
                            double tau, float grad_scale, d4pg_stream_t stream,
                            double weight_decay, double max_grad_norm, double* partials, float* norm_out);
/* update_target_parameters alone (ddpg.py:110-116): target <- (1-tau)*target + tau*src */
int32_t d4pg_polyak(float* target, const float* src, int64_t n, double tau, d4pg_stream_t stream);
/* hard_update (ddpg.py:92-94) / load_state_dict copies */
int32_t d4pg_copy_f32(float* dst, const float* src, int64_t n, d4pg_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * The learner: one DDPG.train() body (ddpg.py:200-255) per d4pg_learner_step call,
 * captured once into a CUDA graph and replayed.
 * ------------------------------------------------------------------------------------- */
typedef struct {
  int32_t obs_dim, act_dim, n_atoms, batch;
  double  v_min, v_max, gamma;
  int32_t n_steps;
  int32_t proj_mode;          /* 0 = reproject2 (live, discount gamma), 1 = n-step (gamma**n) */
  double  tau;
  double  lr_actor, lr_critic, beta1, beta2, adam_eps;
  int32_t prioritized;        /* 1 = PrioritizedReplayBuffer path, 0 = uniform Replay path */
  double  per_beta0, per_beta_final; int64_t per_beta_iters;   /* LinearSchedule, ddpg.py:81-86 */
  double  prio_eps;           /* ddpg.py:87 */
  int32_t precision;          /* 0 exact fp32 FFMA, 1 3xTF32 wgmma (hi/lo split, fp32-accurate: meets the 1e-5 parity bar),
                                 2 one TF32 pass (not parity-grade) whose rounding follows the step plan: the wgmma
                                 chains and plan 0 truncate each operand to TF32 (round toward zero), the mma.sync
                                 chain tiles (|s| or |a| > 32, or > 256 atoms) round to nearest, ties away from zero;
                                 dW is exact fp32 FFMA on both chain plans and TF32 (truncated) on plan 0,
                                 3 one bf16 wgmma pass: the operands of every
                                 MLP GEMM (X and W forward, dZ and W for dX, dZ and X for dW) are rounded to bf16 (nearest
                                 even) as they are staged, products accumulate in fp32; activations, deltas, bias terms,
                                 bias gradients, the loss heads, Adam and the weights stay fp32 (not parity-grade) */
  int32_t sample_mode;        /* 0 = caller uniforms/positions (parity), 1 = device Philox */
  uint64_t philox_seed;
  int32_t world_size;         /* >1: gradients are averaged over ranks before Adam */
  int32_t use_graph;          /* 1 = capture the step into a CUDA graph */
  int32_t loss_flags;         /* corrected-semantics switches, 0 = reference behaviour:
                                 1 = importance-weighted critic CE (the reference samples the weights but
                                     ignores them, ddpg.py:217), 2 = priority = CE_i + eps instead of
                                     |sum_j m_ij q_ij| + eps (ddpg.py:221-222,253), 4 = the actor gradient flows
                                     through the critic AFTER this step's critic update (the reference uses the stale
                                     pre-update local copy, ddpg.py:229-247); needs the tensor-core chain plan, one GPU */
  int32_t chain;              /* step plan of the MLP passes (batches above 512 rows always use plan 0): 0 = one grouped launch per dependency
                                 level (18 kernels/step); 1 = cluster-fused layer chains: forward passes, dX passes
                                 and all dW are ONE launch each (7 kernels/step; precision 0: FFMA tiles, bit-identical
                                 to plan 0; precision 1/2: wgmma tiles, 64-row clusters, pre-packed hi/lo weight images).
                                 Precision 3 always runs plan 0 */
  int32_t prefetch;           /* 1 (sample_mode 1 only): step t samples batch t+1 on a side branch, right after its own
                                 priorities are in the trees, while its backward pass and Adam still run.  Same
                                 Philox counters and the same trees as sampling at the start of step t+1, so results
                                 are identical; any replay mutation by the caller (add / set / update) between two
                                 steps discards the prefetched batch and step t+1 samples again at its start.
                                 With sample_mode 0 (host-drawn uniforms / positions) and use_graph: the HOST pipeline --
                                 d4pg_learner_step_host* samples batch k on the library's ingest stream
                                 (d4pg_learner_ingest_stream), behind the add()s the caller issued on that stream and
                                 gated on step k-1's priority write-back, while step k-1's backward pass, dW and Adam
                                 still run.  Tree operations keep the reference's order update(k-1) -> add(k) ->
                                 sample(k) (ddpg.py:200-255 + main.py's add loop): results are identical */
  int32_t dist_type;          /* critic head: 0 = categorical (n_atoms, v_min, v_max), 1 = mixture of Gaussians with
                                 n_components = K in [1, 32] (d4pg_mog_loss): n_atoms / v_min / v_max are ignored and the
                                 critic's fc3 and every raw-head plane are 3K wide.  loss_flags & 2 is not supported with
                                 the mixture (the cross-entropy of a density can be negative).  2 = quantile regression
                                 (d4pg_qr_loss): n_atoms carries the number of quantiles N in [2, D4PG_MAX_ATOMS], v_min /
                                 v_max are ignored, qr_kappa is the Huber threshold; loss_flags & 2 gives
                                 priority = L_i + eps (the quantile-Huber loss is non-negative) */
  int32_t n_components;
  double  qr_kappa;           /* dist_type 2: Huber threshold kappa, finite and > 0 (1.0 is the usual choice) */
  /* Optimiser options, per network; all zero = the plain update.  On the step's complete gradient g (the flat buffer,
   * which keeps the UNCLIPPED gradient) and the pre-update parameters p:
   *   norm = sqrt(sum g_i^2) (fp64, fixed order);  coef = float(min(1, max_grad_norm / (norm + 1e-6)))
   *   g_eff = coef * g + weight_decay * p, then Adam on g_eff  (torch clip_grad_norm_ + torch.optim.Adam(weight_decay=))
   * max_grad_norm: 0 = off, +inf = measure and report only (coef is exactly 1), otherwise > 0.  A threshold on either
   * network adds one grad_sqnorm_kernel launch before each Adam launch; the norms land in losses[2], losses[3].
   * Not supported with world_size > 1 (the ranks' gradients are summed inside the Adam kernel).
   * weight_decay: 0 = off, otherwise finite and > 0 (L2 decay added to the gradient, not AdamW); any world size. */
  double  max_grad_norm_actor, max_grad_norm_critic;
  double  weight_decay_actor, weight_decay_critic;
  int32_t obs_norm;           /* 1: s and s2 of every batch go through the replay's observation normalizer as they are
                                 gathered (d4pg_replay_set_obs_norm, which must be registered before d4pg_learner_create
                                 and stay registered, with the same buffers and clip, for the learner's lifetime).
                                 0 = off.  Not supported with world_size > 1 (D4PG_EINVAL): each rank would normalize with
                                 the statistics of its own shard */
  int32_t nstep_tails;        /* 1: batches carry per-row horizons (d4pg_replay_set_horizons, registered before
                                 d4pg_learner_create and kept for the learner's lifetime): a row of horizon k > 0 that is
                                 not done bootstraps with gamma^k, computed on the host with pow(gamma, k) like the
                                 gamma^n_steps of full rows; every critic type.  D4PG_EINVAL with proj_mode 0 and
                                 n_steps > 1 (its gamma-for-every-row rule has no horizon) or without a horizon column.
                                 0 = off */
} d4pg_learner_config_t;

/* Caller-owned device buffers.  P_a / P_c = d4pg_*_layout().total. */
typedef struct {
  float* actor;  float* actor_target;  float* critic;  float* critic_target;
  float* grad_actor;  float* grad_critic;          /* contiguous: grad_critic == grad_actor + P_a */
  float* adam_m_actor; float* adam_v_actor; float* adam_m_critic; float* adam_v_critic;
  double*   uniforms;      /* [B] f64 (sample_mode 0, prioritized) */
  int32_t*  positions;     /* [B] i32 (sample_mode 0, uniform replay) */
  int32_t*  idx;           /* [B] i32 out: sampled indices */
  float*    weights;       /* [B] f32 out: IS weights (unused by the loss, SURVEY.md H3) */
  float*    prio;          /* [B] f32 out: new priorities */
  float*    td;            /* [B] f32 out */
  float*    losses;        /* [4]  f32 out: critic loss, actor loss, then the gradient norm (before clipping) of the actor
                              and of the critic -- each written only when that network has a max_grad_norm, else untouched */
  float*    workspace;     /* f32 [d4pg_learner_workspace_floats()] */
} d4pg_learner_buffers_t;

typedef struct d4pg_learner d4pg_learner_t;
typedef struct d4pg_comm    d4pg_comm_t;

int64_t d4pg_learner_workspace_floats(const d4pg_learner_config_t* cfg);
int32_t d4pg_learner_create(const d4pg_learner_config_t* cfg, const d4pg_learner_buffers_t* buf,
                            d4pg_replay_t* replay, d4pg_comm_t* comm, d4pg_learner_t** out);
int32_t d4pg_learner_destroy(d4pg_learner_t* h);
/* One gradient step.  Everything is stream-ordered; results land in buf->losses etc. */
int32_t d4pg_learner_step(d4pg_learner_t* h, d4pg_stream_t stream);
/* Host-facing step: everything `DDPG.train()` needs per call in ONE library call.
 *   d4pg_learner_step_host: order the learner stream after `caller_stream`, copy this step's host inputs
 *     (uniforms f64[B] for prioritized replay / positions i32[B] for uniform replay; NULL with device-side sampling)
 *     to the device, run the step on `learner_stream`, order `caller_stream` after it.  The inputs may live in
 *     ordinary host memory and may be reused as soon as the call returns: they are staged in library-owned pinned
 *     buffers (allocated by d4pg_learner_create, double-buffered by step parity, a buffer is rewritten only after the
 *     H2D copy out of it has completed).
 *   d4pg_learner_step_host_mt: the same for prioritized replay, taking the 2*B raw 32-bit MT19937 outputs of
 *     `random.randbytes(8*B)` instead of B doubles: uniform i = ((w[2i] >> 5) * 2^26 + (w[2i+1] >> 6)) / 2^53, which is
 *     CPython's random.random() -- the draws of prioritized_replay_memory.py:262, same generator state afterwards.
 *   d4pg_learner_read_losses: D2H of {critic loss, actor loss, -, -} and wait for it (the step's result). */
int32_t d4pg_learner_step_host(d4pg_learner_t* h, const double* uniforms, const int32_t* positions,
                               d4pg_stream_t caller_stream, d4pg_stream_t learner_stream);
int32_t d4pg_learner_step_host_mt(d4pg_learner_t* h, const uint32_t* mt_words,
                                  d4pg_stream_t caller_stream, d4pg_stream_t learner_stream);
int32_t d4pg_learner_read_losses(d4pg_learner_t* h, float* out4, d4pg_stream_t learner_stream);
/* Every d4pg_learner_step_host* call also queues an async D2H copy of its {critic loss, actor loss, -, -} into a pinned
 * two-slot ring.  d4pg_learner_fetch_losses waits for and returns the result of the most recent host-facing step (lag 0)
 * or of the one before it (lag 1: usually complete already, so a caller can read step k-1 while step k runs). */
int32_t d4pg_learner_fetch_losses(d4pg_learner_t* h, int32_t lag, float* out4);
/* n_steps back-to-back gradient steps without returning to the caller in between (device-side
 * sampling keeps advancing; caller-supplied uniforms/positions would be reused). */
int32_t d4pg_learner_run(d4pg_learner_t* h, int32_t n_steps, d4pg_stream_t stream);
/* Named intermediate (for parity tests): returns device pointer + element count.
 * names: "s","a","r","s2","done","target_logits","q_logits","pi_logits","m","q_probs",
 *        "target_probs","dlogits_q","dlogits_pi","actor_out","loss_rows","pi_rows"
 * 2-D tensors are stored with a row pitch of `*ld` floats (>= the logical width). */
int32_t d4pg_learner_tensor(d4pg_learner_t* h, const char* name, void** ptr, int64_t* count, int32_t* ld);
/* One EAGER (non-graph) step with a CUDA-event pair around every launch; synchronises.
 * ms_out[i] = device time of launch i, names_out[i*name_stride] = its launcher name. */
int32_t d4pg_learner_profile_step(d4pg_learner_t* h, d4pg_stream_t stream, int32_t max_launches,
                                  float* ms_out, char* names_out, int32_t name_stride, int32_t* n_out);
int64_t d4pg_learner_steps_done(const d4pg_learner_t* h);
/* host pipeline (cfg.prefetch with sample_mode 0): the stream buffer adds should be issued on so they overlap the
 * running step (NULL when the pipeline is off).  Owned by the learner.  With the pipeline on, d4pg_learner_step_host*
 * samples on this stream and does NOT wait for caller_stream first (that stream is ordered after the whole previous
 * step, which would serialise the pipeline): a caller that WROTE the buffer on another stream since the last step (add,
 * add_steps, add_goal_steps, add_nstep, update_priorities, set_leaves, a normalizer refresh ...) calls
 * d4pg_replay_order_after(replay, that_stream, ingest_stream) before the next step; without it the step may sample
 * rows, trees or normalizer statistics from before that write, and on the wgmma plans, whose forward chains poll the
 * sample's epochs, a sample drawn before the previous step advanced the step clock leaves the step waiting forever.
 * Reads on another stream need no edge before a step. */
void* d4pg_learner_ingest_stream(const d4pg_learner_t* h);
/* The tensor-core plans consume pre-split hi/lo weight IMAGES that the library's Adam / Polyak kernel keeps current.  Every
 * CUDA-graph step that samples in the graph re-packs them from the fp32 parameters first (any external write is picked
 * up); the host pipeline's steps (above) re-pack only after this call -- make it whenever actor / critic / target
 * parameters were written from outside the library (state_dict load, hard update, manual edits) since the last step.
 * A new learner starts "changed". */
int32_t d4pg_learner_weights_changed(d4pg_learner_t* h);
int32_t d4pg_learner_kernels_per_step(const d4pg_learner_t* h);
/* restore the optimiser step counters / beta-schedule clock (checkpoint resume) */
int32_t d4pg_learner_set_counters(d4pg_learner_t* h, int64_t adam_step, int64_t beta_t, d4pg_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Data-parallel communicator (one process per GPU).  The reference has no collective (its
 * multi-worker mode is Hogwild over shared CPU memory, main.py:394-405, ddpg.py:104-108);
 * this build is synchronous DP: one all-reduce of the flat [P_a+P_c] gradient per step.
 * NCCL is resolved at run time (dlopen of the torch-bundled libnccl.so.2).
 * ------------------------------------------------------------------------------------- */
int32_t d4pg_comm_unique_id(uint8_t* id128);                       /* ncclGetUniqueId, 128 bytes */
int32_t d4pg_comm_create(const uint8_t* id128, int32_t rank, int32_t world, d4pg_comm_t** out);
int32_t d4pg_comm_destroy(d4pg_comm_t* c);
int32_t d4pg_comm_allreduce_sum(d4pg_comm_t* c, float* buf, int64_t n, d4pg_stream_t stream);
/* Fused gradient all-reduce over peer memory (one node, <= 8 ranks) instead of the NCCL kernel: every rank allocates
 * an exchange block ([2][n_floats] gradient halves + flags) and exports it with CUDA IPC (64-byte handle); after the
 * handles of all ranks were gathered (rank order) every rank maps them.  A learner created with such a communicator
 * writes its dW into its own half, a flag barrier orders the ranks, and the fused Adam kernel sums all ranks' halves
 * (fixed rank order: replicas stay bit-identical) while it updates the parameters. */
int32_t d4pg_comm_peer_alloc(d4pg_comm_t* c, int64_t n_floats, uint8_t* handle64);
int32_t d4pg_comm_peer_open(d4pg_comm_t* c, const uint8_t* all_handles /* world x 64 bytes */);
int32_t d4pg_comm_peer_ready(const d4pg_comm_t* c);
int32_t d4pg_comm_peer_disable(d4pg_comm_t* c);      /* collective decision: fall back to the NCCL all-reduce */

/* In-switch gradient reduction (NVLS): ONE multicast object spans every rank's [2][n] gradient buffer; the fused Adam
 * kernel then reads the sum over all ranks with multimem.ld_reduce (the NVSwitch adds) -- one NVLink hop, n floats inbound
 * per rank whatever the rank count.  Collective setup, driven by the host binding after d4pg_comm_peer_open:
 *   every rank: d4pg_comm_mc_supported;  rank 0: d4pg_comm_mc_create -> POSIX file descriptor, passed to the other ranks
 *   (SCM_RIGHTS over a Unix socket) which d4pg_comm_mc_import it;  every rank: d4pg_comm_mc_add_device;  barrier;  every
 *   rank: d4pg_comm_mc_bind (allocates its buffer, binds it, maps the unicast and the multicast view);  barrier.
 * d4pg_comm_mc_selftest copies `src` (n floats, device) into this rank's buffer and/or writes the switch-reduced sum over
 * all ranks to `out`; the binding uses it to check that every rank reads bit-identical sums before enabling the path. */
int32_t d4pg_comm_mc_supported(d4pg_comm_t* c);
int32_t d4pg_comm_mc_create(d4pg_comm_t* c, int32_t* fd_out);
int32_t d4pg_comm_mc_import(d4pg_comm_t* c, int32_t fd);
int32_t d4pg_comm_mc_add_device(d4pg_comm_t* c);
int32_t d4pg_comm_mc_bind(d4pg_comm_t* c);
int32_t d4pg_comm_mc_ready(const d4pg_comm_t* c);
int32_t d4pg_comm_mc_disable(d4pg_comm_t* c);
int32_t d4pg_comm_mc_selftest(d4pg_comm_t* c, const float* src, float* out, int64_t n, d4pg_stream_t stream);

/* Debug: %globaltimer (ns) phase stamps written by the step kernels when
 * the environment variable D4PG_TC_TRACE is set (out16 = 32 x uint64, host memory). */
int32_t d4pg_debug_tc_trace(unsigned long long* out16);
/* first n (<= 512) stamps of the same buffer: the chain kernels write 6-8 per layer slot of one CTA */
int32_t d4pg_debug_trace_read(unsigned long long* out, int32_t n);
/* Watchdog record of the tensor-core chain kernels (16 x uint64, host memory): every mbarrier wait inside them is bounded;
 * a wait that times out traps the launch and leaves {1, code | slot<<8 | rank<<16 | parity<<24 | block<<32, aux, ...}
 * in host-mapped memory, readable here even after the failed launch invalidated the context; words [4 + 2k, 5 + 2k] hold
 * the first timed-out wait of kind k = 1..5 (loader: MMAs of the slot done, MMA: weights / A chunk landed).  All zero = never fired. */
int32_t d4pg_debug_watchdog(unsigned long long* out16);

#ifdef __cplusplus
}
#endif
#endif /* D4PG_B200_H_ */
