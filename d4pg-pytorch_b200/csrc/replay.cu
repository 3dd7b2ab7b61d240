// GPU-resident prioritized replay: fp32 sum/min segment trees + SoA transition storage.
//
// Replaces (reference, relative to its repository root):
//   prioritized_replay_memory.py:33-113   SegmentTree (__setitem__, reduce, _reduce_helper)
//   prioritized_replay_memory.py:114-162  SumSegmentTree.sum/find_prefixsum_idx, MinSegmentTree.min
//   prioritized_replay_memory.py:164-222  ReplayBuffer.add/_encode_sample
//   prioritized_replay_memory.py:224-335  PrioritizedReplayBuffer.add/_sample_proportional/sample/
//                                         update_priorities
//   replay_memory.py:14-19,61-80          Replay.add / Replay.sample (gather only)
//
// Tree layout is the reference's: root at 1, leaves at [cap, 2cap), V[i] = op(V[2i], V[2i+1]).
// Node dtype is fp32 -- what the reference's Python evaluates to under NumPy 2 (SURVEY.md H11).
// Everything is HBM/L2 pointer chasing + row gathers: no tensor-core work here.
#include "replay_dev.cuh"
#include <stdlib.h>
#include <new>
#include <string.h>
#include <algorithm>

struct d4pg_replay {
  int64_t size, cap; int log2cap;
  int obs_dim, act_dim;
  double alpha; float alpha_f32;
  float* sum; float* mn;
  float* obs; float* act; double* rew; float* obs2; uint8_t* done;
  int32_t* scratch; float* state;
  int64_t len, next_idx;
  int pristine;
  int64_t gen;            // bumped by every external mutation (add / set / update): a learner's prefetched batch is stale
  // host ingest staging (caller-owned buffers registered by d4pg_replay_set_staging)
  // two slots (halves of the registered buffers) so the host can stage add k+1 while add k still waits on the device
  uint8_t* stage_host; uint8_t* stage_dev; int64_t stage_bytes; cudaEvent_t stage_ev[2]; bool stage_busy[2]; int stage_slot;
  // ingest gate (learner host pipeline): the next kernel that touches the store / trees on the ingest stream first waits
  // until *gate_flag >= gate_target (the priority write-back of the last launched learner step)
  // The flag lives with the buffer (learners come and go); every gated step bumps it once and arms target = #armed.
  unsigned long long* gate_flag; unsigned long long gate_target; bool gate_pending;
  cudaEvent_t order_ev;
  // observation normalizer (d4pg_replay_set_obs_norm): caller-owned stats / affine, updated by every insert
  double* norm_stats; float* norm_affine; double norm_clip, norm_eps;
  // per-row horizon column (d4pg_replay_set_horizons): k of an episode-tail row, 0 for every other row
  uint8_t* horizon;
};

namespace d4pg {
// step timeline (D4PG_TC_TRACE, tools/e2e_timeline.py): ingest kernels stamp slots 10 (gate), 11 (ring write), 12 (tree add)
static unsigned long long* step_trace() { unsigned long long* p = debug_trace_buffer(); return p ? p + STEP_TRACE_BASE : nullptr; }


// NORM: the learner's batch goes through the observation normalizer as it is gathered (sample_body<true, .>); HZ: the
// rows' horizons are gathered too (episode tails).  The instantiations are separate non-template kernels so that the
// plain one compiles to what it was before either option.
template <bool NORM, bool HZ>
__device__ __forceinline__ void sample_gather_body(const SampleArgs& a) {
  __shared__ SampleSmem sm;
  pdl_trigger(a.pdl);
  pdl_wait();
  step_stamp(a.trace, a.trace_slot);
  sample_body<NORM, HZ>(a, blockIdx.x, sm);
  if (a.done_epoch) {                          // the forward chains of the step poll these instead of a stream event
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned long long e = (unsigned long long)(a.clock->s_steps_done + 1);
      asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(a.done_epoch + blockIdx.x), "l"(e) : "memory");
    }
  }
  step_stamp(a.trace, a.trace_slot + 16);
  pdl_trigger_end(a.pdl);
}
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_gather_kernel(const SampleArgs a) { sample_gather_body<false, false>(a); }
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_gather_norm_kernel(const SampleArgs a) { sample_gather_body<true, false>(a); }
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_gather_hz_kernel(const SampleArgs a) { sample_gather_body<false, true>(a); }
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_gather_norm_hz_kernel(const SampleArgs a) { sample_gather_body<true, true>(a); }

template <int MODE>
__global__ void __launch_bounds__(TREE_THREADS) tree_write_kernel(const TreeArgs a) {
  __shared__ float red[32];
  step_stamp(a.trace, 3);
  tree_write_body<MODE, TREE_THREADS>(a, red);
  step_stamp(a.trace, 3 + 16);
}


__global__ void __launch_bounds__(TREE_FAST_MAX) tree_update_fast_kernel(const TreeArgs a, int hs, int D) {
  extern __shared__ __align__(16) unsigned char tree_smem[];
  __shared__ float red[32];
  step_stamp(a.trace, 3);
  tree_update_fast_body(a, tree_smem, hs, red, blockIdx.x, D);
  step_stamp(a.trace, 3 + 16);
}

// add(): the new leaves are one contiguous ring range [start, start+n) (no wrap: the host splits a
// wrapping add), so level l only has the nodes (cap+start)>>l .. (cap+start+n-1)>>l to recompute:
// ~2n node updates in total instead of n*log2(cap), and the narrow top of the tree is finished by
// one warp without block-wide barriers.
__global__ void __launch_bounds__(TREE_THREADS) tree_add_range_kernel(float* sum, float* mn, int64_t cap, int log2cap,
                                                                      int64_t start, int64_t n, const ReplayState* state,
                                                                      float alpha_f32) {
  const int t = threadIdx.x;
  const float leaf = pow_alpha(state->max_priority, alpha_f32);      // :255-256
  for (int64_t i = t; i < n; i += TREE_THREADS) { sum[cap + start + i] = leaf; mn[cap + start + i] = leaf; }
  int lvl = 1;
  for (; lvl <= log2cap; ++lvl) {
    const int64_t lo = (cap + start) >> lvl, hi = (cap + start + n - 1) >> lvl;
    if (hi - lo + 1 <= 32) break;                                     // narrow: hand over to warp 0
    __syncthreads();
    for (int64_t node = lo + t; node <= hi; node += TREE_THREADS) {
      sum[node] = __fadd_rn(__ldcg(sum + 2 * node), __ldcg(sum + 2 * node + 1));
      mn[node] = fminf(__ldcg(mn + 2 * node), __ldcg(mn + 2 * node + 1));
    }
  }
  __syncthreads();
  if (t < 32) {
    for (; lvl <= log2cap; ++lvl) {
      const int64_t lo = (cap + start) >> lvl, hi = (cap + start + n - 1) >> lvl;
      const int64_t node = lo + t;
      if (node <= hi) {
        sum[node] = __fadd_rn(__ldcg(sum + 2 * node), __ldcg(sum + 2 * node + 1));
        mn[node] = fminf(__ldcg(mn + 2 * node), __ldcg(mn + 2 * node + 1));
      }
      __threadfence_block();
      __syncwarp();
    }
  }
}

// The same update with ONE round trip to L2 (n <= TREE_ADD_FAST_MAX): a parent inside the recomputed range has both
// children inside the range of the level below, except at the two edges, where the outside child is an OLD node.
// Those <= 2 old nodes per level (and tree) are fetched up front, in flight together; the levels are then computed
// from shared memory.  Identical arithmetic (fp32 left + right, fminf), so the resulting tree is bit-identical.
constexpr int TREE_ADD_FAST_MAX = 2048;
__global__ void __launch_bounds__(TREE_THREADS) tree_add_range_fast_kernel(float* sum, float* mn, int64_t cap, int log2cap,
                                                                           int64_t start, int64_t n, const ReplayState* state,
                                                                           float alpha_f32, unsigned long long* trace,
                                                                           const unsigned long long* gate_flag,
                                                                           unsigned long long gate_target) {
  __shared__ float vs[2][TREE_ADD_FAST_MAX], vm[2][TREE_ADD_FAST_MAX];
  __shared__ float old_s[2][32], old_m[2][32];                         // [left / right edge][level]
  const int t = threadIdx.x;
  step_stamp(trace, 10);
  if (gate_flag) {                                                     // ingest gate, fused: saves a kernel boundary
    if (t == 0) {
      unsigned long long v;
      do { asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(gate_flag) : "memory"); } while (v < gate_target);
    }
    __syncthreads();
  }
  pdl_trigger_raw();      // a programmatically dependent sample kernel (host pipeline) may become resident now; it still waits for this grid's end
  step_stamp(trace, 12);
  const float leaf = pow_alpha(state->max_priority, alpha_f32);       // :255-256
  if (t < 2 * log2cap) {
    const int lvl = (t >> 1) + 1, side = t & 1;                        // the outside child needed by level `lvl`
    const int64_t plo = (cap + start) >> (lvl - 1), phi = (cap + start + n - 1) >> (lvl - 1);
    float a = 0.f, b = INFINITY;
    if (side == 0 && (plo & 1)) { a = __ldcg(sum + plo - 1); b = __ldcg(mn + plo - 1); }
    if (side == 1 && !(phi & 1)) { a = __ldcg(sum + phi + 1); b = __ldcg(mn + phi + 1); }
    old_s[side][lvl] = a; old_m[side][lvl] = b;
  }
  for (int64_t i = t; i < n; i += TREE_THREADS) {
    sum[cap + start + i] = leaf; mn[cap + start + i] = leaf;
    vs[0][i] = leaf; vm[0][i] = leaf;
  }
  __syncthreads();
  for (int lvl = 1; lvl <= log2cap; ++lvl) {
    const int cur = lvl & 1, prev = cur ^ 1;
    const int64_t lo = (cap + start) >> lvl, hi = (cap + start + n - 1) >> lvl;
    const int64_t plo = (cap + start) >> (lvl - 1), phi = (cap + start + n - 1) >> (lvl - 1);
    for (int64_t j = t; j <= hi - lo; j += TREE_THREADS) {
      const int64_t node = lo + j, l = 2 * node, r = 2 * node + 1;
      const float ls = l >= plo ? vs[prev][l - plo] : old_s[0][lvl], lm = l >= plo ? vm[prev][l - plo] : old_m[0][lvl];
      const float rs = r <= phi ? vs[prev][r - plo] : old_s[1][lvl], rm = r <= phi ? vm[prev][r - plo] : old_m[1][lvl];
      const float s2 = __fadd_rn(ls, rs), m2 = fminf(lm, rm);
      vs[cur][j] = s2; vm[cur][j] = m2;
      sum[node] = s2; mn[node] = m2;
    }
    __syncthreads();
  }
  step_stamp(trace, 12 + 16);
}

// bulk path for large adds: grid-wide leaf fill, then one launch per level
__global__ void leaf_fill_kernel(float* sum, float* mn, int64_t cap, int64_t size, int64_t ring_start,
                                 int64_t n, const ReplayState* state, float alpha_f32) {
  const float leaf = pow_alpha(state->max_priority, alpha_f32);
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t p = (ring_start + i) % size;
    sum[cap + p] = leaf; mn[cap + p] = leaf;
  }
}
__global__ void level_rebuild_kernel(float* sum, float* mn, int64_t first, int64_t count) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < count; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t node = first + i;
    sum[node] = __fadd_rn(sum[2 * node], sum[2 * node + 1]);
    mn[node] = fminf(mn[2 * node], mn[2 * node + 1]);
  }
}

// ring insert of n rows from device staging buffers (ReplayBuffer.add, :180-187)
__global__ void ring_write_kernel(float* obs, float* act, double* rew, float* obs2, uint8_t* done,
                                  const float* s, const float* a, const double* r, const float* s2,
                                  const uint8_t* d, int64_t n, int obs_dim, int act_dim,
                                  int64_t size, int64_t ring_start, ReplayState* state,
                                  int64_t new_len, int64_t new_next, unsigned long long* trace) {
  const int64_t stride = int64_t(gridDim.x) * blockDim.x, t0 = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  step_stamp(trace, 11);
  if (t0 == 0) { state->len = new_len; state->next_idx = new_next; }
  for (int64_t e = t0; e < n * obs_dim; e += stride) {
    const int64_t i = e / obs_dim, c = e - i * obs_dim, p = (ring_start + i) % size;
    obs[p * obs_dim + c] = s[e];
    obs2[p * obs_dim + c] = s2[e];
  }
  for (int64_t e = t0; e < n * act_dim; e += stride) {
    const int64_t i = e / act_dim, c = e - i * act_dim, p = (ring_start + i) % size;
    act[p * act_dim + c] = a[e];
  }
  for (int64_t i = t0; i < n; i += stride) {
    const int64_t p = (ring_start + i) % size;
    rew[p] = r[i]; done[p] = d[i];
  }
  step_stamp(trace, 11 + 16);
}

__global__ void tree_init_kernel(float* sum, float* mn, int32_t* scratch, ReplayState* state, int64_t cap) {
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const int64_t t0 = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  for (int64_t i = t0; i < 2 * cap; i += stride) {
    sum[i] = 0.f; mn[i] = INFINITY;                                  // neutral elements, :116-120,152-156
    if (i < cap) scratch[i] = -1;
  }
  if (t0 == 0) {
    state->max_priority = 1.0f;                                      // :249
    state->pristine = 1; state->len = 0; state->next_idx = 0; state->reserved = 0;
  }
}

__global__ void state_set_kernel(ReplayState* state, int64_t len, int64_t next_idx, int pristine) {
  state->len = len; state->next_idx = next_idx; state->pristine = pristine;
}

// SegmentTree.reduce(start, end+1) for an arbitrary range with _reduce_helper's association
// (:61-96): after the first split the left part is a suffix query (left-nested from the deepest
// node up) and the right part a prefix query (right-nested); IS_SUM selects + or min.
template <bool IS_SUM>
__device__ float range_reduce_ref(const float* __restrict__ V, int64_t cap, int64_t s, int64_t e) {
  auto op = [](float a, float b) { return IS_SUM ? __fadd_rn(a, b) : fminf(a, b); };
  int64_t node = 1, lo = 0, hi = cap - 1;
  while (true) {                                   // descend while the range sits in one child
    if (s == lo && e == hi) return __ldcg(V + node);
    const int64_t mid = (lo + hi) >> 1;
    if (e <= mid) { node = 2 * node; hi = mid; }
    else if (s > mid) { node = 2 * node + 1; lo = mid + 1; }
    else break;
  }
  const int64_t mid = (lo + hi) >> 1;
  // left: suffix [s, mid] of node 2*node
  float terms[40]; int n = 0;
  int64_t nd = 2 * node, l2 = lo, h2 = mid;
  while (s != l2) {
    const int64_t m2 = (l2 + h2) >> 1;
    if (s > m2) { nd = 2 * nd + 1; l2 = m2 + 1; }
    else { terms[n++] = __ldcg(V + 2 * nd + 1); nd = 2 * nd; h2 = m2; }
  }
  float left = __ldcg(V + nd);
  for (int i = n - 1; i >= 0; --i) left = op(left, terms[i]);
  // right: prefix [mid+1, e] of node 2*node+1
  n = 0; nd = 2 * node + 1; l2 = mid + 1; h2 = hi;
  while (e != h2) {
    const int64_t m2 = (l2 + h2) >> 1;
    if (e <= m2) { nd = 2 * nd; h2 = m2; }
    else { terms[n++] = __ldcg(V + 2 * nd); nd = 2 * nd + 1; l2 = m2 + 1; }
  }
  float right = __ldcg(V + nd);
  for (int i = n - 1; i >= 0; --i) right = op(terms[i], right);
  return op(left, right);
}

__global__ void reduce_kernel(const float* sum, const float* mn, int64_t cap, int64_t s, int64_t e, float* out) {
  if (threadIdx.x == 0) { out[0] = range_reduce_ref<true>(sum, cap, s, e); out[1] = range_reduce_ref<false>(mn, cap, s, e); }
}

// SumSegmentTree.find_prefixsum_idx (:126-149) for caller-supplied masses (fp32 descent)
__global__ void find_prefix_kernel(const float* sum, int64_t cap, int n, const double* masses, int32_t* idx) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  float mass = __double2float_rn(masses[t]);
  int64_t i = 1;
  while (i < cap) {
    const float left = __ldcg(sum + 2 * i);
    if (left > mass) i = 2 * i;
    else { mass = __fsub_rn(mass, left); i = 2 * i + 1; }
  }
  idx[t] = int32_t(i - cap);
}

static cudaStream_t g_side_stream = nullptr;          // trace only: which launches are the prefetching sampler's
void trace_set_side_stream(cudaStream_t s) { g_side_stream = s; }
static bool st_is_side(cudaStream_t st) { return g_side_stream != nullptr && st == g_side_stream; }
int launch_sample(const d4pg_replay* h, SampleArgs& a, cudaStream_t st, bool dependent = false) {
  a.sum = h->sum; a.mn = h->mn; a.cap = h->cap; a.state = reinterpret_cast<const ReplayState*>(h->state);
  a.obs = h->obs; a.act = h->act; a.rew = h->rew; a.obs2 = h->obs2; a.done = h->done;
  a.obs_dim = h->obs_dim; a.act_dim = h->act_dim;
  a.pdl = pdl_mode();
  a.trace = (a.clock && debug_trace_buffer()) ? debug_trace_buffer() + STEP_TRACE_BASE : nullptr;
  a.trace_slot = a.pipe_slot >= 0 && a.uniforms == nullptr && st_is_side(st) ? 4 : 0;
  // a.norm (learner with an observation normalizer): s / s2 are normalized as they are gathered; a.hz (learner with
  // episode tails): the rows' horizons are gathered from the ring's column
  a.horizon = a.hz ? h->horizon : nullptr;
  void (*kernel)(const SampleArgs) = a.hz ? (a.norm ? sample_gather_norm_hz_kernel : sample_gather_hz_kernel)
                                          : (a.norm ? sample_gather_norm_kernel : sample_gather_kernel);
  if (a.hz) {
    if (a.norm) D4PG_MAX_CARVEOUT(sample_gather_norm_hz_kernel);
    else D4PG_MAX_CARVEOUT(sample_gather_hz_kernel);
  } else if (a.norm) D4PG_MAX_CARVEOUT(sample_gather_norm_kernel);
  else D4PG_MAX_CARVEOUT(sample_gather_kernel);
  if (dependent) {
    // programmatic dependent launch behind the previous kernel of the stream (the host pipeline's tree add): the grid is
    // resident when that kernel ends, griddepcontrol.wait at the top of the kernel holds it until its writes are visible
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(cdiv(a.B, SAMPLE_ROWS)); cfg.blockDim = dim3(SAMPLE_THREADS); cfg.dynamicSmemBytes = 0; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    D4PG_CUDA_OK(cudaLaunchKernelEx(&cfg, kernel, a));
    return D4PG_OK;
  }
  D4PG_CUDA_OK(launch_pdl(kernel, dim3(cdiv(a.B, SAMPLE_ROWS)), dim3(SAMPLE_THREADS), 0, st, a));
  return D4PG_OK;
}

int learner_sample(d4pg_replay* h, int B, int prioritized, const double* uniforms, const int32_t* positions,
                   uint64_t seed, LearnerClock* clock, const ClockParams& cp,
                   int32_t* idx, float* weights, float* s, float* a, double* r, float* s2, uint8_t* d, uint8_t* hz,
                   int ld_obs, int ld_act, const float* norm, float norm_clip, int pipe_slot, cudaStream_t st, bool dependent,
                   unsigned long long* done_epoch) {
  SampleArgs sa{};
  sa.done_epoch = done_epoch; sa.hz = hz;
  sa.norm = norm; sa.norm_clip = norm_clip;
  sa.ld_obs = ld_obs; sa.ld_act = ld_act; sa.pipe_slot = pipe_slot;
  sa.uniforms = uniforms; sa.seed = seed; sa.counter = 0; sa.clock = clock; sa.clock_params = cp;
  sa.beta = 1.f; sa.B = B; sa.idx = idx; sa.weights = prioritized ? weights : nullptr;
  sa.s = s; sa.a = a; sa.r = r; sa.s2 = s2; sa.d = d;
  if (!prioritized) { sa.idx_in = positions; sa.uniform_mode = positions ? 0 : 1; }
  return launch_sample(h, sa, st, dependent);
}

// The tree kernels' view of the store, writing the n leaves idx with the values v0 (priorities, or a set's sums)
static TreeArgs tree_args(const d4pg_replay* h, int n, const int32_t* idx, const float* v0) {
  TreeArgs a{};
  a.sum = h->sum; a.mn = h->mn; a.cap = h->cap; a.log2cap = h->log2cap; a.size = h->size;
  a.n = n; a.idx = idx; a.v0 = v0; a.alpha_f32 = h->alpha_f32; a.scratch = h->scratch;
  a.state = reinterpret_cast<ReplayState*>(h->state);
  return a;
}

int64_t replay_generation(const d4pg_replay* h) { return h->gen; }
const float* replay_obs_norm(const d4pg_replay* h, double* clip) { if (clip) *clip = h->norm_clip; return h->norm_affine; }
const uint8_t* replay_horizons(const d4pg_replay* h) { return h->horizon; }

int launch_gate_signal(unsigned long long* flag, cudaStream_t st);
int launch_tree_update(d4pg_replay* h, int B, const int32_t* idx, const float* prio, cudaStream_t st, unsigned long long* gate) {
  TreeArgs a = tree_args(h, B, idx, prio);
  a.trace = (st_is_side(st) && debug_trace_buffer()) ? debug_trace_buffer() + STEP_TRACE_BASE : nullptr;
  if (B <= TREE_FAST_MAX && h->log2cap < TREE_FAST_LEVELS) {
    int hs = 64;
    while (hs < 2 * B) hs *= 2;
    const int threads = ((B + 31) / 32) * 32;
    const size_t smem = size_t(hs) * 2 * (sizeof(int) + sizeof(float2));     // 12 KB at B = 512
    D4PG_MAX_CARVEOUT(tree_update_fast_kernel);
    const int D = std::min(4, h->log2cap);                     // 2^D CTAs, one per top-level subtree
    if (D > 0) { a.gate = gate; gate = nullptr; }   // the last CTA opens the gate itself
    tree_update_fast_kernel<<<1 << D, threads, smem, st>>>(a, hs, D);
  } else {
    D4PG_MAX_CARVEOUT(tree_write_kernel<TREE_UPDATE>);
    tree_write_kernel<TREE_UPDATE><<<1, TREE_THREADS, 0, st>>>(a);
  }
  D4PG_LAUNCH_OK();
  if (gate) { int rc = launch_gate_signal(gate, st); if (rc) return rc; }
  h->pristine = 0;
  return D4PG_OK;
}

}  // namespace d4pg

using namespace d4pg;

extern "C" int32_t d4pg_replay_capacity(int64_t size, int64_t* cap_out) {
  D4PG_REQUIRE(size > 0 && cap_out, D4PG_EINVAL, "d4pg_replay_capacity: bad arguments");
  int64_t cap = 1;
  while (cap < size) cap *= 2;                                       // :243-245
  *cap_out = cap;
  return D4PG_OK;
}

extern "C" int32_t d4pg_replay_create(int64_t size, int32_t obs_dim, int32_t act_dim, double alpha,
                                      float* sum_tree, float* min_tree,
                                      float* obs, float* act, double* rew, float* obs2, uint8_t* done,
                                      int32_t* scratch, float* state, d4pg_stream_t stream, d4pg_replay_t** out) {
  D4PG_REQUIRE(out && size > 0 && size < (int64_t(1) << 30), D4PG_EINVAL, "d4pg_replay_create: size out of range");
  D4PG_REQUIRE(obs_dim > 0 && act_dim > 0, D4PG_EINVAL, "d4pg_replay_create: dims must be positive");
  D4PG_REQUIRE(alpha >= 0, D4PG_EINVAL, "d4pg_replay_create: alpha must be >= 0");                      // :240
  D4PG_REQUIRE(sum_tree && min_tree && obs && act && rew && obs2 && done && scratch && state, D4PG_EINVAL,
               "d4pg_replay_create: null buffer");
  d4pg_replay* h = new (std::nothrow) d4pg_replay();
  D4PG_REQUIRE(h, D4PG_EINVAL, "d4pg_replay_create: out of host memory");
  h->size = size; d4pg_replay_capacity(size, &h->cap);
  h->log2cap = 0; while ((int64_t(1) << h->log2cap) < h->cap) ++h->log2cap;
  h->obs_dim = obs_dim; h->act_dim = act_dim; h->alpha = alpha; h->alpha_f32 = float(alpha);
  h->sum = sum_tree; h->mn = min_tree; h->obs = obs; h->act = act; h->rew = rew; h->obs2 = obs2; h->done = done;
  h->scratch = scratch; h->state = state; h->len = 0; h->next_idx = 0; h->pristine = 1;
  h->stage_host = nullptr; h->stage_dev = nullptr; h->stage_bytes = 0; h->stage_slot = 0;
  for (int i = 0; i < 2; ++i) { h->stage_ev[i] = nullptr; h->stage_busy[i] = false; }
  h->gate_flag = nullptr; h->gate_target = 0; h->gate_pending = false; h->order_ev = nullptr;
  h->norm_stats = nullptr; h->norm_affine = nullptr; h->norm_clip = 0.0; h->norm_eps = 0.0;
  h->horizon = nullptr;
  tree_init_kernel<<<2 * device_sm_count(), 256, 0, as_stream(stream)>>>(h->sum, h->mn, h->scratch,
                                                        reinterpret_cast<ReplayState*>(h->state), h->cap);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("d4pg_replay_create: %s", cudaGetErrorString(e)); delete h; return D4PG_ECUDA; }
  *out = h;
  return D4PG_OK;
}

extern "C" int32_t d4pg_replay_destroy(d4pg_replay_t* h) {
  if (h) {
    for (int i = 0; i < 2; ++i) if (h->stage_ev[i]) cudaEventDestroy(h->stage_ev[i]);
    if (h->order_ev) cudaEventDestroy(h->order_ev);
    if (h->gate_flag) { cudaDeviceSynchronize(); cudaFree(h->gate_flag); }
  }
  delete h;
  return D4PG_OK;
}

namespace {
// the staging and window layouts start every array that needs it on a 16-byte boundary
int64_t up16(int64_t b) { return (b + 15) & ~int64_t(15); }

struct PackLayout { int64_t obs, obs2, act, rew, done, total; };
PackLayout pack_layout(const d4pg_replay* h, int64_t n) {
  PackLayout p;
  const int64_t S = int64_t(h->obs_dim) * 4, A = int64_t(h->act_dim) * 4;
  p.obs = 0; p.obs2 = p.obs + n * S; p.act = p.obs2 + n * S;
  p.rew = up16(p.act + n * A);
  p.done = p.rew + n * 8;
  p.total = up16(p.done + n);
  return p;
}
}  // namespace

extern "C" int64_t d4pg_replay_staging_bytes(const d4pg_replay_t* h, int64_t rows) {
  return (h && rows > 0) ? 2 * pack_layout(h, rows).total : -1;      // two staging slots
}

extern "C" int32_t d4pg_replay_set_staging(d4pg_replay_t* h, void* pinned_host, void* device, int64_t bytes) {
  D4PG_REQUIRE(h && pinned_host && device && bytes > 0, D4PG_EINVAL, "d4pg_replay_set_staging: bad arguments");
  h->stage_host = static_cast<uint8_t*>(pinned_host); h->stage_dev = static_cast<uint8_t*>(device);
  h->stage_bytes = (bytes / 2) & ~int64_t(15);                        // per slot
  for (int i = 0; i < 2; ++i) {
    if (!h->stage_ev[i]) D4PG_CUDA_OK(cudaEventCreateWithFlags(&h->stage_ev[i], cudaEventDisableTiming));
    h->stage_busy[i] = false;
  }
  h->stage_slot = 0;
  return D4PG_OK;
}

// ---- device-side ingest: n-step return accumulation at insert (replay_memory.py:38-45) ------------------------
// Transition i of an episode of T steps: (s_i, a_i, sum_{k<n} gamma^k r_{i+k}, s'_{i+n-1}, done_{i+n-1}).  Only the
// reward needs arithmetic -- s'/done are the same arrays shifted by n-1 rows -- and it is the reference's own
// left-to-right f64 loop (`cum += exp_gamma * r; exp_gamma *= gamma`) with explicit _rn ops (no FMA contraction).
// nstep_return is that loop over n consecutive rewards; the episode kernel and the streaming windows both call it.
__device__ __forceinline__ double nstep_return(const double* __restrict__ r, int n, double gamma) {
  double cum = 0.0, eg = 1.0;
  for (int k = 0; k < n; ++k) {
    cum = __dadd_rn(cum, __dmul_rn(eg, r[k]));
    eg = __dmul_rn(eg, gamma);
  }
  return cum;
}

__global__ void nstep_returns_kernel(const double* __restrict__ rew, int64_t T, int n, double gamma, double* __restrict__ out) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i + n > T) return;
  out[i] = nstep_return(rew + i, n, gamma);
}

// ---- device-side ingest: streaming n-step windows of E environments (DESIGN.md §3 "Streaming n-step insert") ------
// One call = one vector step.  Environment e appends (s, a, r) to its window; once the window holds n steps of the
// current episode it emits (s_{t-n+1}, a_{t-n+1}, R, s'_t, terminated_t), R = nstep_return over the window's rewards;
// then an episode end clears the window.  Emitting environments take consecutive ring rows in ascending e.
//
// Window state (caller-owned, zero-filled before the first call; d4pg_replay_steps_window_bytes):
//   rec u64 [E]      {bits 0-31: id of the last call, 32-39: fill before it, 40-47: fill after it}
//   wr  f64 [E, 2n]  reward of step u at u % n AND u % n + n, so the last n rewards are contiguous from (fill+1) % n
//   ws  f32 [E, n, S], wa f32 [E, n, A]: s / a of step u at u % n (not written for n = 1)
// fill counts the steps of the current episode, kept in [0, 2n) by subtracting n (u % n is all that is used).
// The emit decision of e needs the fill BEFORE this call; a CTA counts the emitters below its first environment from
// the other CTAs' records, which may or may not have been rewritten yet: a record carrying this call's id holds the
// old fill in bits 32-39.  Every record carries the same call id between calls, because every call steps all E.
//
// TAILS (DESIGN.md §3 "Episode tails"): an episode that ends at a call with fill f leaves P = min(f + 1, n - 1) pending
// tail rows, which environment e emits first thing at its next call, before it appends that call's step: start
// u = f + 1 - P + i (i < P) gives (s_u, a_u, nstep_return over its k = P - i remaining rewards, obs_next and terminated
// of the ending step) with horizon k.  The window also keeps that obs_next (wo f32 [E, S], after wa), and the record
// {bits 48-53: P, 54: terminated, 55-60: (f + 1) % n}; a rewritten record holds the ROWS its call emitted in bits 32-39
// (P, or 1 for a full row), which is what the other CTAs count.  Every row writes its horizon: k, or 0 for a full row.
constexpr int STEPS_THREADS = 256, STEPS_WARPS = STEPS_THREADS / 32;
struct StepsArgs {
  const float* obs; const float* act; const double* rew; const float* obs2; const uint8_t* term; const uint8_t* end;
  int64_t E, chunk; int S, A, n; double gamma;
  unsigned long long* rec; double* wr; float* ws; float* wa;
  float* r_obs; float* r_act; double* r_rew; float* r_obs2; uint8_t* r_done;
  int64_t size, start, n_rows, new_len, new_next; ReplayState* state;
  float* wo; uint8_t* r_hz;          // TAILS only
};

__device__ __forceinline__ int steps_fill_before(unsigned long long rec, unsigned kprev) {
  return int(((unsigned)rec == kprev ? rec >> 40 : rec >> 32) & 0xff);
}
// TAILS: the rows environment `rec` emits at this call (a full row, or its pending tails)
__device__ __forceinline__ int steps_rows(unsigned long long rec, unsigned kprev, int n) {
  if ((unsigned)rec != kprev) return int((rec >> 32) & 0xff);
  return int(((rec >> 40) & 0xff) >= unsigned(n - 1)) + int((rec >> 48) & 0x3f);
}

template <bool TAILS>
__global__ void __launch_bounds__(STEPS_THREADS) replay_add_steps_kernel(const StepsArgs a) {
  __shared__ int red[STEPS_WARPS];
  __shared__ int fill_s[STEPS_THREADS], rank_s[STEPS_THREADS];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5, n = a.n, S = a.S, A = a.A;
  const int64_t e0 = int64_t(blockIdx.x) * a.chunk, e1 = min(a.E, e0 + a.chunk);
  if (blockIdx.x == 0 && t == 0) { a.state->len = a.new_len; a.state->next_idx = a.new_next; }
  // this CTA rewrites its own records only after the barriers below, so rec[e0] still has the previous call's id
  const unsigned kprev = (unsigned)__ldcg(a.rec + e0);
  // emitting environments in [0, e0)
  int c = 0;
  for (int64_t e = t; e < e0; e += STEPS_THREADS)
    c += TAILS ? steps_rows(__ldcg(a.rec + e), kprev, n) : steps_fill_before(__ldcg(a.rec + e), kprev) >= n - 1;
  c = __reduce_add_sync(0xffffffffu, c);
  if (lane == 0) red[w] = c;
  __syncthreads();
  int64_t base = 0;
  for (int i = 0; i < STEPS_WARPS; ++i) base += red[i];
  for (int64_t tile = e0; tile < e1; tile += STEPS_THREADS) {
    // exclusive rank of this tile's emitters (TAILS: of their first rows, by a warp scan of the row counts)
    const int64_t e = tile + t;
    int fill, within = 0;
    unsigned bal = 0u;
    if (TAILS) {
      const unsigned long long rc = e < e1 ? __ldcg(a.rec + e) : 0ull;
      fill = e < e1 ? steps_fill_before(rc, kprev) : 0;
      const int rows = e < e1 ? steps_rows(rc, kprev, n) : 0;
      int incl = rows;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      __syncthreads();                                 // red[] of the previous tile / the prefix count is consumed
      if (lane == 31) red[w] = incl;
      within = incl - rows;
    } else {
      fill = e < e1 ? steps_fill_before(__ldcg(a.rec + e), kprev) : 0;
      const bool emit = e < e1 && fill >= n - 1;
      bal = __ballot_sync(0xffffffffu, emit);
      __syncthreads();                                 // red[] of the previous tile / the prefix count is consumed
      if (lane == 0) red[w] = __popc(bal);
    }
    __syncthreads();
    int before = 0, total = 0;
    for (int i = 0; i < STEPS_WARPS; ++i) { before += i < w ? red[i] : 0; total += red[i]; }
    fill_s[t] = fill;
    rank_s[t] = before + (TAILS ? within : __popc(bal & ((1u << lane) - 1u)));
    __syncthreads();
    const int cnt = int(min(int64_t(STEPS_THREADS), e1 - tile));
    for (int j = w; j < cnt; j += STEPS_WARPS) {
      const int64_t ee = tile + j;
      const int f = fill_s[j], slot = f % n, old = (f + 1) % n;
      const int64_t rank = base + rank_s[j];
      const bool write = f >= n - 1 && rank < a.n_rows;       // never outside [start, start + n_rows)
      const int64_t p = (a.start + rank) % a.size;
      int P = 0;                                              // TAILS: pending tail rows, emitted before the append
      if (TAILS) {
        const unsigned long long rc = __ldcg(a.rec + ee);    // not rewritten yet (lane 0 does that after a __syncwarp)
        P = int((rc >> 48) & 0x3f);
        const uint8_t tterm = uint8_t((rc >> 54) & 1);
        const int endm = int((rc >> 55) & 0x3f);
        const float* tws = a.ws + ee * n * S;
        const float* twa = a.wa + ee * n * A;
        const float* two = a.wo + ee * S;
        int64_t q = p;                                        // ring slot and window slot of tail i, stepped
        int us = (endm - P + n) % n;
        for (int i = 0; i < P && rank + i < a.n_rows; ++i, q = q + 1 == a.size ? 0 : q + 1, us = us + 1 == n ? 0 : us + 1) {
          const int k = P - i;
          for (int c = lane; c < S; c += 32) { a.r_obs[q * S + c] = tws[us * S + c]; a.r_obs2[q * S + c] = two[c]; }
          for (int c = lane; c < A; c += 32) a.r_act[q * A + c] = twa[us * A + c];
          if (lane == 0) {
            a.r_rew[q] = nstep_return(a.wr + ee * 2 * n + us, k, a.gamma);
            a.r_done[q] = tterm;
            a.r_hz[q] = uint8_t(k);
          }
        }
        if (a.term[ee] != 0 || (a.end && a.end[ee] != 0))   // this step ends the episode: keep its obs_next
          for (int c = lane; c < S; c += 32) a.wo[ee * S + c] = a.obs2[ee * S + c];
      }
      const float* s_in = a.obs + ee * S;
      float* ws = a.ws + ee * n * S;
      for (int k = lane; k < S; k += 32) {
        const float v = s_in[k];
        if (n > 1) ws[slot * S + k] = v;
        if (write) {
          a.r_obs[p * S + k] = n > 1 ? ws[old * S + k] : v;
          a.r_obs2[p * S + k] = a.obs2[ee * S + k];
        }
      }
      const float* a_in = a.act + ee * A;
      float* wa = a.wa + ee * n * A;
      for (int k = lane; k < A; k += 32) {
        const float v = a_in[k];
        if (n > 1) wa[slot * A + k] = v;
        if (write) a.r_act[p * A + k] = n > 1 ? wa[old * A + k] : v;
      }
      if (TAILS) __syncwarp();                                // every lane has read the record
      if (lane == 0) {
        double* wr = a.wr + ee * 2 * n;
        if (n > 1) { const double r = a.rew[ee]; wr[slot] = r; wr[slot + n] = r; }
        const bool term = a.term[ee] != 0, ended = term || (a.end && a.end[ee] != 0);
        if (write) {
          a.r_rew[p] = nstep_return(n > 1 ? wr + old : a.rew + ee, n, a.gamma);
          a.r_done[p] = term ? 1 : 0;
          if (TAILS) a.r_hz[p] = 0;
        }
        const int nf = ended ? 0 : (f + 1 >= 2 * n ? f + 1 - n : f + 1);
        if (TAILS) {
          const int pn = ended ? min(f + 1, n - 1) : 0, rows = P + (f >= n - 1 ? 1 : 0);
          a.rec[ee] = (unsigned long long)(kprev + 1u) | ((unsigned long long)rows << 32) | ((unsigned long long)nf << 40) |
                      ((unsigned long long)pn << 48) | ((unsigned long long)(term ? 1 : 0) << 54) |
                      ((unsigned long long)((f + 1) % n) << 55);
        } else {
          a.rec[ee] = (unsigned long long)(kprev + 1u) | ((unsigned long long)f << 32) | ((unsigned long long)nf << 40);
        }
      }
    }
    base += total;
  }
}

extern "C" int32_t d4pg_nstep_returns(const double* rew, int64_t T, int32_t n_steps, double gamma, double* out,
                                      d4pg_stream_t stream) {
  D4PG_REQUIRE(rew && out && T > 0 && n_steps >= 1, D4PG_EINVAL, "d4pg_nstep_returns: bad arguments");
  if (T < n_steps) return D4PG_OK;                        // the reference adds nothing before step n-1 (:38)
  const int64_t m = T - n_steps + 1;
  nstep_returns_kernel<<<unsigned((m + 255) / 256), 256, 0, as_stream(stream)>>>(rew, T, n_steps, gamma, out);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

extern "C" int32_t d4pg_replay_add_nstep(d4pg_replay_t* h, int64_t T, const float* obs, const float* act, const double* rew,
                                         const float* obs2, const uint8_t* done, int32_t n_steps, double gamma,
                                         double* rew_scratch, int32_t prioritized, d4pg_stream_t stream) {
  D4PG_REQUIRE(h && obs && act && rew && obs2 && done && rew_scratch && T > 0 && n_steps >= 1, D4PG_EINVAL,
               "d4pg_replay_add_nstep: bad arguments");
  if (T < n_steps) return D4PG_OK;
  int rc = d4pg_nstep_returns(rew, T, n_steps, gamma, rew_scratch, stream);
  if (rc) return rc;
  const int64_t shift = n_steps - 1;
  return d4pg_replay_add(h, T - shift, obs, act, rew_scratch, obs2 + shift * h->obs_dim, done + shift, prioritized, stream);
}

// ---- device-side ingest: hindsight relabelling (main.py:154-184, "future" strategy) ------------------------------
// Episode of T goal-conditioned steps: obs/obs_next [T, So] f32, goal [T, G] f64 (the desired goal of every step),
// ag_next [T, G] f64 (achieved goal of the NEXT state), act [T, A], rew [T] f64, done [T].  Output rows, in the
// reference's order: for every t the original transition (s = obs_t || goal_t, s' = obs_next_t || goal_t), directly
// followed -- where select[t] != 0 -- by its relabelled copy with the achieved goal of step future[t] >= t as the goal,
// reward = -(||ag_next_t - goal'||_2 > threshold) (the sparse gym-robotics compute_reward, f64, sqrt of the
// left-to-right sum of squares like np.linalg.norm(axis=-1)) and done = (reward == 0).  select / future are the
// caller's random draws (np.random.uniform() < her_ratio, np.random.randint(t, T): main.py:166,170), `dst_row[t]` the
// exclusive prefix count of output rows.  The reference stores the relabelled copy with the LAST action of the rollout
// (`action`, main.py:184, not the step's own `a`): her_action_mode 0 reproduces that, 1 uses a_t.
struct HerArgs {
  const float* obs; const float* obs_next; const double* goal; const double* ag_next; const float* act;
  const double* rew; const uint8_t* done; const uint8_t* select; const int32_t* future; const int32_t* dst_row;
  int T, So, G, A, action_mode; double threshold;
  float* o_s; float* o_a; double* o_r; float* o_s2; uint8_t* o_d;
};
// The relabelled copy's reward: -(||ag[t] - ag[f]||_2 > a.threshold) in f64, ag the achieved goals [*, a.G] of an
// episode (ag[t] after the step, ag[f] after its future step: the new goal), the sum of squares left to right.
// her_relabel_kernel (HerArgs) and the streaming relabel (replay_add_goal_steps_kernel, GoalArgs) both call it.
template <class Args>
__device__ __forceinline__ double her_reward(const Args& a, const double* ag, int t, int f) {
  double ss = 0.0;
  for (int j = 0; j < a.G; ++j) {
    const double d = __dsub_rn(ag[size_t(t) * a.G + j], ag[size_t(f) * a.G + j]);
    ss = __dadd_rn(ss, __dmul_rn(d, d));
  }
  return (__dsqrt_rn(ss) > a.threshold) ? -1.0 : -0.0;     // -(d > threshold), as gym-robotics returns it
}
__global__ void her_relabel_kernel(const HerArgs a) {
  const int t = blockIdx.x;
  if (t >= a.T) return;
  const int S = a.So + a.G, row = a.dst_row[t];
  const bool sel = a.select[t] != 0;
  const int f = sel ? a.future[t] : t;
  for (int j = threadIdx.x; j < S; j += blockDim.x) {
    const bool is_obs = j < a.So;
    const float so = is_obs ? a.obs[size_t(t) * a.So + j] : float(a.goal[size_t(t) * a.G + (j - a.So)]);
    const float sn = is_obs ? a.obs_next[size_t(t) * a.So + j] : so;
    a.o_s[size_t(row) * S + j] = so;
    a.o_s2[size_t(row) * S + j] = sn;
    if (sel) {
      const float g2 = is_obs ? 0.f : float(a.ag_next[size_t(f) * a.G + (j - a.So)]);
      a.o_s[size_t(row + 1) * S + j] = is_obs ? so : g2;
      a.o_s2[size_t(row + 1) * S + j] = is_obs ? sn : g2;
    }
  }
  for (int j = threadIdx.x; j < a.A; j += blockDim.x) {
    a.o_a[size_t(row) * a.A + j] = a.act[size_t(t) * a.A + j];
    if (sel) a.o_a[size_t(row + 1) * a.A + j] = a.act[size_t(a.action_mode ? t : a.T - 1) * a.A + j];
  }
  if (threadIdx.x == 0) {
    a.o_r[row] = a.rew[t];
    a.o_d[row] = a.done[t];
    if (sel) {
      const double r = her_reward(a, a.ag_next, t, f);
      a.o_r[row + 1] = r;
      a.o_d[row + 1] = (r == 0.0) ? 1 : 0;
    }
  }
}

extern "C" int32_t d4pg_her_relabel(int32_t T, int32_t obs_dim, int32_t goal_dim, int32_t act_dim,
                                    const float* obs, const float* obs_next, const double* goal, const double* ag_next,
                                    const float* act, const double* rew, const uint8_t* done,
                                    const uint8_t* select, const int32_t* future, const int32_t* dst_row,
                                    double threshold, int32_t her_action_mode,
                                    float* out_s, float* out_a, double* out_r, float* out_s2, uint8_t* out_d,
                                    d4pg_stream_t stream) {
  D4PG_REQUIRE(T > 0 && obs_dim > 0 && goal_dim > 0 && act_dim > 0 && obs && obs_next && goal && ag_next && act && rew && done &&
               select && future && dst_row && out_s && out_a && out_r && out_s2 && out_d, D4PG_EINVAL, "d4pg_her_relabel: bad arguments");
  HerArgs a{obs, obs_next, goal, ag_next, act, rew, done, select, future, dst_row, T, obs_dim, goal_dim, act_dim,
            her_action_mode ? 1 : 0, threshold, out_s, out_a, out_r, out_s2, out_d};
  her_relabel_kernel<<<T, 64, 0, as_stream(stream)>>>(a);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

extern "C" int32_t d4pg_replay_add_host(d4pg_replay_t* h, int64_t n, const float* obs, const float* act, const double* rew,
                                        const float* obs2, const uint8_t* done, int32_t prioritized, d4pg_stream_t stream) {
  if (h) ++h->gen;
  D4PG_REQUIRE(h && obs && act && rew && obs2 && done && n > 0, D4PG_EINVAL, "d4pg_replay_add_host: null/empty argument");
  D4PG_REQUIRE(h->stage_host, D4PG_ESTATE, "d4pg_replay_add_host: call d4pg_replay_set_staging first");
  const PackLayout p = pack_layout(h, n);
  D4PG_REQUIRE(p.total <= h->stage_bytes, D4PG_EINVAL, "d4pg_replay_add_host: %lld rows do not fit the staging buffer", (long long)n);
  const int slot = h->stage_slot; h->stage_slot ^= 1;
  if (h->stage_busy[slot]) D4PG_CUDA_OK(cudaEventSynchronize(h->stage_ev[slot]));   // the add that used this slot has consumed it
  uint8_t* hp = h->stage_host + size_t(slot) * h->stage_bytes;
  uint8_t* d = h->stage_dev + size_t(slot) * h->stage_bytes;
  memcpy(hp + p.obs, obs, size_t(n) * h->obs_dim * 4);
  memcpy(hp + p.obs2, obs2, size_t(n) * h->obs_dim * 4);
  memcpy(hp + p.act, act, size_t(n) * h->act_dim * 4);
  memcpy(hp + p.rew, rew, size_t(n) * 8);
  memcpy(hp + p.done, done, size_t(n));
  cudaStream_t st = as_stream(stream);
  D4PG_CUDA_OK(cudaMemcpyAsync(d, hp, size_t(p.total), cudaMemcpyHostToDevice, st));   // ahead of the ingest gate
  int rc = d4pg_replay_add(h, n, reinterpret_cast<const float*>(d + p.obs), reinterpret_cast<const float*>(d + p.act),
                           reinterpret_cast<const double*>(d + p.rew), reinterpret_cast<const float*>(d + p.obs2),
                           d + p.done, prioritized, stream);
  D4PG_CUDA_OK(cudaEventRecord(h->stage_ev[slot], st));               // device slot read by the ring write
  h->stage_busy[slot] = true;
  return rc;
}

// ---- ingest gate + stream ordering (learner host pipeline, learner.cu) ------------------------------------------
namespace d4pg {
__global__ void gate_wait_kernel(const unsigned long long* flag, unsigned long long target, unsigned long long* trace) {
  unsigned long long v;
  step_stamp(trace, 10);
  do { asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(flag) : "memory"); } while (v < target);
  step_stamp(trace, 10 + 16);
}
__global__ void gate_signal_kernel(unsigned long long* flag) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(flag) : "memory");
  asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(flag), "l"(v + 1) : "memory");
}
unsigned long long* replay_gate_flag(d4pg_replay* h) {
  if (!h->gate_flag) {
    if (cudaMalloc(reinterpret_cast<void**>(&h->gate_flag), 16) != cudaSuccess || cudaMemset(h->gate_flag, 0, 16) != cudaSuccess) return nullptr;
  }
  return h->gate_flag;
}
void replay_arm_gate(d4pg_replay* h) { ++h->gate_target; h->gate_pending = true; }
int replay_gate_consume(d4pg_replay* h, cudaStream_t st) {
  if (!h->gate_pending) return D4PG_OK;
  gate_wait_kernel<<<1, 1, 0, st>>>(h->gate_flag, h->gate_target, step_trace());
  D4PG_LAUNCH_OK();
  h->gate_pending = false;
  return D4PG_OK;
}
int launch_gate_signal(unsigned long long* flag, cudaStream_t st) {
  gate_signal_kernel<<<1, 1, 0, st>>>(flag);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}
}  // namespace d4pg

extern "C" int32_t d4pg_replay_order_after(d4pg_replay_t* h, d4pg_stream_t first, d4pg_stream_t then) {
  D4PG_REQUIRE(h, D4PG_EINVAL, "d4pg_replay_order_after: null handle");
  if (as_stream(first) == as_stream(then)) return D4PG_OK;
  if (!h->order_ev) D4PG_CUDA_OK(cudaEventCreateWithFlags(&h->order_ev, cudaEventDisableTiming));
  D4PG_CUDA_OK(cudaEventRecord(h->order_ev, as_stream(first)));
  D4PG_CUDA_OK(cudaStreamWaitEvent(as_stream(then), h->order_ev, 0));
  return D4PG_OK;
}
extern "C" int64_t d4pg_replay_len(const d4pg_replay_t* h) { return h ? h->len : -1; }
extern "C" int64_t d4pg_replay_next_idx(const d4pg_replay_t* h) { return h ? h->next_idx : -1; }

extern "C" int32_t d4pg_replay_set_len(d4pg_replay_t* h, int64_t len, int64_t next_idx, int32_t pristine, d4pg_stream_t stream) {
  if (h) ++h->gen;
  D4PG_REQUIRE(h && len >= 0 && len <= h->size && next_idx >= 0 && next_idx < h->size, D4PG_EINVAL,
               "d4pg_replay_set_len: out of range");
  h->len = len; h->next_idx = next_idx; h->pristine = pristine ? 1 : 0;
  state_set_kernel<<<1, 1, 0, as_stream(stream)>>>(reinterpret_cast<ReplayState*>(h->state), len, next_idx, h->pristine);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

extern "C" int32_t d4pg_replay_set_obs_norm(d4pg_replay_t* h, double* stats, float* affine, double clip, double eps,
                                           d4pg_stream_t stream) {
  if (h) ++h->gen;
  D4PG_REQUIRE(h, D4PG_EINVAL, "d4pg_replay_set_obs_norm: null handle");
  if (!stats) {
    h->norm_stats = nullptr; h->norm_affine = nullptr;
    return D4PG_OK;
  }
  D4PG_REQUIRE(affine, D4PG_EINVAL, "d4pg_replay_set_obs_norm: null affine buffer");
  D4PG_REQUIRE(std::isfinite(clip) && clip > 0.0, D4PG_EINVAL, "d4pg_replay_set_obs_norm: clip must be finite and > 0 (got %g)", clip);
  D4PG_REQUIRE(std::isfinite(eps) && eps > 0.0, D4PG_EINVAL, "d4pg_replay_set_obs_norm: eps must be finite and > 0 (got %g)", eps);
  int rc = launch_obs_norm_reset(stats, affine, h->obs_dim, as_stream(stream));
  if (rc) return rc;
  h->norm_stats = stats; h->norm_affine = affine; h->norm_clip = clip; h->norm_eps = eps;
  return D4PG_OK;
}

extern "C" int32_t d4pg_replay_obs_norm_refresh(d4pg_replay_t* h, d4pg_stream_t stream) {
  if (h) ++h->gen;
  D4PG_REQUIRE(h, D4PG_EINVAL, "d4pg_replay_obs_norm_refresh: null handle");
  D4PG_REQUIRE(h->norm_stats, D4PG_ESTATE, "d4pg_replay_obs_norm_refresh: no observation normalizer registered");
  return launch_obs_stats(h->norm_stats, h->norm_affine, h->obs_dim, nullptr, 0, h->obs_dim, h->norm_eps, as_stream(stream));
}

namespace {
// The ring slots of an insert of n rows, [start, start + n) (mod size) from next_idx, and len / next_idx after it; an
// insert of no row leaves len as it is
struct RingRange { int64_t start, new_len, new_next; };
RingRange ring_range(const d4pg_replay* h, int64_t n) {
  const int64_t start = h->next_idx;
  return {start, n ? std::min<int64_t>(h->size, std::max<int64_t>(h->len, start + n)) : h->len, (start + n) % h->size};
}

// What every insert runs after its ring write of n rows at r: the normalizer's fold over the same rows in insertion
// order (rows1 [n1, obs_dim], then rows2 [n - n1, obs_dim]), then, prioritized, the ingest gate and the tree add of the
// new leaves; last, the host mirror of len / next_idx.
int replay_insert_tail(d4pg_replay* h, int64_t n, const RingRange& r, const float* rows1, int64_t n1, const float* rows2,
                       int32_t prioritized, cudaStream_t st) {
  const int64_t start = r.start;
  if (h->norm_stats) {
    // the normalizer's statistics: the same rows, in the same order.  Before the ingest gate and the tree kernels, so
    // the host pipeline's tree add stays the kernel the presample is programmatically dependent on
    int nrc = launch_obs_stats(h->norm_stats, h->norm_affine, h->obs_dim, rows1, n1, h->obs_dim, h->norm_eps, st);
    if (nrc) return nrc;
    if (n1 < n) {
      nrc = launch_obs_stats(h->norm_stats, h->norm_affine, h->obs_dim, rows2, n - n1, h->obs_dim, h->norm_eps, st);
      if (nrc) return nrc;
    }
  }
  if (prioritized) {
    // ingest gate (host pipeline): the rows above only had to follow the previous gather (stream order); the trees wait for
    // the last launched learner step's priority write-back -- inside the first tree kernel when that is the 1-CTA fast one
    const int64_t n1g = std::min<int64_t>(n, h->size - start);
    const unsigned long long* gflag = nullptr; unsigned long long gtarget = 0;
    if (h->gate_pending && n <= 65536 && n1g <= TREE_ADD_FAST_MAX && h->log2cap < 32) {
      gflag = h->gate_flag; gtarget = h->gate_target; h->gate_pending = false;
    } else {
      int grc = replay_gate_consume(h, st); if (grc) return grc;
    }
    if (n <= 65536) {
      // split a wrapping add into its two contiguous pieces
      const int64_t n1 = std::min<int64_t>(n, h->size - start);
      auto add_range = [&](int64_t s0, int64_t cnt) {
        if (cnt <= TREE_ADD_FAST_MAX && h->log2cap < 32) {
          tree_add_range_fast_kernel<<<1, TREE_THREADS, 0, st>>>(h->sum, h->mn, h->cap, h->log2cap, s0, cnt,
                                                                 reinterpret_cast<const ReplayState*>(h->state), h->alpha_f32, step_trace(),
                                                                 gflag, gtarget);
          gflag = nullptr;
        }
        else
          tree_add_range_kernel<<<1, TREE_THREADS, 0, st>>>(h->sum, h->mn, h->cap, h->log2cap, s0, cnt,
                                                            reinterpret_cast<const ReplayState*>(h->state), h->alpha_f32);
      };
      add_range(start, n1);
      D4PG_LAUNCH_OK();
      if (n1 < n) {
        add_range(0, n - n1);
        D4PG_LAUNCH_OK();
      }
    } else {
      leaf_fill_kernel<<<2 * device_sm_count(), 256, 0, st>>>(h->sum, h->mn, h->cap, h->size, start, n,
                                            reinterpret_cast<const ReplayState*>(h->state), h->alpha_f32);
      D4PG_LAUNCH_OK();
      for (int64_t c = h->cap / 2; c >= 1; c /= 2) {
        const int b = int(std::min<int64_t>(2 * device_sm_count(), (c + 255) / 256));
        level_rebuild_kernel<<<b, 256, 0, st>>>(h->sum, h->mn, c, c);
        D4PG_LAUNCH_OK();
      }
    }
  }
  h->len = r.new_len;
  h->next_idx = r.new_next;
  return D4PG_OK;
}

// The insert tail of a kernel that wrote its n rows straight into the ring: the rows are read back from the ring in
// insertion order, [start, size) then [0, ...).  A call that inserted no row has no tail.
int ring_rows_insert_tail(d4pg_replay* h, int64_t n, const RingRange& r, int32_t prioritized, cudaStream_t st) {
  if (n == 0) return D4PG_OK;
  const int64_t n1 = std::min<int64_t>(n, h->size - r.start);
  return replay_insert_tail(h, n, r, h->obs + r.start * h->obs_dim, n1, h->obs, prioritized, st);
}

struct StepsLayout { int64_t rec, wr, ws, wa, wo, total; };
StepsLayout steps_layout(int64_t E, int64_t S, int64_t A, int64_t n, bool tails) {
  StepsLayout l;
  l.rec = 0;
  l.wr = up16(l.rec + E * 8);
  l.ws = up16(l.wr + E * 2 * n * 8);
  l.wa = up16(l.ws + E * n * S * 4);
  l.wo = up16(l.wa + E * n * A * 4);
  l.total = up16(l.wo + (tails ? E * S * 4 : 0));
  return l;
}

// Every insert path but the episode-tails add_steps stores rows of horizon 0: clear the column over [start, start + n)
// (mod size), on the stream of the insert's ring write, so a slot that held a tail row does not keep its horizon
int zero_horizons(d4pg_replay* h, int64_t start, int64_t n, cudaStream_t st) {
  if (!h->horizon || n == 0) return D4PG_OK;
  const int64_t n1 = std::min<int64_t>(n, h->size - start);
  D4PG_CUDA_OK(cudaMemsetAsync(h->horizon + start, 0, size_t(n1), st));
  if (n1 < n) D4PG_CUDA_OK(cudaMemsetAsync(h->horizon, 0, size_t(n - n1), st));
  return D4PG_OK;
}
}  // namespace

extern "C" int32_t d4pg_replay_add(d4pg_replay_t* h, int64_t n, const float* obs, const float* act,
                                   const double* rew, const float* obs2, const uint8_t* done,
                                   int32_t prioritized, d4pg_stream_t stream) {
  if (h) ++h->gen;
  D4PG_REQUIRE(h && obs && act && rew && obs2 && done, D4PG_EINVAL, "d4pg_replay_add: null argument");
  D4PG_REQUIRE(n > 0 && n <= h->size, D4PG_EINVAL, "d4pg_replay_add: need 0 < n <= size (n=%lld)", (long long)n);
  cudaStream_t st = as_stream(stream);
  const RingRange r = ring_range(h, n);
  const int blocks = int(std::min<int64_t>(4 * device_sm_count(), (n * h->obs_dim + 255) / 256));   // grid-stride
  if (int rc = zero_horizons(h, r.start, n, st)) return rc;
  ring_write_kernel<<<blocks, 256, 0, st>>>(h->obs, h->act, h->rew, h->obs2, h->done, obs, act, rew, obs2, done,
                                             n, h->obs_dim, h->act_dim, h->size, r.start,
                                             reinterpret_cast<ReplayState*>(h->state), r.new_len, r.new_next, step_trace());
  D4PG_LAUNCH_OK();
  return replay_insert_tail(h, n, r, obs, n, nullptr, prioritized, st);
}

extern "C" int64_t d4pg_replay_steps_window_bytes(int64_t E, int32_t obs_dim, int32_t act_dim, int32_t n_steps) {
  return d4pg_replay_steps_window_bytes_ex(E, obs_dim, act_dim, n_steps, 0);
}

extern "C" int64_t d4pg_replay_steps_window_bytes_ex(int64_t E, int32_t obs_dim, int32_t act_dim, int32_t n_steps, int32_t tails) {
  if (E <= 0 || obs_dim <= 0 || act_dim <= 0 || n_steps < 1 || n_steps > D4PG_STEPS_MAX_N || (tails != 0 && tails != 1)) return -1;
  return steps_layout(E, obs_dim, act_dim, n_steps, tails != 0).total;
}

extern "C" int32_t d4pg_replay_set_horizons(d4pg_replay_t* h, uint8_t* horizon, d4pg_stream_t stream) {
  if (h) ++h->gen;
  D4PG_REQUIRE(h, D4PG_EINVAL, "d4pg_replay_set_horizons: null handle");
  if (horizon) D4PG_CUDA_OK(cudaMemsetAsync(horizon, 0, size_t(h->size), as_stream(stream)));
  h->horizon = horizon;
  return D4PG_OK;
}

extern "C" int32_t d4pg_replay_add_steps(d4pg_replay_t* h, int64_t E, const float* obs, const float* act, const double* rew,
                                         const float* obs2, const uint8_t* terminated, const uint8_t* episode_end,
                                         int32_t n_steps, double gamma, void* window, int64_t n_rows, int32_t prioritized,
                                         d4pg_stream_t stream) {
  return d4pg_replay_add_steps_ex(h, E, obs, act, rew, obs2, terminated, episode_end, n_steps, gamma, window, n_rows, 0,
                                  prioritized, stream);
}

extern "C" int32_t d4pg_replay_add_steps_ex(d4pg_replay_t* h, int64_t E, const float* obs, const float* act, const double* rew,
                                            const float* obs2, const uint8_t* terminated, const uint8_t* episode_end,
                                            int32_t n_steps, double gamma, void* window, int64_t n_rows, int32_t tails,
                                            int32_t prioritized, d4pg_stream_t stream) {
  if (h && n_rows > 0) ++h->gen;          // a call that inserts no row leaves the store, and a prefetched batch, valid
  D4PG_REQUIRE(h && obs && act && rew && obs2 && terminated && window, D4PG_EINVAL, "d4pg_replay_add_steps: null argument");
  D4PG_REQUIRE(E > 0 && E <= h->size, D4PG_EINVAL, "d4pg_replay_add_steps: need 0 < E <= size (E=%lld)", (long long)E);
  D4PG_REQUIRE(n_steps >= 1 && n_steps <= D4PG_STEPS_MAX_N, D4PG_EINVAL, "d4pg_replay_add_steps: need 1 <= n_steps <= %d (got %d)",
               D4PG_STEPS_MAX_N, n_steps);
  D4PG_REQUIRE(tails == 0 || tails == 1, D4PG_EINVAL, "d4pg_replay_add_steps: tails must be 0 or 1 (got %d)", tails);
  D4PG_REQUIRE(!tails || h->horizon, D4PG_ESTATE, "d4pg_replay_add_steps: episode tails need a horizon column (d4pg_replay_set_horizons)");
  // with tails an environment emits up to n - 1 rows per call
  const int64_t max_rows = tails ? E * std::max(1, n_steps - 1) : E;
  D4PG_REQUIRE(n_rows >= 0 && n_rows <= max_rows && n_rows <= h->size, D4PG_EINVAL,
               "d4pg_replay_add_steps: need 0 <= n_rows <= %s (%lld) and <= size (n_rows=%lld)",
               tails ? "E * max(1, n_steps - 1)" : "E", (long long)max_rows, (long long)n_rows);
  cudaStream_t st = as_stream(stream);
  const RingRange r = ring_range(h, n_rows);
  const StepsLayout l = steps_layout(E, h->obs_dim, h->act_dim, n_steps, tails != 0);
  uint8_t* wb = static_cast<uint8_t*>(window);
  StepsArgs a{};
  a.obs = obs; a.act = act; a.rew = rew; a.obs2 = obs2; a.term = terminated; a.end = episode_end;
  a.E = E; a.S = h->obs_dim; a.A = h->act_dim; a.n = n_steps; a.gamma = gamma;
  a.rec = reinterpret_cast<unsigned long long*>(wb + l.rec); a.wr = reinterpret_cast<double*>(wb + l.wr);
  a.ws = reinterpret_cast<float*>(wb + l.ws); a.wa = reinterpret_cast<float*>(wb + l.wa);
  a.r_obs = h->obs; a.r_act = h->act; a.r_rew = h->rew; a.r_obs2 = h->obs2; a.r_done = h->done;
  if (tails) { a.wo = reinterpret_cast<float*>(wb + l.wo); a.r_hz = h->horizon; }
  a.size = h->size; a.start = r.start; a.n_rows = n_rows; a.new_len = r.new_len; a.new_next = r.new_next;
  a.state = reinterpret_cast<ReplayState*>(h->state);
  // a CTA takes a contiguous chunk of environments, one warp per environment; the grid is at most 4 CTAs per SM
  const int64_t blocks = std::min<int64_t>((E + STEPS_WARPS - 1) / STEPS_WARPS, 4 * device_sm_count());
  a.chunk = (E + blocks - 1) / blocks;
  if (tails) replay_add_steps_kernel<true><<<unsigned((E + a.chunk - 1) / a.chunk), STEPS_THREADS, 0, st>>>(a);
  else {
    if (int rc = zero_horizons(h, r.start, n_rows, st)) return rc;
    replay_add_steps_kernel<false><<<unsigned((E + a.chunk - 1) / a.chunk), STEPS_THREADS, 0, st>>>(a);
  }
  D4PG_LAUNCH_OK();
  return ring_rows_insert_tail(h, n_rows, r, prioritized, st);
}

// ---- device-side ingest: streaming hindsight relabelling (DESIGN.md §3 "Streaming hindsight relabelling") ----------
// One call = one vector step of E goal-conditioned environments.  Environment e appends step t of its current episode
// to its window; an episode that ended at the previous call (its record's end bit) is emitted first, then the window
// restarts with this call's step.  One warp per environment does both, in that order, so the step that starts the new
// episode overwrites slot 0 only after every lane has read the emitted episode (a __syncwarp between them): one
// episode slot per environment is enough, and the emitted rows need no second launch.
//
// Window (caller-owned, zero-filled before the first call; d4pg_replay_goal_window_bytes), M = max_episode_steps:
//   rec u32 [E]        bits 0-30: steps of the current episode, bit 31: it ended at the last call
//   obs, obs2 f32 [E, M, So]   act f32 [E, M, A]   goal, ag f64 [E, M, G]   rew f64 [E, M]   term u8 [E, M]
// Plan (the host's draws, uploaded with one copy; NULL when no episode is emitted), i32:
//   step_off [E]       first draw of e's emitted episode (read only for an environment that emits)
//   future [n_draws]   future step of the relabelled copy of (e, t), -1 = no copy
//   dst [n_draws]      rank of the original row of (e, t) in this call; its copy takes dst + 1
constexpr int GOAL_THREADS = 256, GOAL_WARPS = GOAL_THREADS / 32;
struct GoalArgs {
  const float* obs; const double* goal; const float* act; const double* rew; const float* obs2; const double* ag2;
  const uint8_t* term; const uint8_t* end;
  int64_t E; int So, G, A, M, action_mode, no_step; double threshold;
  uint32_t* rec; float* w_obs; float* w_obs2; float* w_act; double* w_goal; double* w_ag; double* w_rew; uint8_t* w_term;
  const int32_t* step_off; const int32_t* future; const int32_t* dst; int64_t n_draws;
  float* r_obs; float* r_act; double* r_rew; float* r_obs2; uint8_t* r_done;
  int64_t size, start, n_rows, new_len, new_next; ReplayState* state;
};

__global__ void __launch_bounds__(GOAL_THREADS) replay_add_goal_steps_kernel(const GoalArgs a) {
  const int lane = threadIdx.x & 31, So = a.So, G = a.G, A = a.A, M = a.M, S = So + G;
  const int64_t e = int64_t(blockIdx.x) * GOAL_WARPS + (threadIdx.x >> 5);
  if (blockIdx.x == 0 && threadIdx.x == 0) { a.state->len = a.new_len; a.state->next_idx = a.new_next; }
  if (e >= a.E) return;
  const uint32_t rc = a.rec[e];
  const bool ended = (rc >> 31) != 0;
  int fill = int(rc & 0x7fffffffu);
  const int64_t w0 = e * M;                                   // window row of step 0
  if (ended && a.step_off) {
    // emit the ended episode of L steps: the original row of t at dst, its relabelled copy (if any) at dst + 1
    const int L = fill;
    const int64_t d0 = a.step_off[e];
    const float* last_act = a.w_act + (w0 + L - 1) * A;
    for (int t = 0; t < L && d0 + t < a.n_draws; ++t) {
      const int64_t rank = a.dst[d0 + t];
      const int f = a.future[d0 + t];
      const float* so = a.w_obs + (w0 + t) * So;
      const float* sn = a.w_obs2 + (w0 + t) * So;
      const float* at = a.w_act + (w0 + t) * A;
      if (rank < a.n_rows) {                                  // never outside [start, start + n_rows)
        int64_t p = a.start + rank;                            // start < size and rank < n_rows <= size
        if (p >= a.size) p -= a.size;
        const double* g = a.w_goal + (w0 + t) * G;
        for (int j = lane; j < So; j += 32) { a.r_obs[p * S + j] = so[j]; a.r_obs2[p * S + j] = sn[j]; }
        for (int j = lane; j < G; j += 32) { const float v = float(g[j]); a.r_obs[p * S + So + j] = v; a.r_obs2[p * S + So + j] = v; }
        for (int j = lane; j < A; j += 32) a.r_act[p * A + j] = at[j];
        if (lane == 0) { a.r_rew[p] = a.w_rew[w0 + t]; a.r_done[p] = a.w_term[w0 + t]; }
      }
      if (f >= t && f < L && rank + 1 < a.n_rows) {
        int64_t q = a.start + rank + 1;
        if (q >= a.size) q -= a.size;
        const double* g2 = a.w_ag + (w0 + f) * G;             // goal' = the achieved goal after step f
        const float* ac = a.action_mode ? at : last_act;
        for (int j = lane; j < So; j += 32) { a.r_obs[q * S + j] = so[j]; a.r_obs2[q * S + j] = sn[j]; }
        for (int j = lane; j < G; j += 32) { const float v = float(g2[j]); a.r_obs[q * S + So + j] = v; a.r_obs2[q * S + So + j] = v; }
        for (int j = lane; j < A; j += 32) a.r_act[q * A + j] = ac[j];
        if (lane == 0) {
          const double r = her_reward(a, a.w_ag, int(w0 + t), int(w0 + f));   // E * M < size
          a.r_rew[q] = r;
          a.r_done[q] = (r == 0.0) ? 1 : 0;
        }
      }
    }
  }
  if (ended) fill = 0;
  __syncwarp();                                               // every lane has read the record and the emitted episode
  if (a.no_step) {                                            // flush: emit only; running episodes keep their windows
    if (ended && lane == 0) a.rec[e] = 0u;
    return;
  }
  const int slot = fill;
  if (slot < M) {                                             // the host never lets an episode outgrow its window
    const int64_t w = w0 + slot;
    for (int j = lane; j < So; j += 32) { a.w_obs[w * So + j] = a.obs[e * So + j]; a.w_obs2[w * So + j] = a.obs2[e * So + j]; }
    for (int j = lane; j < G; j += 32) { a.w_goal[w * G + j] = a.goal[e * G + j]; a.w_ag[w * G + j] = a.ag2[e * G + j]; }
    for (int j = lane; j < A; j += 32) a.w_act[w * A + j] = a.act[e * A + j];
  }
  if (lane == 0) {
    const bool term = a.term[e] != 0, end_now = term || (a.end && a.end[e] != 0);
    if (slot < M) { a.w_rew[w0 + slot] = a.rew[e]; a.w_term[w0 + slot] = term ? 1 : 0; }
    a.rec[e] = uint32_t(min(slot + 1, M)) | (end_now ? 0x80000000u : 0u);
  }
}

namespace {
struct GoalLayout { int64_t rec, obs, obs2, act, goal, ag, rew, term, total; };
GoalLayout goal_layout(int64_t E, int64_t So, int64_t G, int64_t A, int64_t M) {
  GoalLayout l;
  l.rec = 0;
  l.obs = up16(l.rec + E * 4);
  l.obs2 = up16(l.obs + E * M * So * 4);
  l.act = up16(l.obs2 + E * M * So * 4);
  l.goal = up16(l.act + E * M * A * 4);
  l.ag = up16(l.goal + E * M * G * 8);
  l.rew = up16(l.ag + E * M * G * 8);
  l.term = up16(l.rew + E * M * 8);
  l.total = up16(l.term + E * M);
  return l;
}
}  // namespace

extern "C" int64_t d4pg_replay_goal_window_bytes(int64_t E, int32_t obs_dim, int32_t goal_dim, int32_t act_dim,
                                                 int32_t max_episode_steps) {
  if (E <= 0 || obs_dim <= 0 || goal_dim <= 0 || act_dim <= 0 || max_episode_steps < 1 ||
      max_episode_steps > D4PG_GOAL_MAX_STEPS) return -1;
  return goal_layout(E, obs_dim, goal_dim, act_dim, max_episode_steps).total;
}

extern "C" int32_t d4pg_replay_add_goal_steps(d4pg_replay_t* h, int64_t E, int32_t obs_dim, int32_t goal_dim,
                                              const float* obs, const double* goal, const float* act, const double* rew,
                                              const float* obs2, const double* ag2, const uint8_t* terminated,
                                              const uint8_t* episode_end, int32_t max_episode_steps, void* window,
                                              const int32_t* plan, int64_t n_draws, int64_t n_rows, double threshold,
                                              int32_t her_action_mode, int32_t no_step, int32_t prioritized,
                                              d4pg_stream_t stream) {
  if (h && n_rows > 0) ++h->gen;          // a call that inserts no row leaves the store, and a prefetched batch, valid
  D4PG_REQUIRE(h && window, D4PG_EINVAL, "d4pg_replay_add_goal_steps: null argument");
  D4PG_REQUIRE(no_step == 0 || no_step == 1, D4PG_EINVAL, "d4pg_replay_add_goal_steps: no_step must be 0 or 1 (got %d)", no_step);
  D4PG_REQUIRE(no_step || (obs && goal && act && rew && obs2 && ag2 && terminated), D4PG_EINVAL,
               "d4pg_replay_add_goal_steps: null step input");
  D4PG_REQUIRE(E > 0 && E <= h->size, D4PG_EINVAL, "d4pg_replay_add_goal_steps: need 0 < E <= size (E=%lld)", (long long)E);
  D4PG_REQUIRE(obs_dim > 0 && goal_dim > 0 && int64_t(obs_dim) + goal_dim == h->obs_dim, D4PG_EINVAL,
               "d4pg_replay_add_goal_steps: obs_dim + goal_dim must equal the replay's obs_dim %d (got %d + %d)",
               h->obs_dim, obs_dim, goal_dim);
  D4PG_REQUIRE(max_episode_steps >= 1 && max_episode_steps <= D4PG_GOAL_MAX_STEPS, D4PG_EINVAL,
               "d4pg_replay_add_goal_steps: need 1 <= max_episode_steps <= %d (got %d)", D4PG_GOAL_MAX_STEPS, max_episode_steps);
  D4PG_REQUIRE(std::isfinite(threshold) && threshold >= 0.0, D4PG_EINVAL,
               "d4pg_replay_add_goal_steps: threshold must be finite and >= 0 (got %g)", threshold);
  D4PG_REQUIRE(her_action_mode == 0 || her_action_mode == 1, D4PG_EINVAL,
               "d4pg_replay_add_goal_steps: her_action_mode must be 0 or 1 (got %d)", her_action_mode);
  const int64_t M = max_episode_steps;
  D4PG_REQUIRE(n_draws >= 0 && n_draws <= E * M && (n_draws == 0 || plan), D4PG_EINVAL,
               "d4pg_replay_add_goal_steps: need 0 <= n_draws <= E * max_episode_steps and a plan when n_draws > 0");
  D4PG_REQUIRE(n_rows >= 0 && n_rows <= 2 * n_draws && n_rows <= h->size, D4PG_EINVAL,
               "d4pg_replay_add_goal_steps: need 0 <= n_rows <= 2 * n_draws and <= size (n_rows=%lld)", (long long)n_rows);
  cudaStream_t st = as_stream(stream);
  const RingRange r = ring_range(h, n_rows);
  const GoalLayout l = goal_layout(E, obs_dim, goal_dim, h->act_dim, M);
  uint8_t* wb = static_cast<uint8_t*>(window);
  GoalArgs a{};
  a.obs = obs; a.goal = goal; a.act = act; a.rew = rew; a.obs2 = obs2; a.ag2 = ag2; a.term = terminated; a.end = episode_end;
  a.E = E; a.So = obs_dim; a.G = goal_dim; a.A = h->act_dim; a.M = max_episode_steps;
  a.action_mode = her_action_mode; a.no_step = no_step; a.threshold = threshold;
  a.rec = reinterpret_cast<uint32_t*>(wb + l.rec);
  a.w_obs = reinterpret_cast<float*>(wb + l.obs); a.w_obs2 = reinterpret_cast<float*>(wb + l.obs2);
  a.w_act = reinterpret_cast<float*>(wb + l.act); a.w_goal = reinterpret_cast<double*>(wb + l.goal);
  a.w_ag = reinterpret_cast<double*>(wb + l.ag); a.w_rew = reinterpret_cast<double*>(wb + l.rew); a.w_term = wb + l.term;
  if (n_draws > 0) { a.step_off = plan; a.future = plan + E; a.dst = plan + E + n_draws; }
  a.n_draws = n_draws;
  a.r_obs = h->obs; a.r_act = h->act; a.r_rew = h->rew; a.r_obs2 = h->obs2; a.r_done = h->done;
  a.size = h->size; a.start = r.start; a.n_rows = n_rows; a.new_len = r.new_len; a.new_next = r.new_next;
  a.state = reinterpret_cast<ReplayState*>(h->state);
  if (int rc = zero_horizons(h, r.start, n_rows, st)) return rc;
  replay_add_goal_steps_kernel<<<unsigned((E + GOAL_WARPS - 1) / GOAL_WARPS), GOAL_THREADS, 0, st>>>(a);
  D4PG_LAUNCH_OK();
  return ring_rows_insert_tail(h, n_rows, r, prioritized, st);
}

extern "C" int32_t d4pg_replay_sample(d4pg_replay_t* h, int32_t B, const double* uniforms,
                                      uint64_t philox_seed, uint64_t philox_counter, double beta,
                                      int32_t* idx, float* weights,
                                      float* s, float* a, double* r, float* s2, uint8_t* done,
                                      d4pg_stream_t stream) {
  D4PG_REQUIRE(h && B > 0 && idx && s && a && r && s2 && done, D4PG_EINVAL, "d4pg_replay_sample: null/empty argument");
  D4PG_REQUIRE(h->len >= 2, D4PG_ESTATE, "d4pg_replay_sample: needs at least 2 stored transitions (sum(0,len-1))");
  D4PG_REQUIRE(beta > 0, D4PG_EINVAL, "d4pg_replay_sample: beta must be > 0");                           // :299
  SampleArgs sa{};
  sa.uniforms = uniforms; sa.seed = philox_seed; sa.counter = philox_counter; sa.beta = float(beta);
  sa.B = B; sa.idx = idx; sa.weights = weights; sa.s = s; sa.a = a; sa.r = r; sa.s2 = s2; sa.d = done;
  return launch_sample(h, sa, as_stream(stream));
}

extern "C" int32_t d4pg_replay_gather(d4pg_replay_t* h, int32_t B, const int32_t* idx,
                                      float* s, float* a, double* r, float* s2, uint8_t* done, d4pg_stream_t stream) {
  D4PG_REQUIRE(h && B > 0 && idx && s && a && r && s2 && done, D4PG_EINVAL, "d4pg_replay_gather: null/empty argument");
  SampleArgs sa{};
  sa.B = B; sa.idx_in = idx; sa.s = s; sa.a = a; sa.r = r; sa.s2 = s2; sa.d = done;
  return launch_sample(h, sa, as_stream(stream));
}

extern "C" int32_t d4pg_replay_update_priorities(d4pg_replay_t* h, int32_t B, const int32_t* idx,
                                                 const float* prio, d4pg_stream_t stream) {
  if (h) ++h->gen;
  D4PG_REQUIRE(h && B > 0 && idx && prio, D4PG_EINVAL, "d4pg_replay_update_priorities: null/empty argument");
  return launch_tree_update(h, B, idx, prio, as_stream(stream));
}

extern "C" int32_t d4pg_replay_set_leaves(d4pg_replay_t* h, int32_t n, const int32_t* idx, const float* sum_vals,
                                          const float* min_vals, d4pg_stream_t stream) {
  if (h) ++h->gen;
  D4PG_REQUIRE(h && n > 0 && idx && sum_vals && min_vals, D4PG_EINVAL, "d4pg_replay_set_leaves: null/empty argument");
  TreeArgs a = tree_args(h, n, idx, sum_vals);
  a.v1 = min_vals;
  tree_write_kernel<TREE_SET><<<1, TREE_THREADS, 0, as_stream(stream)>>>(a);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

extern "C" int32_t d4pg_replay_reduce(d4pg_replay_t* h, int64_t start, int64_t end, float* out, d4pg_stream_t stream) {
  D4PG_REQUIRE(h && out, D4PG_EINVAL, "d4pg_replay_reduce: null argument");
  if (end <= 0) end += h->cap;                                        // :91-94 (None / negative end)
  D4PG_REQUIRE(start >= 0 && start < end && end <= h->cap, D4PG_EINVAL, "d4pg_replay_reduce: bad range [%lld,%lld)",
               (long long)start, (long long)end);
  reduce_kernel<<<1, 32, 0, as_stream(stream)>>>(h->sum, h->mn, h->cap, start, end - 1, out);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

extern "C" int32_t d4pg_replay_find_prefixsum(d4pg_replay_t* h, int32_t n, const double* masses, int32_t* idx,
                                              d4pg_stream_t stream) {
  D4PG_REQUIRE(h && n > 0 && masses && idx, D4PG_EINVAL, "d4pg_replay_find_prefixsum: null/empty argument");
  find_prefix_kernel<<<cdiv(n, 128), 128, 0, as_stream(stream)>>>(h->sum, h->cap, n, masses, idx);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}
