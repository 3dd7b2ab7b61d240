// Exploratory action selection: act_chain_kernel, its C ABI d4pg_act, and the row copy that lands observations in a
// 16-byte row pitch.  The kernel runs the actor on the building blocks of the fp32 cluster chain (mlp_chain_dev.cuh).
#include "mlp_chain_dev.cuh"
#include "obs_norm.cuh"
#include <algorithm>
#include <cmath>

namespace d4pg {

// Exploratory action selection (d4pg_act): the actor fc1 -> fc2 -> fc2_2 -> fc3 as a 4-slot chain of the fp32 tile in
// its own kernel.  Slot 0 fills from the observation rows (normalized there when `norm_affine` is set); fc3's tanh
// output gets the exploration noise and the clip (DESIGN §3 "Exploration") before it is stored to `action`.
constexpr int ACT_SLOTS = 4;
enum ActNoise { ACT_NOISE_NONE = 0, ACT_NOISE_GAUSSIAN = 1, ACT_NOISE_OU = 2 };
struct ActArgs {
  ChainSlot slot[ACT_SLOTS];      // slot 0 reads global rows (Ag / ldag), slot l > 0 the plane of slot l - 1
  int B, a_floats, w_floats;
  float* xchg;                    // [row_blocks][ACT_SLOTS - 1][CHAIN_PLANE]
  const float* norm_affine;       // {shift[K0], scale[K0]} or nullptr
  float norm_clip;
  int noise;                      // ActNoise
  double p[5];                    // gaussian {eps, mu, var}; OU {eps, theta, mu, sigma, dt}
  uint64_t seed, counter;         // Philox key / counter of this call's draws
  double* ou_state;               // [B][N3] (OU only)
  const uint8_t* reset;           // [B] or nullptr (OU only)
  float* action;                  // [B][N3]
};

// fill_from_rows<false> with the observation normalizer applied to the rows of the batch (obs_norm_apply, exactly the
// arithmetic of obs_normalize_kernel, so the A plane holds the values the level path's fc1 reads)
__device__ __forceinline__ void fill_from_rows_norm(float* As, const float* __restrict__ src, int ld, int m0, int B, int kn,
                                                    const float* __restrict__ affine, float clip, int tid) {
  const int nq = (kn + 3) >> 2;
  for (int e = tid; e < nq * CHAIN_ROWS; e += GEMM_THREADS) {
    const int row = e & 31, k = (e >> 5) << 2;
    const bool in = m0 + row < B;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (in) v = __ldg(reinterpret_cast<const float4*>(src + size_t(m0 + row) * ld + k));
    const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (k + c < kn)
        As[(k + c) * CHAIN_ROWS + row] = in ? obs_norm_apply(x[c], __ldg(affine + k + c), __ldg(affine + kn + k + c), clip) : 0.f;
  }
}

constexpr double ACT_TWO_PI = 2.0 * 3.14159265358979323846;     // == 2 * numpy.pi

// fc3's tile (tanh applied, k-major [j][32 rows] in shared memory) -> noise, clip, store.  Element i = row * N + j draws
// u1 = uniform53(seed, counter, 2i), u2 = uniform53(seed, counter, 2i + 1); z = sqrt(-2 log(1 - u1)) cos(2 pi u2) in
// fp64.  Every fp64 operation is rounded on its own (no contraction), in the reference's order (random_process.py).
__device__ __forceinline__ void act_epilogue(const ActArgs& a, const float* tile, int m0, int n0, int tid) {
  const int N = a.slot[ACT_SLOTS - 1].N;
  const int nc = min(BN, N - n0);
  for (int e = tid; e < CHAIN_ROWS * nc; e += GEMM_THREADS) {
    const int r = e / nc, j = n0 + (e - r * nc);          // neighbouring threads store neighbouring columns of a row
    const int gi = m0 + r;
    if (gi >= a.B) break;
    const float x = tile[j * CHAIN_ROWS + r];
    const size_t i = size_t(gi) * N + j;
    if (a.noise == ACT_NOISE_NONE) { a.action[i] = x; continue; }
    const double u1 = Philox::uniform53(a.seed, a.counter, uint32_t(2 * i));
    const double u2 = Philox::uniform53(a.seed, a.counter, uint32_t(2 * i + 1));
    const double z = __dmul_rn(__dsqrt_rn(__dmul_rn(-2.0, log(__dsub_rn(1.0, u1)))), cos(__dmul_rn(ACT_TWO_PI, u2)));
    double n;
    if (a.noise == ACT_NOISE_GAUSSIAN) {
      n = __dmul_rn(a.p[0], __dadd_rn(a.p[1], __dmul_rn(a.p[2], z)));                  // eps * (mu + var * z)
    } else {
      const double theta = a.p[1], mu = a.p[2], sigma = a.p[3], dt = a.p[4];
      double s = (a.reset && a.reset[gi]) ? 0.0 : a.ou_state[i];
      s = __dadd_rn(__dadd_rn(s, __dmul_rn(__dmul_rn(theta, __dsub_rn(mu, s)), dt)), __dmul_rn(__dmul_rn(sigma, __dsqrt_rn(dt)), z));
      a.ou_state[i] = s;
      n = __dmul_rn(a.p[0], s);                                                          // eps * x
    }
    a.action[i] = float(fmin(fmax(__dadd_rn(double(x), n), -1.0), 1.0));
  }
}

// The layers run mlp_chain_kernel<0>'s slot loop (FWD slots, no pre-layers): same fills, same chain_tile, same
// barriers, so without noise the action is bit-identical to d4pg_actor_forward at precision 0.  fc3's output tile goes
// to weight buffer 0, which is free in the last slot (its weights sit in buffer 1 and nothing is prefetched).
__global__ void __cluster_dims__(CHAIN_CLUSTER, 1, 1) __launch_bounds__(GEMM_THREADS, 2)
act_chain_kernel(const __grid_constant__ ActArgs args) {
  extern __shared__ __align__(16) float chain_smem[];
  float* As = chain_smem;
  float* W0 = chain_smem + args.a_floats;
  const int wf = args.w_floats;
  const int tid = threadIdx.x;
  const int rank = int(cluster_ctarank());
  const int rb_i = blockIdx.x / CHAIN_CLUSTER;
  const int m0 = rb_i * CHAIN_ROWS, B = args.B;
  float* planes = args.xchg + size_t(rb_i) * ((ACT_SLOTS - 1) * CHAIN_PLANE);
  const int n0 = rank * BN;

  if (n0 < args.slot[0].N) fetch_weights<false>(W0, args.slot[0], n0, tid);
  cp_async_commit();
  for (int l = 0; l < ACT_SLOTS; ++l) {
    const ChainSlot& S = args.slot[l];
    const bool has_tile = n0 < S.N;
    float eop[4] = {0.f, 0.f, 0.f, 0.f};
    if (has_tile) {
      const int gi = m0 + (tid >> 3);
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const int gj = n0 + (tid & 7) + 8 * cc;
        if (gj < S.N && gi < B) eop[cc] = __ldg(S.bias + gj);
      }
    }
    if (l > 0) cluster_wait();
    if (has_tile) {
      if (l > 0) fill_from_plane<false>(As, 0, planes + size_t(l - 1) * CHAIN_PLANE, S.K, tid);
      else if (args.norm_affine) fill_from_rows_norm(As, S.Ag, S.ldag, m0, B, S.K, args.norm_affine, args.norm_clip, tid);
      else fill_from_rows<false>(As, 0, S.Ag, S.ldag, m0, B, S.K, tid);
    }
    cp_async_commit();
    if (l + 1 < ACT_SLOTS && n0 < args.slot[l + 1].N) fetch_weights<false>(W0 + ((l + 1) & 1) * wf, args.slot[l + 1], n0, tid);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    if (has_tile) {
      const bool last = l == ACT_SLOTS - 1;
      chain_tile<GEMM_FWD>(tile_of(S), As, As, W0 + (l & 1) * wf, m0, n0, B, last ? nullptr : planes + size_t(l) * CHAIN_PLANE,
                           last ? W0 : nullptr, eop, nullptr);
    }
    if (l + 1 < ACT_SLOTS) cluster_arrive();
  }
  cp_async_wait<0>();
  if (n0 < args.slot[ACT_SLOTS - 1].N) {
    __syncthreads();                                  // the whole fc3 tile is in buffer 0
    act_epilogue(args, W0, m0, n0, tid);
  }
}

static int64_t act_xchg_floats(int B) { return int64_t(cdiv(B, CHAIN_ROWS)) * (ACT_SLOTS - 1) * CHAIN_PLANE; }

static int act_chain_prepare(ActArgs& a) {
  // chain_add's sizes: the A plane doubles as the reduce buffer; one weight-slice buffer per slot parity
  a.a_floats = GEMM_WARPS * BM * BN;
  a.w_floats = 0;
  for (int l = 0; l < ACT_SLOTS; ++l) {
    a.a_floats = std::max(a.a_floats, int(align4(int64_t(a.slot[l].K) * CHAIN_ROWS)));
    a.w_floats = std::max(a.w_floats, BN * chain_wpitch(a.slot[l].K));
  }
  const size_t smem = size_t(a.a_floats + 2 * a.w_floats) * sizeof(float);
  D4PG_REQUIRE(smem <= 220 * 1024, D4PG_ENOTSUP, "d4pg_act: obs_dim %d needs %zu B of shared memory (at most %d B: obs_dim <= 576)",
               a.slot[0].K, smem, 220 * 1024);
  return D4PG_OK;
}

static int launch_act_chain(ActArgs& a, cudaStream_t st) {
  int rc = act_chain_prepare(a);
  if (rc) return rc;
  const size_t smem = size_t(a.a_floats + 2 * a.w_floats) * sizeof(float);
  static size_t smem_set = 0;
  if (smem > smem_set) {
    D4PG_CUDA_OK(cudaFuncSetAttribute(act_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    D4PG_CUDA_OK(cudaFuncSetAttribute(act_chain_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, int(cudaSharedmemCarveoutMaxShared)));
    smem_set = smem;
  }
  act_chain_kernel<<<cdiv(a.B, CHAIN_ROWS) * CHAIN_CLUSTER, GEMM_THREADS, smem, st>>>(a);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

}  // namespace d4pg

using namespace d4pg;

extern "C" int64_t d4pg_act_workspace_floats(int32_t E, int32_t obs_dim) {
  if (E <= 0 || obs_dim <= 0) return -1;
  return act_xchg_floats(E);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int32_t d4pg_act(const float* actor_params, int32_t obs_dim, int32_t act_dim, const float* s, int64_t lds,
                            int32_t E, const float* norm_affine, double norm_clip, int32_t noise,
                            const double* noise_params, uint64_t seed, uint64_t counter, double* ou_state,
                            const uint8_t* reset, float* action, float* workspace, d4pg_stream_t stream) {
  D4PG_REQUIRE(actor_params && s && action && workspace, D4PG_EINVAL, "d4pg_act: null argument");
  D4PG_REQUIRE(aligned16(actor_params), D4PG_EINVAL, "d4pg_act: actor_params must be 16-B aligned");
  D4PG_REQUIRE(obs_dim > 0 && act_dim > 0 && act_dim <= D4PG_HIDDEN, D4PG_EINVAL,
               "d4pg_act: obs_dim %d / act_dim %d (1 <= act_dim <= %d)", obs_dim, act_dim, D4PG_HIDDEN);
  D4PG_REQUIRE(E >= 1 && 2 * int64_t(E) * act_dim < (int64_t(1) << 31), D4PG_EINVAL,
               "d4pg_act: E = %d rows (need E >= 1 and 2 * E * act_dim < 2^31)", E);
  D4PG_REQUIRE(lds >= obs_dim && lds % 4 == 0 && aligned16(s), D4PG_EINVAL,
               "d4pg_act: s needs a 16-B aligned base and a row pitch that is a multiple of 4 floats >= obs_dim (lds %lld)",
               (long long)lds);
  D4PG_REQUIRE(!norm_affine || (std::isfinite(norm_clip) && norm_clip > 0.0), D4PG_EINVAL,
               "d4pg_act: norm_clip must be finite and > 0 (got %g)", norm_clip);
  D4PG_REQUIRE(noise >= ACT_NOISE_NONE && noise <= ACT_NOISE_OU, D4PG_EINVAL, "d4pg_act: noise %d (0 none, 1 gaussian, 2 OU)", noise);
  const int np = noise == ACT_NOISE_GAUSSIAN ? 3 : noise == ACT_NOISE_OU ? 5 : 0;
  D4PG_REQUIRE(np == 0 || noise_params, D4PG_EINVAL, "d4pg_act: noise %d needs noise_params", noise);
  for (int k = 0; k < np; ++k)
    D4PG_REQUIRE(std::isfinite(noise_params[k]), D4PG_EINVAL, "d4pg_act: noise_params[%d] = %g is not finite", k, noise_params[k]);
  D4PG_REQUIRE(noise != ACT_NOISE_OU || (ou_state && noise_params[4] >= 0.0), D4PG_EINVAL,
               "d4pg_act: Ornstein-Uhlenbeck noise needs ou_state and dt >= 0");

  const NetDims d = actor_dims(obs_dim, act_dim);
  ActArgs a{};
  for (int l = 0; l < ACT_SLOTS; ++l) {
    a.slot[l] = chain_fwd(actor_params + d.w_off[l], d.ld[l], actor_params + d.b_off[l], d.out[l], d.in[l], d.epi[l],
                          nullptr, 0, l + 1 < ACT_SLOTS);
    if (l > 0) chain_src_plane(a.slot[l], l - 1);
  }
  chain_src_global(a.slot[0], s, int(lds));
  a.B = E;
  a.xchg = workspace;
  a.norm_affine = norm_affine;
  a.norm_clip = float(norm_clip);
  a.noise = noise;
  for (int k = 0; k < np; ++k) a.p[k] = noise_params[k];
  a.seed = seed; a.counter = counter;
  a.ou_state = noise == ACT_NOISE_OU ? ou_state : nullptr;
  a.reset = noise == ACT_NOISE_OU ? reset : nullptr;
  a.action = action;
  return launch_act_chain(a, as_stream(stream));
}

extern "C" int32_t d4pg_copy_rows_f32(float* dst, int64_t ldd, const float* src, int64_t lds, int64_t rows, int64_t width,
                                      d4pg_stream_t stream) {
  D4PG_REQUIRE(dst && src && rows > 0 && width > 0 && ldd >= width && lds >= width, D4PG_EINVAL,
               "d4pg_copy_rows_f32: bad arguments");
  D4PG_CUDA_OK(cudaMemcpy2DAsync(dst, size_t(ldd) * sizeof(float), src, size_t(lds) * sizeof(float), size_t(width) * sizeof(float),
                                 size_t(rows), cudaMemcpyDefault, as_stream(stream)));
  return D4PG_OK;
}
