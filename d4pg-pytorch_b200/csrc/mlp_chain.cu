// Cluster-fused MLP chains: every dependent layer of a network chain in ONE launch.
//
// At batch 256 the actor/critic passes of DDPG.train (models.py:32-41,76-88 forward, ddpg.py:230,242
// backward) are 14 dependent layer levels; as separate grouped-GEMM launches most of each level's time is
// the kernel boundary.  Here a thread-block CLUSTER of 8 CTAs owns
// 32 batch rows for a whole chain (e.g. actor_target fc1..fc3 -> critic_target fc1..fc3): CTA r of the
// cluster computes the 32-column slice r of each 256-wide layer, publishes it k-major into an
// L2-resident exchange plane, and a cluster barrier (barrier.cluster arrive.release / wait.acquire)
// replaces the kernel boundary.  The next layer's first weight chunk is prefetched between
// the arrive and the wait.  Rows never mix, so clusters are independent: no grid-wide barrier, no
// co-residency requirement beyond the cluster itself.
//
// Arithmetic is the SAME as gemm_tile (gemm_ffma_dev.cuh): 64-deep K chunks, the 8 warps split each
// chunk, 8x4 lane tiles, partial tiles reduced in warp order -> results are bit-identical to the
// level-by-level path (tests/test_gpu_learner.py::test_chain_equals_levels).
#include "gemm_ffma_dev.cuh"
#include "mlp_chain_dev.cuh"
#include <stdlib.h>
#include <algorithm>

namespace d4pg {

// One 32x32 tile of one slot with A and W resident for the whole K.  The order of the additions is
// gemm_tile's: within every 64-deep chunk warp w owns k = 8w..8w+7, partial tiles are summed w = 0..7.
// ---- tensor-core variant of the tile (PREC 1 = 3xTF32, fp32-accurate; PREC 2 = one TF32 pass) --------------------
// mma.sync.m16n8k8 (the warp-level MMA that exists for a 32-row tile; wgmma tiles start at 64 rows): the operand
// fragments cost 16 LDS.32 per 8-deep k-step instead of 96 LDS wavefronts for the FFMA lane tiles.
// 3xTF32: x = hi + lo with hi = tf32(x), lo = tf32(x - hi);  D += Al*Bh + Ah*Bl + Ah*Bh  (~2^-21 relative).
__device__ __forceinline__ void tf32_split(float x, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  const float r = x - __uint_as_float(hi);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
constexpr int CHAIN_RED_PITCH = 36;   // partial-tile pitch of the tensor-core path

template <int MODE, int PREC>
__device__ __forceinline__ void chain_tile_mma(const ChainSlot& S, float* As, const float* Ws, int m0, int n0, int B, float* xout,
                                               const float (&eop)[4], unsigned long long* tr) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int N = S.N, K = S.K;
  const int P = chain_wpitch(K);
  float acc[2][4][4];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int nn = 0; nn < 4; ++nn)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[m][nn][i] = 0.f;
  const int nks = (K + 7) >> 3;
  for (int ks = warp; ks < nks; ks += GEMM_WARPS) {           // the 8 warps interleave the 8-deep k-steps
    const int ka = ks * 8 + t4, kb = ka + 4;
    const bool va = ka < K, vb = kb < K;                     // operands past K are zero (rows of As / Ws there are stale)
    const int sw = t4 << 3;
    uint32_t ah[2][4], al[2][4], bh[4][2], bl[4][2];
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const int r0 = (m * 16 + g) ^ sw, r1 = (m * 16 + g + 8) ^ sw;      // ka & 3 == kb & 3 == t4
      const float x0 = va ? As[ka * CHAIN_ROWS + r0] : 0.f, x1 = va ? As[ka * CHAIN_ROWS + r1] : 0.f;
      const float x2 = vb ? As[kb * CHAIN_ROWS + r0] : 0.f, x3 = vb ? As[kb * CHAIN_ROWS + r1] : 0.f;
      tf32_split(x0, ah[m][0], al[m][0]); tf32_split(x1, ah[m][1], al[m][1]);
      tf32_split(x2, ah[m][2], al[m][2]); tf32_split(x3, ah[m][3], al[m][3]);
    }
#pragma unroll
    for (int nn = 0; nn < 4; ++nn) {
      float y0, y1;
      if (MODE == GEMM_FWD) { y0 = va ? Ws[(nn * 8 + g) * P + ka] : 0.f; y1 = vb ? Ws[(nn * 8 + g) * P + kb] : 0.f; }
      else { y0 = va ? Ws[ka * BN + ((nn * 8 + g) ^ sw)] : 0.f; y1 = vb ? Ws[kb * BN + ((nn * 8 + g) ^ sw)] : 0.f; }
      tf32_split(y0, bh[nn][0], bl[nn][0]); tf32_split(y1, bh[nn][1], bl[nn][1]);
    }
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int nn = 0; nn < 4; ++nn) {
        if (PREC == 1) { mma_tf32(acc[m][nn], al[m], bh[nn]); mma_tf32(acc[m][nn], ah[m], bl[nn]); }
        mma_tf32(acc[m][nn], ah[m], bh[nn]);
      }
  }
  __syncthreads();                                            // every warp is done with the A plane: reuse it
  if (tr) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); tr[3] = t; }
  float* red = As;                                            // [8 warps][32 rows][CHAIN_RED_PITCH]
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int nn = 0; nn < 4; ++nn) {
      float* q = red + (warp * BM + m * 16 + g) * CHAIN_RED_PITCH + nn * 8 + 2 * t4;
      *reinterpret_cast<float2*>(q) = make_float2(acc[m][nn][0], acc[m][nn][1]);
      *reinterpret_cast<float2*>(q + 8 * CHAIN_RED_PITCH) = make_float2(acc[m][nn][2], acc[m][nn][3]);
    }
  __syncthreads();
  const int orow = tid >> 3, ocol = (tid & 7) * 4;
  float4 sum = *reinterpret_cast<const float4*>(&red[orow * CHAIN_RED_PITCH + ocol]);
#pragma unroll
  for (int w = 1; w < GEMM_WARPS; ++w) {
    const float4 t = *reinterpret_cast<const float4*>(&red[(w * BM + orow) * CHAIN_RED_PITCH + ocol]);
    sum.x += t.x; sum.y += t.y; sum.z += t.z; sum.w += t.w;
  }
  const int gi = m0 + orow;
  const float v[4] = {sum.x, sum.y, sum.z, sum.w};
  const int epi = S.epi;
  float* __restrict__ C = S.C; const int ldc = S.ldc;
#pragma unroll
  for (int cc = 0; cc < 4; ++cc) {
    const int gj = n0 + ocol + cc;
    if (gj >= N) continue;
    float x = v[cc];
    if (gi < B) {
      const float e = eop[cc];
      switch (epi) {
        case EPI_BIAS: x += e; break;
        case EPI_BIAS_RELU: x = fmaxf(x + e, 0.f); break;
        case EPI_BIAS_TANH: x = tanhf(x + e); break;
        case EPI_RELU_MASK: x = (e > 0.f) ? x : 0.f; break;
        case EPI_TANH_MASK: x *= (1.f - e * e); break;
        default: break;
      }
      if (C) C[size_t(gi) * ldc + gj] = x;
    } else x = 0.f;
    if (xout) xout[gj * CHAIN_ROWS + orow] = x;
  }
}

template <int PREC>
__global__ void __cluster_dims__(CHAIN_CLUSTER, 1, 1) __launch_bounds__(GEMM_THREADS, 2)
mlp_chain_kernel(const __grid_constant__ ChainArgs args) {
  constexpr bool SWZ = PREC != 0;                            // tensor-core path: XOR-permuted A plane / dX weight rows
  extern __shared__ __align__(16) float chain_smem[];
  float* As = chain_smem;                              // [ka][32] resident A plane / reduce buffer
  float* W0 = chain_smem + args.a_floats;              // two weight-slice buffers (slot l uses buffer l & 1)
  const int wf = args.w_floats;
  const int tid = threadIdx.x;
  const int rank = int(cluster_ctarank());
  const int cid = blockIdx.x / CHAIN_CLUSTER;
  const int chain = cid / args.row_blocks, rb_i = cid - chain * args.row_blocks;
  const int m0 = rb_i * CHAIN_ROWS, B = args.B;
  const int ns = args.nslots[chain];
  float* planes = args.xchg + (size_t(chain) * args.row_blocks + rb_i) * (size_t(CHAIN_MAX_SLOTS) * CHAIN_PLANE);
  const int n0 = rank * BN;

  if (n0 < args.slot[chain][0].N) fetch_weights<SWZ>(W0, args.slot[chain][0], n0, tid);
  cp_async_commit();
  unsigned long long* tr0 = (args.trace && int(blockIdx.x) == args.trace_cta && tid == 0) ? args.trace : nullptr;
  const long long clk0 = clock64();
  step_stamp(args.step_trace, args.step_slot);
  if (args.step_trace && args.step_slot == 1 && tid == 0 && blockIdx.x < 256) {   // forward launch: which SM runs which CTA
    unsigned smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    reinterpret_cast<unsigned char*>(args.step_trace + (128 - STEP_TRACE_BASE))[blockIdx.x] = (unsigned char)smid;
  }
  for (int l = 0; l < ns; ++l) {
    const ChainSlot& S = args.slot[chain][l];
    const bool has_tile = n0 < S.N;
    unsigned long long* tr = tr0 ? tr0 + 6 * l : nullptr;
    CTRACE(0);
    // this thread's epilogue operands (bias / forward activations) do not depend on the chain: fetch now
    float eop[4] = {0.f, 0.f, 0.f, 0.f};
    if (has_tile && S.epi != EPI_NONE) {
      const int gi = m0 + (tid >> 3);
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const int gj = n0 + ((S.mode == GEMM_FWD && PREC == 0) ? (tid & 7) + 8 * cc : (tid & 7) * 4 + cc);
        if (gj < S.N && gi < B) eop[cc] = (S.mode == GEMM_FWD) ? __ldg(S.bias + gj) : __ldg(S.aux + size_t(gi) * S.ldaux + gj);
      }
    }
    if (l > 0) cluster_wait();                        // previous slot's planes are visible; smem is free
    CTRACE(1);
    if (PREC == 0 && S.has_pre && has_tile) {
      // ---- pre-layer: <= 8 columns, every CTA computes all of them for the cluster's 32 rows --------------------
      float* Wp = W0 + ((l + 1) & 1) * wf;            // the next slot's weight buffer is still free
      fetch_weights<SWZ>(Wp, S.pre_W, S.pre_ldw, S.pre_N, S.pre_K, S.mode, 0, tid);
      fill_from_plane<SWZ>(As, 0, planes + size_t(S.pre_src) * CHAIN_PLANE, S.pre_K, tid);
      cp_async_commit();
      float pe[4] = {0.f, 0.f, 0.f, 0.f};
      {
        const int gi = m0 + (tid >> 3);
#pragma unroll
        for (int cc = 0; cc < 4; ++cc) {
          const int gj = (S.mode == GEMM_FWD) ? (tid & 7) + 8 * cc : (tid & 7) * 4 + cc;
          if (gj < S.pre_N && gi < B)
            pe[cc] = (S.mode == GEMM_FWD) ? __ldg(S.pre_bias + gj) : __ldg(S.pre_aux + size_t(gi) * S.pre_ldaux + gj);
        }
      }
      cp_async_wait<0>();
      __syncthreads();
      const TileDesc D{S.pre_N, S.pre_K, S.pre_epi, rank == 0 ? S.pre_C : nullptr, S.pre_ldc};
      float* sout = As + S.pre_row * CHAIN_ROWS;      // outside the reduce buffer (rows 0..255)
      if (S.mode == GEMM_FWD) chain_tile<GEMM_FWD>(D, As, As, Wp, m0, 0, B, nullptr, sout, pe, nullptr);
      else chain_tile<GEMM_DX>(D, As, As, Wp, m0, 0, B, nullptr, sout, pe, nullptr);
      __syncthreads();                                // reduce buffer dead, pre-layer output in place
    }
    if (has_tile) {
      const int K = S.K, K1 = S.K1;
      if (S.src >= 0) fill_from_plane<SWZ>(As, 0, planes + size_t(S.src) * CHAIN_PLANE, K1, tid);
      else if (S.src == -1) fill_from_rows<SWZ>(As, 0, S.Ag, S.ldag, m0, B, K1, tid);
      if (K > K1) {
        if (S.src2 >= 0) fill_from_plane<SWZ>(As, K1, planes + size_t(S.src2) * CHAIN_PLANE, K - K1, tid);
        else if (S.src2 == -1) fill_from_rows<SWZ>(As, K1, S.A2g, S.lda2g, m0, B, K - K1, tid);
      }
    }
    cp_async_commit();
    // the next layer's weights do not depend on this layer: they travel while it computes
    if (l + 1 < ns && n0 < args.slot[chain][l + 1].N) fetch_weights<SWZ>(W0 + ((l + 1) & 1) * wf, args.slot[chain][l + 1], n0, tid);
    cp_async_commit();
    cp_async_wait<1>();                               // everything but the prefetch has landed
    __syncthreads();
    CTRACE(2);
    if (has_tile) {
      float* xout = S.publish ? planes + size_t(l) * CHAIN_PLANE : nullptr;
      if (PREC == 0) {
        const TileDesc D = tile_of(S);
        const float* Am = As + S.a_row0 * CHAIN_ROWS;
        if (S.mode == GEMM_FWD) chain_tile<GEMM_FWD>(D, Am, As, W0 + (l & 1) * wf, m0, n0, B, xout, nullptr, eop, tr);
        else chain_tile<GEMM_DX>(D, Am, As, W0 + (l & 1) * wf, m0, n0, B, xout, nullptr, eop, tr);
      } else {
        if (S.mode == GEMM_FWD) chain_tile_mma<GEMM_FWD, PREC>(S, As, W0 + (l & 1) * wf, m0, n0, B, xout, eop, tr);
        else chain_tile_mma<GEMM_DX, PREC>(S, As, W0 + (l & 1) * wf, m0, n0, B, xout, eop, tr);
      }
    }
    CTRACE(4);
    if (l + 1 < ns) cluster_arrive();
    CTRACE(5);
  }
  cp_async_wait<0>();
  step_stamp(args.step_trace, args.step_slot + 16);
  if (tr0) tr0[6 * CHAIN_MAX_SLOTS - 1] = (unsigned long long)(clock64() - clk0);    // SM cycles of the whole kernel
}

static unsigned long long* chain_trace_buffer() { return debug_trace_buffer(); }

// ---- host side -------------------------------------------------------------------------------------
int64_t chain_xchg_floats(int B) {
  return int64_t(CHAIN_MAX) * cdiv(B, CHAIN_ROWS) * CHAIN_MAX_SLOTS * CHAIN_PLANE;
}
void chain_args_begin(ChainArgs& a, int B, float* xchg, int precision) {
  a = ChainArgs{};
  a.B = B; a.row_blocks = cdiv(B, CHAIN_ROWS); a.xchg = xchg; a.precision = precision;
  // the A plane doubles as the 8-warp reduce buffer
  a.a_floats = precision ? GEMM_WARPS * BM * CHAIN_RED_PITCH : GEMM_WARPS * BM * BN;
  a.w_floats = 0;
}
int chain_add(ChainArgs& a, int c, const ChainSlot& s) {
  if (c >= a.nchains) a.nchains = c + 1;
  const int l = a.nslots[c]++;
  a.slot[c][l] = s;
  const int af = int(align4(int64_t(s.has_pre ? std::max(s.K, s.pre_row + 8) : s.K) * CHAIN_ROWS));
  const int wf = s.mode == GEMM_FWD ? BN * chain_wpitch(s.K) : int(align4(int64_t(s.K) * BN));
  if (af > a.a_floats) a.a_floats = af;
  if (wf > a.w_floats) a.w_floats = wf;
  return l;
}
size_t chain_smem_bytes(const ChainArgs& a) { return size_t(a.a_floats + 2 * a.w_floats) * sizeof(float); }
bool chain_fits(const ChainArgs& a) {
  for (int c = 0; c < a.nchains; ++c)
    for (int l = 0; l < a.nslots[c]; ++l)
      if (a.slot[c][l].N > CHAIN_CLUSTER * BN) return false;
  return chain_smem_bytes(a) <= CHAIN_SMEM_MAX;
}
ChainSlot chain_fwd(const float* W, int ldw, const float* bias, int N, int K, int epi, float* C, int ldc, int publish) {
  ChainSlot s{};
  s.W = W; s.ldw = ldw; s.bias = bias; s.N = N; s.K = K; s.K1 = K; s.epi = epi; s.C = C; s.ldc = ldc;
  s.mode = GEMM_FWD; s.publish = publish; s.src = -1; s.src2 = -1;
  return s;
}
ChainSlot chain_dx(const float* W, int ldw, int N_in, int K_out, int epi, const float* aux, int ldaux,
                   float* C, int ldc, int publish) {
  ChainSlot s{};
  s.W = W; s.ldw = ldw; s.N = N_in; s.K = K_out; s.K1 = K_out; s.epi = epi; s.aux = aux; s.ldaux = ldaux;
  s.C = C; s.ldc = ldc; s.mode = GEMM_DX; s.publish = publish; s.src = -1; s.src2 = -1;
  return s;
}
void chain_src_global(ChainSlot& s, const float* Ag, int ldag) { s.Ag = Ag; s.ldag = ldag; s.src = -1; }
void chain_src_plane(ChainSlot& s, int slot) { s.src = slot; }
void chain_src2_global(ChainSlot& s, int K1, const float* A2g, int lda2g) { s.K1 = K1; s.A2g = A2g; s.lda2g = lda2g; s.src2 = -1; }
void chain_src2_plane(ChainSlot& s, int K1, int slot) { s.K1 = K1; s.src2 = slot; }
void chain_pre_layer(ChainSlot& s, const float* W, int ldw, const float* bias, const float* aux, int ldaux, int N, int K, int epi,
                     float* C, int ldc, int src_slot, int pre_row, bool whole_operand) {
  s.has_pre = 1; s.pre_W = W; s.pre_ldw = ldw; s.pre_bias = bias; s.pre_aux = aux; s.pre_ldaux = ldaux;
  s.pre_N = N; s.pre_K = K; s.pre_epi = epi; s.pre_C = C; s.pre_ldc = ldc; s.pre_src = src_slot; s.pre_row = pre_row;
  if (whole_operand) { s.src = -2; s.K1 = s.K; s.a_row0 = pre_row; }     // DX: the pre-layer IS the A operand
  else { s.src2 = -2; s.K1 = s.K - N; s.a_row0 = 0; }                     // FWD: the pre-layer is the concatenated tail
}

int launch_mlp_chain(ChainArgs& a, cudaStream_t st) {
  D4PG_REQUIRE(a.nchains > 0 && a.nchains <= CHAIN_MAX, D4PG_EINVAL, "launch_mlp_chain: %d chains", a.nchains);
  for (int c = 0; c < a.nchains; ++c) {
    D4PG_REQUIRE(a.nslots[c] > 0 && a.nslots[c] <= CHAIN_MAX_SLOTS, D4PG_EINVAL, "launch_mlp_chain: chain %d has %d slots", c, a.nslots[c]);
    for (int l = 0; l < a.nslots[c]; ++l) {
      const ChainSlot& s = a.slot[c][l];
      D4PG_REQUIRE(s.N > 0, D4PG_EINVAL, "launch_mlp_chain: slot %d has no columns", l);
      D4PG_REQUIRE(s.ldw % 4 == 0 && (reinterpret_cast<uintptr_t>(s.W) & 15) == 0, D4PG_EINVAL, "launch_mlp_chain: weights must be 16-B pitched");
      D4PG_REQUIRE(s.src < l && s.src2 < l, D4PG_EINVAL, "launch_mlp_chain: slot %d reads a later plane", l);
      D4PG_REQUIRE(s.src >= 0 || s.src == -2 || (s.Ag && s.ldag % 4 == 0 && s.ldag >= s.K1), D4PG_EINVAL, "launch_mlp_chain: bad global A source");
      D4PG_REQUIRE(s.K == s.K1 || s.src2 >= 0 || s.src2 == -2 || (s.A2g && s.lda2g % 4 == 0 && s.lda2g >= s.K - s.K1), D4PG_EINVAL, "launch_mlp_chain: bad second A source");
      D4PG_REQUIRE((s.src != -2 && s.src2 != -2) || s.has_pre, D4PG_EINVAL, "launch_mlp_chain: slot %d expects a pre-layer", l);
      if (s.has_pre) {
        D4PG_REQUIRE(a.precision == 0, D4PG_ENOTSUP, "launch_mlp_chain: pre-layers exist for the fp32 tile only");
        D4PG_REQUIRE(s.pre_N > 0 && s.pre_N <= 8 && s.pre_K <= D4PG_HIDDEN && s.pre_row >= D4PG_HIDDEN && s.pre_src >= 0 && s.pre_src < l &&
                     a.slot[c][s.pre_src].publish && a.slot[c][s.pre_src].N >= s.pre_K && s.pre_ldw % 4 == 0 &&
                     (reinterpret_cast<uintptr_t>(s.pre_W) & 15) == 0, D4PG_EINVAL, "launch_mlp_chain: bad pre-layer in slot %d", l);
      }
      D4PG_REQUIRE(s.src < 0 || (a.slot[c][s.src].publish && a.slot[c][s.src].N >= s.K1), D4PG_EINVAL, "launch_mlp_chain: slot %d reads an unpublished plane", l);
      D4PG_REQUIRE(s.K == s.K1 || s.src2 < 0 || (a.slot[c][s.src2].publish && a.slot[c][s.src2].N >= s.K - s.K1), D4PG_EINVAL, "launch_mlp_chain: slot %d reads an unpublished plane", l);
    }
  }
  const size_t smem = chain_smem_bytes(a);
  // NOT padded to force one CTA per SM: 16 clusters of 8 at one CTA per SM need two free 8-SM groups in every
  // GPC; a single foreign CTA (the concurrent tree update) pushes clusters into a second wave.
  D4PG_REQUIRE(chain_fits(a), D4PG_ENOTSUP, "launch_mlp_chain: %zu B of shared memory needed (at most %zu) or a layer wider than %d",
               smem, CHAIN_SMEM_MAX, CHAIN_CLUSTER * BN);
  D4PG_REQUIRE(a.precision >= 0 && a.precision <= 2, D4PG_EINVAL, "launch_mlp_chain: precision %d", a.precision);
  static size_t smem_set[3] = {0, 0, 0};
  void (*kern)(ChainArgs) = a.precision == 0 ? mlp_chain_kernel<0> : a.precision == 1 ? mlp_chain_kernel<1> : mlp_chain_kernel<2>;
  if (smem > smem_set[a.precision]) {
    D4PG_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    D4PG_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, int(cudaSharedmemCarveoutMaxShared)));
    smem_set[a.precision] = smem;
  }
  a.trace = chain_trace_buffer() ? chain_trace_buffer() + a.trace_base : nullptr;
  a.step_trace = chain_trace_buffer() ? chain_trace_buffer() + STEP_TRACE_BASE : nullptr;
  a.step_slot = a.trace_base ? 5 : 1;
  { const char* e = getenv("D4PG_TRACE_CTA"); a.trace_cta = e ? atoi(e) : 0; if (a.trace_cta >= a.nchains * a.row_blocks * CHAIN_CLUSTER) a.trace_cta = 0; }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(a.nchains * a.row_blocks * CHAIN_CLUSTER); cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cfg.attrs = nullptr; cfg.numAttrs = 0;              // cluster shape is compiled in (__cluster_dims__)
  D4PG_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, a));
  return D4PG_OK;
}

}  // namespace d4pg
