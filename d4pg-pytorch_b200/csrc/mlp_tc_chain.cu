// Cluster chains on the Hopper tensor cores: every dependent layer of an actor/critic network chain in ONE launch,
// each layer a set of wgmma tiles with register accumulators, operands brought in by bulk copies (cp.async.bulk).
//
// Reference ops: actor.forward / critic.forward (models.py:32-41,76-88) for the five forward passes of
// DDPG.train (ddpg.py:205-208,236) and the two backward passes of ddpg.py:230,242 (dX only; dW is gemm_wide).
//
// Decomposition.  A thread-block CLUSTER of 8 CTAs owns 64 batch rows (wgmma M = 64) for a whole chain.  CTA r
// owns output features [32r, 32r+32) of every 256-wide layer, so a layer is eight 64x32xK tiles and the
// layer-to-layer dependency is an all-gather of the 64x256 activation plane inside the cluster.
//
// Precision.  3xTF32: x = hi + lo, hi = x with the low 13 mantissa bits cleared, lo = tf32(x - hi);
// D += Al*Bh + Ah*Bl + Ah*Bh with fp32 accumulation (~2^-21 relative, meets the 1e-5 parity bar).  One TF32 pass
// (TccArgs::passes = 1, precision 2) is D += Ah*Bh alone: both operands truncated to TF32 (round toward zero).
// Nothing is split on the critical path:
//   * weights: hi/lo parts are PRE-PACKED once per step (tcc_pack_kernel, right after Adam changed them) into the
//     exact shared-memory image the MMA reads (K-major SWIZZLE_128B, 32x32 blocks) -- for the backward pass the
//     transposed image -- so a CTA's weight slice of a layer is ONE contiguous cp.async.bulk;
//   * activations: the epilogue that PRODUCES a layer output (bias/ReLU/tanh/mask on the accumulator registers)
//     writes it three times: row-major fp32 (for the loss kernel / dW), and as hi and lo images of its 64x32 tile
//     = K-chunk r of the next layer's A operand, already swizzled.  The consumers fetch chunk c with one 16-KB
//     cp.async.bulk.
//
// Per CTA: warpgroups 0 and 1 = consumers (warpgroup g issues the wgmmas of output group g of a slot and runs
// its epilogue), warp 8 = loader (one lane issues every bulk copy: weight slices one slot ahead, A chunks into
// direct-mapped buffers, completion on mbarriers by byte count).  A slot boundary is a cluster barrier
// (arrive.release / wait.acquire): outputs in L2 are visible, A and weight buffers are free.
#include "mlp_tc_chain.cuh"
#include "tc_common.cuh"
#include <stdlib.h>
#include <string.h>

namespace d4pg {

using namespace tc;

// shared-memory map (bytes from the 1024-B aligned base)
constexpr uint32_t TCC_OFF_A = 0;
constexpr uint32_t TCC_OFF_W = TCC_ABUFS * TCC_A_CHUNK;
constexpr uint32_t TCC_OFF_BAR = TCC_OFF_W + TCC_MAX_CHUNKS * TCC_W_CHUNK;
constexpr uint32_t TCC_SMEM = TCC_OFF_BAR + 256 + 1024;      // barriers + alignment slack
static_assert(TCC_SMEM <= 227 * 1024, "the chain kernel's shared memory exceeds what a Hopper CTA may use");
constexpr int TCC_CONSUMERS = 256;                         // two warpgroups
constexpr int TCC_TRACE_PER_SLOT = 12;

__device__ __forceinline__ void tcc_cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void tcc_cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ unsigned tcc_ctarank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ unsigned long long tcc_gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// 1-D bulk copy global -> this CTA's shared memory, completion by byte count on an mbarrier
__device__ __forceinline__ void tcc_bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// Watchdog: every mbarrier wait of this kernel is bounded (~2 s of SM clocks).  A protocol bug then ends the launch
// with a trap and a record in HOST-mapped memory (readable after the context died: d4pg_debug_watchdog) instead of
// hanging the GPU.  record[0] = 1, [1] = code | slot << 8 | rank << 16 | parity << 24 | block << 32, [2] = seq / nact.
__device__ __forceinline__ void tcc_wait(uint64_t* bar, uint32_t parity, unsigned long long* dbg, unsigned code, unsigned aux) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  bool recorded = false;
  while (!mbar_try_wait(bar, parity)) {
    const long long dt = clock64() - t0;
    if (dt > 4000000000ll && !recorded) {
      recorded = true;
      if (dbg) {
        if (atomicCAS(dbg, 0ull, 1ull) == 0ull) {           // the first wait that timed out anywhere
          dbg[1] = (unsigned long long)code | ((unsigned long long)parity << 24) | ((unsigned long long)blockIdx.x << 32);
          dbg[2] = aux;
        }
        const unsigned kind = code & 0xFFu;                 // and the first one of every kind (2 words each)
        if (kind < 6 && atomicCAS(dbg + 4 + 2 * kind, 0ull, 1ull) == 0ull) {
          dbg[4 + 2 * kind] = (unsigned long long)code | ((unsigned long long)parity << 24) | ((unsigned long long)blockIdx.x << 32);
          dbg[5 + 2 * kind] = aux;
        }
        __threadfence_system();
      }
    }
    if (dt > 5000000000ll) __trap();                        // every stuck waiter had time to leave its record
  }
}
#define TCC_CODE(kind, slot, rank) (unsigned(kind) | (unsigned(slot) << 8) | (unsigned(rank) << 16))
enum { WD_LOADER_DFULL = 2, WD_MMA_WFULL = 3, WD_MMA_FULL = 4 };

__device__ __forceinline__ float4 tcc_hi4(float4 v) { return make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w)); }
__device__ __forceinline__ float4 tcc_lo4(float4 v, float4 h) {
  return make_float4(tf32_lo(v.x, h.x), tf32_lo(v.y, h.y), tf32_lo(v.z, h.z), tf32_lo(v.w, h.w));
}

// [64 rows x 32 k] chunk of a row-major fp32 array -> hi / lo SWIZZLE_128B K-major images (the 256 consumer threads)
__device__ __forceinline__ void tcc_convert_chunk(uint8_t* dst, const float* __restrict__ src, int ld, int k0, int ncols,
                                                  int m0, int B, int et) {
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    const int e = et + p * 256, row = e >> 3, u = e & 7, k = k0 + (u << 2);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m0 + row < B && k < ncols) {
      v = __ldg(reinterpret_cast<const float4*>(src + size_t(m0 + row) * ld + k));     // ld is a multiple of 4 >= ncols
      if (k + 1 >= ncols) v.y = 0.f;
      if (k + 2 >= ncols) v.z = 0.f;
      if (k + 3 >= ncols) v.w = 0.f;
    }
    const float4 h = tcc_hi4(v);
    const uint32_t off = sw128_kmajor_off(row, u << 2);
    *reinterpret_cast<float4*>(dst + off) = h;
    *reinterpret_cast<float4*>(dst + TCC_A_HALF + off) = tcc_lo4(v, h);
  }
}

__device__ __forceinline__ bool tcc_group_active(const TccSlot& S, int g, int n0) { return g < S.ngroups && n0 < S.g[g].N; }
__device__ __forceinline__ bool tcc_slot_active(const TccSlot& S, int n0) { return tcc_group_active(S, 0, n0) || tcc_group_active(S, 1, n0); }

// loader lane: the CTA's weight slices of one slot -> W buffer (one bulk copy per group)
__device__ __forceinline__ void tcc_issue_weights(const TccSlot& S, int rank, int n0, uint8_t* Wb, uint64_t* wfull) {
  const uint32_t gbytes = uint32_t(S.nchunks) * TCC_W_CHUNK;
  uint32_t bytes = 0;
#pragma unroll
  for (int g = 0; g < TCC_MAX_GROUPS; ++g)
    if (tcc_group_active(S, g, n0)) bytes += gbytes;
  mbar_expect_tx(wfull, bytes);
#pragma unroll
  for (int g = 0; g < TCC_MAX_GROUPS; ++g)
    if (tcc_group_active(S, g, n0)) tcc_bulk_load(Wb + g * gbytes, S.g[g].wimg + size_t(rank) * gbytes, gbytes, wfull);
}

// PASSES = 3: 3xTF32 (Ah.Bh + Ah.Bl + Al.Bh); PASSES = 1: one TF32 pass Ah.Bh on the hi images alone (the lo images are
// still written and copied, but never read).  The hi images truncate (tf32_hi), so one pass is round-toward-zero TF32.
template <int PASSES>
__global__ void __cluster_dims__(TCC_CLUSTER, 1, 1) __launch_bounds__(TCC_THREADS, 1)
mlp_tc_chain_kernel(const __grid_constant__ TccArgs args) {
  static_assert(PASSES == 1 || PASSES == 3, "the chain kernel runs one TF32 pass or 3xTF32");
  extern __shared__ uint8_t tcc_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tcc_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* Ab = smem + TCC_OFF_A;        // [TCC_ABUFS] A-chunk buffers; buffer 8 doubles as the resident X chunk
  uint8_t* Xb = Ab + 8 * TCC_A_CHUNK;
  uint8_t* Wb = smem + TCC_OFF_W;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + TCC_OFF_BAR);
  uint64_t* full = bars;                 // [TCC_ABUFS]  bytes of the copy that starts at this buffer have landed
  uint64_t* wfull = bars + TCC_ABUFS;    // weight slices of the current slot have landed
  uint64_t* dfull = wfull + 1;           // all MMAs of the current slot have completed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rank = int(tcc_ctarank());
  const int cid = blockIdx.x / TCC_CLUSTER;
  const int chain = cid / args.row_blocks, rb = cid - chain * args.row_blocks;
  const int m0 = rb * TCC_ROWS, B = args.B;
  const TccChain& CH = args.chain[chain];
  const int ns = CH.nslots;
  const int n0 = rank * TCC_BN;
  uint8_t* planes = args.xchg + (size_t(chain) * args.row_blocks + rb) * (size_t(TCC_PLANES) * TCC_PLANE_BYTES);
  const int npre = CH.pre ? (CH.precols + TCC_KC - 1) / TCC_KC : 0;
  unsigned long long* tr0 = (args.trace && int(blockIdx.x) == args.trace_cta) ? args.trace : nullptr;
  if (args.wait_epoch) {                 // host pipeline: the sample kernel of this step publishes per-CTA epochs
    if (tid < args.wait_n) {
      const unsigned long long target = (unsigned long long)(*reinterpret_cast<const volatile long long*>(args.wait_clock) + 1);
      unsigned long long v;
      do { asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(args.wait_epoch + tid) : "memory"); } while (v < target);
    }
    __syncthreads();
  }
  step_stamp(args.step_trace, args.step_slot);

  if (tid == TCC_CONSUMERS) {
    for (int i = 0; i < TCC_ABUFS + 2; ++i) mbar_init(&bars[i], 1);
    mbar_fence_init();
  }
  if (tid < TCC_CONSUMERS) {
    if (CH.x0) tcc_convert_chunk(Xb, CH.x0, CH.x0ld, 0, CH.x0cols, m0, B, tid);
    for (int p = 0; p < npre; ++p) tcc_convert_chunk(Ab + p * TCC_A_CHUNK, CH.pre, CH.preld, p * TCC_KC, CH.precols, m0, B, tid);
    fence_proxy_async();
  }
  __syncthreads();

  // the pre-converted chunks: complete the first phase of their `full` barriers (the consumers wait on them like on a copy)
  if (tid == TCC_CONSUMERS)
    for (int p = 0; p < npre; ++p) mbar_arrive(&full[p]);
  // per-role state.  fph: bit b = parity of the NEXT completion of full[b] the consumers will wait for
  uint32_t fph = 0;
  int nact = 0;                          // slots this CTA took part in so far: phase of wfull / dfull
  if (tid == TCC_CONSUMERS && tcc_slot_active(CH.slot[0], n0)) tcc_issue_weights(CH.slot[0], rank, n0, Wb, wfull);

  for (int l = 0; l < ns; ++l) {
    const TccSlot& S = CH.slot[l];
    const bool active = tcc_slot_active(S, n0);
    unsigned long long* tr = tr0 ? tr0 + TCC_TRACE_PER_SLOT * l : nullptr;
    bool arrived = false;                  // this thread already arrived on the slot's cluster barrier

    if (tid >= TCC_CONSUMERS) {
      // ============================== loader ==========================================================
      // Every A buffer is free here: the previous slot's MMAs completed before anyone passed the cluster barrier.
      if (lane == 0) {
        if (tr) tr[0] = tcc_gtime();
        if (active && S.nloads > 0) {
          // the cluster's stores to the planes (acquired by the barrier above) -> this thread's bulk-copy reads
          asm volatile("fence.proxy.async.global;" ::: "memory");
          for (int i = 0; i < S.nloads; ++i) {
            const TccLoad L = S.ld[i];
            const uint32_t bytes = uint32_t(L.count) * TCC_A_CHUNK;
            mbar_expect_tx(&full[L.buf0], bytes);
            tcc_bulk_load(Ab + L.buf0 * TCC_A_CHUNK, planes + size_t(L.plane) * TCC_PLANE_BYTES + size_t(L.chunk0) * TCC_A_CHUNK,
                          bytes, &full[L.buf0]);
          }
        }
        if (tr) tr[1] = tcc_gtime();
        // next slot's weights travel while this slot's epilogue and the barrier run
        if (l + 1 < ns && tcc_slot_active(CH.slot[l + 1], n0)) {
          if (active) tcc_wait(dfull, nact & 1, args.watchdog, TCC_CODE(WD_LOADER_DFULL, l, rank), nact);  // the weight buffer is free
          tcc_issue_weights(CH.slot[l + 1], rank, n0, Wb, wfull);
        }
      }
      __syncwarp();
    } else {
      // ============================== consumers: warpgroup g = output group g =========================
      const int g = warp >> 2, wq = warp & 3;
      const bool mine = tcc_group_active(S, g, n0);
      const int rl = 16 * wq + (lane >> 2);                // accumulator rows rl and rl + 8 of the cluster's 64-row block
      const int cl = 2 * (lane & 3);                       // accumulator columns cl + 8 j + {0, 1}, j = 0..3
      if (active) {
        const TccGroup& G = S.g[g];
        // 3xTF32 in two wgmmas per 8-deep k-step: the weight chunk holds the hi image (32 rows) directly followed by
        // the lo image (32 rows) = a 64-row B operand, so d1[64 x 64] = Ah . [Bh; Bl]^T (columns 0-31 Ah.Bh, 32-63
        // Ah.Bl) and d2[64 x 32] = Al . Bh^T (Al.Bl, ~2^-22 relative, is not formed).  One pass: d1[64 x 32] = Ah . Bh^T
        // from the first 32 rows of the chunk, and no d2.
        constexpr int N1 = PASSES == 3 ? 32 : 16;
        float d1[N1], d2[PASSES == 3 ? 16 : 1];
#pragma unroll
        for (int i = 0; i < N1; ++i) d1[i] = 0.f;
        if constexpr (PASSES == 3) {
#pragma unroll
          for (int i = 0; i < 16; ++i) d2[i] = 0.f;
        }
        // this thread's epilogue operands do not depend on the chain: fetch them before the accumulator is ready
        float eop[2][8];
        const int npad = mine ? (G.N + 3) & ~3 : 0;
        const bool fwd = G.epi == EPI_BIAS || G.epi == EPI_BIAS_RELU || G.epi == EPI_BIAS_TANH;
        const bool msk = G.epi == EPI_RELU_MASK || G.epi == EPI_TANH_MASK;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int gi = m0 + rl + 8 * rr;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int gj = n0 + 8 * j + cl;
            float2 v = make_float2(0.f, 0.f);
            if (gj < npad) {
              if (fwd) v = __ldg(reinterpret_cast<const float2*>(G.bias + gj));
              else if (msk && gi < B) v = __ldg(reinterpret_cast<const float2*>(G.aux + size_t(gi) * G.ldaux + gj));
            }
            eop[rr][2 * j] = v.x; eop[rr][2 * j + 1] = v.y;
          }
        }
        const int nch = S.nchunks, boff = S.boff;
        const uint32_t wait_mask = S.wait_mask;
        if (mine) {
          tcc_wait(wfull, nact & 1, args.watchdog, TCC_CODE(WD_MMA_WFULL, l, rank), nact);
          if (tr && tid == 0) tr[2] = tcc_gtime();
          const uint32_t w_base = smem_u32(Wb) + uint32_t(g * nch) * TCC_W_CHUNK;
          const uint32_t a_base = smem_u32(Ab) + uint32_t(boff) * TCC_A_CHUNK;
          wg_fence_regs(d1);
          if constexpr (PASSES == 3) wg_fence_regs(d2);
          // Chunk c of the slot's K lives in A buffer c + boff (checked at launch)
          for (int c = 0; c < nch; ++c) {
            if ((wait_mask >> c) & 1u) {                  // first chunk of a bulk copy / a pre-converted chunk
              const int b = c + boff;
              tcc_wait(&full[b], (fph >> b) & 1u, args.watchdog, TCC_CODE(WD_MMA_FULL, l, rank), b);
              if (tr && tid == 0 && c == 0) tr[3] = tcc_gtime();
            }
            const uint32_t a_hi = a_base + uint32_t(c) * TCC_A_CHUNK, a_lo = a_hi + TCC_A_HALF;
            const uint32_t w = w_base + uint32_t(c) * TCC_W_CHUNK;
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
              const uint64_t bd = wg_desc(w + 32 * ks);
              if constexpr (PASSES == 3) {
                wg_mma_n64(d1, wg_desc(a_hi + 32 * ks), bd);
                wg_mma_n32(d2, wg_desc(a_lo + 32 * ks), bd);
              } else {
                wg_mma_n32(d1, wg_desc(a_hi + 32 * ks), bd);
              }
            }
            wg_commit();
          }
          wg_wait<0>();
          wg_fence_regs(d1);
          if constexpr (PASSES == 3) wg_fence_regs(d2);
          if (tr && tid == 0) tr[4] = tcc_gtime();
        }
        // both warpgroups' MMAs are done: the A buffers may be overwritten and the weight buffer refilled
        for (int c = 0; c < nch; ++c)
          if ((wait_mask >> c) & 1u) fph ^= 1u << (c + boff);
        asm volatile("bar.sync 1, %0;" ::"n"(TCC_CONSUMERS) : "memory");
        if (tid == 0) mbar_arrive(dfull);
        if (tr && tid == 0) tr[5] = tcc_gtime();
        // the resident X chunk is re-used for another array (critic fc2's action columns) now that this slot's MMAs are
        // done -- before any thread arrives on the slot's barrier
        if (S.xsrc) {
          tcc_convert_chunk(Xb, S.xsrc, S.xld, 0, S.xcols, m0, B, tid);
          fence_proxy_async();                             // shared-memory writes -> the tensor core's async-proxy reads
        }
        if (mine) {
          // ---- Ah.Bh + Ah.Bl + Al.Bh (one pass: Ah.Bh), epilogue ------------------------------------------------
          const int epi = G.epi;
          float x[16];                                     // x[4 j + 2 rr + e] = (row rl + 8 rr, column cl + 8 j + e)
          if constexpr (PASSES == 3) {
#pragma unroll
            for (int i = 0; i < 16; ++i) x[i] = (d1[i + 16] + d2[i]) + d1[i];   // the two small cross terms first
          } else {
#pragma unroll
            for (int i = 0; i < 16; ++i) x[i] = d1[i];
          }
          // the epilogue kind is decided ONCE per group, around whole loops (a per-element switch compiles to an
          // indirect branch per element)
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const float e = eop[(i >> 1) & 1][2 * (i >> 2) + (i & 1)];
            if (epi == EPI_BIAS || epi == EPI_BIAS_RELU || epi == EPI_BIAS_TANH) x[i] += e;
            else if (epi == EPI_RELU_MASK) x[i] = (e > 0.f) ? x[i] : 0.f;
            else if (epi == EPI_TANH_MASK) x[i] *= (1.f - e * e);
          }
          if (epi == EPI_BIAS_RELU) {
#pragma unroll
            for (int i = 0; i < 16; ++i) x[i] = fmaxf(x[i], 0.f);
          } else if (epi == EPI_BIAS_TANH) {
#pragma unroll
            for (int i = 0; i < 16; ++i)
              if (n0 + 8 * (i >> 2) + cl + (i & 1) < G.N) x[i] = tanhf(x[i]);   // the action columns only
          }
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int gi = m0 + rl + 8 * ((i >> 1) & 1), gj = n0 + 8 * (i >> 2) + cl + (i & 1);
            x[i] = (gi < B && gj < G.N) ? x[i] : 0.f;      // pad rows / columns stay zero in the images
          }
          if (tr && tid == 0) tr[6] = tcc_gtime();
          if (G.pub >= 0) {
            // K-chunk `rank` of the consumers' A operand: the hi and lo images of this 64 x 32 tile are ONE contiguous
            // 16-KB block of the plane -> staged in shared memory (A buffer 2 + g, free) in the image layout and
            // written with a single bulk store
            uint8_t* stg = Ab + (2 + g) * TCC_A_CHUNK;
#pragma unroll
            for (int i = 0; i < 16; i += 2) {
              const int r = rl + 8 * ((i >> 1) & 1), k = 8 * (i >> 2) + cl;
              const float2 v = make_float2(x[i], x[i + 1]);
              const float2 h = make_float2(tf32_hi(v.x), tf32_hi(v.y));
              const uint32_t off = sw128_kmajor_off(r, k);
              *reinterpret_cast<float2*>(stg + off) = h;
              *reinterpret_cast<float2*>(stg + TCC_A_HALF + off) = make_float2(tf32_lo(v.x, h.x), tf32_lo(v.y, h.y));
            }
            fence_proxy_async();                           // staged tile (generic proxy) -> bulk store (async proxy)
            asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");
            if ((tid & 127) == 0) {
              uint8_t* img = planes + size_t(G.pub) * TCC_PLANE_BYTES + size_t(rank) * TCC_A_CHUNK;
              asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                           ::"l"(img), "r"(smem_u32(stg)), "r"(TCC_A_CHUNK) : "memory");
              asm volatile("cp.async.bulk.commit_group;" ::: "memory");
              asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");      // writes complete: visible before the barrier arrive
            }
          }
          if (tr && tid == 0) tr[8] = tcc_gtime();
          // The row-major outputs are read by later kernels only: they are stored AFTER this thread's barrier arrive, so
          // the cluster does not wait for them to drain.
          if (l + 1 < ns) { tcc_cluster_arrive(); arrived = true; }
          if (G.C) {
#pragma unroll
            for (int i = 0; i < 16; i += 2) {
              const int gi = m0 + rl + 8 * ((i >> 1) & 1), gj = n0 + 8 * (i >> 2) + cl;
              if (gi < B && gj < npad) *reinterpret_cast<float2*>(G.C + size_t(gi) * G.ldc + gj) = make_float2(x[i], x[i + 1]);
            }
          }
        }
      } else if (S.xsrc) {                                 // (an inactive CTA did not read X in this slot)
        tcc_convert_chunk(Xb, S.xsrc, S.xld, 0, S.xcols, m0, B, tid);
        fence_proxy_async();
      }
      if (tr && tid == 0) tr[9] = tcc_gtime();
    }
    if (active) ++nact;
    if (l + 1 < ns) {
      if (!arrived) tcc_cluster_arrive();
      tcc_cluster_wait();
      if (tr && tid == 0) tr[10] = tcc_gtime();
    }
  }
  step_stamp(args.step_trace, args.step_slot + 16);
}

// ---- weight packing -------------------------------------------------------------------------------------
// One CTA per 32x32 block: 256 threads, one float4 of hi and lo each.
__global__ void __launch_bounds__(256) tcc_pack_kernel(const __grid_constant__ TccPackArgs args) {
  int ui = 0;
#pragma unroll 1
  for (int i = 1; i < args.n; ++i)
    if (int(blockIdx.x) >= args.use[i].block_begin) ui = i;
  const TccPackUse& U = args.use[ui];
  const int blk = blockIdx.x - U.block_begin;
  const int slice = blk / U.nchunks, chunk = blk - slice * U.nchunks;
  uint8_t* dst = args.dst + U.dst_off + size_t(blk) * TCC_W_CHUNK;
  const int tid = threadIdx.x;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  int j, u;
  if (U.mode == GEMM_FWD) {
    j = tid >> 3; u = tid & 7;                               // consecutive threads: consecutive 16-B units of a W row
    const int n = slice * TCC_BN + j, k = chunk * TCC_KC + 4 * u;
    if (n < U.N && k < U.K) {
      v = __ldg(reinterpret_cast<const float4*>(U.W + size_t(n) * U.ldw + k));   // row pitch is a multiple of 4 floats
      if (k + 1 >= U.K) v.y = 0.f;
      if (k + 2 >= U.K) v.z = 0.f;
      if (k + 3 >= U.K) v.w = 0.f;
    }
  } else {
    j = tid & 31; u = tid >> 5;                              // consecutive threads: consecutive columns n of a W row (coalesced)
    const int n = slice * TCC_BN + j, k = chunk * TCC_KC + 4 * u;
    if (n < U.N) {
      if (k < U.K) v.x = __ldg(U.W + size_t(k) * U.ldw + n);
      if (k + 1 < U.K) v.y = __ldg(U.W + size_t(k + 1) * U.ldw + n);
      if (k + 2 < U.K) v.z = __ldg(U.W + size_t(k + 2) * U.ldw + n);
      if (k + 3 < U.K) v.w = __ldg(U.W + size_t(k + 3) * U.ldw + n);
    }
  }
  const float4 h = tcc_hi4(v);
  const uint32_t off = sw128_kmajor_off(j, 4 * u);
  *reinterpret_cast<float4*>(dst + off) = h;
  *reinterpret_cast<float4*>(dst + TCC_W_HALF + off) = tcc_lo4(v, h);
}

static unsigned long long* g_tcc_watchdog_host = nullptr;
// allocated once per process, outside of any stream capture (tcc users call this at create time)
unsigned long long* tcc_watchdog_device() {
  static bool tried = false;
  static unsigned long long* dev = nullptr;
  if (!tried) {
    tried = true;
    unsigned long long* host = nullptr;
    if (cudaHostAlloc(reinterpret_cast<void**>(&host), 128, cudaHostAllocMapped) == cudaSuccess) {
      memset(host, 0, 128);
      if (cudaHostGetDevicePointer(reinterpret_cast<void**>(&dev), host, 0) != cudaSuccess) dev = nullptr;
      g_tcc_watchdog_host = host;
    }
    (void)cudaGetLastError();
  }
  return dev;
}
}  // namespace d4pg
// the watchdog record of the chain kernel (host-mapped memory: readable after a trapped launch killed the context)
extern "C" int32_t d4pg_debug_watchdog(unsigned long long* out16) {
  if (!out16) return D4PG_EINVAL;
  for (int i = 0; i < 16; ++i) out16[i] = d4pg::g_tcc_watchdog_host ? d4pg::g_tcc_watchdog_host[i] : 0ull;
  return D4PG_OK;
}
namespace d4pg {

void tcc_pack_begin(TccPackArgs& p, uint8_t* dst) { p.n = 0; p.total_blocks = 0; p.dst = dst; }
int tcc_pack_add(TccPackArgs& p, const float* W, int ldw, int mode, int N, int K) {
  if (p.n >= TCC_MAX_USES) return -1;
  TccPackUse& u = p.use[p.n];
  u.W = W; u.ldw = ldw; u.mode = mode; u.N = N; u.K = K;
  u.nslices = cdiv(N, TCC_BN); u.nchunks = cdiv(K, TCC_KC);
  u.block_begin = p.total_blocks;
  u.dst_off = (long long)(p.total_blocks) * TCC_W_CHUNK;
  p.total_blocks += u.nslices * u.nchunks;
  return p.n++;
}
long long tcc_pack_bytes(const TccPackArgs& p) { return (long long)(p.total_blocks) * TCC_W_CHUNK; }
// the set's images start `first_byte` into the buffer `dst` (dst_off of every use is relative to the set's own start)
void tcc_pack_set_base(TccPackArgs& p, uint8_t* dst, long long first_byte) { p.dst = dst + first_byte; }
int launch_tcc_pack(const TccPackArgs& p, cudaStream_t st) {
  D4PG_REQUIRE(p.n > 0 && p.dst, D4PG_EINVAL, "launch_tcc_pack: nothing to pack");
  tcc_pack_kernel<<<p.total_blocks, 256, 0, st>>>(p);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

// ---- chain construction -----------------------------------------------------------------------------------
int64_t tcc_xchg_floats(int B) {
  return int64_t(TCC_MAX_CHAINS) * cdiv(B, TCC_ROWS) * TCC_PLANES * (TCC_PLANE_BYTES / 4);
}
void tcc_args_begin(TccArgs& a, int B, uint8_t* xchg, int passes) {
  memset(&a, 0, sizeof(a));
  a.B = B; a.row_blocks = cdiv(B, TCC_ROWS); a.xchg = xchg; a.passes = passes;
}
void tcc_chain_x0(TccArgs& a, int c, const float* src, int ld, int cols) {
  a.chain[c].x0 = src; a.chain[c].x0ld = ld; a.chain[c].x0cols = cols;
}
void tcc_chain_pre(TccArgs& a, int c, const float* src, int ld, int cols) {
  a.chain[c].pre = src; a.chain[c].preld = ld; a.chain[c].precols = cols;
}
int tcc_slot_begin(TccArgs& a, int c) {
  if (c >= a.nchains) a.nchains = c + 1;
  TccChain& ch = a.chain[c];
  const int l = ch.nslots++;
  if (l < TCC_MAX_SLOTS) { ch.slot[l] = TccSlot{}; ch.slot[l].g[0].pub = ch.slot[l].g[1].pub = -1; }
  return l;
}
static void tcc_push_chunk(TccSlot& s, int kind, int plane, int chunk) {
  if (s.nchunks < TCC_MAX_CHUNKS) s.ch[s.nchunks] = TccChunk{short(kind), short(plane), short(chunk), 0};
  ++s.nchunks;
}
void tcc_slot_src_x(TccArgs& a, int c, int slot) { tcc_push_chunk(a.chain[c].slot[slot], TCC_SRC_X, 0, 0); }
void tcc_slot_src_pre(TccArgs& a, int c, int slot) {
  const int n = cdiv(a.chain[c].precols, TCC_KC);
  for (int i = 0; i < n; ++i) tcc_push_chunk(a.chain[c].slot[slot], TCC_SRC_PRE, 0, i);
}
void tcc_slot_src_plane(TccArgs& a, int c, int slot, int plane, int nchunks) {
  for (int i = 0; i < nchunks; ++i) tcc_push_chunk(a.chain[c].slot[slot], TCC_SRC_IMG, plane, i);
}
void tcc_slot_reconvert_x(TccArgs& a, int c, int slot, const float* src, int ld, int cols) {
  TccSlot& s = a.chain[c].slot[slot];
  s.xsrc = src; s.xld = ld; s.xcols = cols;
}
int tcc_slot_group(TccArgs& a, int c, int slot, const TccImage& img, int epi, const float* bias,
                   const float* aux, int ldaux, float* C, int ldc, int publish) {
  TccChain& ch = a.chain[c];
  TccSlot& s = ch.slot[slot];
  const int gi = s.ngroups++;
  if (gi >= TCC_MAX_GROUPS) return -1;
  TccGroup& g = s.g[gi];
  g.wimg = img.ptr; g.bias = bias; g.aux = aux; g.ldaux = ldaux; g.C = C; g.ldc = ldc;
  g.N = img.N; g.epi = epi; g.kchunks = img.kchunks;
  g.pub = publish ? ch.nplanes++ : -1;
  return g.pub;
}

int launch_mlp_tc_chain(TccArgs& a, cudaStream_t st) {
  D4PG_REQUIRE(a.nchains > 0 && a.nchains <= TCC_MAX_CHAINS, D4PG_EINVAL, "launch_mlp_tc_chain: %d chains", a.nchains);
  D4PG_REQUIRE(a.passes == 1 || a.passes == 3, D4PG_EINVAL, "launch_mlp_tc_chain: passes %d", a.passes);
  constexpr int gmax = 2;                            // chunks per bulk copy of a plane (see below)
  for (int c = 0; c < a.nchains; ++c) {
    TccChain& ch = a.chain[c];
    bool x_clobbered = false;
    D4PG_REQUIRE(ch.nslots > 0 && ch.nslots <= TCC_MAX_SLOTS, D4PG_EINVAL, "launch_mlp_tc_chain: chain %d has %d slots", c, ch.nslots);
    D4PG_REQUIRE(ch.nplanes <= TCC_PLANES, D4PG_ENOTSUP, "launch_mlp_tc_chain: chain %d publishes %d planes", c, ch.nplanes);
    D4PG_REQUIRE(!ch.x0 || (ch.x0cols <= TCC_KC && ch.x0ld % 4 == 0 && ch.x0ld >= ch.x0cols), D4PG_ENOTSUP, "launch_mlp_tc_chain: bad X source");
    D4PG_REQUIRE(!ch.pre || (ch.precols <= 8 * TCC_KC && ch.preld % 4 == 0 && ch.preld >= ch.precols), D4PG_ENOTSUP,
                 "launch_mlp_tc_chain: bad first-slot source");
    int planes_seen = 0;
    for (int l = 0; l < ch.nslots; ++l) {
      TccSlot& s = ch.slot[l];
      D4PG_REQUIRE(s.ngroups >= 1 && s.ngroups <= TCC_MAX_GROUPS, D4PG_EINVAL, "launch_mlp_tc_chain: slot %d has %d groups", l, s.ngroups);
      D4PG_REQUIRE(s.nchunks >= 1 && s.nchunks <= TCC_MAX_CHUNKS && s.ngroups * s.nchunks <= TCC_MAX_CHUNKS, D4PG_ENOTSUP,
                   "launch_mlp_tc_chain: slot %d: %d groups x %d chunks exceed the weight buffer", l, s.ngroups, s.nchunks);
      // A buffers are direct-mapped: the j-th non-resident chunk of a slot lives in buffer j (0..7); a 9th one takes
      // buffer 8, the resident X chunk's, if this slot does not read X (and X is dead from then on).  Consecutive
      // chunks of one plane in consecutive buffers travel as ONE bulk copy (at most `gmax` chunks each, so that the
      // MMAs of the first chunks overlap the arrival of the rest).
      int nring = 0;
      bool uses_x = false;
      for (int i = 0; i < s.nchunks; ++i) uses_x = uses_x || s.ch[i].kind == TCC_SRC_X;
      s.nloads = 0;
      for (int i = 0; i < s.nchunks; ++i) {
        TccChunk& k = s.ch[i];
        if (k.kind == TCC_SRC_IMG) D4PG_REQUIRE(k.plane >= 0 && k.plane < planes_seen && k.chunk < TCC_CLUSTER, D4PG_EINVAL,
                                                 "launch_mlp_tc_chain: slot %d reads plane %d before it is published", l, k.plane);
        if (k.kind == TCC_SRC_PRE) D4PG_REQUIRE(l == 0 && ch.pre && k.chunk == nring && nring < 8, D4PG_EINVAL, "launch_mlp_tc_chain: pre chunks belong to slot 0, in order");
        if (k.kind == TCC_SRC_X) {
          D4PG_REQUIRE(ch.x0 != nullptr && !x_clobbered, D4PG_EINVAL, "launch_mlp_tc_chain: slot %d reads X but the chain has none (or it was overwritten)", l);
          k.buf = 8;
          continue;
        }
        if (nring < 8) k.buf = short(nring);
        else {
          D4PG_REQUIRE(nring == 8 && !uses_x && k.kind == TCC_SRC_IMG, D4PG_ENOTSUP, "launch_mlp_tc_chain: slot %d needs more than 9 A buffers", l);
          k.buf = 8; x_clobbered = true;
        }
        ++nring;
        if (k.kind == TCC_SRC_IMG) {
          TccLoad* cur = s.nloads ? &s.ld[s.nloads - 1] : nullptr;
          if (cur && cur->plane == k.plane && cur->chunk0 + cur->count == k.chunk && cur->buf0 + cur->count == k.buf && cur->count < gmax) ++cur->count;
          else s.ld[s.nloads++] = TccLoad{k.plane, k.chunk, k.buf, 1};
        }
      }
      // MMA-side view: chunk c <-> A buffer c + boff, wait on full[c + boff] where a copy (or a pre-converted chunk) starts
      s.boff = s.ch[0].buf;
      s.wait_mask = 0;
      for (int i = 0; i < s.nchunks; ++i) {
        D4PG_REQUIRE(s.ch[i].buf == s.boff + i, D4PG_ENOTSUP, "launch_mlp_tc_chain: slot %d: chunk %d is not in A buffer %d", l, i, s.boff + i);
        if (s.ch[i].kind == TCC_SRC_PRE) s.wait_mask |= 1u << i;
      }
      for (int i = 0; i < s.nloads; ++i) s.wait_mask |= 1u << (s.ld[i].buf0 - s.boff);
      for (int g = 0; g < s.ngroups; ++g) {
        const TccGroup& G = s.g[g];
        D4PG_REQUIRE(G.N > 0 && G.N <= TCC_CLUSTER * TCC_BN && G.wimg, D4PG_ENOTSUP, "launch_mlp_tc_chain: group width %d", G.N);
        D4PG_REQUIRE(G.kchunks == s.nchunks, D4PG_EINVAL, "launch_mlp_tc_chain: chain %d slot %d: A operand has %d chunks, the weight image %d", c, l, s.nchunks, G.kchunks);
        D4PG_REQUIRE(!G.C || (G.ldc % 4 == 0 && G.ldc >= ((G.N + 3) & ~3) && (reinterpret_cast<uintptr_t>(G.C) & 15) == 0), D4PG_EINVAL,
                     "launch_mlp_tc_chain: output pitch");
        const bool fwd = G.epi == EPI_BIAS || G.epi == EPI_BIAS_RELU || G.epi == EPI_BIAS_TANH;
        const bool msk = G.epi == EPI_RELU_MASK || G.epi == EPI_TANH_MASK;
        D4PG_REQUIRE(!fwd || (G.bias && (reinterpret_cast<uintptr_t>(G.bias) & 15) == 0), D4PG_EINVAL, "launch_mlp_tc_chain: bias");
        D4PG_REQUIRE(!msk || (G.aux && G.ldaux % 4 == 0 && (reinterpret_cast<uintptr_t>(G.aux) & 15) == 0), D4PG_EINVAL, "launch_mlp_tc_chain: mask operand");
        if (G.pub >= 0) ++planes_seen;
      }
      if (l == 0 && ch.pre) D4PG_REQUIRE(s.g[0].N > (TCC_CLUSTER - 1) * TCC_BN, D4PG_ENOTSUP, "launch_mlp_tc_chain: the first slot must span the cluster");
    }
  }
  void (*kern)(TccArgs) = a.passes == 3 ? mlp_tc_chain_kernel<3> : mlp_tc_chain_kernel<1>;
  static bool attr_set[2] = {false, false};          // per instantiation
  const int ai = a.passes == 3 ? 1 : 0;
  if (!attr_set[ai]) {
    D4PG_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(TCC_SMEM)));
    D4PG_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, int(cudaSharedmemCarveoutMaxShared)));
    attr_set[ai] = true;
  }
  a.watchdog = tcc_watchdog_device();
  unsigned long long* dbg = debug_trace_buffer();
  a.trace = dbg ? dbg + (a.step_slot == 5 ? 384 : 256) : nullptr;
  a.step_trace = dbg ? dbg + STEP_TRACE_BASE : nullptr;
  { const char* e = getenv("D4PG_TRACE_CTA"); a.trace_cta = e ? atoi(e) : 0; if (a.trace_cta >= a.nchains * a.row_blocks * TCC_CLUSTER) a.trace_cta = 0; }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(a.nchains * a.row_blocks * TCC_CLUSTER); cfg.blockDim = dim3(TCC_THREADS);
  cfg.dynamicSmemBytes = TCC_SMEM; cfg.stream = st;
  cfg.attrs = nullptr; cfg.numAttrs = 0;              // cluster shape is compiled in (__cluster_dims__)
  D4PG_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, a));
  return D4PG_OK;
}

}  // namespace d4pg
