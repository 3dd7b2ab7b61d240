// Device code of the fused Adam + Polyak update.
#pragma once
#include "adam.cuh"
#include "tc_common.cuh"

namespace d4pg {

// mean over the batch of the per-row loss terms (ddpg.py:217 `.mean()`, ddpg.py:238 `.mean()`),
// fixed-order single-block reduction so the reported scalars are run-to-run deterministic.
__device__ __forceinline__ void loss_reduce_block(const float* loss_rows, const float* pi_rows, int B, float inv_count,
                                                  float* out, float (*red)[8]) {
  float a = 0.f, b = 0.f;
  for (int i = threadIdx.x; i < B; i += 256) { a += loss_rows[i]; if (pi_rows) b += pi_rows[i]; }
  a = warp_sum(a); b = warp_sum(b);
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = b; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float sa = 0.f, sb = 0.f;
    for (int w = 0; w < 8; ++w) { sa += red[0][w]; sb += red[1][w]; }
    out[0] = sa * inv_count; out[1] = sb * inv_count;
  }
}

// tail: reported losses + advance the base counters for the NEXT step (nobody in the same kernel /
// phase reads them: the derived scalars were written by the step's first kernel).  One 256-thread CTA.
__device__ __forceinline__ void adam_tail(const AdamArgs& a, float (*red)[8]) {
  if (a.loss_out) loss_reduce_block(a.loss_rows, a.pi_rows, a.B, a.inv_count, a.loss_out, red);
  if (threadIdx.x == 0 && a.clock) { a.clock->adam_step += 1; a.clock->beta_t += 1; a.clock->steps_done += 1; }
}

// fp64 sum over a warp, every lane holding the same bits (fp add commutes, so both sides of each exchange agree)
__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Clipping coefficient of segment `s` from the GRAD_NORM_CTAS partial sums grad_sqnorm_kernel left: warp 0 sums them in
// a fixed order and broadcasts through shared memory, so every CTA of the launch derives the same bits and no grid-wide
// synchronisation is needed.  norm = |scale| * sqrt(sum g^2) is the norm of the scaled gradient;
// coef = scale * min(1, max_norm / (norm + 1e-6)) formed in fp64 and cast once: exactly `scale` when nothing is clipped.
__device__ __forceinline__ float clip_coef(const AdamSeg& s, float scale, bool report, double* bcast) {
  if (threadIdx.x < 32) {
    const double sq = warp_sum_f64(s.sq_partials[threadIdx.x] + s.sq_partials[threadIdx.x + 32]);
    if (threadIdx.x == 0) *bcast = fabs(double(scale)) * sqrt(sq);
  }
  __syncthreads();
  const double norm = *bcast;
  if (report && threadIdx.x == 0 && s.norm_out) *s.norm_out = float(norm);
  return float(double(scale) * fmin(1.0, s.max_norm / (norm + GRAD_NORM_EPS)));
}

// segment `seg`, grid-stride over float4 groups: CTA bx of gx (256 threads each).  EX: the launch clips to a global norm
// and / or applies weight decay (a separate instantiation, so the plain update keeps its instructions)
template <bool EX>
__device__ __forceinline__ void adam_segment(const AdamArgs& a, int seg, int bx, int gx, double* bcast = nullptr) {
  const AdamSeg& s = a.seg[seg];
  float coef = a.grad_scale;
  if (EX && s.sq_partials) coef = clip_coef(s, a.grad_scale, bx == 0, bcast);
  float nss = s.neg_step_size, bc2s = a.bc2_sqrt;
  if (a.clock) {
    if (a.pipe_slot >= 0) {
      nss = s.clock_slot >= 0 ? a.clock->d_neg_step_size[a.pipe_slot][s.clock_slot] : nss;
      bc2s = a.clock->d_bc2_sqrt[a.pipe_slot];
    } else {
      nss = s.clock_slot >= 0 ? a.clock->neg_step_size[s.clock_slot] : nss;
      bc2s = a.clock->bc2_sqrt;
    }
  }
  const int64_t n4 = s.n >> 2;
  float4* p4 = reinterpret_cast<float4*>(s.p);
  const float4* g4 = reinterpret_cast<const float4*>(s.g);
  float4* m4 = reinterpret_cast<float4*>(s.m);
  float4* v4 = reinterpret_cast<float4*>(s.v);
  float4* t4 = reinterpret_cast<float4*>(s.target);
  float4* go4 = reinterpret_cast<float4*>(s.g_out);
  if (a.npeers > 0 && a.my_flags) peer_wait_all(a.my_flags, a.npeers);   // every rank signalled this step (local inbox)
  for (int64_t i = bx * int64_t(256) + threadIdx.x; i < n4; i += int64_t(gx) * 256) {
    float4 g;
    if (a.mc_g) {                                           // one instruction, one NVLink hop: the switch adds the N ranks' values
      asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                   : "=f"(g.x), "=f"(g.y), "=f"(g.z), "=f"(g.w) : "l"(reinterpret_cast<const float4*>(a.mc_g + s.g_off) + i) : "memory");
      if (go4) go4[i] = g;
    } else if (a.npeers > 0 && !a.peer_reduced) {
      g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int r = 0; r < D4PG_MAX_PEERS; ++r)
        if (r < a.npeers) {
          const float4 t = __ldcg(reinterpret_cast<const float4*>(a.peer_g[r] + s.g_off) + i);
          g.x += t.x; g.y += t.y; g.z += t.z; g.w += t.w;
        }
      if (go4) go4[i] = g;
    } else {
      g = (a.npeers > 0) ? __ldcg(g4 + i) : g4[i];          // peer mode: written by remote ranks, bypass L1
      if (go4) go4[i] = g;
    }
    float4 p = p4[i], m = m4[i], v = v4[i];
    float4 t = s.target ? t4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    float* pp = &p.x; float* gg = &g.x; float* mm = &m.x; float* vv = &v.x; float* tt = &t.x;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float gr;
      if (EX) {
        gr = __fmul_rn(gg[c], coef);
        if (s.wd != 0.f) gr = __fadd_rn(gr, __fmul_rn(s.wd, pp[c]));
      } else gr = gg[c] * a.grad_scale;
      mm[c] = fmaf(a.w1, gr - mm[c], mm[c]);                                   // lerp, weight < 0.5
      vv[c] = __fadd_rn(__fmul_rn(vv[c], a.beta2), __fmul_rn(__fmul_rn(a.w2, gr), gr));
      const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vv[c]), bc2s), a.eps);
      pp[c] = __fadd_rn(pp[c], __fmul_rn(nss, __fdiv_rn(mm[c], denom)));
      tt[c] = __fadd_rn(__fmul_rn(a.one_minus_tau, tt[c]), __fmul_rn(a.tau, pp[c]));
    }
    p4[i] = p; m4[i] = m; v4[i] = v;
    if (s.target) t4[i] = t;
    if (s.nimg) {                                             // forward operand images of the tensor-core chains
      const int64_t e = i << 2;
#pragma unroll
      for (int L = 0; L < 4; ++L) {
        if (L >= s.nimg || e < s.imgl[L].w_off || e >= s.imgl[L].w_end) continue;
        const AdamImgLayer& I = s.imgl[L];
        const int rel = int(e - I.w_off), n = rel / I.ld, k = rel - n * I.ld;     // row pitch is a multiple of 4: one float4 = 4 k of one row
        const uint32_t off = uint32_t(((n >> 5) * I.nchunks + (k >> 5)) * 8192) + tc::sw128_kmajor_off(n & 31, k & 31);
        const float4 ph = make_float4(tc::tf32_hi(p.x), tc::tf32_hi(p.y), tc::tf32_hi(p.z), tc::tf32_hi(p.w));
        *reinterpret_cast<float4*>(I.img + off) = ph;
        *reinterpret_cast<float4*>(I.img + 4096 + off) =
            make_float4(tc::tf32_lo(p.x, ph.x), tc::tf32_lo(p.y, ph.y), tc::tf32_lo(p.z, ph.z), tc::tf32_lo(p.w, ph.w));
        if (I.img_t) {
          const float4 th = make_float4(tc::tf32_hi(t.x), tc::tf32_hi(t.y), tc::tf32_hi(t.z), tc::tf32_hi(t.w));
          *reinterpret_cast<float4*>(I.img_t + off) = th;
          *reinterpret_cast<float4*>(I.img_t + 4096 + off) =
              make_float4(tc::tf32_lo(t.x, th.x), tc::tf32_lo(t.y, th.y), tc::tf32_lo(t.z, th.z), tc::tf32_lo(t.w, th.w));
        }
      }
    }
  }
}


}  // namespace d4pg
