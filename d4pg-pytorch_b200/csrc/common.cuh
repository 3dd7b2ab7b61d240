// Shared host/device helpers for libd4pg_sm90.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/d4pg_b200.h"

namespace d4pg {

void set_error(const char* fmt, ...);

#define D4PG_CUDA_OK(expr)                                                              \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      ::d4pg::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return D4PG_ECUDA;                                                                \
    }                                                                                   \
  } while (0)

#define D4PG_REQUIRE(cond, code, ...)                                                   \
  do {                                                                                  \
    if (!(cond)) { ::d4pg::set_error(__VA_ARGS__); return (code); }                     \
  } while (0)

#define D4PG_LAUNCH_OK()                                                                \
  do {                                                                                  \
    cudaError_t _e = cudaGetLastError();                                                \
    if (_e != cudaSuccess) {                                                            \
      ::d4pg::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return D4PG_ECUDA;                                                                \
    }                                                                                   \
  } while (0)

// All kernels of a step ask for the same (maximum) shared-memory carve-out: a step mixes kernels
// with 0 KB, 14 KB, 32 KB and 197 KB of shared memory, and letting the driver pick a per-kernel
// L1/shared split makes every kernel boundary an SM reconfiguration.
#define D4PG_MAX_CARVEOUT(kernel)                                                                     \
  do {                                                                                                \
    static bool _carved = false;                                                                      \
    if (!_carved) {                                                                                   \
      cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout,                    \
                           int(cudaSharedmemCarveoutMaxShared));                                      \
      _carved = true;                                                                                 \
    }                                                                                                 \
  } while (0)

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------
// A step is ~18 small dependent kernels; at batch 256 the kernel boundaries (grid drain -> next grid
// launch) cost as much as the kernels.  Every step kernel is launched with the programmatic-stream-
// serialization attribute: it signals `launch_dependents` as soon as it starts, so the next kernel's
// CTAs are scheduled (and run their prologue) while this one is still executing, and blocks in
// `griddepcontrol.wait` until all of this kernel's memory is visible.  Captured into the CUDA graph
// as programmatic dependency edges.  Opt-in with D4PG_PDL=1 (see pdl_enabled()).
// PDL trigger position, carried in every step kernel's argument struct (`pdl` field):
//   1 = `launch_dependents` at kernel entry (next grid becomes resident early), 2 = at kernel exit
__device__ __forceinline__ void pdl_trigger_raw() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger(int mode) { if (mode == 1) pdl_trigger_raw(); }
__device__ __forceinline__ void pdl_trigger_end(int mode) { if (mode == 2) pdl_trigger_raw(); }
int pdl_mode();                      // 0 off, 1 early trigger, 2 late trigger (env D4PG_PDL)
int device_sm_count();               // SMs of the current device (grid-stride kernels size their grids by it)
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
bool pdl_enabled();
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// step timeline (D4PG_TC_TRACE): thread 0 of CTA 0 of every step kernel stamps %globaltimer at entry / exit
__device__ __forceinline__ void step_stamp(unsigned long long* tr, int slot) {
  if (tr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    tr[slot] = t;
  }
}
unsigned long long* debug_trace_buffer();
constexpr int STEP_TRACE_BASE = 96;      // stamps [96, 128) of the debug buffer: entry of kernel k at 96+k, exit at 112+k

static inline cudaStream_t as_stream(d4pg_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

__host__ __device__ static inline int64_t align4(int64_t x) { return (x + 3) & ~int64_t(3); }
__host__ __device__ static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// ---- warp helpers --------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- Philox4x32-10 (counter-based RNG for device-side sampling) -----------------------
struct Philox {
  __device__ static inline void round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
    uint32_t hi0 = __umulhi(M0, c[0]), lo0 = M0 * c[0];
    uint32_t hi1 = __umulhi(M1, c[2]), lo1 = M1 * c[2];
    uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
  }
  // 53-bit uniform in [0,1), same construction as CPython's random.random():
  // (a>>5, b>>6) -> (a*2^26 + b) / 2^53.
  __device__ static inline double uniform53(uint64_t seed, uint64_t counter, uint32_t lane) {
    uint32_t c[4] = {uint32_t(counter), uint32_t(counter >> 32), lane, 0x9E3779B9u};
    uint32_t k0 = uint32_t(seed), k1 = uint32_t(seed >> 32);
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      round(c, k0, k1);
      k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    uint32_t a = c[0] >> 5, b = c[1] >> 6;
    return (double(a) * 67108864.0 + double(b)) * (1.0 / 9007199254740992.0);
  }
};

// ---- network layout ------------------------------------------------------------------
// GEMM epilogues: a forward layer's bias + activation, or the activation derivative a dX applies to its output
enum GemmEpi {
  EPI_NONE = 0, EPI_BIAS = 1, EPI_BIAS_RELU = 2, EPI_BIAS_TANH = 3,
  EPI_RELU_MASK = 4,   // C *= (aux > 0)
  EPI_TANH_MASK = 5    // C *= (1 - aux^2)
};
struct NetDims {
  int in[4], out[4];        // per layer fc1, fc2, fc2_2, fc3
  int ld[4];                // row pitch of each weight matrix in floats: in[] rounded up to 4 (16-B rows,
                            // so every operand is TMA- and float4-addressable); pad columns stay zero
  int epi[4];               // forward epilogue of each layer
  int64_t w_off[4], b_off[4];
  int64_t total;
};
// The mask the dX of layer l applies to its input: the derivative of the activation that produced that input.  A ReLU
// on layer l-1 gives (input > 0); no activation (the actor's fc2), or the network input (l = 0), gives none.
static inline int dx_mask(const NetDims& d, int l) {
  return l > 0 && d.epi[l - 1] == EPI_BIAS_RELU ? EPI_RELU_MASK : EPI_NONE;
}
__host__ __device__ static inline int pitch4(int x) { return (x + 3) & ~3; }
NetDims actor_dims(int obs_dim, int act_dim);
NetDims critic_dims(int obs_dim, int act_dim, int n_atoms);

}  // namespace d4pg
