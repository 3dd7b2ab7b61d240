// Data-parallel communicator: one flat-buffer all-reduce of the gradients per step over
// NVLink 5 / NVSwitch.  The reference has no collective at all (its multi-worker mode is
// Hogwild over shared CPU memory: main.py:394-405, ddpg.py:104-108, shared_adam.py:16-17);
// this is the synchronous-DP equivalent described in SURVEY.md section 8e.
// NCCL is bound at run time (dlopen) so the .so has no link-time dependency on it.
#include "internal.cuh"
#include <cuda.h>          // driver-API types for the multicast (NVLS) objects; entry points are resolved at run time
#include <dlfcn.h>
#include <unistd.h>
#include <stdlib.h>
#include <string.h>
#include <new>
#include <algorithm>

using d4pg::D4PG_MAX_PEERS;
using d4pg::PeerInfo;

namespace {
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
enum { ncclFloat32 = 7, ncclSum = 0 };

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
NcclApi g_nccl;

int load_nccl() {
  if (g_nccl.ok) return D4PG_OK;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  void* lib = nullptr;
  for (const char* n : names) { lib = dlopen(n, RTLD_NOW | RTLD_NOLOAD); if (lib) break; }   // torch's copy, if loaded
  const char* env = getenv("D4PG_NCCL_LIB");
  if (!lib && env) lib = dlopen(env, RTLD_NOW | RTLD_GLOBAL);
  for (const char* n : names) { if (lib) break; lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); }
  if (!lib) { d4pg::set_error("NCCL not loadable: %s (set D4PG_NCCL_LIB)", dlerror()); return D4PG_ENCCL; }
  g_nccl.lib = lib;
  *(void**)(&g_nccl.GetUniqueId) = dlsym(lib, "ncclGetUniqueId");
  *(void**)(&g_nccl.CommInitRank) = dlsym(lib, "ncclCommInitRank");
  *(void**)(&g_nccl.CommDestroy) = dlsym(lib, "ncclCommDestroy");
  *(void**)(&g_nccl.AllReduce) = dlsym(lib, "ncclAllReduce");
  *(void**)(&g_nccl.GetErrorString) = dlsym(lib, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.CommDestroy || !g_nccl.AllReduce) {
    d4pg::set_error("NCCL symbols missing in loaded library");
    return D4PG_ENCCL;
  }
  g_nccl.ok = true;
  return D4PG_OK;
}
#define NCCL_OK(expr)                                                                          \
  do {                                                                                         \
    ncclResult_t _r = (expr);                                                                  \
    if (_r != 0) {                                                                             \
      d4pg::set_error("%s -> NCCL error %d (%s)", #expr, _r,                                   \
                      g_nccl.GetErrorString ? g_nccl.GetErrorString(_r) : "?");                \
      return D4PG_ENCCL;                                                                       \
    }                                                                                          \
  } while (0)
}  // namespace

struct d4pg_comm {
  ncclComm_t comm; int rank, world;
  // ---- fused all-reduce over peer memory (d4pg_comm_peer_*) ----------------------------------------------------
  // One cudaMalloc block per rank, exported with CUDA IPC: [2][n] gradient halves (double buffer), [n] reduced
  // gradient, two flag lines (256 B apart).
  float* xbuf; int64_t xn; unsigned long long* flags;       // local block
  void* peer_base[D4PG_MAX_PEERS];                          // opened IPC mappings (nullptr for self)
  float* peer_x[D4PG_MAX_PEERS]; unsigned long long* peer_flag[D4PG_MAX_PEERS];
  bool peer_ready;
  // ---- in-switch reduction (NVLS): one multicast object over all ranks' gradient buffers (d4pg_comm_mc_*) -------------
  // Every rank binds its own physical [2][n] gradient buffer to the same multicast object; `mc_ptr` is the multicast
  // mapping (a multimem.ld_reduce on it returns the SUM over all ranks, computed by the NVSwitch), `mc_uc` the ordinary
  // mapping of this rank's buffer (what its dW kernel writes).
  CUmemGenericAllocationHandle mc_handle, mc_mem;
  CUdeviceptr mc_ptr, mc_uc; size_t mc_size; int mc_dev;
  bool mc_have_handle, mc_ready;
};

namespace d4pg {
// "my gradient half of this step is complete" + "wait until every peer's is" as a launch of its own (the level plan has
// several dW launches): one CTA publishes, then polls its local inbox.
__global__ void peer_barrier_kernel(PeerSignal sig) {
  if (threadIdx.x == 0) peer_signal_last_cta(sig, 1u);
  __syncthreads();
  peer_wait_all(sig.local, sig.world);
  __threadfence_system();
}

PeerSignal comm_peer_signal(const PeerInfo& info, int kind) {
  PeerSignal s{};
  s.world = info.world;
  s.local = info.flag[info.rank] + kind * 64;
  for (int p = 0; p < info.world; ++p) s.inbox[p] = info.flag[p] + kind * 64 + 8 + info.rank;
  return s;
}

bool comm_peer_info(d4pg_comm* c, PeerInfo* out) {
  if (!c || !c->peer_ready) return false;
  if (!out) return true;
  out->world = c->world; out->rank = c->rank; out->n = c->xn;
  out->mc = c->mc_ready ? reinterpret_cast<const float*>(c->mc_ptr) : nullptr;
  out->mc_uc = c->mc_ready ? reinterpret_cast<float*>(c->mc_uc) : nullptr;
  for (int r = 0; r < c->world; ++r) {
    out->x[r] = c->peer_x[r]; out->red[r] = c->peer_x[r] + 2 * c->xn;
    out->flag[r] = c->peer_flag[r]; out->flag2[r] = c->peer_flag[r] + 64;
  }
  return true;
}
int comm_peer_barrier(d4pg_comm* c, cudaStream_t st) {
  PeerInfo info{};
  D4PG_REQUIRE(comm_peer_info(c, &info), D4PG_ESTATE, "comm_peer_barrier: peers are not open");
  peer_barrier_kernel<<<1, 32, 0, st>>>(comm_peer_signal(info, 0));
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

// ---- reduce-scatter + all-gather over peer memory ---------------------------------------------------------------
// Rank r owns slice r of the flat gradient.  After every rank's dW published flag1 for this step, rank r reads slice r of
// all N halves (N-1 of them over NVLink), sums them IN RANK ORDER and stores the result into slice r of every rank's
// reduced buffer (N-1 remote stores).  Every element is reduced by exactly one rank, so all replicas consume the same
// bits.  Per rank: (N-1)/N x 1.15 MB in and out, instead of pulling all N halves (N x 1.15 MB in).  The last CTA
// publishes flag2; the fused Adam kernel waits for all ranks' flag2 and then streams its LOCAL reduced buffer.
struct PeerRSArgs {
  int world, rank; int64_t n4, lo4, hi4, half_off;
  const float* g[D4PG_MAX_PEERS]; float* red[D4PG_MAX_PEERS];
  const unsigned long long* my_f1;              // this rank's flag block of signal 0 (local inbox: every rank's dW is done)
  d4pg::PeerSignal sig2;                        // signal 1: this rank's slice is reduced and pushed
};
__global__ void __launch_bounds__(256) peer_reduce_scatter_kernel(const PeerRSArgs a) {
  d4pg::peer_wait_all(a.my_f1, a.world);
  for (int64_t i = a.lo4 + int64_t(blockIdx.x) * 256 + threadIdx.x; i < a.hi4; i += int64_t(gridDim.x) * 256) {
    float4 t[D4PG_MAX_PEERS];
#pragma unroll
    for (int r = 0; r < D4PG_MAX_PEERS; ++r)
      if (r < a.world) t[r] = __ldcg(reinterpret_cast<const float4*>(a.g[r] + a.half_off) + i);     // all loads in flight
    float4 s = t[0];
#pragma unroll
    for (int r = 1; r < D4PG_MAX_PEERS; ++r)
      if (r < a.world) { s.x += t[r].x; s.y += t[r].y; s.z += t[r].z; s.w += t[r].w; }
#pragma unroll
    for (int r = 0; r < D4PG_MAX_PEERS; ++r)
      if (r < a.world) reinterpret_cast<float4*>(a.red[r])[i] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) { __threadfence_system(); d4pg::peer_signal_last_cta(a.sig2, gridDim.x); }
}
int comm_peer_reduce_scatter(d4pg_comm* c, int parity, cudaStream_t st) {
  PeerInfo info{};
  D4PG_REQUIRE(comm_peer_info(c, &info), D4PG_ESTATE, "comm_peer_reduce_scatter: peers are not open");
  PeerRSArgs a{};
  a.world = info.world; a.rank = info.rank; a.n4 = info.n >> 2;
  const int64_t per = (a.n4 + info.world - 1) / info.world;
  a.lo4 = std::min<int64_t>(a.n4, per * info.rank); a.hi4 = std::min<int64_t>(a.n4, a.lo4 + per);
  a.half_off = int64_t(parity) * info.n;
  for (int r = 0; r < info.world; ++r) { a.g[r] = info.x[r]; a.red[r] = info.red[r]; }
  a.my_f1 = info.flag[info.rank]; a.sig2 = comm_peer_signal(info, 1);
  const int blocks = int(std::max<int64_t>(1, std::min<int64_t>(2 * device_sm_count(), (a.hi4 - a.lo4 + 255) / 256)));
  peer_reduce_scatter_kernel<<<blocks, 256, 0, st>>>(a);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

// ---- two-phase in-switch reduction (NVLS) ------------------------------------------------------------------------
// Rank r owns slice r: ONE multimem.ld_reduce per element returns the sum over all ranks (added by the NVSwitch), ONE
// multimem.st broadcasts it into slice r of every rank's reduced buffer.  Per GPU 2 x 1.15 MB cross the links instead of
// N x 1.15 MB when every rank ld_reduces everything; the price is a second flag hop (signal 1) before Adam.
struct PeerMC2Args {
  int world; int64_t lo4, hi4;
  const float* mc_half; float* mc_red;          // multicast addresses: this step's gradient half, the reduced buffer
  const unsigned long long* my_f1;              // local inbox of signal 0: every rank's dW is done
  d4pg::PeerSignal sig2;                        // signal 1: my slice is reduced and broadcast
};
__global__ void __launch_bounds__(256) mc_reduce_bcast_kernel(const PeerMC2Args a) {
  d4pg::peer_wait_all(a.my_f1, a.world);
  for (int64_t i = a.lo4 + int64_t(blockIdx.x) * 256 + threadIdx.x; i < a.hi4; i += int64_t(gridDim.x) * 256) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(reinterpret_cast<const float4*>(a.mc_half) + i) : "memory");
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};"
                 :: "l"(reinterpret_cast<float4*>(a.mc_red) + i), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) { __threadfence_system(); d4pg::peer_signal_last_cta(a.sig2, gridDim.x); }
}
int comm_mc_reduce_bcast(d4pg_comm* c, int parity, cudaStream_t st) {
  PeerInfo info{};
  D4PG_REQUIRE(comm_peer_info(c, &info) && info.mc, D4PG_ESTATE, "comm_mc_reduce_bcast: multicast is not set up");
  PeerMC2Args a{};
  a.world = info.world;
  const int64_t n4 = info.n >> 2, per = (n4 + info.world - 1) / info.world;
  a.lo4 = std::min<int64_t>(n4, per * info.rank); a.hi4 = std::min<int64_t>(n4, a.lo4 + per);
  a.mc_half = info.mc + int64_t(parity) * info.n;
  a.mc_red = const_cast<float*>(info.mc) + 2 * info.n;
  a.my_f1 = info.flag[info.rank]; a.sig2 = comm_peer_signal(info, 1);
  const int blocks = int(std::max<int64_t>(1, std::min<int64_t>(2 * device_sm_count(), (a.hi4 - a.lo4 + 255) / 256)));
  mc_reduce_bcast_kernel<<<blocks, 256, 0, st>>>(a);
  D4PG_LAUNCH_OK();
  return D4PG_OK;
}

int comm_allreduce(d4pg_comm* c, float* buf, int64_t n, cudaStream_t st) {
  D4PG_REQUIRE(c && buf && n > 0, D4PG_EINVAL, "comm_allreduce: bad arguments");
  NCCL_OK(g_nccl.AllReduce(buf, buf, size_t(n), ncclFloat32, ncclSum, c->comm, st));
  return D4PG_OK;
}
}  // namespace d4pg

extern "C" int32_t d4pg_comm_unique_id(uint8_t* id128) {
  D4PG_REQUIRE(id128, D4PG_EINVAL, "d4pg_comm_unique_id: null argument");
  int rc = load_nccl();
  if (rc) return rc;
  ncclUniqueId id;
  NCCL_OK(g_nccl.GetUniqueId(&id));
  memcpy(id128, id.internal, 128);
  return D4PG_OK;
}

extern "C" int32_t d4pg_comm_create(const uint8_t* id128, int32_t rank, int32_t world, d4pg_comm_t** out) {
  D4PG_REQUIRE(id128 && out && world >= 1 && rank >= 0 && rank < world, D4PG_EINVAL, "d4pg_comm_create: bad arguments");
  int rc = load_nccl();
  if (rc) return rc;
  ncclUniqueId id;
  memcpy(id.internal, id128, 128);
  d4pg_comm* c = new (std::nothrow) d4pg_comm();
  D4PG_REQUIRE(c, D4PG_EINVAL, "d4pg_comm_create: out of host memory");
  c->rank = rank; c->world = world;
  c->xbuf = nullptr; c->xn = 0; c->flags = nullptr; c->peer_ready = false;
  c->mc_handle = 0; c->mc_mem = 0; c->mc_ptr = 0; c->mc_uc = 0; c->mc_size = 0; c->mc_dev = 0; c->mc_have_handle = false; c->mc_ready = false;
  for (int i = 0; i < D4PG_MAX_PEERS; ++i) { c->peer_base[i] = nullptr; c->peer_x[i] = nullptr; c->peer_flag[i] = nullptr; }
  ncclResult_t r = g_nccl.CommInitRank(&c->comm, world, id, rank);
  if (r != 0) {
    d4pg::set_error("ncclCommInitRank failed: %d (%s)", r, g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    delete c; return D4PG_ENCCL;
  }
  *out = c;
  return D4PG_OK;
}

extern "C" int32_t d4pg_comm_destroy(d4pg_comm_t* c) {
  if (!c) return D4PG_OK;
  if (g_nccl.ok && c->comm) g_nccl.CommDestroy(c->comm);
  for (int i = 0; i < D4PG_MAX_PEERS; ++i) if (c->peer_base[i]) cudaIpcCloseMemHandle(c->peer_base[i]);
  if (c->xbuf) cudaFree(c->xbuf);
  delete c;
  return D4PG_OK;
}

extern "C" int32_t d4pg_comm_allreduce_sum(d4pg_comm_t* c, float* buf, int64_t n, d4pg_stream_t stream) {
  return d4pg::comm_allreduce(c, buf, n, d4pg::as_stream(stream));
}

// ---- fused all-reduce over peer memory -------------------------------------------------------------------------
extern "C" int32_t d4pg_comm_peer_alloc(d4pg_comm_t* c, int64_t n_floats, uint8_t* handle64) {
  D4PG_REQUIRE(c && handle64 && n_floats > 0, D4PG_EINVAL, "d4pg_comm_peer_alloc: bad arguments");
  D4PG_REQUIRE(c->world <= D4PG_MAX_PEERS, D4PG_ENOTSUP, "d4pg_comm_peer_alloc: at most %d ranks (one node)", D4PG_MAX_PEERS);
  D4PG_REQUIRE(!c->xbuf, D4PG_ESTATE, "d4pg_comm_peer_alloc: already allocated");
  const int64_t n = (n_floats + 31) & ~int64_t(31);
  const size_t bytes = size_t(3 * n) * sizeof(float) + 1024;  // [2][n] halves + [n] reduced + two flag blocks of 512 B
  D4PG_CUDA_OK(cudaMalloc(reinterpret_cast<void**>(&c->xbuf), bytes));
  D4PG_CUDA_OK(cudaMemset(c->xbuf, 0, bytes));
  D4PG_CUDA_OK(cudaDeviceSynchronize());
  c->xn = n; c->flags = reinterpret_cast<unsigned long long*>(c->xbuf + 3 * n);
  cudaIpcMemHandle_t h;
  static_assert(sizeof(h) == 64, "CUDA IPC handles are 64 bytes");
  D4PG_CUDA_OK(cudaIpcGetMemHandle(&h, c->xbuf));
  memcpy(handle64, &h, 64);
  return D4PG_OK;
}

extern "C" int32_t d4pg_comm_peer_open(d4pg_comm_t* c, const uint8_t* all_handles) {
  D4PG_REQUIRE(c && all_handles && c->xbuf, D4PG_ESTATE, "d4pg_comm_peer_open: call d4pg_comm_peer_alloc first");
  for (int r = 0; r < c->world; ++r) {
    if (r == c->rank) { c->peer_x[r] = c->xbuf; c->peer_flag[r] = c->flags; continue; }
    cudaIpcMemHandle_t h;
    memcpy(&h, all_handles + size_t(r) * 64, 64);
    void* base = nullptr;
    D4PG_CUDA_OK(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
    c->peer_base[r] = base;
    c->peer_x[r] = static_cast<float*>(base);
    c->peer_flag[r] = reinterpret_cast<unsigned long long*>(static_cast<float*>(base) + 3 * c->xn);
  }
  c->peer_ready = true;
  return D4PG_OK;
}
extern "C" int32_t d4pg_comm_peer_ready(const d4pg_comm_t* c) { return (c && c->peer_ready) ? 1 : 0; }
/* some rank could not map its peers: every rank drops back to the NCCL all-reduce */
extern "C" int32_t d4pg_comm_peer_disable(d4pg_comm_t* c) {
  D4PG_REQUIRE(c, D4PG_EINVAL, "d4pg_comm_peer_disable: null handle");
  c->peer_ready = false;
  for (int i = 0; i < D4PG_MAX_PEERS; ++i) {
    if (c->peer_base[i]) { cudaIpcCloseMemHandle(c->peer_base[i]); c->peer_base[i] = nullptr; }
    c->peer_x[i] = nullptr; c->peer_flag[i] = nullptr;
  }
  return D4PG_OK;
}

// ---- in-switch reduction over NVLink / NVSwitch (NVLS multicast objects) ---------------------------------------------
// Setup is collective and driven by the host binding (dist.py): every rank checks support; rank 0 creates the multicast
// object and exports it as a POSIX file descriptor, the other ranks receive the descriptor over a Unix socket and import
// it; every rank adds its device; after a barrier every rank creates its physical buffer, binds it and maps both views.
namespace {
struct DrvApi {
  CUresult (*DeviceGet)(CUdevice*, int) = nullptr;
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
  CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags) = nullptr;
  CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*) = nullptr;
  CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice) = nullptr;
  CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long) = nullptr;
  CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
  CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  bool ok = false, tried = false;
};
DrvApi g_drv;
bool load_drv() {
  if (g_drv.tried) return g_drv.ok;
  g_drv.tried = true;
  bool ok = true;
  auto get = [&](const char* name, void** fn) {
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(name, fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !*fn) ok = false;
  };
  get("cuDeviceGet", (void**)&g_drv.DeviceGet);
  get("cuDeviceGetAttribute", (void**)&g_drv.DeviceGetAttribute);
  get("cuMulticastGetGranularity", (void**)&g_drv.MulticastGetGranularity);
  get("cuMulticastCreate", (void**)&g_drv.MulticastCreate);
  get("cuMulticastAddDevice", (void**)&g_drv.MulticastAddDevice);
  get("cuMulticastBindMem", (void**)&g_drv.MulticastBindMem);
  get("cuMemExportToShareableHandle", (void**)&g_drv.MemExportToShareableHandle);
  get("cuMemImportFromShareableHandle", (void**)&g_drv.MemImportFromShareableHandle);
  get("cuMemCreate", (void**)&g_drv.MemCreate);
  get("cuMemAddressReserve", (void**)&g_drv.MemAddressReserve);
  get("cuMemMap", (void**)&g_drv.MemMap);
  get("cuMemSetAccess", (void**)&g_drv.MemSetAccess);
  get("cuMemGetAllocationGranularity", (void**)&g_drv.MemGetAllocationGranularity);
  (void)cudaGetLastError();
  g_drv.ok = ok;
  return ok;
}
#define DRV_OK(expr)                                                                            \
  do {                                                                                          \
    CUresult _r = (expr);                                                                       \
    if (_r != CUDA_SUCCESS) { d4pg::set_error("%s -> CUDA driver error %d", #expr, int(_r)); return D4PG_ECUDA; } \
  } while (0)
CUmulticastObjectProp mc_prop(int world, size_t size) {
  CUmulticastObjectProp p{};
  p.numDevices = unsigned(world); p.size = size; p.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR; p.flags = 0;
  return p;
}
}  // namespace

/* 1 if this rank's device supports multicast objects (NVSwitch system, driver with NVLS), else 0 */
extern "C" int32_t d4pg_comm_mc_supported(d4pg_comm_t* c) {
  if (!c || !load_drv()) return 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  CUdevice cd;
  if (g_drv.DeviceGet(&cd, dev) != CUDA_SUCCESS) return 0;
  int v = 0;
  if (g_drv.DeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, cd) != CUDA_SUCCESS) return 0;
  c->mc_dev = dev;
  return v ? 1 : 0;
}
static int mc_size_for(d4pg_comm* c, size_t* out) {
  D4PG_REQUIRE(c->xn > 0, D4PG_ESTATE, "d4pg_comm_mc_*: call d4pg_comm_peer_alloc first (the exchange length comes from it)");
  CUmulticastObjectProp p = mc_prop(c->world, 0);
  size_t gran = 0;
  // [2][n] gradient halves + [n] reduced gradient (two-phase mode: every rank broadcasts its reduced slice into it)
  p.size = size_t(3 * c->xn) * sizeof(float);
  DRV_OK(g_drv.MulticastGetGranularity(&gran, &p, CU_MULTICAST_GRANULARITY_RECOMMENDED));
  *out = ((size_t(3 * c->xn) * sizeof(float) + gran - 1) / gran) * gran;
  return D4PG_OK;
}
/* rank 0: create the multicast object for [2][n] floats per rank and export it; *fd_out is a POSIX file descriptor */
extern "C" int32_t d4pg_comm_mc_create(d4pg_comm_t* c, int32_t* fd_out) {
  D4PG_REQUIRE(c && fd_out && load_drv(), D4PG_ENOTSUP, "d4pg_comm_mc_create: multicast API not available");
  int rc = mc_size_for(c, &c->mc_size);
  if (rc) return rc;
  CUmulticastObjectProp p = mc_prop(c->world, c->mc_size);
  DRV_OK(g_drv.MulticastCreate(&c->mc_handle, &p));
  c->mc_have_handle = true;
  int fd = -1;
  DRV_OK(g_drv.MemExportToShareableHandle(&fd, c->mc_handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  *fd_out = fd;
  return D4PG_OK;
}
/* other ranks: import the object from the descriptor received from rank 0 (the descriptor is closed) */
extern "C" int32_t d4pg_comm_mc_import(d4pg_comm_t* c, int32_t fd) {
  D4PG_REQUIRE(c && fd >= 0 && load_drv(), D4PG_ENOTSUP, "d4pg_comm_mc_import: multicast API not available");
  int rc = mc_size_for(c, &c->mc_size);
  if (rc) return rc;
  DRV_OK(g_drv.MemImportFromShareableHandle(&c->mc_handle, reinterpret_cast<void*>(static_cast<uintptr_t>(fd)), CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
  c->mc_have_handle = true;
  close(fd);
  return D4PG_OK;
}
/* every rank, after it holds the handle: join the multicast team (all ranks must have joined before anyone binds) */
extern "C" int32_t d4pg_comm_mc_add_device(d4pg_comm_t* c) {
  D4PG_REQUIRE(c && c->mc_have_handle, D4PG_ESTATE, "d4pg_comm_mc_add_device: no multicast handle");
  CUdevice cd;
  DRV_OK(g_drv.DeviceGet(&cd, c->mc_dev));
  DRV_OK(g_drv.MulticastAddDevice(c->mc_handle, cd));
  return D4PG_OK;
}
/* every rank, after a barrier: allocate this rank's physical gradient buffer, bind it, map the unicast and multicast views */
extern "C" int32_t d4pg_comm_mc_bind(d4pg_comm_t* c) {
  D4PG_REQUIRE(c && c->mc_have_handle && c->peer_ready, D4PG_ESTATE, "d4pg_comm_mc_bind: handle / peer block missing");
  CUmemAllocationProp ap{};
  ap.type = CU_MEM_ALLOCATION_TYPE_PINNED; ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE; ap.location.id = c->mc_dev;
  ap.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  size_t gran = 0;
  DRV_OK(g_drv.MemGetAllocationGranularity(&gran, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
  D4PG_REQUIRE(c->mc_size % gran == 0 || gran % 4096 == 0, D4PG_ENOTSUP, "d4pg_comm_mc_bind: granularity mismatch");
  const size_t size = ((c->mc_size + gran - 1) / gran) * gran;
  DRV_OK(g_drv.MemCreate(&c->mc_mem, size, &ap, 0));
  DRV_OK(g_drv.MulticastBindMem(c->mc_handle, 0, c->mc_mem, 0, c->mc_size, 0));
  CUmemAccessDesc ad{};
  ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE; ad.location.id = c->mc_dev; ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  DRV_OK(g_drv.MemAddressReserve(&c->mc_uc, size, gran, 0, 0));
  DRV_OK(g_drv.MemMap(c->mc_uc, size, 0, c->mc_mem, 0));
  DRV_OK(g_drv.MemSetAccess(c->mc_uc, size, &ad, 1));
  DRV_OK(g_drv.MemAddressReserve(&c->mc_ptr, c->mc_size, gran, 0, 0));
  DRV_OK(g_drv.MemMap(c->mc_ptr, c->mc_size, 0, c->mc_handle, 0));
  DRV_OK(g_drv.MemSetAccess(c->mc_ptr, c->mc_size, &ad, 1));
  D4PG_CUDA_OK(cudaMemset(reinterpret_cast<void*>(c->mc_uc), 0, size));
  D4PG_CUDA_OK(cudaDeviceSynchronize());
  c->mc_ready = true;
  return D4PG_OK;
}
extern "C" int32_t d4pg_comm_mc_ready(const d4pg_comm_t* c) { return (c && c->mc_ready) ? 1 : 0; }
/* collective decision of the binding: stop using the multicast path (the buffers stay mapped until destroy) */
extern "C" int32_t d4pg_comm_mc_disable(d4pg_comm_t* c) { if (c) c->mc_ready = false; return D4PG_OK; }

// self-test of the in-switch reduction: out[i] = multimem.ld_reduce over all ranks of (rank r's unicast buffer)[i]
namespace d4pg {
__global__ void mc_selftest_kernel(const float* mc, float* out, int n4) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(reinterpret_cast<const float4*>(mc) + i) : "memory");
  reinterpret_cast<float4*>(out)[i] = v;
}
}  // namespace d4pg
/* fill this rank's unicast buffer from `src` (n floats, device), or reduce: out[0..n) = sum over ranks (after a barrier) */
extern "C" int32_t d4pg_comm_mc_selftest(d4pg_comm_t* c, const float* src, float* out, int64_t n, d4pg_stream_t stream) {
  D4PG_REQUIRE(c && c->mc_ready && n > 0 && n % 4 == 0 && size_t(n) * 4 <= c->mc_size, D4PG_EINVAL, "d4pg_comm_mc_selftest: bad arguments");
  cudaStream_t st = d4pg::as_stream(stream);
  if (src) D4PG_CUDA_OK(cudaMemcpyAsync(reinterpret_cast<void*>(c->mc_uc), src, size_t(n) * 4, cudaMemcpyDeviceToDevice, st));
  if (out) {
    d4pg::mc_selftest_kernel<<<unsigned((n / 4 + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float*>(c->mc_ptr), out, int(n / 4));
    D4PG_LAUNCH_OK();
  }
  return D4PG_OK;
}
