// One-sided exchanges over NVLink peer memory for the frame-sharded path (ONE image over several GPUs of a box).
//
// Every rank owns an ARENA (plain cudaMalloc memory, exported with cudaIpcGetMemHandle and mapped by the other ranks of
// the box with cudaIpcOpenMemHandle: the mapped pointers are ordinary global addresses whose loads / stores travel over
// NVLink / NVSwitch).  All arenas have the same layout, so "offset X in rank r's arena" is the whole addressing scheme.
// Three kernels move the data, each ONE launch per exchange and all of them capturable in a CUDA graph (no host
// synchronisation, no NCCL call, no tag matching):
//
//   peer_put_kernel      copies up to 16 contiguous segments into peer (or local) memory with 16-byte stores, then -
//                        after every CTA's stores are fenced system-wide - writes the current EPOCH into flag words
//                        that live in the receivers' arenas (release, system scope);
//   peer_wait_kernel     one thread per flag spins (acquire, system scope) until flag >= epoch;
//   peer_allreduce_f64   GroupNorm statistics: writes the local vector into slot[rank] of every arena, raises
//                        flag[rank] there, waits for all world flags of its own arena and adds the slots in RANK ORDER
//                        (every rank gets bit-identical sums), times `scale`.
//
// The epoch is a device word that a one-thread kernel increments at the start of every sharded forward pass, so a
// captured graph replays with fresh flag values.  Waits are bounded (30 s - ranks can be seconds apart at their first exchange - and only the first wait of a failed transport pays it): a rank that never gets its signal
// records the site in a status word and carries on instead of hanging the device; the host checks the status word.
#include <cstring>

#include "common.cuh"
#include "host_util.cuh"
#include "v3d_b200.h"

namespace v3d {

struct PeerPutArgs {
  const void* src[V3D_PEER_MAX_SEG];
  void* dst[V3D_PEER_MAX_SEG];
  long long bytes[V3D_PEER_MAX_SEG];  // multiples of 16
  unsigned int* flag[V3D_PEER_MAX_FLAG];
  int nseg;
  int nflag;
};

__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
constexpr unsigned long long kWaitLimitNs = 30ull * 1000ull * 1000ull * 1000ull;
// once one wait of a transport has timed out, every later wait falls through at once (the image is invalid anyway):
// a broken exchange costs one time limit, not one per site
__device__ __forceinline__ bool peer_failed(const unsigned int* status) {
  return (*reinterpret_cast<const volatile unsigned int*>(status) & 0x80000000u) != 0u;
}

__global__ void peer_epoch_kernel(unsigned int* epoch) { *epoch += 1u; }

__global__ void __launch_bounds__(512)
peer_put_kernel(const __grid_constant__ PeerPutArgs a, const unsigned int* __restrict__ epoch,
                unsigned int* __restrict__ done_counter) {
  const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long nthr = static_cast<long long>(gridDim.x) * blockDim.x;
  for (int s = 0; s < a.nseg; ++s) {
    const uint4* src = static_cast<const uint4*>(a.src[s]);
    uint4* dst = static_cast<uint4*>(a.dst[s]);
    const long long n = a.bytes[s] >> 4;
    long long i = tid;
    // four independent 16-byte loads in flight per thread
    for (; i + 3 * nthr < n; i += 4 * nthr) {
      const uint4 v0 = ldg_stream(src + i), v1 = ldg_stream(src + i + nthr), v2 = ldg_stream(src + i + 2 * nthr),
                  v3 = ldg_stream(src + i + 3 * nthr);
      dst[i] = v0;
      dst[i + nthr] = v1;
      dst[i + 2 * nthr] = v2;
      dst[i + 3 * nthr] = v3;
    }
    for (; i < n; i += nthr) dst[i] = ldg_stream(src + i);
  }
  if (a.nflag == 0) return;
  // every CTA: stores fenced system-wide, then one arrival; the last CTA raises the flags
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(done_counter, 1u);
    if (prev == gridDim.x - 1) {
      *done_counter = 0u;
      __threadfence_system();
      const unsigned int e = *epoch;
      for (int f = 0; f < a.nflag; ++f) st_release_sys(a.flag[f], e);
    }
  }
}

struct PeerWaitArgs {
  const unsigned int* flag[V3D_PEER_MAX_FLAG];
  int nflag;
  int site;
};

__global__ void peer_wait_kernel(const __grid_constant__ PeerWaitArgs a, const unsigned int* __restrict__ epoch,
                                 unsigned int* __restrict__ status) {
  if (static_cast<int>(threadIdx.x) >= a.nflag) return;
  const unsigned int e = *epoch;
  const unsigned int* f = a.flag[threadIdx.x];
  const unsigned long long t0 = global_ns();
  // signed distance: robust against the 32-bit epoch wrapping
  while (static_cast<int>(ld_acquire_sys(f) - e) < 0) {
    __nanosleep(100);
    if (peer_failed(status)) return;
    if (global_ns() - t0 > kWaitLimitNs) {
      atomicExch(status, 0x80000000u | static_cast<unsigned int>(a.site));
      return;
    }
  }
}

struct PeerReduceArgs {
  double* slot_base[V3D_PEER_MAX_RANKS];         // slot area of every rank's arena: [world][n] doubles
  unsigned int* flag_base[V3D_PEER_MAX_RANKS];   // flag area of every rank's arena: [world] words
  int world;
  int rank;
  int n;
  int site;
};

__global__ void __launch_bounds__(256)
peer_allreduce_f64_kernel(const __grid_constant__ PeerReduceArgs a, double* __restrict__ stats, double scale,
                          const unsigned int* __restrict__ epoch, unsigned int* __restrict__ status) {
  const unsigned int e = *epoch;
  const int t = threadIdx.x;
  // 1) my vector into slot[rank] of every arena (my own included)
  for (int r = 0; r < a.world; ++r)
    for (int i = t; i < a.n; i += blockDim.x) a.slot_base[r][static_cast<size_t>(a.rank) * a.n + i] = stats[i];
  __threadfence_system();
  __syncthreads();
  if (t < a.world) st_release_sys(a.flag_base[t] + a.rank, e);
  // 2) all world contributions have landed here
  if (t < a.world) {
    const unsigned int* f = a.flag_base[a.rank] + t;
    const unsigned long long t0 = global_ns();
    while (static_cast<int>(ld_acquire_sys(f) - e) < 0) {
      __nanosleep(100);
      if (peer_failed(status)) break;
      if (global_ns() - t0 > kWaitLimitNs) {
        atomicExch(status, 0x80000000u | static_cast<unsigned int>(a.site));
        break;
      }
    }
  }
  __syncthreads();
  // 3) rank-ordered sum: the same bits on every rank
  const double* mine = a.slot_base[a.rank];
  for (int i = t; i < a.n; i += blockDim.x) {
    double acc = 0.0;
    for (int r = 0; r < a.world; ++r) {
      double v;
      asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(mine + static_cast<size_t>(r) * a.n + i));
      acc += v;
    }
    stats[i] = acc * scale;
  }
}

}  // namespace v3d

using namespace v3d;

extern "C" {

int v3d_peer_alloc(int64_t bytes, void** out) {
  if (bytes <= 0 || out == nullptr) {
    set_error("v3d_peer_alloc: bad args");
    return V3D_ERR_BAD_ARG;
  }
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, static_cast<size_t>(bytes));
  if (e == cudaSuccess) e = cudaMemset(p, 0, static_cast<size_t>(bytes));
  // the zeroing must have landed before the handle can be exported: cudaMemset only enqueues it behind this process's
  // pending work, and a peer that already holds the handle may write data and epoch flags into the arena at once; a
  // memset that runs after those writes would erase them and leave the owner waiting for a signal that never comes
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    set_error("v3d_peer_alloc(%lld): %s", static_cast<long long>(bytes), cudaGetErrorString(e));
    if (p) cudaFree(p);
    return V3D_ERR_CUDA;
  }
  *out = p;
  return V3D_OK;
}

int v3d_peer_free(void* p) {
  if (p && cudaFree(p) != cudaSuccess) {
    set_error("v3d_peer_free failed");
    return V3D_ERR_CUDA;
  }
  return V3D_OK;
}

int v3d_peer_export(const void* p, void* handle64) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  if (!p || !handle64) {
    set_error("v3d_peer_export: null");
    return V3D_ERR_BAD_ARG;
  }
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, const_cast<void*>(p));
  if (e != cudaSuccess) {
    set_error("cudaIpcGetMemHandle: %s", cudaGetErrorString(e));
    return V3D_ERR_CUDA;
  }
  memcpy(handle64, &h, 64);
  return V3D_OK;
}

int v3d_peer_import(const void* handle64, void** out) {
  if (!handle64 || !out) {
    set_error("v3d_peer_import: null");
    return V3D_ERR_BAD_ARG;
  }
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    set_error("cudaIpcOpenMemHandle: %s", cudaGetErrorString(e));
    return V3D_ERR_CUDA;
  }
  *out = p;
  return V3D_OK;
}

int v3d_peer_close(void* p) {
  if (p && cudaIpcCloseMemHandle(p) != cudaSuccess) {
    set_error("cudaIpcCloseMemHandle failed");
    return V3D_ERR_CUDA;
  }
  return V3D_OK;
}

int v3d_peer_epoch_bump(void* epoch, void* stream) {
  if (!epoch) {
    set_error("v3d_peer_epoch_bump: null");
    return V3D_ERR_BAD_ARG;
  }
  peer_epoch_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<unsigned int*>(epoch));
  V3D_CHECK_LAUNCH("peer_epoch_kernel");
  return V3D_OK;
}

int v3d_peer_put(int32_t nseg, const void* const* src, void* const* dst, const int64_t* bytes, int32_t nflag,
                 void* const* flags, const void* epoch, void* done_counter, void* stream) {
  if (nseg < 0 || nseg > V3D_PEER_MAX_SEG || nflag < 0 || nflag > V3D_PEER_MAX_FLAG || !epoch || !done_counter ||
      (nseg > 0 && (!src || !dst || !bytes)) || (nflag > 0 && !flags)) {
    set_error("v3d_peer_put: bad args nseg=%d nflag=%d", nseg, nflag);
    return V3D_ERR_BAD_ARG;
  }
  PeerPutArgs a;
  memset(&a, 0, sizeof(a));
  a.nseg = nseg;
  a.nflag = nflag;
  long long total = 0;
  for (int i = 0; i < nseg; ++i) {
    if ((bytes[i] & 15) || (reinterpret_cast<uintptr_t>(src[i]) & 15) || (reinterpret_cast<uintptr_t>(dst[i]) & 15)) {
      set_error("v3d_peer_put: segment %d is not 16-byte aligned", i);
      return V3D_ERR_BAD_ARG;
    }
    a.src[i] = src[i];
    a.dst[i] = dst[i];
    a.bytes[i] = bytes[i];
    total += bytes[i];
  }
  for (int i = 0; i < nflag; ++i) a.flag[i] = static_cast<unsigned int*>(flags[i]);
  // enough CTAs to keep NVLink busy without taking the whole GPU: 64 KB per CTA, at most one CTA per SM
  long long ctas = (total + 65535) / 65536;
  if (ctas < 1) ctas = 1;
  if (ctas > num_sms()) ctas = num_sms();
  peer_put_kernel<<<static_cast<unsigned>(ctas), 512, 0, static_cast<cudaStream_t>(stream)>>>(
      a, static_cast<const unsigned int*>(epoch), static_cast<unsigned int*>(done_counter));
  V3D_CHECK_LAUNCH("peer_put_kernel");
  return V3D_OK;
}

int v3d_peer_wait(int32_t nflag, const void* const* flags, const void* epoch, void* status, int32_t site,
                  void* stream) {
  if (nflag <= 0 || nflag > V3D_PEER_MAX_FLAG || !flags || !epoch || !status) {
    set_error("v3d_peer_wait: bad args nflag=%d", nflag);
    return V3D_ERR_BAD_ARG;
  }
  PeerWaitArgs a;
  memset(&a, 0, sizeof(a));
  a.nflag = nflag;
  a.site = site;
  for (int i = 0; i < nflag; ++i) a.flag[i] = static_cast<const unsigned int*>(flags[i]);
  peer_wait_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(a, static_cast<const unsigned int*>(epoch),
                                                                  static_cast<unsigned int*>(status));
  V3D_CHECK_LAUNCH("peer_wait_kernel");
  return V3D_OK;
}

int v3d_peer_allreduce_f64(void* stats, int32_t n, double scale, int32_t world, int32_t rank,
                           void* const* slot_base, void* const* flag_base, const void* epoch, void* status,
                           int32_t site, void* stream) {
  if (!stats || n <= 0 || world <= 0 || world > V3D_PEER_MAX_RANKS || rank < 0 || rank >= world || !slot_base ||
      !flag_base || !epoch || !status) {
    set_error("v3d_peer_allreduce_f64: bad args n=%d world=%d rank=%d", n, world, rank);
    return V3D_ERR_BAD_ARG;
  }
  PeerReduceArgs a;
  memset(&a, 0, sizeof(a));
  a.world = world;
  a.rank = rank;
  a.n = n;
  a.site = site;
  for (int r = 0; r < world; ++r) {
    a.slot_base[r] = static_cast<double*>(slot_base[r]);
    a.flag_base[r] = static_cast<unsigned int*>(flag_base[r]);
  }
  peer_allreduce_f64_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      a, static_cast<double*>(stats), scale, static_cast<const unsigned int*>(epoch),
      static_cast<unsigned int*>(status));
  V3D_CHECK_LAUNCH("peer_allreduce_f64_kernel");
  return V3D_OK;
}

}  // extern "C"
