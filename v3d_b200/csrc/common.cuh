// Shared device-side primitives for the sm_90a kernels: mbarrier, TMA, wgmma fences and descriptors.
// Everything here is inline PTX; there is no CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace v3d {

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------------------------------------
// error codes returned through the C ABI (0 == ok)
// ---------------------------------------------------------------------------------------------
enum {
  V3D_OK = 0,
  V3D_ERR_BAD_ARG = 1,
  V3D_ERR_CUDA = 2,
  V3D_ERR_NO_DRIVER = 3,
  V3D_ERR_UNSUPPORTED = 4,
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trap (-> cudaErrorLaunchFailure), never as a hang.
// The bound is counted in try_wait attempts (each attempt already blocks for a hardware-defined slice);
// %globaltimer is deliberately NOT read on this path: its read latency is microseconds and sat on every
// producer/consumer hand-off.
// try_wait with a suspend-time hint: the thread sleeps in hardware until the phase completes (or the hint expires)
// instead of re-polling shared memory, so waiting role warps leave the issue slots and the MIO queue to the warps
// that do the math.
__device__ __forceinline__ bool mbar_try_wait_suspend(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait_suspend(bar, parity)) {
    if (((++spins) & 0xffu) == 0 && clock64() - t0 > (1ll << 34)) __trap();  // ~8 s at 2 GHz
  }
}

// ---------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) loads, completing on an mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5}], [%2];" ::"r"(smem_u32(dst)),
      "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// TMA stores (shared -> global) tracked by per-thread bulk async-groups
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, uint32_t smem_addr, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(m),
               "r"(smem_addr), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t smem_addr, int c0, int c1, int c2,
                                             int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(m),
               "r"(smem_addr), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): ordering fences and shared-memory matrix descriptors
// ---------------------------------------------------------------------------------------------
// before the first wgmma that reads accumulator registers written by ordinary instructions
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed wgmma groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// move this warpgroup's register budget (producer warps give registers to the MMA warps)
template <int R>
__device__ __forceinline__ void regs_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void regs_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}

// Shared-memory matrix descriptor (sm_90) for a bf16 tile stored as dense 128-byte rows with the 128B TMA swizzle
// (8-row x 128 B atoms, 1024 B apart).
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout type (1 = SWIZZLE_128B)
// K-major operand (rows along M/N, 64 K elements per row): the stride offset steps over 8-row groups, the leading
// offset is unused.  One 16-element K step is +32 bytes inside the atom (+2 in the encoded address).
__device__ __forceinline__ uint64_t gmma_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3fffu);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// MN-major operand: rows of 64 contiguous MN elements (128 B, swizzled), one row per K index; 8-row K groups are
// 1024 B apart (stride byte offset); the leading offset separates 64-element MN groups (one group when MN = 64).
__device__ __forceinline__ uint64_t gmma_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3fffu);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3fffu) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// explicit shared-window accesses (keeps STS/LDS even when the pointer's address space is not inferable)
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}

// ---------------------------------------------------------------------------------------------
// small math helpers
// ---------------------------------------------------------------------------------------------
// two fp32 lanes carried in one 64-bit value; the arithmetic on a pair is two scalar fp32 instructions
__device__ __forceinline__ uint64_t pack2(float lo, float hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpack2(uint64_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  unpack2(c, c0, c1);
  return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ uint64_t add2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  return pack2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ uint64_t mul2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
// 16-byte read-only load that does not allocate in L1 (data consumed once)
__device__ __forceinline__ uint4 ldg_stream(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// SiLU = x * sigmoid(x), sigmoid(x) = 0.5 tanh(0.5 x) + 0.5: one MUFU op (tanh.approx, rel. error 2^-11,
// far below the bf16 resolution of every consumer) instead of ex2 + rcp.
__device__ __forceinline__ float silu_f(float x) {
  return x * fmaf(tanh_approx(0.5f * x), 0.5f, 0.5f);
}
__device__ __forceinline__ float gelu_erf_f(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
// erf-GELU as x * 0.5 (1 + tanh(x P(x^2))), P fitted (minimax over [-8, 8]) to the EXACT erf form:
// max |deviation from x * Phi(x)| = 2.5e-5 (the usual "tanh GELU" constants give 4.7e-4), plus tanh.approx's
// 2^-11 relative error.  8 FP32 ops + 1 MUFU per element instead of ~24 for a direct erf evaluation, which
// matters because the GEGLU GEMM epilogue is issue-bound at K = 320.
// P is only meaningful inside the fitted range (it turns negative beyond |x| ~ 11.1, which would flip the tanh): x^2 is
// clamped to 64 before the polynomial, so for |x| > 8 the argument is x * P(64) = 1.73 x, |.| > 13.8, tanh = +-1 and
// Phi is exactly 0 / 1 as in fp32 erf.
__device__ __forceinline__ float gelu_phi_fast(float x) {
  const float x2 = fminf(x * x, 64.0f);
  float p = fmaf(x2, -0.00035151753388801277f, 0.03700565095560008f);
  p = fmaf(x2, p, 0.7975078784258718f);
  return fmaf(tanh_approx(x * p), 0.5f, 0.5f);  // Phi(x)
}
__device__ __forceinline__ float gelu_erf_fast(float x) { return x * gelu_phi_fast(x); }
// the same function on a packed pair: 6 packed FP32 ops + 2 MUFU for two elements
__device__ __forceinline__ uint64_t gelu_erf_fast2(uint64_t x) {
  float xa, xb;
  unpack2(mul2(x, x), xa, xb);
  const uint64_t xx = pack2(fminf(xa, 64.0f), fminf(xb, 64.0f));  // range guard, see gelu_phi_fast
  uint64_t p = fma2(xx, pack2(-0.00035151753388801277f, -0.00035151753388801277f),
                    pack2(0.03700565095560008f, 0.03700565095560008f));
  p = fma2(xx, p, pack2(0.7975078784258718f, 0.7975078784258718f));
  float a, b;
  unpack2(mul2(x, p), a, b);
  const uint64_t phi = fma2(pack2(tanh_approx(a), tanh_approx(b)), pack2(0.5f, 0.5f), pack2(0.5f, 0.5f));
  return mul2(x, phi);
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
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

}  // namespace v3d
