// Spatial self-attention on the Hopper tensor cores (wgmma; head dim 64, bf16 operands, fp32 softmax).
//
// One CTA = one (sample, head) x 128 queries; it streams 64-key K/V tiles:
//   warp 8      : TMA producer (Q once; K_j, V_j through a 3-stage mbarrier ring, 128B swizzle)
//   warps 0..7  : two consumer warpgroups, 64 query rows each:
//                   S_j = Q K_j^T   wgmma m64n64k16 x 4, A = Q and B = K_j K-major in shared memory -> registers
//                   online softmax on the register fragment (a row lives in the four lanes of a quad)
//                   O  += P_j V_j   wgmma m64n64k16 x 4, A = P straight from registers (the S fragment re-packed as
//                                   bf16), B = V_j MN-major in shared memory
// O and the running max / sum stay in registers for the whole key loop; when the row maximum grows, O and the sum are
// rescaled in place.  Shared memory ~65 KB, so several CTAs share an SM and one CTA's softmax overlaps another's MMAs.
//
// The same kernel serves self-attention (nq = nk = the item's tokens, one tensor map shape for Q, K and V) and
// cross-attention (nq queries of an item against its own nk keys, a separate K/V tensor map whose batch stride picks the
// item's key set).  Keys past nk arrive zero-filled from TMA and are masked to -inf in the tail tile.
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "host_util.cuh"
#include "v3d_b200.h"
#include "wgmma.cuh"

namespace v3d {

constexpr int AT_BM = 128;
constexpr int AT_BN = 64;
constexpr int AT_THREADS = 288;
constexpr int AT_KVSTAGES = 3;
constexpr int AT_QTILE = 128 * 128;                // bytes of a [128][64] bf16 tile (Q)
constexpr int AT_KTILE = 64 * 128;                 // bytes of a [64][64] bf16 tile (K, V)
constexpr int AT_OFF_Q = 0;
constexpr int AT_OFF_K = AT_OFF_Q + AT_QTILE;
constexpr int AT_OFF_V = AT_OFF_K + AT_KVSTAGES * AT_KTILE;
constexpr int AT_OFF_BAR = AT_OFF_V + AT_KVSTAGES * AT_KTILE;
constexpr int AT_SMEM = AT_OFF_BAR + 256 + 1024;   // + slack to align the base to 1024 B

// 2^x for a pair of fp32 values on the FMA pipe (no MUFU): round-to-nearest split x = n + f with the 1.5 * 2^23 magic
// add, degree-3 minimax polynomial for 2^f on [-0.5, 0.5] (max relative error 8.0e-5, a 25th of a bf16 half-ulp), then
// n is added into the exponent field (the integer sits in the low mantissa bits of the magic sum, so `bits << 23` is
// n << 23).  x is clamped to >= -126; x <= 0 here (scores minus the running row maximum).
__device__ __forceinline__ void exp2_poly2(float x0, float x1, float& p0, float& p1) {
  const uint64_t magic = pack2(12582912.0f, 12582912.0f);
  const uint64_t x2 = pack2(fmaxf(x0, -126.0f), fmaxf(x1, -126.0f));
  const uint64_t t2 = add2(x2, magic);
  const uint64_t f2 = add2(x2, fma2(t2, pack2(-1.0f, -1.0f), magic));  // x - (t - magic)
  uint64_t q2 = fma2(f2, pack2(0.05519810691475868f, 0.05519810691475868f),
                     pack2(0.24267712235450745f, 0.24267712235450745f));
  q2 = fma2(q2, f2, pack2(0.6932618021965027f, 0.6932618021965027f));
  q2 = fma2(q2, f2, pack2(0.9999227523803711f, 0.9999227523803711f));
  float q0, q1, t0, t1;
  unpack2(q2, q0, q1);
  unpack2(t2, t0, t1);
  p0 = __int_as_float(__float_as_int(q0) + (__float_as_int(t0) << 23));
  p1 = __int_as_float(__float_as_int(q1) + (__float_as_int(t1) << 23));
}

// POLY: how many of the 8 key chunks of a tile take their exp2 from exp2_poly2 instead of MUFU ex2.approx
// (0 = none, the default; 1 = every 4th chunk, 2 = every 2nd, 3 = three of four): moves part of the softmax's
// exponentials from the MUFU pipe to the FMA pipe.
template <int POLY>
__global__ void __launch_bounds__(AT_THREADS, 2)
attn_tc_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
               const __grid_constant__ CUtensorMap mapV, bf16* __restrict__ O, long long ldo, int nq, int nk,
               float scale_log2e) {
  extern __shared__ uint8_t at_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + AT_OFF_BAR);
  uint64_t* q_full = bars + 0;
  uint64_t* kv_full = bars + 1;    // [3]
  uint64_t* kv_empty = bars + 4;   // [3]  one arrival per consumer warpgroup

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AT_BM;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int nkv = (nk + AT_BN - 1) / AT_BN;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapQ);
    tma_prefetch_desc(&mapK);
    tma_prefetch_desc(&mapV);
    mbar_init(q_full, 1);
    for (int i = 0; i < AT_KVSTAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, AT_QTILE);
      tma_load_3d(smem + AT_OFF_Q, &mapQ, q_full, head * 64, q0, b);
      int st = 0;
      uint32_t ph = 0;
      for (int j = 0; j < nkv; ++j) {
        mbar_wait(&kv_empty[st], ph ^ 1u);
        mbar_arrive_expect_tx(&kv_full[st], 2 * AT_KTILE);
        tma_load_3d(smem + AT_OFF_K + st * AT_KTILE, &mapK, &kv_full[st], head * 64, j * AT_BN, b);
        tma_load_3d(smem + AT_OFF_V + st * AT_KTILE, &mapV, &kv_full[st], head * 64, j * AT_BN, b);
        if (++st == AT_KVSTAGES) {
          st = 0;
          ph ^= 1u;
        }
      }
    }
    return;
  }

  // ---- consumers.  Fragment of a 64 x 64 fp32 wgmma result: x[4 c + 2 h + e] = row 16 wi + lane / 4 + 8 h of the
  // warpgroup's 64, column 8 c + 2 (lane % 4) + e.
  const int cw = warp >> 2;
  const int wi = warp & 3;
  const int cq = (lane & 3) * 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const uint64_t dq = gmma_desc_k_sw128(smem_u32(smem + AT_OFF_Q + cw * 64 * 128));
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait(q_full, 0);

  auto key_tile = [&](int j, int st, auto tail_tag) {
    constexpr bool TAIL = decltype(tail_tag)::value;
    const int kbase = j * AT_BN;
    float s[32];
    const uint64_t dk = gmma_desc_k_sw128(smem_u32(smem + AT_OFF_K + st * AT_KTILE));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      Wgmma<64>::ss(s, dq + static_cast<uint64_t>(2 * k), dk + static_cast<uint64_t>(2 * k), k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    if (TAIL) {
#pragma unroll
      for (int c = 0; c < 8; ++c)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (kbase + 8 * c + cq + e >= nk) s[4 * c + e] = s[4 * c + 2 + e] = -INFINITY;
    }
    float msc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int c = 0; c < 8; ++c) mx = fmaxf(mx, fmaxf(s[4 * c + 2 * h], s[4 * c + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      // every key tile holds at least one key < nk, so mx is finite
      if (mx > m_run[h]) {
        const float fac = ex2_approx((m_run[h] - mx) * scale_log2e);  // 0 on the first tile
        m_run[h] = mx;
        l_run[h] *= fac;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          o[4 * c + 2 * h] *= fac;
          o[4 * c + 2 * h + 1] *= fac;
        }
      }
      msc[h] = m_run[h] * scale_log2e;
    }
    // P = exp2(s * scale - m * scale) as bf16 A fragments: k-chunk kk (keys 16 kk ..) = columns groups 2 kk, 2 kk + 1
    uint32_t pa[4][4];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float x0 = fmaf(s[4 * c + 2 * h], scale_log2e, -msc[h]);
        const float x1 = fmaf(s[4 * c + 2 * h + 1], scale_log2e, -msc[h]);
        float p0, p1;
        if (POLY != 0 && (POLY == 1 ? (c & 3) == 3 : (POLY == 2 ? (c & 1) == 1 : (c & 3) != 0))) {
          exp2_poly2(x0, x1, p0, p1);
          if (TAIL) {  // the polynomial clamps -inf to 2^-126
            if (kbase + 8 * c + cq >= nk) p0 = 0.f;
            if (kbase + 8 * c + cq + 1 >= nk) p1 = 0.f;
          }
        } else {
          p0 = ex2_approx(x0);
          p1 = ex2_approx(x1);
        }
        l_run[h] += p0 + p1;
        pa[c >> 1][(c & 1) * 2 + h] = pack_bf16x2(p0, p1);
      }
    }
    const uint32_t vbase = smem_u32(smem + AT_OFF_V + st * AT_KTILE);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      Wgmma<64>::rs(o, pa[kk], gmma_desc_mn_sw128(vbase + kk * 2048, AT_KTILE), 1u);
    wgmma_commit();
    wgmma_wait<0>();
  };

  int st = 0;
  uint32_t ph = 0;
  for (int j = 0; j < nkv; ++j) {
    mbar_wait(&kv_full[st], ph);
    if (j * AT_BN + AT_BN > nk) key_tile(j, st, std::true_type{});
    else key_tile(j, st, std::false_type{});
    if (wg_leader) mbar_arrive(&kv_empty[st]);
    if (++st == AT_KVSTAGES) {
      st = 0;
      ph ^= 1u;
    }
  }

  // ---- normalise and store
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const int row = q0 + cw * 64 + wi * 16 + (lane >> 2) + 8 * h;
    if (row < nq) {
      bf16* op = O + (static_cast<long long>(b) * nq + row) * ldo + head * 64 + cq;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        *reinterpret_cast<uint32_t*>(op + 8 * c) = pack_bf16x2(o[4 * c + 2 * h] * inv, o[4 * c + 2 * h + 1] * inv);
    }
  }
}

}  // namespace v3d

using namespace v3d;

extern "C" {

/* softmax(q k^T * scale) v per (sample, head), head dim 64, on wgmma tensor cores with TMA-staged operands.
 * q/k/v are column slices of one packed projection matrix (row stride ld_qkv elements), token rows sample-major.
 * Replaces F.scaled_dot_product_attention / xformers FMHA at sgm/modules/attention.py:337-341,432-444. */
int v3d_attention_spatial(const void* q, const void* k, const void* v, void* o, int64_t ld_qkv, int64_t ld_o,
                          int32_t nbatch, int32_t ntok, int32_t nheads, float scale, void* stream) {
  if (!q || !k || !v || !o || ld_qkv % 8 != 0 || ld_o % 8 != 0 || nbatch <= 0 || ntok <= 0 || nheads <= 0 ||
      nheads > 65535 || nbatch > 65535) {
    set_error("v3d_attention_spatial: bad args");
    return V3D_ERR_BAD_ARG;
  }
  CUtensorMap mq, mk, mv;
  const uint64_t dims[3] = {static_cast<uint64_t>(nheads) * 64, static_cast<uint64_t>(ntok),
                            static_cast<uint64_t>(nbatch)};
  const uint64_t str[2] = {static_cast<uint64_t>(ld_qkv) * 2, static_cast<uint64_t>(ld_qkv) * 2 * ntok};
  const uint32_t box_q[3] = {64, AT_BM, 1};
  const uint32_t box_kv[3] = {64, AT_BN, 1};
  int rc;
  if ((rc = make_tmap_bf16(&mq, q, 3, dims, str, box_q))) return rc;
  if ((rc = make_tmap_bf16(&mk, k, 3, dims, str, box_kv))) return rc;
  if ((rc = make_tmap_bf16(&mv, v, 3, dims, str, box_kv))) return rc;
  // V3D_ATTN_POLY = 1 | 2 | 3 (read once per process): opt-in FMA-pipe exp2 for 2 / 4 / 6 of a tile's 8 key chunks.
  // Default 0 = MUFU ex2 only.
  static int poly = -1;
  if (poly < 0) {
    const char* v = getenv("V3D_ATTN_POLY");
    poly = v ? atoi(v) : 0;
    if (poly < 0 || poly > 3) poly = 0;
  }
  using Kern = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, bf16*, long long, int, int, float);
  static const Kern kerns[4] = {attn_tc_kernel<0>, attn_tc_kernel<1>, attn_tc_kernel<2>, attn_tc_kernel<3>};
  static bool cfg[4] = {false, false, false, false};
  if (!cfg[poly]) {
    cudaError_t e = cudaFuncSetAttribute(kerns[poly], cudaFuncAttributeMaxDynamicSharedMemorySize, AT_SMEM);
    if (e != cudaSuccess) {
      set_error("attn_tc smem attr: %s", cudaGetErrorString(e));
      return V3D_ERR_CUDA;
    }
    cfg[poly] = true;
  }
  dim3 grid((ntok + AT_BM - 1) / AT_BM, nheads, nbatch);
  kerns[poly]<<<grid, AT_THREADS, AT_SMEM, static_cast<cudaStream_t>(stream)>>>(
      mq, mk, mv, static_cast<bf16*>(o), ld_o, ntok, ntok, scale * 1.44269504088896340736f);
  V3D_CHECK_LAUNCH("attn_tc_kernel");
  return V3D_OK;
}

/* softmax(q k^T * scale) v per (item, head), head dim 64, queries and keys from different matrices: item b's nq query
 * rows (b*nq + i, row stride ld_q) attend to its own nk key / value rows b*kv_bstride + j (row stride ld_kv; k and v
 * are column slices of one matrix), output rows b*nq + i (row stride ld_o).  kv_bstride >= nk; rows between key sets
 * are never read.  Replaces CrossAttention.forward over a context of nk tokens, sgm/modules/attention.py:286-349:
 * the spatial attn2 (each frame's own context, attention.py:571-572; kv_bstride = nk) and the temporal attn2 (the
 * context of frame 0 of each video, time_context = context[::T], sgm/modules/video_attention.py:244-253,131;
 * kv_bstride = T*nk read in place from the per-frame K/V rows). */
int v3d_attention_cross(const void* q, const void* k, const void* v, void* o, int64_t ld_q, int64_t ld_kv,
                        int64_t ld_o, int32_t nbatch, int32_t nq, int32_t nk, int64_t kv_bstride, int32_t nheads,
                        float scale, void* stream) {
  if (!q || !k || !v || !o || ld_q % 8 != 0 || ld_kv % 8 != 0 || ld_o % 8 != 0 || nbatch <= 0 || nq <= 0 || nk <= 0 ||
      kv_bstride < nk || nheads <= 0 || nheads > 65535 || nbatch > 65535 || ld_q < nheads * 64LL ||
      ld_kv < nheads * 64LL || ld_o < nheads * 64LL) {
    set_error("v3d_attention_cross: bad args");
    return V3D_ERR_BAD_ARG;
  }
  CUtensorMap mq, mk, mv;
  const uint64_t dq[3] = {static_cast<uint64_t>(nheads) * 64, static_cast<uint64_t>(nq), static_cast<uint64_t>(nbatch)};
  const uint64_t sq[2] = {static_cast<uint64_t>(ld_q) * 2, static_cast<uint64_t>(ld_q) * 2 * nq};
  const uint64_t dkv[3] = {static_cast<uint64_t>(nheads) * 64, static_cast<uint64_t>(nk),
                           static_cast<uint64_t>(nbatch)};
  const uint64_t skv[2] = {static_cast<uint64_t>(ld_kv) * 2, static_cast<uint64_t>(ld_kv) * 2 * kv_bstride};
  const uint32_t box_q[3] = {64, AT_BM, 1};
  const uint32_t box_kv[3] = {64, AT_BN, 1};
  int rc;
  if ((rc = make_tmap_bf16(&mq, q, 3, dq, sq, box_q))) return rc;
  if ((rc = make_tmap_bf16(&mk, k, 3, dkv, skv, box_kv))) return rc;
  if ((rc = make_tmap_bf16(&mv, v, 3, dkv, skv, box_kv))) return rc;
  static bool cfg = false;
  if (!cfg) {
    cudaError_t e = cudaFuncSetAttribute(attn_tc_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, AT_SMEM);
    if (e != cudaSuccess) {
      set_error("attn_tc smem attr: %s", cudaGetErrorString(e));
      return V3D_ERR_CUDA;
    }
    cfg = true;
  }
  dim3 grid((nq + AT_BM - 1) / AT_BM, nheads, nbatch);
  attn_tc_kernel<0><<<grid, AT_THREADS, AT_SMEM, static_cast<cudaStream_t>(stream)>>>(
      mq, mk, mv, static_cast<bf16*>(o), ld_o, nq, nk, scale * 1.44269504088896340736f);
  V3D_CHECK_LAUNCH("attn_tc_kernel");
  return V3D_OK;
}

}  // extern "C"
