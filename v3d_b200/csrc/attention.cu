// Attention kernels, head dim 64, bf16 in / fp32 softmax / bf16 out.
//   spatial : flash attention over N tokens per (sample, head); streaming K/V tiles through shared
//             memory with cp.async double buffering, online softmax in registers.
//             (mma.sync m16n8k16 bring-up kernel, exported as v3d_attention_spatial_mma for cross-checks;
//             the product kernel is the tcgen05 one in attention_tc.cu)
//   temporal: sequences of T <= 32 view-frames per (pixel, head); one warp per sequence, whole
//             problem on chip, no online softmax. Reads q/k/v with the frame stride directly from the
//             frame-major token matrix, so "(b t) s c -> (b s) t c" is never materialised.
//             32 < T <= 128: one CTA per sequence, warps split the query tiles (attn_temporal_long_kernel).
#include <cstring>

#include "common.cuh"
#include "host_util.cuh"
#include "v3d_b200.h"

namespace v3d {

constexpr int HD = 64;  // head dim
constexpr float kLog2e = 1.44269504088896340736f;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(sz)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2,
                                          uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// byte offset of 16B chunk `chunk` of row `row` in a [rows][64] bf16 tile with XOR swizzle
__device__ __forceinline__ uint32_t tile_off(int row, int chunk) {
  return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4));
}

constexpr int FA_BN = 64;

template <int BM>
__global__ void __launch_bounds__(BM * 2)
attn_spatial_kernel(const bf16* __restrict__ Q, const bf16* __restrict__ K, const bf16* __restrict__ V,
                    bf16* __restrict__ O, long long ld, long long ldo, int ntok, float scale_log2e) {
  constexpr int NT = BM * 2;  // threads: one warp per 16 query rows
  extern __shared__ __align__(128) uint8_t fa_smem[];
  uint8_t* sQ = fa_smem;                      // BM x 128 B
  uint8_t* sK = sQ + BM * 128;                // 2 x 64 x 128 B
  uint8_t* sV = sK + 2 * FA_BN * 128;         // 2 x 64 x 128 B

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int q0 = blockIdx.x * BM;
  const int head = blockIdx.y;
  const long long tok0 = static_cast<long long>(blockIdx.z) * ntok;
  const bf16* Qb = Q + tok0 * ld + head * HD;
  const bf16* Kb = K + tok0 * ld + head * HD;
  const bf16* Vb = V + tok0 * ld + head * HD;

  // ---- async loads: Q tile + first K/V tile
  for (int i = tid; i < BM * 8; i += NT) {
    const int r = i >> 3, c = i & 7;
    const bool ok = q0 + r < ntok;
    cp_async16(sQ + tile_off(r, c), Qb + static_cast<long long>(ok ? q0 + r : 0) * ld + c * 8, ok);
  }
  auto load_kv = [&](int tile, int buf) {
    const int k0 = tile * FA_BN;
    for (int i = tid; i < FA_BN * 8; i += NT) {
      const int r = i >> 3, c = i & 7;
      const bool ok = k0 + r < ntok;
      const long long off = static_cast<long long>(ok ? k0 + r : 0) * ld + c * 8;
      cp_async16(sK + buf * FA_BN * 128 + tile_off(r, c), Kb + off, ok);
      cp_async16(sV + buf * FA_BN * 128 + tile_off(r, c), Vb + off, ok);
    }
  };
  load_kv(0, 0);
  cp_async_commit();

  const int nkv = (ntok + FA_BN - 1) / FA_BN;
  uint32_t qf[4][4];
  float o_acc[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) o_acc[j][e] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};

  for (int it = 0; it < nkv; ++it) {
    const int buf = it & 1;
    if (it + 1 < nkv) {
      load_kv(it + 1, buf ^ 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (it == 0) {
      // Q fragments for this warp's 16 rows: 4 k-steps of 16 along d
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const int r = warp * 16 + (lane & 15);
        const int c = kk * 2 + (lane >> 4);
        ldsm_x4(smem_u32(sQ + tile_off(r, c)), qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3]);
      }
    }
    const uint8_t* kt = sK + buf * FA_BN * 128;
    const uint8_t* vt = sV + buf * FA_BN * 128;

    // ---- S = Q K^T  (16 x 64 per warp)
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[j][e] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {  // pairs of key n-tiles
        const int mi = lane >> 3;
        const int key = jp * 16 + (mi >> 1) * 8 + (lane & 7);
        const int c = kk * 2 + (mi & 1);
        uint32_t b0, b1, b2, b3;
        ldsm_x4(smem_u32(kt + tile_off(key, c)), b0, b1, b2, b3);
        mma_bf16_16816(s[2 * jp], qf[kk], b0, b1);
        mma_bf16_16816(s[2 * jp + 1], qf[kk], b2, b3);
      }
    }
    // ---- mask keys beyond ntok (only possible in the last tile)
    const int kbase = it * FA_BN;
    if (kbase + FA_BN > ntok) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int key = kbase + j * 8 + 2 * t;
        if (key >= ntok) { s[j][0] = -INFINITY; s[j][2] = -INFINITY; }
        if (key + 1 >= ntok) { s[j][1] = -INFINITY; s[j][3] = -INFINITY; }
      }
    }
    // ---- online softmax (rows g and g+8 of this warp's 16)
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mx[0] = fmaxf(mx[0], fmaxf(s[j][0], s[j][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[j][2], s[j][3]));
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    }
    float corr[2], msc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float mnew = fmaxf(m_run[h], mx[h]);
      corr[h] = exp2f((m_run[h] - mnew) * scale_log2e);  // exp2(-inf) = 0 on the first tile
      m_run[h] = mnew;
      msc[h] = mnew * scale_log2e;
      l_run[h] *= corr[h];
    }
    float rs[2] = {0.f, 0.f};
    uint32_t pf[4][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float p0 = exp2f(s[j][0] * scale_log2e - msc[0]);
      const float p1 = exp2f(s[j][1] * scale_log2e - msc[0]);
      const float p2 = exp2f(s[j][2] * scale_log2e - msc[1]);
      const float p3 = exp2f(s[j][3] * scale_log2e - msc[1]);
      rs[0] += p0 + p1;
      rs[1] += p2 + p3;
      const int kk = j >> 1;
      if ((j & 1) == 0) {
        pf[kk][0] = pack_bf16x2(p0, p1);
        pf[kk][1] = pack_bf16x2(p2, p3);
      } else {
        pf[kk][2] = pack_bf16x2(p0, p1);
        pf[kk][3] = pack_bf16x2(p2, p3);
      }
    }
    l_run[0] += rs[0];
    l_run[1] += rs[1];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o_acc[j][0] *= corr[0]; o_acc[j][1] *= corr[0];
      o_acc[j][2] *= corr[1]; o_acc[j][3] *= corr[1];
    }
    // ---- O += P V   (16 x 64 per warp; k = keys, n = d)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {  // pairs of d n-tiles
        const int mi = lane >> 3;
        const int key = kk * 16 + (mi & 1) * 8 + (lane & 7);
        const int c = jp * 2 + (mi >> 1);
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(smem_u32(vt + tile_off(key, c)), b0, b1, b2, b3);
        mma_bf16_16816(o_acc[2 * jp], pf[kk], b0, b1);
        mma_bf16_16816(o_acc[2 * jp + 1], pf[kk], b2, b3);
      }
    }
    __syncthreads();
  }

  // ---- finalize: quad-reduce row sums, normalise, store
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
  }
  const float inv0 = 1.f / l_run[0], inv1 = 1.f / l_run[1];
  const int r0 = q0 + warp * 16 + g;
  bf16* Ob = O + tok0 * ldo + head * HD;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = j * 8 + 2 * t;
    if (r0 < ntok)
      *reinterpret_cast<uint32_t*>(Ob + static_cast<long long>(r0) * ldo + col) =
          pack_bf16x2(o_acc[j][0] * inv0, o_acc[j][1] * inv0);
    if (r0 + 8 < ntok)
      *reinterpret_cast<uint32_t*>(Ob + static_cast<long long>(r0 + 8) * ldo + col) =
          pack_bf16x2(o_acc[j][2] * inv1, o_acc[j][3] * inv1);
  }
}

// ------------------------------------------------------------------------------------------------
// temporal attention: grid = (pixels, halves b); block = nheads warps. Row of token (b, t, s) is
// (b*T + t)*S + s. Lane t < T owns query frame t.
// ------------------------------------------------------------------------------------------------
constexpr int kMaxT = 32;
constexpr int kTaWarps = 4;
constexpr int kTaTile = 32 * 128;  // one [32 rows][64] bf16 tile, 128-byte rows, XOR-swizzled 16-byte chunks

// Temporal attention over T <= 32 frames: one warp per (pixel, head) sequence, whole problem on tensor cores:
//   S (32x32, keys >= T masked) = Q K^T   : 2 m-tiles x 4 n-tiles x 4 k-steps of mma.m16n8k16
//   O (32x64)                  = P V      : 2 m-tiles x 8 n-tiles x 2 k-steps
// Q/K/V rows are gathered with the frame stride S*ld straight from the frame-major token matrix (cp.async,
// 16-byte chunks), O is staged through the Q tile and written back as 16-byte chunks.
//
// SPLIT (frame-sharded views, SURVEY 8(e)): the T query frames are this rank's block of the video while keys and
// values come from all kv.tk frames of the K|V all-gather buffer, whose rows are rank-major: row of key frame f,
// CFG half b, pixel s is kv.row[f] + b * kv.bstride[f] + s (row stride ldkv).  Keys >= kv.tk are masked.  The dense
// form has kv.tk = T and leaves the table zero.  N = 32 here, 128 for attn_temporal_long_kernel.
template <int N>
struct KvRows {
  int tk;
  int row[N];
  int bstride[N];
};

template <bool SPLIT>
__global__ void __launch_bounds__(kTaWarps * 32)
attn_temporal_kernel(const bf16* __restrict__ Q, const bf16* __restrict__ K, const bf16* __restrict__ V,
                     bf16* __restrict__ O, long long ld, long long ldo, int T, int S, int nheads,
                     float scale_log2e, long long ldkv, const __grid_constant__ KvRows<kMaxT> kv) {
  extern __shared__ __align__(128) uint8_t ta_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int s = blockIdx.x, b = blockIdx.y;
  uint8_t* sq = ta_smem + warp * 3 * kTaTile;
  uint8_t* sk = sq + kTaTile;
  uint8_t* sv = sk + kTaTile;
  const long long row_base = (static_cast<long long>(b) * T) * S + s;
  const int TK = SPLIT ? kv.tk : T;  // key / value frames

  // rows >= T of K and V are never loaded: zero them once (P is 0 there, but 0 * garbage must stay 0)
  if (SPLIT) {
    for (int i = lane; i < (32 - TK) * 8; i += 32) {
      const int r = TK + (i >> 3), c = i & 7;
      *reinterpret_cast<uint4*>(sk + tile_off(r, c)) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(sv + tile_off(r, c)) = make_uint4(0, 0, 0, 0);
    }
    for (int i = lane; i < (32 - T) * 8; i += 32) {
      const int r = T + (i >> 3), c = i & 7;
      *reinterpret_cast<uint4*>(sq + tile_off(r, c)) = make_uint4(0, 0, 0, 0);
    }
  } else {
    for (int i = lane; i < (32 - T) * 8; i += 32) {
      const int r = T + (i >> 3), c = i & 7;
      *reinterpret_cast<uint4*>(sk + tile_off(r, c)) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(sv + tile_off(r, c)) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(sq + tile_off(r, c)) = make_uint4(0, 0, 0, 0);
    }
  }

  for (int head = warp; head < nheads; head += kTaWarps) {
    const long long col = static_cast<long long>(head) * HD;
    __syncwarp();
    if (SPLIT) {
      for (int i = lane; i < T * 8; i += 32) {
        const int r = i >> 3, c = i & 7;
        cp_async16(sq + tile_off(r, c), Q + (row_base + static_cast<long long>(r) * S) * ld + col + c * 8, true);
      }
      for (int i = lane; i < TK * 8; i += 32) {
        const int r = i >> 3, c = i & 7;
        const long long off =
            (static_cast<long long>(kv.row[r]) + static_cast<long long>(b) * kv.bstride[r] + s) * ldkv + col + c * 8;
        cp_async16(sk + tile_off(r, c), K + off, true);
        cp_async16(sv + tile_off(r, c), V + off, true);
      }
    } else {
      for (int i = lane; i < T * 8; i += 32) {
        const int r = i >> 3, c = i & 7;
        const long long off = (row_base + static_cast<long long>(r) * S) * ld + col + c * 8;
        cp_async16(sq + tile_off(r, c), Q + off, true);
        cp_async16(sk + tile_off(r, c), K + off, true);
        cp_async16(sv + tile_off(r, c), V + off, true);
      }
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncwarp();

    // ---- S = Q K^T
    float sc[2][4][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) sc[mt][j][e] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t qa[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
        ldsm_x4(smem_u32(sq + tile_off(mt * 16 + (lane & 15), kk * 2 + (lane >> 4))), qa[mt][0], qa[mt][1],
                qa[mt][2], qa[mt][3]);
#pragma unroll
      for (int jp = 0; jp < 2; ++jp) {  // pairs of key n-tiles
        const int mi = lane >> 3;
        const int key = jp * 16 + (mi >> 1) * 8 + (lane & 7);
        uint32_t b0, b1, b2, b3;
        ldsm_x4(smem_u32(sk + tile_off(key, kk * 2 + (mi & 1))), b0, b1, b2, b3);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma_bf16_16816(sc[mt][2 * jp], qa[mt], b0, b1);
          mma_bf16_16816(sc[mt][2 * jp + 1], qa[mt], b2, b3);
        }
      }
    }
    // ---- softmax over keys (columns), rows g / g+8 of each m-tile; P packed as A fragments
    uint32_t pf[2][2][4];
    float inv[2][2];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int key = j * 8 + 2 * t;
        if (key >= TK) { sc[mt][j][0] = -INFINITY; sc[mt][j][2] = -INFINITY; }
        if (key + 1 >= TK) { sc[mt][j][1] = -INFINITY; sc[mt][j][3] = -INFINITY; }
        mx0 = fmaxf(mx0, fmaxf(sc[mt][j][0], sc[mt][j][1]));
        mx1 = fmaxf(mx1, fmaxf(sc[mt][j][2], sc[mt][j][3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float m0 = mx0 * scale_log2e, m1 = mx1 * scale_log2e;
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float p0 = exp2f(fmaf(sc[mt][j][0], scale_log2e, -m0));
        const float p1 = exp2f(fmaf(sc[mt][j][1], scale_log2e, -m0));
        const float p2 = exp2f(fmaf(sc[mt][j][2], scale_log2e, -m1));
        const float p3 = exp2f(fmaf(sc[mt][j][3], scale_log2e, -m1));
        s0 += p0 + p1;
        s1 += p2 + p3;
        const int kk = j >> 1;
        if ((j & 1) == 0) {
          pf[mt][kk][0] = pack_bf16x2(p0, p1);
          pf[mt][kk][1] = pack_bf16x2(p2, p3);
        } else {
          pf[mt][kk][2] = pack_bf16x2(p0, p1);
          pf[mt][kk][3] = pack_bf16x2(p2, p3);
        }
      }
      s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
      s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
      inv[mt][0] = 1.f / s0;
      inv[mt][1] = 1.f / s1;
    }
    // ---- O = P V
    float oc[2][8][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) oc[mt][j][e] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {  // pairs of d n-tiles
        const int mi = lane >> 3;
        const int key = kk * 16 + (mi & 1) * 8 + (lane & 7);
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(smem_u32(sv + tile_off(key, jp * 2 + (mi >> 1))), b0, b1, b2, b3);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma_bf16_16816(oc[mt][2 * jp], pf[mt][kk], b0, b1);
          mma_bf16_16816(oc[mt][2 * jp + 1], pf[mt][kk], b2, b3);
        }
      }
    }
    // ---- stage O (normalised, bf16) through the Q tile, then 16-byte row-chunk stores
    __syncwarp();
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int r0 = mt * 16 + g;
        const int colb = (j * 8 + 2 * t) * 2;  // byte offset inside the 128-byte row
        *reinterpret_cast<uint32_t*>(sq + tile_off(r0, colb >> 4) + (colb & 15)) =
            pack_bf16x2(oc[mt][j][0] * inv[mt][0], oc[mt][j][1] * inv[mt][0]);
        *reinterpret_cast<uint32_t*>(sq + tile_off(r0 + 8, colb >> 4) + (colb & 15)) =
            pack_bf16x2(oc[mt][j][2] * inv[mt][1], oc[mt][j][3] * inv[mt][1]);
      }
    __syncwarp();
    for (int i = lane; i < T * 8; i += 32) {
      const int r = i >> 3, c = i & 7;
      *reinterpret_cast<uint4*>(O + (row_base + static_cast<long long>(r) * S) * ldo + col + c * 8) =
          *reinterpret_cast<const uint4*>(sq + tile_off(r, c));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// temporal attention over 32 < T <= 128 frames: grid = (pixels, heads, halves b), one (pixel, head) sequence per CTA.
//
// Why not the short kernel's "one warp owns a sequence": at T = 128 a sequence's Q, K and V tiles are 3 x 16 KB, so
// four warp-private sequences would take 192 KB and leave one CTA of 4 warps per SM, far too few loads in flight for
// a kernel that is bound by its HBM gathers.  Here the CTA's 4 warps share one K and one V tile and split the 16-query
// m-tiles between them (warp w takes m-tiles w, w + 4): 48 KB at T = 128, 18 KB at T = 48, all within the 48 KB that
// need no opt-in.  ptxas: 108 / 110 registers (KT = 8) and 82 / 78 (KT = 4), no spills, so 4 CTAs of 128 threads fit an SM by
// registers and by shared memory even at T = 128 (4 x 48 KB), each with its whole gather in flight before its first
// MMA; the launch bounds only keep the compiler from growing past 3 (KT = 8) / 4 (KT = 4) resident CTAs' worth.
//
// Per m-tile, a warp holds the complete score row block in registers (2 KT n-tiles x 4 fp32; Tk <= 128 so KT <= 8), so
// the softmax is single-pass: S = Q K^T on mma.m16n8k16, keys >= Tk set to -inf, row maximum and sum by quad shuffles,
// p = ex2(s * scale*log2e - max * scale*log2e), P packed to bf16 A fragments, O = P V, normalised in fp32.  KT is the
// capacity in 16-key tiles (4: Tk <= 64, 8: Tk <= 128); 16-key tiles at or beyond the padded key count are skipped.
// Rows are gathered with the frame stride by cp.async 16-byte chunks; rows of the last 16-row tile at or beyond T /
// Tk are zero-filled by cp.async itself (source size 0), so 0 x garbage cannot occur.  Each warp stages its m-tile of
// O through the Q rows it alone read and writes it back as 16-byte chunks.
//
// SPLIT: as in attn_temporal_kernel; the row table holds up to kMaxTLong key frames.
// ------------------------------------------------------------------------------------------------
constexpr int kMaxTLong = 128;
constexpr int kTlWarps = 4;

template <bool SPLIT, int KT>
__global__ void __launch_bounds__(kTlWarps * 32, KT == 4 ? 4 : 3)
attn_temporal_long_kernel(const bf16* __restrict__ Q, const bf16* __restrict__ K, const bf16* __restrict__ V,
                          bf16* __restrict__ O, long long ld, long long ldo, int T, int S, float scale_log2e,
                          long long ldkv, const __grid_constant__ KvRows<kMaxTLong> kv) {
  extern __shared__ __align__(128) uint8_t tl_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int s = blockIdx.x, b = blockIdx.z;
  const long long col = static_cast<long long>(blockIdx.y) * HD;
  const int TK = SPLIT ? kv.tk : T;                        // key / value frames
  const int Tp = (T + 15) & ~15, TKp = (TK + 15) & ~15;    // rows of the Q tile / of the K and V tiles
  uint8_t* sq = tl_smem;
  uint8_t* sk = sq + Tp * 128;
  uint8_t* sv = sk + TKp * 128;
  const long long row_base = (static_cast<long long>(b) * T) * S + s;

  for (int i = threadIdx.x; i < Tp * 8; i += kTlWarps * 32) {
    const int r = i >> 3, c = i & 7;
    const bool ok = r < T;
    cp_async16(sq + tile_off(r, c), Q + (row_base + static_cast<long long>(ok ? r : 0) * S) * ld + col + c * 8, ok);
  }
  for (int i = threadIdx.x; i < TKp * 8; i += kTlWarps * 32) {
    const int r = i >> 3, c = i & 7;
    const bool ok = r < TK;
    const int f = ok ? r : 0;
    const long long row = SPLIT ? static_cast<long long>(kv.row[f]) + static_cast<long long>(b) * kv.bstride[f] + s
                                : row_base + static_cast<long long>(f) * S;
    const long long off = row * ldkv + col + c * 8;
    cp_async16(sk + tile_off(r, c), K + off, ok);
    cp_async16(sv + tile_off(r, c), V + off, ok);
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();

  const int mi = lane >> 3;
  for (int m0 = warp * 16; m0 < Tp; m0 += kTlWarps * 16) {
    // ---- S = Q K^T for this warp's 16 queries
    uint32_t qa[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      ldsm_x4(smem_u32(sq + tile_off(m0 + (lane & 15), kk * 2 + (lane >> 4))), qa[kk][0], qa[kk][1], qa[kk][2],
              qa[kk][3]);
    float sc[2 * KT][4];
#pragma unroll
    for (int j = 0; j < 2 * KT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) sc[j][e] = 0.f;
#pragma unroll
    for (int jp = 0; jp < KT; ++jp) {  // pairs of key n-tiles
      if (jp * 16 < TKp) {
        const int key = jp * 16 + (mi >> 1) * 8 + (lane & 7);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          uint32_t b0, b1, b2, b3;
          ldsm_x4(smem_u32(sk + tile_off(key, kk * 2 + (mi & 1))), b0, b1, b2, b3);
          mma_bf16_16816(sc[2 * jp], qa[kk], b0, b1);
          mma_bf16_16816(sc[2 * jp + 1], qa[kk], b2, b3);
        }
      }
    }
    // ---- softmax over keys, rows g / g+8; P packed as A fragments
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 2 * KT; ++j) {
      const int key = j * 8 + 2 * t;
      if (key >= TK) { sc[j][0] = -INFINITY; sc[j][2] = -INFINITY; }
      if (key + 1 >= TK) { sc[j][1] = -INFINITY; sc[j][3] = -INFINITY; }
      mx0 = fmaxf(mx0, fmaxf(sc[j][0], sc[j][1]));
      mx1 = fmaxf(mx1, fmaxf(sc[j][2], sc[j][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float m0s = mx0 * scale_log2e, m1s = mx1 * scale_log2e;
    float s0 = 0.f, s1 = 0.f;
    uint32_t pf[KT][4];
#pragma unroll
    for (int j = 0; j < 2 * KT; ++j) {
      const float p0 = ex2_approx(fmaf(sc[j][0], scale_log2e, -m0s));
      const float p1 = ex2_approx(fmaf(sc[j][1], scale_log2e, -m0s));
      const float p2 = ex2_approx(fmaf(sc[j][2], scale_log2e, -m1s));
      const float p3 = ex2_approx(fmaf(sc[j][3], scale_log2e, -m1s));
      s0 += p0 + p1;
      s1 += p2 + p3;
      pf[j >> 1][(j & 1) * 2] = pack_bf16x2(p0, p1);
      pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
    s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
    s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
    const float inv0 = 1.f / s0, inv1 = 1.f / s1;
    // ---- O = P V
    float oc[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) oc[j][e] = 0.f;
#pragma unroll
    for (int kk = 0; kk < KT; ++kk) {
      if (kk * 16 < TKp) {
        const int key = kk * 16 + (mi & 1) * 8 + (lane & 7);
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {  // pairs of d n-tiles
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(smem_u32(sv + tile_off(key, jp * 2 + (mi >> 1))), b0, b1, b2, b3);
          mma_bf16_16816(oc[2 * jp], pf[kk], b0, b1);
          mma_bf16_16816(oc[2 * jp + 1], pf[kk], b2, b3);
        }
      }
    }
    // ---- stage O (normalised, bf16) through this warp's Q rows, then 16-byte row-chunk stores of the rows < T
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int colb = (j * 8 + 2 * t) * 2;  // byte offset inside the 128-byte row
      *reinterpret_cast<uint32_t*>(sq + tile_off(m0 + g, colb >> 4) + (colb & 15)) =
          pack_bf16x2(oc[j][0] * inv0, oc[j][1] * inv0);
      *reinterpret_cast<uint32_t*>(sq + tile_off(m0 + g + 8, colb >> 4) + (colb & 15)) =
          pack_bf16x2(oc[j][2] * inv1, oc[j][3] * inv1);
    }
    __syncwarp();
    for (int i = lane; i < 16 * 8; i += 32) {
      const int r = m0 + (i >> 3), c = i & 7;
      if (r < T)
        *reinterpret_cast<uint4*>(O + (row_base + static_cast<long long>(r) * S) * ldo + col + c * 8) =
            *reinterpret_cast<const uint4*>(sq + tile_off(r, c));
    }
  }
}

// Row table of the frame-sharded form from the host arrays kv_row / kv_bstride.  The dense form passes null and gets a
// zero table, so a negative offset (the error names the _kv entry point) can only come from v3d_attention_temporal_kv.
template <int N>
static bool fill_kv_rows(KvRows<N>& kv, int Tk, const int32_t* kv_row, const int32_t* kv_bstride) {
  memset(&kv, 0, sizeof(kv));
  kv.tk = Tk;
  for (int f = 0; kv_row && f < Tk; ++f) {
    if (kv_row[f] < 0 || kv_bstride[f] < 0) {
      set_error("v3d_attention_temporal_kv: negative row offset for key frame %d", f);
      return false;
    }
    kv.row[f] = kv_row[f];
    kv.bstride[f] = kv_bstride[f];
  }
  return true;
}

// Host side of both temporal entry points: attn_temporal_kernel for Tk <= 32 key frames, attn_temporal_long_kernel
// (KT = 4 up to 64 key frames, 8 above) for 32 < Tk <= 128.
template <bool SPLIT>
static int launch_temporal(const void* q, const void* k, const void* v, void* o, int64_t ld_q, int64_t ld_kv,
                           int64_t ld_o, int nb, int Tq, int Tk, int S, int nheads, float scale,
                           const int32_t* kv_row, const int32_t* kv_bstride, cudaStream_t st) {
  const bf16 *Q = static_cast<const bf16*>(q), *K = static_cast<const bf16*>(k), *V = static_cast<const bf16*>(v);
  bf16* O = static_cast<bf16*>(o);
  const float sl2 = scale * kLog2e;
  if (Tk <= kMaxT) {
    KvRows<kMaxT> kv;
    if (!fill_kv_rows(kv, Tk, kv_row, kv_bstride)) return V3D_ERR_BAD_ARG;
    attn_temporal_kernel<SPLIT><<<dim3(S, nb), kTaWarps * 32, kTaWarps * 3 * kTaTile, st>>>(
        Q, K, V, O, ld_q, ld_o, Tq, S, nheads, sl2, ld_kv, kv);
    V3D_CHECK_LAUNCH(SPLIT ? "attn_temporal_kernel<split>" : "attn_temporal_kernel");
    return V3D_OK;
  }
  KvRows<kMaxTLong> kv;
  if (!fill_kv_rows(kv, Tk, kv_row, kv_bstride)) return V3D_ERR_BAD_ARG;
  const int smem = (((Tq + 15) & ~15) + 2 * ((Tk + 15) & ~15)) * 128;  // <= 48 KB: no opt-in needed
  const dim3 grid(S, nheads, nb);
  if (Tk <= 64)
    attn_temporal_long_kernel<SPLIT, 4><<<grid, kTlWarps * 32, smem, st>>>(Q, K, V, O, ld_q, ld_o, Tq, S, sl2, ld_kv,
                                                                           kv);
  else
    attn_temporal_long_kernel<SPLIT, 8><<<grid, kTlWarps * 32, smem, st>>>(Q, K, V, O, ld_q, ld_o, Tq, S, sl2, ld_kv,
                                                                           kv);
  V3D_CHECK_LAUNCH(SPLIT ? "attn_temporal_long_kernel<split>" : "attn_temporal_long_kernel");
  return V3D_OK;
}

// Host side of the spatial twin: 128-query CTAs (48 KB of shared memory, opted in) from 512 tokens up, 64 below.
template <int BM>
static void launch_spatial(const void* q, const void* k, const void* v, void* o, int64_t ld_qkv, int64_t ld_o,
                           int nbatch, int ntok, int nheads, float scale, cudaStream_t st) {
  const int smem = BM * 128 + 4 * FA_BN * 128;
  if constexpr (BM == 128) {
    static bool cfg = false;
    if (!cfg) {
      cudaFuncSetAttribute(attn_spatial_kernel<BM>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      cfg = true;
    }
  }
  attn_spatial_kernel<BM><<<dim3((ntok + BM - 1) / BM, nheads, nbatch), BM * 2, smem, st>>>(
      static_cast<const bf16*>(q), static_cast<const bf16*>(k), static_cast<const bf16*>(v), static_cast<bf16*>(o),
      ld_qkv, ld_o, ntok, scale * kLog2e);
}

}  // namespace v3d

using namespace v3d;

extern "C" {

/* Bring-up / cross-check implementation of v3d_attention_spatial on mma.sync (kept for validation of the
 * tcgen05 kernel in tests; the product path calls v3d_attention_spatial).
 * softmax(q k^T * scale) v per (sample, head), head dim 64; q/k/v are column slices of one packed
 * projection matrix (row stride ld_qkv), token rows sample-major. Replaces
 * F.scaled_dot_product_attention / xformers FMHA at sgm/modules/attention.py:337-341,432-444. */
int v3d_attention_spatial_mma(const void* q, const void* k, const void* v, void* o, int64_t ld_qkv, int64_t ld_o,
                          int32_t nbatch, int32_t ntok, int32_t nheads, float scale, void* stream) {
  if (!q || !k || !v || !o || ld_qkv % 8 != 0 || ld_o % 8 != 0 || nbatch <= 0 || ntok <= 0 || nheads <= 0 ||
      nheads > 65535 || nbatch > 65535) {
    set_error("v3d_attention_spatial_mma: bad args");
    return V3D_ERR_BAD_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (ntok >= 512)
    launch_spatial<128>(q, k, v, o, ld_qkv, ld_o, nbatch, ntok, nheads, scale, st);
  else
    launch_spatial<64>(q, k, v, o, ld_qkv, ld_o, nbatch, ntok, nheads, scale, st);
  V3D_CHECK_LAUNCH("attn_spatial_kernel");
  return V3D_OK;
}

/* Temporal self-attention across the T view-frames of each pixel (video_attention.py:114,125 around
 * attention.py:337-341), on the frame-major token matrix: row(b,t,s) = (b*T + t)*S + s. */
int v3d_attention_temporal(const void* q, const void* k, const void* v, void* o, int64_t ld_qkv, int64_t ld_o,
                           int32_t nb, int32_t T, int32_t S, int32_t nheads, float scale, void* stream) {
  if (!q || !k || !v || !o || ld_qkv % 8 != 0 || ld_o % 8 != 0 || T <= 0 || T > kMaxTLong || nheads <= 0 ||
      nheads > 65535 || nb <= 0 || nb > 65535 || S <= 0) {
    set_error("v3d_attention_temporal: bad args (T=%d must be 1..%d: a longer sequence needs an online softmax over "
              "key tiles, which this kernel family does not have)", T, kMaxTLong);
    return V3D_ERR_BAD_ARG;
  }
  return launch_temporal<false>(q, k, v, o, ld_qkv, ld_qkv, ld_o, nb, T, T, S, nheads, scale, nullptr, nullptr,
                                static_cast<cudaStream_t>(stream));
}

/* Frame-sharded temporal self-attention (SURVEY.md 8(e); BASELINE.json "temporal-attention KV all-gather"): this
 * rank holds Tq of the video's Tk view-frames.  q / o are the local frame-major token matrices (row(b,t,s) =
 * (b*Tq + t)*S + s); k / v point into the all-gathered K|V buffer (row stride ld_kv) whose rows are rank-major, so
 * key frame f of CFG half b, pixel s sits at row kv_row[f] + b * kv_bstride[f] + s (host int32 arrays of Tk entries).
 * Same arithmetic as v3d_attention_temporal: softmax(q k^T scale) v over the Tk keys (attention.py:337-341 inside
 * video_attention.py:114-125). */
int v3d_attention_temporal_kv(const void* q, const void* k, const void* v, void* o, int64_t ld_q, int64_t ld_kv,
                              int64_t ld_o, int32_t nb, int32_t Tq, int32_t Tk, int32_t S, int32_t nheads,
                              const int32_t* kv_row, const int32_t* kv_bstride, float scale, void* stream) {
  if (!q || !k || !v || !o || !kv_row || !kv_bstride || ld_q % 8 != 0 || ld_kv % 8 != 0 || ld_o % 8 != 0 ||
      Tq <= 0 || Tq > Tk || Tk > kMaxTLong || nheads <= 0 || nheads > 65535 || nb <= 0 || nb > 65535 || S <= 0) {
    set_error("v3d_attention_temporal_kv: bad args (Tq=%d Tk=%d, need 0 < Tq <= Tk <= %d: more key frames need an "
              "online softmax over key tiles, which this kernel family does not have)", Tq, Tk, kMaxTLong);
    return V3D_ERR_BAD_ARG;
  }
  return launch_temporal<true>(q, k, v, o, ld_q, ld_kv, ld_o, nb, Tq, Tk, S, nheads, scale, kv_row, kv_bstride,
                               static_cast<cudaStream_t>(stream));
}

}  // extern "C"
