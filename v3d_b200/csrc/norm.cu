// Memory-bound normalisation kernels on NHWC / token-major bf16 activations (fp32 statistics):
// GroupNorm(32) statistics + apply(+SiLU), LayerNorm (+ fused per-frame add), row softmax.
// All global accesses are 16-byte vectors along the contiguous channel dimension.
#include <cstdlib>

#include "common.cuh"
#include "host_util.cuh"
#include "v3d_b200.h"

namespace v3d {

// ------------------------------------------------------------------------------------------------
// GroupNorm over [samples][rows][C] bf16 (row stride ldx) -> y dense, act = optional SiLU.
// Every kernel uses one thread layout: thread t owns the 8-channel vector column vc = t % vpr (vpr = C / 8) and the
// row lane rl = t / vpr of lanes_r = blockDim.x / vpr; over rows [r0, r1) it visits r0 + rl, r0 + rl + lanes_r, ...
//
// Statistics blocks: a sample's rows, [frames][hw], are cut into blocks of R rows that never straddle a frame (the
// last block of a frame may be short).  Each (block, group) gets ONE fp32 (sum, sumsq) pair from a fixed in-CTA tree,
// and a sample's pairs are folded in fp64 in block order.  No atomics on data, so the result depends only on the block
// geometry and the data:
//   default mode        one block per CTA (hw = rows_per_sample, R = rows per CTA, chosen from the co-resident grid);
//   deterministic mode  R = min(256, hw), whatever the grid, nsamples or sharded plan (the partials of a frame subset
//                       equal those of the same frames inside the whole tensor), so the partials + fold_apply pair,
//                       the single launch and every sharded plan produce the same bits.
// gn_stats_kernel alone sums with atomics (fp64 out, all-reduced by the frame-sharded default path).
// ------------------------------------------------------------------------------------------------
constexpr int kGnThreads = 256;
constexpr int kGnUnroll = 8;  // independent 16-byte loads in flight per thread
constexpr long long kGnDetRows = 256;

__host__ __device__ __forceinline__ long long gn_det_block_rows(long long hw) { return hw < kGnDetRows ? hw : kGnDetRows; }
__host__ __device__ __forceinline__ long long gn_blocks_per_frame(long long hw, long long R) { return (hw + R - 1) / R; }

// rows [r0, r1) of block `blk` of a sample (frames of hw rows, blocks of R rows); ONE_FRAME: the sample is one frame
template <bool ONE_FRAME = false>
__device__ __forceinline__ void gn_block_range(long long blk, long long hw, long long R, long long& r0, long long& r1) {
  const long long nbf = gn_blocks_per_frame(hw, R);
  const long long f = ONE_FRAME ? 0 : blk / nbf, b = blk - f * nbf;
  r0 = f * hw + b * R;
  r1 = r0 + R < (f + 1) * hw ? r0 + R : (f + 1) * hw;
}

// f(u, r) for this thread's rows r of [r0, r1) (u = its 16-byte vector of row r; xb = the sample's first row + its
// column), kGnUnroll loads in flight; ascending rows, or descending when REVERSE.
template <bool REVERSE, class F>
__device__ __forceinline__ void gn_rows(const bf16* __restrict__ xb, long long r0, long long r1, long long ldx,
                                        int lanes_r, int rl, F&& f) {
  if (!REVERSE) {
    long long r = r0 + rl;
    for (; r + static_cast<long long>(kGnUnroll - 1) * lanes_r < r1; r += static_cast<long long>(kGnUnroll) * lanes_r) {
      uint4 u[kGnUnroll];
#pragma unroll
      for (int k = 0; k < kGnUnroll; ++k)
        u[k] = __ldg(reinterpret_cast<const uint4*>(xb + (r + static_cast<long long>(k) * lanes_r) * ldx));
#pragma unroll
      for (int k = 0; k < kGnUnroll; ++k) f(u[k], r + static_cast<long long>(k) * lanes_r);
    }
    for (; r < r1; r += lanes_r) f(__ldg(reinterpret_cast<const uint4*>(xb + r * ldx)), r);
  } else {
    // this thread's rows are r0 + rl + i * lanes_r, i = 0 .. n_i - 1
    const long long span = r1 - r0 - rl;
    long long i = span > 0 ? (span + lanes_r - 1) / lanes_r : 0;
    for (; i >= kGnUnroll; i -= kGnUnroll) {
      uint4 u[kGnUnroll];
#pragma unroll
      for (int k = 0; k < kGnUnroll; ++k)
        u[k] = __ldg(reinterpret_cast<const uint4*>(xb + (r0 + rl + (i - 1 - k) * lanes_r) * ldx));
#pragma unroll
      for (int k = 0; k < kGnUnroll; ++k) f(u[k], r0 + rl + (i - 1 - k) * lanes_r);
    }
    for (; i > 0; --i) {
      const long long r = r0 + rl + (i - 1) * lanes_r;
      f(__ldg(reinterpret_cast<const uint4*>(xb + r * ldx)), r);
    }
  }
}

// this thread's column sums (x, x^2) of its 8 channels over its rows of [r0, r1), in row order
__device__ __forceinline__ void gn_col_sums(const bf16* __restrict__ xb, long long r0, long long r1, long long ldx,
                                            int lanes_r, int rl, float (&s)[8], float (&q)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  gn_rows<false>(xb, r0, r1, ldx, lanes_r, rl, [&](const uint4& u, long long) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      s[2 * j] += f.x; q[2 * j] = fmaf(f.x, f.x, q[2 * j]);
      s[2 * j + 1] += f.y; q[2 * j + 1] = fmaf(f.y, f.y, q[2 * j + 1]);
    }
  });
}

// The CTA's column sums -> ONE (sum, sumsq) pair per group in part[g]: through s_red ([2][lanes_r][C] floats), then
// one warp per group adds the group's (row lane, channel) sums lane-strided and folds the lanes with an xor-shuffle
// tree.  Only FULL warps take part (240-thread CTAs end in a 16-lane warp: a full-mask shuffle there would read lanes
// that do not exist).  Called by every thread; the first sync lets a previous call's tree finish reading s_red.
__device__ __forceinline__ void gn_cta_pairs(const float (&s)[8], const float (&q)[8], int C, int groups, float* s_red,
                                             float2* __restrict__ part) {
  const int vpr = C >> 3;
  const int lanes_r = blockDim.x / vpr;
  const int vc = threadIdx.x % vpr;
  const int rl = threadIdx.x / vpr;
  const int cg = C / groups;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  __syncthreads();
  {
    float* ss = s_red + (static_cast<size_t>(rl) * C + vc * 8);
    float* qq = ss + static_cast<size_t>(lanes_r) * C;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      ss[j] = s[j];
      qq[j] = q[j];
    }
  }
  __syncthreads();
  for (int g = warp < nwarps ? warp : groups; g < groups; g += nwarps) {
    float a = 0.f, b = 0.f;
    const int n = cg * lanes_r;
    for (int i = lane; i < n; i += 32) {
      const int rr = i / cg, cc = g * cg + (i - rr * cg);
      a += s_red[static_cast<size_t>(rr) * C + cc];
      b += s_red[static_cast<size_t>(lanes_r + rr) * C + cc];
    }
    a = warp_sum(a);
    b = warp_sum(b);
    if (lane == 0) part[g] = make_float2(a, b);
  }
}

// s_stat[g] = {mean, rstd} (fp32) of group g from its fp64 (sum, sumsq) over cnt elements
__device__ __forceinline__ void gn_set_stat(float* s_stat, int g, double sum, double sumsq, double cnt, float eps) {
  const double mean = sum / cnt;
  double var = sumsq / cnt - mean * mean;
  if (var < 0.0) var = 0.0;
  s_stat[2 * g] = static_cast<float>(mean);
  s_stat[2 * g + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// mean / rstd of every group of one sample from its nblk block pairs ([nblk][groups]) -> s_stat: one full warp per
// group, lane l adds blocks l, l + 32, ... in fp64, then an xor-shuffle tree.  The order depends on nblk only.  The
// caller synchronises before reading s_stat.
__device__ __forceinline__ void gn_fold(const float2* __restrict__ part, long long nblk, int groups, double cnt,
                                        float eps, float* s_stat) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int g = warp < nwarps ? warp : groups; g < groups; g += nwarps) {
    double a = 0.0, b = 0.0;
    for (long long k = lane; k < nblk; k += 32) {
      const float2 p = __ldcg(&part[k * groups + g]);
      a += static_cast<double>(p.x);
      b += static_cast<double>(p.y);
    }
    a = warp_sum_f64(a);
    b = warp_sum_f64(b);
    if (lane == 0) gn_set_stat(s_stat, g, a, b, cnt, eps);
  }
}

// this thread's scale / shift of its 8 channels from s_stat, gamma and beta
__device__ __forceinline__ void gn_scale_shift(const float* s_stat, const float* __restrict__ gamma,
                                               const float* __restrict__ beta, int C, int groups, float (&sc)[8],
                                               float (&sh)[8]) {
  const int vc = threadIdx.x % (C >> 3);
  const int cg = C / groups;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = vc * 8 + j;
    const int g = c / cg;
    const float a = s_stat[2 * g + 1] * __ldg(gamma + c);
    sc[j] = a;
    sh[j] = __ldg(beta + c) - s_stat[2 * g] * a;
  }
}

// y = act(x * sc + sh) over this thread's rows of [r0, r1) (xb / yb: the sample's first row + this thread's column)
template <bool REVERSE>
__device__ __forceinline__ void gn_apply_rows(const bf16* __restrict__ xb, bf16* __restrict__ yb, long long r0,
                                              long long r1, long long ldx, int C, int lanes_r, int rl,
                                              const float (&sc)[8], const float (&sh)[8], int silu) {
  gn_rows<REVERSE>(xb, r0, r1, ldx, lanes_r, rl, [&](const uint4& u, long long r) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      float a = fmaf(f.x, sc[2 * j], sh[2 * j]);
      float b = fmaf(f.y, sc[2 * j + 1], sh[2 * j + 1]);
      if (silu) {
        a = silu_f(a);
        b = silu_f(b);
      }
      o[j] = pack_bf16x2(a, b);
    }
    *reinterpret_cast<uint4*>(yb + r * static_cast<long long>(C)) = make_uint4(o[0], o[1], o[2], o[3]);
  });
}

// Sense-reversing grid barrier in the workspace: works for any grid size, launch after launch on one stream, provided
// every CTA of the grid is resident at once.
struct GnBarrier {
  unsigned int count;
  unsigned int gen;
};

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(unsigned int* p, unsigned int v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ void gn_grid_barrier(GnBarrier* bar) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int total = gridDim.x * gridDim.y;
    const unsigned int my_gen = ld_acquire_u32(&bar->gen);
    __threadfence();
    const unsigned int prev = atomicAdd(&bar->count, 1u);
    if (prev == total - 1) {
      bar->count = 0;
      __threadfence();
      st_release_u32(&bar->gen, my_gen + 1);
    } else {
      while (ld_acquire_u32(&bar->gen) == my_gen) __nanosleep(64);
    }
  }
  __syncthreads();
}

// stats[sample][group] = {sum, sumsq} (double), accumulated with atomics: smem float atomics per channel, then fp64
// global atomics per group.  grid = (row chunks of rows_per_cta, samples).
__global__ void __launch_bounds__(512)
gn_stats_kernel(const bf16* __restrict__ x, double* __restrict__ stats, long long rows_per_sample, int C,
                long long ldx, int groups, int rows_per_cta) {
  extern __shared__ float s_acc[];  // [2][C]
  const int vpr = C >> 3;
  const int sample = blockIdx.y;
  const long long row0 = static_cast<long long>(blockIdx.x) * rows_per_cta;
  long long row1 = row0 + rows_per_cta;
  if (row1 > rows_per_sample) row1 = rows_per_sample;
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) s_acc[i] = 0.f;
  __syncthreads();
  const int lanes_r = blockDim.x / vpr;
  const int vc = threadIdx.x % vpr;
  const int rl = threadIdx.x / vpr;
  float s[8], q[8];
  gn_col_sums(x + (static_cast<long long>(sample) * rows_per_sample) * ldx + vc * 8, row0, row1, ldx, lanes_r, rl, s, q);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    atomicAdd(&s_acc[vc * 8 + j], s[j]);
    atomicAdd(&s_acc[C + vc * 8 + j], q[j]);
  }
  __syncthreads();
  const int cg = C / groups;
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    double ds = 0.0, dq = 0.0;
    for (int c = 0; c < cg; ++c) {
      ds += static_cast<double>(s_acc[g * cg + c]);
      dq += static_cast<double>(s_acc[C + g * cg + c]);
    }
    double* o = stats + (static_cast<long long>(sample) * groups + g) * 2;
    atomicAdd(o, ds);
    atomicAdd(o + 1, dq);
  }
}

// The block pairs of the deterministic statistics: grid = (blocks per sample, samples), one CTA per block;
// partial = float2 [samples][ldp][groups].
__global__ void __launch_bounds__(512)
gn_partials_kernel(const bf16* __restrict__ x, float2* __restrict__ partial, long long rows_per_sample, long long hw,
                   int C, long long ldx, int groups, long long ldp) {
  extern __shared__ float s_red[];  // [2][lanes_r][C]
  const int vpr = C >> 3;
  const int sample = blockIdx.y;
  long long r0, r1;
  gn_block_range(blockIdx.x, hw, gn_det_block_rows(hw), r0, r1);
  float s[8], q[8];
  gn_col_sums(x + static_cast<long long>(sample) * rows_per_sample * ldx + (threadIdx.x % vpr) * 8, r0, r1, ldx,
              blockDim.x / vpr, threadIdx.x / vpr, s, q);
  gn_cta_pairs(s, q, C, groups, s_red, partial + (static_cast<long long>(sample) * ldp + blockIdx.x) * groups);
}

// Where the apply kernel's mean / rstd come from: fp64 (sum, sumsq) [samples][groups][2] of gn_stats_kernel ...
struct GnStatsF64 {
  const double* stats;
  __device__ __forceinline__ void operator()(int sample, int groups, double cnt, float eps, float* s_stat) const {
    const double* st = stats + static_cast<long long>(sample) * groups * 2;
    for (int g = threadIdx.x; g < groups; g += blockDim.x) gn_set_stat(s_stat, g, st[2 * g], st[2 * g + 1], cnt, eps);
  }
};
// ... or the fold of nblk block pairs per sample ([samples][nblk][groups])
struct GnFoldPartials {
  const float2* partial;
  long long nblk;
  __device__ __forceinline__ void operator()(int sample, int groups, double cnt, float eps, float* s_stat) const {
    gn_fold(partial + static_cast<long long>(sample) * nblk * groups, nblk, groups, cnt, eps, s_stat);
  }
};

// grid = (row chunks of rows_per_cta, samples): mean / rstd of the sample's groups over count_rows x C/groups
// elements, then normalise the CTA's rows.
template <class Stat>
__global__ void __launch_bounds__(512)
gn_apply_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, Stat stat, const float* __restrict__ gamma,
                const float* __restrict__ beta, long long rows_per_sample, long long count_rows, int C, long long ldx,
                int groups, float eps, int silu, int rows_per_cta) {
  extern __shared__ float s_stat[];  // [groups][2]
  const int vpr = C >> 3;
  const int vc = threadIdx.x % vpr;
  const int sample = blockIdx.y;
  stat(sample, groups, static_cast<double>(count_rows) * (C / groups), eps, s_stat);
  __syncthreads();
  float sc[8], sh[8];
  gn_scale_shift(s_stat, gamma, beta, C, groups, sc, sh);
  const long long row0 = static_cast<long long>(blockIdx.x) * rows_per_cta;
  const long long row1 = row0 + rows_per_cta < rows_per_sample ? row0 + rows_per_cta : rows_per_sample;
  const long long srow = static_cast<long long>(sample) * rows_per_sample;
  gn_apply_rows<false>(x + srow * ldx + vc * 8, y + srow * static_cast<long long>(C) + vc * 8, row0, row1, ldx, C,
                       blockDim.x / vpr, threadIdx.x / vpr, sc, sh, silu);
}

// GroupNorm in ONE launch: the CTAs of a sample stride over its blocks (CTA i takes blocks i, i + gridDim.x, ...) and
// write the block pairs, a grid barrier (the grid is sized to be co-resident), then EVERY CTA folds all blocks of its
// sample (so the fold does not depend on gridDim) and normalises the rows of its own blocks, last row first (the rows
// read last are the ones most likely still in the 50 MB L2).  One launch and one HBM read less than a two-kernel pair.
// MAXT / MINB: launch bounds.  <256, 3> (80 registers) is what every width up to C = 2048 uses: three 240-256-thread
// CTAs per SM instead of two keep enough loads in flight for the streaming phases; wider rows take <512, 1>.
// ONE: one block per CTA (the default mode: hw = rows_per_sample, gridDim.x blocks), which drops the block loops and
// their 64-bit divisions from the short per-CTA prologue / epilogue.
template <int MAXT, int MINB, bool ONE>
__global__ void __launch_bounds__(MAXT, MINB)
gn_fused_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, const float* __restrict__ gamma,
                const float* __restrict__ beta, GnBarrier* __restrict__ bar, float2* __restrict__ partial,
                long long rows_per_sample, long long hw, long long R, int C, long long ldx, int groups, float eps,
                int silu) {
  extern __shared__ float s_red[];  // [2][lanes_r][C] thread sums, reused as s_stat [groups][2]
  const int vpr = C >> 3;
  const int lanes_r = blockDim.x / vpr;
  const int vc = threadIdx.x % vpr;
  const int rl = threadIdx.x / vpr;
  const int sample = blockIdx.y;
  const long long nblk = ONE ? gridDim.x : rows_per_sample / hw * gn_blocks_per_frame(hw, R);
  const long long srow = static_cast<long long>(sample) * rows_per_sample;
  const bf16* xb = x + srow * ldx + vc * 8;
  float2* ps = partial + static_cast<long long>(sample) * nblk * groups;
  for (long long blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
    long long r0, r1;
    gn_block_range<ONE>(blk, hw, R, r0, r1);
    float s[8], q[8];
    gn_col_sums(xb, r0, r1, ldx, lanes_r, rl, s, q);
    gn_cta_pairs(s, q, C, groups, s_red, ps + blk * groups);
  }
  gn_grid_barrier(bar);
  gn_fold(ps, nblk, groups, static_cast<double>(rows_per_sample) * (C / groups), eps, s_red);
  __syncthreads();
  float sc[8], sh[8];
  gn_scale_shift(s_red, gamma, beta, C, groups, sc, sh);
  if (static_cast<long long>(blockIdx.x) >= nblk) return;
  bf16* yb = y + srow * static_cast<long long>(C) + vc * 8;
  const long long last = ONE ? blockIdx.x : blockIdx.x + (nblk - 1 - blockIdx.x) / gridDim.x * gridDim.x;
  for (long long blk = last; blk >= 0; blk -= gridDim.x) {
    long long r0, r1;
    gn_block_range<ONE>(blk, hw, R, r0, r1);
    gn_apply_rows<true>(xb, yb, r0, r1, ldx, C, lanes_r, rl, sc, sh, silu);
  }
}
// ------------------------------------------------------------------------------------------------
// LayerNorm over C (<= 2048), one warp per row, row held in registers.
//   z = x[row] + add[row / rows_per_frame]   (add optional, fp32)
//   ysum[row] = bf16(z)                      (optional)
//   y[row] = (z - mean) * rstd * gamma + beta
// ------------------------------------------------------------------------------------------------
constexpr int kLnMaxVec = 8;  // 8 vectors * 8 elements * 32 lanes = 2048 channels

template <int VPL>  // 16-byte vectors per lane: C <= VPL * 256
__global__ void __launch_bounds__(256)
layernorm_kernel(const bf16* __restrict__ x, const float* __restrict__ add, bf16* __restrict__ ysum,
                 bf16* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta,
                 long long rows, int C, int rows_per_frame, float eps) {
  const int warps = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int vpr = C >> 3;
  for (long long row = static_cast<long long>(blockIdx.x) * warps + (threadIdx.x >> 5); row < rows;
       row += static_cast<long long>(gridDim.x) * warps) {
    float v[VPL][8];
    const bf16* xr = x + row * C;
    const float* ar = add ? add + (row / rows_per_frame) * C : nullptr;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int vc = lane + i * 32;
      if (vc < vpr) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(xr + vc * 8));
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(w[j]);
          v[i][2 * j] = f.x;
          v[i][2 * j + 1] = f.y;
        }
        if (ar) {
          const float4 a0 = __ldg(reinterpret_cast<const float4*>(ar + vc * 8));
          const float4 a1 = __ldg(reinterpret_cast<const float4*>(ar + vc * 8 + 4));
          v[i][0] += a0.x; v[i][1] += a0.y; v[i][2] += a0.z; v[i][3] += a0.w;
          v[i][4] += a1.x; v[i][5] += a1.y; v[i][6] += a1.z; v[i][7] += a1.w;
          if (ysum) {
            // round once so that the residual stream and the LN input agree bit-for-bit
#pragma unroll
            for (int j = 0; j < 8; ++j) v[i][j] = __bfloat162float(__float2bfloat16_rn(v[i][j]));
            *reinterpret_cast<uint4*>(ysum + row * C + vc * 8) =
                make_uint4(pack_bf16x2(v[i][0], v[i][1]), pack_bf16x2(v[i][2], v[i][3]),
                           pack_bf16x2(v[i][4], v[i][5]), pack_bf16x2(v[i][6], v[i][7]));
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[i][j];
      }
    }
    s = warp_sum(s);
    const float mean = s / static_cast<float>(C);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      if (lane + i * 32 < vpr) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[i][j] - mean;
          q += d * d;
        }
      }
    }
    q = warp_sum(q);
    const float rstd = rsqrtf(q / static_cast<float>(C) + eps);
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int vc = lane + i * 32;
      if (vc < vpr) {
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + vc * 8));
        const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + vc * 8 + 4));
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + vc * 8));
        const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + vc * 8 + 4));
        const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * gg[j] + bb[j];
        *reinterpret_cast<uint4*>(y + row * C + vc * 8) =
            make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]),
                       pack_bf16x2(o[6], o[7]));
      }
    }
  }
}

// LayerNorm, C = LPR * 40 (320 / 640 / 1280): LPR lanes per row, 5 vectors (40 channels) per lane, 32/LPR rows per
// warp in flight.  Compared with one-warp-per-row this keeps every lane busy at C = 320 (40 vectors), cuts the
// shuffle reductions to log2(LPR) steps and quadruples the bytes in flight per warp.
template <int LPR>
__global__ void __launch_bounds__(256)
layernorm40_kernel(const bf16* __restrict__ x, const float* __restrict__ add, bf16* __restrict__ ysum,
                   bf16* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta,
                   long long rows, int rows_per_frame, float eps) {
  constexpr int C = LPR * 40;
  constexpr int RPW = 32 / LPR;  // rows per warp per iteration
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR;     // which row of the warp's group
  const int l = lane % LPR;       // lane within the row
  const long long warp_id = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  for (long long row0 = warp_id * RPW; row0 < rows; row0 += nwarps * RPW) {
    const long long row = row0 + sub;
    const bool ok = row < rows;
    float v[5][8];
    float s = 0.f;
    if (ok) {
      const bf16* xr = x + row * C;
      uint4 u[5];
#pragma unroll
      for (int i = 0; i < 5; ++i) u[i] = __ldg(reinterpret_cast<const uint4*>(xr + (l + i * LPR) * 8));
      const float* ar = add ? add + (row / rows_per_frame) * C : nullptr;
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const uint32_t w[4] = {u[i].x, u[i].y, u[i].z, u[i].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(w[j]);
          v[i][2 * j] = f.x;
          v[i][2 * j + 1] = f.y;
        }
        if (ar) {
          const int c0 = (l + i * LPR) * 8;
          const float4 a0 = __ldg(reinterpret_cast<const float4*>(ar + c0)), a1 = __ldg(reinterpret_cast<const float4*>(ar + c0 + 4));
          v[i][0] += a0.x; v[i][1] += a0.y; v[i][2] += a0.z; v[i][3] += a0.w;
          v[i][4] += a1.x; v[i][5] += a1.y; v[i][6] += a1.z; v[i][7] += a1.w;
          if (ysum) {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[i][j] = __bfloat162float(__float2bfloat16_rn(v[i][j]));
            *reinterpret_cast<uint4*>(ysum + row * C + c0) =
                make_uint4(pack_bf16x2(v[i][0], v[i][1]), pack_bf16x2(v[i][2], v[i][3]), pack_bf16x2(v[i][4], v[i][5]),
                           pack_bf16x2(v[i][6], v[i][7]));
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[i][j];
      }
    } else {
#pragma unroll
      for (int i = 0; i < 5; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) v[i][j] = 0.f;
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * (1.0f / C);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 5; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[i][j] - mean;
        q = fmaf(d, d, q);
      }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q * (1.0f / C) + eps);
    if (ok) {
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const int c0 = (l + i * LPR) * 8;
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c0)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c0 + 4));
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c0)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c0 + 4));
        const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf((v[i][j] - mean) * rstd, gg[j], bb[j]);
        *reinterpret_cast<uint4*>(y + row * C + (l + i * LPR) * 8) =
            make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// In-place row softmax over bf16 scores (decoder AttnBlock, one 4096-wide row per CTA).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
softmax_rows_kernel(bf16* __restrict__ x, int n, float scale) {
  __shared__ float red[8];
  __shared__ float bcast;
  bf16* row = x + static_cast<long long>(blockIdx.x) * n;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nv = n >> 3;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + i * 8);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      m = fmaxf(m, fmaxf(f.x, f.y));
    }
  }
  m = warp_max(m);
  if (lane == 0) red[warp] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = red[0];
    for (int i = 1; i < (blockDim.x >> 5); ++i) t = fmaxf(t, red[i]);
    bcast = t;
  }
  __syncthreads();
  m = bcast * scale;
  float s = 0.f;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + i * 8);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      s += __expf(f.x * scale - m) + __expf(f.y * scale - m);
    }
  }
  s = warp_sum(s);
  __syncthreads();
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += red[i];
    bcast = 1.f / t;
  }
  __syncthreads();
  const float inv = bcast;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + i * 8);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      o[j] = pack_bf16x2(__expf(f.x * scale - m) * inv, __expf(f.y * scale - m) * inv);
    }
    *reinterpret_cast<uint4*>(row + i * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// fp32 scores -> bf16 probabilities (separate buffers): keeps the decoder's 4096-wide softmax input in fp32.
__global__ void __launch_bounds__(256)
softmax_rows_f32_kernel(const float* __restrict__ x, bf16* __restrict__ y, int n, float scale) {
  __shared__ float red[8];
  __shared__ float bcast;
  const float* row = x + static_cast<long long>(blockIdx.x) * n;
  bf16* orow = y + static_cast<long long>(blockIdx.x) * n;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nv = n >> 2;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const float4 f = *reinterpret_cast<const float4*>(row + i * 4);
    m = fmaxf(m, fmaxf(fmaxf(f.x, f.y), fmaxf(f.z, f.w)));
  }
  m = warp_max(m);
  if (lane == 0) red[warp] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = red[0];
    for (int i = 1; i < (blockDim.x >> 5); ++i) t = fmaxf(t, red[i]);
    bcast = t;
  }
  __syncthreads();
  m = bcast * scale;
  float s = 0.f;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const float4 f = *reinterpret_cast<const float4*>(row + i * 4);
    s += __expf(f.x * scale - m) + __expf(f.y * scale - m) + __expf(f.z * scale - m) + __expf(f.w * scale - m);
  }
  s = warp_sum(s);
  __syncthreads();
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += red[i];
    bcast = 1.f / t;
  }
  __syncthreads();
  const float inv = bcast;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const float4 f = *reinterpret_cast<const float4*>(row + i * 4);
    *reinterpret_cast<uint2*>(orow + i * 4) =
        make_uint2(pack_bf16x2(__expf(f.x * scale - m) * inv, __expf(f.y * scale - m) * inv),
                   pack_bf16x2(__expf(f.z * scale - m) * inv, __expf(f.w * scale - m) * inv));
  }
}

static int pick_rows_per_cta(long long rows_per_sample, int nsamples) {
  // a few CTAs per SM, each with enough rows that the per-CTA prologue / reduction tail stays small next to the
  // streaming loop (V3D_GN_WAVES overrides the CTA-per-SM target: tuning knob)
  static int waves = 0;
  if (waves == 0) {
    const char* v = getenv("V3D_GN_WAVES");
    waves = v ? atoi(v) : 4;
    if (waves < 1) waves = 1;
  }
  const long long target = static_cast<long long>(waves) * num_sms();
  long long chunks = (target + nsamples - 1) / nsamples;
  if (chunks < 1) chunks = 1;
  long long rpc = (rows_per_sample + chunks - 1) / chunks;
  if (rpc < 32) rpc = 32;
  if (rpc > rows_per_sample) rpc = rows_per_sample;
  return static_cast<int>(rpc);
}

// Launch shape of the GroupNorm kernels at width C: C / 8 vector columns x lanes_r row lanes (about kGnThreads
// threads), and the [2][lanes_r][C] floats of the CTA tree (gn_cta_pairs).
struct GnShape {
  int lanes_r, threads;
  size_t smem;
};
static GnShape gn_shape(int C) {
  const int vpr = C / 8;
  const int lanes_r = kGnThreads / vpr > 0 ? kGnThreads / vpr : 1;
  return {lanes_r, vpr * lanes_r, sizeof(float) * 2 * static_cast<size_t>(lanes_r) * C};
}

// What every GroupNorm entry point requires of the shape
static bool gn_shape_ok(int C, int ldx, int groups, long long rows_per_sample, int nsamples) {
  return C > 0 && C % 8 == 0 && groups > 0 && C % groups == 0 && C / 8 <= 512 && ldx % 8 == 0 &&
         rows_per_sample > 0 && nsamples > 0;
}

// Workspace of the single launch: the barrier words, then the block pairs (float2 [samples][blocks][groups]).
constexpr size_t kGnWsHeader = 256;
constexpr int kGnMaxCtas = 4096;  // CTAs the default mode's fixed-size workspace has pairs for
static int64_t gn_ws_bytes(long long pairs) { return static_cast<int64_t>(kGnWsHeader + sizeof(float2) * pairs); }

// gn_fused_kernel over nsamples x (CTAs per sample).  det: the blocks of min(256, hw) rows, which the CTAs of a
// sample stride over; otherwise one block per CTA.  The grid barrier needs every CTA resident at once, so the grid is
// held to the co-resident capacity (occupancy x SMs, at most 4 CTAs per SM and kGnMaxCtas in all);
// V3D_ERR_UNSUPPORTED when nsamples exceeds it (the caller then takes the two-kernel form).
static int gn_fused(const char* who, bool det, const void* x, void* y, const void* gamma, const void* beta,
                    long long rows_per_sample, long long hw, int nsamples, int C, int ldx, int groups, float eps,
                    int silu, void* workspace, void* stream) {
  const GnShape sh = gn_shape(C);
  auto kern = sh.threads <= 256 ? (det ? gn_fused_kernel<256, 3, false> : gn_fused_kernel<256, 3, true>)
                                 : (det ? gn_fused_kernel<512, 1, false> : gn_fused_kernel<512, 1, true>);
  int per_sm = 0;
  const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, sh.threads, sh.smem);
  if (e != cudaSuccess || per_sm < 1) {
    set_error("%s: occupancy query failed (%s)", who, cudaGetErrorString(e));
    return V3D_ERR_CUDA;
  }
  long long cap = static_cast<long long>(per_sm < 4 ? per_sm : 4) * num_sms();
  if (cap > kGnMaxCtas) cap = kGnMaxCtas;
  if (nsamples > cap) {
    set_error("%s: %d samples exceed the co-resident grid (%lld CTAs)", who, nsamples, cap);
    return V3D_ERR_UNSUPPORTED;
  }
  long long ctas = cap / nsamples, R;
  if (det) {
    R = gn_det_block_rows(hw);
    const long long nblk = rows_per_sample / hw * gn_blocks_per_frame(hw, R);
    if (ctas > nblk) ctas = nblk;
  } else {
    // >= 16 rows per thread: the barrier and the pairs must stay small next to the streaming loops
    long long max_ctas = rows_per_sample / (16LL * sh.lanes_r);
    if (max_ctas < 1) max_ctas = 1;
    if (ctas > max_ctas) ctas = max_ctas;
    hw = rows_per_sample;
    R = (rows_per_sample + ctas - 1) / ctas;
    ctas = (rows_per_sample + R - 1) / R;
  }
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  kern<<<dim3(static_cast<unsigned>(ctas), nsamples), sh.threads, sh.smem, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const bf16*>(x), static_cast<bf16*>(y), static_cast<const float*>(gamma),
      static_cast<const float*>(beta), reinterpret_cast<GnBarrier*>(ws), reinterpret_cast<float2*>(ws + kGnWsHeader),
      rows_per_sample, hw, R, C, ldx, groups, eps, silu);
  V3D_CHECK_LAUNCH("gn_fused_kernel");
  return V3D_OK;
}

// gn_apply_kernel over row chunks of pick_rows_per_cta rows x nsamples
template <class Stat>
static int gn_apply(Stat stat, const void* x, void* y, const void* gamma, const void* beta, long long rows_per_sample,
                    long long count_rows, int nsamples, int C, int ldx, int groups, float eps, int silu, void* stream) {
  const int rpc = pick_rows_per_cta(rows_per_sample, nsamples);
  gn_apply_kernel<<<dim3(static_cast<unsigned>((rows_per_sample + rpc - 1) / rpc), nsamples), gn_shape(C).threads,
                    sizeof(float) * 2 * groups, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const bf16*>(x), static_cast<bf16*>(y), stat, static_cast<const float*>(gamma),
      static_cast<const float*>(beta), rows_per_sample, count_rows, C, ldx, groups, eps, silu, rpc);
  V3D_CHECK_LAUNCH("gn_apply_kernel");
  return V3D_OK;
}

}  // namespace v3d

using namespace v3d;

extern "C" {

/* GroupNorm statistics over [nsamples][rows_per_sample][C] (bf16, row stride ldx) -> stats double
 * [nsamples][groups][2] = {sum, sumsq}. rows_per_sample = H*W for 2-D GroupNorm32/Normalize
 * (diffusionmodules/util.py:259-276, attention.py:130-133, model.py:52-55) and T*H*W for the 3-D
 * time_stack ResBlock (openaimodel.py:267-271 with dims=3: reduction over (C/32, T, H, W)). */
int v3d_groupnorm_stats(const void* x, void* stats, int64_t rows_per_sample, int32_t nsamples, int32_t C,
                        int32_t ldx, int32_t groups, int32_t pre_zeroed, void* stream) {
  if (!x || !stats || !gn_shape_ok(C, ldx, groups, rows_per_sample, nsamples)) {
    set_error("v3d_groupnorm_stats: bad args C=%d groups=%d ldx=%d", C, groups, ldx);
    return V3D_ERR_BAD_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!pre_zeroed) {
    cudaError_t e = cudaMemsetAsync(stats, 0, sizeof(double) * 2 * groups * nsamples, st);
    if (e != cudaSuccess) {
      set_error("memset stats: %s", cudaGetErrorString(e));
      return V3D_ERR_CUDA;
    }
  }
  const int rpc = pick_rows_per_cta(rows_per_sample, nsamples);
  gn_stats_kernel<<<dim3(static_cast<unsigned>((rows_per_sample + rpc - 1) / rpc), nsamples), gn_shape(C).threads,
                    2 * C * sizeof(float), st>>>(static_cast<const bf16*>(x), static_cast<double*>(stats),
                                                 rows_per_sample, C, ldx, groups, rpc);
  V3D_CHECK_LAUNCH("gn_stats_kernel");
  return V3D_OK;
}

/* y[dense, ld=C] = act(GroupNorm(x; stats, gamma, beta, eps)), act = SiLU when silu != 0
 * (fuses normalization() + nn.SiLU of openaimodel.py:267-271,300-303; model.py:131-143 nonlinearity). */
int v3d_groupnorm_apply(const void* x, void* y, const void* stats, const void* gamma, const void* beta,
                        int64_t rows_per_sample, int32_t nsamples, int32_t C, int32_t ldx, int32_t groups,
                        float eps, int32_t silu, void* stream) {
  if (!x || !y || !stats || !gamma || !beta || !gn_shape_ok(C, ldx, groups, rows_per_sample, nsamples)) {
    set_error("v3d_groupnorm_apply: bad args C=%d groups=%d ldx=%d", C, groups, ldx);
    return V3D_ERR_BAD_ARG;
  }
  return gn_apply(GnStatsF64{static_cast<const double*>(stats)}, x, y, gamma, beta, rows_per_sample, rows_per_sample,
                  nsamples, C, ldx, groups, eps, silu, stream);
}

/* Bytes of the workspace v3d_groupnorm needs (barrier words + per-CTA partials); the caller allocates it once per
 * stream, ZEROED, and passes the same buffer to every call on that stream. */
int64_t v3d_groupnorm_workspace_bytes(void) { return gn_ws_bytes(32LL * kGnMaxCtas); }

/* y[dense, ld=C] = act(GroupNorm(x; gamma, beta, eps)) in ONE launch (statistics + grid barrier + apply); same
 * operand meaning as the v3d_groupnorm_stats / v3d_groupnorm_apply pair it replaces on the unsharded path
 * (GroupNorm32 + SiLU openaimodel.py:267-271,300-303, diffusionmodules/util.py:259-276; Normalize model.py:52-55,
 * attention.py:130-133).  Deterministic (no atomics on data).  Calls sharing a workspace must be stream-ordered. */
int v3d_groupnorm(const void* x, void* y, const void* gamma, const void* beta, int64_t rows_per_sample,
                  int32_t nsamples, int32_t C, int32_t ldx, int32_t groups, float eps, int32_t silu,
                  void* workspace, int64_t workspace_bytes, void* stream) {
  if (!x || !y || !gamma || !beta || !workspace || !gn_shape_ok(C, ldx, groups, rows_per_sample, nsamples) ||
      groups > 32 || workspace_bytes < v3d_groupnorm_workspace_bytes()) {
    set_error("v3d_groupnorm: bad args C=%d groups=%d ldx=%d workspace=%lld", C, groups, ldx,
              static_cast<long long>(workspace_bytes));
    return V3D_ERR_BAD_ARG;
  }
  return gn_fused("v3d_groupnorm", false, x, y, gamma, beta, rows_per_sample, rows_per_sample, nsamples, C, ldx,
                  groups, eps, silu, workspace, stream);
}

/* Deterministic GroupNorm: blocks per sample of the statistics definition (rows_per_sample = frames x hw, blocks of
 * min(256, hw) rows that never straddle a frame); -1 if hw does not divide rows_per_sample. */
int64_t v3d_groupnorm_det_blocks(int64_t rows_per_sample, int64_t hw) {
  if (hw <= 0 || rows_per_sample <= 0 || rows_per_sample % hw != 0) return -1;
  return rows_per_sample / hw * gn_blocks_per_frame(hw, gn_det_block_rows(hw));
}

/* Bytes of the workspace v3d_groupnorm_det needs for this shape (barrier words + one fp32 pair per block and group). */
int64_t v3d_groupnorm_det_workspace_bytes(int64_t rows_per_sample, int64_t hw, int32_t nsamples, int32_t groups) {
  const int64_t nblk = v3d_groupnorm_det_blocks(rows_per_sample, hw);
  if (nblk < 0 || nsamples <= 0 || groups <= 0) return -1;
  return gn_ws_bytes(nblk * nsamples * groups);
}

/* Block partials of the deterministic statistics: partials = float2 [nsamples][ldp][groups], block k of sample s at
 * [s][k] (k < v3d_groupnorm_det_blocks(rows_per_sample, hw) <= ldp). */
int v3d_groupnorm_partials(const void* x, void* partials, int64_t rows_per_sample, int64_t hw, int32_t nsamples,
                           int32_t C, int32_t ldx, int32_t groups, int64_t ldp, void* stream) {
  const int64_t nblk = v3d_groupnorm_det_blocks(rows_per_sample, hw);
  if (!x || !partials || !gn_shape_ok(C, ldx, groups, rows_per_sample, nsamples) || groups > 32 || nblk <= 0 ||
      ldp < nblk || nsamples > 65535) {
    set_error("v3d_groupnorm_partials: bad args C=%d groups=%d ldx=%d hw=%lld ldp=%lld", C, groups, ldx,
              static_cast<long long>(hw), static_cast<long long>(ldp));
    return V3D_ERR_BAD_ARG;
  }
  const GnShape sh = gn_shape(C);
  gn_partials_kernel<<<dim3(static_cast<unsigned>(nblk), nsamples), sh.threads, sh.smem,
                       static_cast<cudaStream_t>(stream)>>>(static_cast<const bf16*>(x), static_cast<float2*>(partials),
                                                            rows_per_sample, hw, C, ldx, groups, ldp);
  V3D_CHECK_LAUNCH("gn_partials_kernel");
  return V3D_OK;
}

/* y[dense, ld=C] = act(GroupNorm(x)) from block partials: each sample's nblocks pairs (float2 [nsamples][nblocks]
 * [groups]) are folded in block order, over count_rows x C/groups elements (count_rows = rows the partials cover: the
 * whole video's when x holds one rank's frames of it). */
int v3d_groupnorm_fold_apply(const void* x, void* y, const void* partials, const void* gamma, const void* beta,
                             int64_t rows_per_sample, int32_t nsamples, int32_t C, int32_t ldx, int32_t groups,
                             int64_t nblocks, int64_t count_rows, float eps, int32_t silu, void* stream) {
  if (!x || !y || !partials || !gamma || !beta || !gn_shape_ok(C, ldx, groups, rows_per_sample, nsamples) ||
      groups > 32 || nblocks <= 0 || count_rows <= 0 || nsamples > 65535) {
    set_error("v3d_groupnorm_fold_apply: bad args C=%d groups=%d ldx=%d nblocks=%lld", C, groups, ldx,
              static_cast<long long>(nblocks));
    return V3D_ERR_BAD_ARG;
  }
  return gn_apply(GnFoldPartials{static_cast<const float2*>(partials), nblocks}, x, y, gamma, beta, rows_per_sample,
                  count_rows, nsamples, C, ldx, groups, eps, silu, stream);
}

/* The deterministic normalisation in ONE launch; bit-identical to v3d_groupnorm_partials + v3d_groupnorm_fold_apply.
 * workspace: >= v3d_groupnorm_det_workspace_bytes(rows_per_sample, hw, nsamples, groups) bytes, zeroed once by the
 * caller, then passed unchanged to every call on the same stream. */
int v3d_groupnorm_det(const void* x, void* y, const void* gamma, const void* beta, int64_t rows_per_sample, int64_t hw,
                      int32_t nsamples, int32_t C, int32_t ldx, int32_t groups, float eps, int32_t silu,
                      void* workspace, int64_t workspace_bytes, void* stream) {
  const int64_t need = v3d_groupnorm_det_workspace_bytes(rows_per_sample, hw, nsamples, groups);
  if (!x || !y || !gamma || !beta || !workspace || !gn_shape_ok(C, ldx, groups, rows_per_sample, nsamples) ||
      groups > 32 || need < 0 || workspace_bytes < need) {
    set_error("v3d_groupnorm_det: bad args C=%d groups=%d ldx=%d hw=%lld workspace=%lld (need %lld)", C, groups, ldx,
              static_cast<long long>(hw), static_cast<long long>(workspace_bytes), static_cast<long long>(need));
    return V3D_ERR_BAD_ARG;
  }
  return gn_fused("v3d_groupnorm_det", true, x, y, gamma, beta, rows_per_sample, hw, nsamples, C, ldx, groups, eps,
                  silu, workspace, stream);
}

/* LayerNorm (attention.py:525-527, video_attention.py:51,79,93-94) with the optional fused
 * "x_mix = x + emb" of video_attention.py:286-287 (add = per-frame fp32 vectors, ysum receives x+emb). */
int v3d_layernorm(const void* x, const void* add, void* ysum, void* y, const void* gamma, const void* beta,
                  int64_t rows, int32_t C, int32_t rows_per_frame, float eps, void* stream) {
  if (!x || !y || !gamma || !beta || C % 8 != 0 || C > kLnMaxVec * 256 || rows <= 0) {
    set_error("v3d_layernorm: bad args C=%d", C);
    return V3D_ERR_BAD_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int warps = 8;
  long long blocks = (rows + warps - 1) / warps;
  const long long cap = 32LL * num_sms();
  if (blocks > cap) blocks = cap;
  if (C == 320 || C == 640 || C == 1280) {
    const int lpr = C / 40;
    const long long rows_per_cta = 8LL * (32 / lpr);
    long long nb = (rows + rows_per_cta - 1) / rows_per_cta;
    // grid-stride over rows: V3D_LN_CTAS_PER_SM (tuning knob) bounds the grid in CTAs per SM
    static int ln_ctas = 0;
    if (ln_ctas == 0) {
      const char* v = getenv("V3D_LN_CTAS_PER_SM");
      // 8: fastest of 2 / 4 / 6 / 8 / 12 at the UNet's three LayerNorm shapes on one H100 (0.076 / 0.042 / 0.024 ms)
      ln_ctas = v ? atoi(v) : 8;
      if (ln_ctas < 1) ln_ctas = 1;
    }
    const long long cap2 = static_cast<long long>(ln_ctas) * num_sms();
    if (nb > cap2) nb = cap2;
#define V3D_LN40(L)                                                                                              \
  layernorm40_kernel<L><<<static_cast<unsigned>(nb), 256, 0, st>>>(                                             \
      static_cast<const bf16*>(x), static_cast<const float*>(add), static_cast<bf16*>(ysum), static_cast<bf16*>(y), \
      static_cast<const float*>(gamma), static_cast<const float*>(beta), rows, rows_per_frame > 0 ? rows_per_frame : 1, eps)
    if (lpr == 8) V3D_LN40(8);
    else if (lpr == 16) V3D_LN40(16);
    else V3D_LN40(32);
#undef V3D_LN40
    V3D_CHECK_LAUNCH("layernorm40_kernel");
    return V3D_OK;
  }
  const int vpl = (C / 8 + 31) / 32;
#define V3D_LN_LAUNCH(V)                                                                                   \
  layernorm_kernel<V><<<static_cast<unsigned>(blocks), warps * 32, 0, st>>>(                                \
      static_cast<const bf16*>(x), static_cast<const float*>(add), static_cast<bf16*>(ysum),               \
      static_cast<bf16*>(y), static_cast<const float*>(gamma), static_cast<const float*>(beta), rows, C,   \
      rows_per_frame > 0 ? rows_per_frame : 1, eps)
  switch (vpl) {
    case 1: V3D_LN_LAUNCH(1); break;
    case 2: V3D_LN_LAUNCH(2); break;
    case 3: V3D_LN_LAUNCH(3); break;
    case 4: V3D_LN_LAUNCH(4); break;
    case 5: V3D_LN_LAUNCH(5); break;
    default: V3D_LN_LAUNCH(8); break;
  }
#undef V3D_LN_LAUNCH
  V3D_CHECK_LAUNCH("layernorm_kernel");
  return V3D_OK;
}

/* In-place softmax(scale * x) over rows of n bf16 scores (decoder AttnBlock, model.py:190-192). */
int v3d_softmax_rows(void* x, int64_t rows, int32_t n, float scale, void* stream) {
  if (!x || n % 8 != 0 || rows <= 0 || rows > 0x7fffffffLL) {
    set_error("v3d_softmax_rows: bad args");
    return V3D_ERR_BAD_ARG;
  }
  softmax_rows_kernel<<<static_cast<unsigned>(rows), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<bf16*>(x), n, scale);
  V3D_CHECK_LAUNCH("softmax_rows_kernel");
  return V3D_OK;
}

/* softmax(scale * x) from fp32 scores to bf16 probabilities (decoder AttnBlock, model.py:190-192). */
int v3d_softmax_rows_f32(const void* x, void* y, int64_t rows, int32_t n, float scale, void* stream) {
  if (!x || !y || n % 4 != 0 || rows <= 0 || rows > 0x7fffffffLL) {
    set_error("v3d_softmax_rows_f32: bad args");
    return V3D_ERR_BAD_ARG;
  }
  softmax_rows_f32_kernel<<<static_cast<unsigned>(rows), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(x), static_cast<bf16*>(y), n, scale);
  V3D_CHECK_LAUNCH("softmax_rows_f32_kernel");
  return V3D_OK;
}

}  // extern "C"
