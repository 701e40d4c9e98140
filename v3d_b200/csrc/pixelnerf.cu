// PixelNeRF scene conditioning (sgm/modules/encoders/pixelnerf.py): rays, fused sample render, per-ray decoder.
//
//   pnerf_rays_kernel     one thread per target ray: origin / unit direction (RayGenerator.forward) and the [-1, 1]^3
//                         box limits (math_utils.get_ray_limits_box); the min / max of t_start over valid rays is
//                         reduced on the device (ordered-uint atomicMin) for the reference's miss fallback.
//   pnerf_render_kernel   persistent, 2 warpgroups per CTA, each warpgroup one ray at a time in 64-sample tiles:
//                         jittered depth -> projection into every source -> bilinear / nearest fetch -> mean, std,
//                         positional encoding -> bf16 A tile (128B swizzle) -> d_in->128->128->129 MLP on wgmma
//                         (weights resident in shared memory) -> online softmax over the sample axis with a running
//                         weighted sum of the 128 feature columns.  Only the per-ray [rays, 128] result reaches HBM.
//   pnerf_decode_kernel   the 128->128->128->131 decoder MLP on 64-ray tiles (same wgmma stages), sigmoid on rgb,
//                         NCHW fp32 stores.
// Everything is row-local with a fixed summation order: the same inputs give the same bytes.
#include "common.cuh"
#include "host_util.cuh"
#include "v3d_b200.h"
#include "wgmma.cuh"

namespace v3d {

constexpr int PN_THREADS = 256;  // two warpgroups
constexpr int PN_N3 = 136;       // 129 / 131 output columns, zero-padded to the n136 wgmma tile
constexpr int PN_W23 = 128 * 256 + PN_N3 * 256;
constexpr int PN_WG_BYTES_BASE = 16384 + 2048 + 1024;  // H tile + column-sum scratch + logits (rounded up)
constexpr uint32_t PN_NO_VALID = 0xffffffffu;

__host__ __device__ constexpr int pn_wg_bytes(int kp) { return kp * 8192 + PN_WG_BYTES_BASE; }
__host__ __device__ constexpr int pn_smem_bytes(int kp) { return kp * 16384 + PN_W23 + 2 * pn_wg_bytes(kp) + 1024; }

__device__ __forceinline__ void wg_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void sts16(uint32_t addr, uint16_t v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// byte offset of element (row, col) in a K-major bf16 tile of `rows` rows: 64-column panels of 128-byte rows with the
// 128B swizzle (16-byte chunk index XOR row % 8), panels rows * 128 bytes apart
__device__ __forceinline__ uint32_t sw_off(int rows, int row, int col) {
  return (col >> 6) * rows * 128 + row * 128 + ((((col & 63) >> 3) ^ (row & 7)) << 4) + (col & 7) * 2;
}
__device__ __forceinline__ void sts_bf16(uint32_t base, int row, int col, float v) {
  __nv_bfloat16 b = __float2bfloat16_rn(v);
  sts16(base + sw_off(64, row, col), *reinterpret_cast<uint16_t*>(&b));
}
// ordered-uint image of a float: a < b  <=>  key(a) < key(b)
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// torch.max / torch.min propagate NaN
__device__ __forceinline__ float nmax(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : fmaxf(a, b); }
__device__ __forceinline__ float nmin(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : fminf(a, b); }

// row-major bf16 W [n][kpad] (global) -> swizzled K-major panels at smem byte address dst
__device__ void load_weight(uint32_t dst, const bf16* __restrict__ w, int n, int kpad) {
  const int chunks_per_row = kpad / 8;
  for (int i = threadIdx.x; i < n * chunks_per_row; i += blockDim.x) {
    const int r = i / chunks_per_row, j = i - r * chunks_per_row;
    const uint4 v = *reinterpret_cast<const uint4*>(w + static_cast<long long>(r) * kpad + j * 8);
    sts128(dst + (j >> 3) * n * 128 + r * 128 + (((j & 7) ^ (r & 7)) << 4), v.x, v.y, v.z, v.w);
  }
}

// ReLU(acc + bias) of a 64 x 128 fragment -> bf16 H tile.  Fragment: acc[4 c + 2 h + e] = row 16 wi + lane / 4 + 8 h,
// column 8 c + 2 (lane % 4) + e.
__device__ __forceinline__ void store_hidden(const float (&acc)[64], const float* __restrict__ bias, uint32_t sH) {
  const int lane = threadIdx.x & 31, wi = (threadIdx.x >> 5) & 3;
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    const int col = 8 * c + 2 * (lane & 3);
    const float b0 = __ldg(bias + col), b1 = __ldg(bias + col + 1);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = 16 * wi + (lane >> 2) + 8 * h;
      sts32(sH + sw_off(64, row, col),
            pack_bf16x2(fmaxf(acc[4 * c + 2 * h] + b0, 0.f), fmaxf(acc[4 * c + 2 * h + 1] + b1, 0.f)));
    }
  }
}

// The three linear layers on one 64-row A tile (KP 64-column panels, already written and fenced): ReLU hidden layers
// rounded to bf16 in sH, the last layer's fp32 accumulators (no bias) in acc3.  Weights: sW1 [128][64 KP],
// sW2 [128][128], sW3 [136][128], all K-major swizzled.
template <int KP>
__device__ __forceinline__ void mlp3(uint32_t sA, uint32_t sW1, uint32_t sW2, uint32_t sW3, const float* __restrict__ b1,
                                     const float* __restrict__ b2, uint32_t sH, int bar, float (&acc3)[68]) {
  float acc[64];
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4 * KP; ++kk)
    Wgmma<128>::ss(acc, gmma_desc_k_sw128(sA + (kk >> 2) * 8192) + 2 * (kk & 3),
                   gmma_desc_k_sw128(sW1 + (kk >> 2) * 16384) + 2 * (kk & 3), kk != 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  store_hidden(acc, b1, sH);
  fence_proxy_async_smem();
  wg_bar(bar);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 8; ++kk)
    Wgmma<128>::ss(acc, gmma_desc_k_sw128(sH + (kk >> 2) * 8192) + 2 * (kk & 3),
                   gmma_desc_k_sw128(sW2 + (kk >> 2) * 16384) + 2 * (kk & 3), kk != 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  wg_bar(bar);  // every warp's reads of H are done before H is overwritten
  store_hidden(acc, b2, sH);
  fence_proxy_async_smem();
  wg_bar(bar);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 8; ++kk)
    Wgmma<PN_N3>::ss(acc3, gmma_desc_k_sw128(sH + (kk >> 2) * 8192) + 2 * (kk & 3),
                     gmma_desc_k_sw128(sW3 + (kk >> 2) * (PN_N3 * 128)) + 2 * (kk & 3), kk != 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
}

// ---------------------------------------------------------------------------------------------------------------
// rays
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pnerf_rays_kernel(const float* __restrict__ cams, int ncam, int rs,
                                                         float box_half, int box, float* __restrict__ rays,
                                                         uint32_t* __restrict__ limits) {
  const long long hw = static_cast<long long>(rs) * rs;
  const long long ray = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  bool valid = false;
  float ts = 0.f;
  if (ray < ncam * hw) {
    const int cam = static_cast<int>(ray / hw);
    const int pix = static_cast<int>(ray - cam * hw);
    const float* m = cams + cam * 25;  // c2w row-major 4x4, then the normalised 3x3 intrinsics
    const float fx = m[16], sk = m[17], cx = m[18], fy = m[20], cy = m[21];
    // uv = meshgrid(ij).flip(0): u = column, v = row
    const float inv = 1.0f / static_cast<float>(rs), half = 0.5f / static_cast<float>(rs);
    const float xc = __fadd_rn(__fmul_rn(static_cast<float>(pix % rs), inv), half);
    const float yc = __fadd_rn(__fmul_rn(static_cast<float>(pix / rs), inv), half);
    float xl = __fadd_rn(__fsub_rn(xc, cx), __fdiv_rn(__fmul_rn(cy, sk), fy));
    xl = __fdiv_rn(__fsub_rn(xl, __fdiv_rn(__fmul_rn(sk, yc), fy)), fx);
    const float yl = __fdiv_rn(__fsub_rn(yc, cy), fy);
    // c2w @ diag(1, -1, -1, 1) @ (xl, yl, 1, 1) - camera centre
    float d[3], o[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      o[i] = m[4 * i + 3];
      const float w = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[4 * i], xl), __fmul_rn(-m[4 * i + 1], yl)), -m[4 * i + 2]),
                                o[i]);
      d[i] = __fsub_rn(w, o[i]);
    }
    const float nrm = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2]))),
                            1e-12f);
#pragma unroll
    for (int i = 0; i < 3; ++i) d[i] = __fdiv_rn(d[i], nrm);
    float te = 0.f;
    if (box) {
      // slab test against [-box_half, box_half]^3, in the reference's order (YZ, XZ, then XY planes)
      float lo[3], hi[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const float id = __fdiv_rn(1.0f, d[i]);
        const float bmin = id < 0.f ? box_half : -box_half, bmax = id < 0.f ? -box_half : box_half;
        lo[i] = __fmul_rn(__fsub_rn(bmin, o[i]), id);
        hi[i] = __fmul_rn(__fsub_rn(bmax, o[i]), id);
      }
      valid = !(lo[0] > hi[1] || lo[1] > hi[0]);
      float tmin = nmax(lo[0], lo[1]), tmax = nmin(hi[0], hi[1]);
      if (tmin > hi[2] || lo[2] > tmax) valid = false;
      tmin = nmax(tmin, lo[2]);
      tmax = nmin(tmax, hi[2]);
      if (!valid) {
        tmin = -1.f;
        tmax = -2.f;
      }
      ts = tmin;
      te = tmax;
      valid = te > ts;
    }
    float* r = rays + ray * 8;
    *reinterpret_cast<float4*>(r) = make_float4(o[0], o[1], o[2], d[0]);
    *reinterpret_cast<float4*>(r + 4) = make_float4(d[1], d[2], ts, te);
  }
  if (box) {
    const uint32_t kmin = __reduce_min_sync(0xffffffffu, valid ? f2key(ts) : PN_NO_VALID);
    const uint32_t kmax = __reduce_min_sync(0xffffffffu, valid ? ~f2key(ts) : PN_NO_VALID);
    if ((threadIdx.x & 31) == 0 && kmin != PN_NO_VALID) {
      atomicMin(limits, kmin);
      atomicMin(limits + 1, kmax);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// render
// ---------------------------------------------------------------------------------------------------------------
struct PnRenderArgs {
  const float* rays;        // [R][8]
  const uint32_t* limits;   // 2 ordered keys (box mode)
  const float* jitter;      // box: [ns][R] uniforms; disparity: z[ns]
  const float* src;         // [B][S][C][H][W]
  const float* src_w2c;     // [B][S][12]
  const float* src_k;       // [B][S][4]: fx, fy, cx, cy
  const bf16* w1;           // [128][64 KP]
  const float* b1;
  const bf16* w2;           // [128][128]
  const float* b2;
  const bf16* w3;           // [136][128]
  const float* b3;          // [136]
  float* feat;              // [R][128]
  long long nrays, rays_per_batch;
  int S, C, H, W, ns, d_in, flags;
  float inv_near, inv_far;
};

template <int KP>
__global__ void __launch_bounds__(PN_THREADS, 1) pnerf_render_kernel(const PnRenderArgs a) {
  extern __shared__ uint8_t pn_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(pn_smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const uint32_t sW1 = smem_u32(smem), sW2 = sW1 + KP * 16384, sW3 = sW2 + 32768;
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127, lane = threadIdx.x & 31, wi = tid >> 5;
  uint8_t* wgp = smem + KP * 16384 + PN_W23 + wg * pn_wg_bytes(KP);
  const uint32_t sA = smem_u32(wgp), sH = sA + KP * 8192;
  float* red = reinterpret_cast<float*>(wgp + KP * 8192 + 16384);  // [4 warps][128]
  float* lg = red + 512;                                           // [64] logits
  const int bar = 1 + wg;

  load_weight(sW1, a.w1, 128, 64 * KP);
  load_weight(sW2, a.w2, 128, 128);
  load_weight(sW3, a.w3, PN_N3, 128);
  // zero the A tile once: padding columns d_in .. 64 KP stay zero (0 * weight must not meet garbage)
  for (int i = tid; i < KP * 8192 / 16; i += 128) sts128(sA + i * 16, 0u, 0u, 0u, 0u);
  fence_proxy_async_smem();
  __syncthreads();

  const bool use_std = a.flags & V3D_PNERF_STD, use_pe = a.flags & V3D_PNERF_POSENC;
  const bool nearest = a.flags & V3D_PNERF_NEAREST, zeros = a.flags & V3D_PNERF_ZEROS;
  const bool disparity = a.flags & V3D_PNERF_DISPARITY;
  const int S = a.S, C = a.C, H = a.H, W = a.W, ns = a.ns;
  const long long plane = static_cast<long long>(H) * W;
  const int row = tid >> 1, half = tid & 1;
  const float wm1 = static_cast<float>(W - 1), hm1 = static_cast<float>(H - 1);
  const float nsm1 = static_cast<float>(ns - 1);
  const bool have_valid = a.limits[0] != PN_NO_VALID;
  const float gmin = have_valid ? key2f(a.limits[0]) : 0.f, gmax = have_valid ? key2f(~a.limits[1]) : 0.f;

  for (long long ray = static_cast<long long>(blockIdx.x) * 2 + wg; ray < a.nrays; ray += static_cast<long long>(gridDim.x) * 2) {
    const float4 r0 = *reinterpret_cast<const float4*>(a.rays + ray * 8);
    const float4 r1 = *reinterpret_cast<const float4*>(a.rays + ray * 8 + 4);
    float ts = r1.z, te = r1.w;
    if (!disparity && have_valid && !(te > ts)) {  // RaySampler: misses take the global limits (both from t_start)
      ts = gmin;
      te = gmax;
    }
    const float diff = __fsub_rn(te, ts);
    const int b = static_cast<int>(ray / a.rays_per_batch);
    const float* srcb = a.src + static_cast<long long>(b) * S * C * plane;
    float m_run = -INFINITY, l_run = 0.f, acc_run = 0.f;

    for (int t0 = 0; t0 < ns; t0 += 64) {
      // ---- gather: two threads per sample row, channels split even / odd
      const int k = t0 + row;
      if (k < ns) {
        float depth;
        if (disparity) {
          const float z = __ldg(a.jitter + k);
          depth = __fdiv_rn(1.0f, __fadd_rn(__fmul_rn(a.inv_near, __fsub_rn(1.0f, z)), __fmul_rn(a.inv_far, z)));
        } else {
          const float u = __ldg(a.jitter + static_cast<long long>(k) * a.nrays + ray);
          depth = __fadd_rn(ts, __fmul_rn(__fdiv_rn(static_cast<float>(k), nsm1), diff));
          depth = __fadd_rn(depth, __fdiv_rn(__fmul_rn(u, diff), nsm1));
        }
        const float p[3] = {__fadd_rn(r0.x, __fmul_rn(r0.w, depth)), __fadd_rn(r0.y, __fmul_rn(r1.x, depth)),
                            __fadd_rn(r0.z, __fmul_rn(r1.y, depth))};
        for (int cb = 0; cb < C; cb += 16) {
          float mean[8], m2[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) mean[j] = m2[j] = 0.f;
          for (int s = 0; s < S; ++s) {
            const float* wm = a.src_w2c + (static_cast<long long>(b) * S + s) * 12;
            const float* km = a.src_k + (static_cast<long long>(b) * S + s) * 4;
            float q[3];
#pragma unroll
            for (int i = 0; i < 3; ++i)
              q[i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(wm + 4 * i), p[0]), __fmul_rn(__ldg(wm + 4 * i + 1), p[1])),
                                         __fmul_rn(__ldg(wm + 4 * i + 2), p[2])),
                               __ldg(wm + 4 * i + 3));
            const float qx = __fdiv_rn(-q[0], q[2]), qy = __fdiv_rn(-q[1], q[2]);
            const float x = __fadd_rn(__fmul_rn(qx, __ldg(km)), __ldg(km + 2));
            const float y = __fadd_rn(__fmul_rn(-qy, __ldg(km + 1)), __ldg(km + 3));
            // grid_sample(align_corners=True) of the grid value 2 x - 1
            float ix = __fmul_rn(__fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(x, 2.f), 1.f), 1.f), 0.5f), wm1);
            float iy = __fmul_rn(__fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(y, 2.f), 1.f), 1.f), 0.5f), hm1);
            if (!zeros) {
              ix = fminf(fmaxf(ix, 0.f), wm1);
              iy = fminf(fmaxf(iy, 0.f), hm1);
            }
            long long off[4];
            float wt[4];
            if (nearest) {
              const float nx = rintf(ix), ny = rintf(iy);
              const bool in = nx >= 0.f && nx <= wm1 && ny >= 0.f && ny <= hm1;
              off[0] = in ? static_cast<long long>(ny) * W + static_cast<long long>(nx) : -1;
              wt[0] = 1.f;
              off[1] = off[2] = off[3] = -1;
              wt[1] = wt[2] = wt[3] = 0.f;
            } else {
              const float x0 = floorf(ix), y0 = floorf(iy), x1 = x0 + 1.f, y1 = y0 + 1.f;
              wt[0] = __fmul_rn(__fsub_rn(x1, ix), __fsub_rn(y1, iy));  // nw
              wt[1] = __fmul_rn(__fsub_rn(ix, x0), __fsub_rn(y1, iy));  // ne
              wt[2] = __fmul_rn(__fsub_rn(x1, ix), __fsub_rn(iy, y0));  // sw
              wt[3] = __fmul_rn(__fsub_rn(ix, x0), __fsub_rn(iy, y0));  // se
              const float xs[2] = {x0, x1}, ys[2] = {y0, y1};
#pragma unroll
              for (int tp = 0; tp < 4; ++tp) {
                const float tx = xs[tp & 1], ty = ys[tp >> 1];
                const bool in = tx >= 0.f && tx <= wm1 && ty >= 0.f && ty <= hm1;
                off[tp] = in ? static_cast<long long>(ty) * W + static_cast<long long>(tx) : -1;
              }
            }
            const float* img = srcb + static_cast<long long>(s) * C * plane;
            const float inv_n = 1.0f / static_cast<float>(s + 1);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int c = cb + half + 2 * j;
              if (c < C) {
                const float* ip = img + c * plane;
                float v = 0.f;
#pragma unroll
                for (int tp = 0; tp < 4; ++tp) v += (off[tp] >= 0 ? __ldg(ip + off[tp]) : 0.f) * wt[tp];
                const float dl = v - mean[j];  // Welford
                mean[j] = fmaf(dl, inv_n, mean[j]);
                m2[j] = fmaf(dl, v - mean[j], m2[j]);
              }
            }
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int c = cb + half + 2 * j;
            if (c < C) {
              sts_bf16(sA, row, c, mean[j]);
              if (use_std) sts_bf16(sA, row, C + c, S > 1 ? sqrtf(m2[j] / static_cast<float>(S - 1)) : 0.f);
            }
          }
        }
        if (use_pe) {  // NeRF positional encoding of the world sample: x, then sin(x f_i + phase) as (N C)
          const int base = use_std ? 2 * C : C;
          for (int i = half; i < 39; i += 2) {
            float v;
            if (i < 3) {
              v = p[i];
            } else {
              const int n = (i - 3) / 3, cc = (i - 3) - 3 * n;
              const float f = 3.14159265358979323846f * static_cast<float>(1 << (n >> 1));
              v = sinf(__fadd_rn(__fmul_rn(p[cc], f), (n & 1) ? 1.57079632679489661923f : 0.f));
            }
            sts_bf16(sA, row, base + i, v);
          }
        }
      } else {
        for (int c = half; c < a.d_in; c += 2) sts_bf16(sA, row, c, 0.f);
      }
      fence_proxy_async_smem();
      wg_bar(bar);

      float acc3[68];
      mlp3<KP>(sA, sW1, sW2, sW3, a.b1, a.b2, sH, bar, acc3);

      // ---- online softmax over the samples of this tile
      if ((lane & 3) == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int rr = 16 * wi + (lane >> 2) + 8 * h;
          lg[rr] = (t0 + rr < ns) ? acc3[64 + 2 * h] + __ldg(a.b3 + 128) : -INFINITY;
        }
      }
      wg_bar(bar);
      float tmax = -INFINITY;
      for (int i = 0; i < 64; ++i) tmax = fmaxf(tmax, lg[i]);
      const float m_new = fmaxf(m_run, tmax);
      const float scale = expf(m_run - m_new);
      float psum = 0.f;
      for (int i = 0; i < 64; ++i) psum += expf(lg[i] - m_new);
      const float p0 = expf(lg[16 * wi + (lane >> 2)] - m_new), p1 = expf(lg[16 * wi + (lane >> 2) + 8] - m_new);
#pragma unroll
      for (int c = 0; c < 16; ++c) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float bc = __ldg(a.b3 + 8 * c + 2 * (lane & 3) + e);
          float v = p0 * (acc3[4 * c + e] + bc) + p1 * (acc3[4 * c + 2 + e] + bc);
          v += __shfl_xor_sync(0xffffffffu, v, 4);
          v += __shfl_xor_sync(0xffffffffu, v, 8);
          v += __shfl_xor_sync(0xffffffffu, v, 16);
          if (lane < 4) red[wi * 128 + 8 * c + 2 * lane + e] = v;
        }
      }
      wg_bar(bar);
      acc_run = acc_run * scale + (((red[tid] + red[128 + tid]) + red[256 + tid]) + red[384 + tid]);
      l_run = l_run * scale + psum;
      m_run = m_new;
    }
    a.feat[ray * 128 + tid] = acc_run / l_run;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// decoder
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PN_THREADS, 1) pnerf_decode_kernel(const float* __restrict__ feat, long long nrays,
                                                                     long long hw, const bf16* w1, const float* b1,
                                                                     const bf16* w2, const float* b2, const bf16* w3,
                                                                     const float* b3, float* __restrict__ rgb,
                                                                     float* __restrict__ feats) {
  constexpr int KP = 2;
  extern __shared__ uint8_t pn_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(pn_smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const uint32_t sW1 = smem_u32(smem), sW2 = sW1 + KP * 16384, sW3 = sW2 + 32768;
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127, lane = threadIdx.x & 31, wi = tid >> 5;
  const uint32_t sA = smem_u32(smem + KP * 16384 + PN_W23 + wg * pn_wg_bytes(KP)), sH = sA + KP * 8192;
  const int bar = 1 + wg;
  load_weight(sW1, w1, 128, 128);
  load_weight(sW2, w2, 128, 128);
  load_weight(sW3, w3, PN_N3, 128);
  fence_proxy_async_smem();
  __syncthreads();

  const long long ntiles = (nrays + 63) / 64;
  for (long long tile = static_cast<long long>(blockIdx.x) * 2 + wg; tile < ntiles; tile += static_cast<long long>(gridDim.x) * 2) {
    const int row = tid >> 1, half = tid & 1;
    const long long r = tile * 64 + row;
#pragma unroll 4
    for (int j = 0; j < 32; ++j) {
      const int col = half * 64 + 2 * j;
      float2 v = make_float2(0.f, 0.f);
      if (r < nrays) v = *reinterpret_cast<const float2*>(feat + r * 128 + col);
      sts32(sA + sw_off(64, row, col), pack_bf16x2(v.x, v.y));
    }
    fence_proxy_async_smem();
    wg_bar(bar);
    float acc3[68];
    mlp3<KP>(sA, sW1, sW2, sW3, b1, b2, sH, bar, acc3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long rr = tile * 64 + 16 * wi + (lane >> 2) + 8 * h;
      if (rr >= nrays) continue;
      const long long img = rr / hw, pix = rr - img * hw;
#pragma unroll
      for (int c = 0; c < 17; ++c) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * c + 2 * (lane & 3) + e;
          if (col >= 131) continue;
          const float v = acc3[4 * c + 2 * h + e] + __ldg(b3 + col);
          if (col < 3) rgb[(img * 3 + col) * hw + pix] = 1.0f / (1.0f + expf(-v));
          else feats[(img * 128 + col - 3) * hw + pix] = v;
        }
      }
    }
    wg_bar(bar);  // A is rewritten by the next tile only after every warp's layer-1 reads
  }
}

template <typename K>
int pn_set_smem(K kern, int bytes, bool& done) {
  if (!done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) {
      set_error("pixelnerf smem attr (%d bytes): %s", bytes, cudaGetErrorString(e));
      return V3D_ERR_CUDA;
    }
    done = true;
  }
  return V3D_OK;
}

}  // namespace v3d

using namespace v3d;

extern "C" {

/* RayGenerator.forward (sgm/modules/encoders/pixelnerf.py:77-158) and, with `box`, get_ray_limits_box
 * (math_utils.py) for a box of half side `box_half`, plus the miss fallback reduction of RaySampler.forward
 * (pixelnerf.py:182-188) without its host sync.  cams: [ncam][25] fp32 rows (c2w, normalised K); rays out:
 * [ncam * rs * rs][8] = (origin, unit direction, t_start, t_end), pixel-major within a camera; limits: 2 words of
 * caller-owned scratch (overwritten). */
int v3d_pixelnerf_rays(const void* cams, int32_t ncam, int32_t render_size, float box_half, int32_t box, void* rays,
                       void* limits, void* stream) {
  if (!cams || !rays || !limits || ncam <= 0 || render_size <= 0 ||
      static_cast<long long>(ncam) * render_size * render_size > (1LL << 31) - 256) {
    set_error("v3d_pixelnerf_rays: bad args");
    return V3D_ERR_BAD_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(limits, 0xff, 8, st);
  if (e != cudaSuccess) {
    set_error("v3d_pixelnerf_rays: memset: %s", cudaGetErrorString(e));
    return V3D_ERR_CUDA;
  }
  const long long n = static_cast<long long>(ncam) * render_size * render_size;
  pnerf_rays_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(
      static_cast<const float*>(cams), ncam, render_size, box_half, box, static_cast<float*>(rays),
      static_cast<uint32_t*>(limits));
  V3D_CHECK_LAUNCH("pnerf_rays_kernel");
  return V3D_OK;
}

/* The per-sample half of PixelNeRF.forward (pixelnerf.py:160-182 depths, 263-303 project / grid_sample / reduce /
 * feature_aggregator / softmax / weighted sum) fused: nothing per sample leaves the chip. */
int v3d_pixelnerf_render(const void* rays, const void* limits, const void* jitter, const void* src, const void* src_w2c,
                         const void* src_k, int64_t nrays, int64_t rays_per_batch, int32_t S, int32_t C, int32_t H,
                         int32_t W, int32_t ns, int32_t flags, float inv_near, float inv_far, const void* w1,
                         int32_t d_in, const void* b1, const void* w2, const void* b2, const void* w3, const void* b3,
                         void* feat, void* stream) {
  const int kp = (d_in + 63) / 64;
  const int want = C * ((flags & V3D_PNERF_STD) ? 2 : 1) + ((flags & V3D_PNERF_POSENC) ? 39 : 0);
  if (!rays || !limits || !jitter || !src || !src_w2c || !src_k || !w1 || !b1 || !w2 || !b2 || !w3 || !b3 || !feat ||
      nrays <= 0 || rays_per_batch <= 0 || nrays % rays_per_batch != 0 || S <= 0 || C <= 0 || H <= 0 || W <= 0 ||
      ns < 2 || d_in != want || kp > 3) {
    set_error("v3d_pixelnerf_render: bad args (d_in = %d, expected %d, at most 192; ns = %d, at least 2)", d_in, want,
              ns);
    return V3D_ERR_BAD_ARG;
  }
  PnRenderArgs a;
  a.rays = static_cast<const float*>(rays);
  a.limits = static_cast<const uint32_t*>(limits);
  a.jitter = static_cast<const float*>(jitter);
  a.src = static_cast<const float*>(src);
  a.src_w2c = static_cast<const float*>(src_w2c);
  a.src_k = static_cast<const float*>(src_k);
  a.w1 = static_cast<const bf16*>(w1);
  a.b1 = static_cast<const float*>(b1);
  a.w2 = static_cast<const bf16*>(w2);
  a.b2 = static_cast<const float*>(b2);
  a.w3 = static_cast<const bf16*>(w3);
  a.b3 = static_cast<const float*>(b3);
  a.feat = static_cast<float*>(feat);
  a.nrays = nrays;
  a.rays_per_batch = rays_per_batch;
  a.S = S, a.C = C, a.H = H, a.W = W, a.ns = ns, a.d_in = d_in, a.flags = flags;
  a.inv_near = inv_near, a.inv_far = inv_far;
  const long long want_ctas = (nrays + 1) / 2;
  const unsigned grid = static_cast<unsigned>(want_ctas < num_sms() ? want_ctas : num_sms());
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static bool cfg[3] = {false, false, false};
  int rc;
  switch (kp) {
    case 1:
      if ((rc = pn_set_smem(pnerf_render_kernel<1>, pn_smem_bytes(1), cfg[0])) != V3D_OK) return rc;
      pnerf_render_kernel<1><<<grid, PN_THREADS, pn_smem_bytes(1), st>>>(a);
      break;
    case 2:
      if ((rc = pn_set_smem(pnerf_render_kernel<2>, pn_smem_bytes(2), cfg[1])) != V3D_OK) return rc;
      pnerf_render_kernel<2><<<grid, PN_THREADS, pn_smem_bytes(2), st>>>(a);
      break;
    default:
      if ((rc = pn_set_smem(pnerf_render_kernel<3>, pn_smem_bytes(3), cfg[2])) != V3D_OK) return rc;
      pnerf_render_kernel<3><<<grid, PN_THREADS, pn_smem_bytes(3), st>>>(a);
      break;
  }
  V3D_CHECK_LAUNCH("pnerf_render_kernel");
  return V3D_OK;
}

/* PixelNeRF.decoder + split / sigmoid / rearrange (pixelnerf.py:305-313) over the per-ray features feat [nrays][128]
 * fp32: rgb [nrays / hw][3][hw] and feats [nrays / hw][128][hw], fp32 NCHW. */
int v3d_pixelnerf_decode(const void* feat, int64_t nrays, int64_t hw, const void* w1, const void* b1, const void* w2,
                         const void* b2, const void* w3, const void* b3, void* rgb, void* feats, void* stream) {
  if (!feat || !w1 || !b1 || !w2 || !b2 || !w3 || !b3 || !rgb || !feats || nrays <= 0 || hw <= 0 ||
      nrays % hw != 0) {
    set_error("v3d_pixelnerf_decode: bad args");
    return V3D_ERR_BAD_ARG;
  }
  static bool cfg = false;
  int rc = pn_set_smem(pnerf_decode_kernel, pn_smem_bytes(2), cfg);
  if (rc != V3D_OK) return rc;
  const long long want_ctas = ((nrays + 63) / 64 + 1) / 2;
  const unsigned grid = static_cast<unsigned>(want_ctas < num_sms() ? want_ctas : num_sms());
  pnerf_decode_kernel<<<grid, PN_THREADS, pn_smem_bytes(2), static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(feat), nrays, hw, static_cast<const bf16*>(w1), static_cast<const float*>(b1),
      static_cast<const bf16*>(w2), static_cast<const float*>(b2), static_cast<const bf16*>(w3),
      static_cast<const float*>(b3), static_cast<float*>(rgb), static_cast<float*>(feats));
  V3D_CHECK_LAUNCH("pnerf_decode_kernel");
  return V3D_OK;
}

}  // extern "C"
