// wgmma GEMM / temporal-conv / implicit-GEMM 3x3 conv for sm_90a.
//
// One persistent, warp-specialised kernel, 128 x BN output tiles:
//   warpgroup 0    : TMA producer (one thread; A tile 128x64 bf16 + B tile BNx64 bf16 per pipeline stage, 128B swizzle)
//                    and, for the bf16 epilogues, one epilogue I/O thread (warp 1): it loads each tile's residual
//                    sub-tiles into the staging buffer by TMA while the consumers still run the tile's main loop, and
//                    writes the finished tile out of the same buffer by TMA.
//   warpgroups 1-2 : consumers.  Each owns 64 rows of the tile: wgmma.mma_async m64nBNk16 from shared memory into
//                    fp32 register accumulators, then the epilogue straight from those registers (bias / per-frame
//                    bias / SiLU / GEGLU / residual blend -> bf16 sub-tiles staged in shared memory and written by TMA,
//                    or fp32 stores).  While the consumers run the epilogue the producer already fills the ring with
//                    the next tile's operands.
// Operand gather modes (see include/v3d_b200.h): linear rows, 3-tap temporal shift, 3x3 spatial taps.
// The im2row never exists in memory: each (tap, 64-channel) K-block is one TMA box whose out-of-bounds
// part is zero-filled by the hardware, which is exactly the conv zero padding.
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "host_util.cuh"
#include "v3d_b200.h"
#include "wgmma.cuh"

namespace v3d {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kThreads = 384;  // warpgroup 0 TMA, warpgroups 1 and 2 MMA + epilogue
constexpr int kConsumerThreads = 256;
constexpr int kSmemBudget = 227 * 1024;

struct GemmEpi {
  void* D;
  const float* bias;
  const float* fbias;
  const bf16* R1;
  const bf16* R2;
  long long ldd, ldr1, ldr2, ldfb;
  int batch, rows_per_batch, tiles_per_batch;
  int N, kpt, ntaps, tap_shift;  // kpt = K-blocks per tap
  int rows_per_frame, act, out_fp32;
  int b_batched;
  int transposed, valid_cols, accumulate;  // small-M mode: D is fp32 [cols][ldd], D[col][row]; bias per row
  // conv3x3 geometry
  int cn, ch, cw, bw, bh, bn, tiles_w, tiles_h, bw_shift, bh_shift, tw_shift, th_shift;  // t*_shift < 0: not pow2
  int num_m_tiles, num_n_tiles;
  float s0, s1, s2;
  int tap0;  // A row coordinate of tap 0 relative to the output row: a_row0 - (ntaps / 2) * tap_shift
  // residuals fetched into shared memory by TMA (mapR1 / mapR2) instead of __ldg from the epilogue: every residual's
  // base and row pitch are 16-byte aligned.  R2 is staged only by the variants that have room for it (Cfg::R2_STAGED).
  int res_tma;
};

// Fused GEMM -> all-gather over peer memory: output sub-tiles whose first column is >= col0 are stored a second time
// through each of these tensor maps (destination matrices that may live on other GPUs: IPC-mapped arenas), by the same
// epilogue I/O thread with the same cp.async.bulk.tensor instruction.  n = 0: off (every launch but the frame-sharded K|V
// projection).
struct alignas(64) KvMaps {
  CUtensorMap m[8];
  int n;
  int col0;
};

// epilogue variants (compile-time): what is stored and how
constexpr int EPI_BF16 = 0;   // bf16 sub-tiles staged in shared memory, written by TMA; at most one residual (R1)
constexpr int EPI_BF16R2 = 4; // as EPI_BF16 with both residuals (blend epilogue); the only variant that carries R2
constexpr int EPI_GEGLU = 1;  // value * gelu(gate) then as EPI_BF16 (linear mode only)
constexpr int EPI_F32 = 2;    // fp32 direct stores (optional SiLU)
constexpr int EPI_TRANS = 3;  // fp32 transposed store with per-row bias (small-M mode, linear only)

template <int BN, int EPI>
struct Cfg {
  static constexpr bool STAGED = EPI == EPI_BF16 || EPI == EPI_BF16R2 || EPI == EPI_GEGLU;
  static constexpr int OUT_COLS = EPI == EPI_GEGLU ? BN / 2 : BN;
  // bf16 output leaves as 128-row x SUBW-column TMA stores (64B-swizzled rows when SUBW = 32)
  static constexpr int SUBW = OUT_COLS % 32 == 0 ? 32 : 16;
  static constexpr int NSUB = OUT_COLS / SUBW;
  static constexpr int SUB_BYTES = BM * SUBW * 2;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int TILE_OUT_BYTES = NSUB * SUB_BYTES;
  // R2 takes a second staging buffer, but only where the operand ring keeps at least 4 stages with it (BN <= 160);
  // BN = 256 would drop to 2 stages, so there R2 stays an __ldg from the epilogue.
  static constexpr bool R2_STAGED =
      EPI == EPI_BF16R2 && (kSmemBudget - 2048 - 2 * TILE_OUT_BYTES) / STAGE_BYTES >= 4;
  static constexpr int STAGING_BYTES = STAGED ? (R2_STAGED ? 2 : 1) * TILE_OUT_BYTES : 0;
  static constexpr int NSTAGE_RAW = (kSmemBudget - 2048 - STAGING_BYTES) / STAGE_BYTES;
  static constexpr int NSTAGE = NSTAGE_RAW > 8 ? 8 : NSTAGE_RAW;
  static constexpr int SMEM_BYTES = NSTAGE * STAGE_BYTES + STAGING_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(NSTAGE >= 2, "pipeline too shallow");
};

// Persistent tile walk without per-tile divisions: tile = first + i * step, n fastest.
struct TileWalk {
  int n_tile, m_tile, step_n, step_m, num_n;
  __device__ __forceinline__ explicit TileWalk(const GemmEpi& p) {
    num_n = p.num_n_tiles;
    n_tile = static_cast<int>(blockIdx.x) % num_n;
    m_tile = static_cast<int>(blockIdx.x) / num_n;
    step_n = static_cast<int>(gridDim.x) % num_n;
    step_m = static_cast<int>(gridDim.x) / num_n;
  }
  __device__ __forceinline__ void next() {
    n_tile += step_n;
    m_tile += step_m;
    if (n_tile >= num_n) {
      n_tile -= num_n;
      ++m_tile;
    }
  }
};

__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

// m_tile -> tile origin. conv: (w0, h0, img0); linear: (batch index, first row, 0)
template <bool CONV>
__device__ __forceinline__ void tile_origin(const GemmEpi& p, int m_tile, int& t0, int& t1, int& t2) {
  if (CONV) {
    int tw, th, tn;
    if (p.tw_shift >= 0) {
      tw = m_tile & (p.tiles_w - 1);
      th = (m_tile >> p.tw_shift) & (p.tiles_h - 1);
      tn = m_tile >> (p.tw_shift + p.th_shift);
    } else {
      tw = m_tile % p.tiles_w;
      th = (m_tile / p.tiles_w) % p.tiles_h;
      tn = m_tile / (p.tiles_w * p.tiles_h);
    }
    t0 = tw * p.bw;
    t1 = th * p.bh;
    t2 = tn * p.bn;
  } else {
    if (p.batch == 1) {
      t0 = 0;
      t1 = m_tile * BM;
    } else {
      t0 = m_tile / p.tiles_per_batch;
      t1 = (m_tile - t0 * p.tiles_per_batch) * BM;
    }
    t2 = 0;
  }
}

template <int BN, bool CONV, int EPI>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
               const __grid_constant__ CUtensorMap mapD, const __grid_constant__ CUtensorMap mapR1,
               const __grid_constant__ CUtensorMap mapR2, const GemmEpi p, const __grid_constant__ KvMaps kv) {
  using C = Cfg<BN, EPI>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* staging = smem + C::NSTAGE * C::STAGE_BYTES;  // output tile (and R1), then R2 when C::R2_STAGED
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + C::STAGING_BYTES);
  uint64_t* empty_bar = full_bar + C::NSTAGE;
  uint64_t* stg_ready = empty_bar + C::NSTAGE;  // staging free for the next tile and its residuals have landed
  uint64_t* stg_full = stg_ready + 1;           // the consumers have written the tile's output into staging
  const bool res_staged = (EPI == EPI_BF16 || EPI == EPI_BF16R2) && p.res_tma != 0;  // GEGLU takes no residual
  const bool r2_staged = C::R2_STAGED && p.res_tma != 0 && p.R2 != nullptr;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
    if (C::STAGED) tma_prefetch_desc(&mapD);
    if (res_staged) tma_prefetch_desc(&mapR1);
    if (r2_staged) tma_prefetch_desc(&mapR2);
    for (int i = 0; i < C::NSTAGE; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);  // one arrival per consumer warpgroup
    }
    mbar_init(stg_ready, 1);  // the I/O thread (plus the residual bytes)
    mbar_init(stg_full, 1);   // one consumer thread, after a barrier over all 256
    fence_barrier_init();
  }
  __syncthreads();

  const int total_tiles = p.num_m_tiles * p.num_n_tiles;
  const int num_kb = p.ntaps * p.kpt;

  if (threadIdx.x < 128) {
    // ------------------------------ TMA producer ------------------------------
    regs_dec<40>();
    if (C::STAGED && threadIdx.x == 32) {
      // ---- epilogue I/O: per tile, residuals in, then output out, through the one staging buffer.
      // Ordering: the residual load of tile t is issued only after bulk_wait_read has seen every TMA store of tile
      // t-1 finish reading staging (same thread, so its bulk group covers them all), and the consumers touch staging
      // for tile t only after stg_ready completes for t, i.e. after that load's bytes have arrived (or, without a
      // staged residual, after the plain arrive that follows the same wait).  The stores of tile t are issued only
      // after stg_full says both consumer warpgroups wrote it, each thread having fenced its generic-proxy writes
      // for the async proxy first.  Each barrier is at most one phase ahead of its waiter.
      uint32_t sphase = 0;
      const uint32_t stg = smem_u32(staging);
      TileWalk tw(p);
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, tw.next()) {
        int t0, t1, t2;
        tile_origin<CONV>(p, tw.m_tile, t0, t1, t2);
        const int obase = tw.n_tile * C::OUT_COLS;
        if (res_staged) {
          // a tile's residual rows are its own output rows: TMA zero-fills the rows past the end, the store clips them
          mbar_arrive_expect_tx(stg_ready, C::TILE_OUT_BYTES * (r2_staged ? 2 : 1));
#pragma unroll 1
          for (int sub = 0; sub < C::NSUB; ++sub) {
            uint8_t* dst = staging + sub * C::SUB_BYTES;
            const int col0 = obase + sub * C::SUBW;
            if (CONV) tma_load_4d(dst, &mapR1, stg_ready, col0, t0, t1, t2);
            else tma_load_3d(dst, &mapR1, stg_ready, col0, t1, t0);
            if (r2_staged) {
              if (CONV) tma_load_4d(dst + C::TILE_OUT_BYTES, &mapR2, stg_ready, col0, t0, t1, t2);
              else tma_load_3d(dst + C::TILE_OUT_BYTES, &mapR2, stg_ready, col0, t1, t0);
            }
          }
        } else {
          mbar_arrive(stg_ready);
        }
        mbar_wait(stg_full, sphase);
        sphase ^= 1u;
        // the whole bf16 tile is in shared memory: TMA clips it at row / image tails
#pragma unroll 1
        for (int sub = 0; sub < C::NSUB; ++sub) {
          const uint32_t src = stg + static_cast<uint32_t>(sub * C::SUB_BYTES);
          const int col0 = obase + sub * C::SUBW;
          if (CONV) tma_store_4d(&mapD, src, col0, t0, t1, t2);
          else tma_store_3d(&mapD, src, col0, t1, t0);
          if (!CONV && EPI == EPI_BF16 && kv.n > 0 && col0 >= kv.col0) {
            // fused all-gather: the same sub-tile into every rank's gather buffer (peer memory over NVLink)
            for (int i = 0; i < kv.n; ++i) tma_store_3d(&kv.m[i], src, col0 - kv.col0, t1, t0);
          }
        }
        bulk_commit();
        bulk_wait_read<0>();
      }
      bulk_wait_all();  // the last stores have landed before the CTA (and its staging buffer) goes away
    }
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      TileWalk tw(p);
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, tw.next()) {
        int c1, c2, c3;
        if (CONV) tile_origin<true>(p, tw.m_tile, c1, c2, c3);
        else tile_origin<false>(p, tw.m_tile, c2, c1, c3);
        const int bz = p.b_batched ? c2 : 0;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem + stage * C::STAGE_BYTES;
          uint8_t* sb = sa + C::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);
          const int tap = kb / p.kpt;
          const int kc = (kb - tap * p.kpt) * BK;
          if (CONV) {
            const int ky = tap / 3, kx = tap - ky * 3;
            tma_load_4d(sa, &mapA, &full_bar[stage], kc, c1 + kx - 1, c2 + ky - 1, c3);
          } else {
            tma_load_3d(sa, &mapA, &full_bar[stage], kc, c1 + tap * p.tap_shift + p.tap0, c2);
          }
          tma_load_3d(sb, &mapB, &full_bar[stage], kb * BK, tw.n_tile * BN, bz);
          if (++stage == C::NSTAGE) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
    return;
  }

  // ------------------------------ consumers: MMA + epilogue ------------------------------
  regs_inc<232>();
  constexpr bool GEGLU = EPI == EPI_GEGLU;
  constexpr bool DUAL = EPI == EPI_BF16R2 || EPI == EPI_F32;  // variants that may take a second residual
  constexpr int OUT_COLS = C::OUT_COLS;
  constexpr int SUBW = C::SUBW;
  const int ct = threadIdx.x - 128;       // 0..255
  const int cw = ct >> 7;                 // consumer warpgroup: tile rows [64 cw, 64 cw + 64)
  const int wi = (ct >> 5) & 3;           // warp inside the warpgroup: 16 of those rows
  const int lane = ct & 31;
  const bool wg_leader = (ct & 127) == 0;
  const bool store_leader = ct == 0;
  const int cq = (lane & 3) * 2;          // first of the thread's two columns inside each 8-column group
  const int tr_base = cw * 64 + wi * 16 + (lane >> 2);  // tile rows tr_base and tr_base + 8
  const bool has_bias = p.bias != nullptr;
  // the GEGLU variant carries no residual / per-frame bias code (rejected on the host): registers
  const bool has_fb = !GEGLU && p.fbias != nullptr;
  const bool has_r1 = !GEGLU && p.R1 != nullptr;
  const bool has_r2 = DUAL && p.R2 != nullptr;
  const bool do_silu = p.act == V3D_ACT_SILU;
  const float s0 = p.s0, s1 = p.s1, s2 = p.s2;
  const uint32_t stg = smem_u32(staging);

  // tile row -> (valid, global row). bw/bh are powers of two (checked on the host).
  auto map_row = [&](int tr, int o0, int o1, int o2, long long& grow) -> bool {
    if (CONV) {
      const int w = tr & (p.bw - 1);
      const int h = (tr >> p.bw_shift) & (p.bh - 1);
      const int img = o2 + (tr >> (p.bw_shift + p.bh_shift));
      grow = (static_cast<long long>(img) * p.ch + (o1 + h)) * p.cw + (o0 + w);
      return img < p.cn;
    } else {
      const int m = o1 + tr;
      grow = static_cast<long long>(o0) * p.rows_per_batch + m;
      return m < p.rows_per_batch;
    }
  };

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  int stage = 0;
  uint32_t phase = 0;
  uint32_t sphase = 0;
  TileWalk tw(p);
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int n_tile = tw.n_tile;
    int t0, t1, t2;
    tile_origin<CONV>(p, tw.m_tile, t0, t1, t2);
    tw.next();

    // ---- main loop: one wgmma group per K-block; the stage of block kb-1 is released once block kb is issued
    int prev = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * C::STAGE_BYTES);
      const uint64_t adesc = gmma_desc_k_sw128(sa + static_cast<uint32_t>(cw * 64 * 128));
      const uint64_t bdesc = gmma_desc_k_sw128(sa + C::A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        Wgmma<BN>::ss(acc, adesc + static_cast<uint64_t>(2 * k), bdesc + static_cast<uint64_t>(2 * k),
                      (kb | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && wg_leader) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == C::NSTAGE) {
        stage = 0;
        phase ^= 1u;
      }
    }
    wgmma_wait<0>();
    if (prev >= 0 && wg_leader) mbar_arrive(&empty_bar[prev]);

    // ---- epilogue from registers.  acc[4 j + 2 h + e] = tile row tr_base + 8 h, column 8 j + cq + e.
    if (C::STAGED) {
      // the previous tile's TMA stores have finished reading the staging buffer, and this tile's residuals are in it
      mbar_wait(stg_ready, sphase);
      sphase ^= 1u;
    }
    const int obase = n_tile * OUT_COLS;  // first output column of this tile
    const int nbase = n_tile * BN;        // first column in the (packed) N space
    // operand pointers at this thread's first column (cq), so that every load of the unrolled column loop below is
    // one instruction with an immediate offset instead of a re-derived address
    const float* bcol = has_bias && EPI != EPI_TRANS ? p.bias + nbase + cq : nullptr;
    // RS: residuals staged in shared memory.  A compile-time flag, so that the unrolled column loop of either form
    // branches on nothing but the launch-uniform flags above.
    auto rows = [&](auto staged_tag) {
      constexpr bool RS = decltype(staged_tag)::value;
      constexpr bool R2S = RS && C::R2_STAGED;
  #pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int tr = tr_base + 8 * h;
        long long row = 0;
        const bool valid = map_row(tr, t0, t1, t2, row);
        // Rows past the end (tail tiles) read row 0 of the per-frame bias and of the __ldg residuals instead: their
        // results are never stored (the TMA store clips them, the fp32 stores check `valid`), and the column loop then
        // branches on launch-uniform flags only.  Staged residuals read the zeros TMA filled in for those rows.
        const long long orow = valid ? row : 0;
        const float* fb = has_fb ? p.fbias + static_cast<long long>(static_cast<int>(orow) / p.rows_per_frame) * p.ldfb +
                                       nbase + cq
                                 : nullptr;
        const bf16* r1p = has_r1 && !RS ? p.R1 + orow * p.ldr1 + obase + cq : nullptr;
        const bf16* r2p = has_r2 && !R2S ? p.R2 + orow * p.ldr2 + obase + cq : nullptr;
        float row_bias = 0.f;
        if (EPI == EPI_TRANS && has_bias && valid) row_bias = __ldg(p.bias + row);
        const uint32_t swz = SUBW == 32 ? static_cast<uint32_t>((tr >> 1) & 3) : 0u;  // 64B-swizzle XOR of the chunk
        const uint32_t srow = stg + static_cast<uint32_t>(tr * SUBW * 2 + cq * 2);  // staged row, this thread's column
  #pragma unroll
        for (int j = 0; j < OUT_COLS / 8; ++j) {
          const int oc = 8 * j + cq;
          // sub-tile and 16-byte chunk of column 8 j + cq fold to constants once j is unrolled (cq < 8, SUBW % 8 == 0);
          // a staged residual sits at the very address the output goes to
          const int sub = 8 * j / SUBW;
          const int chunk = (8 * j - sub * SUBW) >> 3;
          const uint32_t addr = srow + static_cast<uint32_t>(sub * C::SUB_BYTES) + ((static_cast<uint32_t>(chunk) ^ swz) << 4);
          float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if (EPI == EPI_TRANS) {
            v0 += row_bias;
            v1 += row_bias;
          } else if (has_bias) {
            v0 += __ldg(bcol + 8 * j);
            v1 += __ldg(bcol + 8 * j + 1);
          }
          if (has_fb) {
            v0 += __ldg(fb + 8 * j);
            v1 += __ldg(fb + 8 * j + 1);
          }
          if (GEGLU) {
            constexpr int JG = BN / 16;  // the gate of column c is column c + BN / 2 of the packed tile
            float g0 = acc[4 * (j + JG) + 2 * h], g1 = acc[4 * (j + JG) + 2 * h + 1];
            if (has_bias) {
              g0 += __ldg(bcol + BN / 2 + 8 * j);
              g1 += __ldg(bcol + BN / 2 + 8 * j + 1);
            }
            v0 *= gelu_erf_fast(g0);
            v1 *= gelu_erf_fast(g1);
          } else if (EPI == EPI_F32 && do_silu) {
            v0 = silu_f(v0);
            v1 = silu_f(v1);
          }
          if (RS || has_r1 || has_r2) {
            if (RS || has_r1) {
              const float2 x = unpack_bf16x2(RS ? lds32(addr) : __ldg(reinterpret_cast<const unsigned int*>(r1p + 8 * j)));
              v0 = fmaf(v0, s0, x.x * s1);
              v1 = fmaf(v1, s0, x.y * s1);
            } else {
              v0 *= s0;
              v1 *= s0;
            }
            if (has_r2) {
              const float2 x = unpack_bf16x2(R2S ? lds32(addr + C::TILE_OUT_BYTES)
                                                 : __ldg(reinterpret_cast<const unsigned int*>(r2p + 8 * j)));
              v0 = fmaf(x.x, s2, v0);
              v1 = fmaf(x.y, s2, v1);
            }
          } else {  // s0 = 1 scales exactly
            v0 *= s0;
            v1 *= s0;
          }
          if (EPI == EPI_TRANS) {
            if (valid) {
              float* dp = static_cast<float*>(p.D) + row;
              if (obase + oc < p.valid_cols) {
                float* o = dp + static_cast<long long>(obase + oc) * p.ldd;
                *o = p.accumulate ? *o + v0 : v0;
              }
              if (obase + oc + 1 < p.valid_cols) {
                float* o = dp + static_cast<long long>(obase + oc + 1) * p.ldd;
                *o = p.accumulate ? *o + v1 : v1;
              }
            }
          } else if (EPI == EPI_F32) {
            if (valid)
              *reinterpret_cast<float2*>(static_cast<float*>(p.D) + row * p.ldd + obase + oc) = make_float2(v0, v1);
          } else {
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_bf16x2(v0, v1)) : "memory");
          }
        }
      }
    };
    if (res_staged) rows(std::true_type{});
    else rows(std::false_type{});
    if (C::STAGED) {
      // the whole bf16 tile is in shared memory: hand it to the I/O thread, which writes it out by TMA
      fence_proxy_async_smem();
      asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
      if (store_leader) mbar_arrive(stg_full);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int pick_block_n(int N, int act) {
  static const int cands[] = {256, 160, 128, 64, 32, 16};
  for (int c : cands) {
    if (N % c != 0) continue;
    if (act == V3D_ACT_GEGLU && (c / 2) % 16 != 0) continue;
    return c;
  }
  return 0;
}

// bf16 output and the residuals staged in its place: one tensor map each, same box and swizzle (zeroed when unused)
struct OutMaps {
  CUtensorMap d, r1, r2;
};

static KvMaps g_kv_none;  // zero-initialised: n = 0
static const KvMaps* g_kv = &g_kv_none;  // set by v3d_gemm_bf16 around the one launch that scatters K|V

template <int BN, bool CONV, int EPI>
static int launch(const CUtensorMap& ma, const CUtensorMap& mb, const OutMaps& mo, const GemmEpi& epi,
                  cudaStream_t st) {
  using C = Cfg<BN, EPI>;
  static bool configured = false;
  auto kern = gemm_tc_kernel<BN, CONV, EPI>;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(smem=%d) failed: %s", C::SMEM_BYTES, cudaGetErrorString(e));
      return V3D_ERR_CUDA;
    }
    configured = true;
  }
  const int total = epi.num_m_tiles * epi.num_n_tiles;
  const int grid = total < num_sms() ? total : num_sms();
  kern<<<grid, kThreads, C::SMEM_BYTES, st>>>(ma, mb, mo.d, mo.r1, mo.r2, epi, *g_kv);
  V3D_CHECK_LAUNCH("gemm_tc_kernel");
  return V3D_OK;
}

template <int BN, bool CONV>
static int dispatch_epi(int epi_kind, const CUtensorMap& ma, const CUtensorMap& mb, const OutMaps& mo,
                        const GemmEpi& epi, cudaStream_t st) {
  switch (epi_kind) {
    case EPI_BF16: return launch<BN, CONV, EPI_BF16>(ma, mb, mo, epi, st);
    case EPI_BF16R2: return launch<BN, CONV, EPI_BF16R2>(ma, mb, mo, epi, st);
    case EPI_F32: return launch<BN, CONV, EPI_F32>(ma, mb, mo, epi, st);
    case EPI_GEGLU:
      if constexpr (!CONV && (BN / 2) % 16 == 0) return launch<BN, false, EPI_GEGLU>(ma, mb, mo, epi, st);
      break;
    case EPI_TRANS:  // at most 128 columns: the per-element transposed stores of wider tiles spill (host caps bn)
      if constexpr (!CONV && BN <= 128) return launch<BN, false, EPI_TRANS>(ma, mb, mo, epi, st);
      break;
  }
  set_error("unsupported epilogue %d for this mode/tile", epi_kind);
  return V3D_ERR_BAD_ARG;
}

template <bool CONV>
static int dispatch_bn(int bn, int epi_kind, const CUtensorMap& ma, const CUtensorMap& mb, const OutMaps& mo,
                       const GemmEpi& epi, cudaStream_t st) {
  switch (bn) {
    case 256: return dispatch_epi<256, CONV>(epi_kind, ma, mb, mo, epi, st);
    case 160: return dispatch_epi<160, CONV>(epi_kind, ma, mb, mo, epi, st);
    case 128: return dispatch_epi<128, CONV>(epi_kind, ma, mb, mo, epi, st);
    case 64: return dispatch_epi<64, CONV>(epi_kind, ma, mb, mo, epi, st);
    case 32: return dispatch_epi<32, CONV>(epi_kind, ma, mb, mo, epi, st);
    case 16: return dispatch_epi<16, CONV>(epi_kind, ma, mb, mo, epi, st);
    default: set_error("unsupported block_n %d", bn); return V3D_ERR_BAD_ARG;
  }
}

}  // namespace v3d

using namespace v3d;

/* diagnostics hook of an earlier GEMM (per-role clock64 timelines); this kernel records none: NULL is accepted,
 * anything else is refused. */
extern "C" int v3d_debug_set_trace(void* buf) {
  if (buf != nullptr) {
    set_error("v3d_debug_set_trace: the GEMM records no role timelines");
    return V3D_ERR_UNSUPPORTED;
  }
  return V3D_OK;
}

extern "C" int v3d_gemm_pick_block_n(int32_t N, int32_t act) { return pick_block_n(N, act); }

extern "C" int v3d_geglu_pack_rows(int32_t n_out, int32_t block_n, int32_t* perm) {
  if (n_out <= 0 || block_n <= 0 || (block_n & 1) || (2 * n_out) % block_n != 0 || perm == nullptr) {
    set_error("v3d_geglu_pack_rows: bad n_out=%d block_n=%d", n_out, block_n);
    return V3D_ERR_BAD_ARG;
  }
  const int half = block_n / 2;
  const int tiles = 2 * n_out / block_n;
  for (int t = 0; t < tiles; ++t) {
    for (int j = 0; j < half; ++j) {
      perm[t * block_n + j] = t * half + j;                 // value rows
      perm[t * block_n + half + j] = n_out + t * half + j;  // gate rows
    }
  }
  return V3D_OK;
}

extern "C" int v3d_gemm_args_size(void) { return static_cast<int>(sizeof(v3d_gemm_args)); }

extern "C" int v3d_gemm_bf16(const v3d_gemm_args* a, void* stream) {
  if (a == nullptr || a->A == nullptr || a->B == nullptr || a->D == nullptr) {
    set_error("v3d_gemm_bf16: null pointer");
    return V3D_ERR_BAD_ARG;
  }
  const bool conv = a->conv_w > 0;
  const int ntaps = conv ? 9 : (a->ntaps > 0 ? a->ntaps : 1);
  if (a->K <= 0 || a->K % BK != 0 || a->N <= 0 || a->N % 16 != 0) {
    set_error("v3d_gemm_bf16: K=%d must be a multiple of 64 and N=%d of 16", a->K, a->N);
    return V3D_ERR_BAD_ARG;
  }
  if (a->out_transposed && (conv || ntaps != 1 || !a->out_fp32 || a->batch > 1 || a->act == V3D_ACT_GEGLU || a->R1 || a->R2 || a->fbias)) {
    set_error("v3d_gemm_bf16: out_transposed needs a plain fp32 linear GEMM (no taps/conv/batch/residual/geglu)");
    return V3D_ERR_BAD_ARG;
  }
  if (a->act == V3D_ACT_GEGLU && (a->R1 || a->R2 || a->fbias)) {
    set_error("v3d_gemm_bf16: GEGLU takes no residual or per-frame bias");
    return V3D_ERR_BAD_ARG;
  }
  if (!conv && ntaps != 1 && ntaps != 3) {
    set_error("v3d_gemm_bf16: ntaps must be 1 or 3");
    return V3D_ERR_BAD_ARG;
  }
  if ((a->lda % 8) || (a->ldb % 8) || (a->ldd % 8) || (a->ldfb % 4)) {
    set_error("v3d_gemm_bf16: leading dimensions must be multiples of 8 elements");
    return V3D_ERR_BAD_ARG;
  }
  // the epilogue reads residuals two columns at a time (4 bytes); TMA staging needs 16-byte alignment on top
  auto res_ok = [](const void* r, int64_t ld) { return r == nullptr || (ld % 2 == 0 && (reinterpret_cast<uintptr_t>(r) & 3) == 0); };
  auto res_tma = [](const void* r, int64_t ld) { return r != nullptr && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(r) & 15) == 0; };
  if (!res_ok(a->R1, a->ldr1) || !res_ok(a->R2, a->ldr2)) {
    set_error("v3d_gemm_bf16: residuals need an even row pitch and a 4-byte aligned base (ldr1=%lld ldr2=%lld)",
              static_cast<long long>(a->ldr1), static_cast<long long>(a->ldr2));
    return V3D_ERR_BAD_ARG;
  }
  int bn = a->block_n > 0 ? a->block_n : pick_block_n(a->N, a->act);
  if (a->block_n <= 0 && a->act != V3D_ACT_GEGLU && bn >= 128) {
    // wave quantisation: among the wide tiles that divide N, take the one that fills the SMs best
    // (e.g. M = 2304, N = 1280: 90 tiles of 128x256 leave 58 SMs idle, 144 tiles of 128x160 do not)
    long long mt;
    if (a->conv_w > 0) {
      const int bw = a->conv_w < BM ? a->conv_w : BM;
      int bh = BM / bw;
      if (bh > a->conv_h) bh = a->conv_h;
      const int bnimg = BM / (bw * (bh > 0 ? bh : 1));
      mt = static_cast<long long>(a->conv_w / bw) * (a->conv_h / (bh > 0 ? bh : 1)) * ((a->conv_n + bnimg - 1) / bnimg);
    } else {
      mt = static_cast<long long>(a->batch > 0 ? a->batch : 1) * ((a->rows_per_batch + BM - 1) / BM);
    }
    static const int cands[] = {256, 160, 128};
    static const double mma_eff[] = {1.0, 0.97, 0.80};  // 128-wide tiles are shared-memory-bandwidth bound
    double best = -1.0;
    const int sms = num_sms();
    for (int i = 0; i < 3; ++i) {
      if (a->N % cands[i] != 0) continue;
      const long long tiles = mt * (a->N / cands[i]);
      const long long waves = (tiles + sms - 1) / sms;
      const double score = mma_eff[i] * static_cast<double>(tiles) / static_cast<double>(waves * sms);
      if (score > best + 1e-9) {
        best = score;
        bn = cands[i];
      }
    }
  }
  if (a->out_transposed && a->block_n <= 0 && bn > 128) {  // the transposed fp32 epilogue exists up to 128 columns
    for (int c : {128, 64, 32, 16}) {
      if (a->N % c == 0) {
        bn = c;
        break;
      }
    }
  }
  if (bn == 0 || a->N % bn != 0 || (a->act == V3D_ACT_GEGLU && (bn / 2) % 16 != 0)) {
    set_error("v3d_gemm_bf16: no valid N tile for N=%d act=%d block_n=%d", a->N, a->act, a->block_n);
    return V3D_ERR_BAD_ARG;
  }

  GemmEpi e;
  memset(&e, 0, sizeof(e));
  e.D = a->D;
  e.bias = a->bias;
  e.fbias = a->fbias;
  e.R1 = static_cast<const bf16*>(a->R1);
  e.R2 = static_cast<const bf16*>(a->R2);
  e.ldd = a->ldd;
  e.ldr1 = a->ldr1;
  e.ldr2 = a->ldr2;
  e.ldfb = a->ldfb > 0 ? a->ldfb : a->N;
  e.N = a->N;
  e.kpt = a->K / BK;
  e.ntaps = ntaps;
  e.tap_shift = a->tap_shift;
  e.tap0 = a->a_row0 - (ntaps >> 1) * a->tap_shift;
  e.rows_per_frame = a->rows_per_frame > 0 ? a->rows_per_frame : 1;
  e.act = a->act;
  e.out_fp32 = a->out_fp32;
  e.transposed = a->out_transposed;
  e.valid_cols = a->valid_cols > 0 ? a->valid_cols : a->N;
  e.accumulate = a->accumulate;
  e.s0 = a->s0;
  e.s1 = a->s1;
  e.s2 = a->s2;
  e.num_n_tiles = a->N / bn;

  CUtensorMap ma, mb;
  int rc;
  int b_batch = 1;
  if (conv) {
    const int W = a->conv_w, H = a->conv_h, NI = a->conv_n;
    if (H <= 0 || NI <= 0) {
      set_error("v3d_gemm_bf16: bad conv geometry");
      return V3D_ERR_BAD_ARG;
    }
    const int bw = W < BM ? W : BM;
    if (BM % bw != 0 || W % bw != 0) {
      set_error("conv3x3: width %d does not tile into 128-pixel boxes", W);
      return V3D_ERR_UNSUPPORTED;
    }
    int bh = BM / bw;
    if (bh > H) bh = H;
    if (H % bh != 0 || (BM / bw) % bh != 0) {
      set_error("conv3x3: height %d does not tile into 128-pixel boxes (bw=%d)", H, bw);
      return V3D_ERR_UNSUPPORTED;
    }
    const int bnimg = BM / (bw * bh);
    if ((bw & (bw - 1)) != 0 || (bh & (bh - 1)) != 0) {
      set_error("conv3x3: tile box %dx%d is not a power of two", bw, bh);
      return V3D_ERR_UNSUPPORTED;
    }
    e.cn = NI; e.ch = H; e.cw = W; e.bw = bw; e.bh = bh; e.bn = bnimg;
    e.bw_shift = __builtin_ctz(bw);
    e.bh_shift = __builtin_ctz(bh);
    e.tiles_w = W / bw;
    e.tiles_h = H / bh;
    {
      const bool p2 = (e.tiles_w & (e.tiles_w - 1)) == 0 && (e.tiles_h & (e.tiles_h - 1)) == 0;
      e.tw_shift = p2 ? __builtin_ctz(e.tiles_w) : -1;
      e.th_shift = p2 ? __builtin_ctz(e.tiles_h) : -1;
    }
    e.num_m_tiles = e.tiles_w * e.tiles_h * ((NI + bnimg - 1) / bnimg);
    e.batch = 1; e.rows_per_batch = NI * H * W; e.tiles_per_batch = 1;
    const uint64_t dims[4] = {(uint64_t)a->K, (uint64_t)W, (uint64_t)H, (uint64_t)NI};
    const uint64_t str[3] = {(uint64_t)a->lda * 2, (uint64_t)a->lda * 2 * W, (uint64_t)a->lda * 2 * W * H};
    const uint32_t box[4] = {BK, (uint32_t)bw, (uint32_t)bh, (uint32_t)bnimg};
    rc = make_tmap_bf16(&ma, a->A, 4, dims, str, box);
    if (rc) return rc;
  } else {
    if (a->batch <= 0 || a->rows_per_batch <= 0) {
      set_error("v3d_gemm_bf16: bad batch/rows");
      return V3D_ERR_BAD_ARG;
    }
    e.batch = a->batch;
    e.rows_per_batch = a->rows_per_batch;
    e.tiles_per_batch = (a->rows_per_batch + BM - 1) / BM;
    e.num_m_tiles = e.batch * e.tiles_per_batch;
    const uint64_t abs_ = a->batch > 1 ? (uint64_t)a->a_batch_stride
                                       : (uint64_t)(a->a_rows > 0 ? a->a_rows : a->rows_per_batch) * a->lda;
    if (abs_ % 8 != 0) {
      set_error("v3d_gemm_bf16: a_batch_stride must be a multiple of 8");
      return V3D_ERR_BAD_ARG;
    }
    // halo'd operand (frame-sharded temporal convs): the tensor map spans a_rows >= rows_per_batch rows per batch
    // item and output row r reads A rows a_row0 + r (+ tap shifts); rows outside [0, a_rows) are zero-filled
    if (a->a_rows < 0 || a->a_row0 < 0 || (a->a_rows > 0 && a->a_rows < a->a_row0 + a->rows_per_batch)) {
      set_error("v3d_gemm_bf16: bad halo geometry a_rows=%d a_row0=%d rows_per_batch=%d", a->a_rows, a->a_row0,
                a->rows_per_batch);
      return V3D_ERR_BAD_ARG;
    }
    const uint64_t a_rows = a->a_rows > 0 ? (uint64_t)a->a_rows : (uint64_t)a->rows_per_batch + (uint64_t)a->a_row0;
    const uint64_t dims[3] = {(uint64_t)a->K, a_rows, (uint64_t)a->batch};
    const uint64_t str[2] = {(uint64_t)a->lda * 2, abs_ * 2};
    const uint32_t box[3] = {BK, BM, 1};
    rc = make_tmap_bf16(&ma, a->A, 3, dims, str, box);
    if (rc) return rc;
    if (a->b_batch_stride != 0) {
      b_batch = a->batch;
      e.b_batched = 1;
    }
  }
  {
    const uint64_t ktot = (uint64_t)ntaps * a->K;
    const uint64_t bbs = b_batch > 1 ? (uint64_t)a->b_batch_stride : (uint64_t)a->N * a->ldb;
    const uint64_t dims[3] = {ktot, (uint64_t)a->N, (uint64_t)b_batch};
    const uint64_t str[2] = {(uint64_t)a->ldb * 2, bbs * 2};
    const uint32_t box[3] = {BK, (uint32_t)bn, 1};
    rc = make_tmap_bf16(&mb, a->B, 3, dims, str, box);
    if (rc) return rc;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int epi_kind = EPI_BF16;
  if (a->out_transposed) epi_kind = EPI_TRANS;
  else if (a->out_fp32) epi_kind = EPI_F32;
  else if (a->act == V3D_ACT_GEGLU) epi_kind = EPI_GEGLU;
  if ((a->act == V3D_ACT_GEGLU && epi_kind != EPI_GEGLU) || (a->act == V3D_ACT_SILU && epi_kind != EPI_F32)) {
    set_error("v3d_gemm_bf16: act=%d is not available with this output mode", a->act);
    return V3D_ERR_UNSUPPORTED;
  }
  OutMaps mo;
  memset(&mo, 0, sizeof(mo));
  if (e.R2 != nullptr && e.R1 == nullptr) {  // a lone residual always travels as R1
    e.R1 = e.R2; e.ldr1 = e.ldr2; e.s1 = e.s2;
    e.R2 = nullptr;
  }
  if (epi_kind == EPI_BF16 && e.R2 != nullptr) epi_kind = EPI_BF16R2;
  if (epi_kind == EPI_BF16 || epi_kind == EPI_BF16R2 || epi_kind == EPI_GEGLU) {
    const uint64_t out_cols = static_cast<uint64_t>(e.num_n_tiles) * (epi_kind == EPI_GEGLU ? bn / 2 : bn);
    const uint32_t ocols_tile = epi_kind == EPI_GEGLU ? bn / 2 : bn;
    const uint32_t subw = ocols_tile % 32 == 0 ? 32 : 16;  // must match SUBW in the kernel
    const int swz = subw == 32 ? 64 : 0;
    // the output's tile boxes over a matrix of pitch ld: the output itself, and the residuals, whose rows are the
    // output rows in every mode (a temporal GEMM's residual is not tap-shifted)
    auto out_map = [&](CUtensorMap* m, const void* base, long long ld) {
      if (conv) {
        const uint64_t dims[4] = {out_cols, (uint64_t)e.cw, (uint64_t)e.ch, (uint64_t)e.cn};
        const uint64_t str[3] = {(uint64_t)ld * 2, (uint64_t)ld * 2 * e.cw, (uint64_t)ld * 2 * e.cw * e.ch};
        const uint32_t box[4] = {subw, (uint32_t)e.bw, (uint32_t)e.bh, (uint32_t)e.bn};
        return make_tmap_bf16(m, base, 4, dims, str, box, swz);
      }
      const uint64_t dims[3] = {out_cols, (uint64_t)e.rows_per_batch, (uint64_t)e.batch};
      const uint64_t str[2] = {(uint64_t)ld * 2, (uint64_t)ld * 2 * e.rows_per_batch};
      const uint32_t box[3] = {subw, BM, 1};
      return make_tmap_bf16(m, base, 3, dims, str, box, swz);
    };
    rc = out_map(&mo.d, a->D, a->ldd);
    if (rc) return rc;
    // residuals are staged only if TMA can address all of them (16-byte aligned bases and pitches); otherwise the
    // epilogue reads them with __ldg
    if (res_tma(e.R1, e.ldr1) && (e.R2 == nullptr || res_tma(e.R2, e.ldr2))) {
      e.res_tma = 1;
      rc = out_map(&mo.r1, e.R1, e.ldr1);
      if (rc) return rc;
      if (e.R2 != nullptr) {
        rc = out_map(&mo.r2, e.R2, e.ldr2);
        if (rc) return rc;
      }
    }
  }
  // fused GEMM -> all-gather (K|V scatter into peer memory): plain linear bf16-output launches only
  KvMaps kvm;
  memset(&kvm, 0, sizeof(kvm));
  if (a->kv_n > 0) {
    if (conv || ntaps != 1 || epi_kind != EPI_BF16 || a->batch > 1 || a->kv_n > 8 || a->kv_col0 <= 0 ||
        a->kv_col0 % 32 != 0 || a->kv_col0 >= a->N || a->kv_ld < a->N - a->kv_col0 || a->kv_ld % 8 != 0 || bn % 32 != 0) {
      set_error("v3d_gemm_bf16: K|V scatter needs a plain linear bf16 GEMM without a second residual (kv_col0=%d kv_n=%d "
                "N=%d block_n=%d epilogue=%d)", a->kv_col0, a->kv_n, a->N, bn, epi_kind);
      return V3D_ERR_BAD_ARG;
    }
    kvm.n = a->kv_n;
    kvm.col0 = a->kv_col0;
    const uint64_t dims[3] = {(uint64_t)(a->N - a->kv_col0), (uint64_t)e.rows_per_batch, 1};
    const uint64_t str[2] = {(uint64_t)a->kv_ld * 2, (uint64_t)a->kv_ld * 2 * e.rows_per_batch};
    const uint32_t box[3] = {32, BM, 1};
    for (int i = 0; i < a->kv_n; ++i) {
      if (a->kv_dst[i] == nullptr) {
        set_error("v3d_gemm_bf16: kv_dst[%d] is null", i);
        return V3D_ERR_BAD_ARG;
      }
      rc = make_tmap_bf16(&kvm.m[i], a->kv_dst[i], 3, dims, str, box, 64);
      if (rc) return rc;
    }
    g_kv = &kvm;
  }
  rc = conv ? dispatch_bn<true>(bn, epi_kind, ma, mb, mo, e, st) : dispatch_bn<false>(bn, epi_kind, ma, mb, mo, e, st);
  g_kv = &g_kv_none;
  return rc;
}
