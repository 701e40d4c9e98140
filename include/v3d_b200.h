/*
 * v3d_b200 — C ABI of the H100 (sm_90a) kernels behind V3D's denoising hot path.
 *
 * The reference (heheyas/V3D) has no FFI of its own: every GPU op on the path is a PyTorch library
 * call.  Each entry point below therefore names the reference call site(s) it replaces
 * (file:line under the reference tree).  Conventions, identical for every function:
 *   - plain pointers to DEVICE memory + sizes; no allocation inside; caller owns all buffers;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - activations are bf16 NHWC / token-major ([rows, channels], channels contiguous) unless said
 *     otherwise; norm statistics, biases, sampler state are fp32;
 *   - return value 0 = ok; non-zero = error code (V3D_ERR_*), message via v3d_last_error().
 *   - launches are asynchronous on `stream`; nothing here synchronises the device.
 */
#ifndef V3D_B200_H
#define V3D_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define V3D_ABI_VERSION 1

#define V3D_ERR_OK 0
#define V3D_ERR_BAD_ARG 1
#define V3D_ERR_CUDA 2
#define V3D_ERR_NO_DRIVER 3
#define V3D_ERR_UNSUPPORTED 4

#define V3D_ACT_NONE 0
#define V3D_ACT_SILU 1
#define V3D_ACT_GEGLU 2 /* out[j] = (v[j]) * gelu_erf(g[j]); weight rows packed per N-tile, see v3d_geglu_pack_rows */

int v3d_abi_version(void);
const char* v3d_last_error(void);
/* number of kernels launched through this library since load (bench.py's gpu_launches) */
int64_t v3d_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Tensor-core GEMM family (wgmma, register accumulators, TMA-staged operands).
 *
 *   D[row, n] = s0 * act( sum_k A[row, k] * B[n, k] + bias[n] + fbias[row / rows_per_frame, n] )
 *               + s1 * R1[row, n] + s2 * R2[row, n]
 *
 * One kernel, three operand-gather modes:
 *   linear   (conv_w == 0, ntaps == 1): A is [batch][rows_per_batch][K], row stride lda.
 *            replaces nn.Linear / 1x1 Conv2d: sgm/modules/attention.py:95,277-283,680,704;
 *            sgm/modules/diffusionmodules/openaimodel.py:324; model.py:167-178 (AttnBlock q,k,v,proj).
 *   temporal (conv_w == 0, ntaps == 3): K-loop runs over 3 taps; tap t reads rows shifted by
 *            (t-1)*tap_shift inside the batch item, zero outside -> Conv3d k=(3,1,1) pad (1,0,0) on a
 *            frame-major [b][t*hw][C] tensor.  replaces sgm/modules/diffusionmodules/video_model.py:42-55
 *            (time_stack ResBlock convs) and sgm/modules/autoencoding/temporal_ae.py:31-44,94-99.
 *   conv3x3  (conv_w > 0): A is an NHWC image batch [conv_n][conv_h][conv_w][K] (pixel stride lda); the
 *            K-loop runs over the 9 taps with implicit zero padding (TMA out-of-bounds fill).
 *            replaces nn.Conv2d 3x3 s1 p1: openaimodel.py:145-147,267-315; video_model.py:189,439;
 *            model.py:65-66,111-120,651-653.
 * B is always [N][ntaps*K] (K-major, tap-major then channel), optionally batched.
 * All of K, lda, ldb, ldd, ldr* are in elements; K % 64 == 0; N % 16 == 0; lda, ldb, ldd % 8 == 0.
 * A residual needs an even ldr* and a 4-byte aligned base.  With a 16-byte aligned base and ldr* % 8 == 0 (the
 * usual case) the bf16-output epilogues load it into shared memory by TMA during the main loop; otherwise the
 * epilogue reads it from global memory.  Both give the same bits.
 * ------------------------------------------------------------------------------------------ */
typedef struct v3d_gemm_args {
  const void* A;      /* bf16 */
  const void* B;      /* bf16 [b_batch][N][ntaps*K] */
  void* D;            /* bf16, or fp32 when out_fp32 */
  const float* bias;  /* [N] or NULL */
  const float* fbias; /* [nframes][N] or NULL: per-frame (per-sample) additive row vector */
  const void* R1;     /* bf16 [rows][ldr1] or NULL */
  const void* R2;     /* bf16 [rows][ldr2] or NULL */
  int64_t lda, ldb, ldd, ldr1, ldr2;
  int64_t ldfb; /* row stride of fbias in floats; 0 -> N */
  int64_t a_batch_stride, b_batch_stride; /* elements; b_batch_stride == 0 -> B shared by all batch items */
  int32_t batch, rows_per_batch;
  int32_t N, K;
  int32_t ntaps, tap_shift;
  int32_t rows_per_frame; /* rows sharing one fbias vector (>=1) */
  int32_t act;            /* V3D_ACT_* */
  int32_t out_fp32;
  int32_t conv_n, conv_h, conv_w; /* conv3x3 mode when conv_w > 0 (then batch/rows_per_batch ignored) */
  int32_t block_n;                /* 0 = auto; else force the N tile (16,32,64,128,160,256) */
  /* small-M mode (the M<=64 embedding linears run as W[N_w,K] x X[64,K]^T): D is fp32 [valid_cols][ldd] written
   * transposed (D[col][row] = acc + bias[row]), optionally accumulated into; columns >= valid_cols are dropped */
  int32_t out_transposed, valid_cols, accumulate;
  float s0, s1, s2;
  /* halo'd A operand (linear / temporal modes; both 0 = none): every batch item of A holds a_rows >= a_row0 +
   * rows_per_batch rows and output row r reads A row a_row0 + r (+ the tap shifts); rows outside [0, a_rows) read as
   * zero.  Frame-sharded temporal convs pass a buffer with one halo frame on each side (a_row0 = tap_shift,
   * a_rows = rows_per_batch + 2 * tap_shift): the neighbours' boundary frames of video_model.py:42-55 /
   * temporal_ae.py:94-99 when the T view-frames are split across GPUs. */
  int32_t a_rows, a_row0;
  /* fused GEMM -> all-gather over peer memory (plain linear GEMMs with bf16 output; kv_n = 0: off).  Output columns
   * >= kv_col0 are ALSO stored - by the same epilogue, with the same TMA sub-tile stores - into kv_n destination matrices
   * kv_dst[i] (row stride kv_ld elements, column c - kv_col0, row = the output row), which may be IPC-mapped memory of
   * other GPUs (v3d_peer_import): the frame-sharded temporal attention's K|V all-gather (video_attention.py:114-125
   * around attention.py:337-341) leaves the projection GEMM tile by tile over NVLink instead of through a packing copy
   * and a separate collective.  kv_col0 must be a multiple of 32. */
  int32_t kv_col0, kv_n;
  int64_t kv_ld;
  void* kv_dst[8];
} v3d_gemm_args;

int v3d_gemm_bf16(const v3d_gemm_args* args, void* stream);
/* sizeof(v3d_gemm_args) as this library was compiled: bindings check their mirror of the struct against it. */
int v3d_gemm_args_size(void);

/* Permutation used to pack GEGLU projection rows so that each N-tile of width block_n holds
 * block_n/2 "value" rows followed by the matching block_n/2 "gate" rows
 * (reference split: attention.py:97-99, value = first half, gate = second half).
 * perm[i] = source row of packed row i; n_out = inner dim (proj has 2*n_out rows). Host function. */
int v3d_geglu_pack_rows(int32_t n_out, int32_t block_n, int32_t* perm);
/* N-tile width the GEMM will choose for a given N (so packers and callers agree). Host function. */
int v3d_gemm_pick_block_n(int32_t N, int32_t act);
/* diagnostics only: device buffer (>= 3072 int64) that CTA 0 of subsequent v3d_gemm_bf16 launches fills with per-role
 * clock64() timelines; NULL disables. */
int v3d_debug_set_trace(void* buf);

/* ------------------------------------------------------------------------------------------
 * Normalisation (norm.cu). GroupNorm is split into a statistics pass and an apply(+SiLU) pass; both
 * work on NHWC bf16 with fp32/fp64 statistics, like GroupNorm32 (diffusionmodules/util.py:274-276).
 * ------------------------------------------------------------------------------------------ */
/* stats: double [nsamples][groups][2] = {sum, sumsq} over rows_per_sample x (C/groups). rows_per_sample is
 * H*W for 2-D norms (util.py:259-276; attention.py:130-133; model.py:52-55) and T*H*W for the 3-D
 * time_stack ResBlock norms (openaimodel.py:267-271 with dims=3). The kernel accumulates with atomics: stats is
 * cleared first unless pre_zeroed != 0 (callers that carve many stats slices out of one zeroed pool). */
int v3d_groupnorm_stats(const void* x, void* stats, int64_t rows_per_sample, int32_t nsamples, int32_t C,
                        int32_t ldx, int32_t groups, int32_t pre_zeroed, void* stream);
/* y (dense, ld = C) = act(GN(x)); silu != 0 fuses the nn.SiLU / nonlinearity that always follows
 * (openaimodel.py:267-271,300-303; model.py:131-143). */
int v3d_groupnorm_apply(const void* x, void* y, const void* stats, const void* gamma, const void* beta,
                        int64_t rows_per_sample, int32_t nsamples, int32_t C, int32_t ldx, int32_t groups,
                        float eps, int32_t silu, void* stream);
/* The same normalisation in ONE launch (statistics -> grid-wide barrier -> apply): what the unsharded path calls;
 * the pair above remains for the frame-sharded path, where the statistics are all-reduced between the two passes.
 * Deterministic (per-CTA fp32 partials folded by warp-shuffle trees, summed in fp64 in a fixed order; no atomics on
 * data).  `workspace`: >= v3d_groupnorm_workspace_bytes() bytes of device memory, zeroed once by the caller and then
 * passed unchanged to every call issued on the same stream (it holds the barrier state and the partials). */
int64_t v3d_groupnorm_workspace_bytes(void);
int v3d_groupnorm(const void* x, void* y, const void* gamma, const void* beta, int64_t rows_per_sample,
                  int32_t nsamples, int32_t C, int32_t ldx, int32_t groups, float eps, int32_t silu,
                  void* workspace, int64_t workspace_bytes, void* stream);
/* Deterministic GroupNorm (opt-in): statistics that depend on the shape and the data only, never on the launch grid,
 * nsamples or a sharded plan.  A sample's rows_per_sample = frames x hw rows are cut into blocks of min(256, hw) rows
 * that never straddle a frame (the last block of a frame may be short); each (block, group) gets one fp32
 * (sum, sumsq) pair from a fixed in-CTA tree; the pairs are folded in fp64 in block order (lane l of one warp adds
 * blocks l, l + 32, ..., then an xor-shuffle tree).  The same shape and data give the same bits on the same GPU model
 * and library build.  hw = H*W for 2-D norms and for the 3-D time_stack norms alike.
 *   v3d_groupnorm_det_blocks            blocks per sample (-1 if hw does not divide rows_per_sample); host function
 *   v3d_groupnorm_partials              the block partials: float2 [nsamples][ldp][groups], ldp >= blocks per sample
 *   v3d_groupnorm_fold_apply            fold the nblocks partials of each sample ([nsamples][nblocks][groups]) over
 *                                       count_rows x C/groups elements, then y (dense, ld = C) = act(GN(x)); a frame-
 *                                       sharded caller passes the whole video's partials and count_rows
 *   v3d_groupnorm_det                   both in one launch (grid barrier), bit-identical to the pair; workspace >=
 *                                       v3d_groupnorm_det_workspace_bytes(...) bytes, zeroed once by the caller and
 *                                       passed unchanged to every call on the same stream */
int64_t v3d_groupnorm_det_blocks(int64_t rows_per_sample, int64_t hw);
int64_t v3d_groupnorm_det_workspace_bytes(int64_t rows_per_sample, int64_t hw, int32_t nsamples, int32_t groups);
int v3d_groupnorm_partials(const void* x, void* partials, int64_t rows_per_sample, int64_t hw, int32_t nsamples,
                           int32_t C, int32_t ldx, int32_t groups, int64_t ldp, void* stream);
int v3d_groupnorm_fold_apply(const void* x, void* y, const void* partials, const void* gamma, const void* beta,
                             int64_t rows_per_sample, int32_t nsamples, int32_t C, int32_t ldx, int32_t groups,
                             int64_t nblocks, int64_t count_rows, float eps, int32_t silu, void* stream);
int v3d_groupnorm_det(const void* x, void* y, const void* gamma, const void* beta, int64_t rows_per_sample, int64_t hw,
                      int32_t nsamples, int32_t C, int32_t ldx, int32_t groups, float eps, int32_t silu,
                      void* workspace, int64_t workspace_bytes, void* stream);
/* LayerNorm over C (attention.py:525-527; video_attention.py:51,79,93-94). Optional fused
 * z = x + add[row / rows_per_frame] (fp32 vectors; video_attention.py:286-287), z stored to ysum. */
int v3d_layernorm(const void* x, const void* add, void* ysum, void* y, const void* gamma, const void* beta,
                  int64_t rows, int32_t C, int32_t rows_per_frame, float eps, void* stream);
/* in-place softmax(scale * x) over rows of n bf16 scores (decoder AttnBlock, model.py:190-192). */
int v3d_softmax_rows(void* x, int64_t rows, int32_t n, float scale, void* stream);
/* same, fp32 scores in, bf16 probabilities out (separate buffers). */
int v3d_softmax_rows_f32(const void* x, void* y, int64_t rows, int32_t n, float scale, void* stream);

/* ------------------------------------------------------------------------------------------
 * Attention (attention.cu), head dim 64. q/k/v are column slices of one packed projection output
 * (row stride ld_qkv elements); heads are 64-column groups.
 * ------------------------------------------------------------------------------------------ */
/* F.scaled_dot_product_attention / xformers FMHA, attention.py:337-341,432-444: per (sample, head)
 * softmax(q k^T scale) v over ntok tokens; token rows are sample-major. wgmma MMAs (S = QK^T and O = PV with
 * register accumulators), TMA-staged Q/K/V tiles, fp32 online softmax. */
int v3d_attention_spatial(const void* q, const void* k, const void* v, void* o, int64_t ld_qkv, int64_t ld_o,
                          int32_t nbatch, int32_t ntok, int32_t nheads, float scale, void* stream);
/* validation twin of v3d_attention_spatial on mma.sync (same contract); not used by the product path. */
int v3d_attention_spatial_mma(const void* q, const void* k, const void* v, void* o, int64_t ld_qkv, int64_t ld_o,
                              int32_t nbatch, int32_t ntok, int32_t nheads, float scale, void* stream);
/* the same attention across the T view-frames of each pixel (video_attention.py:114,125), reading the
 * frame-major token matrix in place: row(b,t,s) = (b*T + t)*S + s, 1 <= T <= 128.  T <= 32 runs one warp per
 * (pixel, head) sequence; 33..128 runs one CTA per sequence with the 16-query tiles split over its warps and a
 * single-pass softmax over the whole key row (same arithmetic).  T > 128 is V3D_ERR_BAD_ARG: it would need an online
 * softmax over key tiles. */
int v3d_attention_temporal(const void* q, const void* k, const void* v, void* o, int64_t ld_qkv, int64_t ld_o,
                           int32_t nb, int32_t T, int32_t S, int32_t nheads, float scale, void* stream);
/* frame-sharded form (SURVEY.md 8(e); the "temporal-attention KV all-gather" of BASELINE.json): q / o hold this rank's
 * Tq frames (row(b,t,s) = (b*Tq + t)*S + s); k / v point into the all-gathered K|V buffer (row stride ld_kv) where key
 * frame f of CFG half b, pixel s is row kv_row[f] + b*kv_bstride[f] + s (host int32[Tk] arrays, rank-major layout).
 * 1 <= Tq <= Tk <= 128; the kernel is chosen by Tk as v3d_attention_temporal chooses it by T, and gives the same bits as
 * the dense form on the same rows. */
int v3d_attention_temporal_kv(const void* q, const void* k, const void* v, void* o, int64_t ld_q, int64_t ld_kv,
                              int64_t ld_o, int32_t nb, int32_t Tq, int32_t Tk, int32_t S, int32_t nheads,
                              const int32_t* kv_row, const int32_t* kv_bstride, float scale, void* stream);
/* CrossAttention over a context of nk >= 1 tokens (attention.py:286-349; the spatial and temporal attn2 of a
 * multi-token context), on the wgmma kernel of v3d_attention_spatial: item b's nq query rows b*nq + i (row stride ld_q)
 * attend to its own key / value rows b*kv_bstride + j, j < nk (row stride ld_kv, kv_bstride >= nk; rows between key
 * sets are not read); output rows b*nq + i, row stride ld_o. */
int v3d_attention_cross(const void* q, const void* k, const void* v, void* o, int64_t ld_q, int64_t ld_kv,
                        int64_t ld_o, int32_t nbatch, int32_t nq, int32_t nk, int64_t kv_bstride, int32_t nheads,
                        float scale, void* stream);

/* ------------------------------------------------------------------------------------------
 * Data movement / small matrices (elementwise.cu)
 * ------------------------------------------------------------------------------------------ */
/* F.interpolate(scale_factor=2, mode="nearest") on NHWC bf16 (openaimodel.py:164; model.py:68). */
int v3d_upsample_nearest2x(const void* x, void* y, int32_t N, int32_t H, int32_t W, int32_t C, void* stream);
/* [rows][ncols] bf16 block copy between row-strided buffers (th.cat skip concat, video_model.py:483). */
int v3d_copy_channels(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, int64_t rows, int32_t ncols,
                      void* stream);
/* explicit im2row for the 3x3 convs the TMA gather does not cover (Cin % 64 != 0: video_model.py:189,
 * model.py:651; stride 2: openaimodel.py:202-209, model.py:82-90). y[n,oh,ow][tap*C + c], zero-padded to Kpad. */
int v3d_im2col3x3(const void* x, void* y, int32_t N, int32_t H, int32_t W, int32_t C, int32_t stride, int32_t pad,
                  int32_t Hout, int32_t Wout, int32_t Kpad, void* stream);
/* sgm boundary layout conversion: NCHW fp32 (wrappers.py:27; video_diffusion.py:184) <-> NHWC. */
int v3d_nchw_f32_to_nhwc_bf16(const void* x, void* y, int32_t N, int32_t C, int32_t H, int32_t W, float scale,
                              void* stream);
int v3d_nhwc_to_nchw_f32(const void* x, void* y, int32_t N, int32_t C, int32_t HW, int64_t ldx, int32_t src_fp32,
                         float scale, void* stream);
/* y[M,N] fp32 (+)= act_out(act_in(x[M,K] fp32) W[N,K]^T (bf16) + bias), M <= 64, row strides ldx/ldy
 * in floats (0 -> dense): time_embed/label_emb
 * (video_model.py:151-182,456-461), emb_layers (openaimodel.py:291-297), time_pos_embed
 * (video_attention.py:220-224,275), single-token cross-attention to_out(to_v(ctx)) (attention.py:277-283). */
int v3d_small_linear(const void* x, const void* W, const void* bias, void* y, int32_t M, int32_t K, int32_t N,
                     int32_t act_in, int32_t act_out, int32_t accumulate, int64_t ldx, int64_t ldy, void* stream);
/* operand prep for the tensor-core small-M path: y bf16 [64][K] = act_in(x fp32 [M][ldx]), rows >= M zero. */
int v3d_prep_small_x(const void* x, int64_t ldx, void* y, int32_t M, int32_t K, int32_t act_in, void* stream);
/* timestep_embedding (diffusionmodules/util.py:207-231): out[n][dim] = cos | sin, fp32. */
int v3d_timestep_embedding(const void* t, void* out, int32_t n, int32_t dim, float max_period, void* stream);
int v3d_add_rows(const void* a, const void* b, void* out, int32_t rows, int32_t cols, void* stream);
/* AE3DConv.time_mix_conv (temporal_ae.py:94-107): Conv3d(C,C,(3,1,1)) over frames, C <= 4; x NHWC fp32 (row
 * stride ldx), w [C][C][3] fp32, y NCHW fp32 [nb*T][C][HW]. */
int v3d_time_mix_conv(const void* x, int64_t ldx, const void* w, const void* bias, void* y, int32_t nb, int32_t T,
                      int64_t HW, int32_t C, void* stream);

/* ------------------------------------------------------------------------------------------
 * EDM sampler arithmetic, fp32 (sampler.cu)
 * ------------------------------------------------------------------------------------------ */
/* y = x * c_in(sigma), c_noise = 0.25 log sigma (denoiser.py:31-39; denoiser_scaling.py:51-59). */
int v3d_edm_scale_input(const void* x, const void* sigma, void* y, void* c_noise, int32_t nsamples,
                        int64_t per_sample, void* stream);
/* out = net * c_out + x * c_skip (denoiser.py:36-39). */
int v3d_edm_denoise_combine(const void* net, const void* x, const void* sigma, void* out, int32_t nsamples,
                            int64_t per_sample, void* stream);
/* LinearPredictionGuider.__call__ (guiders.py:78-86), batch order [uc; c]. */
int v3d_cfg_combine(const void* den, const void* scale, void* out, int32_t B, int32_t T, int64_t per_sample,
                    void* stream);
/* to_d + euler_step (sampling_utils.py:34-35; sampling.py:81-82,103-106); out may alias x. */
int v3d_euler_step(const void* x, const void* den, const void* sigma_hat, const void* sigma_next, void* out,
                   int32_t nsamples, int64_t per_sample, void* stream);
/* HeunEDMSampler.possible_correction_step (sampling.py:221-237): x + dt * (d + d_new) / 2 where sigma_next > 0,
 * else the Euler proposal; x_euler = euler step of x, den2 = denoised(x_euler, sigma_next). out may alias x. */
int v3d_heun_step(const void* x, const void* den, const void* x_euler, const void* den2, const void* sigma_hat,
                  const void* sigma_next, void* out, int32_t nsamples, int64_t per_sample, void* stream);
/* The ancestral, DPM++ and linear-multistep samplers (sampling.py:136-211,240-365; sampling_utils.py:7-43).  One pass
 * over the fp32 state per call; every sample shares the step's sigma, so the schedule-derived multipliers are host
 * scalars computed in fp32 like the reference's.  Each operation is rounded on its own, in the reference's order
 * (e.g. (noise * s_noise) * sigma_up), so the results are the reference's to the last bit.  The noise term is added
 * only where sigma_next > 0 (ancestral_step's torch.where); the caller still draws that step's noise, as the
 * reference does, so later draws stay in the reference's order. */
#define V3D_LMS_MAX_ORDER 8
/* EulerAncestralSampler step: d = (x - den)/sigma; x_euler = x + (sigma_down - sigma) d; out = sigma_next > 0 ?
 * x_euler + (noise * s_noise) * sigma_up : x_euler (sampling.py:144-156,240-247; sampling_utils.py:22-35).
 * out may alias x. */
int v3d_ancestral_euler_step(const void* x, const void* den, const void* noise, void* out, float sigma,
                             float sigma_down, float sigma_up, float sigma_next, float s_noise, int32_t nsamples,
                             int64_t per_sample, void* stream);
/* DPM++ 2S ancestral midpoint: out = m1 x - m2 den (sampling.py:257-279).  out may alias x. */
int v3d_dpmpp2s_stage(const void* x, const void* den, void* out, float m1, float m2, int32_t nsamples,
                      int64_t per_sample, void* stream);
/* DPM++ 2S ancestral combine: sigma_down > 0 ? m3 x - m4 den2 : the ancestral Euler step of (x, den), then the
 * ancestral noise term (sampling.py:265-287).  out may alias x. */
int v3d_dpmpp2s_step(const void* x, const void* den, const void* den2, const void* noise, void* out, float sigma,
                     float sigma_down, float sigma_up, float sigma_next, float s_noise, float m3, float m4,
                     int32_t nsamples, int64_t per_sample, void* stream);
/* DPM++ 2M: out = m1 x - m2 den, or with second_order != 0: m1 x - m2 (m3 den - m4 hist); then hist := den
 * (sampling.py:290-345).  out may alias x; hist aliases nothing. */
int v3d_dpmpp2m_step(const void* x, const void* den, void* hist, void* out, float m1, float m2, float m3, float m4,
                     int32_t second_order, int32_t nsamples, int64_t per_sample, void* stream);
/* LMS: ring[slots[0]] := d = (x - den)/sigma; out = x + sum_{j<order} coeffs[j] ring[slots[j]], summed left to right
 * (sampling.py:194-209).  ring: ring_slots x nsamples x per_sample floats; coeffs / slots are HOST arrays of `order`
 * entries; 1 <= order <= V3D_LMS_MAX_ORDER <= ring_slots.  out may alias x. */
int v3d_lms_step(const void* x, const void* den, void* ring, void* out, float sigma, const float* coeffs,
                 const int32_t* slots, int32_t order, int32_t ring_slots, int32_t nsamples, int64_t per_sample,
                 void* stream);
/* clamp((x+1)/2,0,1)*255 -> uint8 THWC from the decoder's NHWC output (scripts/pub/V3D_512.py:286-303). */
int v3d_decode_to_u8(const void* x, int64_t ldx, int32_t src_fp32, void* y, int64_t npix, void* stream);
/* same, from NCHW fp32 frames [T][3][HW] (decode_first_stage's return layout) to uint8 [T][HW][3]. */
int v3d_frames_nchw_to_u8(const void* x, void* y, int32_t T, int64_t HW, void* stream);

/* ------------------------------------------------------------------------------------------
 * PixelNeRF scene conditioning (pixelnerf.cu): the PixelNeRFEmbedder of sparse-view scene generation
 * (sgm/modules/encoders/pixelnerf.py, math_utils.py).  Three launches: rays, the fused per-sample render (the
 * feature MLP on wgmma, online softmax over the sample axis) and the per-ray decoder MLP.  MLP weights are bf16
 * row-major [out][in] with zero padding: w1 [128][64 * ceil(d_in / 64)], w2 [128][128], w3 [136][128] (129 / 131 real
 * rows); biases fp32, b3 [136].
 * ------------------------------------------------------------------------------------------ */
#define V3D_PNERF_STD 1        /* append the unbiased std over sources (zeros when S = 1) */
#define V3D_PNERF_POSENC 2     /* append the 39-value NeRF positional encoding of the world sample */
#define V3D_PNERF_NEAREST 4    /* grid_sample mode "nearest" (default "bilinear") */
#define V3D_PNERF_ZEROS 8      /* grid_sample padding "zeros" (default "border") */
#define V3D_PNERF_DISPARITY 16 /* disparity sampling: jitter holds z[ns], depth = 1 / (inv_near (1 - z) + inv_far z) */
/* cams [ncam][25] -> rays [ncam * rs^2][8] = (origin, direction, t_start, t_end); limits: 2 words of scratch. */
int v3d_pixelnerf_rays(const void* cams, int32_t ncam, int32_t render_size, float box_half, int32_t box, void* rays,
                       void* limits, void* stream);
/* rays + limits from v3d_pixelnerf_rays; jitter [ns][nrays] uniforms (box mode); src [B][S][C][H][W] fp32;
 * src_w2c [B][S][3][4]; src_k [B][S][4] = (fx, fy, cx, cy); feat out [nrays][128] fp32.  ns >= 2, d_in <= 192. */
int v3d_pixelnerf_render(const void* rays, const void* limits, const void* jitter, const void* src, const void* src_w2c,
                         const void* src_k, int64_t nrays, int64_t rays_per_batch, int32_t S, int32_t C, int32_t H,
                         int32_t W, int32_t ns, int32_t flags, float inv_near, float inv_far, const void* w1,
                         int32_t d_in, const void* b1, const void* w2, const void* b2, const void* w3, const void* b3,
                         void* feat, void* stream);
/* feat [nrays][128] -> rgb [nrays / hw][3][hw] (sigmoid) and feats [nrays / hw][128][hw], fp32. */
int v3d_pixelnerf_decode(const void* feat, int64_t nrays, int64_t hw, const void* w1, const void* b1, const void* w2,
                         const void* b2, const void* w3, const void* b3, void* rgb, void* feats, void* stream);

/* ------------------------------------------------------------------------------------------
 * One-sided exchanges over NVLink peer memory (peer.cu): the transport of the frame-sharded path - ONE image over
 * several GPUs of a box (BASELINE.json north_star; SURVEY.md 8(e)).  They replace, on the data path, the three
 * torch.distributed exchanges that the reference's single-GPU modules imply once the T frames are split over ranks:
 * the temporal-attention K|V all-gather (video_attention.py:114-125 around attention.py:337-341), the 1-frame halos
 * of the (3,1,1) temporal convolutions (video_model.py:42-55, temporal_ae.py:94-99) and the (sum, sumsq) all-reduce
 * of the 3-D GroupNorm (openaimodel.py:267-271 with dims=3).  Every rank owns an arena (v3d_peer_alloc) that the
 * other ranks map through a 64-byte IPC handle; kernels then store straight into the mapped arenas and raise /
 * wait on epoch-valued flag words, so a whole sharded forward is stream-ordered and CUDA-graph capturable.
 * ------------------------------------------------------------------------------------------ */
#define V3D_PEER_MAX_SEG 16
#define V3D_PEER_MAX_FLAG 16
#define V3D_PEER_MAX_RANKS 8
/* zeroed device memory that can be exported (plain cudaMalloc, not the framework's caching allocator) */
int v3d_peer_alloc(int64_t bytes, void** out);
int v3d_peer_free(void* p);
/* 64-byte handle of an arena (cudaIpcGetMemHandle) / mapping of another rank's arena (cudaIpcOpenMemHandle) */
int v3d_peer_export(const void* p, void* handle64);
int v3d_peer_import(const void* handle64, void** out);
int v3d_peer_close(void* p);
/* *epoch += 1 on the stream: once at the start of every sharded forward (flags carry the epoch) */
int v3d_peer_epoch_bump(void* epoch, void* stream);
/* copy nseg contiguous segments src[i] -> dst[i] (bytes[i], multiples of 16; dst may be mapped peer memory), then -
 * once all stores are fenced system-wide - store *epoch into the nflag flag words (usually in the receivers' arenas).
 * done_counter: one zeroed u32 of local scratch per stream. */
int v3d_peer_put(int32_t nseg, const void* const* src, void* const* dst, const int64_t* bytes, int32_t nflag,
                 void* const* flags, const void* epoch, void* done_counter, void* stream);
/* block the stream until every flag word >= *epoch (bounded: after 30 s the site id is recorded in *status and every later wait
 * of the transport returns at once) */
int v3d_peer_wait(int32_t nflag, const void* const* flags, const void* epoch, void* status, int32_t site,
                  void* stream);
/* stats[n] (fp64) := scale * sum over ranks, rank-ordered (bit-identical on every rank): slot_base[r] / flag_base[r]
 * = rank r's slot area [world][n] doubles / flag area [world] words of this exchange site. */
int v3d_peer_allreduce_f64(void* stats, int32_t n, double scale, int32_t world, int32_t rank,
                           void* const* slot_base, void* const* flag_base, const void* epoch, void* status,
                           int32_t site, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* V3D_B200_H */
