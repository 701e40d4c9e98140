// EDM sampler arithmetic (fp32, per-sample sigma broadcast) and the output wire format.
// These are the O(T*4*64*64) elementwise pieces between UNet evaluations: one kernel each instead of the
// reference's ~15 tiny ATen launches per step.
#include "common.cuh"
#include "host_util.cuh"
#include "v3d_b200.h"

namespace v3d {

static inline unsigned ew_blocks(long long n) {
  long long b = (n + 255) / 256;
  const long long cap = 16LL * num_sms();
  if (b > cap) b = cap;
  return static_cast<unsigned>(b < 1 ? 1 : b);
}

// y = x * c_in(sigma_n);  c_noise[n] = 0.25 ln sigma_n      (VScalingWithEDMcNoise)
__global__ void edm_scale_input_kernel(const float* __restrict__ x, const float* __restrict__ sigma,
                                       float* __restrict__ y, float* __restrict__ c_noise, int nsamples,
                                       long long per_sample) {
  const long long total = nsamples * per_sample;
  const long long i0 = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (c_noise != nullptr && i0 < nsamples) c_noise[i0] = 0.25f * logf(sigma[i0]);
  for (long long i = i0; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float s = sigma[i / per_sample];
    y[i] = x[i] * (1.0f / sqrtf(s * s + 1.0f));
  }
}

// out = net * c_out + x * c_skip
__global__ void edm_denoise_combine_kernel(const float* __restrict__ net, const float* __restrict__ x,
                                           const float* __restrict__ sigma, float* __restrict__ out,
                                           int nsamples, long long per_sample) {
  const long long total = nsamples * per_sample;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float s = sigma[i / per_sample];
    const float d = s * s + 1.0f;
    const float c_skip = 1.0f / d;
    const float c_out = -s / sqrtf(d);
    out[i] = net[i] * c_out + x[i] * c_skip;
  }
}

// out[b,t] = x_u[b,t] + scale[t] * (x_c[b,t] - x_u[b,t]); den = [uncond (B*T samples) ; cond (B*T samples)]
__global__ void cfg_combine_kernel(const float* __restrict__ den, const float* __restrict__ scale,
                                   float* __restrict__ out, int B, int T, long long per_sample) {
  const long long half = static_cast<long long>(B) * T * per_sample;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < half;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int t = static_cast<int>((i / per_sample) % T);
    const float xu = den[i], xc = den[half + i];
    out[i] = xu + scale[t] * (xc - xu);
  }
}

// d = (x - denoised) / sigma_hat; out = x + (sigma_next - sigma_hat) * d
__global__ void euler_step_kernel(const float* __restrict__ x, const float* __restrict__ den,
                                  const float* __restrict__ sigma_hat, const float* __restrict__ sigma_next,
                                  float* __restrict__ out, int nsamples, long long per_sample) {
  const long long total = nsamples * per_sample;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long n = i / per_sample;
    const float sh = sigma_hat[n];
    const float d = (x[i] - den[i]) / sh;
    out[i] = x[i] + (sigma_next[n] - sh) * d;
  }
}

// Heun correction: d = (x - den)/sigma_hat, d2 = (x_euler - den2)/sigma_next,
// out = sigma_next > 0 ? x + (sigma_next - sigma_hat) * (d + d2) / 2 : x_euler
__global__ void heun_step_kernel(const float* __restrict__ x, const float* __restrict__ den,
                                 const float* __restrict__ x_euler, const float* __restrict__ den2,
                                 const float* __restrict__ sigma_hat, const float* __restrict__ sigma_next,
                                 float* __restrict__ out, int nsamples, long long per_sample) {
  const long long total = nsamples * per_sample;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long n = i / per_sample;
    const float sh = sigma_hat[n], sn = sigma_next[n];
    const float xe = x_euler[i];
    float r = xe;
    if (sn > 0.0f) {
      const float d = (x[i] - den[i]) / sh;
      const float d2 = (xe - den2[i]) / sn;
      r = x[i] + ((d + d2) / 2.0f) * (sn - sh);
    }
    out[i] = r;
  }
}

// The ancestral / DPM++ / LMS steps below round every operation separately (__f*_rn: no FMA contraction), in the
// order of the reference's torch expressions, so that they reproduce its fp32 results bit for bit.

// x + (noise * s_noise) * sigma_up where sigma_next > 0, else x   (AncestralSampler.ancestral_step)
__device__ __forceinline__ float add_ancestral_noise(float x, const float* __restrict__ noise, long long i,
                                                     float s_noise, float sigma_up, float sigma_next) {
  return sigma_next > 0.0f ? __fadd_rn(x, __fmul_rn(__fmul_rn(noise[i], s_noise), sigma_up)) : x;
}

// d = (x - den) / sigma; x_euler = x + (sigma_down - sigma) * d; then the ancestral noise term
__global__ void ancestral_euler_step_kernel(const float* __restrict__ x, const float* __restrict__ den,
                                            const float* __restrict__ noise, float* __restrict__ out, float sigma,
                                            float sigma_down, float sigma_up, float sigma_next, float s_noise,
                                            long long total) {
  const float dt = __fsub_rn(sigma_down, sigma);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float xi = x[i];
    const float d = __fdiv_rn(__fsub_rn(xi, den[i]), sigma);
    out[i] = add_ancestral_noise(__fadd_rn(xi, __fmul_rn(dt, d)), noise, i, s_noise, sigma_up, sigma_next);
  }
}

// out = m1 * x - m2 * den   (DPM++ 2S midpoint, DPM++ 2M first-order step)
__global__ void dpm_first_order_kernel(const float* __restrict__ x, const float* __restrict__ den,
                                       float* __restrict__ out, float m1, float m2, long long total) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    out[i] = __fsub_rn(__fmul_rn(m1, x[i]), __fmul_rn(m2, den[i]));
}

// sigma_down > 0 ? m3 * x - m4 * den2 : x_euler(x, den); then the ancestral noise term
__global__ void dpmpp2s_step_kernel(const float* __restrict__ x, const float* __restrict__ den,
                                    const float* __restrict__ den2, const float* __restrict__ noise,
                                    float* __restrict__ out, float sigma, float sigma_down, float sigma_up,
                                    float sigma_next, float s_noise, float m3, float m4, long long total) {
  const float dt = __fsub_rn(sigma_down, sigma);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float xi = x[i];
    float r;
    if (sigma_down > 0.0f) {
      r = __fsub_rn(__fmul_rn(m3, xi), __fmul_rn(m4, den2[i]));
    } else {
      const float d = __fdiv_rn(__fsub_rn(xi, den[i]), sigma);
      r = __fadd_rn(xi, __fmul_rn(dt, d));
    }
    out[i] = add_ancestral_noise(r, noise, i, s_noise, sigma_up, sigma_next);
  }
}

// x_std = m1 x - m2 D; with history and sigma_next > 0: m1 x - m2 (m3 D - m4 D_old).  hist <- D afterwards.
__global__ void dpmpp2m_step_kernel(const float* __restrict__ x, const float* __restrict__ den, float* hist,
                                    float* out, float m1, float m2, float m3, float m4, int second_order,
                                    long long total) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float xi = x[i], di = den[i];
    float dd = di;
    if (second_order) dd = __fsub_rn(__fmul_rn(m3, di), __fmul_rn(m4, hist[i]));
    hist[i] = di;
    out[i] = __fsub_rn(__fmul_rn(m1, xi), __fmul_rn(m2, dd));
  }
}

struct LmsTerms {
  float c[V3D_LMS_MAX_ORDER];
  int slot[V3D_LMS_MAX_ORDER];
};

// ring[slot[0]] <- d = (x - den) / sigma;  out = x + (((c0 d_i + c1 d_{i-1}) + c2 d_{i-2}) + ...)
__global__ void lms_step_kernel(const float* x, const float* __restrict__ den, float* ring, float* out, float sigma,
                                LmsTerms terms, int order, long long total) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float xi = x[i];
    const float d = __fdiv_rn(__fsub_rn(xi, den[i]), sigma);
    ring[terms.slot[0] * total + i] = d;
    float acc = __fmul_rn(terms.c[0], d);
#pragma unroll
    for (int j = 1; j < V3D_LMS_MAX_ORDER; ++j)
      if (j < order) acc = __fadd_rn(acc, __fmul_rn(terms.c[j], ring[terms.slot[j] * total + i]));
    out[i] = __fadd_rn(xi, acc);
  }
}

// frames[p][c] = uint8(clamp((x[p][c] + 1) / 2, 0, 1) * 255)  (truncating cast, like numpy astype)
template <typename T>
__global__ void decode_to_u8_kernel(const T* __restrict__ x, long long ldx, uint8_t* __restrict__ y, long long npix) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < npix * 3;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / 3;
    const int c = static_cast<int>(i - p * 3);
    float v = (static_cast<float>(x[p * ldx + c]) + 1.0f) / 2.0f;
    v = fminf(fmaxf(v, 0.0f), 1.0f) * 255.0f;
    y[i] = static_cast<uint8_t>(v);
  }
}

// same wire format straight from the decoder's NCHW fp32 output: y[t][p][c] = u8(x[t][c][p])
__global__ void frames_nchw_to_u8_kernel(const float* __restrict__ x, uint8_t* __restrict__ y, int T, long long HW) {
  const long long total = static_cast<long long>(T) * HW * 3;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % 3);
    const long long p = (i / 3) % HW;
    const long long t = i / (3 * HW);
    float v = (x[(t * 3 + c) * HW + p] + 1.0f) / 2.0f;
    v = fminf(fmaxf(v, 0.0f), 1.0f) * 255.0f;
    y[i] = static_cast<uint8_t>(v);
  }
}

}  // namespace v3d

using namespace v3d;

extern "C" {

/* Denoiser.forward input side: network input = x * c_in, c_noise = 0.25 log sigma
 * (denoiser.py:31-39, denoiser_scaling.py:51-59). */
int v3d_edm_scale_input(const void* x, const void* sigma, void* y, void* c_noise, int32_t nsamples,
                        int64_t per_sample, void* stream) {
  if (!x || !sigma || !y || nsamples <= 0 || per_sample <= 0) {
    set_error("v3d_edm_scale_input: bad args");
    return V3D_ERR_BAD_ARG;
  }
  edm_scale_input_kernel<<<ew_blocks(nsamples * per_sample), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(x), static_cast<const float*>(sigma), static_cast<float*>(y),
      static_cast<float*>(c_noise), nsamples, per_sample);
  V3D_CHECK_LAUNCH("edm_scale_input_kernel");
  return V3D_OK;
}

/* Denoiser.forward output side: net * c_out + x * c_skip (denoiser.py:36-39). */
int v3d_edm_denoise_combine(const void* net, const void* x, const void* sigma, void* out, int32_t nsamples,
                            int64_t per_sample, void* stream) {
  if (!net || !x || !sigma || !out || nsamples <= 0 || per_sample <= 0) {
    set_error("v3d_edm_denoise_combine: bad args");
    return V3D_ERR_BAD_ARG;
  }
  edm_denoise_combine_kernel<<<ew_blocks(nsamples * per_sample), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(net), static_cast<const float*>(x), static_cast<const float*>(sigma),
      static_cast<float*>(out), nsamples, per_sample);
  V3D_CHECK_LAUNCH("edm_denoise_combine_kernel");
  return V3D_OK;
}

/* LinearPredictionGuider.__call__ (guiders.py:78-86): x_u + scale_t (x_c - x_u), [uc; c] batch order. */
int v3d_cfg_combine(const void* den, const void* scale, void* out, int32_t B, int32_t T, int64_t per_sample,
                    void* stream) {
  if (!den || !scale || !out || B <= 0 || T <= 0 || per_sample <= 0) {
    set_error("v3d_cfg_combine: bad args");
    return V3D_ERR_BAD_ARG;
  }
  cfg_combine_kernel<<<ew_blocks(static_cast<long long>(B) * T * per_sample), 256, 0,
                       static_cast<cudaStream_t>(stream)>>>(static_cast<const float*>(den),
                                                            static_cast<const float*>(scale),
                                                            static_cast<float*>(out), B, T, per_sample);
  V3D_CHECK_LAUNCH("cfg_combine_kernel");
  return V3D_OK;
}

/* to_d + euler_step (sampling_utils.py:34-35, sampling.py:81-82,103-106). out may alias x. */
int v3d_euler_step(const void* x, const void* den, const void* sigma_hat, const void* sigma_next, void* out,
                   int32_t nsamples, int64_t per_sample, void* stream) {
  if (!x || !den || !sigma_hat || !sigma_next || !out || nsamples <= 0 || per_sample <= 0) {
    set_error("v3d_euler_step: bad args");
    return V3D_ERR_BAD_ARG;
  }
  euler_step_kernel<<<ew_blocks(nsamples * per_sample), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(x), static_cast<const float*>(den), static_cast<const float*>(sigma_hat),
      static_cast<const float*>(sigma_next), static_cast<float*>(out), nsamples, per_sample);
  V3D_CHECK_LAUNCH("euler_step_kernel");
  return V3D_OK;
}

/* HeunEDMSampler.possible_correction_step (sampling.py:221-237): second-order correction from the Euler proposal
 * x_euler and its denoised estimate den2 at sigma_next; samples with sigma_next == 0 keep the Euler proposal.
 * out may alias x or x_euler. */
int v3d_heun_step(const void* x, const void* den, const void* x_euler, const void* den2, const void* sigma_hat,
                  const void* sigma_next, void* out, int32_t nsamples, int64_t per_sample, void* stream) {
  if (!x || !den || !x_euler || !den2 || !sigma_hat || !sigma_next || !out || nsamples <= 0 || per_sample <= 0) {
    set_error("v3d_heun_step: bad args");
    return V3D_ERR_BAD_ARG;
  }
  heun_step_kernel<<<ew_blocks(nsamples * per_sample), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(x), static_cast<const float*>(den), static_cast<const float*>(x_euler),
      static_cast<const float*>(den2), static_cast<const float*>(sigma_hat), static_cast<const float*>(sigma_next),
      static_cast<float*>(out), nsamples, per_sample);
  V3D_CHECK_LAUNCH("heun_step_kernel");
  return V3D_OK;
}

/* EulerAncestralSampler.sampler_step: AncestralSampler.ancestral_euler_step + ancestral_step (sampling.py:144-156,
 * 240-247) with sigma_down / sigma_up of get_ancestral_step (sampling_utils.py:22-31).  out may alias x. */
int v3d_ancestral_euler_step(const void* x, const void* den, const void* noise, void* out, float sigma,
                             float sigma_down, float sigma_up, float sigma_next, float s_noise, int32_t nsamples,
                             int64_t per_sample, void* stream) {
  if (!x || !den || !noise || !out || nsamples <= 0 || per_sample <= 0 || !(sigma > 0.0f)) {
    set_error("v3d_ancestral_euler_step: bad args");
    return V3D_ERR_BAD_ARG;
  }
  const long long total = nsamples * per_sample;
  ancestral_euler_step_kernel<<<ew_blocks(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(x), static_cast<const float*>(den), static_cast<const float*>(noise),
      static_cast<float*>(out), sigma, sigma_down, sigma_up, sigma_next, s_noise, total);
  V3D_CHECK_LAUNCH("ancestral_euler_step_kernel");
  return V3D_OK;
}

/* DPMPP2SAncestralSampler.sampler_step midpoint (sampling.py:257-279): x2 = m1 * x - m2 * den with
 * m1 = sigma(s) / sigma(t), m2 = expm1(-h / 2).  out may alias x. */
int v3d_dpmpp2s_stage(const void* x, const void* den, void* out, float m1, float m2, int32_t nsamples,
                      int64_t per_sample, void* stream) {
  if (!x || !den || !out || nsamples <= 0 || per_sample <= 0) {
    set_error("v3d_dpmpp2s_stage: bad args");
    return V3D_ERR_BAD_ARG;
  }
  const long long total = nsamples * per_sample;
  dpm_first_order_kernel<<<ew_blocks(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(x), static_cast<const float*>(den), static_cast<float*>(out), m1, m2, total);
  V3D_CHECK_LAUNCH("dpm_first_order_kernel");
  return V3D_OK;
}

/* DPMPP2SAncestralSampler.sampler_step final combine (sampling.py:265-287): sigma_down > 0 ? m3 * x - m4 * den2 :
 * the ancestral Euler step of (x, den), then ancestral_step's noise term; m3 = sigma(t_next) / sigma(t),
 * m4 = expm1(-h), den2 = denoised(x2, sigma(s)).  out may alias x. */
int v3d_dpmpp2s_step(const void* x, const void* den, const void* den2, const void* noise, void* out, float sigma,
                     float sigma_down, float sigma_up, float sigma_next, float s_noise, float m3, float m4,
                     int32_t nsamples, int64_t per_sample, void* stream) {
  if (!x || !den || !den2 || !noise || !out || nsamples <= 0 || per_sample <= 0 || !(sigma > 0.0f)) {
    set_error("v3d_dpmpp2s_step: bad args");
    return V3D_ERR_BAD_ARG;
  }
  const long long total = nsamples * per_sample;
  dpmpp2s_step_kernel<<<ew_blocks(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(x), static_cast<const float*>(den), static_cast<const float*>(den2),
      static_cast<const float*>(noise), static_cast<float*>(out), sigma, sigma_down, sigma_up, sigma_next, s_noise,
      m3, m4, total);
  V3D_CHECK_LAUNCH("dpmpp2s_step_kernel");
  return V3D_OK;
}

/* DPMPP2MSampler.sampler_step (sampling.py:290-345): m1 = sigma(t_next) / sigma(t), m2 = expm1(-h);
 * second_order != 0 (previous step exists and sigma_next > 0): m3 = 1 + 1/(2r), m4 = 1/(2r) with the previous
 * denoised estimate read from hist.  hist is overwritten with den (the next step's old_denoised).  out may alias x;
 * hist must not alias x, den or out. */
int v3d_dpmpp2m_step(const void* x, const void* den, void* hist, void* out, float m1, float m2, float m3, float m4,
                     int32_t second_order, int32_t nsamples, int64_t per_sample, void* stream) {
  if (!x || !den || !hist || !out || nsamples <= 0 || per_sample <= 0) {
    set_error("v3d_dpmpp2m_step: bad args");
    return V3D_ERR_BAD_ARG;
  }
  const long long total = nsamples * per_sample;
  dpmpp2m_step_kernel<<<ew_blocks(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(x), static_cast<const float*>(den), static_cast<float*>(hist),
      static_cast<float*>(out), m1, m2, m3, m4, second_order, total);
  V3D_CHECK_LAUNCH("dpmpp2m_step_kernel");
  return V3D_OK;
}

/* LinearMultistepSampler.__call__ loop body (sampling.py:194-209): ring holds `ring_slots` slopes of
 * nsamples * per_sample floats each; d = (x - den) / sigma is stored in slot slots[0], then
 * out = x + sum_j coeffs[j] * ring[slots[j]] for j < order (slots[j] = the slot of d_{i-j}; coeffs, slots: host
 * arrays of `order` entries, order <= V3D_LMS_MAX_ORDER).  out may alias x. */
int v3d_lms_step(const void* x, const void* den, void* ring, void* out, float sigma, const float* coeffs,
                 const int32_t* slots, int32_t order, int32_t ring_slots, int32_t nsamples, int64_t per_sample,
                 void* stream) {
  if (!x || !den || !ring || !out || !coeffs || !slots || nsamples <= 0 || per_sample <= 0 || !(sigma > 0.0f) ||
      order < 1 || order > V3D_LMS_MAX_ORDER || ring_slots < order) {
    set_error("v3d_lms_step: bad args (order must be 1..8 and fit the ring)");
    return V3D_ERR_BAD_ARG;
  }
  LmsTerms terms{};
  for (int j = 0; j < order; ++j) {
    if (slots[j] < 0 || slots[j] >= ring_slots) {
      set_error("v3d_lms_step: ring slot out of range");
      return V3D_ERR_BAD_ARG;
    }
    terms.c[j] = coeffs[j];
    terms.slot[j] = slots[j];
  }
  const long long total = nsamples * per_sample;
  lms_step_kernel<<<ew_blocks(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(x), static_cast<const float*>(den), static_cast<float*>(ring),
      static_cast<float*>(out), sigma, terms, order, total);
  V3D_CHECK_LAUNCH("lms_step_kernel");
  return V3D_OK;
}

/* Output wire format of sample_one (scripts/pub/V3D_512.py:286-303): clamp((x+1)/2,0,1)*255 -> uint8 THWC.
 * x is the decoder's NHWC output (row stride ldx, first 3 channels), fp32 or bf16. */
int v3d_decode_to_u8(const void* x, int64_t ldx, int32_t src_fp32, void* y, int64_t npix, void* stream) {
  if (!x || !y || npix <= 0 || ldx < 3) {
    set_error("v3d_decode_to_u8: bad args");
    return V3D_ERR_BAD_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (src_fp32)
    decode_to_u8_kernel<float><<<ew_blocks(npix * 3), 256, 0, st>>>(static_cast<const float*>(x), ldx,
                                                                    static_cast<uint8_t*>(y), npix);
  else
    decode_to_u8_kernel<bf16><<<ew_blocks(npix * 3), 256, 0, st>>>(static_cast<const bf16*>(x), ldx,
                                                                   static_cast<uint8_t*>(y), npix);
  V3D_CHECK_LAUNCH("decode_to_u8_kernel");
  return V3D_OK;
}

/* The same conversion from the decoder's NCHW fp32 frames [T][3][HW] -> uint8 [T][HW][3]
 * (rearrange "t c h w -> t h w c" + clamp + *255 + astype(uint8), scripts/pub/V3D_512.py:286-303). */
int v3d_frames_nchw_to_u8(const void* x, void* y, int32_t T, int64_t HW, void* stream) {
  if (!x || !y || T <= 0 || HW <= 0) {
    set_error("v3d_frames_nchw_to_u8: bad args");
    return V3D_ERR_BAD_ARG;
  }
  frames_nchw_to_u8_kernel<<<ew_blocks(static_cast<long long>(T) * HW * 3), 256, 0,
                             static_cast<cudaStream_t>(stream)>>>(static_cast<const float*>(x),
                                                                  static_cast<uint8_t*>(y), T, HW);
  V3D_CHECK_LAUNCH("frames_nchw_to_u8_kernel");
  return V3D_OK;
}

}  // extern "C"
