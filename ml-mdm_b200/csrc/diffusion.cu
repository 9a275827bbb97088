// Diffusion algebra of the path as single-pass kernels over NCHW fp32 images with PER-SAMPLE
// gamma scalars (the reference materialises gamma as full (B,C,H,W) maps, samplers.py:196-199).
//   q-sample            samplers.py:244-246 (+ NestedSampler.get_xt :625-637)
//   targets / loss      samplers.py:266-279,347-390 ; diffusion.py:123-136,160-168,367-386
//   reverse step        samplers.py:281-345 (DDPM posterior mean or DDIM(eta)), clip :500-508
//   CFG combine         samplers.py:449-455
//   avg_pool pyramid    diffusion.py:346
#include <math.h>

#include "engine.cuh"
#include "mdm_b200.h"

namespace mdm {
namespace {

enum { PT_DDPM = 3, PT_DDIM = 4, PT_V = 5 };  // values of samplers.PredictionType

__device__ __forceinline__ float x0_from_pred(int ptype, float xt, float pred, float a, float c) {
  // a = sqrt(g), c = sqrt(1-g)   (samplers.py:359-367)
  if (ptype == PT_V) return xt * a - pred * c;
  return (xt - pred * c) / a;
}
// x0 * image_scale with one rounding per operation (no FMA contraction): the dynamic-threshold kernels rank these
// values and the step kernel clips them -- both must see the same bits
__device__ __forceinline__ float x0_scaled(int ptype, float xt, float pred, float a, float c, float image_scale) {
  float x0;
  if (ptype == PT_V) x0 = __fsub_rn(__fmul_rn(xt, a), __fmul_rn(pred, c));
  else x0 = __fdiv_rn(__fsub_rn(xt, __fmul_rn(pred, c)), a);
  return __fmul_rn(x0, image_scale);
}
__device__ __forceinline__ float pred_from_x0(int ltype, float xt, float x0, float a, float c) {
  // samplers.py:381-389
  if (ltype == PT_V) return (a * xt - x0) / c;
  return (xt - x0 * a) / c;
}

__global__ void q_sample_kernel(const float* __restrict__ x, const float* __restrict__ eps,
                                const long long* __restrict__ t, const float* __restrict__ gammas, int t_off,
                                float image_div, float* __restrict__ xt, long long per, long long total) {
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const int b = static_cast<int>(i / per);
    const float g = gammas[t[b] + t_off];
    float xi = x[i];
    if (image_div != 1.0f) xi = xi / image_div;
    // no FMA contraction: bit-identical to the reference's separate fp32 mul/add (samplers.py:245)
    xt[i] = __fadd_rn(__fmul_rn(sqrtf(g), xi), __fmul_rn(sqrtf(1.0f - g), eps[i]));
  }
}


// uint8 NHWC image -> normalised fp32 NCHW image x = (u - 127) / 128 (clis/train_parallel.py:193-195) and, in the same
// pass, x_t = sqrt(g) x / div + sqrt(1-g) eps. One thread per pixel: reads its C interleaved bytes, writes C planes.
__global__ void q_sample_u8_kernel(const uint8_t* __restrict__ u8, const float* __restrict__ eps,
                                   const long long* __restrict__ t, const float* __restrict__ gammas, int t_off,
                                   float image_div, float* __restrict__ x, float* __restrict__ xt, int C, long long HW,
                                   long long total_pix) {
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total_pix; i += gs) {
    const long long b = i / HW, p = i - b * HW;
    float sg = 0.f, sn = 0.f;
    if (xt != nullptr) {
      const float g = gammas[t[b] + t_off];
      sg = sqrtf(g);
      sn = sqrtf(1.0f - g);
    }
    for (int c = 0; c < C; ++c) {
      // same two fp32 roundings as the reference's (x.float() - 127.0) / 128.0 (both exact here)
      const float v = __fdiv_rn(__fsub_rn(static_cast<float>(u8[i * C + c]), 127.0f), 128.0f);
      const long long o = (b * C + c) * HW + p;
      x[o] = v;
      if (xt != nullptr) {
        const float vi = image_div != 1.0f ? v / image_div : v;
        xt[o] = __fadd_rn(__fmul_rn(sg, vi), __fmul_rn(sn, eps[o]));
      }
    }
  }
}

// loss[b] = mean_chw (pred_loss - target)^2 * weight ; optionally writes pred_loss / target.
// One block per (sample, chunk); partial sums by atomics into loss (zeroed by the launcher).
__global__ void __launch_bounds__(256)
loss_fwd_kernel(const float* __restrict__ model_out, const float* __restrict__ xt, const float* __restrict__ x,
                const float* __restrict__ eps, const long long* __restrict__ t, const float* __restrict__ gammas,
                int ptype, int ltype, float image_div, float weight, float* __restrict__ loss,
                float* __restrict__ pred_out, float* __restrict__ tgt_out, long long per) {
  const int b = blockIdx.y;
  const float g = gammas[t[b] + 1];
  const float a = sqrtf(g), c = sqrtf(1.0f - g);
  float acc = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < per;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long k = static_cast<long long>(b) * per + i;
    const float v = model_out[k], xti = xt[k];
    float xi = x[k];
    if (image_div != 1.0f) xi = xi / image_div;
    const float tgt = (ltype == PT_V) ? (a * eps[k] - c * xi) : eps[k];
    float p = v;
    if (ltype != ptype) p = pred_from_x0(ltype, xti, x0_from_pred(ptype, xti, v, a, c), a, c);
    if (pred_out != nullptr) pred_out[k] = p;
    if (tgt_out != nullptr) tgt_out[k] = tgt;
    const float d = p - tgt;
    acc += d * d;
  }
  __shared__ float sh[8];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += sh[w];
    atomicAdd(&loss[b], weight * s / static_cast<float>(per));
  }
}

// d model_out = dloss[b] * weight * 2 (p - tgt) / per * dp/dv
__global__ void loss_bwd_kernel(const float* __restrict__ model_out, const float* __restrict__ xt,
                                const float* __restrict__ x, const float* __restrict__ eps,
                                const long long* __restrict__ t, const float* __restrict__ gammas, int ptype,
                                int ltype, float image_div, float weight, const float* __restrict__ dloss,
                                float* __restrict__ dout, long long per, long long total) {
  long long k = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; k < total; k += gs) {
    const int b = static_cast<int>(k / per);
    const float g = gammas[t[b] + 1];
    const float a = sqrtf(g), c = sqrtf(1.0f - g);
    const float v = model_out[k], xti = xt[k];
    float xi = x[k];
    if (image_div != 1.0f) xi = xi / image_div;
    const float tgt = (ltype == PT_V) ? (a * eps[k] - c * xi) : eps[k];
    float p = v, dpdv = 1.0f;
    if (ltype != ptype) {
      p = pred_from_x0(ltype, xti, x0_from_pred(ptype, xti, v, a, c), a, c);
      const float dx0dv = (ptype == PT_V) ? -c : (-c / a);
      const float dpdx0 = (ltype == PT_V) ? (-1.0f / c) : (-a / c);
      dpdv = dpdx0 * dx0dv;
    }
    dout[k] = dloss[b] * weight * 2.0f * (p - tgt) / static_cast<float>(per) * dpdv;
  }
}

// Thresholded x0 of element k, shared by the reverse-step kernels so that they produce the same bits.
__device__ __forceinline__ float thresholded_x0(int ptype, float x, float p, float a, float c, int clip,
                                                float image_scale, const float* __restrict__ bound, long long k,
                                                long long per) {
  if (bound != nullptr) {  // dynamic thresholding (samplers.py:461-508): clamp(x0 s, -b, b) / b / s, b per sample
    const float b = bound[k / per];
    return __fdiv_rn(__fdiv_rn(fminf(fmaxf(x0_scaled(ptype, x, p, a, c, image_scale), -b), b), b), image_scale);
  }
  float x0 = x0_from_pred(ptype, x, p, a, c);
  if (clip) x0 = fminf(fmaxf(x0 * image_scale, -1.0f), 1.0f) / image_scale;
  return x0;
}

// One reverse step for one resolution level (samplers.py:281-345).
//   mode 0: DDPM posterior mean (ddim_eta is None); mode 1: DDIM with eta (>= 0)
__global__ void sampler_step_kernel(const float* __restrict__ xt, const float* __restrict__ pred,
                                    const float* __restrict__ noise, const float* __restrict__ gammas, int t_idx,
                                    int s_idx, int ptype, int clip, float image_scale, int mode, float eta,
                                    int need_noise, float* __restrict__ x0_out, float* __restrict__ xs_out,
                                    long long total, const float* __restrict__ bound, long long per) {
  const float g = gammas[t_idx], gl = gammas[s_idx];
  const float alpha = g / gl;
  const float beta = 1.0f - alpha;
  float beta_tilde = beta * (1.0f - gl) / (1.0f - g);
  const float a = sqrtf(g), c = sqrtf(1.0f - g);
  long long k = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; k < total; k += gs) {
    const float x = xt[k];
    const float x0 = thresholded_x0(ptype, x, pred[k], a, c, clip, image_scale, bound, k, per);
    float xs;
    float bt = beta_tilde;
    int nn = need_noise;
    if (mode == 0) {
      xs = x0 * beta * sqrtf(gl) / (1.0f - g) + x * sqrtf(alpha) * (1.0f - gl) / (1.0f - g);
    } else {
      const float e = (x - x0 * a) / c;
      if (eta > 0.f) {
        bt = (eta * eta) * beta_tilde;
        xs = x0 * sqrtf(gl) + e * sqrtf(1.0f - gl - bt);
      } else {
        nn = 0;
        xs = x0 * sqrtf(gl) + e * sqrtf(1.0f - gl);
      }
    }
    if (nn) xs = xs + sqrtf(bt) * noise[k];
    if (x0_out != nullptr) x0_out[k] = x0;
    xs_out[k] = xs;
  }
}

// One DPM-Solver++ multistep update of one level (2M, or 2M SDE with noise): x0 as sampler_step_kernel computes it,
// then x_s = A x_t + B x0 + C x0_prev + S z with the step's coefficients from the host (C = 0: no x0_prev read;
// S = 0: no noise read). One pass: at most four reads and two writes per element.
__global__ void multistep_kernel(const float* __restrict__ xt, const float* __restrict__ pred,
                                 const float* __restrict__ x0_prev, const float* __restrict__ noise,
                                 const float* __restrict__ gammas, int t_idx, int ptype, int clip, float image_scale,
                                 const float* __restrict__ bound, long long per, float A, float B, float Cc, float S,
                                 float* __restrict__ x0_out, float* __restrict__ xs_out, long long total) {
  const float g = gammas[t_idx];
  const float a = sqrtf(g), c = sqrtf(1.0f - g);
  long long k = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; k < total; k += gs) {
    const float x = xt[k];
    const float x0 = thresholded_x0(ptype, x, pred[k], a, c, clip, image_scale, bound, k, per);
    float xs = fmaf(B, x0, A * x);
    if (x0_prev != nullptr) xs = fmaf(Cc, x0_prev[k], xs);
    if (noise != nullptr) xs = fmaf(S, noise[k], xs);
    x0_out[k] = x0;
    xs_out[k] = xs;
  }
}


// ---- dynamic thresholding (samplers.py:461-508): bound[b] = clamp(quantile(|x0 * image_scale|, q), 1, max_value) over
// the C*H*W values of sample b, with torch.quantile's arithmetic: rank = q * (n - 1) in fp32, the two order statistics
// at floor(rank) / ceil(rank), torch's lerp. The order statistics are EXACT: a 3-pass radix select (11 + 10 + 10 bits)
// over the bit patterns of the non-negative floats, one CTA per sample, x0 recomputed from (x_t, pred) in every pass
// so nothing is materialised.
constexpr int DT_THREADS = 1024;

__device__ __forceinline__ unsigned dt_key(int ptype, float xt, float pred, float a, float c, float image_scale) {
  return __float_as_uint(fabsf(x0_scaled(ptype, xt, pred, a, c, image_scale)));
}

// Block-wide: which of the 2048 bins holds rank `r` (0-based among the counted elements)? Returns the bin and
// rewrites r to the rank inside it. hist: 2048 counters in shared memory.
__device__ unsigned dt_find_bin(const unsigned* hist, unsigned* r_io, unsigned* scratch) {
  const int t = threadIdx.x;
  const unsigned c0 = hist[2 * t], c1 = hist[2 * t + 1];
  unsigned v = c0 + c1;
  // inclusive scan over the 1024 threads
  unsigned incl = v;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned n = __shfl_up_sync(0xffffffffu, incl, o);
    if ((t & 31) >= o) incl += n;
  }
  if ((t & 31) == 31) scratch[t >> 5] = incl;
  __syncthreads();
  if (t < 32) {
    unsigned w = scratch[t];
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned n = __shfl_up_sync(0xffffffffu, w, o);
      if (t >= o) w += n;
    }
    scratch[32 + t] = w;  // inclusive totals per warp
  }
  __syncthreads();
  const unsigned before_warp = (t >> 5) == 0 ? 0u : scratch[32 + (t >> 5) - 1];
  incl += before_warp;
  const unsigned excl = incl - v;
  const unsigned r = *r_io;
  __syncthreads();
  if (r >= excl && r < incl) {  // exactly one thread
    if (r - excl < c0) {
      scratch[64] = 2 * t;
      scratch[65] = r - excl;
    } else {
      scratch[64] = 2 * t + 1;
      scratch[65] = r - excl - c0;
    }
    scratch[66] = (r - excl < c0) ? c0 : c1;
  }
  __syncthreads();
  *r_io = scratch[65];
  return scratch[64];
}

__global__ void __launch_bounds__(DT_THREADS)
dyn_threshold_kernel(const float* __restrict__ xt, const float* __restrict__ pred, const float* __restrict__ gammas,
                     int t_idx, int ptype, float image_scale, float q, float max_value, float* __restrict__ bound,
                     long long per) {
  __shared__ unsigned hist[2048];
  __shared__ unsigned scratch[72];
  const int b = blockIdx.x, t = threadIdx.x;
  const float g = gammas[t_idx];
  const float a = sqrtf(g), c = sqrtf(1.0f - g);
  const float* xb = xt + static_cast<long long>(b) * per;
  const float* pb = pred + static_cast<long long>(b) * per;
  // torch.quantile: ranks = q * (n - 1) as fp32; below = floor, above = ceil, weight = ranks - below
  const float rank = __fmul_rn(q, static_cast<float>(per - 1));
  const float below = floorf(rank);
  const unsigned kb = static_cast<unsigned>(below), ka = static_cast<unsigned>(ceilf(rank));
  const float w = __fsub_rn(rank, below);
  unsigned prefix = 0, mask = 0, r = kb;
  const int shifts[3] = {20, 10, 0}, widths[3] = {11, 10, 10};
  unsigned count_in_bin = 0;
  for (int ps = 0; ps < 3; ++ps) {
    for (int i = t; i < 2048; i += DT_THREADS) hist[i] = 0;
    __syncthreads();
    const unsigned bm = (1u << widths[ps]) - 1u;
    for (long long i = t; i < per; i += DT_THREADS) {
      const unsigned u = dt_key(ptype, xb[i], pb[i], a, c, image_scale);
      if ((u & mask) == prefix) atomicAdd(&hist[(u >> shifts[ps]) & bm], 1u);
    }
    __syncthreads();
    const unsigned bin = dt_find_bin(hist, &r, scratch);
    count_in_bin = scratch[66];
    prefix |= bin << shifts[ps];
    mask |= bm << shifts[ps];
    __syncthreads();
  }
  const unsigned u_below = prefix;  // all 31 bits fixed: the value at rank kb; r = its index among its duplicates
  unsigned u_above = u_below;
  if (ka != kb && r + 1 >= count_in_bin) {  // the next order statistic is the smallest value above u_below
    if (t == 0) scratch[67] = 0xffffffffu;
    __syncthreads();
    unsigned m = 0xffffffffu;
    for (long long i = t; i < per; i += DT_THREADS) {
      const unsigned u = dt_key(ptype, xb[i], pb[i], a, c, image_scale);
      if (u > u_below && u < m) m = u;
    }
    for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((t & 31) == 0) atomicMin(&scratch[67], m);
    __syncthreads();
    u_above = scratch[67];
  }
  if (t == 0) {
    const float vb = __uint_as_float(u_below), va = __uint_as_float(u_above);
    // at::lerp: |w| < 0.5 ? a + w (b - a) : b - (b - a)(1 - w)
    const float d = __fsub_rn(va, vb);
    const float s = (fabsf(w) < 0.5f) ? __fadd_rn(vb, __fmul_rn(w, d)) : __fsub_rn(va, __fmul_rn(d, __fsub_rn(1.0f, w)));
    bound[b] = fminf(fmaxf(s, 1.0f), max_value);
  }
}

__global__ void cfg_combine_kernel(const float* __restrict__ uncond, const float* __restrict__ cond, float w,
                                   float* __restrict__ out, long long n) {
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < n; i += gs) out[i] = uncond[i] + w * (cond[i] - uncond[i]);
}

__global__ void avg_pool_kernel(const float* __restrict__ x, float* __restrict__ y, int planes, int H, int W,
                                int r) {
  const int Ho = H / r, Wo = W / r;
  const long long total = static_cast<long long>(planes) * Ho * Wo;
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < total; i += gs) {
    const int wo = static_cast<int>(i % Wo);
    const long long tt = i / Wo;
    const int ho = static_cast<int>(tt % Ho);
    const long long pl = tt / Ho;
    const float* src = x + (pl * H + static_cast<long long>(ho) * r) * W + static_cast<long long>(wo) * r;
    float s = 0.f;
    for (int a = 0; a < r; ++a)
      for (int b = 0; b < r; ++b) s += src[static_cast<long long>(a) * W + b];
    y[i] = s / static_cast<float>(r * r);
  }
}

__global__ void clip_scale_kernel(const float* __restrict__ x, float scale, int clip, float* __restrict__ y,
                                  long long n) {
  long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long gs = static_cast<long long>(gridDim.x) * blockDim.x;
  for (; i < n; i += gs) {
    float v = x[i] * scale;
    if (clip) v = fminf(fmaxf(v, -1.0f), 1.0f);
    y[i] = v;
  }
}

inline int grid_for(long long n) {
  long long g = (n + 255) / 256;
  if (g > 132 * 16) g = 132 * 16;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

}  // namespace
}  // namespace mdm

#define MDM_TRY(...)                     \
  try {                                  \
    __VA_ARGS__;                         \
    return 0;                            \
  } catch (const std::exception& e) {    \
    mdm::set_error("%s", e.what());      \
    return -1;                           \
  }

extern "C" {

int mdm_q_sample(const float* x, const float* eps, const int64_t* t, const float* gammas, int t_offset,
                 float image_div, float* x_t, int batch, int64_t per_sample, mdm_stream_t stream) {
  MDM_TRY({
    const long long total = static_cast<long long>(batch) * per_sample;
    mdm::q_sample_kernel<<<mdm::grid_for(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, eps, reinterpret_cast<const long long*>(t), gammas, t_offset, image_div, x_t, per_sample, total);
    ++mdm::g_launch_count;
    MDM_CUDA(cudaGetLastError());
  })
}

int mdm_q_sample_u8(const uint8_t* images_u8, const float* eps, const int64_t* t, const float* gammas, int t_offset,
                    float image_div, float* x, float* x_t, int batch, int channels, int height, int width,
                    mdm_stream_t stream) {
  MDM_TRY({
    if (x == nullptr || images_u8 == nullptr) throw mdm::MdmFail("mdm_q_sample_u8: images_u8 and x are required");
    if (x_t != nullptr && (eps == nullptr || t == nullptr || gammas == nullptr))
      throw mdm::MdmFail("mdm_q_sample_u8: eps, t and gammas are required when x_t is requested");
    const long long HW = static_cast<long long>(height) * width, total = HW * batch;
    mdm::q_sample_u8_kernel<<<mdm::grid_for(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        images_u8, eps, reinterpret_cast<const long long*>(t), gammas, t_offset, image_div, x, x_t, channels, HW, total);
    ++mdm::g_launch_count;
    MDM_CUDA(cudaGetLastError());
  })
}

int mdm_loss_fwd(const float* model_out, const float* x_t, const float* x, const float* eps, const int64_t* t,
                 const float* gammas, int prediction_type, int loss_type, float image_div, float weight,
                 float* loss, float* pred_out, float* tgt_out, int batch, int64_t per_sample, mdm_stream_t stream) {
  MDM_TRY({
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int chunks = static_cast<int>(std::min<long long>((per_sample + 1023) / 1024, 64));
    if (chunks < 1) chunks = 1;
    dim3 grid(chunks, batch);
    mdm::loss_fwd_kernel<<<grid, 256, 0, st>>>(model_out, x_t, x, eps, reinterpret_cast<const long long*>(t), gammas,
                                               prediction_type, loss_type, image_div, weight, loss, pred_out, tgt_out,
                                               per_sample);
    ++mdm::g_launch_count;
    MDM_CUDA(cudaGetLastError());
  })
}

int mdm_loss_bwd(const float* model_out, const float* x_t, const float* x, const float* eps, const int64_t* t,
                 const float* gammas, int prediction_type, int loss_type, float image_div, float weight,
                 const float* dloss, float* dmodel_out, int batch, int64_t per_sample, mdm_stream_t stream) {
  MDM_TRY({
    const long long total = static_cast<long long>(batch) * per_sample;
    mdm::loss_bwd_kernel<<<mdm::grid_for(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        model_out, x_t, x, eps, reinterpret_cast<const long long*>(t), gammas, prediction_type, loss_type, image_div,
        weight, dloss, dmodel_out, per_sample, total);
    ++mdm::g_launch_count;
    MDM_CUDA(cudaGetLastError());
  })
}

int mdm_sampler_step(const float* x_t, const float* pred, const float* noise, const float* gammas, int t_index,
                     int s_index, int prediction_type, int clip, float image_scale, int use_ddim, float ddim_eta,
                     int need_noise, float* x0_out, float* x_s_out, int64_t numel, mdm_stream_t stream) {
  MDM_TRY({
    if (need_noise && !(use_ddim && ddim_eta <= 0.f) && noise == nullptr)
      throw mdm::MdmFail("mdm_sampler_step: noise tensor required for a stochastic step");
    mdm::sampler_step_kernel<<<mdm::grid_for(numel), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x_t, pred, noise, gammas, t_index, s_index, prediction_type, clip, image_scale, use_ddim ? 1 : 0, ddim_eta,
        need_noise, x0_out, x_s_out, numel, nullptr, 1);
    ++mdm::g_launch_count;
    MDM_CUDA(cudaGetLastError());
  })
}

int mdm_dynamic_threshold(const float* x_t, const float* pred, const float* gammas, int t_index, int prediction_type,
                          float image_scale, float ratio, float max_value, float* bound, int batch, int64_t per_sample,
                          mdm_stream_t stream) {
  MDM_TRY({
    if (batch < 1 || per_sample < 2 || per_sample >= (1ll << 31)) throw mdm::MdmFail("mdm_dynamic_threshold: bad sizes");
    mdm::dyn_threshold_kernel<<<batch, mdm::DT_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        x_t, pred, gammas, t_index, prediction_type, image_scale, ratio, max_value, bound, per_sample);
    ++mdm::g_launch_count;
    MDM_CUDA(cudaGetLastError());
  })
}

int mdm_sampler_step_dynamic(const float* x_t, const float* pred, const float* noise, const float* gammas, int t_index,
                             int s_index, int prediction_type, const float* bound, float image_scale, int use_ddim,
                             float ddim_eta, int need_noise, float* x0_out, float* x_s_out, int batch, int64_t per_sample,
                             mdm_stream_t stream) {
  MDM_TRY({
    if (bound == nullptr) throw mdm::MdmFail("mdm_sampler_step_dynamic: bound required");
    if (need_noise && !(use_ddim && ddim_eta <= 0.f) && noise == nullptr)
      throw mdm::MdmFail("mdm_sampler_step_dynamic: noise tensor required for a stochastic step");
    const long long numel = static_cast<long long>(batch) * per_sample;
    mdm::sampler_step_kernel<<<mdm::grid_for(numel), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x_t, pred, noise, gammas, t_index, s_index, prediction_type, 1, image_scale, use_ddim ? 1 : 0, ddim_eta,
        need_noise, x0_out, x_s_out, numel, bound, per_sample);
    ++mdm::g_launch_count;
    MDM_CUDA(cudaGetLastError());
  })
}

int mdm_sampler_multistep(const float* x_t, const float* pred, const float* x0_prev, const float* noise,
                          const float* gammas, int t_index, int prediction_type, int clip, const float* bound,
                          float image_scale, float coef_xt, float coef_x0, float coef_x0_prev, float coef_noise,
                          float* x0_out, float* x_s_out, int batch, int64_t per_sample, mdm_stream_t stream) {
  MDM_TRY({
    if (x_t == nullptr || pred == nullptr || gammas == nullptr || x0_out == nullptr || x_s_out == nullptr)
      throw mdm::MdmFail("mdm_sampler_multistep: x_t, pred, gammas, x0_out and x_s_out are required");
    if (batch < 1 || per_sample < 1) throw mdm::MdmFail("mdm_sampler_multistep: bad sizes");
    if (coef_x0_prev != 0.f && x0_prev == nullptr)
      throw mdm::MdmFail("mdm_sampler_multistep: x0_prev required for a second-order step");
    if (coef_noise != 0.f && noise == nullptr)
      throw mdm::MdmFail("mdm_sampler_multistep: noise tensor required for a stochastic step");
    const long long numel = static_cast<long long>(batch) * per_sample;
    mdm::multistep_kernel<<<mdm::grid_for(numel), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x_t, pred, coef_x0_prev != 0.f ? x0_prev : nullptr, coef_noise != 0.f ? noise : nullptr, gammas, t_index,
        prediction_type, clip, image_scale, bound, per_sample, coef_xt, coef_x0, coef_x0_prev, coef_noise, x0_out,
        x_s_out, numel);
    ++mdm::g_launch_count;
    MDM_CUDA(cudaGetLastError());
  })
}

int mdm_cfg_combine(const float* uncond, const float* cond, float guidance_scale, float* out, int64_t numel,
                    mdm_stream_t stream) {
  MDM_TRY({
    mdm::cfg_combine_kernel<<<mdm::grid_for(numel), 256, 0, static_cast<cudaStream_t>(stream)>>>(uncond, cond,
                                                                                                guidance_scale, out,
                                                                                                numel);
    ++mdm::g_launch_count;
    MDM_CUDA(cudaGetLastError());
  })
}

int mdm_avg_pool(const float* x, float* y, int planes, int H, int W, int ratio, mdm_stream_t stream) {
  MDM_TRY({
    if (ratio < 1 || H % ratio != 0 || W % ratio != 0) throw mdm::MdmFail("mdm_avg_pool: size not divisible");
    const long long total = static_cast<long long>(planes) * (H / ratio) * (W / ratio);
    mdm::avg_pool_kernel<<<mdm::grid_for(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, planes, H, W,
                                                                                             ratio);
    ++mdm::g_launch_count;
    MDM_CUDA(cudaGetLastError());
  })
}

int mdm_clip_scale(const float* x, float scale, int clip, float* y, int64_t numel, mdm_stream_t stream) {
  MDM_TRY({
    mdm::clip_scale_kernel<<<mdm::grid_for(numel), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, scale, clip, y,
                                                                                               numel);
    ++mdm::g_launch_count;
    MDM_CUDA(cudaGetLastError());
  })
}

}  // extern "C"
