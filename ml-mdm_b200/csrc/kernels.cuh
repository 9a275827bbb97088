// Non-GEMM kernels of the denoising path: GroupNorm(+FiLM+SiLU) forward/backward, softmax,
// LayerNorm, activations, layout/precision packing, resampling, and the diffusion algebra.
// All are HBM-bound streaming kernels: 128-bit loads along the channel (contiguous) dimension,
// per-channel register accumulation, warp-shuffle / shared-memory reductions.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mdm {

// A channel-concatenated NHWC fp32 tensor made of one or two sources (torch.cat((x, skip), 1),
// reference unet.py:547, is never materialised in fp32).
struct Src2 {
  const float* p0;
  const float* p1;
  int c0, c1;  // channels of each source (c1 == 0: single source)
};
struct Dst2 {
  float* p0;
  float* p1;
  int c0, c1;
  int acc0, acc1;  // 1: += into existing contents, 0: overwrite
  // alternative single-consumer destination: fp16 operand + column sums (bias gradient); p0/p1 unused
  __half* h16;
  float* colsum;
  const float* inv_scale;
  __half* h16lo;  // optional second fp16 plane of h16: fp16(v - h16)
};

// ---- dropout on the output of a GroupNorm apply (ResNet.dropout, reference unet.py:208,233-235)
// Element i (NHWC linear index of the [N][HW][C] output) is kept when u >= p, where u * 2^32 is word i % 4 of
// Philox4x32-10 with key = *seed and counter = (i / 4 as two words, stream, 0); kept elements are scaled by 1/(1-p) and
// p == 1 drops everything. The mask is a pure function of (seed, stream, i): the backward regenerates it.
struct Dropout {
  float p = 0.f;                           // 0: off (the kernels take their plain form)
  const unsigned long long* seed = nullptr;  // device slot, read by the kernels (a replayed graph sees its new value)
  uint32_t stream = 0;
};
// *slot = seed, one thread on st (no host synchronisation)
void dropout_set_seed(unsigned long long* slot, unsigned long long seed, cudaStream_t st);
// out[i] = the factor (0 or 1/(1-p)) the fused kernels apply to element i, i < n
void dropout_mask(unsigned long long seed, uint32_t stream, long long n, float p, float* out, cudaStream_t st);

// ---- GroupNorm family (reference: nn.GroupNorm(32, C) in unet.py:198,207,259,268,749)
// sums: [N][G][2] (sum, sumsq), must be zero on entry.
void gn_stats(const Src2& x, int N, int HW, int G, float* sums, cudaStream_t st);
// y16 = drop(act(gn(x) * (1 + ta) + tb)); film = [N][film_ld] fp32 rows with ta at film_off, tb at
// film_off + C (null: no FiLM). raw16 (optional) receives the un-normalised fp16 copy of x.
void gn_apply(const Src2& x, int N, int HW, int G, const float* sums, const float* gamma,
              const float* beta, const float* film, int film_ld, int film_off, int silu, __half* y16,
              __half* raw16, cudaStream_t st, const Dropout& drop = Dropout());
// Backward. dy: fp32 or fp16 (dy_f16) [N][HW][C] gradient w.r.t. y16; `drop` as in the forward.
// ab: [N][C][2] scratch, zero on entry.
void gn_bwd_reduce(const Src2& x, const void* dy, int dy_f16, int N, int HW, int G, const float* sums,
                   const float* gamma, const float* beta, const float* film, int film_ld, int film_off,
                   int silu, float* ab, cudaStream_t st, const Dropout& drop = Dropout());
// pg: [N][G][2] scratch (written). dgamma/dbeta: += inv_scale * grad. dfilm (optional): dense
// [N][2C] rows (d_ta | d_tb), overwritten.
void gn_bwd_finalize(int N, int C, int G, int HW, const float* ab, const float* gamma, const float* beta,
                     const float* film, int film_ld, int film_off, float* pg, float* dgamma,
                     float* dbeta, float* dfilm, const float* inv_scale, cudaStream_t st);
// dx = rstd * (du*(1+ta)*gamma - P1/m - xhat*P2/m) + extra ; written/accumulated into dst.
void gn_bwd_apply(const Src2& x, const void* dy, int dy_f16, int N, int HW, int G, const float* sums,
                  const float* gamma, const float* beta, const float* film, int film_ld, int film_off,
                  int silu, const float* pg, const float* extra, const Dst2& dst, cudaStream_t st,
                  const Dropout& drop = Dropout());

// ---- precision / reductions
// out16 = half(in) and colsum[c] += inv_scale * sum_rows(in[:, c]) (colsum may be null).
void cast_colsum(const float* in, __half* out16, long long rows, int C, float* colsum,
                 const float* inv_scale, cudaStream_t st);
void colsum_f16(const __half* in, long long rows, int C, float* colsum, const float* inv_scale,
                cudaStream_t st);
void cast_f32_to_f16(const float* in, __half* out, long long n, cudaStream_t st);
// out16[r][:] = half(in[r][:] * rowscale[r]); D % 4 == 0
void cast_rowscale_f16(const float* in, const float* rowscale, __half* out16, long long rows, int D, cudaStream_t st);
void add_f32(float* dst, const float* a, const float* b, long long n, cudaStream_t st);  // dst = a + b
void axpy_f32(float* dst, const float* a, float alpha, long long n, int acc, cudaStream_t st);
void scale_f32(float* dst, const float* a, const float* scale, long long n, cudaStream_t st);  // dst = *scale * a

// ---- attention pieces (reference unet.py:276-294)
// P16[r][:] = softmax(scores[r][:]) ; mask (optional) is [B][S] with row r belonging to batch
// r / rows_per_batch; masked columns get -inf.
// ld = row stride in elements (>= S; padded so TMA strides stay 16-byte aligned).
void softmax_rows(const float* scores, __half* P16, long long rows, int S, int ld, const float* mask,
                  long long rows_per_batch, cudaStream_t st);
// dS16 = P * (dP - sum(dP * P)) * scale
void softmax_bwd_rows(const __half* P16, const float* dP, __half* dS16, long long rows, int S, int ld, float scale,
                      cudaStream_t st);

// ---- LayerNorm over the last dim (reference unet.py:263, eps 1e-5)
void layernorm_fwd(const float* x, const float* w, const float* b, __half* y16, float* stats, long long rows,
                   int D, cudaStream_t st);
void layernorm_bwd(const float* x, const float* w, const float* stats, const float* dy, float* dx,
                   int acc_dx, float* dw, float* db, const float* inv_scale, long long rows, int D,
                   cudaStream_t st);

// LayerNorm affine folded into the Linear that follows it (w, b may be null in layernorm_fwd/bwd: plain xhat)
// lo (optional): the second fp16 plane, fp16(W w - out)
void fold_ln_weight(const float* W, const float* w, __half* out, __half* lo, long long rows, int D, cudaStream_t st);
void f16_residual(const float* in, float* out, long long n, cudaStream_t st);  // out = in - fp16(in)
// lo = fp16(in - fp16(in)): the second fp16 plane of an fp16 copy of `in` (n a multiple of 4, 16-byte aligned)
void f16_lo_plane(const float* in, __half* lo, long long n, cudaStream_t st);
void fold_ln_bias(const float* W, const float* b, const float* bias, float* out, int rows, int D, cudaStream_t st);
void unfold_ln_grads(const float* dWf, const float* dbf, const float* W, const float* w, const float* b, float* dW,
                     float* dw, float* db, int rows, int D, cudaStream_t st);

// ---- embeddings / small elementwise
// The micro-conditioning keys of one level, in its order (unet.py:920-933).
constexpr int kMaxMicroKeys = 8;  // MDM_MAX_MICRO
struct MicroKeys {
  int num;
  const float* values[kMaxMicroKeys];  // (B,) fp32, or null: the key takes its default
  float defaults[kMaxMicroKeys];
  unsigned scale_mask;  // bit k: key k is "scale" (clamp(v/default, max=1)*default); otherwise v*1000
};
// e16[b][0:half]=sin(v*w_i), [half:2half]=cos(v*w_i); w = the reference's t_emb buffer
// exp(-ln(1e4) i/half) (unet.py:600-603,834-836), bound from the host so it is bit-identical.
// Exactly one of times / micro is non-null. times (int64): one embedding, v = times[b]. micro: one embedding per key
// k, at e16 + k * key_stride, of v = the key's transform of its value (unet.py:924-929).
void sinusoid_embed(const long long* times, const MicroKeys* micro, const float* freq, int B, int half,
                    long long key_stride, __half* e16, cudaStream_t st);
void silu_f16(const float* x, __half* y16, long long n, cudaStream_t st);
// dx (=|+=) dy * silu'(x)
void silu_bwd(const float* x, const float* dy, float* dx, long long n, int acc, cudaStream_t st);
// du16 = dg * gelu'(u16)  (exact erf GELU, unet.py:270)
void gelu_bwd(const __half* u16, const float* dg, __half* du16, long long n, cudaStream_t st);
// masked mean over tokens: y[b][d] = sum_s mask[b][s]*x[b][s][d] / sum_s mask[b][s]  (unet.py:857-861)
void masked_mean(const float* x, const float* mask, float* y, __half* y16, int B, int S, int D,
                 cudaStream_t st);
// dx[b][s][d] (+)= mask[b][s] * dy[b][d] / sum_s mask
void masked_mean_bwd(const float* dy, const float* mask, float* dx, int acc, int B, int S, int D,
                     cudaStream_t st);

// ---- conv helpers
// col16[(n,ho,wo)][tap*C + c] for a 3x3 / pad 1 / given stride conv over NHWC fp32 x.
void im2col3x3(const float* x, __half* col16, int N, int H, int W, int C, int stride, cudaStream_t st);
// dx[n,h,w,c] (+)= sum over taps of dcol (gather form of col2im for the same geometry).
void col2im3x3(const float* dcol, float* dx, int acc, int N, int H, int W, int C, int stride,
               cudaStream_t st);
// conv_in: NCHW fp32 image (Cin channels, 9*Cin <= 32) -> [N*H*W][32] fp16, k = tap*Cin + c.
// inv_std (optional, [N]) divides the image (nested_unet.py:184-186 input normalisation).
void im2col_input(const float* x_nchw, const float* inv_std, __half* col16, int N, int Cin, int H, int W,
                  cudaStream_t st);
void upsample2x_f16(const float* x, __half* y16, int N, int H, int W, int C, cudaStream_t st);
// dx[n,h,w,c] (+)= sum of the 2x2 block of dy (backward of nearest x2)
void upsample2x_bwd(const float* dy, float* dx, int acc, int N, int H, int W, int C, cudaStream_t st);
// tanh_scale = s != 0 (model_output_scale): y = s * tanh(x / s), also stored to keep when keep != nullptr
void nhwc_to_nchw(const float* x, int ldc, float* y, int N, int C, int HW, cudaStream_t st, float tanh_scale = 0.f,
                  float* keep = nullptr);
// dy16[pix][ldo] = half(scale * dy_nchw) (columns >= C zero-filled); with tanh_scale = s != 0 and y_out (the NCHW
// output s * tanh(o / s)) dy_nchw is first multiplied by 1 - (y_out / s)^2
void nchw_to_nhwc_f16(const float* x_nchw, const float* scale, __half* y16, int ldo, int N, int C, int HW,
                      cudaStream_t st, float tanh_scale = 0.f, const float* y_out = nullptr);
// per-sample unbiased std over (C,H,W): inv_std[n] = 1/std  (nested_unet.py:872)
void sample_inv_std(const float* x, float* inv_std, int N, long long per, cudaStream_t st);

// ---- weight packing (fp32 master parameters -> fp16 operand layouts) and gradient unpacking
void pack_conv_w(const float* w_oihw, __half* packed, int Co, int Ci, int taps, cudaStream_t st);
void pack_conv_in_w(const float* w_oihw, __half* packed, int Co, int Ci, cudaStream_t st);  // [Co][32]
// W-folded 3x3 weights [2Co][9][2Ci] (two adjacent pixels as one pixel with twice the channels) and the matching
// gradient un-fold: g_oihw += inv_scale * fold^T(packed [2Co][9][2Ci])
void pack_conv_w_fold(const float* w_oihw, __half* packed, int Co, int Ci, cudaStream_t st);
void unpack_conv_wgrad_fold(const float* packed, float* g_oihw, int Co, int Ci, const float* inv_scale,
                            cudaStream_t st);
// g_oihw += inv_scale * packed  (packed: [Co][taps][ci_ld] fp32, only ci < Ci used)
void unpack_conv_wgrad(const float* packed, float* g_oihw, int Co, int Ci, int taps, int ci_ld,
                       const float* inv_scale, cudaStream_t st);
void unpack_conv_in_wgrad(const float* packed, float* g_oihw, int Co, int Ci, const float* inv_scale,
                          cudaStream_t st);

// ---- gradient scaling: scale = 2^k with amax(|g|) * scale in [2^3, 2^4); inv = 1/scale.
// amax_buf must be zero on entry; call grad_amax for every tensor, then grad_scale_finalize.
// tanh_scale / y_out as in nchw_to_nhwc_f16: the max is taken over g * (1 - (y_out / s)^2)
void grad_amax(const float* g, long long n, float* amax_buf, cudaStream_t st, float tanh_scale = 0.f,
               const float* y_out = nullptr);
void grad_scale_finalize(const float* amax_buf, float* scale, float* inv_scale, cudaStream_t st);

}  // namespace mdm
