/*
 * mdm_b200 -- C ABI of the H100-native (sm_90a) Matryoshka denoising path.
 *
 * The reference (apple/ml-mdm) is pure Python/PyTorch and has no FFI of its own; the entry points
 * below are what a binding for its hot path would call.  Each one names the reference interface it
 * stands behind (paths relative to ml-mdm-matryoshka/ml_mdm/):
 *
 *   mdm_net_*            models/unet.py:579-987 (UNet), models/nested_unet.py:96-230 (NestedUNet):
 *                        construction from UNetConfig / NestedUNetConfig, forward(), and the autograd
 *                        backward that `loss.backward()` (trainer.py:46,75) runs through it.
 *   mdm_gammas_*         samplers.py:126-170,201-231,255-264 (noise schedules, shifted schedule)
 *   mdm_set_timesteps    samplers.py:601-609
 *   mdm_q_sample*, mdm_loss*   samplers.py:233-279, diffusion.py:123-168,315-387
 *   mdm_sampler_step     samplers.py:281-345 (get_prediction_xt_last) as used by :392-433,:655-713
 *   mdm_op_*             single fused operators, exported so parity tests can pin each kernel
 *
 * Conventions: every function returns 0 on success and a negative code on failure; the message is
 * available from mdm_last_error().  Pointers are raw device pointers unless named host_*.  Nothing
 * is allocated on the hot path after the first call with a given shape.  All work is enqueued on
 * the cudaStream_t passed by the caller (pass torch.cuda.current_stream().cuda_stream).
 * There is no CPU fallback: without an sm_90a device every compute entry point fails.
 */
#ifndef MDM_B200_H_
#define MDM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* mdm_stream_t; /* cudaStream_t */

const char* mdm_last_error(void);
int mdm_version(void);
/* sizeof() of the structs of this header as the library was compiled (0 = mdm_tmap_spec, 1 = mdm_gemm_params,
 * 2 = mdm_level_cfg, 3 = mdm_net_cfg, 4 = mdm_net_io, 5 = mdm_net_grad_io, 6 = mdm_opt_chunk, 7 = mdm_adam_cfg; -1 for
 * anything else): a binding written in another language (the ctypes mirror in mdm_b200/, a cgo / JNI stub) checks its own
 * struct layout against this instead of trusting that two copies of a declaration stayed in step. */
long long mdm_abi_sizeof(int which);
/* Number of CUDA kernels this library has launched since load (bench.py's gpu_launches). */
unsigned long long mdm_launch_count(void);

/* ---------------------------------------------------------------- low-level wgmma GEMM engine */

/* 4-D TMA view of an fp16 operand; dims[0] is contiguous.
 * rows mode: (inner, rows, z1, z2); patch mode: (channels, W, H, image). Strides in elements. */
typedef struct mdm_tmap_spec {
  const void* ptr;
  uint64_t dims[4];
  uint64_t strides[4];
  uint32_t box[4];
} mdm_tmap_spec;

enum { MDM_GEMM_PLAIN = 0, MDM_GEMM_CONV = 1, MDM_GEMM_CONV_WGRAD = 2 };
enum { MDM_ACT_NONE = 0, MDM_ACT_GELU = 1 };

typedef struct mdm_gemm_params {
  int32_t kind;
  int32_t M, N, K;
  int32_t block_n;
  int32_t nz1, nz2, nsplit;
  int32_t a_z1_off, b_z1_off, a_use_z, b_use_z;
  int32_t H, W, PW, PH, tiles_w, tiles_h, nimg;
  int32_t taps, flip, kblocks_c;
  int32_t num_kblocks;
  int32_t num_stages; /* filled by the launcher */
  float alpha;
  const float* alpha_dev;
  const float* bias;
  const float* residual;
  float* out_f32;
  void* out_f16;     /* __half* */
  void* out_act_f16; /* __half*: act(v); out_f16 then receives the pre-activation */
  int64_t ldc, c_z1_stride, c_z2_stride;
  int32_t act;
  int32_t atomic;
  int32_t epi_tma; /* filled by the launcher: 1 = TMA epilogue (with epi_op = 1): the residual or GELU' source is loaded
                    * by TMA into the staging tile while the tile's MMAs run, the consumers fold their accumulators into
                    * it, and the outputs are written by TMA stores. Chosen for plain products with a GELU or GELU'
                    * epilogue or at most 8 k blocks, where tensor maps can describe every epilogue buffer: 16 B-aligned
                    * bases, ldc and batch strides multiples of 16 B, a tile width that is a multiple of 32 columns up
                    * to 128, fp32 buffers (residual, out_f32) or fp16 ones (GELU' source, out_f16, out_act_f16) but
                    * not both, no split-K atomics. 0 = the epilogue loads and stores with ordinary instructions */
  const void* gelu_grad_src; /* optional __half*, indexed like the output: result *= gelu'(src) (FFN backward) */
  int32_t cluster; /* reserved (the launcher sets 1): every CTA loads its own B tile */
  int32_t kfactor; /* MDM_GEMM_CONV_WGRAD only: pixel rows per pipeline stage = 64 * kfactor (0/1: 64). Narrow layers
                    * (<= 64 channels) move only 4-8 KB per 64-pixel stage, so the stage round trip, not HBM, sets
                    * the pace; 256-pixel stages cut the round trips four-fold. Needs a PW x PH = 64 * kfactor patch. */
  int32_t pair;   /* reserved (the launcher sets 0) */
  int32_t epi_op; /* filled by the launcher: 1 = the persistent kernel's epilogue runs from a shared-memory staging
                   * tile on warps of its own, overlapped with the next tile's MMAs; 0 = from the accumulator registers */
} mdm_gemm_params;

/* Measurement aid for bench.py's roofline leg: while enabled every launch of the wgmma GEMM kernel
 * is bracketed by CUDA events on its stream; mdm_profile_read returns and clears their sum. */
int mdm_profile_gemm(int enable);
int mdm_profile_read(double* total_ms, long long* launches);
/* Writes one CSV row per profiled launch (shape, grid parameters, milliseconds, and the lo planes it multiplied:
 * planes = 0 none, 1 B lo, 2 A lo, 3 both); call before mdm_profile_read. */
int mdm_profile_dump(const char* path);

int mdm_gemm_raw(const mdm_tmap_spec* A, const mdm_tmap_spec* B, int a_mn, int b_mn,
                 const mdm_gemm_params* p, mdm_stream_t stream);
/* mdm_gemm_raw with the split operand planes the engine gives its weight products: b_lo (or NULL) is a second fp16
 * plane laid out exactly like B, a_lo (or NULL) one laid out exactly like A; the result is A B + A b_lo + a_lo B.
 * MDM_GEMM_CONV_WGRAD uses neither plane, and a_lo is used only with a K-major A (a_mn = 0). */
int mdm_gemm_raw_split(const mdm_tmap_spec* A, const mdm_tmap_spec* B, int a_mn, int b_mn, const mdm_gemm_params* p,
                       const void* b_lo, const void* a_lo, mdm_stream_t stream);


/* ---------------------------------------------------------------- the (nested) U-Net denoiser */

#define MDM_MAX_RES 8
#define MDM_MAX_LEVELS 4

/* One U-Net of the nest.  Field meaning follows UNetConfig (models/unet.py:62-156) after
 * __post_init__: lists are per resolution; num_attn[i] is already 0 when i is not in
 * attention_levels; cond_level[i] = 1 when i is in attention_levels. */
typedef struct mdm_level_cfg {
  int32_t num_res;
  int32_t channels[MDM_MAX_RES];
  int32_t num_resnets[MDM_MAX_RES];
  int32_t num_attn[MDM_MAX_RES];
  int32_t cond_level[MDM_MAX_RES];
  int32_t temporal_dim;
  int32_t groups;
  int32_t use_attention_ffn;
  int32_t skip_mid_blocks;
  int32_t nesting;            /* this U-Net sits inside another one (UNetConfig.nesting) */
  int32_t skip_normalization; /* NestedUNetConfig.skip_normalization (outer levels only) */
  int32_t has_micro_scale;    /* micro_conditioning == "scale:<default>" (mdm_net_create; other strings: mdm_micro_cfg) */
  float micro_scale_default;
  /* ResNetConfig.dropout in [0, 1]: nn.Dropout between SiLU(norm2) and conv2 of every ResNet of this level
   * (unet.py:208,233-235), applied when mdm_net_io.dropout is 1 */
  float dropout;
} mdm_level_cfg;

typedef struct mdm_net_cfg {
  int32_t num_levels; /* 1: UNet; >1: NestedUNet, levels[0] outermost (nested_unet.py:96-160) */
  mdm_level_cfg levels[MDM_MAX_LEVELS];
  int32_t in_channels, out_channels;
  int32_t lm_dim;      /* width of lm_outputs */
  int32_t cond_dim;    /* width seen by cross-attention (conditioning_feature_proj_dim when projecting) */
  int32_t has_lm_proj; /* unet.py:760-765 */
  int32_t has_cond_emb;
  int32_t masked_cross_attention;
  int32_t num_heads; /* 8 (unet.py:245) */
  /* UNetConfig.num_lm_head_layers of the innermost level: SelfAttention1DBlock layers over the conditioning tokens
   * after lm_proj (unet.py:766-771,849-853); needs has_cond_emb */
  int32_t num_lm_head_layers;
} mdm_net_cfg;

typedef struct mdm_net mdm_net;

int mdm_net_create(const mdm_net_cfg* cfg, mdm_net** out);
void mdm_net_destroy(mdm_net* net);

/* Parameter table: same names and shapes as the reference module's state_dict() (OIHW fp32). */
int mdm_net_num_params(const mdm_net* net);
int mdm_net_param_info(const mdm_net* net, int index, const char** name, int32_t* ndim, int64_t shape[4]);
/* Bind caller-owned fp32 storage. grad may be NULL (no gradient wanted); gradients are ACCUMULATED
 * (+=) into it by mdm_net_backward.  Pointers are borrowed until rebound. */
int mdm_net_bind_param(mdm_net* net, const char* name, void* weight, void* grad);
/* Tell the engine the fp32 weights changed (optimizer step / load): fp16 operand copies are rebuilt
 * at the next forward. */
int mdm_net_weights_changed(mdm_net* net);

typedef struct mdm_net_io {
  int32_t batch;
  int32_t tokens;
  int32_t res[MDM_MAX_LEVELS];      /* image height per level, outermost (largest) first; width: res_w */
  const float* x_t[MDM_MAX_LEVELS]; /* NCHW fp32, (batch, in_channels, res, res_w) */
  const int64_t* times;             /* (batch,) */
  const float* lm;                  /* (batch, tokens, lm_dim) fp32 */
  const float* lm_mask;             /* (batch, tokens) fp32 0/1, or NULL */
  const float* micro_scale;         /* (batch,) fp32 or NULL => per-level default (unet.py:924): the key "scale" */
  float* out[MDM_MAX_LEVELS];       /* NCHW fp32 predictions, same shapes as x_t */
  int32_t save_for_backward;
  /* Mixed-resolution batches (NestedDiffusionConfig.mixed_ratio, diffusion.py:262-274; nested_unet.py:180,
   * 193-204,209): level l processes only the FIRST level_batch[l] samples (0 => batch). Must not decrease from
   * outer to inner levels and the innermost level runs the whole batch; x_t[l] / out[l] / dout[l] then hold
   * level_batch[l] samples. Where an outer level is narrower than its inner one the in_adapter output is
   * zero-padded and only the leading rows of the out_adapter result are used, as in the reference. */
  int32_t level_batch[MDM_MAX_LEVELS];
  /* 1: lm is the raw encoder output and is multiplied by lm_mask on the way in (what language_models/factory.py:101
   * does as a separate (B,S,D) pass before the model is called); needs lm_mask and the lm_proj layer. */
  int32_t apply_lm_mask;
  /* Image width per level (0 => res[l], a square image). Both sides must divide by the level's downsampling
   * 2^(num_res - 1), and the bottleneck of an outer level must equal the next level's (res, res_w). */
  int32_t res_w[MDM_MAX_LEVELS];
  /* DiffusionConfig.model_output_scale (diffusion.py:83-85): s != 0 returns s * tanh(out / s) at every level, and
   * the backward multiplies the incoming output gradient by 1 - (out / s)^2. 0 = off. */
  float output_scale;
  /* Operand precision of the weight products (what torch autocast asks of the reference's convs and linears, whose
   * operands it rounds to bf16 / fp16). 0: weights enter every product as two fp16 planes, hi = fp16(w) and
   * lo = fp16(w - hi), ~22 significant bits, and the ResNet data gradients that feed a GroupNorm backward as two planes
   * too. 1: the hi planes only (11 bits; bf16 keeps 8): the weight products skip the B lo plane, the ResNet data
   * gradients their A lo plane, and a weight refresh repacks the hi planes only (the lo planes are refilled before the
   * next call with 0). The backward runs in the mode of its forward. */
  int32_t single_plane;
  /* 1: apply each level's ResNet dropout (the module is in training mode; independent of save_for_backward).
   * Element i of the [level_batch][H][W][C] output of a ResNet's SiLU(norm2) is kept when Philox4x32-10 with
   * key = dropout_seed and counter = (i / 4, stream id) gives a word w (word i % 4) with w / 2^32 >= p; the stream id
   * is the mdm_net_param_info index of that ResNet's conv2.weight. mdm_op_dropout_mask rebuilds a mask. The backward
   * regenerates the masks of the forward it follows. */
  int32_t dropout;
  uint64_t dropout_seed;
} mdm_net_io;

/* CUDA-graph execution of forward / backward (off by default). With it on, the first call with a given shape
 * signature (batch, per-level batch, per-level height and width, tokens, mask presence, which micro keys have
 * values, save_for_backward, dropout, output_scale, single_plane, stage,
 * cond_cache, cond_emb presence; stage-1 calls always run eagerly) runs
 * eagerly, the
 * second is captured and later ones replay the captured graphs: inputs / output gradients are copied into static
 * buffers, ONE graph launch runs the ~1-2.5 k kernels of the pass, outputs are copied out. Gradient-ready
 * notifications (mdm_net_set_grad_ready) keep working: the backward is then recorded as one graph per reported range
 * and fn is called between the segment launches. Rebinding parameters or gradients drops the recorded graphs. */
int mdm_net_set_graph_mode(mdm_net* net, int enable);
/* Number of graph launches issued by this library since load; kernels inside replayed graphs are included in
 * mdm_launch_count(). */
unsigned long long mdm_graph_launch_count(void);

/* SMs to leave to a concurrently running collective (process-wide; 0 = none), set beside the overlapped gradient
 * all-reduce (NCCL_MAX_CTAS = sms). The GEMM kernel runs one tile per CTA, so the collective's CTAs get SMs between
 * tiles whatever the value; it is recorded, and kept so that callers need not change. */
int mdm_set_sm_reserve(int sms);

/* UNet.forward / NestedUNet.forward (unet.py:971-987). */
int mdm_net_forward(mdm_net* net, const mdm_net_io* io, mdm_stream_t stream);

/* The split forward: what mdm_net_forward_stage runs beside the mdm_net_io it is given. A zero-initialised struct (or
 * NULL) is mdm_net_forward. */
typedef struct mdm_net_stage_io {
  /* UNet.forward_conditioning / forward_denoising (unet.py:847-865, 935-969; nested_unet.py:165-230) as separate calls.
   * 0: both, as mdm_net_forward always did. 1: conditioning only: lm_proj (with apply_lm_mask), the lm_head layers,
   * the pooled mean (the plain mean with lm_head and unmasked cross-attention, else the masked mean over lm_mask) and
   * cond_emb; writes cond_out and cond_emb_out and nothing else (x_t / times / out are not read). Its backward
   * recomputes the text path from the same inputs, so lm / lm_mask must stay valid until then. 2: denoising only:
   * cond / cond_emb / cross_mask replace the text path; the token LayerNorm and the kv_cond products of the
   * cross-attention blocks (unet.py:263-264,304) belong to this stage. temb = time MLP + cond_emb + micro. */
  int32_t stage;
  float* cond_out;         /* stage 1: (batch, tokens, cond_dim) fp32 */
  float* cond_emb_out;     /* stage 1: (batch, temporal_dim of the innermost level) fp32; unused without cond_emb */
  const float* cond;       /* stage 2: (batch, tokens, cond_dim) fp32 (may be NULL with cond_cache 2) */
  const float* cond_emb;   /* stage 2: (batch, temporal_dim) fp32 or NULL (nothing added to temb) */
  const float* cross_mask; /* stage 2: (batch, tokens) fp32 0/1 key mask of cross-attention, or NULL */
  /* Stage 2 without save_for_backward: reuse of the text encoding across calls, one slot per net.
   * 1: the fp16 K/V every cross-attention block computes from cond are kept in net-owned memory (at fixed addresses,
   * so replayed graphs read them directly). 2: they are read from there; the token LayerNorm and every kv_cond
   * product are skipped and cond is not read. Mode 2 fails (nothing runs) unless a mode-1 call with the same batch,
   * level_batch, tokens and mdm_net_io.single_plane filled the slot and neither mdm_net_weights_changed nor
   * mdm_net_bind_param came since.
   * Whether cond itself is unchanged is the caller's to know. */
  int32_t cond_cache;
} mdm_net_stage_io;
int mdm_net_forward_stage(mdm_net* net, const mdm_net_io* io, const mdm_net_stage_io* stage, mdm_stream_t stream);

/* ---- general micro-conditioning (UNetConfig.micro_conditioning = "LABEL:DEFAULT,LABEL:DEFAULT,...", unet.py:615-629,
 * 920-933). Each level of the nest has its own keys, order and defaults. Per key, in the level's order, the level owns
 * cond_layers.<key>.0 = Linear(td/4, td) and cond_layers.<key>.1 = Linear(td, td), and adds
 *   layer1(silu(layer0(sincos(m * t_emb))))   with m = clamp(v / default, max=1) * default for the key "scale",
 *                                             and m = v * 1000 for every other key
 * to its temb, v being the key's value of the sample or, when absent, the level's default. mdm_net_create is
 * mdm_net_create_micro with the table {"scale": micro_scale_default} at every level that sets has_micro_scale, and the
 * old forward entry points pass mdm_net_io.micro_scale as the value of the key "scale". Unlike the reference, a "scale"
 * default of 0 (0/0 there) is refused. */
#define MDM_MAX_MICRO 8       /* distinct keys of a nest */
#define MDM_MICRO_NAME_LEN 32 /* bytes of a key name, the terminating NUL included */

typedef struct mdm_micro_cfg {
  int32_t num_keys;                              /* distinct keys of the nest: first appearance, outermost level first */
  char names[MDM_MAX_MICRO][MDM_MICRO_NAME_LEN]; /* NUL-terminated, non-empty, distinct */
  int32_t level_num_keys[MDM_MAX_LEVELS];
  int32_t level_keys[MDM_MAX_LEVELS][MDM_MAX_MICRO];   /* indices into names, in the level's order, no repeats */
  float level_defaults[MDM_MAX_LEVELS][MDM_MAX_MICRO]; /* the level's default of each of its keys */
} mdm_micro_cfg;

/* cfg must not set has_micro_scale at any level: the table says everything about micro-conditioning. */
int mdm_net_create_micro(const mdm_net_cfg* cfg, const mdm_micro_cfg* micro, mdm_net** out);

typedef struct mdm_net_micro_io {
  /* values[k]: (batch,) fp32 values of the table's key k, or NULL => each level's default. Level l reads the leading
   * level_batch[l] rows. */
  const float* values[MDM_MAX_MICRO];
} mdm_net_micro_io;

/* mdm_net_forward_stage (stage NULL: mdm_net_forward) with the values of the micro table's keys (micro NULL: every key
 * takes its default). io->micro_scale must be NULL. Stage-1 forwards read no micro values. */
int mdm_net_forward_micro(mdm_net* net, const mdm_net_io* io, const mdm_net_stage_io* stage,
                          const mdm_net_micro_io* micro, mdm_stream_t stream);

typedef struct mdm_net_grad_io {
  const float* dout[MDM_MAX_LEVELS]; /* d loss / d out[l], NCHW fp32; NULL => zero */
  /* split forward (mdm_net_stage_io.stage). 1: differentiate the last stage-1 forward with save_for_backward=1; otherwise
   * the last stage-0 / stage-2 one. Each keeps its own saved state, so the two backwards may run in either order. */
  int32_t stage;
  float* dcond;              /* stage 2 out: d loss / d cond (batch, tokens, cond_dim) fp32, overwritten; or NULL */
  float* dcond_emb;          /* stage 2 out: d loss / d cond_emb (batch, temporal_dim) fp32, overwritten; or NULL */
  const float* dcond_in;     /* stage 1 in: d loss / d cond_out, or NULL (zero) */
  const float* dcond_emb_in; /* stage 1 in: d loss / d cond_emb_out, or NULL (zero) */
} mdm_net_grad_io;

/* Backward of the last mdm_net_forward(save_for_backward=1): accumulates parameter gradients. A split backward
 * (stage 1 or 2) reports no gradient-ready ranges: its caller reduces the gradients afterwards. */
int mdm_net_backward(mdm_net* net, const mdm_net_grad_io* gio, mdm_stream_t stream);

/* Overlap of the data-parallel gradient all-reduce with backward (replaces DDP's bucket hooks,
 * reference clis/train_parallel.py:147-154). While mdm_net_backward enqueues its kernels it calls
 * fn(user, lo, hi) on the calling host thread each time another >= min_bytes of gradient memory became
 * final: every bound gradient buffer that lies in the address range [lo, hi) has received its last
 * write (as enqueued on `stream`), so a collective ordered after the current stream position may
 * start on it. Ranges are reported from high addresses to low and never overlap; whatever was not reported
 * (the first backward after create/structure change reports nothing) must be reduced by the caller
 * afterwards. fn == NULL disables the notification. */
typedef void (*mdm_grad_ready_fn)(void* user, void* lo, void* hi);
int mdm_net_set_grad_ready(mdm_net* net, mdm_grad_ready_fn fn, void* user, uint64_t min_bytes);
/* After at least one mdm_net_backward: rank[i] = how late the gradient of parameter i (mdm_net_param_info
 * index) becomes final, as the index of the last backward closure that uses it (0 = final only at the very
 * end, larger = earlier, INT32_MAX = never written). Gradient buffers laid out in ascending rank order
 * make the notification above cover the arena from the top down. Returns -1 before the first backward. */
int mdm_net_grad_order(const mdm_net* net, int32_t* rank, int32_t n);

/* Device bytes currently reserved by the engine's pool / its high-water mark of live bytes. */
uint64_t mdm_net_workspace_bytes(const mdm_net* net);
uint64_t mdm_net_workspace_high_water(const mdm_net* net);
/* Debug: copy a named fp32 intermediate of the last forward (e.g. "down_blocks.0.0") to dst.
 * Returns its element count, or negative if unknown. Layout NHWC. "cond_kv" copies the valid K/V cache
 * (mdm_net_stage_io.cond_cache) as raw fp16 bits, two per float, in the cache's block-major layout. */
int64_t mdm_net_debug_fetch(mdm_net* net, const char* name, float* dst, int64_t max_elems, mdm_stream_t stream);


/* ---------------------------------------------------------------- post-backward sweep (SURVEY.md 8f)
 * Replaces, in one pass over the flat gradient arena, the reference's
 *   nn.utils.clip_grad_norm_(model.parameters(), clip)      ml_mdm/trainer.py:78-80
 *   optimizer.step()  (torch.optim.Adam / AdamW)            ml_mdm/trainer.py:81, clis/train_parallel.py:122-134
 *   ema_model.update(vision_model)                          ml_mdm/trainer.py:82-85, models/model_ema.py:25-34
 *   optimizer.zero_grad()                                   ml_mdm/trainer.py:92-93
 * All pointers are device fp32. */

/* One contiguous run of parameters (a tensor or a slice of one). ema may be NULL. */
typedef struct mdm_opt_chunk {
  float* p;   /* parameter values, updated in place */
  float* g;   /* gradient (read; overwritten with 0 when zero_grad, else with the scaled/clipped value) */
  float* m;   /* Adam exp_avg */
  float* v;   /* Adam exp_avg_sq */
  float* ema; /* EMA copy of p, or NULL */
  int64_t n;  /* elements */
} mdm_opt_chunk;

typedef struct mdm_adam_cfg {
  /* hyper-parameters as the doubles torch holds them: the float constants the kernels use (1 - beta, lr / (1 -
   * beta1^step), sqrt(1 - beta2^step), 1 - lr * wd, 1 - ema_decay) are derived in double first, like torch does */
  double lr, beta1, beta2, eps, weight_decay;
  double ema_decay;    /* effective decay of this EMA update: (counter >= warmup) * decay (model_ema.py:26) */
  float grad_scale;    /* gradients are multiplied by this first (1/world, 1/accumulation, ...) */
  float max_norm;      /* clip_grad_norm_ threshold on the scaled gradients; <= 0 disables clipping */
  int32_t adamw;       /* 0: Adam (L2 added to the gradient), 1: AdamW (decoupled decay) */
  int32_t step;        /* 1-based step count of this update (bias corrections 1 - beta^step) */
  int32_t zero_grad;   /* 1: leave the gradients zeroed (the next backward needs no memset) */
} mdm_adam_cfg;

#define MDM_GRAD_NORM_SCRATCH 1184 /* doubles of scratch mdm_grad_norm needs */
/* out_norm[0] = grad_scale * sqrt(sum grads[i]^2) over the n elements (gaps of the arena must be zero), left on
 * the device; deterministic (fixed reduction tree, fp64 partial sums). */
int mdm_grad_norm(const float* grads, int64_t n, float grad_scale, double* scratch, int32_t scratch_elems,
                  float* out_norm, mdm_stream_t stream);
/* chunks_dev: device array of nchunks descriptors (one CTA each; keep n <= ~64K per chunk). norm_dev is the
 * value written by mdm_grad_norm (may be NULL when max_norm <= 0). Element formulas follow
 * torch/optim/adam.py::_single_tensor_adam, torch/nn/utils/clip_grad.py and ModelEma.update op for op. */
int mdm_adam_ema_sweep(const mdm_opt_chunk* chunks_dev, int32_t nchunks, const mdm_adam_cfg* cfg,
                       const float* norm_dev, mdm_stream_t stream);


/* ---------------------------------------------------------------- diffusion algebra (NCHW fp32) */
/* gammas: device fp32 table of num_diffusion_steps+1 entries (Sampler.gammas, samplers.py:201-231),
 * for nested pipelines the per-level shifted table (samplers.py:255-264,613-623).
 * prediction/loss types use the values of samplers.PredictionType: DDPM=3, DDIM=4, V_PREDICTION=5. */

/* x_t = sqrt(g) * (x / image_div) + sqrt(1-g) * eps with g = gammas[t[b] + t_offset]  (samplers.py:244-246) */
int mdm_q_sample(const float* x, const float* eps, const int64_t* t, const float* gammas, int t_offset,
                 float image_div, float* x_t, int batch, int64_t per_sample, mdm_stream_t stream);
/* Input side of the path (SURVEY.md 8f rank 3; clis/train_parallel.py:193-199): the data loader hands over uint8 NHWC
 * images and the trainer computes images = (x.float() - 127) / 128, permuted to NCHW, before get_loss noises them.
 * One pass: x (batch, channels, H, W) fp32 = (u8 - 127) / 128 and, when x_t != NULL, x_t = q-sample of it as
 * mdm_q_sample does. images_u8: (batch, H, W, channels). */
int mdm_q_sample_u8(const uint8_t* images_u8, const float* eps, const int64_t* t, const float* gammas, int t_offset,
                    float image_div, float* x, float* x_t, int batch, int channels, int height, int width,
                    mdm_stream_t stream);
/* loss[b] += weight * mean_chw (pred_for_training - target)^2 with g = gammas[t[b] + 1]
 * (diffusion.py:123-136,160-168; samplers.py:266-279). loss must be zero-initialised by the caller.
 * pred_out / tgt_out (optional) receive the converted prediction and the target. */
int mdm_loss_fwd(const float* model_out, const float* x_t, const float* x, const float* eps, const int64_t* t,
                 const float* gammas, int prediction_type, int loss_type, float image_div, float weight,
                 float* loss, float* pred_out, float* tgt_out, int batch, int64_t per_sample, mdm_stream_t stream);
/* d loss / d model_out given dloss (batch,) */
int mdm_loss_bwd(const float* model_out, const float* x_t, const float* x, const float* eps, const int64_t* t,
                 const float* gammas, int prediction_type, int loss_type, float image_div, float weight,
                 const float* dloss, float* dmodel_out, int batch, int64_t per_sample, mdm_stream_t stream);
/* Sampler.get_prediction_xt_last (samplers.py:281-345) for one level: g = gammas[t_index],
 * g_last = gammas[s_index]. use_ddim=0: DDPM posterior mean (ddim_eta is None). x0_out optional. */
int mdm_sampler_step(const float* x_t, const float* pred, const float* noise, const float* gammas, int t_index,
                     int s_index, int prediction_type, int clip, float image_scale, int use_ddim, float ddim_eta,
                     int need_noise, float* x0_out, float* x_s_out, int64_t numel, mdm_stream_t stream);
/* Dynamic thresholding, Sampler._threshold_sample / clip_sample (samplers.py:461-508), DYNAMIC = (0.995, 100),
 * DYNAMIC_IF = (0.95, 1.5): bound[b] = clamp(quantile(|x0 * image_scale|, ratio), 1, max_value) over sample b's
 * per_sample values, x0 recomputed from (x_t, pred, g = gammas[t_index]); exact order statistics (radix select) combined
 * with torch.quantile's fp32 rank / lerp arithmetic. bound: (batch,) fp32, device. */
int mdm_dynamic_threshold(const float* x_t, const float* pred, const float* gammas, int t_index, int prediction_type,
                          float image_scale, float ratio, float max_value, float* bound, int batch, int64_t per_sample,
                          mdm_stream_t stream);
/* mdm_sampler_step with x0 = clamp(x0 * image_scale, -bound[b], bound[b]) / bound[b] / image_scale. */
int mdm_sampler_step_dynamic(const float* x_t, const float* pred, const float* noise, const float* gammas, int t_index,
                             int s_index, int prediction_type, const float* bound, float image_scale, int use_ddim,
                             float ddim_eta, int need_noise, float* x0_out, float* x_s_out, int batch, int64_t per_sample,
                             mdm_stream_t stream);
/* classifier-free guidance: out = uncond + w * (cond - uncond)  (samplers.py:449-455) */
int mdm_cfg_combine(const float* uncond, const float* cond, float guidance_scale, float* out, int64_t numel,
                    mdm_stream_t stream);
/* F.avg_pool2d(x, ratio) over `planes` = batch*channels images of H x W  (diffusion.py:346) */
int mdm_avg_pool(const float* x, float* y, int planes, int H, int W, int ratio, mdm_stream_t stream);
/* y = clip(x * scale, -1, 1) if clip else x * scale  (Sampler._postprocess, samplers.py:580-599) */
int mdm_clip_scale(const float* x, float scale, int clip, float* y, int64_t numel, mdm_stream_t stream);


/* ---------------------------------------------------------------- fused attention (single operator, for tests)
 * SelfAttention.attention of both branches (models/unet.py:276-294,300-307): qkv16 (B*T, 3C) fp16 = [q|k|v]
 * channel thirds, kv16 (B*S, 2C) fp16 = [k_c|v_c] or NULL, mask (B,S) fp32 or NULL.
 * h16 (B*T, C) = softmax(qk^T/sqrt d) v + softmax(qk_c^T/sqrt d) v_c.  stats (B,heads,2,T,2) fp32 and
 * oself16 are the forward's residue for the backward (may be NULL for inference). */
int mdm_op_attention_fwd(const void* qkv16, const void* kv16, const float* mask, int B, int T, int S, int C, int heads,
                         void* h16, void* oself16, float* stats, mdm_stream_t stream);
/* Backward: dO16 (B*T, C) -> dqkv16 (B*T, 3C) and dkv16 (B*S, 2C). Dterm (B,heads,2,T) and dq32 (B*T, C) are
 * fp32 scratch. */
int mdm_op_attention_bwd(const void* qkv16, const void* kv16, const float* mask, const void* dO16, const void* h16,
                         const void* oself16, const float* stats, int B, int T, int S, int C, int heads, float* Dterm,
                         float* dq32, void* dqkv16, void* dkv16, mdm_stream_t stream);

/* ---------------------------------------------------------------- ResNet dropout mask (single operator, for tests)
 * out_f32[i] (i < n) = the factor the fused GroupNorm kernels apply to element i of a ResNet with this stream id under
 * this seed (mdm_net_io.dropout): 1/(1-p) when kept, else 0 (always 0 for p == 1). p in [0, 1]. */
int mdm_op_dropout_mask(uint64_t seed, uint32_t stream_id, int64_t n, float p, float* out_f32, mdm_stream_t stream);

/* ---------------------------------------------------------------- token self-attention (single operator, for tests)
 * SelfAttention1D.attention of the lm_head layers (models/unet.py:350-375): qkv16 (B*T, 3D) fp16 = [q|k|v] thirds,
 * `heads` heads of d = D/heads columns (d a multiple of 8, 8 <= d <= 256), key mask (B,T) fp32 0/1 or NULL.
 * o16 (B*T, D) = softmax(qk^T/sqrt d, masked keys -inf) v; stats (B,heads,T,2) fp32 is the residue for the backward
 * (may be NULL for inference). A sample whose keys are all masked gets zero output rows and zero gradients. */
int mdm_op_token_attention_fwd(const void* qkv16, const float* mask, int B, int T, int D, int heads, void* o16,
                               float* stats, mdm_stream_t stream);
/* Backward: dO16 (B*T, D) -> dqkv16 (B*T, 3D). Dterm (B,heads,T) and dq32 (B*T, D) are fp32 scratch. */
int mdm_op_token_attention_bwd(const void* qkv16, const float* mask, const void* dO16, const void* o16,
                               const float* stats, int B, int T, int D, int heads, float* Dterm, float* dq32,
                               void* dqkv16, mdm_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* MDM_B200_H_ */
