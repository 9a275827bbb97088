// The (nested) U-Net denoiser on the engine: forward with a recorded tape, backward by replaying it.
//
// Structure and arithmetic follow the reference modules (ml-mdm-matryoshka/ml_mdm/):
//   UNet.__init__ / forward_denoising        models/unet.py:581-773, 935-969
//   ResNet.forward                            models/unet.py:223-238
//   SelfAttention.forward / attention         models/unet.py:276-313
//   ResNetBlock.forward                       models/unet.py:534-576
//   NestedUNet.forward_denoising              models/nested_unet.py:168-230
// but nothing of their code structure is kept: activations are NHWC, every contraction runs on
// the wgmma engine in fp16 x fp16 -> fp32, GroupNorm/FiLM/SiLU/concat live in the pass that
// produces a conv's operand, and gradients come from an explicit tape (the reference uses autograd).
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <memory>

#include <algorithm>

#include "engine.cuh"
#include "mdm_b200.h"

namespace mdm {

unsigned long long g_graph_launches = 0;

// what one forward call is given: the io, the split-forward fields beside it (mdm_net_forward_stage) and the values of
// the micro-conditioning keys (mdm_net_forward_micro; mdm_net_io.micro_scale is moved to the key "scale" on entry)
struct StepIO : mdm_net_io, mdm_net_stage_io, mdm_net_micro_io {};
static_assert(kMaxMicroKeys == MDM_MAX_MICRO, "MicroKeys holds one level's keys");

namespace {

struct ResSpec {
  std::string pre;
  int cin, cout;
  int film_off;  // column of this ResNet's (ta|tb) in the level's FiLM matrix
};
struct AttnSpec {
  std::string pre;
  int C;
  bool cond, ffn;
  float* kv_bias_fold = nullptr;  // W b_ln + bias of kv_cond with the LayerNorm affine folded in (persistent)
  long long kv_col = 0;            // offset of this block's K/V in the cache, in units of batch * tokens (Net::kv_cache)
};
struct BlockSpec {
  std::string pre;
  std::vector<ResSpec> res;
  std::vector<AttnSpec> attn;  // nattn per resnet, index i * nattn + j
  int nattn = 0;
  bool cond = false, down = false, up = false;
};
struct LevelSpec {
  std::string pre;
  mdm_level_cfg c;
  std::vector<BlockSpec> down, mid, up;
  int film_total = 0;
  int feat_ch = 0;
  bool innermost = false;
  // micro-conditioning keys in the level's order: "<pre>cond_layers.<key>", the key's index in the net's table
  // (mdm_net_micro_io.values) and its default / transform (values are bound per step)
  std::vector<std::string> micro_pre;
  std::vector<int> micro_slot;
  MicroKeys micro{};
  // persistent packed time-layer operands
  __half* tl_w16 = nullptr;  // [film_total][td]
  float* tl_bias = nullptr;  // [film_total]
};

int round8(int x) { return (x + 7) / 8 * 8; }

}  // namespace

struct Net {
  mdm_net_cfg cfg;
  mdm_micro_cfg micro{};  // the nest's micro-conditioning table (mdm_net_create_micro)
  int scale_slot = -1;    // index of the key "scale" in it, -1 if absent: where mdm_net_io.micro_scale goes
  std::vector<LevelSpec> levels;
  std::vector<Param> plist;
  std::unordered_map<std::string, int> pindex;
  Engine eng;
  bool weights_dirty = true;
  // the lo planes of the packed weights lag the fp32 masters: a single-plane pass repacked only the hi planes
  bool lo_stale = false;
  bool fused_attention = getenv("MDM_UNFUSED_ATTENTION") == nullptr;
  bool have_tape = false;
  std::vector<void*> persistent;  // cudaMalloc'd for the life of the net
  std::unordered_map<std::string, Act*> debug_acts;

  // ---- split forward (mdm_net_stage_io.stage)
  int tape_stage = 0;          // stage (0 or 2) of the forward whose tape is held
  bool tape_single = false;    // plane mode (mdm_net_io.single_plane) of that forward: its backward runs in it too
  Pool text_pool;              // workspace of the stage-1 passes, which run beside a held stage-0/2 tape
  bool have_cond_io = false;   // a stage-1 forward with save_for_backward ran: its backward recomputes from cond_io
  StepIO cond_io{};
  // K/V cache of the cross-attention blocks (mdm_net_stage_io.cond_cache): block a's dense (batch * tokens, 2C) fp16 [k_c|v_c]
  // starts at element a.kv_col * batch * tokens (kv_row = sum of 2C); valid for the (batch, tokens, level batches) it
  // was filled with
  long long kv_row = 0;
  __half* kv_cache = nullptr;
  size_t kv_cap = 0;           // elements allocated
  uint64_t kv_epoch = 0;       // bumped on reallocation: graphs that read or write the cache record it
  bool kv_valid = false;
  int kv_key[2 + MDM_MAX_LEVELS] = {0, 0, 0, 0, 0, 0};
  bool kv_single = false;      // plane mode of the forward that filled it

  // per-step state
  struct CondStep {
    int B = 0, S = 0, cd = 0;
    const float* lm = nullptr;
    const float* mask = nullptr;       // pooling mask
    const float* cross_mask = nullptr; // mask for cross-attention (null when masked_cross_attention == 0)
    __half* lm16 = nullptr;
    float* cond32 = nullptr;  // (B*S, cd)
    float* dcond = nullptr;
    bool dcond_init = false;
    float* y32 = nullptr;
    __half* y16 = nullptr;
    __half* xhat16 = nullptr;  // LayerNorm(cond) without affine, shared by every cross-attention block
    float* lnstats = nullptr;  // (B*S, 2) mean, rstd
    float* dxhat = nullptr;    // gradient w.r.t. xhat, accumulated over the blocks
    bool dxhat_init = false;
    float* cemb = nullptr;  // (B, td)
    float* dcemb = nullptr;
    bool dcemb_init = false;
    int kv_mode = 0;  // stage 2: mdm_net_stage_io.cond_cache
  } cs;
  struct LevelStep {
    float* temb = nullptr;      // (B, td) fp32
    __half* stemb16 = nullptr;  // silu(temb)
    float* film = nullptr;      // (B, film_total)
    float* dstemb = nullptr;
    bool dstemb_init = false;
  };
  std::deque<LevelStep> lsteps;
  const StepIO* io = nullptr;
  struct OutRec {
    float* nhwc = nullptr;  // [pix][out_ch]
    __half* d16 = nullptr;  // [pix][8] scaled gradient (filled by backward)
    int h = 0, w = 0;
    int batch = 0;
    float scale = 0.f;      // model_output_scale of the forward; != 0: y holds its NCHW output s * tanh(o / s)
    float* y = nullptr;
  } outs[MDM_MAX_LEVELS];
  // samples level li processes (mixed-resolution batches run only a leading part of the batch on outer levels)
  int level_batch(int li) const {
    const int b = io->level_batch[li];
    return b > 0 ? b : io->batch;
  }
  static int width_of(const mdm_net_io* q, int l) { return q->res_w[l] > 0 ? q->res_w[l] : q->res[l]; }

  ~Net() {
    for (cudaEvent_t e : eng.events) cudaEventDestroy(e);
    if (eng.side != nullptr) cudaStreamDestroy(eng.side);
    for (auto& r : graphs) free_rec(r);
    if (cap_st != nullptr) cudaStreamDestroy(cap_st);
    for (void* p : persistent) cudaFree(p);
    cudaFree(kv_cache);
  }

  // ---------------------------------------------------------------- parameters
  void add_param(const std::string& name, std::vector<int64_t> shape, int pack) {
    Param p;
    p.name = name;
    p.shape = shape;
    p.numel = 1;
    for (auto d : shape) p.numel *= d;
    p.pack = pack;
    pindex[name] = static_cast<int>(plist.size());
    plist.push_back(p);
  }
  // ---- gradient-ready notification (mdm_net_set_grad_ready): which parameters each tape closure looks
  // up is learned from earlier replays; while replaying, the addresses above the highest gradient any
  // remaining closure may still touch are final and are reported so the caller can start reducing them.
  mdm_grad_ready_fn ready_fn = nullptr;
  void* ready_user = nullptr;
  size_t ready_min_bytes = 0;
  std::vector<std::vector<int>> learned;  // per closure (tape order): parameter indices seen during replay
  int replay_idx = -1;                    // closure being replayed, -1 outside backward
  std::vector<int> cur_lookup;
  uintptr_t final_lo = UINTPTR_MAX;       // gradient addresses >= final_lo were reported final

  Param& P(const std::string& name) {
    auto it = pindex.find(name);
    if (it == pindex.end()) throw MdmFail("unknown parameter " + name);
    Param& p = plist[it->second];
    if (p.w == nullptr) throw MdmFail("parameter not bound: " + name);
    if (replay_idx >= 0) {
      cur_lookup.push_back(it->second);
      if (p.g != nullptr && reinterpret_cast<uintptr_t>(p.g) >= final_lo)
        throw MdmFail("gradient of " + name + " was reported ready before its last use in backward");
    }
    return p;
  }
  void* persist(size_t bytes) {
    void* p = nullptr;
    MDM_CUDA(cudaMalloc(&p, bytes));
    persistent.push_back(p);
    return p;
  }
  // an fp16 weight copy of n elements as two planes [hi | lo] (Engine::weight_planes); returns the hi plane
  __half* persist_w16(size_t n) {
    const size_t plane = (n + 63) / 64 * 64;  // keeps the lo plane of every view as aligned as its hi plane
    auto* p = static_cast<__half*>(persist(sizeof(__half) * 2 * plane));
    eng.add_weight_planes(p, plane);
    return p;
  }
  // Fills the lo plane of a packed copy: the packer applied to the fp16 rounding residual of the fp32 master, written
  // to the lo-plane address of `hi` (packers only copy, permute or zero, so the residual packs like the weight).
  template <typename Packer>
  void pack_lo(const float* w, long long numel, const __half* hi, Packer&& packer) {
    float* r = eng.alloc<float>(numel);
    f16_residual(w, r, numel, eng.st);
    packer(r, const_cast<__half*>(eng.lo_plane(hi)));
    eng.rel(r);
  }

  void add_resnet(const ResSpec& r, int td) {
    add_param(r.pre + ".norm1.weight", {r.cin}, 0);
    add_param(r.pre + ".norm1.bias", {r.cin}, 0);
    add_param(r.pre + ".conv1.weight", {r.cout, r.cin, 3, 3}, 2);
    add_param(r.pre + ".conv1.bias", {r.cout}, 0);
    add_param(r.pre + ".time_layer.weight", {2 * r.cout, td}, 4);  // packed into the level's FiLM matrix
    add_param(r.pre + ".time_layer.bias", {2 * r.cout}, 0);
    add_param(r.pre + ".norm2.weight", {r.cout}, 0);
    add_param(r.pre + ".norm2.bias", {r.cout}, 0);
    add_param(r.pre + ".conv2.weight", {r.cout, r.cout, 3, 3}, 2);
    add_param(r.pre + ".conv2.bias", {r.cout}, 0);
    if (r.cin != r.cout) {
      add_param(r.pre + ".conv3.weight", {r.cout, r.cin, 1, 1}, 1);
      add_param(r.pre + ".conv3.bias", {r.cout}, 0);
    }
  }
  void add_attn(const AttnSpec& a) {
    const int C = a.C;
    add_param(a.pre + ".norm.weight", {C}, 0);
    add_param(a.pre + ".norm.bias", {C}, 0);
    add_param(a.pre + ".qkv.weight", {3 * C, C, 1, 1}, 1);
    add_param(a.pre + ".qkv.bias", {3 * C}, 0);
    if (a.cond) {
      add_param(a.pre + ".norm_cond.weight", {cfg.cond_dim}, 0);
      add_param(a.pre + ".norm_cond.bias", {cfg.cond_dim}, 0);
      add_param(a.pre + ".kv_cond.weight", {2 * C, cfg.cond_dim}, 5);  // packed with norm_cond folded in
      add_param(a.pre + ".kv_cond.bias", {2 * C}, 0);
    }
    add_param(a.pre + ".proj_out.weight", {C, C, 1, 1}, 1);
    add_param(a.pre + ".proj_out.bias", {C}, 0);
    if (a.ffn) {
      add_param(a.pre + ".ffn.0.weight", {C}, 0);
      add_param(a.pre + ".ffn.0.bias", {C}, 0);
      add_param(a.pre + ".ffn.1.weight", {4 * C, C, 1, 1}, 1);
      add_param(a.pre + ".ffn.1.bias", {4 * C}, 0);
      add_param(a.pre + ".ffn.3.weight", {C, 4 * C, 1, 1}, 1);
      add_param(a.pre + ".ffn.3.bias", {C}, 0);
    }
  }
  void add_block(LevelSpec& L, BlockSpec& b, int td) {
    for (size_t i = 0; i < b.res.size(); ++i) {
      b.res[i].film_off = L.film_total;
      L.film_total += 2 * b.res[i].cout;
      add_resnet(b.res[i], td);
    }
    for (auto& a : b.attn) add_attn(a);
    if (b.down || b.up) {
      const int C = b.res.back().cout;
      add_param(b.pre + ".resample.weight", {C, C, 3, 3}, 2);
      add_param(b.pre + ".resample.bias", {C}, 0);
    }
  }

  // Mirrors the bookkeeping of UNet.__init__ (unet.py:631-747): channel/skip arithmetic only.
  // the micro table of mdm_net_create_micro: well-formed names, per-level keys and defaults
  void check_micro() {
    MDM_CHECK(micro.num_keys >= 0 && micro.num_keys <= MDM_MAX_MICRO, "mdm_micro_cfg.num_keys must lie in [0, MDM_MAX_MICRO]");
    for (int k = 0; k < micro.num_keys; ++k) {
      const char* nm = micro.names[k];
      MDM_CHECK(memchr(nm, 0, MDM_MICRO_NAME_LEN) != nullptr && nm[0] != 0,
                "micro-conditioning key names must be non-empty and shorter than MDM_MICRO_NAME_LEN");
      for (int j = 0; j < k; ++j)
        if (strcmp(nm, micro.names[j]) == 0) throw MdmFail(std::string("micro-conditioning key '") + nm + "' is listed twice");
      if (strcmp(nm, "scale") == 0) scale_slot = k;
    }
    for (int li = 0; li < cfg.num_levels; ++li) {
      const int n = micro.level_num_keys[li];
      MDM_CHECK(n >= 0 && n <= micro.num_keys, "mdm_micro_cfg.level_num_keys must lie in [0, num_keys]");
      for (int j = 0; j < n; ++j) {
        const int k = micro.level_keys[li][j];
        MDM_CHECK(k >= 0 && k < micro.num_keys, "mdm_micro_cfg.level_keys must index the table");
        for (int i = 0; i < j; ++i) MDM_CHECK(micro.level_keys[li][i] != k, "a level lists a micro-conditioning key twice");
        const float d = micro.level_defaults[li][j];
        if (!isfinite(d)) throw MdmFail(std::string("micro-conditioning key '") + micro.names[k] + "' has a non-finite default");
        // the reference divides by the default of "scale" (unet.py:926): 0 would give 0/0
        if (k == scale_slot && d == 0.f)
          throw MdmFail("micro-conditioning key 'scale' needs a non-zero default (clamp(v / default, max=1) * default)");
      }
    }
  }

  void build() {
    MDM_CHECK(cfg.num_levels >= 1 && cfg.num_levels <= MDM_MAX_LEVELS, "bad num_levels");
    check_micro();
    MDM_CHECK(cfg.in_channels * 9 <= 32, "conv_in packs 9*Cin into one 32-wide k block");
    std::string pre;
    for (int li = 0; li < cfg.num_levels; ++li) {
      LevelSpec L;
      L.pre = pre;
      L.c = cfg.levels[li];
      L.innermost = (li == cfg.num_levels - 1);
      const mdm_level_cfg& c = L.c;
      const int td = c.temporal_dim;
      const bool cond_here = cfg.cond_dim > 0;
      MDM_CHECK(c.num_res >= 1 && c.num_res <= MDM_MAX_RES, "bad num_res");
      MDM_CHECK(td % 8 == 0, "temporal_dim must be a multiple of 8");
      MDM_CHECK(c.dropout >= 0.f && c.dropout <= 1.f, "dropout must lie in [0, 1]");
      // Parameter registration order follows nn.Module registration order of the reference so that
      // index order == state_dict order.
      add_param(pre + "t_emb", {1, td / 8}, 0);  // non-persistent buffer of the reference (unet.py:600-603)
      add_param(pre + "temb_layer1.weight", {td, td / 4}, 1);
      add_param(pre + "temb_layer1.bias", {td}, 0);
      add_param(pre + "temb_layer2.weight", {td, td}, 1);
      add_param(pre + "temb_layer2.bias", {td}, 0);
      if (L.innermost && cfg.has_cond_emb) add_param(pre + "cond_emb.weight", {td, cfg.cond_dim}, 1);
      MDM_CHECK(!c.has_micro_scale, "has_micro_scale is for mdm_net_create; with mdm_net_create_micro the table says it");
      L.micro.num = micro.level_num_keys[li];
      for (int j = 0; j < L.micro.num; ++j) {
        const int k = micro.level_keys[li][j];
        const std::string cl = pre + "cond_layers." + micro.names[k];
        add_param(cl + ".0.weight", {td, td / 4}, 1);
        add_param(cl + ".0.bias", {td}, 0);
        add_param(cl + ".1.weight", {td, td}, 1);
        add_param(cl + ".1.bias", {td}, 0);
        L.micro_pre.push_back(cl);
        L.micro_slot.push_back(k);
        L.micro.defaults[j] = micro.level_defaults[li][j];
        if (strcmp(micro.names[k], "scale") == 0) L.micro.scale_mask |= 1u << j;
      }
      add_param(pre + "conv_in.weight", {c.channels[0], cfg.in_channels, 3, 3}, 3);
      add_param(pre + "conv_in.bias", {c.channels[0]}, 0);

      int ch = c.channels[0];
      std::vector<int> skips{ch};
      for (int i = 0; i < c.num_res; ++i) {
        BlockSpec b;
        b.pre = pre + "down_blocks." + std::to_string(i);
        b.nattn = c.num_attn[i];
        b.cond = c.cond_level[i] != 0;
        b.down = (i != c.num_res - 1);
        for (int j = 0; j < c.num_resnets[i]; ++j) {
          ResSpec r{b.pre + ".resnets." + std::to_string(j), ch, c.channels[i], 0};
          ch = c.channels[i];
          skips.push_back(ch);
          b.res.push_back(r);
        }
        if (b.down) skips.push_back(ch);
        for (int j = 0; j < c.num_resnets[i] * b.nattn; ++j)
          b.attn.push_back(AttnSpec{b.pre + ".attn." + std::to_string(j), c.channels[i], b.cond && cond_here,
                                    c.use_attention_ffn != 0});
        L.down.push_back(b);
      }
      if (!c.skip_mid_blocks) {
        BlockSpec m0, m1;
        m0.pre = pre + "mid_blocks.0";
        m0.nattn = 1;
        m0.cond = true;
        m0.res.push_back(ResSpec{m0.pre + ".resnets.0", ch, ch, 0});
        m0.attn.push_back(AttnSpec{m0.pre + ".attn.0", ch, cond_here, c.use_attention_ffn != 0});
        m1.pre = pre + "mid_blocks.1";
        m1.res.push_back(ResSpec{m1.pre + ".resnets.0", ch, ch, 0});
        L.mid.push_back(m0);
        L.mid.push_back(m1);
      }
      for (int i = c.num_res - 1; i >= 0; --i) {
        BlockSpec b;
        b.pre = pre + "up_blocks." + std::to_string(c.num_res - 1 - i);
        b.nattn = c.num_attn[i];
        b.cond = c.cond_level[i] != 0;
        b.up = (i != 0);
        for (int j = 0; j < c.num_resnets[i] + 1; ++j) {
          const int sk = skips.back();
          skips.pop_back();
          ResSpec r{b.pre + ".resnets." + std::to_string(j), ch + sk, c.channels[i], 0};
          ch = c.channels[i];
          b.res.push_back(r);
        }
        for (int j = 0; j < (c.num_resnets[i] + 1) * b.nattn; ++j)
          b.attn.push_back(AttnSpec{b.pre + ".attn." + std::to_string(j), c.channels[i], b.cond && cond_here,
                                    c.use_attention_ffn != 0});
        L.up.push_back(b);
      }
      L.feat_ch = ch;
      // register block parameters in module order: down, mid, up
      for (auto& b : L.down) add_block(L, b, td);
      for (auto& b : L.mid) add_block(L, b, td);
      for (auto& b : L.up) add_block(L, b, td);
      add_param(pre + "norm_out.weight", {ch}, 0);
      add_param(pre + "norm_out.bias", {ch}, 0);
      add_param(pre + "conv_out.weight", {cfg.out_channels, ch, 3, 3}, 2);
      add_param(pre + "conv_out.bias", {cfg.out_channels}, 0);
      if (L.innermost && cfg.has_lm_proj) {
        add_param(pre + "lm_proj.weight", {cfg.cond_dim, cfg.lm_dim}, 1);
        add_param(pre + "lm_proj.bias", {cfg.cond_dim}, 0);
      }
      if (L.innermost) {
        MDM_CHECK(cfg.num_lm_head_layers >= 0 && (cfg.num_lm_head_layers == 0 || cfg.has_cond_emb),
                  "lm_head layers exist only beside cond_emb");
        const int D = cfg.cond_dim;
        for (int i = 0; i < cfg.num_lm_head_layers; ++i) {  // SelfAttention1DBlock (unet.py:439-446)
          const std::string h = pre + "lm_head." + std::to_string(i);
          add_param(h + ".attn.norm.weight", {D}, 0);
          add_param(h + ".attn.norm.bias", {D}, 0);
          add_param(h + ".attn.qkv.weight", {3 * D, D}, 1);
          add_param(h + ".attn.qkv.bias", {3 * D}, 0);
          add_param(h + ".attn.proj_out.weight", {D, D}, 1);
          add_param(h + ".attn.proj_out.bias", {D}, 0);
          add_param(h + ".mlp.main.0.weight", {D}, 0);
          add_param(h + ".mlp.main.0.bias", {D}, 0);
          add_param(h + ".mlp.main.1.weight", {4 * D, D}, 1);
          add_param(h + ".mlp.main.1.bias", {4 * D}, 0);
          add_param(h + ".mlp.main.3.weight", {D, 4 * D}, 1);
          add_param(h + ".mlp.main.3.bias", {D}, 0);
        }
      }
      levels.push_back(L);
      pre += "inner_unet.";
    }
    // adapters belong to the outer level of each nesting step (registered after the inner net)
    for (int li = cfg.num_levels - 2; li >= 0; --li) {
      const mdm_level_cfg& o = cfg.levels[li];
      const mdm_level_cfg& in = cfg.levels[li + 1];
      const int co = o.channels[o.num_res - 1], ci = in.channels[0];
      add_param(levels[li].pre + "in_adapter.weight", {ci, co, 3, 3}, 2);
      add_param(levels[li].pre + "in_adapter.bias", {ci}, 0);
      add_param(levels[li].pre + "out_adapter.weight", {co, ci, 3, 3}, 2);
      add_param(levels[li].pre + "out_adapter.bias", {co}, 0);
    }
    MDM_CUDA(cudaMalloc(&eng.d_scale, 3 * sizeof(float)));
    eng.d_inv_scale = eng.d_scale + 1;
    eng.d_amax = eng.d_scale + 2;
    persistent.push_back(eng.d_scale);
    eng.d_drop_seed = static_cast<unsigned long long*>(persist(sizeof(unsigned long long)));
    for (auto& L : levels)
      for (auto* blocks : {&L.down, &L.mid, &L.up})
        for (auto& b : *blocks)
          for (auto& a : b.attn)
            if (a.cond) {
              a.kv_col = kv_row;
              kv_row += 2 * a.C;
            }
  }

  // ---------------------------------------------------------------- weight packing
  // Packs the fp16 operand copies a pass in this plane mode reads. A single-plane pass packs the hi planes and leaves
  // the lo planes stale (still allocated, so addresses baked into captured graphs stay valid); the next two-plane pass
  // packs both again.
  void prepare_weights(bool single) {
    if (!weights_dirty && (single || !lo_stale)) return;
    const bool lo = !single;
    cudaStream_t st = eng.st;
    for (auto& L : levels) {
      if (L.tl_w16 == nullptr && L.film_total > 0) {
        L.tl_w16 = persist_w16(static_cast<size_t>(L.film_total) * L.c.temporal_dim);
        L.tl_bias = static_cast<float*>(persist(sizeof(float) * L.film_total));
      }
    }
    for (auto& p : plist) {
      if (p.pack == 0) continue;
      MDM_CHECK(p.w != nullptr, ("parameter not bound: " + p.name).c_str());
      if (p.pack == 4 || p.pack == 5) continue;  // handled per level / per attention block below
      if (p.w16 == nullptr) {
        size_t n = static_cast<size_t>(p.numel);
        if (p.pack == 3) n = static_cast<size_t>(p.shape[0]) * 32;
        p.w16 = persist_w16(n);
      }
      if (p.pack == 1) {
        cast_f32_to_f16(p.w, p.w16, p.numel, st);
        if (lo) pack_lo(p.w, p.numel, p.w16, [&](const float* r, __half* l) { cast_f32_to_f16(r, l, p.numel, st); });
      } else if (p.pack == 2) {
        const int Co = static_cast<int>(p.shape[0]), Ci = static_cast<int>(p.shape[1]);
        pack_conv_w(p.w, p.w16, Co, Ci, 9, st);
        if (lo) pack_lo(p.w, p.numel, p.w16, [&](const float* r, __half* l) { pack_conv_w(r, l, Co, Ci, 9, st); });
        if (Engine::fold_ok(Ci, Co) && Co % 4 == 0) {  // narrow layer: W-folded copy + doubled bias (engine.cu)
          if (p.w16f == nullptr) {
            p.w16f = persist_w16(36ull * Co * Ci);
            p.bias_f = static_cast<float*>(persist(sizeof(float) * 2ull * Co));
          }
          pack_conv_w_fold(p.w, p.w16f, Co, Ci, st);
          if (lo) pack_lo(p.w, p.numel, p.w16f, [&](const float* r, __half* l) { pack_conv_w_fold(r, l, Co, Ci, st); });
          auto bi = pindex.find(p.name.substr(0, p.name.size() - 6) + "bias");  // "...weight" -> "...bias"
          MDM_CHECK(bi != pindex.end() && plist[bi->second].w != nullptr, "conv bias not bound");
          for (int r = 0; r < 2; ++r)
            MDM_CUDA(cudaMemcpyAsync(p.bias_f + r * Co, plist[bi->second].w, sizeof(float) * Co, cudaMemcpyDeviceToDevice, st));
        }
      }
      else if (p.pack == 3) {
        const int Co = static_cast<int>(p.shape[0]), Ci = static_cast<int>(p.shape[1]);
        pack_conv_in_w(p.w, p.w16, Co, Ci, st);
        if (lo) pack_lo(p.w, p.numel, p.w16, [&](const float* r, __half* l) { pack_conv_in_w(r, l, Co, Ci, st); });
      }
    }
    for (auto& L : levels) {
      const int td = L.c.temporal_dim;
      auto pack_block = [&](BlockSpec& b) {
        for (auto& r : b.res) {
          Param& w = P(r.pre + ".time_layer.weight");
          Param& bb = P(r.pre + ".time_layer.bias");
          w.w16 = L.tl_w16 + static_cast<size_t>(r.film_off) * td;
          cast_f32_to_f16(w.w, w.w16, w.numel, st);
          if (lo) pack_lo(w.w, w.numel, w.w16, [&](const float* r, __half* l) { cast_f32_to_f16(r, l, w.numel, st); });
          MDM_CUDA(cudaMemcpyAsync(L.tl_bias + r.film_off, bb.w, sizeof(float) * 2 * r.cout,
                                   cudaMemcpyDeviceToDevice, st));
        }
      };
      for (auto& b : L.down) pack_block(b);
      for (auto& b : L.mid) pack_block(b);
      for (auto& b : L.up) pack_block(b);
    }
    for (auto& L : levels) {
      auto fold_block = [&](BlockSpec& b) {
        for (auto& a : b.attn) {
          if (!a.cond) continue;
          Param &kw = P(a.pre + ".kv_cond.weight"), &kb = P(a.pre + ".kv_cond.bias");
          Param &lw = P(a.pre + ".norm_cond.weight"), &lb = P(a.pre + ".norm_cond.bias");
          const int rows = 2 * a.C, D = cfg.cond_dim;
          if (kw.w16 == nullptr) kw.w16 = persist_w16(static_cast<size_t>(rows) * D);
          if (a.kv_bias_fold == nullptr) a.kv_bias_fold = static_cast<float*>(persist(sizeof(float) * rows));
          fold_ln_weight(kw.w, lw.w, kw.w16, lo ? const_cast<__half*>(eng.lo_plane(kw.w16)) : nullptr, rows, D, st);
          fold_ln_bias(kw.w, lb.w, kb.w, a.kv_bias_fold, rows, D, st);
        }
      };
      for (auto& b : L.down) fold_block(b);
      for (auto& b : L.mid) fold_block(b);
      for (auto& b : L.up) fold_block(b);
    }
    weights_dirty = false;
    lo_stale = single;
  }

  // ---------------------------------------------------------------- small building blocks
  const float* inv_scale() const { return eng.d_inv_scale; }

  // y = x W^T + b backward. dy16: fp16 gradient (M x N). Accumulates W.g / b.g; optional dx.
  void linear_bwd(const __half* dy16, long long ldy, int M, int N, int K, const __half* x16, long long ldx,
                  Param& W, Param* b, bool bias_from_f16, float* dx32, int acc_dx) {
    if (b != nullptr && b->g != nullptr && bias_from_f16) {
      MDM_CHECK(ldy == N, "colsum needs dense rows");
      colsum_f16(dy16, M, N, b->g, inv_scale(), eng.st);
    }
    if (W.g != nullptr) {
      eng.side_begin();
      Epi e;
      e.out_f32 = W.g;
      e.alpha_dev = inv_scale();
      e.atomic_ok = true;
      eng.gemm_tn(dy16, ldy, x16, ldx, N, K, M, e);
      eng.side_end();
    }
    if (dx32 != nullptr) {
      Epi e;
      e.out_f32 = dx32;
      if (acc_dx) e.residual = dx32;
      eng.gemm_nn(dy16, ldy, W.w16, K, M, K, N, e);
    }
  }

  // 3x3 weight gradient into w.g (+=): folded form for the narrow layers (engine.cu), else the plain one.
  // wtmp must hold 36 * cin * cout floats.
  void conv_wgrad_into(const __half* dy16, int ldy, const __half* x16, int ldx, int N, int H, int W, int cin, int cout,
                       float* wtmp, Param& w) {
    eng.side_begin();  // beside the data-gradient chain of the same layer (engine.cuh); joined at the end of the closure
    const bool folded = eng.conv3x3_wgrad(dy16, ldy, x16, ldx, N, H, W, cin, cout, wtmp, w.w16f != nullptr);
    if (folded) unpack_conv_wgrad_fold(wtmp, w.g, cout, cin, inv_scale(), eng.st);
    else unpack_conv_wgrad(wtmp, w.g, cout, cin, 9, cin, inv_scale(), eng.st);
    eng.side_end();
  }

  struct GnOut {
    float* sums;
    __half* y16;
    __half* raw16;
  };
  GnOut gn_fwd(const Src2& x, int N, int HW, int G, Param& gw, Param& gb, const float* film, int film_ld,
               int film_off, int silu, bool want_raw, const Dropout& drop = Dropout()) {
    const int C = x.c0 + x.c1;
    MDM_CHECK(C % G == 0 && C % 4 == 0 && x.c0 % 4 == 0, "GroupNorm channel layout");
    GnOut o;
    o.sums = eng.zeros_f32(2ll * N * G);
    gn_stats(x, N, HW, G, o.sums, eng.st);
    o.y16 = eng.alloc<__half>(static_cast<long long>(N) * HW * C);
    o.raw16 = want_raw ? eng.alloc<__half>(static_cast<long long>(N) * HW * C) : nullptr;
    gn_apply(x, N, HW, G, o.sums, gw.w, gb.w, film, film_ld, film_off, silu, o.y16, o.raw16, eng.st, drop);
    return o;
  }
  // Backward through gn_apply. dy: gradient w.r.t. its fp16 output, fp16 (dy_f16) or fp32.
  // Destination: Act gradients dst0/dst1 (accumulating), or -- when h16_out is given -- a plain fp16
  // tensor plus bias-gradient column sums (single consumer, nothing to accumulate).
  void gn_bwd(const Src2& x, const void* dy, bool dy_f16, int N, int HW, int G, const float* sums, Param& gw, Param& gb,
              const float* film, int film_ld, int film_off, int silu, float* dfilm, const float* extra, Act* dst0,
              Act* dst1, __half* h16_out = nullptr, float* colsum = nullptr, __half* h16_lo = nullptr,
              const Dropout& drop = Dropout()) {
    const int C = x.c0 + x.c1;
    float* ab = eng.zeros_f32(2ll * N * C);
    float* pg = eng.alloc<float>(2ll * N * G);
    gn_bwd_reduce(x, dy, dy_f16 ? 1 : 0, N, HW, G, sums, gw.w, gb.w, film, film_ld, film_off, silu, ab, eng.st, drop);
    // dgamma/dbeta always have somewhere to go: when a grad buffer is missing use scratch
    float* dg = gw.g != nullptr ? gw.g : eng.zeros_f32(C);
    float* db = gb.g != nullptr ? gb.g : eng.zeros_f32(C);
    gn_bwd_finalize(N, C, G, HW, ab, gw.w, gb.w, film, film_ld, film_off, pg, dg, db, dfilm, inv_scale(), eng.st);
    Dst2 d{};
    if (h16_out != nullptr) {
      d.h16 = h16_out;
      d.h16lo = h16_lo;
      d.colsum = colsum;
      d.inv_scale = inv_scale();
      d.c0 = C;
    } else {
      int a0 = 0, a1 = 0;
      d.p0 = eng.grad_buf(dst0, &a0);
      d.c0 = x.c0;
      d.acc0 = a0;
      if (dst1 != nullptr) {
        d.p1 = eng.grad_buf(dst1, &a1);
        d.c1 = x.c1;
        d.acc1 = a1;
      }
    }
    gn_bwd_apply(x, dy, dy_f16 ? 1 : 0, N, HW, G, sums, gw.w, gb.w, film, film_ld, film_off, silu, pg, extra, d, eng.st,
                 drop);
    eng.rel(ab);
    eng.rel(pg);
  }

  // ---------------------------------------------------------------- ResNet (unet.py:223-238)
  Act* resnet_fwd(const LevelSpec& L, LevelStep* ls, const ResSpec& r, Act* x, Act* skip) {
    const int N = x->n, H = x->h, W = x->w, HW = H * W;
    const int cin = r.cin, cout = r.cout, G = L.c.groups;
    MDM_CHECK(x->c + (skip ? skip->c : 0) == cin, "resnet input channels");
    Src2 src{x->p, skip ? skip->p : nullptr, x->c, skip ? skip->c : 0};
    Param &n1w = P(r.pre + ".norm1.weight"), &n1b = P(r.pre + ".norm1.bias");
    Param &c1w = P(r.pre + ".conv1.weight"), &c1b = P(r.pre + ".conv1.bias");
    Param &n2w = P(r.pre + ".norm2.weight"), &n2b = P(r.pre + ".norm2.bias");
    Param &c2w = P(r.pre + ".conv2.weight"), &c2b = P(r.pre + ".conv2.bias");
    const bool proj = cin != cout;
    GnOut g1 = gn_fwd(src, N, HW, G, n1w, n1b, nullptr, 0, 0, 1, proj);
    float* h = eng.alloc<float>(static_cast<long long>(N) * HW * cout);
    {
      Epi e;
      e.bias = c1b.w;
      e.out_f32 = h;
      eng.conv3x3_fwd(g1.y16, cin, N, H, W, cin, c1w.w16, cout, e, c1w.w16f, c1w.bias_f);
    }
    Src2 hs{h, nullptr, cout, 0};
    // ResNet.dropout sits between SiLU(norm2) and conv2 (unet.py:233-235); its mask stream is conv2's parameter index
    Dropout drop;
    if (io->dropout && L.c.dropout > 0.f) {
      drop.p = L.c.dropout;
      drop.seed = eng.d_drop_seed;
      drop.stream = static_cast<uint32_t>(pindex.at(r.pre + ".conv2.weight"));
    }
    GnOut g2 = gn_fwd(hs, N, HW, G, n2w, n2b, ls->film, L.film_total, r.film_off, 1, false, drop);
    const float* res = x->p;
    float* sproj = nullptr;
    if (proj) {
      Param &c3w = P(r.pre + ".conv3.weight"), &c3b = P(r.pre + ".conv3.bias");
      sproj = eng.alloc<float>(static_cast<long long>(N) * HW * cout);
      Epi e;
      e.bias = c3b.w;
      e.out_f32 = sproj;
      eng.gemm_nt(g1.raw16, cin, c3w.w16, cin, N * HW, cout, cin, e);
      res = sproj;
    }
    Act* out = eng.new_act(N, H, W, cout);
    {
      Epi e;
      e.bias = c2b.w;
      e.residual = res;
      e.out_f32 = out->p;
      eng.conv3x3_fwd(g2.y16, cout, N, H, W, cout, c2w.w16, cout, e, c2w.w16f, c2w.bias_f);
    }
    if (!eng.training) {
      eng.rel(g1.y16);
      eng.rel(g1.raw16);
      eng.rel(g1.sums);
      eng.rel(g2.y16);
      eng.rel(g2.sums);
      eng.rel(h);
      eng.rel(sproj);
      return out;
    }
    const LevelSpec* Lp = &L;
    eng.tape.push_back([=]() {
      if (out->g == nullptr) return;  // nothing flowed back
      Engine& E = eng;
      const long long rows = static_cast<long long>(N) * HW;
      Param &n1w = P(r.pre + ".norm1.weight"), &n1b = P(r.pre + ".norm1.bias");
      Param &c1w = P(r.pre + ".conv1.weight"), &c1b = P(r.pre + ".conv1.bias");
      Param &n2w = P(r.pre + ".norm2.weight"), &n2b = P(r.pre + ".norm2.bias");
      Param &c2w = P(r.pre + ".conv2.weight"), &c2b = P(r.pre + ".conv2.bias");
      Param &tlw = P(r.pre + ".time_layer.weight"), &tlb = P(r.pre + ".time_layer.bias");
      // conv2
      __half* d16 = E.alloc<__half>(rows * cout);
      float* bias_scratch = E.zeros_f32(cout);
      cast_colsum(out->g, d16, rows, cout, bias_scratch, inv_scale(), E.st);
      if (c2b.g != nullptr) axpy_f32(c2b.g, bias_scratch, 1.f, cout, 1, E.st);
      float* wtmp = E.alloc<float>(std::max((Engine::fold_ok(cin, cout) ? 36ll : 9ll) * cin * cout,
                                             (Engine::fold_ok(cout, cout) ? 36ll : 9ll) * cout * cout));
      if (c2w.g != nullptr) conv_wgrad_into(d16, cout, g2.y16, cout, N, H, W, cout, cout, wtmp, c2w);
      // the data gradient entering a GroupNorm backward stays fp32: it is no GEMM operand, and the GroupNorm backward
      // subtracts its group means, so an fp16 rounding here dominates the (cancelling) conv bias gradients before it
      float* da2 = E.alloc<float>(rows * cout);
      {
        // (a single-plane pass takes the gradient at fp16 only)
        __half* d16lo = E.single_plane ? nullptr : E.alloc<__half>(rows * cout);
        if (d16lo != nullptr) f16_lo_plane(out->g, d16lo, rows * cout, E.st);
        Epi e;
        e.out_f32 = da2;
        e.a_lo = d16lo;
        E.conv3x3_dgrad(d16, cout, N, H, W, cout, c2w.w16, cout, e, c2w.w16f);
        E.rel(d16lo);
      }
      // norm2 + FiLM + SiLU: h has a single consumer, so its gradient goes straight to the fp16 operand
      // of conv1's backward, with conv1's bias gradient as column sums
      __half* dh16 = E.alloc<__half>(rows * cout);
      __half* dh16lo = E.single_plane ? nullptr : E.alloc<__half>(rows * cout);
      float* dfilm = E.alloc<float>(2ll * N * cout);
      gn_bwd(Src2{h, nullptr, cout, 0}, da2, false, N, HW, G, g2.sums, n2w, n2b, ls->film, Lp->film_total, r.film_off, 1,
             dfilm, nullptr, nullptr, nullptr, dh16, c1b.g, dh16lo, drop);
      E.rel(da2);
      // time layer: film = silu(temb) Wt^T + bt  (batch rows)
      {
        __half* df16 = E.alloc<__half>(2ll * N * cout);
        cast_colsum(dfilm, df16, N, 2 * cout, tlb.g, inv_scale(), E.st);
        int acc = ls->dstemb_init ? 1 : 0;
        ls->dstemb_init = true;
        linear_bwd(df16, 2 * cout, N, 2 * cout, Lp->c.temporal_dim, ls->stemb16, Lp->c.temporal_dim, tlw, nullptr,
                   false, ls->dstemb, acc);
        E.rel(df16);
        E.rel(dfilm);
      }
      // conv1
      if (c1w.g != nullptr) conv_wgrad_into(dh16, cout, g1.y16, cin, N, H, W, cin, cout, wtmp, c1w);
      float* da1 = E.alloc<float>(rows * cin);
      {
        Epi e;
        e.out_f32 = da1;
        e.a_lo = dh16lo;
        E.conv3x3_dgrad(dh16, cout, N, H, W, cout, c1w.w16, cin, e, c1w.w16f);
      }
      E.rel(dh16);
      E.rel(dh16lo);
      // norm1 + SiLU -> x (and skip). Identity residual folds in as `extra`.
      gn_bwd(src, da1, false, N, HW, G, g1.sums, n1w, n1b, nullptr, 0, 0, 1, nullptr, proj ? nullptr : out->g, x, skip);
      E.rel(da1);
      if (proj) {
        Param &c3w = P(r.pre + ".conv3.weight"), &c3b = P(r.pre + ".conv3.bias");
        if (c3b.g != nullptr) axpy_f32(c3b.g, bias_scratch, 1.f, cout, 1, E.st);
        if (c3w.g != nullptr) {
          E.side_begin();
          Epi e;
          e.out_f32 = c3w.g;
          e.alpha_dev = inv_scale();
          e.atomic_ok = true;
          E.gemm_tn(d16, cout, g1.raw16, cin, cout, cin, static_cast<int>(rows), e);
          E.side_end();
        }
        // dX (+)= d16 * W3, split over the two concat sources
        {
          Epi e;
          e.out_f32 = x->g;  // already initialised by gn_bwd above
          e.residual = x->g;
          e.ldc = x->c;
          E.gemm_nn(d16, cout, c3w.w16, cin, static_cast<int>(rows), x->c, cout, e);
        }
        if (skip != nullptr) {
          Epi e;
          e.out_f32 = skip->g;
          e.residual = skip->g;
          e.ldc = skip->c;
          E.gemm_nn(d16, cout, c3w.w16 + x->c, cin, static_cast<int>(rows), skip->c, cout, e);
        }
      }
      E.rel(wtmp);
      E.rel(d16);
      E.rel(bias_scratch);
      E.rel(out->g);
    });
    return out;
  }

  // ---------------------------------------------------------------- attention (unet.py:276-313)
  struct BOp {
    const __half* p;
    int inner, rows;
    long long row_stride;
    int slots;
    long long slot_stride, batch_stride;
    int z_off;
    bool mn;
  };
  void gemm_batched(const BOp& A, const BOp& B, int M, int N, int K, int nz1, int nz2, const Epi& e, long long ldc,
                    long long cz1, long long cz2) {
    GemmParams p{};
    p.kind = GEMM_PLAIN;
    p.M = M; p.N = N; p.K = K;
    const long long mt = (M + 127) / 128;
    int bn = N >= 256 ? 256 : (N + 15) / 16 * 16;
    p.block_n = bn;
    p.nz1 = nz1; p.nz2 = nz2; p.nsplit = 1;
    p.a_use_z = p.b_use_z = 1;
    p.a_z1_off = A.z_off;
    p.b_z1_off = B.z_off;
    p.num_kblocks = (K + 63) / 64;
    p.alpha = e.alpha; p.alpha_dev = e.alpha_dev; p.bias = e.bias; p.residual = e.residual;
    p.out_f32 = e.out_f32; p.out_f16 = e.out_f16; p.out_act_f16 = e.out_act_f16; p.act = e.act;
    p.ldc = ldc; p.c_z1_stride = cz1; p.c_z2_stride = cz2;
    auto mk = [&](const BOp& o, bool is_a) {
      TmapSpec s;
      s.ptr = o.p;
      s.dims[0] = o.inner; s.dims[1] = o.rows; s.dims[2] = o.slots; s.dims[3] = nz2;
      s.strides[0] = 1; s.strides[1] = o.row_stride; s.strides[2] = o.slot_stride; s.strides[3] = o.batch_stride;
      s.box[0] = 64;
      s.box[1] = o.mn ? 64 : (is_a ? 128 : bn);
      s.box[2] = 1; s.box[3] = 1;
      return s;
    };
    (void)mt;
    TmapSpec a = mk(A, true), b = mk(B, false);
    const int rc = launch_gemm(a, b, A.mn ? 1 : 0, B.mn ? 1 : 0, p, eng.st);
    if (rc != 0) throw MdmFail("batched attention GEMM failed rc=" + std::to_string(rc));
  }

  Act* attn_fwd(const LevelSpec& L, const AttnSpec& a, Act* x) {
    Engine& E = eng;
    const int B = x->n, H = x->h, W = x->w, T = H * W, C = a.C, nh = cfg.num_heads, d = C / nh;
    MDM_CHECK(x->c == C && C % nh == 0 && d % 8 == 0, "attention channels (head dim must be a multiple of 8)");
    const long long rows = static_cast<long long>(B) * T;
    const float alpha = 1.0f / sqrtf(static_cast<float>(d));
    Param &nw = P(a.pre + ".norm.weight"), &nb = P(a.pre + ".norm.bias");
    Param &qw = P(a.pre + ".qkv.weight"), &qb = P(a.pre + ".qkv.bias");
    Param &pw = P(a.pre + ".proj_out.weight"), &pb = P(a.pre + ".proj_out.bias");
    GnOut g1 = gn_fwd(Src2{x->p, nullptr, C, 0}, B, T, 32, nw, nb, nullptr, 0, 0, 0, false);
    __half* qkv = E.alloc<__half>(rows * 3 * C);
    {
      Epi e;
      e.bias = qb.w;
      e.out_f16 = qkv;
      E.gemm_nt(g1.y16, C, qw.w16, C, static_cast<int>(rows), 3 * C, C, e);
    }
    const int Tp = round8(T);
    const long long nrow = static_cast<long long>(B) * nh * T;
    const bool cross = a.cond;
    const int S = cs.S, cd = cs.cd, Sp = round8(S);
    const bool fused = fused_attention && d <= 128;
    __half* h16 = E.alloc<__half>(rows * C);
    __half *Pm = nullptr, *cn16 = nullptr, *kv = nullptr, *Pc = nullptr, *oself = nullptr;
    float *lnstats = nullptr, *astats = nullptr;
    bool kv_cached = false;
    BOp Q{qkv, d, T, 3ll * C, 3 * nh, d, static_cast<long long>(T) * 3 * C, 0, false};
    if (cross) {
      // k_c, v_c = kv_cond(LayerNorm(cond))  (unet.py:304-305)
      Param &lw = P(a.pre + ".norm_cond.weight"), &lb = P(a.pre + ".norm_cond.bias");
      Param &kw = P(a.pre + ".kv_cond.weight"), &kb = P(a.pre + ".kv_cond.bias");
      const long long crow = static_cast<long long>(B) * S;
      (void)lw; (void)lb; (void)kb;
      // with the K/V cache on (stage 2, no tape) this block's slab of it: filled here (1) or read as it is (2)
      kv_cached = cs.kv_mode != 0;
      kv = kv_cached ? kv_cache + a.kv_col * cs.B * S : E.alloc<__half>(crow * 2 * C);
      if (cs.kv_mode != 2) {
        Epi e2;
        e2.bias = a.kv_bias_fold;
        e2.out_f16 = kv;
        E.gemm_nt(cs.xhat16, cd, kw.w16, cd, static_cast<int>(crow), 2 * C, cd, e2);
      }
    }
    if (fused) {
      if (E.training) {
        astats = E.alloc<float>(static_cast<long long>(B) * nh * 2 * T * 2);
        if (cross) oself = E.alloc<__half>(rows * C);
      }
      attention_forward(qkv, kv, cross ? cs.cross_mask : nullptr, B, T, S, C, nh, h16, oself, astats, E.st);
    } else {
      float* sc = E.alloc<float>(nrow * Tp);
      Pm = E.alloc<__half>(nrow * Tp);
      BOp Kk = Q;
      Kk.z_off = nh;
      BOp Vm{qkv, d, T, 3ll * C, 3 * nh, d, static_cast<long long>(T) * 3 * C, 2 * nh, true};
      {
        Epi e;
        e.alpha = alpha;
        e.out_f32 = sc;
        gemm_batched(Q, Kk, T, T, d, nh, B, e, Tp, static_cast<long long>(T) * Tp, static_cast<long long>(nh) * T * Tp);
      }
      softmax_rows(sc, Pm, nrow, T, Tp, nullptr, 1, E.st);
      E.rel(sc);
      BOp Pk{Pm, T, T, Tp, nh, static_cast<long long>(T) * Tp, static_cast<long long>(nh) * T * Tp, 0, false};
      if (!cross) {
        Epi e;
        e.out_f16 = h16;
        gemm_batched(Pk, Vm, T, d, T, nh, B, e, C, d, static_cast<long long>(T) * C);
      } else {
        float* hs32 = E.alloc<float>(rows * C);
        Epi e;
        e.out_f32 = hs32;
        gemm_batched(Pk, Vm, T, d, T, nh, B, e, C, d, static_cast<long long>(T) * C);
        float* scc = E.alloc<float>(nrow * Sp);
        Pc = E.alloc<__half>(nrow * Sp);
        BOp Kc{kv, d, S, 2ll * C, 2 * nh, d, static_cast<long long>(S) * 2 * C, 0, false};
        BOp Vc{kv, d, S, 2ll * C, 2 * nh, d, static_cast<long long>(S) * 2 * C, nh, true};
        {
          Epi e3;
          e3.alpha = alpha;
          e3.out_f32 = scc;
          gemm_batched(Q, Kc, T, S, d, nh, B, e3, Sp, static_cast<long long>(T) * Sp, static_cast<long long>(nh) * T * Sp);
        }
        softmax_rows(scc, Pc, nrow, S, Sp, cs.cross_mask, static_cast<long long>(nh) * T, E.st);
        E.rel(scc);
        BOp Pck{Pc, S, T, Sp, nh, static_cast<long long>(T) * Sp, static_cast<long long>(nh) * T * Sp, 0, false};
        {
          Epi e4;
          e4.residual = hs32;
          e4.out_f16 = h16;
          gemm_batched(Pck, Vc, T, d, S, nh, B, e4, C, d, static_cast<long long>(T) * C);
        }
        E.rel(hs32);
      }
    }
    Act* x1 = E.new_act(B, H, W, C);
    {
      Epi e;
      e.bias = pb.w;
      e.residual = x->p;
      e.out_f32 = x1->p;
      E.gemm_nt(h16, C, pw.w16, C, static_cast<int>(rows), C, C, e);
    }
    Act* out = x1;
    GnOut g2{};
    __half *u16 = nullptr, *gl16 = nullptr;
    if (a.ffn) {
      Param &fw0 = P(a.pre + ".ffn.0.weight"), &fb0 = P(a.pre + ".ffn.0.bias");
      Param &fw1 = P(a.pre + ".ffn.1.weight"), &fb1 = P(a.pre + ".ffn.1.bias");
      Param &fw3 = P(a.pre + ".ffn.3.weight"), &fb3 = P(a.pre + ".ffn.3.bias");
      g2 = gn_fwd(Src2{x1->p, nullptr, C, 0}, B, T, 32, fw0, fb0, nullptr, 0, 0, 0, false);
      u16 = E.training ? E.alloc<__half>(rows * 4 * C) : nullptr;  // pre-activation: only the backward needs it
      gl16 = E.alloc<__half>(rows * 4 * C);
      {
        Epi e;
        e.bias = fb1.w;
        e.out_f16 = u16;
        e.out_act_f16 = gl16;
        e.act = ACT_GELU;
        E.gemm_nt(g2.y16, C, fw1.w16, C, static_cast<int>(rows), 4 * C, C, e);
      }
      out = E.new_act(B, H, W, C);
      {
        Epi e;
        e.bias = fb3.w;
        e.residual = x1->p;
        e.out_f32 = out->p;
        E.gemm_nt(gl16, 4 * C, fw3.w16, 4 * C, static_cast<int>(rows), C, 4 * C, e);
      }
    }
    if (!E.training) {
      E.rel(g1.y16); E.rel(g1.sums); E.rel(qkv); E.rel(Pm);
      E.rel(h16); E.rel(cn16); E.rel(lnstats); E.rel(Pc);
      if (!kv_cached) E.rel(kv);
      E.rel(oself); E.rel(astats);
      if (a.ffn) {
        E.rel(g2.y16); E.rel(g2.sums); E.rel(u16); E.rel(gl16);
        E.rel(x1->p);
      }
      return out;
    }
    E.tape.push_back([=]() {
      Engine& E = eng;
      const int irows = static_cast<int>(rows);
      Param &nw = P(a.pre + ".norm.weight"), &nb = P(a.pre + ".norm.bias");
      Param &qw = P(a.pre + ".qkv.weight"), &qb = P(a.pre + ".qkv.bias");
      Param &pw = P(a.pre + ".proj_out.weight"), &pb = P(a.pre + ".proj_out.bias");
      if (a.ffn) {
        if (out->g == nullptr) return;
        Param &fw0 = P(a.pre + ".ffn.0.weight"), &fb0 = P(a.pre + ".ffn.0.bias");
        Param &fw1 = P(a.pre + ".ffn.1.weight"), &fb1 = P(a.pre + ".ffn.1.bias");
        Param &fw3 = P(a.pre + ".ffn.3.weight"), &fb3 = P(a.pre + ".ffn.3.bias");
        __half* d16 = E.alloc<__half>(rows * C);
        cast_colsum(out->g, d16, rows, C, fb3.g, inv_scale(), E.st);
        // ffn.3 backward: weight gradient, then dU = (dY W3) * gelu'(U) straight out of the dgrad epilogue
        linear_bwd(d16, C, irows, C, 4 * C, gl16, 4 * C, fw3, nullptr, false, nullptr, 0);
        __half* du16 = E.alloc<__half>(rows * 4 * C);
        {
          Epi e;
          e.out_f16 = du16;
          e.gelu_grad_src = u16;
          E.gemm_nn(d16, C, fw3.w16, 4 * C, irows, 4 * C, C, e);
        }
        E.rel(d16);
        float* dm32 = E.alloc<float>(rows * C);
        linear_bwd(du16, 4 * C, irows, 4 * C, C, g2.y16, C, fw1, &fb1, true, dm32, 0);
        E.rel(du16);
        gn_bwd(Src2{x1->p, nullptr, C, 0}, dm32, false, B, T, 32, g2.sums, fw0, fb0, nullptr, 0, 0, 0, nullptr, out->g, x1,
               nullptr);
        E.rel(dm32);
        E.rel(out->g);
      }
      if (x1->g == nullptr) return;
      // proj_out
      __half* d16 = E.alloc<__half>(rows * C);
      cast_colsum(x1->g, d16, rows, C, pb.g, inv_scale(), E.st);
      if (pw.g != nullptr) {
        E.side_begin();
        Epi e;
        e.out_f32 = pw.g;
        e.alpha_dev = inv_scale();
        e.atomic_ok = true;
        E.gemm_tn(d16, C, h16, C, C, C, irows, e);
        E.side_end();
      }
      __half* dh16 = E.alloc<__half>(rows * C);
      {
        Epi e;
        e.out_f16 = dh16;
        E.gemm_nn(d16, C, pw.w16, C, irows, C, C, e);
      }
      E.rel(d16);
      __half* dqkv = E.alloc<__half>(rows * 3 * C);
      __half* dkv = nullptr;
      float* dq32 = nullptr;
      if (fused) {
        const long long crow = static_cast<long long>(B) * S;
        if (cross) dkv = E.alloc<__half>(crow * 2 * C);
        float* Dterm = E.alloc<float>(static_cast<long long>(B) * nh * 2 * T);
        dq32 = E.alloc<float>(rows * C);
        attention_backward(qkv, kv, cross ? cs.cross_mask : nullptr, dh16, h16, oself, astats, B, T, S, C, nh, Dterm, dq32,
                           dqkv, dkv, E.st);
        E.rel(Dterm);
      } else {
        BOp Q{qkv, d, T, 3ll * C, 3 * nh, d, static_cast<long long>(T) * 3 * C, 0, false};
        BOp Qm = Q; Qm.mn = true;
        BOp Kk = Q; Kk.z_off = nh;
        BOp Km = Kk; Km.mn = true;
        BOp Vk = Q; Vk.z_off = 2 * nh;
        BOp dHk{dh16, d, T, C, nh, d, static_cast<long long>(T) * C, 0, false};
        BOp dHm = dHk; dHm.mn = true;
        BOp Pmn{Pm, T, T, Tp, nh, static_cast<long long>(T) * Tp, static_cast<long long>(nh) * T * Tp, 0, true};
        const long long qkv_b = static_cast<long long>(T) * 3 * C;
        // dV = P^T dH
        {
          Epi e;
          e.out_f16 = dqkv + 2 * C;
          gemm_batched(Pmn, dHm, T, d, T, nh, B, e, 3 * C, d, qkv_b);
        }
        // dP = dH V^T ; dS = softmax'(P, dP) * alpha
        float* dP = E.alloc<float>(nrow * Tp);
        {
          Epi e;
          e.out_f32 = dP;
          gemm_batched(dHk, Vk, T, T, d, nh, B, e, Tp, static_cast<long long>(T) * Tp, static_cast<long long>(nh) * T * Tp);
        }
        __half* dS = E.alloc<__half>(nrow * Tp);
        softmax_bwd_rows(Pm, dP, dS, nrow, T, Tp, alpha, E.st);
        E.rel(dP);
        BOp dSk{dS, T, T, Tp, nh, static_cast<long long>(T) * Tp, static_cast<long long>(nh) * T * Tp, 0, false};
        BOp dSm = dSk; dSm.mn = true;
        // dQ = dS K (+ cross term below)
        if (cross) {
          // fp32 partial in the same (ld = 3C) layout as dqkv so the cross term can add it as a residual
          dq32 = E.alloc<float>(rows * 3 * C);
          Epi e;
          e.out_f32 = dq32;
          gemm_batched(dSk, Km, T, d, T, nh, B, e, 3 * C, d, qkv_b);
        } else {
          Epi e;
          e.out_f16 = dqkv;
          gemm_batched(dSk, Km, T, d, T, nh, B, e, 3 * C, d, qkv_b);
        }
        // dK = dS^T Q
        {
          Epi e;
          e.out_f16 = dqkv + C;
          gemm_batched(dSm, Qm, T, d, T, nh, B, e, 3 * C, d, qkv_b);
        }
        E.rel(dS);
        if (cross) {
          Param &lw = P(a.pre + ".norm_cond.weight"), &lb = P(a.pre + ".norm_cond.bias");
          Param &kw = P(a.pre + ".kv_cond.weight"), &kb = P(a.pre + ".kv_cond.bias");
          const long long crow = static_cast<long long>(B) * S;
          const long long kv_b = static_cast<long long>(S) * 2 * C;
          dkv = E.alloc<__half>(crow * 2 * C);
          BOp Kc{kv, d, S, 2ll * C, 2 * nh, d, kv_b, 0, false};
          BOp Kcm = Kc; Kcm.mn = true;
          BOp Vck = Kc; Vck.z_off = nh;
          BOp Pcm{Pc, S, T, Sp, nh, static_cast<long long>(T) * Sp, static_cast<long long>(nh) * T * Sp, 0, true};
          {  // dVc = Pc^T dH
            Epi e;
            e.out_f16 = dkv + C;
            gemm_batched(Pcm, dHm, S, d, T, nh, B, e, 2 * C, d, kv_b);
          }
          float* dPc = E.alloc<float>(nrow * Sp);
          {
            Epi e;
            e.out_f32 = dPc;
            gemm_batched(dHk, Vck, T, S, d, nh, B, e, Sp, static_cast<long long>(T) * Sp, static_cast<long long>(nh) * T * Sp);
          }
          __half* dSc = E.alloc<__half>(nrow * Sp);
          softmax_bwd_rows(Pc, dPc, dSc, nrow, S, Sp, alpha, E.st);
          E.rel(dPc);
          BOp dSck{dSc, S, T, Sp, nh, static_cast<long long>(T) * Sp, static_cast<long long>(nh) * T * Sp, 0, false};
          BOp dScm = dSck; dScm.mn = true;
          {  // dQ = dq32 + dSc Kc -> fp16
            Epi e;
            e.residual = dq32;
            e.out_f16 = dqkv;
            gemm_batched(dSck, Kcm, T, d, S, nh, B, e, 3 * C, d, qkv_b);
          }
          {  // dKc = dSc^T Q
            Epi e;
            e.out_f16 = dkv;
            gemm_batched(dScm, Qm, S, d, T, nh, B, e, 2 * C, d, kv_b);
          }
          E.rel(dSc);
        }

      }
      if (cross) {
        Param &lw = P(a.pre + ".norm_cond.weight"), &lb = P(a.pre + ".norm_cond.bias");
        Param &kw = P(a.pre + ".kv_cond.weight"), &kb = P(a.pre + ".kv_cond.bias");
        const long long crow = static_cast<long long>(B) * S;
        // kv = xhat (W diag(w_ln))^T + (W b_ln + bias): gradients of the folded operands, then unfold
        float* dbf = E.zeros_f32(2 * C);
        colsum_f16(dkv, crow, 2 * C, dbf, inv_scale(), E.st);
        if (kb.g != nullptr) axpy_f32(kb.g, dbf, 1.f, 2 * C, 1, E.st);
        float* dWf = E.zeros_f32(2ll * C * cd);
        {
          Epi e;
          e.out_f32 = dWf;
          e.alpha_dev = inv_scale();
          e.atomic_ok = true;
          E.gemm_tn(dkv, 2 * C, cs.xhat16, cd, 2 * C, cd, static_cast<int>(crow), e);
        }
        unfold_ln_grads(dWf, dbf, kw.w, lw.w, lb.w, kw.g, lw.g, lb.g, 2 * C, cd, E.st);
        E.rel(dWf);
        E.rel(dbf);
        const bool whole = B == cs.B;  // a level that ran only part of the batch touches the leading rows only
        if (cs.dxhat == nullptr) {
          cs.dxhat = whole ? E.alloc<float>(crow * cd) : E.zeros_f32(static_cast<long long>(cs.B) * S * cd);
          cs.dxhat_init = !whole;
        }
        {
          Epi e;
          e.out_f32 = cs.dxhat;
          if (cs.dxhat_init) e.residual = cs.dxhat;
          E.gemm_nn(dkv, 2 * C, kw.w16, cd, static_cast<int>(crow), cd, 2 * C, e);
        }
        cs.dxhat_init = true;
        E.rel(dkv);
      }
      // qkv conv + norm
      float* dn32 = E.alloc<float>(rows * C);
      linear_bwd(dqkv, 3 * C, irows, 3 * C, C, g1.y16, C, qw, &qb, true, dn32, 0);
      E.rel(dqkv);
      E.rel(dh16);
      E.rel(dq32);
      gn_bwd(Src2{x->p, nullptr, C, 0}, dn32, false, B, T, 32, g1.sums, nw, nb, nullptr, 0, 0, 0, nullptr, x1->g, x, nullptr);
      E.rel(dn32);
      E.rel(x1->g);
    });
    return out;
  }

  // ---------------------------------------------------------------- resampling (unet.py:514-532,563-569)
  Act* downsample_fwd(const BlockSpec& b, Act* x) {
    Engine& E = eng;
    const int N = x->n, H = x->h, W = x->w, C = x->c;
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    Param &w = P(b.pre + ".resample.weight"), &bb = P(b.pre + ".resample.bias");
    const long long orow = static_cast<long long>(N) * Ho * Wo;
    __half* col = E.alloc<__half>(orow * 9 * C);
    im2col3x3(x->p, col, N, H, W, C, 2, E.st);
    Act* y = E.new_act(N, Ho, Wo, C);
    Epi e;
    e.bias = bb.w;
    e.out_f32 = y->p;
    E.gemm_nt(col, 9ll * C, w.w16, 9ll * C, static_cast<int>(orow), C, 9 * C, e);
    if (!E.training) {
      E.rel(col);
      return y;
    }
    E.tape.push_back([=]() {
      if (y->g == nullptr) return;
      Engine& E = eng;
      Param &w = P(b.pre + ".resample.weight"), &bb = P(b.pre + ".resample.bias");
      __half* d16 = E.alloc<__half>(orow * C);
      cast_colsum(y->g, d16, orow, C, bb.g, inv_scale(), E.st);
      if (w.g != nullptr) {
        float* wtmp = E.zeros_f32(9ll * C * C);
        Epi e;
        e.out_f32 = wtmp;
        e.atomic_ok = true;
        E.gemm_tn(d16, C, col, 9ll * C, C, 9 * C, static_cast<int>(orow), e);
        unpack_conv_wgrad(wtmp, w.g, C, C, 9, C, inv_scale(), E.st);
        E.rel(wtmp);
      }
      float* dcol = E.alloc<float>(orow * 9 * C);
      {
        Epi e;
        e.out_f32 = dcol;
        E.gemm_nn(d16, C, w.w16, 9ll * C, static_cast<int>(orow), 9 * C, C, e);
      }
      int acc = 0;
      float* dx = E.grad_buf(x, &acc);
      col2im3x3(dcol, dx, acc, N, H, W, C, 2, E.st);
      E.rel(dcol);
      E.rel(d16);
      E.rel(y->g);
    });
    return y;
  }

  // generic 3x3 stride-1 conv on an fp16 NHWC operand producing a new Act (+ optional residual)
  // n_alloc > N: the Act holds n_alloc samples, the conv fills the first N and the rest is zero
  // (nested_unet.py:200-204 pads the in_adapter output for the samples the outer level did not run)
  Act* conv_act(const std::string& wname, const std::string& bname, const __half* x16, int N, int H, int W, int Cin,
                int Cout, const float* residual, int n_alloc = 0) {
    Param &w = P(wname), &bb = P(bname);
    Act* y = eng.new_act(std::max(N, n_alloc), H, W, Cout);
    Epi e;
    e.bias = bb.w;
    e.residual = residual;
    e.out_f32 = y->p;
    eng.conv3x3_fwd(x16, Cin, N, H, W, Cin, w.w16, Cout, e, w.w16f, w.bias_f);
    if (n_alloc > N) {
      const long long lead = static_cast<long long>(N) * H * W * Cout;
      MDM_CUDA(cudaMemsetAsync(y->p + lead, 0, sizeof(float) * (y->numel() - lead), eng.st));
    }
    return y;
  }
  // backward of conv_act: returns fp32 gradient w.r.t. the fp16 operand (caller releases)
  float* conv_act_bwd(const std::string& wname, const std::string& bname, const __half* x16, Act* y, int Cin,
                      int n_lead = 0) {
    Engine& E = eng;
    Param &w = P(wname), &bb = P(bname);
    const int N = n_lead > 0 ? n_lead : y->n, H = y->h, W = y->w, Cout = y->c;
    const long long rows = static_cast<long long>(N) * H * W;
    __half* d16 = E.alloc<__half>(rows * Cout);
    cast_colsum(y->g, d16, rows, Cout, bb.g, inv_scale(), E.st);
    if (w.g != nullptr) {
      float* wtmp = E.alloc<float>((Engine::fold_ok(Cin, Cout) ? 36ll : 9ll) * Cin * Cout);
      conv_wgrad_into(d16, Cout, x16, Cin, N, H, W, Cin, Cout, wtmp, w);
      E.rel(wtmp);
    }
    float* dx = E.alloc<float>(rows * Cin);
    Epi e;
    e.out_f32 = dx;
    E.conv3x3_dgrad(d16, Cout, N, H, W, Cout, w.w16, Cin, e, w.w16f);
    E.rel(d16);
    return dx;
  }

  Act* upsample_fwd(const BlockSpec& b, Act* x) {
    Engine& E = eng;
    const int N = x->n, H = x->h, W = x->w, C = x->c;
    __half* u16 = E.alloc<__half>(static_cast<long long>(N) * 4 * H * W * C);
    upsample2x_f16(x->p, u16, N, H, W, C, E.st);
    Act* y = conv_act(b.pre + ".resample.weight", b.pre + ".resample.bias", u16, N, 2 * H, 2 * W, C, C, nullptr);
    if (!E.training) {
      E.rel(u16);
      return y;
    }
    E.tape.push_back([=]() {
      if (y->g == nullptr) return;
      Engine& E = eng;
      float* du = conv_act_bwd(b.pre + ".resample.weight", b.pre + ".resample.bias", u16, y, C);
      int acc = 0;
      float* dx = E.grad_buf(x, &acc);
      upsample2x_bwd(du, dx, acc, N, H, W, C, E.st);
      E.rel(du);
      E.rel(y->g);
    });
    return y;
  }

  // ---------------------------------------------------------------- block (unet.py:534-576)
  Act* block_fwd(const LevelSpec& L, LevelStep* ls, const BlockSpec& b, Act* x, std::vector<Act*>* skips_in,
                 std::vector<Act*>* acts_out) {
    for (size_t i = 0; i < b.res.size(); ++i) {
      Act* skip = nullptr;
      if (skips_in != nullptr) {
        skip = skips_in->front();
        skips_in->erase(skips_in->begin());
      }
      x = resnet_fwd(L, ls, b.res[i], x, skip);
      for (int j = 0; j < b.nattn; ++j) x = attn_fwd(L, b.attn[i * b.nattn + j], x);
      if (acts_out != nullptr) acts_out->push_back(x);
      debug_acts[b.pre + "." + std::to_string(i)] = x;
    }
    if (b.down) {
      x = downsample_fwd(b, x);
      if (acts_out != nullptr) acts_out->push_back(x);
    } else if (b.up) {
      x = upsample_fwd(b, x);
    }
    return x;
  }

  // ---------------------------------------------------------------- embeddings
  // out32 = W2 silu(W1 e + b1) + b2 ; records backward that consumes `dsrc` (gradient of out32)
  struct MlpRec {
    __half* e16;
    float* h1;
    __half* sh16;
  };
  float* embed_mlp_fwd(const std::string& l1, const std::string& l2, __half* e16, int B, int td, MlpRec* rec) {
    Engine& E = eng;
    Param &w1 = P(l1 + ".weight"), &b1 = P(l1 + ".bias"), &w2 = P(l2 + ".weight"), &b2 = P(l2 + ".bias");
    float* h1 = E.alloc<float>(static_cast<long long>(B) * td);
    {
      Epi e;
      e.bias = b1.w;
      e.out_f32 = h1;
      E.gemm_nt(e16, td / 4, w1.w16, td / 4, B, td, td / 4, e);
    }
    __half* sh16 = E.alloc<__half>(static_cast<long long>(B) * td);
    silu_f16(h1, sh16, static_cast<long long>(B) * td, E.st);
    float* out = E.alloc<float>(static_cast<long long>(B) * td);
    {
      Epi e;
      e.bias = b2.w;
      e.out_f32 = out;
      E.gemm_nt(sh16, td, w2.w16, td, B, td, td, e);
    }
    rec->e16 = e16;
    rec->h1 = h1;
    rec->sh16 = sh16;
    return out;
  }
  void embed_mlp_bwd(const std::string& l1, const std::string& l2, const MlpRec& rec, const float* dout, int B, int td) {
    Engine& E = eng;
    Param &w1 = P(l1 + ".weight"), &b1 = P(l1 + ".bias"), &w2 = P(l2 + ".weight"), &b2 = P(l2 + ".bias");
    const long long n = static_cast<long long>(B) * td;
    __half* d16 = E.alloc<__half>(n);
    cast_colsum(dout, d16, B, td, b2.g, inv_scale(), E.st);
    float* dsh = E.alloc<float>(n);
    linear_bwd(d16, td, B, td, td, rec.sh16, td, w2, nullptr, false, dsh, 0);
    float* dh1 = E.alloc<float>(n);
    silu_bwd(rec.h1, dsh, dh1, n, 0, E.st);
    // (a second buffer: the weight-gradient GEMM of layer 2 may still be reading d16 on the side stream)
    __half* d16b = E.alloc<__half>(n);
    cast_colsum(dh1, d16b, B, td, b1.g, inv_scale(), E.st);
    linear_bwd(d16b, td, B, td, td / 4, rec.e16, td / 4, w1, nullptr, false, nullptr, 0);
    E.rel(d16b);
    E.rel(d16);
    E.rel(dsh);
    E.rel(dh1);
  }

  // forward_conditioning (unet.py:847-865) on the innermost level. Stage 0 also runs the token LayerNorm of the
  // cross-attention blocks (cond_norm_fwd), which belongs to forward_denoising; stage 1 stops at cond_emb.
  void conditioning_fwd(int stage) {
    Engine& E = eng;
    const LevelSpec& L = levels.back();
    const int B = io->batch, S = io->tokens, td = L.c.temporal_dim;
    cs = CondStep();
    cs.B = B;
    cs.S = S;
    cs.cd = cfg.cond_dim;
    cs.lm = io->lm;
    // with lm_head layers and unmasked cross-attention the pooled y is the plain mean over all tokens (unet.py:854-856)
    cs.mask = (cfg.num_lm_head_layers > 0 && !cfg.masked_cross_attention) ? nullptr : io->lm_mask;
    cs.cross_mask = cfg.masked_cross_attention ? io->lm_mask : nullptr;
    if (cfg.cond_dim <= 0) return;
    const long long crow = static_cast<long long>(B) * S;
    if (cfg.has_lm_proj) {
      Param &w = P(L.pre + "lm_proj.weight"), &b = P(L.pre + "lm_proj.bias");
      cs.lm16 = E.alloc<__half>(crow * cfg.lm_dim);
      if (io->apply_lm_mask) {
        MDM_CHECK(io->lm_mask != nullptr && cfg.lm_dim % 4 == 0, "apply_lm_mask needs lm_mask");
        cast_rowscale_f16(io->lm, io->lm_mask, cs.lm16, crow, cfg.lm_dim, E.st);
      } else {
        cast_f32_to_f16(io->lm, cs.lm16, crow * cfg.lm_dim, E.st);
      }
      cs.cond32 = E.alloc<float>(crow * cfg.cond_dim);
      Epi e;
      e.bias = b.w;
      e.out_f32 = cs.cond32;
      E.gemm_nt(cs.lm16, cfg.lm_dim, w.w16, cfg.lm_dim, static_cast<int>(crow), cfg.cond_dim, cfg.lm_dim, e);
      if (E.training) {
        // runs after the lm_head backward closures have turned cs.dcond into the gradient of lm_proj's output
        E.tape.push_back([=]() {
          if (cs.dcond == nullptr) return;
          Engine& E = eng;
          const LevelSpec& L = levels.back();
          Param &w = P(L.pre + "lm_proj.weight"), &b = P(L.pre + "lm_proj.bias");
          __half* d16 = E.alloc<__half>(crow * cfg.cond_dim);
          cast_colsum(cs.dcond, d16, crow, cfg.cond_dim, b.g, inv_scale(), E.st);
          linear_bwd(d16, cfg.cond_dim, static_cast<int>(crow), cfg.cond_dim, cfg.lm_dim, cs.lm16, cfg.lm_dim, w,
                     nullptr, false, nullptr, 0);
          E.rel(d16);
        });
      }
    } else {
      MDM_CHECK(!io->apply_lm_mask, "apply_lm_mask is only built for models with an lm_proj layer");
      cs.cond32 = const_cast<float*>(io->lm);
    }
    for (int i = 0; i < cfg.num_lm_head_layers; ++i) lm_head_fwd(L.pre + "lm_head." + std::to_string(i), B, S);
    if (stage == 0) cond_norm_fwd();
    if (!cfg.has_cond_emb) return;
    Param& cw = P(L.pre + "cond_emb.weight");
    cs.y32 = E.alloc<float>(static_cast<long long>(B) * cfg.cond_dim);
    cs.y16 = E.alloc<__half>(static_cast<long long>(B) * cfg.cond_dim);
    masked_mean(cs.cond32, cs.mask, cs.y32, cs.y16, B, S, cfg.cond_dim, E.st);
    cs.cemb = E.alloc<float>(static_cast<long long>(B) * td);
    {
      Epi e;
      e.out_f32 = cs.cemb;
      E.gemm_nt(cs.y16, cfg.cond_dim, cw.w16, cfg.cond_dim, B, td, cfg.cond_dim, e);
    }
    if (!E.training) return;
    // replayed before the LayerNorm closure of stage 0: cs.dcond starts with the pooled-mean term
    E.tape.push_back([=]() {
      if (cs.dcemb == nullptr) return;
      Engine& E = eng;
      const LevelSpec& L = levels.back();
      const long long crow = static_cast<long long>(B) * S;
      Param& cw = P(L.pre + "cond_emb.weight");
      __half* d16 = E.alloc<__half>(static_cast<long long>(B) * td);
      cast_colsum(cs.dcemb, d16, B, td, nullptr, nullptr, E.st);
      float* dy = E.alloc<float>(static_cast<long long>(B) * cfg.cond_dim);
      linear_bwd(d16, td, B, td, cfg.cond_dim, cs.y16, cfg.cond_dim, cw, nullptr, false, dy, 0);
      if (cfg.has_lm_proj || cfg.num_lm_head_layers > 0) {
        if (cs.dcond == nullptr) cs.dcond = E.alloc<float>(crow * cfg.cond_dim);
        masked_mean_bwd(dy, cs.mask, cs.dcond, cs.dcond_init ? 1 : 0, B, S, cfg.cond_dim, E.st);
        cs.dcond_init = true;
      }
      E.rel(d16);
      E.rel(dy);
    });
  }

  // LayerNorm(cond) without its affine part, once per forward: every cross-attention block folds its norm_cond affine
  // into kv_cond and reads this (unet.py:263,304). Its closure adds the blocks' gradient to cs.dcond.
  void cond_norm_fwd() {
    Engine& E = eng;
    const long long crow = static_cast<long long>(cs.B) * cs.S;
    cs.xhat16 = E.alloc<__half>(crow * cfg.cond_dim);
    cs.lnstats = E.alloc<float>(crow * 2);
    layernorm_fwd(cs.cond32, nullptr, nullptr, cs.xhat16, cs.lnstats, crow, cfg.cond_dim, E.st);
    if (!E.training) return;
    E.tape.push_back([=]() {
      if (!cs.dxhat_init) return;
      Engine& E = eng;
      if (cs.dcond == nullptr) cs.dcond = E.alloc<float>(crow * cfg.cond_dim);
      layernorm_bwd(cs.cond32, nullptr, cs.lnstats, cs.dxhat, cs.dcond, cs.dcond_init ? 1 : 0, nullptr, nullptr, nullptr,
                    crow, cfg.cond_dim, E.st);
      cs.dcond_init = true;
    });
  }

  // forward_denoising's side of the text (stage 2): the caller's tokens, pooled embedding and key mask
  void cond_input_fwd() {
    cs = CondStep();
    cs.B = io->batch;
    cs.S = io->tokens;
    cs.cd = cfg.cond_dim;
    cs.cross_mask = io->cross_mask;
    cs.cemb = const_cast<float*>(io->cond_emb);
    cs.kv_mode = io->cond_cache;
    if (cfg.cond_dim <= 0) return;
    cs.cond32 = const_cast<float*>(io->cond);
    if (cs.kv_mode != 2) cond_norm_fwd();
  }

  // One SelfAttention1DBlock of lm_head (unet.py:316-446) on the fp32 token stream cs.cond32 (B*S rows of D):
  //   x1 = x + proj_out(attn(qkv(LayerNorm(x)), mask)),  x2 = x1 + W3 gelu(W1 LayerNorm(x1) + b1) + b3
  // cs.cond32 becomes x2. The backward closure turns cs.dcond (gradient of x2) into the gradient of x, in place.
  void lm_head_fwd(const std::string& pre, int B, int S) {
    Engine& E = eng;
    const int D = cfg.cond_dim, nh = cfg.num_heads;
    const long long rows = static_cast<long long>(B) * S;
    const int irows = static_cast<int>(rows);
    const float* mask = cs.cross_mask;  // the reference passes cond_mask only with masked_cross_attention
    Param &nw = P(pre + ".attn.norm.weight"), &nb = P(pre + ".attn.norm.bias");
    Param &qw = P(pre + ".attn.qkv.weight"), &qb = P(pre + ".attn.qkv.bias");
    Param &pw = P(pre + ".attn.proj_out.weight"), &pb = P(pre + ".attn.proj_out.bias");
    Param &mw0 = P(pre + ".mlp.main.0.weight"), &mb0 = P(pre + ".mlp.main.0.bias");
    Param &mw1 = P(pre + ".mlp.main.1.weight"), &mb1 = P(pre + ".mlp.main.1.bias");
    Param &mw3 = P(pre + ".mlp.main.3.weight"), &mb3 = P(pre + ".mlp.main.3.bias");
    const float* x = cs.cond32;
    float* ln1 = E.alloc<float>(rows * 2);
    __half* xn16 = E.alloc<__half>(rows * D);
    layernorm_fwd(x, nw.w, nb.w, xn16, ln1, rows, D, E.st);
    __half* qkv = E.alloc<__half>(rows * 3 * D);
    {
      Epi e;
      e.bias = qb.w;
      e.out_f16 = qkv;
      E.gemm_nt(xn16, D, qw.w16, D, irows, 3 * D, D, e);
    }
    __half* o16 = E.alloc<__half>(rows * D);
    float* stats = E.training ? E.alloc<float>(rows * nh * 2) : nullptr;
    token_attention_forward(qkv, mask, B, S, D, nh, o16, stats, E.st);
    float* x1 = E.alloc<float>(rows * D);
    {
      Epi e;
      e.bias = pb.w;
      e.residual = x;
      e.out_f32 = x1;
      E.gemm_nt(o16, D, pw.w16, D, irows, D, D, e);
    }
    float* ln2 = E.alloc<float>(rows * 2);
    __half* y16 = E.alloc<__half>(rows * D);
    layernorm_fwd(x1, mw0.w, mb0.w, y16, ln2, rows, D, E.st);
    __half* u16 = E.training ? E.alloc<__half>(rows * 4 * D) : nullptr;  // pre-activation: only the backward needs it
    __half* g16 = E.alloc<__half>(rows * 4 * D);
    {
      Epi e;
      e.bias = mb1.w;
      e.out_f16 = u16;
      e.out_act_f16 = g16;
      e.act = ACT_GELU;
      E.gemm_nt(y16, D, mw1.w16, D, irows, 4 * D, D, e);
    }
    float* x2 = E.alloc<float>(rows * D);
    {
      Epi e;
      e.bias = mb3.w;
      e.residual = x1;
      e.out_f32 = x2;
      E.gemm_nt(g16, 4 * D, mw3.w16, 4 * D, irows, D, 4 * D, e);
    }
    cs.cond32 = x2;
    if (!E.training) {
      E.rel(ln1); E.rel(xn16); E.rel(qkv); E.rel(o16);
      E.rel(x1); E.rel(ln2); E.rel(y16); E.rel(g16);
      return;
    }
    E.tape.push_back([=]() {
      if (cs.dcond == nullptr) return;  // no gradient reached the tokens
      Engine& E = eng;
      Param &nw = P(pre + ".attn.norm.weight"), &nb = P(pre + ".attn.norm.bias");
      Param &qw = P(pre + ".attn.qkv.weight"), &qb = P(pre + ".attn.qkv.bias");
      Param &pw = P(pre + ".attn.proj_out.weight"), &pb = P(pre + ".attn.proj_out.bias");
      Param &mw0 = P(pre + ".mlp.main.0.weight"), &mb0 = P(pre + ".mlp.main.0.bias");
      Param &mw1 = P(pre + ".mlp.main.1.weight"), &mb1 = P(pre + ".mlp.main.1.bias");
      Param &mw3 = P(pre + ".mlp.main.3.weight"), &mb3 = P(pre + ".mlp.main.3.bias");
      float* g = cs.dcond;
      // MLP: dW3, then dU = (dX2 W3) * gelu'(U) straight out of the dgrad epilogue
      __half* d16 = E.alloc<__half>(rows * D);
      cast_colsum(g, d16, rows, D, mb3.g, inv_scale(), E.st);
      linear_bwd(d16, D, irows, D, 4 * D, g16, 4 * D, mw3, nullptr, false, nullptr, 0);
      __half* du16 = E.alloc<__half>(rows * 4 * D);
      {
        Epi e;
        e.out_f16 = du16;
        e.gelu_grad_src = u16;
        E.gemm_nn(d16, D, mw3.w16, 4 * D, irows, 4 * D, D, e);
      }
      E.rel(d16);
      float* dy32 = E.alloc<float>(rows * D);
      linear_bwd(du16, 4 * D, irows, 4 * D, D, y16, D, mw1, &mb1, true, dy32, 0);
      E.rel(du16);
      layernorm_bwd(x1, mw0.w, ln2, dy32, g, 1, mw0.g, mb0.g, inv_scale(), rows, D, E.st);  // g: gradient of x1
      E.rel(dy32);
      // attention: dW_proj, dO = dX1 W_proj, token attention backward, then qkv and its LayerNorm
      __half* dx16 = E.alloc<__half>(rows * D);
      cast_colsum(g, dx16, rows, D, pb.g, inv_scale(), E.st);
      linear_bwd(dx16, D, irows, D, D, o16, D, pw, nullptr, false, nullptr, 0);
      __half* do16 = E.alloc<__half>(rows * D);
      {
        Epi e;
        e.out_f16 = do16;
        E.gemm_nn(dx16, D, pw.w16, D, irows, D, D, e);
      }
      E.rel(dx16);
      __half* dqkv = E.alloc<__half>(rows * 3 * D);
      float* Dterm = E.alloc<float>(rows * nh);
      float* dq32 = E.alloc<float>(rows * D);
      token_attention_backward(qkv, mask, do16, o16, stats, B, S, D, nh, Dterm, dq32, dqkv, E.st);
      E.rel(Dterm);
      E.rel(dq32);
      E.rel(do16);
      float* dn32 = E.alloc<float>(rows * D);
      linear_bwd(dqkv, 3 * D, irows, 3 * D, D, xn16, D, qw, &qb, true, dn32, 0);
      E.rel(dqkv);
      layernorm_bwd(x, nw.w, ln1, dn32, g, 1, nw.g, nb.g, inv_scale(), rows, D, E.st);  // g: gradient of x
      E.rel(dn32);
    });
  }

  // temb of one level (unet.py:939-943 / nested_unet.py:172-176) + the level's FiLM matrix
  LevelStep* temb_fwd(const LevelSpec& L, int B) {
    Engine& E = eng;
    const int td = L.c.temporal_dim, half = td / 8;
    lsteps.emplace_back();
    LevelStep* ls = &lsteps.back();
    const long long n = static_cast<long long>(B) * td;
    __half* e16 = E.alloc<__half>(static_cast<long long>(B) * (td / 4));
    const float* freq = P(L.pre + "t_emb").w;
    sinusoid_embed(reinterpret_cast<const long long*>(io->times), nullptr, freq, B, half, 0, e16, E.st);
    MlpRec trec{};
    float* t = embed_mlp_fwd(L.pre + "temb_layer1", L.pre + "temb_layer2", e16, B, td, &trec);
    ls->temb = t;
    if (cs.cemb != nullptr) add_f32(t, t, cs.cemb, n, E.st);
    // micro-conditioning (unet.py:920-933): the keys' terms are summed in the level's order, then added to temb
    const int nkeys = L.micro.num;
    std::vector<MlpRec> mrec(nkeys);
    if (nkeys > 0) {
      MicroKeys keys = L.micro;
      for (int j = 0; j < nkeys; ++j) keys.values[j] = io->values[L.micro_slot[j]];
      const long long stride = (static_cast<long long>(B) * (td / 4) + 127) / 128 * 128;  // 256-byte aligned operands
      __half* m16 = E.alloc<__half>(stride * nkeys);
      sinusoid_embed(nullptr, &keys, freq, B, half, stride, m16, E.st);
      float* m = nullptr;
      for (int j = 0; j < nkeys; ++j) {
        float* mj = embed_mlp_fwd(L.micro_pre[j] + ".0", L.micro_pre[j] + ".1", m16 + j * stride, B, td, &mrec[j]);
        if (m == nullptr) {
          m = mj;
        } else {
          add_f32(m, m, mj, n, E.st);
          E.rel(mj);
        }
      }
      add_f32(t, t, m, n, E.st);
      E.rel(m);
    }
    ls->stemb16 = E.alloc<__half>(n);
    silu_f16(t, ls->stemb16, n, E.st);
    ls->film = E.alloc<float>(static_cast<long long>(B) * L.film_total);
    {
      Epi e;
      e.bias = L.tl_bias;
      e.out_f32 = ls->film;
      E.gemm_nt(ls->stemb16, td, L.tl_w16, td, B, L.film_total, td, e);
    }
    if (!E.training) return ls;
    ls->dstemb = E.alloc<float>(n);
    const LevelSpec* Lp = &L;
    E.tape.push_back([=]() {
      if (!ls->dstemb_init) return;
      Engine& E = eng;
      float* dt = E.alloc<float>(n);
      silu_bwd(ls->temb, ls->dstemb, dt, n, 0, E.st);
      embed_mlp_bwd(Lp->pre + "temb_layer1", Lp->pre + "temb_layer2", trec, dt, B, td);
      for (int j = 0; j < nkeys; ++j)
        embed_mlp_bwd(Lp->micro_pre[j] + ".0", Lp->micro_pre[j] + ".1", mrec[j], dt, B, td);
      if (cs.cemb != nullptr) {
        if (cs.dcemb == nullptr) cs.dcemb = E.zeros_f32(static_cast<long long>(cs.B) * td);  // whole batch
        axpy_f32(cs.dcemb, dt, 1.f, n, 1, E.st);  // this level's leading rows
        cs.dcemb_init = true;
      }
      E.rel(dt);
    });
    return ls;
  }

  // ---------------------------------------------------------------- one level (recursive for nesting)
  // Returns the pre-head feature Act; writes the level's prediction to io->out[li].
  Act* level_fwd(int li, Act* x_feat) {
    Engine& E = eng;
    const LevelSpec& L = levels[li];
    const int B = level_batch(li), H = io->res[li], W = width_of(io, li), C0 = L.c.channels[0];
    MDM_CHECK(x_feat == nullptr || x_feat->n == B, "x_feat batch");
    LevelStep* ls = temb_fwd(L, B);
    // conv_in (+ x_feat when nested)  (unet.py:867-874,946-950; nested_unet.py:184-188)
    float* inv_std = nullptr;
    if (li < cfg.num_levels - 1 && !L.c.skip_normalization) {
      inv_std = E.alloc<float>(B);
      sample_inv_std(io->x_t[li], inv_std, B, static_cast<long long>(cfg.in_channels) * H * W, E.st);
    }
    const long long rows = static_cast<long long>(B) * H * W;
    __half* col = E.alloc<__half>(rows * 32);
    im2col_input(io->x_t[li], inv_std, col, B, cfg.in_channels, H, W, E.st);
    Param &ciw = P(L.pre + "conv_in.weight"), &cib = P(L.pre + "conv_in.bias");
    Act* x = E.new_act(B, H, W, C0);
    {
      Epi e;
      e.bias = cib.w;
      e.residual = x_feat != nullptr ? x_feat->p : nullptr;
      e.out_f32 = x->p;
      E.gemm_nt(col, 32, ciw.w16, 32, static_cast<int>(rows), C0, 32, e);
    }
    debug_acts[L.pre + "conv_in"] = x;
    if (E.training) {
      const LevelSpec* Lp = &L;
      E.tape.push_back([=]() {
        if (x->g == nullptr) return;
        Engine& E = eng;
        Param &ciw = P(Lp->pre + "conv_in.weight"), &cib = P(Lp->pre + "conv_in.bias");
        __half* d16 = E.alloc<__half>(rows * C0);
        cast_colsum(x->g, d16, rows, C0, cib.g, inv_scale(), E.st);
        if (ciw.g != nullptr) {
          float* wtmp = E.zeros_f32(static_cast<long long>(C0) * 32);
          Epi e;
          e.out_f32 = wtmp;
          e.atomic_ok = true;
          E.gemm_tn(d16, C0, col, 32, C0, 32, static_cast<int>(rows), e);
          unpack_conv_in_wgrad(wtmp, ciw.g, C0, cfg.in_channels, inv_scale(), E.st);
          E.rel(wtmp);
        }
        if (x_feat != nullptr) {
          int acc = 0;
          float* g = E.grad_buf(x_feat, &acc);
          axpy_f32(g, x->g, 1.f, x->numel(), acc, E.st);
        }
        E.rel(d16);
        E.rel(x->g);
      });
    } else {
      E.rel(col);
    }

    // down path
    std::vector<Act*> skips{x};
    for (auto& b : L.down) {
      std::vector<Act*> acts;
      x = block_fwd(L, ls, b, x, nullptr, &acts);
      skips.insert(skips.end(), acts.begin(), acts.end());
    }
    // middle: own mid blocks, or the inner U-Net between the adapters
    if (li == cfg.num_levels - 1) {
      for (auto& b : L.mid) x = block_fwd(L, ls, b, x, nullptr, nullptr);
    } else {
      MDM_CHECK(L.mid.empty(), "outer levels of a nest have no mid blocks");
      const int N = x->n, Hb = x->h, Wb = x->w, Co = x->c;
      const int Ci = levels[li + 1].c.channels[0];
      MDM_CHECK(Hb == io->res[li + 1] && Wb == width_of(io, li + 1),
                "outer bottleneck resolution must equal the inner image size (both sides)");
      __half* x16 = E.alloc<__half>(x->numel());
      cast_f32_to_f16(x->p, x16, x->numel(), E.st);
      const int Bin = level_batch(li + 1);  // >= N; the inner level's extra samples see a zero feature
      MDM_CHECK(Bin >= N, "level_batch must not decrease from outer to inner levels");
      Act* xin = conv_act(L.pre + "in_adapter.weight", L.pre + "in_adapter.bias", x16, N, Hb, Wb, Co, Ci, nullptr, Bin);
      Act* xo_in = x;
      if (E.training) {
        const LevelSpec* Lp = &L;
        E.tape.push_back([=]() {
          if (xin->g == nullptr) return;
          Engine& E = eng;
          float* dx16 = conv_act_bwd(Lp->pre + "in_adapter.weight", Lp->pre + "in_adapter.bias", x16, xin, Co, N);
          int acc = 0;
          float* g = E.grad_buf(xo_in, &acc);
          axpy_f32(g, dx16, 1.f, xo_in->numel(), acc, E.st);
          E.rel(dx16);
          E.rel(xin->g);
        });
      } else {
        E.rel(x16);
      }
      Act* feat = level_fwd(li + 1, xin);
      // out_adapter on the leading N samples only: the reference convolves all Bin and slices [:N] (nested_unet.py:208-209),
      // so the dropped rows contribute neither to the output nor to any gradient
      const long long lead = static_cast<long long>(N) * Hb * Wb * Ci;
      __half* f16 = E.alloc<__half>(lead);
      cast_f32_to_f16(feat->p, f16, lead, E.st);
      Act* xn = conv_act(L.pre + "out_adapter.weight", L.pre + "out_adapter.bias", f16, N, Hb, Wb, Ci, Co, x->p);
      if (E.training) {
        const LevelSpec* Lp = &L;
        E.tape.push_back([=]() {
          if (xn->g == nullptr) return;
          Engine& E = eng;
          float* df = conv_act_bwd(Lp->pre + "out_adapter.weight", Lp->pre + "out_adapter.bias", f16, xn, Ci);
          int acc = 0;
          float* g = E.grad_buf(feat, &acc);
          axpy_f32(g, df, 1.f, lead, acc, E.st);
          if (!acc && feat->numel() > lead)
            MDM_CUDA(cudaMemsetAsync(g + lead, 0, sizeof(float) * (feat->numel() - lead), E.st));
          E.rel(df);
          g = E.grad_buf(xo_in, &acc);
          axpy_f32(g, xn->g, 1.f, xo_in->numel(), acc, E.st);
          E.rel(xn->g);
        });
      } else {
        E.rel(f16);
      }
      x = xn;
    }
    // up path
    for (auto& b : L.up) {
      const size_t n = b.res.size();
      std::vector<Act*> sk(skips.end() - n, skips.end());
      std::reverse(sk.begin(), sk.end());
      skips.resize(skips.size() - n);
      x = block_fwd(L, ls, b, x, &sk, nullptr);
    }
    // head (unet.py:876-880)
    Act* feat = x;
    {
      const int Cf = feat->c, HW = H * W;
      Param &nw = P(L.pre + "norm_out.weight"), &nb = P(L.pre + "norm_out.bias");
      Param &ow = P(L.pre + "conv_out.weight"), &ob = P(L.pre + "conv_out.bias");
      GnOut g = gn_fwd(Src2{feat->p, nullptr, Cf, 0}, B, HW, L.c.groups, nw, nb, nullptr, 0, 0, 1, false);
      const int oc = cfg.out_channels;
      float* o = E.alloc<float>(rows * oc);
      Epi e;
      e.bias = ob.w;
      e.out_f32 = o;
      E.conv3x3_fwd(g.y16, Cf, B, H, W, Cf, ow.w16, oc, e, ow.w16f, ow.bias_f);
      // model_output_scale: s * tanh(o / s) on the way out; a training forward keeps that output for the backward seed
      const float s = io->output_scale;
      float* keep = s != 0.f && E.training ? E.alloc<float>(rows * oc) : nullptr;
      nhwc_to_nchw(o, oc, io->out[li], B, oc, HW, E.st, s, keep);
      E.rel(o);
      outs[li].h = H;
      outs[li].w = W;
      outs[li].batch = B;
      outs[li].scale = s;
      outs[li].y = keep;
      if (E.training) {
        const LevelSpec* Lp = &L;
        OutRec* orec = &outs[li];
        E.tape.push_back([=]() {
          if (orec->d16 == nullptr) return;  // no gradient supplied for this level
          Engine& E = eng;
          Param &nw = P(Lp->pre + "norm_out.weight"), &nb = P(Lp->pre + "norm_out.bias");
          Param &ow = P(Lp->pre + "conv_out.weight"), &ob = P(Lp->pre + "conv_out.bias");
          float* bs = E.zeros_f32(8);
          colsum_f16(orec->d16, rows, 8, bs, inv_scale(), E.st);
          if (ob.g != nullptr) axpy_f32(ob.g, bs, 1.f, oc, 1, E.st);
          if (ow.g != nullptr) {
            float* wtmp = E.alloc<float>(9ll * Cf * oc);
            E.conv3x3_wgrad(orec->d16, 8, g.y16, Cf, B, H, W, Cf, oc, wtmp);
            unpack_conv_wgrad(wtmp, ow.g, oc, Cf, 9, Cf, inv_scale(), E.st);
            E.rel(wtmp);
          }
          float* da = E.alloc<float>(rows * Cf);
          Epi e;
          e.out_f32 = da;
          E.conv3x3_dgrad(orec->d16, 8, B, H, W, oc, ow.w16, Cf, e);
          gn_bwd(Src2{feat->p, nullptr, Cf, 0}, da, false, B, HW, Lp->c.groups, g.sums, nw, nb, nullptr, 0, 0, 1, nullptr,
                 nullptr, feat, nullptr);
          E.rel(da);
          E.rel(bs);
        });
      } else {
        E.rel(g.y16);
        E.rel(g.sums);
      }
    }
    return feat;
  }

  // ---------------------------------------------------------------- entry points
  void forward_body(const StepIO* io_, cudaStream_t st) {
    eng.st = st;
    eng.training = io_->save_for_backward != 0;
    eng.tape.clear();
    eng.acts.clear();
    eng.pool.reset();
    lsteps.clear();
    debug_acts.clear();
    have_tape = false;
    io = io_;
    for (int l = 0; l < MDM_MAX_LEVELS; ++l) outs[l] = OutRec();
    MDM_CHECK(io->batch > 0, "batch");
    MDM_CHECK(level_batch(cfg.num_levels - 1) == io->batch, "the innermost level runs the whole batch");
    for (int l = 0; l < cfg.num_levels; ++l) {
      MDM_CHECK(level_batch(l) >= 1 && level_batch(l) <= io->batch, "level_batch out of range");
      MDM_CHECK(io->x_t[l] != nullptr && io->out[l] != nullptr, "missing x_t/out pointer");
      const int f = 1 << (cfg.levels[l].num_res - 1);
      MDM_CHECK(io->res[l] > 0 && io->res_w[l] >= 0 && io->res[l] % f == 0 && width_of(io, l) % f == 0,
                "image height and width must both divide by the level's downsampling");
    }
    if (cfg.cond_dim > 0 && io->stage == 0) MDM_CHECK(io->lm != nullptr && io->tokens > 0, "conditioning required");
    if (cfg.cond_dim > 0 && io->stage == 2)
      MDM_CHECK(io->tokens > 0 && (io->cond != nullptr || io->cond_cache == 2), "stage 2 needs cond (batch, tokens, cond_dim)");
    tape_stage = io->stage;
    {  // weight gradients on a side stream (engine.cuh); MDM_SIDE_WGRAD=0 keeps everything on one stream
      static const char* sw = getenv("MDM_SIDE_WGRAD");
      eng.side_enabled = sw != nullptr ? atoi(sw) != 0 : true;
      eng.ev_next = 0;
    }
    eng.single_plane = io->single_plane != 0;
    tape_single = eng.single_plane;
    prepare_weights(eng.single_plane);
    if (io->stage == 2) cond_input_fwd();
    else conditioning_fwd(0);
    level_fwd(0, nullptr);
    have_tape = eng.training;
    io = nullptr;
  }

  void backward_body(const mdm_net_grad_io* gio, cudaStream_t st) {
    MDM_CHECK(have_tape, "mdm_net_backward needs a preceding forward with save_for_backward=1");
    eng.st = st;
    eng.single_plane = tape_single;
    // gradient scale from the largest |dout| (fp16 operands need the seed in range)
    MDM_CUDA(cudaMemsetAsync(eng.d_amax, 0, sizeof(float), st));
    for (int l = 0; l < cfg.num_levels; ++l) {
      if (gio->dout[l] == nullptr) continue;
      const long long n = static_cast<long long>(outs[l].batch) * cfg.out_channels * outs[l].h * outs[l].w;
      // with model_output_scale the seed is dout * (1 - (y / s)^2): the power-of-two scale is chosen from that product
      grad_amax(gio->dout[l], n, eng.d_amax, st, outs[l].scale, outs[l].y);
    }
    grad_scale_finalize(eng.d_amax, eng.d_scale, eng.d_inv_scale, st);
    for (int l = 0; l < cfg.num_levels; ++l) {
      if (gio->dout[l] == nullptr) continue;
      const int HW = outs[l].h * outs[l].w;
      const int B = outs[l].batch;
      outs[l].d16 = eng.alloc<__half>(static_cast<long long>(B) * HW * 8);
      nchw_to_nhwc_f16(gio->dout[l], eng.d_scale, outs[l].d16, 8, B, cfg.out_channels, HW, st, outs[l].scale, outs[l].y);
      if (outs[l].y != nullptr) {
        eng.rel(outs[l].y);
        outs[l].y = nullptr;
      }
    }
    replay_tape(tape_stage == 0);
    if (tape_stage == 2) {  // gradients of the caller's cond / cond_emb, unscaled
      const long long n = static_cast<long long>(cs.B) * cs.S * cfg.cond_dim;
      if (gio->dcond != nullptr && n > 0) {
        if (cs.dcond_init) scale_f32(gio->dcond, cs.dcond, eng.d_inv_scale, n, st);
        else MDM_CUDA(cudaMemsetAsync(gio->dcond, 0, sizeof(float) * n, st));
      }
      if (gio->dcond_emb != nullptr && cs.cemb != nullptr) {
        const long long m = static_cast<long long>(cs.B) * levels.back().c.temporal_dim;
        if (cs.dcemb != nullptr) scale_f32(gio->dcond_emb, cs.dcemb, eng.d_inv_scale, m, st);
        else MDM_CUDA(cudaMemsetAsync(gio->dcond_emb, 0, sizeof(float) * m, st));
      }
    }
    eng.tape.clear();
    have_tape = false;
  }

  // ---------------------------------------------------------------- stage 1: forward_conditioning alone
  // Runs beside a held stage-0/2 tape (and any captured graph): on text_pool, with a tape of its own, and restores the
  // held state when done. Its backward recomputes the text path from the recorded inputs and replays that tape at
  // once, so the two stages' backwards can come in either order.
  struct TextScope {
    Net* n;
    std::vector<std::function<void()>> tape;
    CondStep cs;
    const StepIO* io;
    bool training, single;
    TextScope(Net* net, bool train, bool single_plane)
        : n(net), cs(net->cs), io(net->io), training(net->eng.training), single(net->eng.single_plane) {
      tape.swap(n->eng.tape);
      n->eng.training = train;
      n->eng.single_plane = single_plane;
      n->text_pool.reset();
      n->eng.alt = &n->text_pool;
    }
    ~TextScope() {
      n->eng.alt = nullptr;
      n->eng.tape.swap(tape);
      n->cs = cs;
      n->io = io;
      n->eng.training = training;
      n->eng.single_plane = single;
    }
  };

  void stage1_forward(const StepIO* q, cudaStream_t st) {
    MDM_CHECK(cfg.cond_dim > 0, "stage 1 needs a model with text conditioning (conditioning_feature_dim > 0)");
    MDM_CHECK(q->batch > 0 && q->tokens > 0 && q->lm != nullptr && q->cond_out != nullptr,
              "stage 1 needs batch, tokens, lm and cond_out");
    MDM_CHECK(!cfg.has_cond_emb || q->cond_emb_out != nullptr, "stage 1 needs cond_emb_out: the model has cond_emb");
    have_cond_io = false;
    eng.st = st;
    {
      TextScope scope(this, false, q->single_plane != 0);
      prepare_weights(q->single_plane != 0);
      io = q;
      conditioning_fwd(1);
      const long long n = static_cast<long long>(q->batch) * q->tokens * cfg.cond_dim;
      MDM_CUDA(cudaMemcpyAsync(q->cond_out, cs.cond32, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
      if (cs.cemb != nullptr)
        MDM_CUDA(cudaMemcpyAsync(q->cond_emb_out, cs.cemb,
                                 sizeof(float) * q->batch * levels.back().c.temporal_dim, cudaMemcpyDeviceToDevice, st));
    }
    if (q->save_for_backward) {
      cond_io = *q;
      have_cond_io = true;
    }
  }

  void stage1_backward(const mdm_net_grad_io* gio, cudaStream_t st) {
    MDM_CHECK(have_cond_io, "a stage-1 backward needs a preceding stage-1 forward with save_for_backward=1");
    have_cond_io = false;
    eng.st = st;
    TextScope scope(this, true, cond_io.single_plane != 0);  // the mode of the forward it differentiates
    prepare_weights(cond_io.single_plane != 0);
    io = &cond_io;
    conditioning_fwd(1);
    Engine& E = eng;
    const long long n = static_cast<long long>(cs.B) * cs.S * cfg.cond_dim;
    const long long m = static_cast<long long>(cs.B) * levels.back().c.temporal_dim;
    // one gradient scale for both incoming gradients, derived as backward_body derives it from the output gradients
    MDM_CUDA(cudaMemsetAsync(E.d_amax, 0, sizeof(float), st));
    if (gio->dcond_in != nullptr) grad_amax(gio->dcond_in, n, E.d_amax, st);
    if (gio->dcond_emb_in != nullptr && cs.cemb != nullptr) grad_amax(gio->dcond_emb_in, m, E.d_amax, st);
    grad_scale_finalize(E.d_amax, E.d_scale, E.d_inv_scale, st);
    cs.dcond = E.alloc<float>(n);
    if (gio->dcond_in != nullptr) scale_f32(cs.dcond, gio->dcond_in, E.d_scale, n, st);
    else MDM_CUDA(cudaMemsetAsync(cs.dcond, 0, sizeof(float) * n, st));
    cs.dcond_init = true;
    if (cs.cemb != nullptr) {
      cs.dcemb = E.alloc<float>(m);
      if (gio->dcond_emb_in != nullptr) scale_f32(cs.dcemb, gio->dcond_emb_in, E.d_scale, m, st);
      else MDM_CUDA(cudaMemsetAsync(cs.dcemb, 0, sizeof(float) * m, st));
    }
    for (int i = static_cast<int>(E.tape.size()) - 1; i >= 0; --i) {
      E.tape[i]();
      E.side_join();
    }
  }

  // ---------------------------------------------------------------- K/V cache (mdm_net_stage_io.cond_cache)
  void kv_cache_begin(const StepIO* q) {
    if (q->cond_cache == 0) return;
    int key[2 + MDM_MAX_LEVELS] = {q->batch, q->tokens, 0, 0, 0, 0};
    for (int l = 0; l < cfg.num_levels; ++l) key[2 + l] = level_batch_of(q, l);
    if (q->cond_cache == 2) {
      if (!kv_valid)
        throw MdmFail("cond_cache 2: the K/V cache holds nothing valid (fill it with a cond_cache 1 forward; weight "
                      "changes and rebinding parameters invalidate it)");
      if (memcmp(key, kv_key, sizeof(key)) != 0)
        throw MdmFail("cond_cache 2: the K/V cache was filled for batch " + std::to_string(kv_key[0]) + ", tokens " +
                      std::to_string(kv_key[1]) + " (level batches " + std::to_string(kv_key[2]) + "..); this call has batch " +
                      std::to_string(q->batch) + ", tokens " + std::to_string(q->tokens));
      if (kv_single != (q->single_plane != 0))
        throw MdmFail(std::string("cond_cache 2: the K/V cache was filled by a ") + (kv_single ? "single" : "two") +
                      "-plane forward; this call is " + (q->single_plane ? "single" : "two") +
                      "-plane (mdm_net_io.single_plane): fill it again with cond_cache 1");
      return;
    }
    kv_valid = false;
    const size_t need = static_cast<size_t>(q->batch) * q->tokens * kv_row;
    if (need > kv_cap) {
      if (kv_cache != nullptr) MDM_CUDA(cudaDeviceSynchronize());  // replayed graphs may still read the old slot
      cudaFree(kv_cache);
      kv_cache = nullptr;
      kv_cap = 0;
      MDM_CUDA(cudaMalloc(&kv_cache, need * sizeof(__half)));
      kv_cap = need;
      ++kv_epoch;
    }
    memcpy(kv_key, key, sizeof(key));
    kv_single = q->single_plane != 0;
  }
  static int level_batch_of(const mdm_net_io* q, int l) { return q->level_batch[l] > 0 ? q->level_batch[l] : q->batch; }


  // ---------------------------------------------------------------- CUDA graphs
  // One step is ~1-2.5 k launches. With graph mode on, the second call with a given shape signature is captured
  // (forward and backward separately, on an internal stream -- torch's default stream is the legacy stream, which
  // cannot capture) and later calls replay it: inputs are staged into per-signature static buffers, the graph is
  // launched on the caller's stream, outputs are copied out. The first call of a signature runs eagerly and sizes the
  // pool; pool addresses, TMA descriptors and gradient pointers are baked into the graph, so anything that moves them
  // (rebinding parameters, the pool returning memory to the driver) drops the recorded graphs.
  struct GraphRec {
    int training = 0, batch = 0, tokens = 0, has_mask = 0, apply_lm_mask = 0, dropout = 0;
    int micro_mask = 0;  // bit k: the micro table's key k has values (staged in micro[k])
    int stage = 0, cond_cache = 0, has_cemb = 0;  // stage 2: the K/V cache mode and whether cond_emb is given
    uint64_t kv_epoch = 0;
    int lb[MDM_MAX_LEVELS] = {0, 0, 0, 0}, res[MDM_MAX_LEVELS] = {0, 0, 0, 0}, res_w[MDM_MAX_LEVELS] = {0, 0, 0, 0};
    float output_scale = 0.f;  // baked into the head kernels' arguments
    int single_plane = 0;      // which kernels and operand planes the weight products were captured with
    uint64_t bind_epoch = 0, pool_epoch = 0;
    float* x_t[MDM_MAX_LEVELS] = {nullptr, nullptr, nullptr, nullptr};
    float* out[MDM_MAX_LEVELS] = {nullptr, nullptr, nullptr, nullptr};
    float* dout[MDM_MAX_LEVELS] = {nullptr, nullptr, nullptr, nullptr};
    size_t x_bytes[MDM_MAX_LEVELS] = {0, 0, 0, 0};
    long long* times = nullptr;
    float *lm = nullptr, *mask = nullptr;  // mask: lm_mask (stage 0) or cross_mask (stage 2)
    float* micro[MDM_MAX_MICRO] = {};
    size_t lm_bytes = 0, mask_bytes = 0;
    float *cond = nullptr, *cemb = nullptr, *dcond = nullptr, *dcemb = nullptr;  // stage 2
    size_t cond_bytes = 0, cemb_bytes = 0;
    cudaGraphExec_t fwd = nullptr;
    // backward: one graph, or -- with a gradient-ready callback installed -- one graph per reported range, so the
    // caller's collective on range i is enqueued right after segment i and overlaps segments i+1..
    std::vector<cudaGraphExec_t> bwd;
    std::vector<std::pair<uintptr_t, uintptr_t>> bwd_ranges;  // (lo, hi) reported after segment i; (0, 0): none
    bool bwd_notifies = false;
    unsigned long long fwd_kernels = 0, bwd_kernels = 0;
    int dout_mask = 0;
    int seen = 0;
    uint64_t last_use = 0;
  };
  std::vector<GraphRec> graphs;
  bool graph_mode = false;
  int active_graph = -1;  // record whose forward ran last (its backward replays/captures), -1: eager
  uint64_t bind_epoch = 1, use_clock = 0;
  cudaStream_t cap_st = nullptr;
  int rebinds_while_graphed = 0;

  void drop_graph(GraphRec& r) {
    if (r.fwd != nullptr) cudaGraphExecDestroy(r.fwd);
    for (cudaGraphExec_t g : r.bwd) cudaGraphExecDestroy(g);
    r.fwd = nullptr;
    r.bwd.clear();
    r.bwd_ranges.clear();
  }
  void free_rec(GraphRec& r) {
    drop_graph(r);
    for (int l = 0; l < MDM_MAX_LEVELS; ++l) {
      cudaFree(r.x_t[l]);
      cudaFree(r.out[l]);
      cudaFree(r.dout[l]);
    }
    cudaFree(r.times);
    cudaFree(r.lm);
    cudaFree(r.mask);
    for (float* m : r.micro) cudaFree(m);
    cudaFree(r.cond);
    cudaFree(r.cemb);
    cudaFree(r.dcond);
    cudaFree(r.dcemb);
  }
  static const float* key_mask(const StepIO* q) { return q->stage == 2 ? q->cross_mask : q->lm_mask; }
  int micro_mask(const StepIO* q) const {
    int m = 0;
    for (int k = 0; k < micro.num_keys; ++k)
      if (q->values[k] != nullptr) m |= 1 << k;
    return m;
  }
  bool same_key(const GraphRec& r, const StepIO* q) const {
    if (r.training != (q->save_for_backward != 0) || r.batch != q->batch || r.tokens != q->tokens ||
        r.apply_lm_mask != (q->apply_lm_mask != 0) || r.dropout != (q->dropout != 0) ||
        r.has_mask != (key_mask(q) != nullptr) || r.micro_mask != micro_mask(q) || r.stage != q->stage ||
        r.cond_cache != q->cond_cache || r.has_cemb != (q->stage == 2 && q->cond_emb != nullptr) ||
        r.output_scale != q->output_scale || r.single_plane != (q->single_plane != 0))
      return false;
    // both sides: a 32x48 and a 48x32 input move the same number of bytes but run different kernels
    for (int l = 0; l < cfg.num_levels; ++l)
      if (r.res[l] != q->res[l] || r.res_w[l] != width_of(q, l) ||
          r.lb[l] != (q->level_batch[l] > 0 ? q->level_batch[l] : q->batch))
        return false;
    return true;
  }
  int find_rec(const StepIO* q) {
    for (size_t i = 0; i < graphs.size(); ++i)
      if (same_key(graphs[i], q)) return static_cast<int>(i);
    if (graphs.size() >= 6) {  // bounded cache: evict the least recently used signature
      size_t v = 0;
      for (size_t i = 1; i < graphs.size(); ++i)
        if (graphs[i].last_use < graphs[v].last_use) v = i;
      free_rec(graphs[v]);
      graphs.erase(graphs.begin() + v);
    }
    GraphRec r;
    r.training = q->save_for_backward != 0;
    r.batch = q->batch;
    r.tokens = q->tokens;
    r.has_mask = key_mask(q) != nullptr;
    r.micro_mask = micro_mask(q);
    r.stage = q->stage;
    r.cond_cache = q->cond_cache;
    r.has_cemb = q->stage == 2 && q->cond_emb != nullptr;
    r.apply_lm_mask = q->apply_lm_mask != 0;
    r.dropout = q->dropout != 0;
    r.output_scale = q->output_scale;
    r.single_plane = q->single_plane != 0;
    for (int l = 0; l < cfg.num_levels; ++l) {
      r.res[l] = q->res[l];
      r.res_w[l] = width_of(q, l);
      r.lb[l] = q->level_batch[l] > 0 ? q->level_batch[l] : q->batch;
      r.x_bytes[l] = sizeof(float) * static_cast<size_t>(r.lb[l]) * cfg.in_channels * r.res[l] * r.res_w[l];
      MDM_CUDA(cudaMalloc(&r.x_t[l], r.x_bytes[l]));
      MDM_CUDA(cudaMalloc(&r.out[l], r.x_bytes[l] / cfg.in_channels * cfg.out_channels));
      if (r.training) MDM_CUDA(cudaMalloc(&r.dout[l], r.x_bytes[l] / cfg.in_channels * cfg.out_channels));
    }
    MDM_CUDA(cudaMalloc(&r.times, sizeof(long long) * r.batch));
    if (q->stage == 0 && q->lm != nullptr) {
      r.lm_bytes = sizeof(float) * static_cast<size_t>(r.batch) * r.tokens * cfg.lm_dim;
      MDM_CUDA(cudaMalloc(&r.lm, r.lm_bytes));
    }
    if (q->stage == 2 && cfg.cond_dim > 0) {
      r.cond_bytes = sizeof(float) * static_cast<size_t>(r.batch) * r.tokens * cfg.cond_dim;
      if (q->cond_cache != 2) MDM_CUDA(cudaMalloc(&r.cond, r.cond_bytes));  // mode 2 does not read cond
      if (r.training) MDM_CUDA(cudaMalloc(&r.dcond, r.cond_bytes));
    }
    if (r.has_cemb) {
      r.cemb_bytes = sizeof(float) * static_cast<size_t>(r.batch) * levels.back().c.temporal_dim;
      MDM_CUDA(cudaMalloc(&r.cemb, r.cemb_bytes));
      if (r.training) MDM_CUDA(cudaMalloc(&r.dcemb, r.cemb_bytes));
    }
    if (r.has_mask) {
      r.mask_bytes = sizeof(float) * static_cast<size_t>(r.batch) * r.tokens;
      MDM_CUDA(cudaMalloc(&r.mask, r.mask_bytes));
    }
    for (int k = 0; k < micro.num_keys; ++k)
      if ((r.micro_mask >> k) & 1) MDM_CUDA(cudaMalloc(&r.micro[k], sizeof(float) * r.batch));
    graphs.push_back(r);
    return static_cast<int>(graphs.size()) - 1;
  }
  cudaGraphExec_t end_capture() {
    cudaGraph_t g = nullptr;
    MDM_CUDA(cudaStreamEndCapture(cap_st, &g));
    cudaGraphExec_t ex = nullptr;
    cudaError_t e = cudaGraphInstantiate(&ex, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) throw MdmFail(std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e));
    return ex;
  }
  void abort_capture() {
    cudaStreamCaptureStatus stt = cudaStreamCaptureStatusNone;
    if (cap_st != nullptr && cudaStreamIsCapturing(cap_st, &stt) == cudaSuccess && stt != cudaStreamCaptureStatusNone) {
      cudaGraph_t g = nullptr;
      cudaStreamEndCapture(cap_st, &g);
      if (g != nullptr) cudaGraphDestroy(g);
    }
    (void)cudaGetLastError();
  }

  void forward(const StepIO* io_, cudaStream_t st) {
    if (io_->stage == 1) {  // eager: once per sampling run / training step, and it leaves any held tape alone
      stage1_forward(io_, st);
      return;
    }
    MDM_CHECK(io_->stage == 0 || io_->stage == 2, "mdm_net_stage_io.stage must be 0, 1 or 2");
    MDM_CHECK(io_->cond_cache >= 0 && io_->cond_cache <= 2, "mdm_net_stage_io.cond_cache must be 0, 1 or 2");
    MDM_CHECK(io_->cond_cache == 0 || (io_->stage == 2 && !io_->save_for_backward),
              "cond_cache applies to stage-2 forwards without save_for_backward");
    kv_cache_begin(io_);
    forward_pass(io_, st);
    if (io_->cond_cache == 1) kv_valid = true;
  }

  void forward_pass(const StepIO* io_, cudaStream_t st) {
    active_graph = -1;
    // on the caller's stream ahead of the eager, captured or replayed pass: the kernels read the seed from its slot
    if (io_->dropout) dropout_set_seed(eng.d_drop_seed, io_->dropout_seed, st);
    if (!graph_mode || g_profile) {
      forward_body(io_, st);
      return;
    }
    const int idx = find_rec(io_);
    GraphRec& r = graphs[idx];
    r.last_use = ++use_clock;
    if (r.seen == 0) {  // first call of this signature: eager, sizes the pool
      r.seen = 1;
      forward_body(io_, st);
      return;
    }
    // stage the inputs at the addresses the graph reads
    for (int l = 0; l < cfg.num_levels; ++l)
      MDM_CUDA(cudaMemcpyAsync(r.x_t[l], io_->x_t[l], r.x_bytes[l], cudaMemcpyDeviceToDevice, st));
    MDM_CUDA(cudaMemcpyAsync(r.times, io_->times, sizeof(long long) * r.batch, cudaMemcpyDeviceToDevice, st));
    if (r.lm != nullptr) MDM_CUDA(cudaMemcpyAsync(r.lm, io_->lm, r.lm_bytes, cudaMemcpyDeviceToDevice, st));
    if (r.has_mask) MDM_CUDA(cudaMemcpyAsync(r.mask, key_mask(io_), r.mask_bytes, cudaMemcpyDeviceToDevice, st));
    if (r.cond != nullptr) MDM_CUDA(cudaMemcpyAsync(r.cond, io_->cond, r.cond_bytes, cudaMemcpyDeviceToDevice, st));
    if (r.cemb != nullptr) MDM_CUDA(cudaMemcpyAsync(r.cemb, io_->cond_emb, r.cemb_bytes, cudaMemcpyDeviceToDevice, st));
    for (int k = 0; k < micro.num_keys; ++k)
      if (r.micro[k] != nullptr)
        MDM_CUDA(cudaMemcpyAsync(r.micro[k], io_->values[k], sizeof(float) * r.batch, cudaMemcpyDeviceToDevice, st));
    eng.st = st;
    prepare_weights(io_->single_plane != 0);  // outside the graph: only when the masters changed or lo planes are stale
    const bool valid = r.fwd != nullptr && r.bind_epoch == bind_epoch && r.pool_epoch == eng.pool.epoch() &&
                       (r.cond_cache == 0 || r.kv_epoch == kv_epoch) &&
                       (!r.training || (!r.bwd.empty() && r.bwd_notifies == (ready_fn != nullptr)));
    if (!valid) {
      drop_graph(r);
      if (cap_st == nullptr) MDM_CUDA(cudaStreamCreateWithFlags(&cap_st, cudaStreamNonBlocking));
      StepIO sio = *io_;
      for (int l = 0; l < cfg.num_levels; ++l) {
        sio.x_t[l] = r.x_t[l];
        sio.out[l] = r.out[l];
      }
      sio.times = reinterpret_cast<const int64_t*>(r.times);
      sio.lm = r.lm;
      if (r.stage == 2) {
        sio.cond = r.cond;
        sio.cond_emb = r.cemb;
        sio.cross_mask = r.has_mask ? r.mask : nullptr;
      } else {
        sio.lm_mask = r.has_mask ? r.mask : nullptr;
      }
      for (int k = 0; k < MDM_MAX_MICRO; ++k) sio.values[k] = r.micro[k];
      const unsigned long long k0 = g_launch_count;
      MDM_CUDA(cudaStreamBeginCapture(cap_st, cudaStreamCaptureModeRelaxed));
      try {
        forward_body(&sio, cap_st);
        r.fwd = end_capture();
      } catch (...) {
        abort_capture();
        eng.st = st;
        throw;
      }
      r.fwd_kernels = g_launch_count - k0;
      g_launch_count = k0;
      r.bind_epoch = bind_epoch;
      r.pool_epoch = eng.pool.epoch();
      r.kv_epoch = kv_epoch;
      eng.st = st;
    }
    MDM_CUDA(cudaGraphLaunch(r.fwd, st));
    g_launch_count += r.fwd_kernels;
    ++g_graph_launches;
    for (int l = 0; l < cfg.num_levels; ++l)
      MDM_CUDA(cudaMemcpyAsync(io_->out[l], r.out[l], r.x_bytes[l] / cfg.in_channels * cfg.out_channels,
                               cudaMemcpyDeviceToDevice, st));
    active_graph = idx;
  }

  void backward(const mdm_net_grad_io* gio, cudaStream_t st) {
    if (gio->stage == 1) {
      stage1_backward(gio, st);
      return;
    }
    if (active_graph < 0) {
      backward_body(gio, st);
      return;
    }
    GraphRec& r = graphs[active_graph];
    active_graph = -1;
    MDM_CHECK(r.training, "mdm_net_backward needs a preceding forward with save_for_backward=1");
    int mask = 0;
    for (int l = 0; l < cfg.num_levels; ++l) {
      if (gio->dout[l] == nullptr) continue;
      mask |= 1 << l;
      MDM_CUDA(cudaMemcpyAsync(r.dout[l], gio->dout[l], r.x_bytes[l] / cfg.in_channels * cfg.out_channels,
                               cudaMemcpyDeviceToDevice, st));
    }
    if (r.bwd.empty()) {
      MDM_CHECK(have_tape, "graph mode: no recorded tape for this backward");
      mdm_net_grad_io sg{};
      for (int l = 0; l < cfg.num_levels; ++l) sg.dout[l] = (mask >> l) & 1 ? r.dout[l] : nullptr;
      sg.dcond = r.dcond;
      sg.dcond_emb = r.dcemb;
      const unsigned long long k0 = g_launch_count;
      MDM_CUDA(cudaStreamBeginCapture(cap_st, cudaStreamCaptureModeRelaxed));
      eng.capturing = true;  // weight gradients may fork onto the side stream (graph branches)
      try {
        // a reported range closes the current segment: its graph ends here and the next one begins
        seg_cut = [&](uintptr_t lo, uintptr_t hi) {
          r.bwd.push_back(end_capture());
          r.bwd_ranges.emplace_back(lo, hi);
          MDM_CUDA(cudaStreamBeginCapture(cap_st, cudaStreamCaptureModeRelaxed));
        };
        backward_body(&sg, cap_st);
        seg_cut = nullptr;
        eng.capturing = false;
        r.bwd.push_back(end_capture());
        r.bwd_ranges.emplace_back(0, 0);
      } catch (...) {
        seg_cut = nullptr;
        eng.capturing = false;
        abort_capture();
        drop_graph(r);
        eng.st = st;
        throw;
      }
      r.bwd_kernels = g_launch_count - k0;
      g_launch_count = k0;
      r.dout_mask = mask;
      r.bwd_notifies = ready_fn != nullptr;
      eng.st = st;
      if (r.pool_epoch != eng.pool.epoch()) {  // the pool grew by freeing cached blocks: addresses in the forward graph died
        drop_graph(r);
        throw MdmFail("graph mode: device memory pool was trimmed during capture; retry the step");
      }
    } else {
      MDM_CHECK(mask == r.dout_mask, "graph mode: the set of output gradients changed between steps");
      MDM_CHECK(r.bind_epoch == bind_epoch, "graph mode: parameters or gradients were rebound between forward and backward");
    }
    for (size_t i = 0; i < r.bwd.size(); ++i) {
      MDM_CUDA(cudaGraphLaunch(r.bwd[i], st));
      ++g_graph_launches;
      if (r.bwd_ranges[i].second > r.bwd_ranges[i].first && ready_fn != nullptr)
        ready_fn(ready_user, reinterpret_cast<void*>(r.bwd_ranges[i].first), reinterpret_cast<void*>(r.bwd_ranges[i].second));
    }
    g_launch_count += r.bwd_kernels;
    if (gio->dcond != nullptr && r.dcond != nullptr)
      MDM_CUDA(cudaMemcpyAsync(gio->dcond, r.dcond, r.cond_bytes, cudaMemcpyDeviceToDevice, st));
    if (gio->dcond_emb != nullptr && r.dcemb != nullptr)
      MDM_CUDA(cudaMemcpyAsync(gio->dcond_emb, r.dcemb, r.cemb_bytes, cudaMemcpyDeviceToDevice, st));
  }

  std::function<void(uintptr_t, uintptr_t)> seg_cut;  // set while a segmented backward is being captured

  // learn = false (a split backward): neither learns the closures' parameters nor reports ready ranges -- the text
  // path's gradients are written by the other stage's backward, so no range is final here
  void replay_tape(bool learn) {
    const int n = static_cast<int>(eng.tape.size());
    uintptr_t arena_lo = UINTPTR_MAX, arena_hi = 0;
    for (const Param& p : plist) {
      if (p.g == nullptr) continue;
      const uintptr_t a = reinterpret_cast<uintptr_t>(p.g);
      arena_lo = std::min(arena_lo, a);
      arena_hi = std::max(arena_hi, a + static_cast<uintptr_t>(p.numel) * sizeof(float));
    }
    // (while a backward is being captured the report cuts the graph into segments instead: see backward())
    const bool notify = learn && ready_fn != nullptr && static_cast<int>(learned.size()) == n && n > 0 && arena_hi > arena_lo;
    std::vector<uintptr_t> hi_prefix;  // highest gradient end address touched by closures 0..i
    if (notify) {
      hi_prefix.assign(n, arena_lo);
      uintptr_t run = arena_lo;
      for (int i = 0; i < n; ++i) {
        for (int idx : learned[i]) {
          const Param& p = plist[idx];
          if (p.g != nullptr)
            run = std::max(run, reinterpret_cast<uintptr_t>(p.g) + static_cast<uintptr_t>(p.numel) * sizeof(float));
        }
        hi_prefix[i] = run;
      }
    }
    if (notify && getenv("MDM_DEBUG_GRAD_READY") != nullptr) {
      // which closure pins how much of the arena: the highest gradient each of the earliest closures touches
      for (int i = 0; i < n && i < 12; ++i) {
        const Param* top = nullptr;
        for (int idx : learned[i])
          if (plist[idx].g != nullptr && (top == nullptr || plist[idx].g > top->g)) top = &plist[idx];
        fprintf(stderr, "[grad_ready] closure %d/%d: %zu params, highest %s at +%.1f MB of %.1f MB\n", i, n,
                learned[i].size(), top ? top->name.c_str() : "-",
                top ? (reinterpret_cast<uintptr_t>(top->g) - arena_lo) / 1048576.0 : 0.0, (arena_hi - arena_lo) / 1048576.0);
      }
    }
    if (learn && static_cast<int>(learned.size()) != n) learned.assign(n, {});
    uintptr_t prev = arena_hi;
    final_lo = UINTPTR_MAX;
    struct Guard {
      Net* n;
      ~Guard() {
        n->replay_idx = -1;
        n->final_lo = UINTPTR_MAX;
        n->eng.side_end();  // (an exception inside a side scope must not leave the engine on the side stream)
      }
    } guard{this};
    for (int i = n - 1; i >= 0; --i) {
      replay_idx = i;
      cur_lookup.clear();
      eng.tape[i]();
      eng.side_join();  // weight-gradient work of this closure is ordered before anything later (and before a report)
      if (!learn) continue;
      std::vector<int>& seen = learned[i];
      for (int idx : cur_lookup)
        if (std::find(seen.begin(), seen.end(), idx) == seen.end()) seen.push_back(idx);
      if (notify) {
        const uintptr_t x = i > 0 ? hi_prefix[i - 1] : arena_lo;
        if (x < prev && (prev - x >= ready_min_bytes || i == 0)) {
          final_lo = x;
          if (seg_cut) seg_cut(x, prev);
          else ready_fn(ready_user, reinterpret_cast<void*>(x), reinterpret_cast<void*>(prev));
          prev = x;
        }
      }
    }
  }
};

}  // namespace mdm

// ====================================================================== C ABI
using mdm::Net;

struct mdm_net {
  Net net;
};

#define MDM_TRY(...)                                 \
  try {                                              \
    __VA_ARGS__;                                     \
    return 0;                                        \
  } catch (const std::exception& e) {                \
    mdm::set_error("%s", e.what());                  \
    return -1;                                       \
  }

extern "C" {

int mdm_net_create(const mdm_net_cfg* cfg, mdm_net** out) {
  // the one-key table {"scale": micro_scale_default} of every level that sets has_micro_scale
  mdm_micro_cfg m{};
  mdm_net_cfg c = *cfg;
  for (int l = 0; l < std::min<int>(c.num_levels, MDM_MAX_LEVELS); ++l) {
    if (!c.levels[l].has_micro_scale) continue;
    m.num_keys = 1;
    strcpy(m.names[0], "scale");
    m.level_num_keys[l] = 1;
    m.level_defaults[l][0] = c.levels[l].micro_scale_default;
    c.levels[l].has_micro_scale = 0;
  }
  return mdm_net_create_micro(&c, &m, out);
}

int mdm_net_create_micro(const mdm_net_cfg* cfg, const mdm_micro_cfg* micro, mdm_net** out) {
  MDM_TRY({
    int dev = 0, major = 0, minor = 0;
    MDM_CUDA(cudaGetDevice(&dev));
    MDM_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    MDM_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    if (major != 9 || minor != 0)
      throw mdm::MdmFail("mdm_b200 requires an sm_90a (H100) device; there is no fallback path");
    auto* n = new mdm_net();
    n->net.cfg = *cfg;
    if (micro != nullptr) n->net.micro = *micro;
    try {
      n->net.build();
    } catch (...) {
      delete n;
      throw;
    }
    *out = n;
  })
}

void mdm_net_destroy(mdm_net* net) { delete net; }

int mdm_net_num_params(const mdm_net* net) { return static_cast<int>(net->net.plist.size()); }

int mdm_net_param_info(const mdm_net* net, int index, const char** name, int32_t* ndim, int64_t shape[4]) {
  if (index < 0 || index >= static_cast<int>(net->net.plist.size())) return -1;
  const mdm::Param& p = net->net.plist[index];
  *name = p.name.c_str();
  *ndim = static_cast<int32_t>(p.shape.size());
  for (size_t i = 0; i < 4; ++i) shape[i] = i < p.shape.size() ? p.shape[i] : 1;
  return 0;
}

int mdm_net_bind_param(mdm_net* net, const char* name, void* weight, void* grad) {
  MDM_TRY({
    auto it = net->net.pindex.find(name);
    if (it == net->net.pindex.end()) throw mdm::MdmFail(std::string("unknown parameter ") + name);
    mdm::Param& p = net->net.plist[it->second];
    if (p.w != static_cast<float*>(weight) || p.g != static_cast<float*>(grad)) ++net->net.bind_epoch;
    p.w = static_cast<float*>(weight);
    p.g = static_cast<float*>(grad);
    net->net.weights_dirty = true;
    net->net.kv_valid = false;
  })
}

int mdm_net_grad_order(const mdm_net* net, int32_t* rank, int32_t n) {
  if (net == nullptr || rank == nullptr) return -1;
  const mdm::Net& N = net->net;
  if (N.learned.empty() || n != static_cast<int32_t>(N.plist.size())) return -1;
  for (int32_t i = 0; i < n; ++i) rank[i] = INT32_MAX;
  for (size_t c = 0; c < N.learned.size(); ++c)
    for (int idx : N.learned[c]) rank[idx] = std::min<int32_t>(rank[idx], static_cast<int32_t>(c));
  return 0;
}

int mdm_net_set_grad_ready(mdm_net* net, mdm_grad_ready_fn fn, void* user, uint64_t min_bytes) {
  if (net == nullptr) return -1;
  net->net.ready_fn = fn;
  net->net.ready_user = user;
  net->net.ready_min_bytes = static_cast<size_t>(min_bytes);
  return 0;
}

int mdm_net_set_graph_mode(mdm_net* net, int enable) {
  if (net == nullptr) return -1;
  net->net.graph_mode = enable != 0;
  if (!enable) {
    for (auto& r : net->net.graphs) net->net.drop_graph(r);
    net->net.active_graph = -1;
  }
  return 0;
}

unsigned long long mdm_graph_launch_count(void) { return mdm::g_graph_launches; }

int mdm_set_sm_reserve(int sms) {
  mdm::g_sm_reserve = sms < 0 ? 0 : (sms > 64 ? 64 : sms);
  return 0;
}

int mdm_net_weights_changed(mdm_net* net) {
  net->net.weights_dirty = true;
  net->net.kv_valid = false;
  return 0;
}

int mdm_net_forward(mdm_net* net, const mdm_net_io* io, mdm_stream_t stream) {
  return mdm_net_forward_stage(net, io, nullptr, stream);
}

static int forward_with(mdm_net* net, const mdm_net_io* io, const mdm_net_stage_io* stage, const mdm_net_micro_io& micro,
                        mdm_stream_t stream) {
  MDM_TRY({
    mdm::StepIO q{};
    static_cast<mdm_net_io&>(q) = *io;
    q.micro_scale = nullptr;
    if (stage != nullptr) static_cast<mdm_net_stage_io&>(q) = *stage;
    for (int k = 0; k < net->net.micro.num_keys; ++k) q.values[k] = micro.values[k];
    net->net.forward(&q, static_cast<cudaStream_t>(stream));
    MDM_CUDA(cudaGetLastError());
  })
}

int mdm_net_forward_stage(mdm_net* net, const mdm_net_io* io, const mdm_net_stage_io* stage, mdm_stream_t stream) {
  mdm_net_micro_io m{};
  if (net->net.scale_slot >= 0) m.values[net->net.scale_slot] = io->micro_scale;
  return forward_with(net, io, stage, m, stream);
}

int mdm_net_forward_micro(mdm_net* net, const mdm_net_io* io, const mdm_net_stage_io* stage,
                          const mdm_net_micro_io* micro, mdm_stream_t stream) {
  if (io->micro_scale != nullptr) {
    mdm::set_error("mdm_net_forward_micro: io->micro_scale must be NULL (pass the key \"scale\" in micro->values)");
    return -1;
  }
  mdm_net_micro_io m{};
  if (micro != nullptr) m = *micro;
  return forward_with(net, io, stage, m, stream);
}

int mdm_net_backward(mdm_net* net, const mdm_net_grad_io* gio, mdm_stream_t stream) {
  MDM_TRY({
    net->net.backward(gio, static_cast<cudaStream_t>(stream));
    MDM_CUDA(cudaGetLastError());
  })
}

uint64_t mdm_net_workspace_bytes(const mdm_net* net) { return net->net.eng.pool.reserved(); }
uint64_t mdm_net_workspace_high_water(const mdm_net* net) { return net->net.eng.pool.high_water(); }

int64_t mdm_net_debug_fetch(mdm_net* net, const char* name, float* dst, int64_t max_elems, mdm_stream_t stream) {
  const Net& N = net->net;
  if (strcmp(name, "cond_kv") == 0) {  // the K/V cache as raw fp16 bits, two per float
    if (!N.kv_valid) return -1;
    const int64_t halves = static_cast<int64_t>(N.kv_key[0]) * N.kv_key[1] * N.kv_row, n = (halves + 1) / 2;
    if (n > max_elems) return -2;
    cudaMemcpyAsync(dst, N.kv_cache, sizeof(__half) * halves, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream));
    return n;
  }
  auto it = net->net.debug_acts.find(name);
  if (it == net->net.debug_acts.end() || it->second->p == nullptr) return -1;
  const int64_t n = it->second->numel();
  if (n > max_elems) return -2;
  cudaMemcpyAsync(dst, it->second->p, sizeof(float) * n, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream));
  return n;
}

}  // extern "C"
