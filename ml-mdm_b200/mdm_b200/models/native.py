"""Bridge between the parameter-container modules and the native engine (mdm_net_* in
include/mdm_b200.h).  torch is used for device memory, streams and autograd bookkeeping only."""
import ctypes as C
import os
import weakref

import torch

from .. import _lib

MAX_RES, MAX_LEVELS = 8, 4
MAX_MICRO, MICRO_NAME_LEN = 8, 32  # MDM_MAX_MICRO, MDM_MICRO_NAME_LEN


class LevelCfg(C.Structure):
    _fields_ = [
        ("num_res", C.c_int32),
        ("channels", C.c_int32 * MAX_RES),
        ("num_resnets", C.c_int32 * MAX_RES),
        ("num_attn", C.c_int32 * MAX_RES),
        ("cond_level", C.c_int32 * MAX_RES),
        ("temporal_dim", C.c_int32),
        ("groups", C.c_int32),
        ("use_attention_ffn", C.c_int32),
        ("skip_mid_blocks", C.c_int32),
        ("nesting", C.c_int32),
        ("skip_normalization", C.c_int32),
        ("has_micro_scale", C.c_int32),
        ("micro_scale_default", C.c_float),
        ("dropout", C.c_float),
    ]


class NetCfg(C.Structure):
    _fields_ = [
        ("num_levels", C.c_int32),
        ("levels", LevelCfg * MAX_LEVELS),
        ("in_channels", C.c_int32),
        ("out_channels", C.c_int32),
        ("lm_dim", C.c_int32),
        ("cond_dim", C.c_int32),
        ("has_lm_proj", C.c_int32),
        ("has_cond_emb", C.c_int32),
        ("masked_cross_attention", C.c_int32),
        ("num_heads", C.c_int32),
        ("num_lm_head_layers", C.c_int32),
    ]


class NetIO(C.Structure):
    _fields_ = [
        ("batch", C.c_int32),
        ("tokens", C.c_int32),
        ("res", C.c_int32 * MAX_LEVELS),
        ("x_t", C.c_void_p * MAX_LEVELS),
        ("times", C.c_void_p),
        ("lm", C.c_void_p),
        ("lm_mask", C.c_void_p),
        ("micro_scale", C.c_void_p),
        ("out", C.c_void_p * MAX_LEVELS),
        ("save_for_backward", C.c_int32),
        ("level_batch", C.c_int32 * MAX_LEVELS),
        ("apply_lm_mask", C.c_int32),
        ("res_w", C.c_int32 * MAX_LEVELS),
        ("output_scale", C.c_float),
        ("single_plane", C.c_int32),
        ("dropout", C.c_int32),
        ("dropout_seed", C.c_uint64),
    ]


class StageIO(C.Structure):
    """mdm_net_stage_io: which part of the denoiser mdm_net_forward_stage runs, and its text inputs / outputs."""
    _fields_ = [
        ("stage", C.c_int32),
        ("cond_out", C.c_void_p),
        ("cond_emb_out", C.c_void_p),
        ("cond", C.c_void_p),
        ("cond_emb", C.c_void_p),
        ("cross_mask", C.c_void_p),
        ("cond_cache", C.c_int32),
    ]


class MicroCfg(C.Structure):
    """mdm_micro_cfg: the nest's micro-conditioning keys (first appearance, outermost level first) and each level's
    keys, as indices into that table in the level's order, with their defaults."""
    _fields_ = [
        ("num_keys", C.c_int32),
        ("names", (C.c_char * MICRO_NAME_LEN) * MAX_MICRO),
        ("level_num_keys", C.c_int32 * MAX_LEVELS),
        ("level_keys", (C.c_int32 * MAX_MICRO) * MAX_LEVELS),
        ("level_defaults", (C.c_float * MAX_MICRO) * MAX_LEVELS),
    ]


class MicroIO(C.Structure):
    """mdm_net_micro_io: (batch,) fp32 values per table key, NULL = the levels' defaults."""
    _fields_ = [("values", C.c_void_p * MAX_MICRO)]


class NetGradIO(C.Structure):
    _fields_ = [
        ("dout", C.c_void_p * MAX_LEVELS),
        ("stage", C.c_int32),
        ("dcond", C.c_void_p),
        ("dcond_emb", C.c_void_p),
        ("dcond_in", C.c_void_p),
        ("dcond_emb_in", C.c_void_p),
    ]


def _ints(v, n=None):
    if v is None:
        return []
    if isinstance(v, str):
        v = [int(x) for x in v.split(",")] if v else []
    v = [int(x) for x in v]
    if n is not None and len(v) == 1:
        v = v * n
    return v


def build_net_cfg(module) -> NetCfg:
    """module: UNet / NestedUNet container. Translates its config objects into the C struct."""
    cfgs = module._level_configs()
    mods = module._levels()
    nc = NetCfg()
    nc.num_levels = len(cfgs)
    scale_only = _scale_only(mods)
    for li, (cfg, m) in enumerate(zip(cfgs, mods)):
        lc = nc.levels[li]
        ch = _ints(cfg.resolution_channels)
        L = len(ch)
        assert L <= MAX_RES
        nres = _ints(cfg.num_resnets_per_resolution, L)
        nattn = _ints(cfg.num_attention_layers, L)
        levels = _ints(cfg.attention_levels)
        lc.num_res = L
        for i in range(L):
            lc.channels[i] = ch[i]
            lc.num_resnets[i] = nres[i]
            lc.num_attn[i] = nattn[i] if i in levels else 0
            lc.cond_level[i] = 1 if i in levels else 0
        lc.temporal_dim = m.temporal_dim
        lc.groups = cfg.resnet_config.num_groups_norm
        lc.use_attention_ffn = int(bool(cfg.resnet_config.use_attention_ffn))
        lc.skip_mid_blocks = int(bool(cfg.skip_mid_blocks))
        lc.nesting = int(bool(cfg.nesting))
        lc.skip_normalization = int(bool(getattr(cfg, "skip_normalization", True)))
        # "scale:<default>" nests keep the one-key fields of mdm_net_create; any other keys go in build_micro_cfg's table
        if scale_only:
            lc.has_micro_scale = int(m.conditions is not None)
            lc.micro_scale_default = float(m.conditions["scale"]) if m.conditions is not None else 0.0
        lc.dropout = float(cfg.resnet_config.dropout)
    inner = mods[-1]
    icfg = cfgs[-1]
    nc.in_channels = module.input_channels
    nc.out_channels = module.output_channels
    nc.lm_dim = max(int(inner.input_conditioning_feature_dim), 0)
    nc.cond_dim = max(int(icfg.conditioning_feature_dim), 0)
    nc.has_lm_proj = int(hasattr(inner, "lm_proj"))
    nc.has_cond_emb = int(inner.cond_emb is not None)
    nc.masked_cross_attention = int(icfg.masked_cross_attention)
    nc.num_heads = 8
    nc.num_lm_head_layers = len(inner.lm_head) if getattr(inner, "lm_head", None) is not None else 0
    return nc


def autocast_active():
    """Whether the call being entered runs inside an active CUDA autocast region (bf16 or fp16). The engine then runs
    its weight products on the hi fp16 plane of the weights only (mdm_net_io.single_plane): autocast rounds the
    reference's conv and linear operands to 8 (bf16) or 11 (fp16) significand bits, so the lo plane that carries the
    weights to ~22 bits for the fp32 path buys nothing there."""
    return torch.is_autocast_enabled("cuda")


def _scale_only(mods):
    return all(m.conditions is None or list(m.conditions) == ["scale"] for m in mods)


def build_micro_cfg(module) -> MicroCfg:
    """The micro-conditioning table of the nest (mdm_net_create_micro) from every level's `conditions`."""
    mc = MicroCfg()
    names = []
    for li, m in enumerate(module._levels()):
        conds = m.conditions or {}
        for j, (key, default) in enumerate(conds.items()):
            if key not in names:
                if len(names) == MAX_MICRO:
                    raise _lib.MdmError(f"micro_conditioning: the nest has more than {MAX_MICRO} distinct keys")
                raw = key.encode()
                if len(raw) >= MICRO_NAME_LEN:
                    raise _lib.MdmError(f"micro_conditioning key '{key}' is longer than {MICRO_NAME_LEN - 1} bytes")
                mc.names[len(names)].value = raw
                names.append(key)
            mc.level_keys[li][j] = names.index(key)
            mc.level_defaults[li][j] = float(default)
        mc.level_num_keys[li] = len(conds)
    mc.num_keys = len(names)
    return mc


class _DenoiseFn(torch.autograd.Function):
    """One autograd node for the whole denoiser: forward = mdm_net_forward, backward = mdm_net_backward.
    Parameters are passed so autograd routes their gradients (DDP hooks, accumulation, clipping work
    on ordinary .grad tensors). The plane mode is read here, at forward time (autocast_active); the engine runs the
    backward in the mode of its forward, so a backward called outside the autocast region still matches it."""

    @staticmethod
    def forward(ctx, native, nlev, need_grad, times, lm, mask, micro, *rest):
        xs = rest[:nlev]
        outs = native._forward(list(xs), times, lm, mask, micro, save=need_grad, apply_lm_mask=native.apply_lm_mask,
                               output_scale=native.output_scale, single_plane=autocast_active())
        ctx.native = native
        ctx.nlev = nlev
        ctx.set_materialize_grads(False)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gouts):
        native = ctx.native
        grads = native._backward(list(gouts))
        return (None,) * 7 + (None,) * ctx.nlev + tuple(grads)


class _ConditioningFn(torch.autograd.Function):
    """forward_conditioning as one autograd node (mdm_net_io.stage = 1): lm_proj, the lm_head layers, the pooled mean
    and cond_emb. Its backward (stage 1) recomputes the text path from the saved inputs and routes the gradients of
    the text parameters only; the denoising node routes the others."""

    @staticmethod
    def forward(ctx, native, need_grad, apply_lm_mask, lm, mask, *text_params):
        # (the engine recomputes the text path for the stage-1 backward in this mode)
        cond, cemb = native._conditioning(lm, mask, save=need_grad, apply_lm_mask=apply_lm_mask,
                                          single_plane=autocast_active())
        ctx.native = native
        ctx.set_materialize_grads(False)
        if not need_grad:
            ctx.mark_non_differentiable(cond, cemb)
        return cond, cemb

    @staticmethod
    def backward(ctx, dcond, dcemb):
        native = ctx.native
        grads = native._backward([], stage=1, dcond_in=dcond, dcemb_in=dcemb)
        return (None,) * 5 + tuple(g for g, k in zip(grads, native.param_names) if k in native._text_names)


class _DenoisingFn(torch.autograd.Function):
    """forward_denoising as one autograd node (mdm_net_io.stage = 2), differentiable with respect to the tokens, the
    pooled embedding and every parameter outside the text path."""

    @staticmethod
    def forward(ctx, native, nlev, need_grad, cache, times, cond, cond_emb, cross_mask, micro, *rest):
        xs = rest[:nlev]
        outs = native._forward(list(xs), times, None, None, micro, save=need_grad, stage=2, cond=cond,
                               cond_emb=cond_emb, cross_mask=cross_mask, cache=cache, output_scale=native.output_scale,
                               single_plane=autocast_active())
        ctx.native = native
        ctx.nlev = nlev
        ctx.want = (cond is not None and cond.requires_grad, cond_emb is not None and cond_emb.requires_grad)
        ctx.set_materialize_grads(False)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gouts):
        grads, dcond, dcemb = ctx.native._backward(list(gouts), stage=2, want=ctx.want)
        return (None,) * 5 + (dcond, dcemb, None, None) + (None,) * ctx.nlev + tuple(grads)


ARENA_ALIGN = 64  # elements: every gradient view starts on a 256-byte boundary (vector loads in the optimiser sweep)


def _pad(n):
    return (n + ARENA_ALIGN - 1) // ARENA_ALIGN * ARENA_ALIGN


def arena_views(arena, params, offsets):
    """Fresh per-parameter views of a flat gradient arena for autograd. They must not be referenced anywhere
    else: AccumulateGrad adopts an incoming gradient as `.grad` only when it holds the sole reference and clones
    it otherwise, and the flat-arena paths (one NCCL all-reduce, GradientOverlap, FusedAdam) rely on `.grad`
    aliasing the arena."""
    return [arena[off:off + p.numel()].view_as(p) for p, off in zip(params, offsets)]


class NativeNet:
    def __init__(self, module):
        self.module = module
        self.lib = _lib.lib()
        self.cfg = build_net_cfg(module)
        self.handle = C.c_void_p()
        self.micro_cfg = build_micro_cfg(module)
        self.micro_keys = [self.micro_cfg.names[k].value.decode() for k in range(self.micro_cfg.num_keys)]
        if _scale_only(module._levels()):
            _lib.check(self.lib.mdm_net_create(C.byref(self.cfg), C.byref(self.handle)), "mdm_net_create")
        else:
            _lib.check(self.lib.mdm_net_create_micro(C.byref(self.cfg), C.byref(self.micro_cfg), C.byref(self.handle)),
                       "mdm_net_create_micro")
        self.lib.mdm_net_workspace_bytes.restype = C.c_uint64
        self.lib.mdm_net_workspace_high_water.restype = C.c_uint64
        self.lib.mdm_net_debug_fetch.restype = C.c_int64
        # parameter table of the engine
        self.names, self.shapes = [], {}
        n = self.lib.mdm_net_num_params(self.handle)
        for i in range(n):
            name = C.c_char_p()
            nd = C.c_int32()
            shape = (C.c_int64 * 4)()
            _lib.check(self.lib.mdm_net_param_info(self.handle, i, C.byref(name), C.byref(nd), shape), "param_info")
            nm = name.value.decode()
            self.names.append(nm)
            self.shapes[nm] = tuple(shape[j] for j in range(nd.value))
        self._check_tree()
        self.params = None
        self.sig = None
        self.grad_arena = None
        self.active_arena = None
        self.order = None
        self.arena_zeroed = False
        self.offsets = None
        self._ready_cb = None
        self._keep = None
        self.apply_lm_mask = False
        self.output_scale = 0.0  # model_output_scale of the forward being entered (diffusion.Model sets it)
        # ResNet dropout: the largest p of the nest, the modules whose train/eval flag it follows, and the
        # (flag, seed) of the forward being entered
        self.max_dropout = max(self.cfg.levels[i].dropout for i in range(self.cfg.num_levels))
        self._dropouts = [m for m in module.modules() if isinstance(m, torch.nn.Dropout)]
        self.dropout = (0, 0)
        # CUDA-graph replay of forward / backward (mdm_net_set_graph_mode): on unless MDM_NO_GRAPH is set; switched
        # off for this net by gradient accumulation (a fresh arena per backward would re-record every step). With a
        # gradient-ready callback installed the backward is recorded as one graph per reported range.
        self.graphs = os.environ.get("MDM_NO_GRAPH") is None
        self.lib.mdm_net_set_graph_mode(self.handle, int(self.graphs))
        # split forward: the text path's parameters (stage 1) and the state of the engine's K/V cache (stage 2)
        inner = "inner_unet." * (self.cfg.num_levels - 1)
        self._text_names = {k for k in self.names
                            if k.startswith((inner + "lm_proj.", inner + "lm_head.", inner + "cond_emb."))}
        self._text_clean = False  # the text parameters' arena slots are zero (a stage-2 backward just cleared it)
        self.weights_epoch = 0    # bumped whenever the engine is told its weights changed or they are rebound
        self._kv = None           # what the engine's K/V cache was filled from (see _cache_mode)
        self._keep_text = None    # inputs of a stage-1 forward, kept for its backward
        self._split_shapes = (None, None)

    def set_graph_mode(self, on):
        self.graphs = bool(on)
        _lib.check(self.lib.mdm_net_set_graph_mode(self.handle, int(self.graphs)), "mdm_net_set_graph_mode")

    def __del__(self):
        try:
            if self.handle:
                self.lib.mdm_net_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def _tensors(self):
        d = dict(self.module.named_parameters())
        for k, v in self.module.named_buffers():
            if k.endswith("t_emb"):
                d[k] = v
        return d

    def _check_tree(self):
        t = self._tensors()
        mine, theirs = set(t), set(self.names)
        if mine != theirs:
            raise _lib.MdmError(f"parameter tree mismatch: only in module {sorted(mine - theirs)[:5]}, "
                                f"only in engine {sorted(theirs - mine)[:5]}")
        for k in self.names:
            if tuple(t[k].shape) != self.shapes[k]:
                raise _lib.MdmError(f"shape mismatch for {k}: module {tuple(t[k].shape)} engine {self.shapes[k]}")

    # ---------------------------------------------------------------- binding
    def _bind(self):
        t = self._tensors()
        plist = [(k, t[k]) for k in self.names]
        for k, p in plist:
            if not p.is_cuda:
                raise _lib.MdmError("mdm_b200 runs on a CUDA (sm_90a) device only; move the model with .to('cuda'). "
                                    "There is no CPU path.")
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise _lib.MdmError(f"parameter {k} must be contiguous fp32")
        sig = tuple(p.data_ptr() for _, p in plist) + tuple(p.requires_grad for _, p in plist)
        if sig == self.sig:
            return
        dev = plist[0][1].device
        total = sum(_pad(p.numel()) for k, p in plist if not k.endswith("t_emb"))
        self.grad_arena = torch.zeros(total, device=dev, dtype=torch.float32)
        self.arena_zeroed = True
        off = 0
        self.params, self.param_names, self.offsets = [], [], []
        # Arena layout: registration order at first; optimize_arena_layout() re-sorts it by how late each
        # gradient becomes final so that mdm_net_set_grad_ready can report it from the top down.
        if self.order is not None:
            by_name = dict(plist)
            plist = [(k, by_name[k]) for k in self.order]
        for k, p in plist:
            if k.endswith("t_emb"):
                _lib.check(self.lib.mdm_net_bind_param(self.handle, k.encode(), C.c_void_p(p.data_ptr()), None), "bind")
                continue
            self.param_names.append(k)
            self.offsets.append(off)
            g = self.grad_arena[off:off + p.numel()].view_as(p)
            off += _pad(p.numel())
            # frozen parameters (requires_grad=False, e.g. freeze_inner_unet, nested_unet.py:147-150) get no
            # gradient pointer: the engine skips their weight gradients, their arena slot stays zero and the
            # global norm / optimiser sweep never see them (clip_grad_norm_ ignores them in the reference too)
            _lib.check(self.lib.mdm_net_bind_param(self.handle, k.encode(), C.c_void_p(p.data_ptr()),
                                                   C.c_void_p(g.data_ptr()) if p.requires_grad else None), "bind")
            self.params.append(p)
        self.sig = sig
        self.versions = None
        self.weights_epoch += 1

    def _sync_weights(self):
        v = sum(p._version for p in self.params)
        if v != self.versions:
            self.lib.mdm_net_weights_changed(self.handle)
            self.versions = v
            self.weights_epoch += 1

    # ---------------------------------------------------------------- public
    def run(self, xs, times, lm, mask, micros, apply_lm_mask=False, output_scale=0.0):
        self._bind()
        self.apply_lm_mask = bool(apply_lm_mask)
        self.output_scale = float(output_scale)
        micro = self._enter(micros, xs[-1].shape[0])
        # (Function.forward runs with grad mode off, so the decision is taken here)
        need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in self.params)
        return _DenoiseFn.apply(self, len(xs), need_grad, times, lm, mask, micro, *xs, *self.params)

    def run_conditioning(self, lm, mask, apply_lm_mask=False):
        """forward_conditioning: (cond (B,S,cond_dim), cond_emb (B,temporal_dim) or None)."""
        if self.cfg.cond_dim <= 0:
            raise _lib.MdmError("forward_conditioning needs a model with text conditioning (conditioning_feature_dim > 0)")
        if lm is None:
            raise _lib.MdmError("forward_conditioning needs the conditioning tensor")
        self._bind()
        text = [p for p, k in zip(self.params, self.param_names) if k in self._text_names]
        need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in text)
        cond, cemb = _ConditioningFn.apply(self, need_grad, bool(apply_lm_mask), lm, mask, *text)
        return cond, (cemb if self.cfg.has_cond_emb else None)

    def run_denoising(self, xs, times, cond_emb, cond, cross_mask, micros, output_scale=0.0):
        """forward_denoising on the engine (stage 2). Without autograd the K/V the cross-attention blocks compute from
        `cond` are kept by the engine and reused while `cond`, `cross_mask` and the weights stay what they were."""
        self._bind()
        self.output_scale = float(output_scale)
        micro = self._enter(micros, xs[-1].shape[0])
        need_grad = torch.is_grad_enabled() and (any(p.requires_grad for p in self.params) or any(
            t is not None and t.requires_grad for t in (cond, cond_emb)))
        if self.cfg.cond_dim > 0 and cond is None:
            raise _lib.MdmError("forward_denoising needs `conditioning` for a model with text conditioning")
        cache = 0 if need_grad or self.cfg.cond_dim <= 0 else self._cache_mode(xs, cond, cross_mask)
        outs = _DenoisingFn.apply(self, len(xs), need_grad, cache, times, cond, cond_emb, cross_mask, micro, *xs,
                                  *self.params)
        if cache == 1:
            self._kv = self._kv_key(xs, cond, cross_mask)
        return outs

    def _kv_key(self, xs, cond, mask):
        # identity (a weak reference: a freed tensor's address is reused) and in-place version of the tokens and mask,
        # the weight state, the shapes the cache was laid out for and the plane mode its K/V were computed in
        def ident(t):
            return None if t is None else (weakref.ref(t), t._version)
        return (ident(cond), ident(mask), self.weights_epoch, tuple(x.shape[0] for x in xs), tuple(cond.shape),
                autocast_active())

    def _cache_mode(self, xs, cond, mask):
        """2 when the engine's K/V cache was filled from this very `cond` / `mask` (unchanged since) under the current
        weights and in the current plane mode, else 1 (fill it)."""
        self._sync_weights()  # an in-place weight update bumps weights_epoch here, before the comparison
        old = self._kv
        if old is None:
            return 1
        new = self._kv_key(xs, cond, mask)

        def same(a, b):
            if a is None or b is None:
                return a is None and b is None
            return a[0]() is not None and a[0]() is b[0]() and a[1] == b[1]
        ok = same(old[0], new[0]) and same(old[1], new[1]) and old[2:] == new[2:]
        return 2 if ok else 1

    def _enter(self, micros, batch):
        """The micro-conditioning values of the forward being entered, one (batch,) fp32 tensor or None per key of the
        engine's table (keys no level configures are ignored, as the reference ignores them), and its dropout
        (flag, seed). A one-element value is broadcast over the batch, as torch broadcasting does in the reference."""
        micro = []
        for key in self.micro_keys:
            v = micros.get(key) if micros else None
            if v is not None:
                if not isinstance(v, torch.Tensor):
                    raise _lib.MdmError(f"micro-conditioning value '{key}' must be a CUDA tensor")
                if v.numel() not in (1, batch):
                    raise _lib.MdmError(f"micro-conditioning value '{key}' has {v.numel()} elements; the batch is "
                                        f"{batch} (one value per sample, or one for all)")
                if not v.is_cuda:
                    raise _lib.MdmError(f"micro-conditioning value '{key}' must be a CUDA tensor")
                v = v.detach().reshape(-1).float().expand(batch).contiguous()
            micro.append(v)
        self.dropout = (0, 0)
        if self.max_dropout > 0:
            training = self.module.training
            if any(d.training != training for d in self._dropouts):
                raise _lib.MdmError("the ResNets' nn.Dropout modules disagree with the model's train/eval mode; the "
                                    "engine applies dropout to every ResNet or to none (use model.train() / .eval())")
            if training:
                # from torch's default CPU generator: reproducible under torch.manual_seed, no device sync
                self.dropout = (1, int(torch.randint(2**63 - 1, ())))
        return micro

    def _forward(self, xs, times, lm, mask, micro, save, apply_lm_mask=False, stage=0, cond=None, cond_emb=None,
                 cross_mask=None, cache=0, output_scale=0.0, single_plane=False):
        self._sync_weights()
        if save and self.graphs and self.grad_arena is not None:
            lo, hi = self.grad_arena.data_ptr(), self.grad_arena.data_ptr() + self.grad_arena.numel() * 4
            if any(p.grad is not None and lo <= p.grad.data_ptr() < hi for p in self.params):
                self.set_graph_mode(False)  # gradient accumulation: this backward needs a fresh arena (see _backward)
        io = NetIO()
        B = xs[-1].shape[0]  # the innermost level always runs the whole batch (nested_unet.py:180,200-204)
        io.batch = B
        keep = []

        def f32(t):
            t = t.detach()
            if t.dtype != torch.float32 or not t.is_contiguous():
                t = t.float().contiguous()
            keep.append(t)
            return t

        outs = []
        for i, x in enumerate(xs):
            if not x.is_cuda:
                raise _lib.MdmError("inputs must be CUDA tensors")
            if x.dim() != 4:
                raise _lib.MdmError(f"level {i} input must be (batch, channels, height, width); got {tuple(x.shape)}")
            if i > 0:
                # the outer level's bottleneck feeds this level: both sides are the outer sides / 2^(num_res - 1)
                r = 1 << (self.cfg.levels[i - 1].num_res - 1)
                want = (xs[i - 1].shape[2] // r, xs[i - 1].shape[3] // r)
                if tuple(x.shape[2:]) != want:
                    raise _lib.MdmError(f"level {i} input is {tuple(x.shape[2:])} (height, width); the level above is "
                                        f"{tuple(xs[i - 1].shape[2:])} and downsamples by {r}, so it must be {want}")
            x = f32(x)
            if not (1 <= x.shape[0] <= B) or (i > 0 and x.shape[0] < xs[i - 1].shape[0]):
                raise _lib.MdmError("mixed-resolution batches: each level runs a leading part of the batch and inner "
                                    f"levels at least as many samples as outer ones; got {[t.shape[0] for t in xs]}")
            io.level_batch[i] = x.shape[0]
            io.res[i] = x.shape[2]
            io.res_w[i] = x.shape[3]
            io.x_t[i] = x.data_ptr()
            o = torch.empty_like(x)
            outs.append(o)
            io.out[i] = o.data_ptr()
        t64 = times.detach().to(torch.int64).contiguous()
        keep.append(t64)
        io.times = t64.data_ptr()
        if lm is not None:
            lm = f32(lm)
            io.tokens = lm.shape[1]
            io.lm = lm.data_ptr()
            if mask is not None:
                mask = f32(mask)
                io.lm_mask = mask.data_ptr()
        sio = StageIO()
        if stage == 2:
            sio.stage = 2
            sio.cond_cache = int(cache)
            if cond is not None:
                cond = f32(cond)
                io.tokens = cond.shape[1]
                sio.cond = cond.data_ptr()
            if cond_emb is not None:
                sio.cond_emb = f32(cond_emb).data_ptr()
            if cross_mask is not None:
                sio.cross_mask = f32(cross_mask).data_ptr()
        mio = MicroIO()
        for k, v in enumerate(micro):
            if v is not None:
                keep.append(v)
                mio.values[k] = v.data_ptr()
        io.save_for_backward = int(save)
        if stage == 2 and save:
            td = self.cfg.levels[self.cfg.num_levels - 1].temporal_dim
            self._split_shapes = (tuple(cond.shape) if cond is not None else None, (B, td))
        io.apply_lm_mask = int(bool(apply_lm_mask))
        io.dropout, io.dropout_seed = self.dropout
        io.output_scale = float(output_scale)
        io.single_plane = int(bool(single_plane))
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(self.lib.mdm_net_forward_micro(self.handle, C.byref(io), C.byref(sio) if stage else None,
                                                  C.byref(mio), C.c_void_p(st)), "mdm_net_forward_micro")
        self._keep = keep if save else None  # inputs must outlive the tape
        return outs

    def _conditioning(self, lm, mask, save, apply_lm_mask=False, single_plane=False):
        """mdm_net_forward with stage 1: (cond, cond_emb); cond_emb is an empty tensor for a model without one."""
        self._sync_weights()
        io = NetIO()
        keep = []

        def f32(t):
            t = t.detach()
            if t.dtype != torch.float32 or not t.is_contiguous():
                t = t.float().contiguous()
            keep.append(t)
            return t
        lm = f32(lm)
        if not lm.is_cuda:
            raise _lib.MdmError("inputs must be CUDA tensors")
        B, S = lm.shape[0], lm.shape[1]
        sio = StageIO()
        sio.stage = 1
        io.batch, io.tokens = B, S
        io.lm = lm.data_ptr()
        if mask is not None:
            io.lm_mask = f32(mask).data_ptr()
        io.apply_lm_mask = int(bool(apply_lm_mask))
        io.save_for_backward = int(save)
        io.single_plane = int(bool(single_plane))
        cond = torch.empty(B, S, self.cfg.cond_dim, device=lm.device, dtype=torch.float32)
        td = self.cfg.levels[self.cfg.num_levels - 1].temporal_dim
        cemb = torch.empty(B, td if self.cfg.has_cond_emb else 0, device=lm.device, dtype=torch.float32)
        sio.cond_out = cond.data_ptr()
        sio.cond_emb_out = cemb.data_ptr() if self.cfg.has_cond_emb else None
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(self.lib.mdm_net_forward_stage(self.handle, C.byref(io), C.byref(sio), C.c_void_p(st)),
                   "mdm_net_forward_stage (stage 1)")
        self._keep_text = keep if save else None  # the stage-1 backward recomputes from these
        return cond, cemb

    def _backward(self, gouts, stage=0, dcond_in=None, dcemb_in=None, want=(False, False)):
        """Stage 0: gradients of every parameter. Stage 1 (forward_conditioning): of the text parameters only, from the
        incoming dcond_in / dcemb_in. Stage 2 (forward_denoising): of the other parameters, plus (d cond, d cond_emb)
        where `want` asks for them. Parameters outside the stage get None."""
        gio = NetGradIO()
        gio.stage = stage
        keep = []

        def f32(g):
            g = g.detach()
            if g.dtype != torch.float32 or not g.is_contiguous():
                g = g.float().contiguous()
            keep.append(g)
            return g
        for i, g in enumerate(gouts):
            if g is None:
                continue
            gio.dout[i] = f32(g).data_ptr()
        if stage == 1:
            if dcond_in is not None:
                gio.dcond_in = f32(dcond_in).data_ptr()
            if dcemb_in is not None and dcemb_in.numel() > 0:
                gio.dcond_emb_in = f32(dcemb_in).data_ptr()
        mine = [stage == 0 or (k in self._text_names) == (stage == 1) for k in self.param_names]
        # fresh arena when existing .grad tensors alias the persistent one (gradient accumulation)
        arena = self.grad_arena
        lo, hi = arena.data_ptr(), arena.data_ptr() + arena.numel() * 4
        aliased = any(p.grad is not None and lo <= p.grad.data_ptr() < hi for p, m in zip(self.params, mine) if m)
        if aliased:
            arena = torch.zeros_like(self.grad_arena)
            views = self._views(arena)
            for k, p, g in zip(self.param_names, self.params, views):
                _lib.check(self.lib.mdm_net_bind_param(self.handle, k.encode(), C.c_void_p(p.data_ptr()),
                                                       C.c_void_p(g.data_ptr()) if p.requires_grad else None), "bind")
            self.sig = None  # rebinding to the persistent arena happens at the next forward
        else:
            views = self._views(arena)
            if stage == 1:
                # autograd runs the stage-2 backward first, which cleared the whole arena: zero only what is not clean
                if not (self.arena_zeroed or self._text_clean):
                    for v, m in zip(views, mine):
                        if m:
                            v.zero_()
            elif not self.arena_zeroed:  # the fused optimiser sweep (optim.FusedAdam) leaves it zeroed
                arena.zero_()
            self.arena_zeroed = False
        self._text_clean = stage == 2
        dcond = dcemb = None
        if stage == 2:
            if want[0]:
                dcond = torch.empty(self._split_shapes[0], device=arena.device, dtype=torch.float32)
                gio.dcond = dcond.data_ptr()
            if want[1]:
                dcemb = torch.empty(self._split_shapes[1], device=arena.device, dtype=torch.float32)
                gio.dcond_emb = dcemb.data_ptr()
        st = torch.cuda.current_stream().cuda_stream
        self.active_arena = arena  # what a gradient-ready callback (parallel.GradientOverlap) indexes into
        _lib.check(self.lib.mdm_net_backward(self.handle, C.byref(gio), C.c_void_p(st)), "mdm_net_backward")
        if stage == 1:
            self._keep_text = None
        else:
            self._keep = None
        grads = [g if (p.requires_grad and m) else None for p, g, m in zip(self.params, views, mine)]
        if stage == 2:
            return grads, dcond, dcemb
        return grads

    def _views(self, arena):
        return arena_views(arena, self.params, self.offsets)

    def optimize_arena_layout(self):
        """Re-sort the gradient arena by the order gradients become final in backward (learned by the
        engine during a previous backward, mdm_net_grad_order), latest at the lowest address. Returns
        False when nothing has been learned yet. Takes effect at the next forward; gradients already
        handed out keep their (old) storage."""
        n = len(self.names)
        rank = (C.c_int32 * n)()
        if self.lib.mdm_net_grad_order(self.handle, rank, C.c_int32(n)) != 0:
            return False
        idx = sorted(range(n), key=lambda i: (rank[i], i))
        order = [self.names[i] for i in idx]
        if order != self.order:
            self.order = order
            self.sig = None  # rebind at the next forward
        return True

    def set_grad_ready(self, fn, min_bytes=0):
        """Install (or with fn=None remove) the engine's gradient-ready notification: fn(lo_ptr, hi_ptr) is
        called from inside mdm_net_backward whenever the gradient bytes at addresses [lo, hi) are final."""
        if fn is None:
            self._ready_cb = None
            _lib.check(self.lib.mdm_net_set_grad_ready(self.handle, None, None, C.c_uint64(0)), "set_grad_ready")
            return
        cb = _lib.GRAD_READY_FN(lambda user, lo, hi: fn(int(lo or 0), int(hi or 0)))
        self._ready_cb = cb  # keep the trampoline alive as long as the engine may call it
        _lib.check(self.lib.mdm_net_set_grad_ready(self.handle, cb, None, C.c_uint64(int(min_bytes))), "set_grad_ready")

    def workspace_bytes(self):
        return int(self.lib.mdm_net_workspace_bytes(self.handle)), int(self.lib.mdm_net_workspace_high_water(self.handle))

    def debug_fetch(self, name, shape):
        out = torch.empty(shape, device="cuda", dtype=torch.float32)
        st = torch.cuda.current_stream().cuda_stream
        n = self.lib.mdm_net_debug_fetch(self.handle, name.encode(), C.c_void_p(out.data_ptr()), C.c_int64(out.numel()),
                                         C.c_void_p(st))
        if n < 0:
            raise _lib.MdmError(f"no debug tensor {name} ({n})")
        return out
