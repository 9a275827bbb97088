"""Drop-in `UNet` for ml_mdm.models.unet.UNet (reference models/unet.py:579-987).

Same constructor signature `(input_channels, output_channels, config)`, same `forward(x_t, times,
conditioning, cond_mask, micros)`, same attributes used by the reference's pipelines/CLIs, and the
same parameter tree (names, shapes, OIHW fp32, default torch initialisation and zero-initialised
layers) -- so `state_dict()`, checkpoints, EMA deep copies and optimizers are interchangeable.

The modules below are parameter containers only: the arithmetic runs in libmdm_b200.so
(`mdm_net_forward` / `mdm_net_backward`), entered through one `torch.autograd.Function`.
There is no PyTorch fallback path.
"""
import copy
import ctypes as C
import logging
import math

import torch
import torch.nn as nn

from .. import _lib
from .native import MAX_MICRO, MICRO_NAME_LEN, NativeNet


def zero_module(module):
    for p in module.parameters():
        p.detach().zero_()
    return module


def _cfg_get(cfg, name, default=None):
    return getattr(cfg, name, default)


def _ints(v, n=None):
    if v is None:
        return []
    if isinstance(v, str):
        v = [int(x) for x in v.split(",")] if v else []
    v = [int(x) for x in v]
    if n is not None and len(v) == 1:
        v = v * n
    return v


def check_micro_conditions(conditions):
    """What the engine accepts of one level's micro-conditioning keys ({key: default}, unet.py:615-620)."""
    if len(conditions) > MAX_MICRO:
        raise ValueError(f"micro_conditioning: {len(conditions)} keys, the native path takes at most {MAX_MICRO}")
    for key, default in conditions.items():
        if len(key.encode()) >= MICRO_NAME_LEN:
            raise ValueError(f"micro_conditioning key '{key}' is longer than {MICRO_NAME_LEN - 1} bytes")
        if key == "scale" and default == 0:
            # the reference computes (micro / default).clamp(max=1) * default (unet.py:926): 0/0
            raise ValueError("micro_conditioning key 'scale' needs a non-zero default")


class _ResNet(nn.Module):
    """Parameters of one residual unit (reference ResNet, unet.py:193-221)."""

    def __init__(self, temporal_dim, cin, cout, groups, dropout):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.time_layer = nn.Linear(temporal_dim, cout * 2)
        self.norm2 = nn.GroupNorm(groups, cout)
        # no parameters; carries the train/eval flag the engine's fused dropout follows (native.py)
        self.dropout = nn.Dropout(dropout)
        self.conv2 = zero_module(nn.Conv2d(cout, cout, 3, padding=1))
        if cin != cout:
            self.conv3 = nn.Conv2d(cin, cout, 1)


class _Attention(nn.Module):
    """Parameters of one attention unit (reference SelfAttention, unet.py:241-274)."""

    def __init__(self, channels, cond_dim, use_ffn):
        super().__init__()
        self.norm = nn.GroupNorm(32, channels)
        self.qkv = nn.Conv2d(channels, channels * 3, 1)
        if cond_dim is not None and cond_dim > 0:
            self.norm_cond = nn.LayerNorm(cond_dim)
            self.kv_cond = nn.Linear(cond_dim, channels * 2)
        self.proj_out = zero_module(nn.Conv2d(channels, channels, 1))
        if use_ffn:
            self.ffn = nn.Sequential(
                nn.GroupNorm(32, channels),
                nn.Conv2d(channels, 4 * channels, 1),
                nn.GELU(),
                zero_module(nn.Conv2d(4 * channels, channels, 1)),
            )


class _MLP(nn.Module):
    """Parameters of the reference MLP (unet.py:425-436): x + Linear(GELU(Linear(LayerNorm(x))))."""

    def __init__(self, channels, multiplier=4):
        super().__init__()
        self.main = nn.Sequential(
            nn.LayerNorm(channels),
            nn.Linear(channels, multiplier * channels),
            nn.GELU(),
            zero_module(nn.Linear(multiplier * channels, channels)),
        )


class _SelfAttention1D(nn.Module):
    """Parameters of the reference SelfAttention1D without FFN (unet.py:316-346)."""

    def __init__(self, channels):
        super().__init__()
        self.norm = nn.LayerNorm(channels)
        self.qkv = nn.Linear(channels, channels * 3)
        self.proj_out = zero_module(nn.Linear(channels, channels))


class SelfAttention1DBlock(nn.Module):
    """Parameters of one lm_head layer (reference SelfAttention1DBlock, unet.py:439-446): 8-head self-attention over
    the conditioning tokens, then an MLP."""

    def __init__(self, channels):
        super().__init__()
        self.attn = _SelfAttention1D(channels)
        self.mlp = _MLP(channels)


class _Block(nn.Module):
    """Parameters of one resolution block (reference ResNetBlock, unet.py:449-532)."""

    def __init__(self, temporal_dim, res_io, nattn, down, up, cond_dim, groups, use_ffn, dropout):
        super().__init__()
        self.resnets = nn.ModuleList([_ResNet(temporal_dim, ci, co, groups, dropout) for ci, co in res_io])
        if nattn > 0:
            self.attn = nn.ModuleList(
                [_Attention(co, cond_dim, use_ffn) for (_, co) in res_io for _ in range(nattn)])
        if down or up:
            c = res_io[-1][1]
            self.resample = nn.Conv2d(c, c, 3, stride=2 if down else 1, padding=1)


class UNet(nn.Module):
    def __init__(self, input_channels: int, output_channels: int, config):
        super().__init__()
        self.config = config
        self._config = config
        self.input_channels = input_channels
        self.output_channels = output_channels
        rc = config.resnet_config
        groups = rc.num_groups_norm
        use_ffn = bool(rc.use_attention_ffn)
        dropout = rc.dropout
        channels_list = _ints(config.resolution_channels)
        L = len(channels_list)
        nres = _ints(config.num_resnets_per_resolution, L)
        nattn = _ints(config.num_attention_layers, L)
        attn_levels = _ints(config.attention_levels)
        if _cfg_get(config, "temporal_mode", False):
            raise NotImplementedError("temporal mode is inactive in all shipped configs "
                                      "and is not part of the native path (SURVEY.md 8f)")
        # mirrors unet.py:588-598: projected conditioning replaces the feature dim
        self.input_conditioning_feature_dim = config.conditioning_feature_dim
        if config.conditioning_feature_dim > 0 and config.conditioning_feature_proj_dim > 0:
            config.conditioning_feature_dim = config.conditioning_feature_proj_dim
        cond_dim = config.conditioning_feature_dim
        self.temporal_dim = channels_list[0] * 4 if config.temporal_dim is None else config.temporal_dim
        td = self.temporal_dim

        half = td // 8
        emb = math.log(10000) / half
        emb = torch.exp(torch.arange(half, dtype=torch.float) * -emb)
        self.register_buffer("t_emb", emb.unsqueeze(0), persistent=False)
        self.temb_layer1 = nn.Linear(td // 4, td)
        self.temb_layer2 = nn.Linear(td, td)
        has_cond_emb = cond_dim > 0 and not config.skip_cond_emb
        self.cond_emb = nn.Linear(cond_dim, td, bias=False) if has_cond_emb else None

        self.conditions = None
        if config.micro_conditioning is not None:
            self.conditions = {c.split(":")[0]: float(c.split(":")[1])
                               for c in config.micro_conditioning.split(",")}
            check_micro_conditions(self.conditions)
            self.cond_layers = nn.ModuleDict({
                k: nn.ModuleList([nn.Linear(td // 4, td), zero_module(nn.Linear(td, td))])
                for k in self.conditions})

        ch = channels_list[0]
        self.conv_in = nn.Conv2d(input_channels, ch, 3, padding=1)
        skips = [ch]
        down, mid, up = [], [], []
        for i in range(L):
            io = []
            for _ in range(nres[i]):
                io.append((ch, channels_list[i]))
                ch = channels_list[i]
                skips.append(ch)
            if i != L - 1:
                skips.append(ch)
            na = nattn[i] if i in attn_levels else 0
            down.append(_Block(td, io, na, i != L - 1, False, cond_dim if i in attn_levels else -1, groups, use_ffn,
                               dropout))
        if not config.skip_mid_blocks:
            mid = [_Block(td, [(ch, ch)], 1, False, False, cond_dim, groups, use_ffn, dropout),
                   _Block(td, [(ch, ch)], 0, False, False, -1, groups, use_ffn, dropout)]
        for i in reversed(range(L)):
            io = []
            for _ in range(nres[i] + 1):
                io.append((ch + skips.pop(), channels_list[i]))
                ch = channels_list[i]
            na = nattn[i] if i in attn_levels else 0
            up.append(_Block(td, io, na, False, i != 0, cond_dim if i in attn_levels else -1, groups, use_ffn,
                             dropout))
        self.norm_out = nn.GroupNorm(groups, ch)
        self.conv_out = zero_module(nn.Conv2d(ch, output_channels, 3, padding=1))
        self.down_blocks = nn.ModuleList(down)
        if not config.skip_mid_blocks:
            self.mid_blocks = nn.ModuleList(mid)
        self.up_blocks = nn.ModuleList(up)
        self.masked_cross_attention = config.masked_cross_attention
        if has_cond_emb:
            if config.conditioning_feature_proj_dim > 0:
                self.lm_proj = nn.Linear(self.input_conditioning_feature_dim, cond_dim)
            self.lm_head = nn.ModuleList(
                [SelfAttention1DBlock(cond_dim) for _ in range(_cfg_get(config, "num_lm_head_layers", 0) or 0)])
        self.is_temporal = []
        self._native = None

    # ------------------------------------------------------------------ reference surface
    @property
    def model_type(self):
        return "unet"

    def print_size(self, target_image_size: int = 64):
        n = sum(p.numel() for p in self.parameters())
        logging.info(f"{type(self).__name__}: {n / 1e6:.2f} M parameters")

    def save(self, fname: str, other_items=None):
        logging.info(f"Saving model file: {fname}")
        ckpt = {"state_dict": self.state_dict()}
        if other_items is not None:
            ckpt.update(other_items)
        torch.save(ckpt, fname)

    def load(self, fname: str):
        """Key-filtered, non-strict load; returns the checkpoint's other items (unet.py:802-832)."""
        logging.info(f"Loading model file: {fname}")
        ckpt = torch.load(fname, map_location="cpu", weights_only=False)
        mine = self.state_dict()
        sd = {k: v for k, v in ckpt["state_dict"].items() if k in mine}
        extra = {k for k in ckpt["state_dict"] if k not in mine}
        missing = {k for k in mine if k not in sd}
        if extra or missing:
            print(extra, missing)
        self.load_state_dict(sd, strict=False)
        return {k: copy.copy(v) for k, v in ckpt.items() if k != "model_state_dict"}

    # ------------------------------------------------------------------ native path
    def _level_configs(self):
        """Configs of the nest, outermost first."""
        return [self._config]

    def _levels(self):
        """Modules of the nest, outermost first."""
        return [self]

    def _lm_dim(self):
        return self._levels()[-1].input_conditioning_feature_dim

    def native(self) -> NativeNet:
        if self._native is None:
            self._native = NativeNet(self)
        return self._native

    def __deepcopy__(self, memo):
        # the native handle is per-module state, not copied (ModelEma deep-copies the vision model)
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = None if k == "_native" else copy.deepcopy(v, memo)
        return new

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_native"] = None
        return d

    def forward(self, x_t, times, conditioning=None, cond_mask=None, micros={}):
        """UNet.forward (unet.py:971-987). x_t: (B, C, H, W) fp32 cuda tensor; H and W divide by the downsampling."""
        single = not isinstance(x_t, (list, tuple))
        xs = [x_t] if single else list(x_t)
        # fuse_lm_mask: `conditioning` is the raw encoder output; the engine multiplies it by cond_mask on the way in
        # (language_models/factory.py:101 does that as a separate pass before the model is called)
        outs = self.native().run(xs, times, conditioning, cond_mask, micros,
                                 apply_lm_mask=bool(getattr(self, "fuse_lm_mask", False)),
                                 output_scale=self._output_scale())
        return outs[0] if single else list(outs)

    def _require_top(self, what):
        if bool(_cfg_get(self._config, "nesting", False)):
            raise _lib.MdmError(f"{what}: this U-Net was built with nesting=True; the engine runs it as part of its "
                                f"NestedUNet parent, so call {what} on the outermost NestedUNet")

    def forward_conditioning(self, conditioning, cond_mask):
        """UNet.forward_conditioning (unet.py:847-865): lm_proj, the lm_head layers, the pooled mean and cond_emb.
        Returns (cond_emb, conditioning, cond_mask): cond_emb is None when the model has none, cond_mask is None unless
        masked_cross_attention. Differentiable with respect to the text parameters."""
        self._require_top("forward_conditioning")
        native = self.native()
        cond, cemb = native.run_conditioning(conditioning, cond_mask,
                                             apply_lm_mask=bool(getattr(self, "fuse_lm_mask", False)))
        return cemb, cond, (cond_mask if native.cfg.masked_cross_attention else None)

    def forward_denoising(self, x_t, times, cond_emb=None, conditioning=None, cond_mask=None, micros={}):
        """UNet.forward_denoising (unet.py:935-969) / NestedUNet.forward_denoising (nested_unet.py:168-230): the
        denoiser on given text features. x_t is a tensor for a UNet, a list (high -> low resolution) for a NestedUNet.
        Differentiable with respect to conditioning, cond_emb and the parameters outside the text path. Without
        autograd, the K/V the cross-attention blocks compute from `conditioning` are kept by the engine and reused by
        the next call with the same (unmodified) conditioning / cond_mask tensors under unchanged weights."""
        self._require_top("forward_denoising")
        single = not isinstance(x_t, (list, tuple))
        xs = [x_t] if single else list(x_t)
        outs = self.native().run_denoising(xs, times, cond_emb, conditioning, cond_mask, micros,
                                           output_scale=self._output_scale())
        return outs[0] if single else list(outs)

    def _output_scale(self):
        # model_output_scale, set by diffusion.Model around its own calls only: the reference applies s * tanh(out / s)
        # in Model.forward (diffusion.py:83-85), so a U-Net called directly is never scaled
        return float(getattr(self, "output_scale", 0.0))
