"""Pipelines behind the reference's `ml_mdm.diffusion` interface (diffusion.py:53-387):

  Model / NestedModel             wrap the vision model (DDP wraps this object in the reference)
  Diffusion / NestedDiffusion     get_loss(sample) -> (loss(B,), time, x_t, pred, tgt, weights),
                                  sample(num_examples, sample, image_side, device, **kwargs)

Noising, the v->eps conversion, the per-sample MSE and its gradient are fused CUDA kernels
(mdm_q_sample, mdm_loss_fwd, mdm_loss_bwd, mdm_avg_pool); the denoiser is the native engine.
torch supplies RNG draws, device tensors and the autograd graph only.
"""
import ctypes as C
import logging
from typing import List

import numpy as np
import torch
import torch.nn as nn

from . import _lib, samplers
from .config import DiffusionConfig, NestedDiffusionConfig  # noqa: F401
from .samplers import _f32c, _ptr, _stream


def _off(t, nbytes):
    return C.c_void_p(t.data_ptr() + nbytes) if t is not None else None


class _LossFn(torch.autograd.Function):
    """loss(B,) = sum_levels w_l * mean_chw (pred_for_training_l - target_l)^2 and its gradient w.r.t.
    the model outputs (diffusion.py:160-168, 367-386)."""

    @staticmethod
    def forward(ctx, spec, time, *tensors):
        # tensors: per level (model_out, x_t, x, eps)
        L = len(spec["levels"])
        B = tensors[0].shape[0]
        loss = torch.zeros(B, device=tensors[0].device, dtype=torch.float32)
        preds, tgts = [], []
        lib = _lib.lib()
        saved = []
        for l in range(L):
            mo, xt, x, eps = (_f32c(t) for t in tensors[4 * l:4 * l + 4])
            lv = spec["levels"][l]
            per = mo.numel() // B
            want = lv["want_outputs"]
            p = torch.empty_like(mo) if want else None
            tg = torch.empty_like(mo) if want else None
            if lv["weight"] != 0.0 or want:
                valid = min(int(lv.get("valid", B)), B)
                # rows [0, valid) carry the loss; the rest (mixed-resolution batches) only produce pred / target
                for lo, hi, wgt in ((0, valid, lv["weight"]), (valid, B, 0.0)):
                    if hi <= lo or (wgt == 0.0 and not want):
                        continue
                    o4, o1 = lo * per * 4, lo * 4
                    _lib.check(lib.mdm_loss_fwd(_off(mo, o4), _off(xt, o4), _off(x, o4), _off(eps, o4),
                                                _off(time, lo * 8), _ptr(lv["table"]), spec["ptype"], spec["ltype"],
                                                C.c_float(lv["image_div"]), C.c_float(wgt), _off(loss, o1),
                                                _off(p, o4), _off(tg, o4), hi - lo, C.c_int64(per), _stream()),
                               "mdm_loss_fwd")
            preds.append(p)
            tgts.append(tg)
            saved += [mo, xt, x, eps]
        ctx.spec = spec
        ctx.time = time
        ctx.saved = saved
        outs = [loss] + [t for t in preds + tgts if t is not None]
        ctx.mark_non_differentiable(*outs[1:])
        return tuple(outs)

    @staticmethod
    def backward(ctx, dloss, *unused):
        spec, time, saved = ctx.spec, ctx.time, ctx.saved
        dloss = _f32c(dloss)
        lib = _lib.lib()
        grads = []
        for l, lv in enumerate(spec["levels"]):
            mo, xt, x, eps = saved[4 * l:4 * l + 4]
            if lv["weight"] == 0.0:
                grads += [torch.zeros_like(mo), None, None, None]
                continue
            B = mo.shape[0]
            valid = min(int(lv.get("valid", B)), B)
            d = torch.empty_like(mo)
            if valid < B:
                d[valid:].zero_()
            _lib.check(lib.mdm_loss_bwd(_ptr(mo), _ptr(xt), _ptr(x), _ptr(eps), _ptr(time), _ptr(lv["table"]),
                                        spec["ptype"], spec["ltype"], C.c_float(lv["image_div"]),
                                        C.c_float(lv["weight"]), _ptr(dloss), _ptr(d), valid,
                                        C.c_int64(mo.numel() // B), _stream()), "mdm_loss_bwd")
            grads += [d, None, None, None]
        return (None, None) + tuple(grads)


class Model(nn.Module):
    """diffusion.py:53-87. `forward` returns (outputs, variances placeholder)."""

    def __init__(self, vision_model, diffusion_config=None):
        super().__init__()
        self.diffusion_config = diffusion_config if diffusion_config is not None else DiffusionConfig()
        self._output_scale = self.diffusion_config.model_output_scale
        self.vision_model = vision_model
        self.sampler = None

    def set_sampler(self, sampler):
        self.sampler = sampler

    def load(self, vision_file: str) -> dict:
        return self.vision_model.load(vision_file)

    def save(self, vision_file, other_items=None):
        self.vision_model.save(vision_file, other_items=other_items)

    @property
    def input_channels(self):
        return self.vision_model.input_channels

    def scaled_call(self, fn, *args):
        """fn(*args) (the vision model or one of its methods) with the engine applying
        s * tanh(out / s), s = model_output_scale, to the outputs and its derivative in the backward (diffusion.py:83-85)."""
        vm = self.vision_model
        vm.output_scale = float(self._output_scale or 0.0)
        try:
            return fn(*args)
        finally:
            vm.output_scale = 0.0

    def forward(self, x_t, times, lm_outputs, lm_mask, micros={}):
        outputs = self.scaled_call(self.vision_model, x_t, times, lm_outputs, lm_mask, micros)
        # the reference allocates ones_like(outputs) here; a broadcast view keeps the interface
        return outputs, outputs.new_ones(()).expand_as(outputs)


class NestedModel(Model):
    """diffusion.py:251-292 with no_use_residual=True (the only working mode of the reference). Its forward replaces
    Model.forward, so model_output_scale is accepted and not applied, as in the reference."""

    def forward(self, x_t: List[torch.Tensor], times, lm_outputs, lm_mask, micros={}, mixed_ratio=None):
        if not self.diffusion_config.no_use_residual:
            raise NotImplementedError("NestedModel residual mode references an undefined variable in the reference "
                                      "(diffusion.py:288); shipped configs set no_use_residual: true")
        if mixed_ratio is None:
            return self.vision_model(x_t, times, lm_outputs, lm_mask, micros)
        # diffusion.py:262-274: each level sees only a leading part of the batch (the engine slices temb /
        # conditioning and zero-pads the in_adapter output itself); predictions are zero-padded back to the batch
        batch_size = x_t[0].size(0)
        x_t = [x[: int(m * x.size(0))] for x, m in zip(x_t, mixed_ratio)]
        p_t = self.vision_model(x_t, times, lm_outputs, lm_mask, micros)
        return [torch.cat([p, p.new_zeros(batch_size - p.size(0), *p.size()[1:])], 0) if p.size(0) < batch_size else p
                for p in p_t]


class Diffusion(nn.Module):
    def __init__(self, denoising_model, diffusion_config):
        super().__init__()
        logging.info(f"Diffusion config: {diffusion_config}")
        self.model = Model(denoising_model, diffusion_config)
        self.sampler = samplers.Sampler(diffusion_config.sampler_config)
        self.model.set_sampler(self.sampler)
        self._config = diffusion_config

    def get_model(self):
        return self.model.module if hasattr(self.model, "module") else self.model

    def to(self, device):
        self.model = self.model.to(device)
        self.sampler = self.sampler.to(device)
        return self

    def train(self, mode: bool = True):
        self.model.train(mode)
        return self

    def eval(self):
        self.model.eval()
        self.sampler.eval()
        return self

    def get_micro_conditioning(self, sample: dict) -> dict:
        micros, conditions = {}, self.get_model().vision_model.conditions
        if conditions is not None:
            micros = {key: sample[key] for key in conditions if key in sample}
        return micros

    def _types(self):
        sc = self._config.sampler_config
        return int(sc.prediction_type.value), int(sc.loss_target_type.value)

    def _inputs(self, sample):
        """(images or uint8 batch, lm_outputs, lm_mask). Besides the reference's keys, the raw reader batch is accepted:
        sample["image"] uint8 NHWC instead of "images" (the (x - 127) / 128 + permute of train_parallel.py:193-195 is
        then fused into the q-sample kernel), and sample["lm_mask_applied"] = False when lm_outputs has not been
        multiplied by lm_mask yet (language_models/factory.py:101; fused into the engine's input cast)."""
        self.get_model().vision_model.fuse_lm_mask = sample.get("lm_mask_applied", True) is False
        images = sample["images"] if "images" in sample else sample["image"]
        return images, sample["lm_outputs"], sample["lm_mask"]

    def _draw(self, images):
        """get_eps_time for a float NCHW or a uint8 NHWC batch (same generator draws either way)."""
        if images.dtype == torch.uint8:
            B, H, W, Cc = images.shape
            like = torch.empty(B, Cc, H, W, device=images.device, dtype=torch.float32)
            return self.sampler.get_eps_time(like)
        return self.sampler.get_eps_time(images)

    def get_loss(self, sample: dict):
        """diffusion.py:144-168."""
        images, lm_outputs, lm_mask = self._inputs(sample)
        sc = self._config.sampler_config
        eps, time, weights = self._draw(images)
        if not self._config.use_vdm_loss_weights:
            weights = None
        rs = sc.rescale_signal
        if images.dtype == torch.uint8:
            images, x_t = self.sampler.q_sample_u8(images, eps, time, scale=1.0, image_div=float(rs) if rs else 1.0)
        else:
            x_t = self.sampler.q_sample(images, eps, time, scale=1.0, image_div=float(rs) if rs else 1.0)
        micros = self.get_micro_conditioning(sample)
        means, _ = self.model(x_t, time, lm_outputs, lm_mask, micros)
        ptype, ltype = self._types()
        spec = dict(ptype=ptype, ltype=ltype,
                    levels=[dict(table=self.sampler.level_table(1.0, images.device), image_div=1.0, weight=1.0,
                                 want_outputs=True)])
        loss, pred, tgt = _LossFn.apply(spec, time, means, x_t, _f32c(images), eps)
        self.get_model().vision_model.fuse_lm_mask = False
        return loss, time, x_t, means, tgt, weights

    def get_noise(self, num_examples, input_channels, image_side, device):
        return torch.randn(num_examples, input_channels, image_side, image_side).to(device)

    def sample(self, num_examples: int, sample: dict, image_side: int, device, **kwargs):
        """diffusion.py:181-197 (noise is drawn on the CPU generator and copied, as in the reference)."""
        self.eval()
        noise = self.get_noise(num_examples, self.get_model().input_channels, image_side, device)
        lm_outputs, lm_mask = sample["lm_outputs"], sample["lm_mask"]
        micros = self.get_micro_conditioning(sample)
        return self.sampler.sample(self.get_model(), noise, lm_outputs, lm_mask, micros, **kwargs)


class NestedDiffusion(Diffusion):
    def __init__(self, denoising_model, diffusion_config):
        nn.Module.__init__(self)
        logging.info(f"Diffusion config: {diffusion_config}")
        self.model = NestedModel(denoising_model, diffusion_config)
        self.sampler = samplers.NestedSampler(diffusion_config.sampler_config)
        self.model.set_sampler(self.sampler)
        self._config = diffusion_config
        self.mixed_ratio = None
        if getattr(self._config, "mixed_ratio", None):  # diffusion.py:309-313, e.g. '2:1' -> [2/3, 1]
            mr = np.cumsum(np.asarray([float(x) for x in str(self._config.mixed_ratio).split(":")]))
            self.mixed_ratio = mr / mr[-1]

    @staticmethod
    def avg_pool(x, r):
        x = _f32c(x)
        b, c, h, w = x.shape
        y = torch.empty(b, c, h // r, w // r, device=x.device, dtype=torch.float32)
        _lib.check(_lib.lib().mdm_avg_pool(_ptr(x), _ptr(y), b * c, h, w, int(r), _stream()), "mdm_avg_pool")
        return y

    def get_loss(self, sample: dict):
        """diffusion.py:315-387: image pyramid by average pooling, fresh low-resolution noise,
        per-level shifted schedule, weighted sum of per-level MSE."""
        images, lm_outputs, lm_mask = self._inputs(sample)
        micros = self.get_micro_conditioning(sample)
        vm = self.get_model().vision_model
        scales = vm.nest_ratio + [1]
        ratios = [scales[0] // s for s in scales]
        if any(vm.is_temporal):
            raise NotImplementedError("temporal mode")
        eps0, time, weights = self._draw(images)
        if not self._config.use_vdm_loss_weights:
            weights = None
        xt0 = None
        if images.dtype == torch.uint8:  # fused (x - 127) / 128, NHWC -> NCHW and the full-resolution q-sample
            images, xt0 = self.sampler.q_sample_u8(images, eps0, time, scale=scales[0],
                                                   image_div=self.sampler.level_image_div(scales[0]))
        imgs, epss = [_f32c(images)], [eps0]
        for iz in range(1, len(ratios)):
            rr = ratios[iz] // ratios[iz - 1]
            imgs.append(self.avg_pool(imgs[-1], rr))
        for iz in range(1, len(ratios)):
            epss.append(torch.empty_like(imgs[iz]).normal_())
        x_t = [xt0 if (i == 0 and xt0 is not None) else
               self.sampler.q_sample(x, e, time, scale=s, image_div=self.sampler.level_image_div(s))
               for i, (x, e, s) in enumerate(zip(imgs, epss, scales))]
        p_t = self.model(x_t, time, lm_outputs, lm_mask, micros, self.mixed_ratio)
        if self._config.multi_res_weights is not None:
            assert self._config.use_double_loss, "only makes sense when applying more losses"
            w = [float(v) for v in self._config.multi_res_weights.split(":")]
        else:
            w = [1.0] * len(x_t)
        ptype, ltype = self._types()
        levels, flat = [], []
        for i, (p, xt, x, e, s) in enumerate(zip(p_t, x_t, imgs, epss, scales)):
            active = (i == 0) or self._config.use_double_loss
            lv = dict(table=self.sampler.level_table(s, images.device),
                      image_div=self.sampler.level_image_div(s), weight=w[i] if active else 0.0,
                      want_outputs=(i == 0))
            if self.mixed_ratio is not None and active:
                # diffusion.py:378-382: loss_ / mixed_ratio[i], rows beyond int(mixed_ratio[i] * B) discarded
                lv["weight"] = w[i] / float(self.mixed_ratio[i])
                lv["valid"] = int(self.mixed_ratio[i] * p.shape[0])
            levels.append(lv)
            flat += [p, xt, x, e]
        loss, pred0, tgt0 = _LossFn.apply(dict(ptype=ptype, ltype=ltype, levels=levels), time, *flat)
        vm.fuse_lm_mask = False
        return loss, time, x_t[0], pred0, tgt0, weights
