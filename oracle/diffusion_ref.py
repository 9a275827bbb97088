"""ORACLE (test infrastructure only -- never on the product path).

CPU restatement of the reference's diffusion algebra for the denoising path, in numpy (index and
schedule math, float64 -> float32 exactly as the reference) and elementwise torch on CPU tensors:

  schedules / shifted schedule     ml_mdm/samplers.py:126-170, 201-231, 255-264
  set_timesteps                    samplers.py:601-609
  q-sample, targets, x0/eps/v      samplers.py:244-246, 266-279, 347-390
  training loss (base / nested)    diffusion.py:123-168, 315-387
  reverse step, p_sample loop      samplers.py:281-345, 392-433, 516-578, 655-713

Pinned against the unmodified reference run here (tests/test_oracle.py) and the golden fixtures in
tests/golden/ generated from it (tests/golden/make_golden.py).  Gamma here is a per-sample scalar
broadcast over (C,H,W); the reference builds the same values as full maps.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

DDPM, DDIM, V_PREDICTION = 3, 4, 5


def schedule_table(schedule_type: str, n_steps: int, beta_start=0.0001, beta_end=0.02) -> np.ndarray:
    """float64 table of n_steps + 1 gammas, index 0 == 1.0."""
    st = schedule_type.upper()
    if st == "DEEPFLOYD":
        def abar(s):
            return math.cos((s + 0.008) / 1.008 * math.pi / 2) ** 2
        betas = [0]
        for i in range(n_steps):
            betas.append(min(1 - abar((i + 1) / n_steps) / abar(i / n_steps), 0.999))
        return np.exp(np.cumsum(np.log(1.0 - np.asarray(betas))))
    if st == "DDPM":
        betas = np.concatenate(([0], np.linspace(beta_start, beta_end, num=n_steps)))
        return np.exp(np.cumsum(np.log(1.0 - betas)))
    if st == "COSINE":
        t = np.linspace(0.0, 1.0, num=n_steps)
        b = np.arctan(np.exp(-0.5 * 5.0))
        a = np.arctan(np.exp(-0.5 * -5.0)) - b
        logsnrs = -2.0 * np.log(np.tan(a * t + b))
        return np.concatenate(([1.0], 1 / (1 + np.exp(-logsnrs))))
    raise ValueError(schedule_type)


def shift_table(gammas: torch.Tensor, scale, power=1) -> torch.Tensor:
    """get_schedule_shifted: fp32 elementwise on the (already float32) table."""
    if scale is None or scale <= 1:
        return gammas
    sf = scale ** power
    snr = gammas / (1 - gammas)
    return 1 / (1 + 1 / (snr / sf))


def gammas_f32(schedule_type, n_steps, rescale_schedule=1.0, power=1, **kw) -> torch.Tensor:
    g = torch.tensor(schedule_table(schedule_type, n_steps, **kw)).float()
    return shift_table(g.clone(), rescale_schedule, power)


def vdm_weights(gammas: torch.Tensor) -> torch.Tensor:
    g, gl = gammas[2:], gammas[1:-1]
    w = gl * (1 - g) / (1 - gl) / g - 1
    return torch.cat([w[:1], w[:1], w])


def set_timesteps(num_diffusion_steps: int, num_inference_steps: int) -> np.ndarray:
    ratio = (num_diffusion_steps + 1) / (num_inference_steps + 1)
    return (np.arange(0, num_inference_steps + 1) * ratio).round()[::-1].copy().astype(np.int64)


def _b(g):
    return g.view(-1, 1, 1, 1)


def q_sample(x, eps, g):
    return _b(g).sqrt() * x + (1 - _b(g)).sqrt() * eps


def x0_from_pred(x_t, pred, g, ptype):
    g = _b(g)
    if ptype == V_PREDICTION:
        return x_t * g.sqrt() - pred * (1 - g).sqrt()
    return (x_t - pred * (1 - g).sqrt()) / g.sqrt()


def pred_from_x0(x_t, x0, g, ptype):
    g = _b(g)
    if ptype == V_PREDICTION:
        return (g.sqrt() * x_t - x0) / (1 - g).sqrt()
    return (x_t - x0 * g.sqrt()) / (1 - g).sqrt()


def target(x, eps, g, ltype):
    g = _b(g)
    if ltype == V_PREDICTION:
        return g.sqrt() * eps - (1 - g).sqrt() * x
    return eps


def pred_for_training(x_t, pred, g, ptype, ltype):
    if ptype == ltype:
        return pred
    return pred_from_x0(x_t, x0_from_pred(x_t, pred, g, ptype), g, ltype)


def level_loss(model_out, x_t, x, eps, g, ptype, ltype):
    p = pred_for_training(x_t, model_out, g, ptype, ltype)
    t = target(x, eps, g, ltype)
    return ((p - t) ** 2).mean(dim=(1, 2, 3)), p, t


def threshold_sample(sample, ratio=0.995, max_value=100.0):
    """Sampler._threshold_sample (samplers.py:461-498): per-image quantile of |x|, clamp to [1, max], clip and divide.
    torch.quantile (third-party arithmetic, linear interpolation on fp32 ranks) is the anchor."""
    b = sample.shape[0]
    flat = sample.reshape(b, -1)
    # tensor methods only, so that tests/algebra_cases.Mag (an fp64 value with its error magnitude) runs this too
    s = flat.abs().quantile(ratio, dim=1)
    s = s.clamp(min=1, max=max_value).unsqueeze(1)
    return (flat.clamp(-s, s) / s).reshape(sample.shape)


def clip_sample(x0, image_scale, mode):
    """Sampler.clip_sample (samplers.py:500-508). mode: True/'CLIP', 'DYNAMIC', 'DYNAMIC_IF', False/'NONE'."""
    if mode is True or mode == "CLIP":
        return (x0 * image_scale).clip(-1, 1) / image_scale
    if mode == "DYNAMIC":
        return threshold_sample(x0 * image_scale, 0.995, 100.0) / image_scale
    if mode == "DYNAMIC_IF":
        return threshold_sample(x0 * image_scale, 0.95, 1.5) / image_scale
    return x0


def reverse_step(x_t, pred, g, g_last, ptype, clip, image_scale, ddim_eta, need_noise, noise=None):
    """get_prediction_xt_last with scalar g, g_last (0-dim tensors). Returns (x0, x_s).
    clip: bool or the ThresholdType name."""
    alpha = g / g_last
    beta = 1 - alpha
    beta_tilde = beta * (1 - g_last) / (1 - g)
    x0 = x0_from_pred(x_t, pred, g.expand(x_t.shape[0]), ptype)
    if clip:
        x0 = clip_sample(x0, image_scale, clip)
    if ddim_eta is None:
        x_s = x0 * beta * g_last.sqrt() / (1 - g) + x_t * alpha.sqrt() * (1 - g_last) / (1 - g)
    else:
        e = (x_t - x0 * g.sqrt()) / (1 - g).sqrt()
        if ddim_eta > 0:
            beta_tilde = (ddim_eta ** 2) * beta_tilde
            x_s = x0 * g_last.sqrt() + e * (1 - g_last - beta_tilde).sqrt()
        else:
            need_noise = False
            x_s = x0 * g_last.sqrt() + e * (1 - g_last).sqrt()
    if need_noise:
        if noise is None:
            noise = torch.randn_like(x_s)
        x_s = x_s + beta_tilde.sqrt() * noise
    return x0, x_s


def nested_pyramid(images, ratios):
    out = [images]
    for i in range(1, len(ratios)):
        out.append(F.avg_pool2d(out[-1], ratios[i] // ratios[i - 1]))
    return out


def mixed_ratio_fractions(spec):
    """NestedDiffusion.__init__ (diffusion.py:308-313): '2:1' -> cumulative fractions [2/3, 1]."""
    if not spec:
        return None
    mr = np.cumsum(np.asarray([float(x) for x in str(spec).split(":")]))
    return mr / mr[-1]


def training_loss(net, P, images, eps_list, time, lm, mask, gammas, scales, ptype, ltype, shifted, power,
                  weights=None, double_loss=True, mixed_ratio=None, rescale_signal=None):
    """Base (scales == [1]) or nested get_loss given the noise tensors. Returns (loss(B,), x_t list, outs).
    weights: per-level multi_res_weights (diffusion.py:368-374), double_loss: use_double_loss.
    mixed_ratio: cumulative fractions per level (diffusion.py:262-274, 378-382).
    rescale_signal (base pipeline only): x_t is made from images / r, the targets from the unrescaled images
    (diffusion.py:156, 163-165)."""
    nested = len(scales) > 1
    ratios = [scales[0] // s for s in scales]
    imgs = nested_pyramid(images, ratios) if nested else [images]
    g_base = gammas[time + 1]
    gs = [shift_table(g_base, s, power) if (nested and shifted) else g_base for s in scales]
    divs = [1.0 if (not nested or shifted) else float(s) for s in scales]
    xdivs = [float(rescale_signal)] if (not nested and rescale_signal) else divs
    x_t = [q_sample(x / d if d != 1.0 else x, e, g) for x, e, g, d in zip(imgs, eps_list, gs, xdivs)]
    B = images.shape[0]
    x_in = x_t
    if mixed_ratio is not None:  # NestedModel.forward: leading part of the batch per level, zero-padded predictions
        x_in = [x[: int(m * x.size(0))] for x, m in zip(x_t, mixed_ratio)]
    outs = net.forward(P, x_in if nested else x_in[0], time, lm, mask, {})
    outs = list(outs) if nested else [outs]
    if mixed_ratio is not None:
        outs = [torch.cat([p, p.new_zeros(B - p.size(0), *p.size()[1:])], 0) for p in outs]
    w = weights or [1.0] * len(scales)
    loss = 0
    for i in range(len(scales)):
        if i == 0 or double_loss:
            li, _, _ = level_loss(outs[i], x_t[i], imgs[i] / divs[i] if divs[i] != 1.0 else imgs[i], eps_list[i], gs[i],
                                  ptype, ltype)
            if mixed_ratio is not None:
                li = li / float(mixed_ratio[i])
                keep = torch.zeros_like(li)
                keep[: int(mixed_ratio[i] * B)] = 1
                li = li * keep
            loss = loss + li * w[i]
    return loss, x_t, outs


def sample_loop(net, P, x_init, lm, mask, gammas, scales, ptype, n_diffusion, num_inference_steps, ddim_eta, clip=True,
                shifted=False, power=1, guidance_scale=1.0, rescale_signal=None, noises=None, tabs=None, trace=None):
    """p_sample loop (samplers.py:516-578, 655-713) with resampled steps; x_init is a list per level. A full-length
    loop is num_inference_steps == n_diffusion. Returns the final images per level, scaled and clipped as _postprocess
    does (samplers.py:580-599, 715-739).
    clip: the threshold mode (bool or ThresholdType name). noises: per step, the list of per-level noise tensors of
    the stochastic steps (drawn from torch's generator when None). tabs: per-level gamma tables (default: gammas,
    shifted per level when `shifted`). trace: a list that receives (x0 list, x_s list) of every step."""
    nested = len(scales) > 1
    ts = set_timesteps(n_diffusion, num_inference_steps)
    x_t = [x.clone() for x in x_init]
    if tabs is None:
        tabs = [shift_table(gammas, s, power) if (nested and shifted) else gammas for s in scales]
    img_scales = [1.0 if shifted else float(sc) for sc in scales] if nested else \
        [float(rescale_signal) if rescale_signal else 1.0]
    B = x_t[0].shape[0]
    with torch.no_grad():
        for i, t in enumerate(ts[:-1]):
            s = ts[i + 1]
            times = torch.full((B,), int(t) - 1, dtype=torch.long)
            if guidance_scale != 1:
                xin = [torch.cat([x, x]) for x in x_t]
                o = net.forward(P, xin if nested else xin[0], torch.cat([times, times]), lm, mask, {})
                o = list(o) if nested else [o]
                o = [a.chunk(2)[0] + guidance_scale * (a.chunk(2)[1] - a.chunk(2)[0]) for a in o]
            else:
                o = net.forward(P, x_t if nested else x_t[0], times, lm, mask, {})
                o = list(o) if nested else [o]
            nxt, x0s = [], []
            for lv, (x, p, tab, sc) in enumerate(zip(x_t, o, tabs, img_scales)):
                need = (int(t) != 1) if nested else (int(s) != 0)
                nz = noises[i][lv] if noises is not None else None
                x0, xs = reverse_step(x, p, tab[int(t)], tab[int(s)], ptype, clip, sc, ddim_eta, need, noise=nz)
                nxt.append(xs)
                x0s.append(x0)
            x_t = nxt
            if trace is not None:
                trace.append((x0s, nxt))
    return [(x * sc).clip(-1, 1) if sc != 1.0 else x.clip(-1, 1) for x, sc in zip(x_t, img_scales)]
