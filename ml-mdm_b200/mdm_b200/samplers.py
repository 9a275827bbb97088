"""Noise schedules and the DDPM/DDIM p_sample loop behind the reference's `ml_mdm.samplers` interface.

  schedule_*            samplers.py:126-170   (float64 numpy -> float32 table; bit-exact restatement)
  Sampler               samplers.py:177-609   (get_eps_time, get_xt, get_xt_minus_1, forward_model,
                                               sample/_sample generator protocol, _postprocess, set_timesteps)
  NestedSampler         samplers.py:612-793   (per-resolution shifted schedules, list inputs/outputs)
  solver=               DPM-Solver++ 2M / 2M SDE multistep sampling (no counterpart in the reference)

Per-pixel algebra runs in libmdm_b200.so (mdm_q_sample / mdm_sampler_step / mdm_sampler_multistep / mdm_cfg_combine); gamma
is a per-sample table lookup on the device, never a (B,C,H,W) map.  Index math (time steps, table
indices) is integer/float64 on the host exactly as in the reference.
"""
import ctypes as C
import logging
import math

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .config import PredictionType, SamplerConfig, ScheduleType, ThresholdType  # noqa: F401


# ------------------------------------------------------------------ schedules (host, float64)
def schedule_cosine(timesteps: int, logsnr_min: float = -5.0, logsnr_max: float = 5.0) -> np.ndarray:
    """samplers.py:126-136."""
    t = np.linspace(0.0, 1.0, num=timesteps)
    b = np.arctan(np.exp(-0.5 * logsnr_max))
    a = np.arctan(np.exp(-0.5 * logsnr_min)) - b
    logsnrs = -2.0 * np.log(np.tan(a * t + b))
    gammas = 1 / (1 + np.exp(-logsnrs))
    return np.concatenate(([1.0], gammas))


def schedule_ddpm_defults(timesteps: int, beta_start: float, beta_end: float) -> np.ndarray:
    """samplers.py:139-146 (name kept, typo included, for drop-in imports)."""
    betas = np.concatenate(([0], np.linspace(beta_start, beta_end, num=timesteps)))
    return np.exp(np.cumsum(np.log(1.0 - betas)))


def squaredcos_cap_v2(timesteps: int) -> np.ndarray:
    """samplers.py:149-165: beta_i = min(1 - abar((i+1)/T)/abar(i/T), 0.999), gamma = cumprod(1-beta)."""
    def abar(s):
        return math.cos((s + 0.008) / 1.008 * math.pi / 2) ** 2

    betas = [0]
    for i in range(timesteps):
        betas.append(min(1 - abar((i + 1) / timesteps) / abar(i / timesteps), 0.999))
    return np.exp(np.cumsum(np.log(1.0 - np.asarray(betas))))


SOLVERS = ("dpmpp_2m", "dpmpp_2m_sde")


def multistep_coefficients(solver: str, gammas, t: int, s: int, h_prev=None):
    """DPM-Solver++ (Lu et al. 2022) step t -> s of one level: (A, B, C, S, h) with
    x_s = A x_t + B x0_t + C x0_prev + S z, in float64 from the level's gamma table.

    alpha = sqrt(g), sigma = sqrt(1 - g), lambda = log alpha - log sigma, h = lambda_s - lambda_t, r = h_prev / h.
      dpmpp_2m      A = sigma_s / sigma_t,          E = 1 - e^-h
      dpmpp_2m_sde  A = sigma_s / sigma_t e^-h,     E = 1 - e^-2h,   S = sigma_s sqrt(E)
    first order (no previous x0): B = alpha_s E, C = 0; second order: B = alpha_s E (1 + 1/2r), C = -alpha_s E / 2r.
    The final step (s = 0, sigma_s = 0) returns x0: A = C = S = 0, B = 1, h = None.
    h_prev: the level's previous h (None on its first step, or after a step of zero length)."""
    if s == 0:
        return 0.0, 1.0, 0.0, 0.0, None
    g_t, g_s = float(gammas[t]), float(gammas[s])
    a_t, a_s = math.sqrt(g_t), math.sqrt(g_s)
    sig_t, sig_s = math.sqrt(1.0 - g_t), math.sqrt(1.0 - g_s)
    h = (math.log(a_s) - math.log(sig_s)) - (math.log(a_t) - math.log(sig_t))
    if solver == "dpmpp_2m_sde":
        A, E = sig_s / sig_t * math.exp(-h), -math.expm1(-2.0 * h)
        S = sig_s * math.sqrt(E)
    else:
        A, E, S = sig_s / sig_t, -math.expm1(-h), 0.0
    B, Cc = a_s * E, 0.0
    if h_prev:
        half_inv_r = h / (2.0 * h_prev)
        B, Cc = a_s * E * (1.0 + half_inv_r), -a_s * E * half_inv_r
    return A, B, Cc, S, h


def check_solver(solver, ddim_eta):
    if solver is None:
        return
    if solver not in SOLVERS:
        raise ValueError(f"unknown solver {solver!r}: expected None or one of {SOLVERS}")
    if ddim_eta is not None:
        raise ValueError(f"solver={solver!r} does not take ddim_eta (got {ddim_eta!r})")


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _f32c(t):
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.float().contiguous()
    return t


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


class Sampler(nn.Module):
    def __init__(self, sampler_config: SamplerConfig):
        super().__init__()
        self.n_steps = sampler_config.num_diffusion_steps
        self._config = sampler_config
        self.get_noise_schedule(sampler_config.schedule_type, sampler_config.num_diffusion_steps, sampler_config)
        logging.info(f"Step gammas: {self.gammas}")
        if self._config.loss_target_type is None:
            self._config.loss_target_type = self._config.prediction_type
        self._level_tables = {}
        self._text = None  # (lm_outputs, lm_mask, forward_conditioning of them) during a sampling run

    # ---- schedule (samplers.py:201-231,255-264)
    def get_noise_schedule(self, schedule_type, n_steps: int, sampler_config):
        st = getattr(schedule_type, "name", schedule_type)
        if st == "COSINE":
            g = schedule_cosine(n_steps)
        elif st == "DDPM":
            g = schedule_ddpm_defults(n_steps, sampler_config.beta_start, sampler_config.beta_end)
        elif st == "DEEPFLOYD":
            g = squaredcos_cap_v2(n_steps)
        else:
            raise Exception("Unknown")
        self.register_buffer(name="_gammas", tensor=torch.tensor(g).float())
        gammas = self.get_schedule_shifted(self._gammas.clone(), sampler_config.rescale_schedule)
        g2, g_last = gammas[2:], gammas[1:-1]
        weights = g_last * (1 - g2) / (1 - g_last) / g2 - 1
        weights = torch.cat([weights[:1], weights[:1], weights])
        self.register_buffer("gammas", gammas)
        self.register_buffer("vdm_loss_weights", weights)

    def get_schedule_shifted(self, gammas: torch.Tensor, scale_factor: float = None) -> torch.Tensor:
        """gamma' = 1 / (1 + s^p (1-gamma)/gamma) in fp32 on the table (host-side torch, once)."""
        if (scale_factor is not None) and (scale_factor > 1):
            p = self._config.schedule_shifted_power
            scale_factor = scale_factor ** p
            snr = gammas / (1 - gammas)
            scaled_snr = snr / scale_factor
            gammas = 1 / (1 + 1 / scaled_snr)
        return gammas

    def level_table(self, scale, device):
        """Device table of gammas for one resolution level (identity for the base sampler)."""
        key = (float(scale), str(device))
        tab = self._level_tables.get(key)
        if tab is None or tab.device != torch.device(device):
            base = self.gammas.detach().cpu()
            tab = self._shift_for_level(base, scale).contiguous().to(device)
            self._level_tables[key] = tab
        return tab

    def _shift_for_level(self, base, scale):
        return base

    def read_gamma(self, time: torch.Tensor, image: torch.Tensor = None) -> torch.Tensor:
        """Per-sample gamma (B,1,1,1) -- broadcastable where the reference returns a full map."""
        return self.gammas[time].view(-1, 1, 1, 1)

    # ---- training-side draws (samplers.py:233-246)
    def get_eps_time(self, images, time=None):
        batch_size = images.shape[0]
        if time is None:
            time = torch.randint(0, self.n_steps, (batch_size,), device=images.device)
        else:
            time = time * torch.ones(batch_size, dtype=torch.long, device=images.device)
        weights = self.vdm_loss_weights[time + 1]
        eps = torch.randn_like(images)
        return eps, time, weights

    def get_image_rescaled(self, images, scale_factor=None):
        raise NotImplementedError("use the image_div argument of the native q-sample / loss kernels")

    def q_sample(self, images, eps, time, scale=1.0, image_div=1.0):
        """x_t = sqrt(g) x + sqrt(1-g) eps with g = gammas_level[time + 1] (get_xt, samplers.py:244)."""
        images, eps = _f32c(images), _f32c(eps)
        tab = self.level_table(scale, images.device)
        x_t = torch.empty_like(images)
        B = images.shape[0]
        _lib.check(_lib.lib().mdm_q_sample(_ptr(images), _ptr(eps), _ptr(time), _ptr(tab), 1, C.c_float(image_div),
                                           _ptr(x_t), B, C.c_int64(images.numel() // B), _stream()), "mdm_q_sample")
        return x_t

    def q_sample_u8(self, images_u8, eps, time, scale=1.0, image_div=1.0):
        """uint8 NHWC batch (as the data loader yields it, train_parallel.py:193-195) -> (normalised fp32 NCHW images,
        x_t) in one pass (mdm_q_sample_u8)."""
        assert images_u8.dtype == torch.uint8 and images_u8.dim() == 4 and images_u8.is_contiguous()
        B, H, W, Cc = images_u8.shape
        x = torch.empty(B, Cc, H, W, device=images_u8.device, dtype=torch.float32)
        x_t = torch.empty_like(x)
        tab = self.level_table(scale, images_u8.device)
        _lib.check(_lib.lib().mdm_q_sample_u8(_ptr(images_u8), _ptr(_f32c(eps)), _ptr(time), _ptr(tab), 1,
                                              C.c_float(image_div), _ptr(x), _ptr(x_t), B, Cc, H, W, _stream()),
                   "mdm_q_sample_u8")
        return x, x_t

    # ---- reverse process
    _DYNAMIC = {"DYNAMIC": (0.995, 100.0), "DYNAMIC_IF": (0.95, 1.5)}  # clip_sample, samplers.py:500-508

    def _threshold_name(self):
        tf = self._config.threshold_function  # the CLIs overwrite this with an enum or a plain name
        return getattr(tf, "name", tf if isinstance(tf, str) else {0: "NONE", 1: "CLIP", 2: "DYNAMIC", 3: "DYNAMIC_IF"}.get(tf))

    def _clip_flag(self):
        tf = self._threshold_name()
        if tf == "CLIP":
            return 1
        if tf == "NONE":
            return 0
        if tf in self._DYNAMIC:
            return 2
        raise ValueError(f"unknown threshold_function {self._config.threshold_function!r}")

    def _dynamic_bound(self, x_t, pred, tab, t_idx, ptype, image_scale):
        """Per-sample clip bound of dynamic thresholding (mdm_dynamic_threshold): clamp(quantile(|x0 s|, r), 1, max)."""
        ratio, vmax = self._DYNAMIC[self._threshold_name()]
        B = x_t.shape[0]
        bound = torch.empty(B, device=x_t.device, dtype=torch.float32)
        _lib.check(_lib.lib().mdm_dynamic_threshold(_ptr(x_t), _ptr(pred), _ptr(tab), int(t_idx), int(ptype),
                                                    C.c_float(image_scale), C.c_float(ratio), C.c_float(vmax),
                                                    _ptr(bound), B, C.c_int64(x_t.numel() // B), _stream()),
                   "mdm_dynamic_threshold")
        return bound

    def _step_level(self, x_t, pred, t_idx, s_idx, scale, need_noise, ddim_eta, image_scale):
        x_t, pred = _f32c(x_t), _f32c(pred)
        tab = self.level_table(scale, x_t.device)
        x0 = torch.empty_like(x_t)
        x_s = torch.empty_like(x_t)
        use_ddim = ddim_eta is not None
        eta = float(ddim_eta) if use_ddim else 0.0
        stochastic = bool(need_noise) and not (use_ddim and eta <= 0)
        noise = torch.randn_like(x_t) if stochastic else None
        ptype = self._config.prediction_type.value
        clip = self._clip_flag()
        if clip == 2:  # dynamic thresholding: exact per-sample quantile, then the same fused step kernel
            B = x_t.shape[0]
            bound = self._dynamic_bound(x_t, pred, tab, t_idx, ptype, image_scale)
            _lib.check(_lib.lib().mdm_sampler_step_dynamic(_ptr(x_t), _ptr(pred), _ptr(noise), _ptr(tab), int(t_idx),
                                                           int(s_idx), int(ptype), _ptr(bound), C.c_float(image_scale),
                                                           int(use_ddim), C.c_float(eta), int(stochastic), _ptr(x0),
                                                           _ptr(x_s), B, C.c_int64(x_t.numel() // B), _stream()),
                       "mdm_sampler_step_dynamic")
            return x0, x_s
        _lib.check(_lib.lib().mdm_sampler_step(_ptr(x_t), _ptr(pred), _ptr(noise), _ptr(tab), int(t_idx), int(s_idx),
                                               int(ptype), clip, C.c_float(image_scale), int(use_ddim),
                                               C.c_float(eta), int(stochastic), _ptr(x0), _ptr(x_s),
                                               C.c_int64(x_t.numel()), _stream()), "mdm_sampler_step")
        return x0, x_s

    def _multistep_level(self, x_t, pred, t_idx, s_idx, scale, image_scale, solver, hist):
        """One DPM-Solver++ step of one level (mdm_sampler_multistep): x0 thresholded as _step_level does, then
        x_s = A x_t + B x0 + C x0_prev (+ S z). hist: the level's (x0, h) of its previous step, or None.
        Returns (x0, x_s, the level's new hist)."""
        x_t, pred = _f32c(x_t), _f32c(pred)
        tab = self.level_table(scale, x_t.device)
        x0_prev, h_prev = hist if hist is not None else (None, None)
        A, Bc, Cc, S, h = multistep_coefficients(solver, self.level_table(scale, "cpu"), t_idx, s_idx, h_prev)
        noise = torch.randn_like(x_t) if S != 0.0 else None
        ptype = self._config.prediction_type.value
        clip = self._clip_flag()
        bound = self._dynamic_bound(x_t, pred, tab, t_idx, ptype, image_scale) if clip == 2 else None
        x0 = torch.empty_like(x_t)
        x_s = torch.empty_like(x_t)
        B = x_t.shape[0]
        _lib.check(_lib.lib().mdm_sampler_multistep(_ptr(x_t), _ptr(pred), _ptr(x0_prev), _ptr(noise), _ptr(tab),
                                                    int(t_idx), int(ptype), clip, _ptr(bound), C.c_float(image_scale),
                                                    C.c_float(A), C.c_float(Bc), C.c_float(Cc), C.c_float(S),
                                                    _ptr(x0), _ptr(x_s), B, C.c_int64(x_t.numel() // B), _stream()),
                   "mdm_sampler_multistep")
        return x0, x_s, (x0, h)

    def _solver_step(self, model, t, s, x_t, lm_outputs, lm_mask, micros, guidance_scale, solver, hist):
        """One DPM-Solver++ step t -> s (the model sees t - 1). hist: per level index, the level's previous (x0, h);
        updated in place. Returns (x0, x_s, (gamma_t, gamma_s)) as get_xt_minus_1(return_details=True) does."""
        B = x_t.shape[0]
        times = torch.full((B,), t - 1, dtype=torch.long, device=x_t.device)
        pred, _ = self.forward_model(model, x_t, times, lm_outputs, lm_mask, micros, guidance_scale)
        rs = self._config.rescale_signal
        x0, x_s, hist[0] = self._multistep_level(x_t, pred, t, s, 1.0, 1.0 if rs is None else rs, solver, hist.get(0))
        return x0, x_s, (self.gammas[t], self.gammas[s])

    def get_xt_minus_1(self, model, time_step, x_t, lm_outputs, lm_mask, micros={}, time_step_last=None,
                       guidance_scale: float = 1, ddim_eta=None, return_details: bool = False):
        """One reverse step (samplers.py:392-433). The model sees t-1."""
        t = int(time_step)
        s = t - 1 if time_step_last is None else int(time_step_last)
        B = x_t.shape[0]
        times = torch.full((B,), t - 1, dtype=torch.long, device=x_t.device)
        pred, _ = self.forward_model(model, x_t, times, lm_outputs, lm_mask, micros, guidance_scale)
        rs = self._config.rescale_signal
        x0, x_s = self._step_level(x_t, pred, t, s, 1.0, s != 0, ddim_eta, 1.0 if rs is None else rs)
        if return_details:
            return x0, x_s, (self.gammas[t], self.gammas[s])
        return x_s

    def forward_model(self, model, x_t, t, lm_outputs, lm_mask, micros={}, guidance_scale: float = 1):
        """Classifier-free guidance wrapper (samplers.py:435-459): rows are [uncond; cond]."""
        if guidance_scale != 1:
            assert x_t.shape[0] * 2 == lm_outputs.shape[0]
            pred, extras = self._model(model, torch.cat([x_t] * 2), torch.cat([t, t]), lm_outputs, lm_mask, micros)
            u, c = pred.chunk(2)
            pred = self._cfg(u, c, guidance_scale)
            extras = extras.chunk(2)[1]
        else:
            pred, extras = self._model(model, x_t, t, lm_outputs, lm_mask, micros)
        return pred, extras

    # ---- text encoded once per sampling run
    def _encode_text(self, model, lm_outputs, lm_mask):
        """forward_conditioning of the whole run, when `model` is this package's Model / NestedModel (a subclass that
        overrides forward, or any other wrapper, is called as it is at every step). The steps then evaluate
        forward_denoising on it, and the engine reuses the cross-attention K/V it computed at the first step."""
        from .diffusion import Model, NestedModel
        from .models import UNet

        if lm_outputs is None or getattr(type(model), "forward", None) not in (Model.forward, NestedModel.forward):
            return None
        if isinstance(model, NestedModel) and not getattr(model.diffusion_config, "no_use_residual", False):
            return None  # NestedModel.forward raises for the residual mode; let it
        vm = model.vision_model
        if not isinstance(vm, UNet) or vm.native().cfg.cond_dim <= 0:
            return None
        return lm_outputs, lm_mask, vm.forward_conditioning(lm_outputs, lm_mask)

    def _model(self, model, x_t, t, lm_outputs, lm_mask, micros):
        """model(x_t, t, lm_outputs, lm_mask, micros), through the run's encoded text when there is one for exactly
        these lm_outputs / lm_mask tensors."""
        enc = getattr(self, "_text", None)
        if enc is None or enc[0] is not lm_outputs or enc[1] is not lm_mask:
            return model(x_t, t, lm_outputs, lm_mask, micros)
        from .diffusion import NestedModel

        cond_emb, cond, cmask = enc[2]
        vm = model.vision_model
        if isinstance(model, NestedModel):  # NestedModel.forward applies no model_output_scale
            return vm.forward_denoising(x_t, t, cond_emb, cond, cmask, micros)
        out = model.scaled_call(vm.forward_denoising, x_t, t, cond_emb, cond, cmask, micros)
        return out, out.new_ones(()).expand_as(out)  # Model.forward's (outputs, variances placeholder)

    @staticmethod
    def _cfg(u, c, w):
        u, c = _f32c(u), _f32c(c)
        out = torch.empty_like(u)
        _lib.check(_lib.lib().mdm_cfg_combine(_ptr(u), _ptr(c), C.c_float(w), _ptr(out), C.c_int64(u.numel()),
                                              _stream()), "mdm_cfg_combine")
        return out

    def clip_sample(self, pred_x0, image_scale=1):
        """samplers.py:500-508 on an x0 tensor (the sampling loop itself uses the fused step kernels)."""
        clip = self._clip_flag()
        if clip == 0:
            return pred_x0
        x = _f32c(pred_x0)
        s = float(image_scale)
        if clip == 1:
            y = self._scale_clip(x, s, True)
            return y if s == 1.0 else self._scale_clip(y, 1.0 / s, False)
        # dynamic: the kernels rebuild x0 from (x_t, pred) as x_t sqrt(g) - pred sqrt(1-g); with g = 1 that is x_t itself
        one = torch.ones(1, device=x.device, dtype=torch.float32)
        B = x.shape[0]
        bound = self._dynamic_bound(x, x, one, 0, PredictionType.V_PREDICTION.value, s)
        x0 = torch.empty_like(x)
        xs = torch.empty_like(x)
        _lib.check(_lib.lib().mdm_sampler_step_dynamic(_ptr(x), _ptr(x), None, _ptr(one), 0, 0,
                                                       int(PredictionType.V_PREDICTION.value), _ptr(bound), C.c_float(s),
                                                       1, C.c_float(0.0), 0, _ptr(x0), _ptr(xs), B,
                                                       C.c_int64(x.numel() // B), _stream()), "mdm_sampler_step_dynamic")
        return x0

    @staticmethod
    def _scale_clip(x, scale, clip):
        x = _f32c(x)
        y = torch.empty_like(x)
        _lib.check(_lib.lib().mdm_clip_scale(_ptr(x), C.c_float(scale), int(bool(clip)), _ptr(y), C.c_int64(x.numel()),
                                             _stream()), "mdm_clip_scale")
        return y

    def sample(self, *args, **kwargs):
        if not kwargs.get("yield_output", False):
            return next(self._sample(*args, **kwargs))
        return self._sample(*args, **kwargs)

    def _sample(self, model, x_t, lm_outputs, lm_mask, micros, return_sequence: bool = False,
                use_beta_tilde: bool = False, t: int = -1, num_inference_steps: int = 2000, ddim_eta=None,
                guidance_scale: float = 1, resample_steps: bool = False, disable_bar: bool = True,
                yield_output: bool = False, solver=None, **post_args):
        """p_sample loop (samplers.py:516-578), generator protocol preserved.
        solver: None (DDPM, or DDIM with ddim_eta) or one of SOLVERS, DPM-Solver++ multistep over the same time steps."""
        assert not (yield_output and return_sequence), "not allowed."
        check_solver(solver, ddim_eta)
        if not resample_steps:
            num_inference_steps = self.n_steps
        timesteps = self.set_timesteps(num_inference_steps)
        if t > -1:
            timesteps = timesteps[timesteps <= t]
        seq = [x_t] if return_sequence else []
        x0, extra = None, None
        hist = {}
        with torch.no_grad():
            self._text = self._encode_text(model, lm_outputs, lm_mask)
            try:
                for i, tt in enumerate(timesteps[:-1]):
                    t_last = timesteps[i + 1] if resample_steps else None
                    if solver is not None:
                        x0, x_t, extra = self._solver_step(model, int(tt), int(timesteps[i + 1]), x_t, lm_outputs,
                                                           lm_mask, micros, guidance_scale, solver, hist)
                    else:
                        x0, x_t, extra = self.get_xt_minus_1(model, int(tt), x_t, lm_outputs, lm_mask, micros,
                                                             time_step_last=None if t_last is None else int(t_last),
                                                             guidance_scale=guidance_scale, ddim_eta=ddim_eta,
                                                             return_details=True)
                    if yield_output:
                        yield self._postprocess(x_t, x0, extra, **post_args)
                    if return_sequence:
                        seq.append(self._postprocess(x_t))
            finally:
                self._text = None
            if return_sequence:
                seq[-1] = self._scale_clip(seq[-1], 1.0, True)
                yield seq
            else:
                yield self._postprocess(x_t, x0, extra, clip=True, **post_args)

    def _postprocess(self, x_t, x0=None, extra=None, yield_full: bool = False, clip: bool = False,
                     image_scale: float = None, **unused):
        if image_scale is None:
            image_scale = self._config.rescale_signal
        sc = float(image_scale) if image_scale else 1.0
        if sc != 1.0 or clip:
            x_t = self._scale_clip(x_t, sc, clip)
            if x0 is not None and sc != 1.0:
                x0 = self._scale_clip(x0, sc, False)
        if yield_full:
            return (x0, x_t, extra)
        return x_t

    def set_timesteps(self, num_inference_steps: int = 250) -> np.ndarray:
        """round-half-even of arange * (T+1)/(N+1), descending, int64 (samplers.py:601-609)."""
        step_ratio = (self._config.num_diffusion_steps + 1) / (num_inference_steps + 1)
        return (np.arange(0, num_inference_steps + 1) * step_ratio).round()[::-1].copy().astype(np.int64)


class NestedSampler(Sampler):
    def _shift_for_level(self, base, scale):
        if not self._config.schedule_shifted:
            return base
        return self.get_schedule_shifted(base, scale)

    def get_gammas(self, gamma, scales, images=None):
        """Per-level gammas of per-sample values (samplers.py:613-623)."""
        if not self._config.schedule_shifted:
            return [gamma for _ in scales]
        return [self.get_schedule_shifted(gamma, s) for s in scales]

    def level_image_div(self, scale):
        return 1.0 if self._config.schedule_shifted else float(scale)

    def get_xt_minus_1(self, model, time_step, x_t, lm_outputs, lm_mask, micros={}, time_step_last=None,
                       guidance_scale=1, ddim_eta=None, return_details=False):
        """samplers.py:655-713. x_t: full-resolution tensor (first call) or list high -> low."""
        scales = model.vision_model.nest_ratio + [1]
        x_t = self._level_inputs(x_t, scales)
        t = int(time_step)
        s_idx = t - 1 if time_step_last is None else int(time_step_last)
        B = x_t[0].shape[0]
        times = torch.full((B,), t - 1, dtype=torch.long, device=x_t[0].device)
        p_t = self.forward_model(model, x_t, times, lm_outputs, lm_mask, micros, guidance_scale)
        x0, x_s = [], []
        for x, p, sc in zip(x_t, p_t, scales):
            a, b = self._step_level(x, p, t, s_idx, sc, t != 1, ddim_eta,
                                    1.0 if self._config.schedule_shifted else float(sc))
            x0.append(a)
            x_s.append(b)
        if return_details:
            tab = self.level_table(scales[-1], x_t[0].device)
            return x0, x_s, (tab[t], tab[s_idx])
        return x_s

    @staticmethod
    def _level_inputs(x_t, scales):
        """The first step's full-resolution tensor -> one tensor per level, the lower ones drawn with normal_
        (samplers.py:664-672); a list is returned as it is."""
        if not isinstance(x_t, torch.Tensor):
            return x_t
        out = [x_t]
        for s in scales[1:]:
            ratio = scales[0] // s
            b, c, h, w = x_t.shape
            out.append(torch.empty(b, c, h // ratio, w // ratio, device=x_t.device, dtype=x_t.dtype).normal_())
        return out

    def _solver_step(self, model, t, s, x_t, lm_outputs, lm_mask, micros, guidance_scale, solver, hist):
        """Sampler._solver_step per level, each with its own table and history (x_t as in get_xt_minus_1)."""
        scales = model.vision_model.nest_ratio + [1]
        x_t = self._level_inputs(x_t, scales)
        B = x_t[0].shape[0]
        times = torch.full((B,), t - 1, dtype=torch.long, device=x_t[0].device)
        p_t = self.forward_model(model, x_t, times, lm_outputs, lm_mask, micros, guidance_scale)
        x0, x_s = [], []
        for l, (x, p, sc) in enumerate(zip(x_t, p_t, scales)):
            a, b, hist[l] = self._multistep_level(x, p, t, s, sc, 1.0 if self._config.schedule_shifted else float(sc),
                                                  solver, hist.get(l))
            x0.append(a)
            x_s.append(b)
        tab = self.level_table(scales[-1], x_t[0].device)
        return x0, x_s, (tab[t], tab[s])

    def _postprocess(self, x_t, x0=None, extra=None, yield_full: bool = False, clip: bool = False,
                     output_inner: bool = False, **unused):
        """samplers.py:715-772: level 0 (optionally all levels side by side, low resolution first)."""
        scales = [x_t[i].size(-1) / x_t[-1].size(-1) if not self._config.schedule_shifted else 1
                  for i in range(len(x_t))]
        out = super()._postprocess(x_t[0], x0[0] if x0 is not None else x0, extra, yield_full=yield_full, clip=clip,
                                   image_scale=scales[0], **unused)
        if output_inner:
            # visualisation only (web demo): outside the denoising loop, resized with torch's bilinear kernel
            import torch.nn.functional as F

            outs = [out]
            for i in range(1, len(x_t)):
                outs.append(super()._postprocess(x_t[i], x0[i] if x0 is not None else None, extra,
                                                 yield_full=yield_full, clip=clip, image_scale=scales[i], **unused))
            # both sides, for rectangles: a case the reference's nested pipeline never reaches (its gamma maps are
            # resized to a square, samplers.py:618-622); for square images this is its int size
            size = tuple(x_t[0].shape[-2:])
            if not yield_full:
                out = torch.cat([F.interpolate(o, size, mode="bilinear") for o in outs[::-1]], -1)
            else:
                a, b, e = zip(*outs)
                out = (torch.cat([F.interpolate(o, size, mode="bilinear") for o in a[::-1]], -1),
                       torch.cat([F.interpolate(o, size, mode="bilinear") for o in b[::-1]], -1), e[-1])
        return out

    def forward_model(self, model, x_t, t, lm_outputs, lm_mask, micros={}, guidance_scale=1):
        """samplers.py:774-793."""
        if guidance_scale != 1:
            assert x_t[0].shape[0] * 2 == lm_outputs.shape[0]
            p_t = self._model(model, [torch.cat([x] * 2) for x in x_t], torch.cat([t] * 2), lm_outputs, lm_mask, micros)
            return [self._cfg(*p.chunk(2), guidance_scale) for p in p_t]
        return self._model(model, x_t, t, lm_outputs, lm_mask, micros)
