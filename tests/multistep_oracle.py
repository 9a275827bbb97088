"""fp64 oracle of DPM-Solver++ multistep sampling (mdm_sampler_multistep, Sampler(..., solver=...)) and analytic
denoisers whose E[x0 | x_t] is known in closed form.

Solver      x_s = A x_t + B x0_t + C x0_prev + S z, restated from DPM-Solver++ (Lu et al. 2022, 2M; the SDE variant
            of its section 5) with alpha = sqrt(g), sigma = sqrt(1 - g), lambda = log alpha - log sigma,
            h = lambda_s - lambda_t and r = h_prev / h. x0 is the thresholded data prediction of
            oracle/diffusion_ref.reverse_step. step() uses tensor operations only, so it also runs on
            tests/algebra_cases.Mag values (fp64 value and forward-error magnitude).
Denoisers   per-pixel data distributions, x0 ~ N(mu, s^2) or a two-component Gaussian mixture inside [-1, 1]; at
            x_t = alpha x0 + sigma eps the posterior mean is exact. For the single Gaussian the probability-flow ODE
            maps x_T to x0 = mu + s (x_T - alpha_T mu) / sqrt(alpha_T^2 s^2 + sigma_T^2) (gaussian_flow).
"""
import math

import numpy as np
import torch

from oracle import diffusion_ref as dref

SOLVERS = ("dpmpp_2m", "dpmpp_2m_sde")


# ---------------------------------------------------------------- the solver
def lam(g):
    g = float(g)
    return 0.5 * math.log(g) - 0.5 * math.log(1.0 - g)


def coefficients(solver, g_t, g_s, s, h_prev):
    """(A, B, C, S, h) of one step t -> s of one level in float64; g_t, g_s: the level's table entries.
    h_prev: the level's previous h, None on its first step. s == 0: the final step returns x0."""
    if s == 0:
        return 0.0, 1.0, 0.0, 0.0, None
    g_t, g_s = float(g_t), float(g_s)
    alpha_s, sigma_t, sigma_s = math.sqrt(g_s), math.sqrt(1 - g_t), math.sqrt(1 - g_s)
    h = lam(g_s) - lam(g_t)
    sde = solver == "dpmpp_2m_sde"
    e = 1 - math.exp(-2 * h) if sde else 1 - math.exp(-h)
    A = sigma_s / sigma_t * (math.exp(-h) if sde else 1.0)
    S = sigma_s * math.sqrt(e) if sde else 0.0
    if not h_prev:
        return A, alpha_s * e, 0.0, S, h
    r = h_prev / h
    return A, alpha_s * e * (1 + 1 / (2 * r)), -alpha_s * e / (2 * r), S, h


def x0_of(x_t, pred, g_t, ptype, threshold, image_scale):
    """Thresholded data prediction, as the reverse step computes it. threshold: ThresholdType name."""
    x0 = dref.x0_from_pred(x_t, pred, g_t.expand(x_t.shape[0]), ptype)
    return dref.clip_sample(x0, image_scale, False if threshold == "NONE" else threshold)


def step(x_t, pred, g_t, ptype, threshold, image_scale, coef, x0_prev=None, z=None):
    """(x0, x_s) of one multistep update with coefficients coef = (A, B, C, S) (floats or 0-dim tensors)."""
    A, B, Cc, S = coef
    x0 = x0_of(x_t, pred, g_t, ptype, threshold, image_scale)
    x_s = x_t * A + x0 * B
    if x0_prev is not None and float(Cc) != 0.0:
        x_s = x_s + x0_prev * Cc
    if z is not None and float(S) != 0.0:
        x_s = x_s + z * S
    return x0, x_s


def ddim_step(x_t, pred, g_t, g_s, ptype, threshold, image_scale):
    """The package's DDIM eta = 0 step (oracle/diffusion_ref.reverse_step)."""
    return dref.reverse_step(x_t, pred, g_t, g_s, ptype, False if threshold == "NONE" else threshold, image_scale,
                             0.0, False)


# ---------------------------------------------------------------- analytic denoisers
class Gaussian:
    """x0 ~ N(mu, s^2) per pixel (mu, s: tensors broadcastable to the image)."""

    def __init__(self, mu, s):
        self.mu, self.s = mu.double(), s.double()

    def x0(self, x_t, g):
        a2 = g
        return self.mu + math.sqrt(a2) * self.s ** 2 * (x_t - math.sqrt(a2) * self.mu) / (a2 * self.s ** 2 + 1 - a2)

    def flow(self, x_T, g_T, g=1.0):
        """Probability-flow ODE solution from x_T at g_T to g (g = 1: the endpoint x0)."""
        scale = math.sqrt(g) ** 2 * self.s ** 2 + 1 - g
        return math.sqrt(g) * self.mu + scale.sqrt() * (x_T - math.sqrt(g_T) * self.mu) / \
            (g_T * self.s ** 2 + 1 - g_T).sqrt()


class Mixture:
    """x0 ~ w N(mu1, s1^2) + (1 - w) N(mu2, s2^2) per pixel, components inside [-1, 1]."""

    def __init__(self, w, mu1, s1, mu2, s2):
        self.w, self.comp = float(w), ((mu1.double(), s1.double()), (mu2.double(), s2.double()))

    def x0(self, x_t, g):
        a = math.sqrt(g)
        logs, means = [], []
        for wk, (mu, s) in zip((self.w, 1 - self.w), self.comp):
            var = g * s ** 2 + 1 - g
            logs.append(math.log(wk) - 0.5 * torch.log(var) - 0.5 * (x_t - a * mu) ** 2 / var)
            means.append(mu + a * s ** 2 * (x_t - a * mu) / var)
        r1 = torch.sigmoid(logs[0] - logs[1])
        return r1 * means[0] + (1 - r1) * means[1]


def as_prediction(x0, x_t, g, ptype):
    """E[x0 | x_t] as the model output of prediction type ptype (eps or v)."""
    if ptype == dref.V_PREDICTION:
        return (math.sqrt(g) * x_t - x0) / math.sqrt(1 - g)
    return (x_t - math.sqrt(g) * x0) / math.sqrt(1 - g)


def gaussian_case(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return Gaussian(torch.rand(shape, generator=g) - 0.5, 0.3 + 0.2 * torch.rand(shape, generator=g))


def mixture_case(shape, seed):
    g = torch.Generator().manual_seed(seed)
    u = lambda lo, hi: lo + (hi - lo) * torch.rand(shape, generator=g)  # noqa: E731
    return Mixture(0.4, u(-0.6, -0.4), u(0.15, 0.25), u(0.3, 0.5), u(0.15, 0.25))


# ---------------------------------------------------------------- sampling loops
def sample_loop(den, x_T, tab, timesteps, solver, ptype, threshold="NONE", image_scale=1.0, noises=None, trace=None):
    """fp64 loop of Sampler.sample over `timesteps` (descending, ending at 0) on one level with the analytic
    denoiser: solver 'ddim' (eta 0) or one of SOLVERS. tab: the level's fp32 gamma table (values read as float64).
    noises: per step the SDE's z (or None). trace: receives (x_t, pred, x0, x_s) of every step.
    Returns the final x_s (= the last step's x0)."""
    x = x_T.double()
    x0_prev, h_prev = None, None
    for i, t in enumerate(timesteps[:-1]):
        t, s = int(t), int(timesteps[i + 1])
        g_t = float(tab[t])
        pred = as_prediction(den.x0(x, g_t), x, g_t, ptype)
        gt = torch.tensor(g_t, dtype=torch.float64)
        if solver == "ddim":
            x0, xs = ddim_step(x, pred, gt, torch.tensor(float(tab[s]), dtype=torch.float64), ptype, threshold,
                               image_scale)
        else:
            A, B, Cc, S, h = coefficients(solver, g_t, tab[s], s, h_prev)
            z = noises[i] if (noises is not None and S != 0.0) else None
            x0, xs = step(x, pred, gt, ptype, threshold, image_scale, (A, B, Cc, S), x0_prev, z)
            x0_prev, h_prev = x0, h
        if trace is not None:
            trace.append((x, pred, x0, xs))
        x = xs
    return x


def fine_flow(den, x, g_from, g_to, n=2000):
    """Probability-flow ODE from g_from to g_to (both < 1) by 2M on n steps uniform in lambda: the reference solution
    where no closed form exists (its error is checked against Gaussian.flow in tests/test_multistep_host.py)."""
    l0, l1 = lam(g_from), lam(g_to)
    gs = [1 / (1 + math.exp(-2 * (l0 + (l1 - l0) * i / n))) for i in range(n + 1)]
    x = x.double()
    x0_prev, h_prev = None, None
    for i in range(n):
        x0 = den.x0(x, gs[i])
        A, B, Cc, _, h = coefficients("dpmpp_2m", gs[i], gs[i + 1], 1, h_prev)
        x = x * A + x0 * B + (x0_prev * Cc if x0_prev is not None else 0.0)
        x0_prev, h_prev = x0, h
    return x


def table(schedule, n=1000):
    return np.asarray(dref.gammas_f32(schedule, n).double())


def exact_endpoint(den, x_T, tab, ts):
    """What a loop over time steps ts returns without discretisation error: the exact flow from ts[0] to the last
    non-zero step ts[-2], then the final step's x0 = E[x0 | x] there, which every solver takes as it is."""
    g_T, g_1 = float(tab[int(ts[0])]), float(tab[int(ts[-2])])
    x_1 = den.flow(x_T, g_T, g_1) if isinstance(den, Gaussian) else fine_flow(den, x_T, g_T, g_1)
    return den.x0(x_1, g_1)


def rms(a, b):
    return float((a - b).pow(2).mean().sqrt())
