"""Shared cases of the diffusion-algebra tests (tests/test_algebra_oracle.py on the CPU, tests/test_algebra_gpu.py on
the GPU, tests/golden/make_golden_algebra.py for the reference fixture tests/golden/algebra.npz).

Stub        a small deterministic denoiser standing in for the U-Net, so the algebra around it (q-sample, the
            per-sample loss and its gradient, the reverse step, CFG, the pyramid, clip / scale) can be compared at
            fp32 rounding level instead of behind the network's 1e-3:
                out_c = tanh(w_c x_t + b_c) + k_c t / 1000 + q_c lm_outputs[b, 0, 0]    per channel c
            (the lm term makes the conditional and unconditional rows of classifier-free guidance differ).
            NestedStub applies one such stub per resolution level.
Grids       the sampler / loss options of the reference's SamplerConfig and (Nested)DiffusionConfig covered, pairwise.
Mag         an fp64 value with the magnitude of its forward error bound. Evaluating the oracle on Mag values gives
            the same fp64 result, and alongside it `mag`: the same expression with |.| on every operand and + for every
            -. An fp32 evaluation of the expression is within c * 2^-24 * mag of the fp64 value, c about the number of
            roundings on the longest path. The c used per quantity is stated below (C_*).
"""
import math

import numpy as np
import torch
import torch.nn as nn

from oracle import diffusion_ref as dref

U = 2.0 ** -24  # unit roundoff of fp32

# c per quantity, for |got - ref64| <= c * U * mag
C_XT = 8      # q-sample: sqrt, sqrt, 1 - g, /div, two products, one sum
C_ELEM = 32   # pred_for_training / target / reverse step / clip: at most ~12 roundings on a path, x2 for the kernels'
              # and torch's different association (FMA contraction, the reference's separate products)
C_GRAD = 32   # d loss / d model output: 2 (p - tgt) / per * dloss * weight * dp/dv
C_PARAM = 256  # stub-parameter gradients: torch's fp32 reductions over B*H*W terms in the stub's backward
C_STEP_LOOP = 32  # per reverse step of a sampling loop (the stub, the step, the clip); times the number of steps


def loss_c(per):
    """c of the per-sample loss, from mdm_loss_fwd's summation order: a serial sum per thread over
    ceil(per / (chunks * 256)) values, 5 warp-shuffle and 8 per-warp additions, one fp32 atomic per chunk
    (chunks = min(ceil(per / 1024), 64)), the weight / per scaling, plus 2 C_ELEM for the squared difference."""
    chunks = max(1, min(-(-per // 1024), 64))
    return -(-per // (chunks * 256)) + 5 + 8 + chunks + 4 + 2 * C_ELEM


# ---------------------------------------------------------------- error-bound arithmetic
class Mag:
    """fp64 value `v` and error magnitude `m` (>= |v|). Operands read exactly from fp32 data are `exact`: an operation
    on two exact operands rounds once, so its result has m = |v|; otherwise + and - add magnitudes, * multiplies
    them, / divides by |denominator|, sqrt divides by sqrt(|v|), clamping to a computed bound adds its magnitude."""

    __slots__ = ("v", "m", "exact")

    def __init__(self, v, m=None, exact=False):
        self.v = v
        self.m = v.abs() if m is None else m
        self.exact = exact

    @staticmethod
    def of(x):
        if isinstance(x, Mag):
            return x
        return Mag(torch.as_tensor(x).double(), exact=True)

    def _bin(self, o, f, fm, rev=False):
        o = Mag.of(o)
        a, b = (o, self) if rev else (self, o)
        v = f(a.v, b.v)
        return Mag(v) if (a.exact and b.exact) else Mag(v, fm(a, b))

    def __add__(self, o):
        return self._bin(o, torch.add, lambda a, b: a.m + b.m)

    def __radd__(self, o):
        return self._bin(o, torch.add, lambda a, b: a.m + b.m, True)

    def __sub__(self, o):
        return self._bin(o, torch.sub, lambda a, b: a.m + b.m)

    def __rsub__(self, o):
        return self._bin(o, torch.sub, lambda a, b: a.m + b.m, True)

    def __mul__(self, o):
        return self._bin(o, torch.mul, lambda a, b: a.m * b.m)

    def __rmul__(self, o):
        return self._bin(o, torch.mul, lambda a, b: a.m * b.m, True)

    def __truediv__(self, o):
        return self._bin(o, torch.div, lambda a, b: a.m / b.v.abs())

    def __rtruediv__(self, o):
        return self._bin(o, torch.div, lambda a, b: a.m / b.v.abs(), True)

    def __neg__(self):
        return Mag(-self.v, self.m, self.exact)

    def __pow__(self, p):
        assert p == 2
        return self * self

    def sqrt(self):
        v = self.v.sqrt()
        if self.exact:
            return Mag(v)
        return Mag(v, torch.where(self.m == 0, self.m, self.m / v.clamp_min(1e-300)))

    def tanh(self):
        v = self.v.tanh()
        return Mag(v) if self.exact else Mag(v, (1 - v * v) * self.m + v.abs())

    def abs(self):
        return Mag(self.v.abs(), self.m, self.exact)

    def clamp(self, min=None, max=None):  # noqa: A002 -- torch's names
        lo, hi = (b.v if isinstance(b, Mag) else b for b in (min, max))
        v = torch.clamp(self.v, lo, hi)
        m = self.m
        for b in (min, max):  # a clamped value carries the bound's error, which adds to the value's once divided by it
            if isinstance(b, Mag):
                m = m + b.m
        return Mag(v, m, self.exact)

    def clip(self, lo, hi):
        return self.clamp(lo, hi)

    def quantile(self, q, dim):  # an order statistic moves by at most the largest input error
        return Mag(torch.quantile(self.v, q, dim=dim), self.m.amax(dim=dim))

    def mean(self, dim):
        return Mag(self.v.mean(dim=dim), self.m.mean(dim=dim))

    def _map(self, f):
        return Mag(f(self.v), f(self.m), self.exact)

    def view(self, *s):
        return self._map(lambda t: t.view(*s))

    def reshape(self, *s):
        return self._map(lambda t: t.reshape(*s))

    def expand(self, *s):
        return self._map(lambda t: t.expand(*s))

    def unsqueeze(self, d):
        return self._map(lambda t: t.unsqueeze(d))

    def clone(self):
        return self._map(torch.clone)

    def __getitem__(self, i):
        return self._map(lambda t: t[i])

    def chunk(self, n):
        return [Mag(v, m, self.exact) for v, m in zip(self.v.chunk(n), self.m.chunk(n))]

    @property
    def shape(self):
        return self.v.shape

    def size(self, *d):
        return self.v.size(*d)

    def new_zeros(self, *s):
        return self.v.new_zeros(*s)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func is torch.cat:
            xs = [Mag.of(x) for x in args[0]]
            d = args[1] if len(args) > 1 else kwargs.get("dim", 0)
            return Mag(torch.cat([x.v for x in xs], d), torch.cat([x.m for x in xs], d), all(x.exact for x in xs))
        if func is torch.zeros_like:
            return torch.zeros_like(args[0].v)
        if func is torch.nn.functional.avg_pool2d:
            x = args[0]
            return Mag(func(x.v, *args[1:], **kwargs), func(x.m, *args[1:], **kwargs))
        return NotImplemented


def excess(got, ref, c):
    """max |got - ref.v| / (c U ref.m): <= 1 passes the bound. got: a tensor (any device), ref: a Mag."""
    d = (got.detach().double().cpu() - ref.v.cpu()).abs()
    return float((d / (c * U * ref.m.cpu()).clamp_min(1e-300)).max())


def assert_bound(got, ref, c, what, worst=None):
    r = excess(got, ref, c)
    if worst is not None:
        worst[what.split("/")[0]] = max(worst.get(what.split("/")[0], 0.0), r * c)
    assert r <= 1.0, f"{what}: |got - ref| reaches {r:.3g} x the bound c={c}"


# ---------------------------------------------------------------- the stub denoiser
def stub_out(w, b, k, q, x, times, lm):
    """The stub's arithmetic, on torch tensors or on Mag values; w, b, k, q shaped (1, C, 1, 1)."""
    B = x.shape[0]
    dt = x.v.dtype if isinstance(x, Mag) else x.dtype
    tt = times[:B].view(-1, 1, 1, 1).to(dt)
    lv = lm[:B, 0, 0].reshape(-1, 1, 1, 1).to(dt)
    return (x * w + b).tanh() + k * (tt / 1000.0) + q * lv


def stub_params(seed, levels, channels=3):
    g = torch.Generator().manual_seed(seed)
    return dict(w=0.5 + torch.rand(levels, channels, generator=g), b=torch.randn(levels, channels, generator=g) * 0.3,
                k=torch.randn(levels, channels, generator=g) * 0.5, q=torch.randn(levels, channels, generator=g))


class Stub(nn.Module):
    """Plain denoiser stub with the attributes the pipelines read (conditions, input_channels, output_scale,
    fuse_lm_mask). model_output_scale stays 0: the package applies it in its engine, not in Model.forward.
    `outputs` keeps the outputs of the last call, with retain_grad() when they need a gradient."""

    nested = False

    def __init__(self, seed=0, levels=1, channels=3):
        super().__init__()
        for n, v in stub_params(seed, levels, channels).items():
            setattr(self, n, nn.Parameter(v))
        self.conditions = None
        self.input_channels = channels
        self.output_scale = 0.0
        self.fuse_lm_mask = False
        self.outputs = []

    def level(self, l, x, times, lm):
        P = [getattr(self, n)[l].view(1, -1, 1, 1) for n in "wbkq"]
        out = stub_out(*P, x, times, lm)
        if out.requires_grad:
            out.retain_grad()
        return out

    def forward(self, x_t, times, lm_outputs, lm_mask, micros={}):
        out = self.level(0, x_t, times, lm_outputs)
        self.outputs = [out]
        return out


class NestedStub(Stub):
    """One stub per level, high resolution first; nest_ratio as in NestedUNetConfig (scales = nest_ratio + [1])."""

    nested = True

    def __init__(self, nest_ratio, seed=0, channels=3):
        super().__init__(seed, len(nest_ratio) + 1, channels)
        self.nest_ratio = list(nest_ratio)
        self.is_temporal = [False] * len(nest_ratio)

    def forward(self, x_t, times, lm_outputs, lm_mask, micros={}):
        self.outputs = [self.level(l, x, times, lm_outputs) for l, x in enumerate(x_t)]
        return self.outputs


class StubNet:
    """The stub in the oracle's net.forward(P, x, times, lm, mask, micros) form. P: dict of (levels, C) tensors
    (fp64 leaves for autograd) or of Mag; x a tensor / Mag (plain) or a list of them (nested)."""

    @staticmethod
    def forward(P, x, times, lm, mask, micros):
        def lv(l, xi):
            return stub_out(*[P[n][l].view(1, -1, 1, 1) for n in "wbkq"], xi, times, lm)

        if isinstance(x, (list, tuple)):
            return [lv(l, xi) for l, xi in enumerate(x)]
        return lv(0, x)


def mag_params(stub):
    return {n: Mag.of(getattr(stub, n).detach().cpu()) for n in "wbkq"}


def f64_params(stub):
    return {n: getattr(stub, n).detach().cpu().double().requires_grad_(True) for n in "wbkq"}


def param_grad_mag(P64, x_list, times, lm, gmags):
    """Per stub parameter, sum over elements of |d loss / d out|-magnitude * |d out / d parameter|."""
    out = {n: torch.zeros_like(P64[n], dtype=torch.float64) for n in "wbkq"}
    for l, (x, gm) in enumerate(zip(x_list, gmags)):
        B = x.shape[0]
        xv = x.v if isinstance(x, Mag) else x.double()
        w, b = P64["w"][l].detach().view(1, -1, 1, 1), P64["b"][l].detach().view(1, -1, 1, 1)
        s2 = 1 - ((xv * w + b).tanh()) ** 2
        tt = times[:B].double().view(-1, 1, 1, 1) / 1000.0
        lv = lm[:B, 0, 0].double().reshape(-1, 1, 1, 1)
        for n, d in (("w", s2 * xv.abs()), ("b", s2), ("k", tt.expand_as(xv)), ("q", lv.abs().expand_as(xv))):
            out[n][l] = (gm * d).sum(dim=(0, 2, 3))
    return out


# ---------------------------------------------------------------- option grids
PT = {"DDPM": dref.DDPM, "DDIM": dref.DDIM, "V_PREDICTION": dref.V_PREDICTION}
_ST = "V_PREDICTION"


def _loss(name, ptype=_ST, ltype="DDPM", schedule="DEEPFLOYD", nest=None, **kw):
    return dict(name=name, ptype=ptype, ltype=ltype, schedule=schedule, nest=nest, **kw)


LOSS_GRID = (
    [_loss(f"{p}_{l}", p, l) for p in PT for l in PT]                       # all 9 prediction / target pairs
    + [_loss(f"{s}_{p}_{l}", p, l, s) for s in ("DDPM", "COSINE") for p, l in ((_ST, "DDPM"), ("DDPM", _ST))]
    + [_loss("rescale2_V_DDPM", rescale_signal=2), _loss("rescale2_DDPM_V", "DDPM", _ST, rescale_signal=2),
       _loss("vdm_weights", use_vdm_loss_weights=True)]
    + [_loss("n2_shift", nest=[4], shifted=True),
       _loss("n2_unshift_V_DDPM", nest=[4], shifted=False),
       _loss("n2_unshift_DDPM_V", "DDPM", _ST, nest=[4], shifted=False),
       _loss("n3_p2_weights", nest=[4, 2], shifted=True, power=2, multi_res_weights="16:4:1"),
       _loss("n2_single_loss", "DDIM", _ST, nest=[4], shifted=True, double_loss=False),
       _loss("n2_mixed", nest=[4], shifted=True, mixed_ratio="2:1", B=3),
       _loss("n3_mixed_weights", _ST, _ST, nest=[4, 2], shifted=True, power=2, multi_res_weights="16:4:1",
             mixed_ratio="1:1:2")]
)
LOSS_B, LOSS_SIDE = 4, 8          # plain batches; nested: top level LOSS_SIDE * 2


def loss_side(case):
    return LOSS_SIDE * 2 if case["nest"] else LOSS_SIDE


# sampler pipelines: (nest ratio, shifted, power, rescale_signal, schedule, num_diffusion_steps)
PIPES = {
    "plain": (None, False, 1, None, "DEEPFLOYD", 1000),
    "plain_rs2": (None, False, 1, 2, "DEEPFLOYD", 1000),
    "plain_cos": (None, False, 1, None, "COSINE", 1000),
    "n2_shift": ([4], True, 1, None, "DEEPFLOYD", 1000),
    "n2_unshift": ([4], False, 1, None, "DEEPFLOYD", 1000),
    "n3_p2": ([4, 2], True, 2, None, "DEEPFLOYD", 1000),
    "plain20": (None, False, 1, 2, "DEEPFLOYD", 20),
    "n3_p2_20": ([4, 2], True, 2, None, "DEEPFLOYD", 20),
    "n2_unshift20": ([4], False, 1, None, "DDPM", 20),
}

# reverse steps: (name, pipe, prediction type, ddim_eta, threshold, guidance, t, s)
STEP_GRID = [
    ("ddpm_clip", "plain", _ST, None, "CLIP", 1, 500, 499),
    ("ddim0_clip", "plain", _ST, 0.0, "CLIP", 1, 500, 480),
    ("ddim05_none", "plain", _ST, 0.5, "NONE", 1, 500, 480),
    ("ddim1_dyn_cfg", "plain", _ST, 1.0, "DYNAMIC", 3, 500, 480),
    ("eps_ddpm_dynif", "plain", "DDPM", None, "DYNAMIC_IF", 1, 500, 480),
    ("eps_ddim05_clip_cfg", "plain", "DDPM", 0.5, "CLIP", 3, 300, 250),
    ("final_t1", "plain", _ST, None, "NONE", 1, 1, 0),
    ("final_resampled", "plain", _ST, 1.0, "CLIP", 1, 20, 0),
    ("cos_ddim05", "plain_cos", "DDPM", 0.5, "CLIP", 1, 900, 850),
    ("rs2_ddim05_clip", "plain_rs2", _ST, 0.5, "CLIP", 1, 500, 480),
    ("rs2_eps_ddpm_dyn", "plain_rs2", "DDPM", None, "DYNAMIC", 1, 500, 499),
    ("n2s_ddim05_cfg", "n2_shift", _ST, 0.5, "CLIP", 3, 500, 480),
    ("n2u_ddpm_clip", "n2_unshift", _ST, None, "CLIP", 1, 500, 499),
    ("n2u_eps_ddim1_dyn", "n2_unshift", "DDPM", 1.0, "DYNAMIC", 1, 700, 650),
    ("n3_ddim0_dynif_final", "n3_p2", _ST, 0.0, "DYNAMIC_IF", 1, 1, 0),
    ("n3_ddpm_none_cfg", "n3_p2", _ST, None, "NONE", 3, 40, 0),
]

# sampling loops: (name, pipe, prediction type, ddim_eta, threshold, guidance, resample steps (None: full length))
LOOP_GRID = [
    ("plain_ddim05_4", "plain", _ST, 0.5, "CLIP", 1, 4),
    ("plain_rs2_full_ddpm_dyn", "plain20", "DDPM", None, "DYNAMIC", 3, None),
    ("n2u_ddim1_3_cfg", "n2_unshift", _ST, 1.0, "NONE", 3, 3),
    ("n3_full_ddpm_clip", "n3_p2_20", _ST, None, "CLIP", 1, None),
    ("n2u_full_eps_ddim0", "n2_unshift20", "DDPM", 0.0, "DYNAMIC_IF", 1, None),
]
SAMPLE_B, SAMPLE_SIDE = 2, 8      # plain; nested top level SAMPLE_SIDE * 2


def sample_side(pipe):
    return SAMPLE_SIDE * 2 if PIPES[pipe][0] else SAMPLE_SIDE


def scales_of(nest):
    return (list(nest) + [1]) if nest else [1]


def level_shapes(B, side, nest):
    sc = scales_of(nest)
    return [(B, 3, side * s // sc[0], side * s // sc[0]) for s in sc]


# ---------------------------------------------------------------- configuration dicts (package and reference schema)
def loss_config(case):
    sc = dict(num_diffusion_steps=1000, reproject_signal=False, schedule_type=case["schedule"],
              prediction_type=case["ptype"], loss_target_type=case["ltype"], beta_start=0.0001, beta_end=0.02,
              threshold_function="CLIP", rescale_schedule=1.0, rescale_signal=case.get("rescale_signal", None),
              schedule_shifted=case.get("shifted", False), schedule_shifted_power=case.get("power", 1))
    d = dict(sampler_config=sc, model_output_scale=0, use_vdm_loss_weights=case.get("use_vdm_loss_weights", False))
    if case["nest"]:
        d.update(use_double_loss=case.get("double_loss", True), multi_res_weights=case.get("multi_res_weights"),
                 mixed_ratio=case.get("mixed_ratio"), no_use_residual=True)
    return d


def sampler_config(pipe, ptype, threshold):
    nest, shifted, power, rs, schedule, n = PIPES[pipe]
    case = _loss("", ptype, ptype, schedule, nest, shifted=shifted, power=power, rescale_signal=rs)
    d = loss_config(case)
    d["sampler_config"].update(threshold_function=threshold, num_diffusion_steps=n)
    return d


# ---------------------------------------------------------------- seeded inputs
def images(B, side, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 3, side, side, generator=g) * 2 - 1


def text(B, seed, tokens=4, dim=8):
    g = torch.Generator().manual_seed(seed + 1)
    return torch.randn(B, tokens, dim, generator=g), torch.ones(B, tokens)


def step_inputs(pipe, guidance, seed):
    """x_t per level and the text batch (rows [uncond; cond] under guidance) of a reverse-step case."""
    nest = PIPES[pipe][0]
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(*s, generator=g) * 1.5 for s in level_shapes(SAMPLE_B, sample_side(pipe), nest)]
    lm, mask = text(SAMPLE_B, seed)
    if guidance != 1:
        lm, mask = torch.cat([torch.zeros_like(lm), lm]), torch.cat([mask, mask])
    return xs, lm, mask


def loop_inputs(pipe, guidance, seed):
    """step_inputs with the lower levels of a nest drawn as the reference's first nested step draws them (normal_
    on the CPU generator seeded with `seed`), so a loop started from the full-resolution tensor sees the same values."""
    xs, lm, mask = step_inputs(pipe, guidance, seed)
    torch.manual_seed(seed)
    return [xs[0]] + [torch.empty(x.shape).normal_() for x in xs[1:]], lm, mask


def case_seed(name):
    return 1000 + sum(ord(ch) * (i + 1) for i, ch in enumerate(name)) % 100000


# ---------------------------------------------------------------- fp64 oracle with error magnitudes
def gamma_tables(schedule, n, nest, shifted, power):
    """fp32 tables per level, exactly as the package and the reference build them."""
    base = dref.gammas_f32(schedule, n)
    return [dref.shift_table(base, s, power) if (nest and shifted) else base for s in scales_of(nest)]


def mag_step(x_t, pred, tab, t, s, ptype, threshold, image_scale, eta, need, noise):
    """One reverse step on Mag values (x_t, pred exact fp32 operands unless given as Mag)."""
    clip = False if threshold == "NONE" else threshold
    return dref.reverse_step(Mag.of(x_t), Mag.of(pred), Mag.of(tab[t]), Mag.of(tab[s]), ptype, clip, image_scale, eta,
                             need, noise=noise)


def stochastic(need, eta):
    return bool(need) and not (eta is not None and eta <= 0)


def oracle_step(stub, pipe, ptype, eta, threshold, guidance, t, s, xs, lm, noises):
    """fp64 oracle of get_xt_minus_1 with the stub: per level (x0, x_s) Mags. xs: exact fp32 x_t per level;
    noises: per level, the noise the step drew (or None)."""
    nest, shifted, power, rs, schedule, n = PIPES[pipe]
    tabs = gamma_tables(schedule, n, nest, shifted, power)
    P = mag_params(stub)
    B = xs[0].shape[0]
    times = torch.full((B,), t - 1, dtype=torch.long)
    xm = [Mag.of(x.cpu()) for x in xs]
    lm = lm.cpu()
    if guidance != 1:
        o = StubNet.forward(P, [torch.cat([x, x]) for x in xm], torch.cat([times, times]), lm, None, {})
        o = [a.chunk(2)[0] + guidance * (a.chunk(2)[1] - a.chunk(2)[0]) for a in o]
    else:
        o = StubNet.forward(P, xm, times, lm, None, {})
    out = []
    for l, (x, p, tab, sc) in enumerate(zip(xm, o, tabs, scales_of(nest))):
        need = (t != 1) if nest else (s != 0)
        img_scale = (1.0 if shifted else float(sc)) if nest else (float(rs) if rs else 1.0)
        nz = noises[l].cpu() if noises[l] is not None else None
        out.append(mag_step(x, p, tab, t, s, PT[ptype], threshold, img_scale, eta, need, nz))
    return out


def replay_loss_draws(B, shapes, n_steps, seed, device):
    """The draws of get_loss in the package's order: time, eps at full resolution, then one normal_ per lower level."""
    torch.manual_seed(seed)
    time = torch.randint(0, n_steps, (B,), device=device)
    eps = [torch.randn(*shapes[0], device=device)]
    for s in shapes[1:]:
        eps.append(torch.empty(*s, device=device).normal_())
    return time, eps


def oracle_loss(case, stub, imgs, eps, time, lm, mask):
    """fp64 oracle of get_loss with the stub: (loss Mag, x_t Mags, outs Mags, autograd results)."""
    nest = case["nest"]
    scales = scales_of(nest)
    gam = dref.gammas_f32(case["schedule"], 1000)
    mr = dref.mixed_ratio_fractions(case.get("mixed_ratio"))
    w = [float(v) for v in case["multi_res_weights"].split(":")] if case.get("multi_res_weights") else None
    kw = dict(weights=w, double_loss=case.get("double_loss", True), mixed_ratio=mr,
              rescale_signal=case.get("rescale_signal"))
    args = (scales, PT[case["ptype"]], PT[case["ltype"]], case.get("shifted", False), case.get("power", 1))
    time = time.cpu()
    lm, mask = lm.cpu(), mask.cpu()
    eps = [e.cpu() for e in eps]
    imgs = imgs.cpu()
    lossm, xtm, outm = dref.training_loss(StubNet, mag_params(stub), Mag.of(imgs), [Mag.of(e) for e in eps], time, lm,
                                          mask, Mag.of(gam), *args, **kw)
    P64 = f64_params(stub)
    l64, _, o64 = dref.training_loss(StubNet, P64, imgs.double(), [e.double() for e in eps], time, lm.double(),
                                     mask.double(), gam.double(), *args, **kw)
    wrt = list(o64) + [P64[n] for n in "wbkq"]
    grads = [torch.zeros_like(a) if g is None else g
             for a, g in zip(wrt, torch.autograd.grad(l64.mean(), wrt, allow_unused=True))]
    gout, gpar = grads[:len(o64)], dict(zip("wbkq", grads[len(o64):]))
    # magnitude of d loss / d out = 2 w_l (p - tgt) / (per B) * dp/dv per level, from the level's (p, tgt) Mags
    B, ptype, ltype = imgs.shape[0], args[1], args[2]
    gmags, ps, ts = [], [], []
    for i, (x, o, e) in enumerate(zip(xtm, outm, eps)):
        g = Mag.of(gam)[time + 1]
        if nest and case.get("shifted", False):
            g = dref.shift_table(g, scales[i], args[4])
        xi = dref.nested_pyramid(Mag.of(imgs), [scales[0] // s for s in scales])[i] if nest else Mag.of(imgs)
        if nest and not case.get("shifted", False) and scales[i] != 1:
            xi = xi / float(scales[i])
        _, p, t = dref.level_loss(o, x, xi, Mag.of(e), g, ptype, ltype)
        wl = (w[i] if w else 1.0) if (i == 0 or kw["double_loss"]) else 0.0
        if mr is not None:
            wl /= float(mr[i])
        v = torch.ones(B, 1, 1, 1, dtype=torch.float64, requires_grad=True)
        dpdv = torch.autograd.grad(dref.pred_for_training(torch.zeros_like(v), v, g.v, ptype, ltype).sum(), v)[0]
        per = o.v[0].numel()
        gmags.append(2 * wl * (p.m + t.m) * dpdv.abs() / (per * B))
        ps.append(p)
        ts.append(t)
    return dict(loss=lossm, x_t=xtm, out=outm, p=ps, t=ts, gout=gout, gpar=gpar, P64=P64, gmags=gmags,
                gpar_mag=param_grad_mag(P64, xtm, time, lm, gmags))
