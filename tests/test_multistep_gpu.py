"""DPM-Solver++ multistep sampling (mdm_sampler_multistep, Sampler.sample(..., solver=...)) on the GPU:

  kernel      every step through Sampler._multistep_level against the fp64 oracle (tests/multistep_oracle.py) within
              c * 2^-24 * mag, as tests/test_algebra_gpu.py bounds the other reverse steps; its x0 bit for bit against
              mdm_sampler_step's
  loops       Sampler / NestedSampler.sample with an analytic stand-in denoiser against the fp64 oracle loop, and the
              host test's convergence orders at 64x64 and on a 256/64 nest
  tiny nets   the U-Nets of tests/tiny_configs.py through Diffusion.sample: every recorded step against the oracle step,
              the generator protocol, the final output
"""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

import algebra_cases as ac
import multistep_oracle as mo
import net_cases as nc
import test_rect_oracle as fx
import tiny_configs as tc
from mdm_b200 import config as mc
from mdm_b200 import samplers
from mdm_b200.diffusion import Diffusion, NestedDiffusion
from oracle import diffusion_ref as dref

pytestmark = pytest.mark.gpu
Mag = ac.Mag
THRESHOLDS = ["NONE", "CLIP", "DYNAMIC", "DYNAMIC_IF"]


@pytest.fixture(scope="module")
def worst():
    w = {}
    yield w
    print("\nworst |got - ref| / (u * mag):", {k: round(v, 2) for k, v in sorted(w.items())})


@pytest.fixture
def steps(monkeypatch):
    """Every Sampler._multistep_level call with its inputs, outputs and the noise it drew."""
    log, randn = [], torch.randn_like
    orig = samplers.Sampler._multistep_level
    drawn = []

    def rec_randn(*a, **k):
        r = randn(*a, **k)
        drawn.append(r.clone())
        return r

    def rec(self, x_t, pred, t_idx, s_idx, scale, image_scale, solver, hist):
        n = len(drawn)
        x0, x_s, new = orig(self, x_t, pred, t_idx, s_idx, scale, image_scale, solver, hist)
        log.append(dict(smp=self, x_t=samplers._f32c(x_t).clone(), pred=samplers._f32c(pred).clone(), t=t_idx,
                        s=s_idx, scale=scale, image_scale=image_scale, solver=solver, hist=hist, x0=x0.clone(),
                        x_s=x_s.clone(), noise=drawn[n] if len(drawn) > n else None))
        return x0, x_s, new

    monkeypatch.setattr(torch, "randn_like", rec_randn)
    monkeypatch.setattr(samplers.Sampler, "_multistep_level", rec)
    return log


def oracle_of(r):
    """fp64 (x0, x_s) Mags of one recorded step, with the fp32 coefficients the kernel received as exact operands."""
    smp = r["smp"]
    tab = smp.level_table(r["scale"], "cpu")
    x0_prev, h_prev = r["hist"] if r["hist"] is not None else (None, None)
    coef = samplers.multistep_coefficients(r["solver"], tab, r["t"], r["s"], h_prev)[:4]
    coef = [float(np.float32(c)) for c in coef]
    nz = r["noise"]
    return mo.step(Mag.of(r["x_t"].cpu()), Mag.of(r["pred"].cpu()), Mag.of(tab[r["t"]]),
                   smp._config.prediction_type.value, smp._threshold_name(), r["image_scale"], coef,
                   None if x0_prev is None else Mag.of(x0_prev.cpu()), None if nz is None else Mag.of(nz.cpu()))


def check_record(r, what, worst):
    r0, rs = oracle_of(r)
    ac.assert_bound(r["x0"], r0, ac.C_ELEM, f"x0/{what}", worst)
    ac.assert_bound(r["x_s"], rs, ac.C_ELEM, f"x_s/{what}", worst)


# ---------------------------------------------------------------- kernel level
# (pipe of algebra_cases.PIPES, level scale): plain, rescale_signal 2, nested level of scale 4 shifted / unshifted
TABLES = [("plain", 1), ("plain_rs2", 1), ("n2_shift", 4), ("n2_unshift", 4)]
SIZES = [(1, 3, 17, 23), (3, 3, 40, 24)]
STEPS = [(1000, 960), (960, 920), (40, 0)]  # first (no history), middle (second order), final


def _sampler(pipe, ptype, thr):
    nest = ac.PIPES[pipe][0]
    cfg = mc.diffusion_config_from_dict(ac.sampler_config(pipe, ptype, thr), bool(nest)).sampler_config
    return (samplers.NestedSampler if nest else samplers.Sampler)(cfg).to("cuda")


def _image_scale(pipe, scale):
    nest, shifted, _, rs, _, _ = ac.PIPES[pipe]
    if nest:
        return 1.0 if shifted else float(scale)
    return float(rs) if rs else 1.0


@pytest.mark.parametrize("thr", THRESHOLDS)
@pytest.mark.parametrize("ptype", ["DDPM", "DDIM", "V_PREDICTION"])
def test_kernel_against_oracle(ptype, thr, steps, worst):
    g = torch.Generator().manual_seed(ac.case_seed(ptype + thr))
    for pipe, scale in TABLES:
        smp = _sampler(pipe, ptype, thr)
        isc = _image_scale(pipe, scale)
        for shape in SIZES:
            for solver in mo.SOLVERS:
                hist = None
                for t, s in STEPS:
                    x = (torch.randn(shape, generator=g) * 1.5).cuda()
                    pred = torch.randn(shape, generator=g).cuda()
                    _, _, hist = smp._multistep_level(x, pred, t, s, scale, isc, solver, hist)
    assert len(steps) == len(TABLES) * len(SIZES) * len(mo.SOLVERS) * len(STEPS)
    for r in steps:
        check_record(r, f"{ptype}/{thr}/{r['solver']}/{r['t']}", worst)
        if r["s"] == 0:
            assert torch.equal(r["x_s"], r["x0"])  # the final step returns x0
        if r["s"] != 0 and r["solver"] == "dpmpp_2m_sde":
            assert r["noise"] is not None
    assert sum(r["noise"] is not None for r in steps) == len(TABLES) * len(SIZES) * 2


@pytest.mark.parametrize("thr", THRESHOLDS)
@pytest.mark.parametrize("ptype", ["DDPM", "DDIM", "V_PREDICTION"])
def test_x0_bits_match_sampler_step(ptype, thr):
    g = torch.Generator().manual_seed(3)
    for pipe, scale in TABLES:
        smp = _sampler(pipe, ptype, thr)
        isc = _image_scale(pipe, scale)
        for shape in SIZES:
            x = (torch.randn(shape, generator=g) * 2).cuda()
            pred = torch.randn(shape, generator=g).cuda()
            for t, s in STEPS:
                ref = smp._step_level(x, pred, t, s, scale, False, 0.0, isc)[0]
                got = smp._multistep_level(x, pred, t, s, scale, isc, "dpmpp_2m", (ref, 0.5))[0]
                assert torch.equal(got, ref), (pipe, shape, t)


def test_argument_checks_of_the_entry_point():
    from mdm_b200 import _lib
    import ctypes as C

    x = torch.zeros(2, 8, device="cuda")
    tab = torch.ones(4, device="cuda")
    p = samplers._ptr
    call = _lib.lib().mdm_sampler_multistep
    args = lambda prev, nz, cprev, cn: (p(x), p(x), prev, nz, p(tab), 1, 5, 0, None, C.c_float(1.0), C.c_float(1.0),  # noqa
                                       C.c_float(1.0), C.c_float(cprev), C.c_float(cn), p(x), p(x), 2, C.c_int64(8),
                                       samplers._stream())
    with pytest.raises(_lib.MdmError, match="x0_prev required"):
        _lib.check(call(*args(None, None, 0.5, 0.0)), "mdm_sampler_multistep")
    with pytest.raises(_lib.MdmError, match="noise tensor required"):
        _lib.check(call(*args(None, None, 0.0, 0.5)), "mdm_sampler_multistep")
    _lib.check(call(*args(None, None, 0.0, 0.0)), "mdm_sampler_multistep")


# ---------------------------------------------------------------- loops with an analytic denoiser
class Analytic(nn.Module):
    """Stand-in denoiser: per level, E[x0 | x_t] of x0 ~ N(mu, s^2) as the sampler's prediction, fp32 on the GPU,
    at g = table[times + 1] (the sampler passes t - 1)."""

    def __init__(self, dens, tabs, ptype, nest_ratio=None):
        super().__init__()
        self.p = [(d.mu.float().cuda(), d.s.float().cuda(), tb.cuda()) for d, tb in zip(dens, tabs)]
        self.ptype = ptype
        self.nested = nest_ratio is not None
        self.nest_ratio = list(nest_ratio or [])
        self.is_temporal = [False] * len(self.nest_ratio)
        self.conditions, self.input_channels, self.output_scale, self.fuse_lm_mask = None, 3, 0.0, False

    def forward(self, x_t, times, lm_outputs, lm_mask, micros={}):
        out = []
        for x, (mu, s, tab) in zip(x_t if self.nested else [x_t], self.p):
            g = tab[times + 1].view(-1, 1, 1, 1)
            a, c = g.sqrt(), (1 - g).sqrt()
            x0 = mu + a * s * s * (x - a * mu) / (g * s * s + 1 - g)
            out.append((a * x - x0) / c if self.ptype == dref.V_PREDICTION else (x - a * x0) / c)
        return out if self.nested else out[0]


def _loop_case(nested, ptype_name, side):
    pname = "n2_shift" if nested else "plain"
    nest = ac.PIPES[pname][0]
    cfg = mc.diffusion_config_from_dict(ac.sampler_config(pname, ptype_name, "NONE"), nested)
    scales = ac.scales_of(nest)
    shapes = [(2, 3, side * sc // scales[0], side * sc // scales[0]) for sc in scales]
    dens = [mo.gaussian_case(sh[1:], 10 + i) for i, sh in enumerate(shapes)]
    base = samplers.NestedSampler(cfg.sampler_config) if nested else samplers.Sampler(cfg.sampler_config)
    tabs = [base.level_table(sc, "cpu") for sc in scales]
    model = Analytic(dens, tabs, ac.PT[ptype_name], nest if nested else None)
    pipe = (NestedDiffusion if nested else Diffusion)(model, cfg).to("cuda")
    g = torch.Generator().manual_seed(5)
    x_T = [torch.randn(sh, generator=g) for sh in shapes]
    lm, mask = ac.text(2, 5)
    return pipe, dens, tabs, x_T, lm.cuda(), mask.cuda()


def _run(pipe, x_T, lm, mask, num, **kw):
    """The final x_s per level, unclipped (the last step's yield_full frame)."""
    init = [x.cuda() for x in x_T] if len(x_T) > 1 else x_T[0].cuda()
    frames = list(pipe.sampler.sample(pipe.get_model(), init, lm, mask, {}, num_inference_steps=num,
                                      resample_steps=True, yield_output=True, yield_full=True, **kw))
    return frames


@pytest.mark.parametrize("nested,side", [(False, 64), (True, 256)], ids=["plain64", "nest256_64"])
@pytest.mark.parametrize("ptype", ["DDPM", "V_PREDICTION"])
def test_loop_matches_oracle_and_converges(nested, side, ptype, steps):
    pipe, dens, tabs, x_T, lm, mask = _loop_case(nested, ptype, side)
    pt = ac.PT[ptype]
    for solver in mo.SOLVERS:
        steps.clear()
        torch.manual_seed(1)
        frames = _run(pipe, x_T, lm, mask, 20, solver=solver)
        assert len(frames) == 21
        nlev = len(x_T)
        # every level's loop against the fp64 oracle loop on the same noise. The bound covers the fp32 stand-in: an eps
        # prediction at the first step (alpha ~ 5e-5) turns its rounding into ~4e-3 of x0, weighted by alpha_s in x_s
        for lv in range(nlev):
            noises = [r["noise"].cpu() if r["noise"] is not None else None for r in steps[lv::nlev]]
            ref = mo.sample_loop(dens[lv], x_T[lv], tabs[lv], dref.set_timesteps(1000, 20), solver, pt, noises=noises)
            got = steps[-nlev + lv]["x_s"]
            assert float((got.cpu().double() - ref).abs().max()) <= (1e-4 if pt == dref.V_PREDICTION else 2e-3), \
                (solver, lv)
    # orders at 200 -> 400 steps against the exact endpoint of every level (host test: DDIM ~1.9x, 2M >= 2.2x)
    err = {}
    for num in (200, 400):
        ts = dref.set_timesteps(1000, num)
        steps.clear()
        _run(pipe, x_T, lm, mask, num, solver="dpmpp_2m")
        for lv in range(nlev):
            exact = mo.exact_endpoint(dens[lv], x_T[lv].double(), tabs[lv], ts)
            err[("dpmpp_2m", num, lv)] = mo.rms(steps[-nlev + lv]["x_s"].cpu().double(), exact)
            err[("ddim", num, lv)] = mo.rms(_final_ddim(pipe, x_T, lm, mask, ts)[lv], exact)
    for lv in range(nlev):
        r_ddim = err[("ddim", 200, lv)] / err[("ddim", 400, lv)]
        r_2m = err[("dpmpp_2m", 200, lv)] / err[("dpmpp_2m", 400, lv)]
        assert 1.7 <= r_ddim <= 2.1 and r_2m >= 2.2 and r_2m >= 1.2 * r_ddim, (lv, r_ddim, r_2m)


def _final_ddim(pipe, x_T, lm, mask, ts):
    """The DDIM (eta 0) loop's final x_s per level, unclipped."""
    x = [v.cuda() for v in x_T] if len(x_T) > 1 else x_T[0].cuda()
    with torch.no_grad():
        for i, t in enumerate(ts[:-1]):
            x = pipe.sampler.get_xt_minus_1(pipe.get_model(), int(t), x, lm, mask, {}, time_step_last=int(ts[i + 1]),
                                            ddim_eta=0.0)
    return [v.cpu().double() for v in (x if len(x_T) > 1 else [x])]


# ---------------------------------------------------------------- tiny nets
TINY = [("unet", None, 1, "CLIP", "dpmpp_2m"), ("unet", (24, 40), 5, "DYNAMIC", "dpmpp_2m_sde"),
        ("nested", None, 5, "CLIP", "dpmpp_2m_sde"), ("nested", fx.NEST_HW, 1, "DYNAMIC", "dpmpp_2m"),
        ("nested", fx.NEST_HW[::-1], 5, "DYNAMIC_IF", "dpmpp_2m")]


@pytest.mark.parametrize("kind,hw,gs,thr,solver", TINY, ids=lambda v: str(v))
def test_tiny_nets(kind, hw, gs, thr, solver, steps, worst):
    nested = kind == "nested"
    model = nc.build(kind)[0]
    dcfg = copy.deepcopy(tc.TINY_NESTED_DIFFUSION if nested else tc.TINY_DIFFUSION)
    dcfg["sampler_config"]["threshold_function"] = thr
    pipe = (NestedDiffusion if nested else Diffusion)(model, mc.diffusion_config_from_dict(dcfg, nested)).to("cuda")
    B, num = 2, 6
    _, _, lm, mask = tc.seeded_inputs(4, B, 8, 6)
    if gs != 1:
        lm, mask = torch.cat([torch.zeros_like(lm), lm]), torch.cat([mask, mask])
    lm, mask = lm.cuda(), mask.cuda()
    kw = dict(num_inference_steps=num, resample_steps=True, guidance_scale=gs, solver=solver)
    side = 32 if nested else 16
    torch.manual_seed(9)
    if hw is None:
        out = pipe.sample(B, {"lm_outputs": lm, "lm_mask": mask}, side, "cuda", **kw)
        hw = (side, side)
    else:
        out = pipe.sampler.sample(pipe.get_model(), torch.randn(B, 3, *hw).cuda(), lm, mask, {}, **kw)
    nlev = 2 if nested else 1
    assert out.shape == (B, 3) + tuple(hw)
    assert len(steps) == num * nlev
    for i, r in enumerate(steps):
        check_record(r, f"tiny/{kind}/{thr}/{solver}/{i}", worst)
        assert (r["hist"] is None) == (i < nlev)
    assert torch.equal(out, steps[-nlev]["x0"].clamp(-1, 1))  # final output: the clipped x0 of the last step
    # generator protocol: per step (x0, x_s, extra) of level 0, then the clipped final frame
    steps.clear()
    torch.manual_seed(9)
    init = torch.randn(B, 3, *hw).cuda()
    frames = list(pipe.sampler.sample(pipe.get_model(), init, lm, mask, {}, yield_output=True, yield_full=True, **kw))
    assert len(frames) == num + 1
    for f, r in zip(frames[:-1], steps[::nlev]):
        assert torch.equal(f[0], r["x0"]) and torch.equal(f[1], r["x_s"]) and len(f[2]) == 2
    assert torch.equal(frames[-1][1], frames[-2][1].clamp(-1, 1))
    if nested:
        steps.clear()
        torch.manual_seed(9)
        inner = list(pipe.sampler.sample(pipe.get_model(), init, lm, mask, {}, yield_output=True, output_inner=True,
                                         **kw))[-1]
        assert inner.shape == (B, 3, hw[0], hw[1] * 2)
