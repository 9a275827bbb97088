"""DPM-Solver++ multistep sampling on the host: the fp64 oracle (tests/multistep_oracle.py) against the DDIM step it
generalises, its convergence on analytic denoisers, the package's coefficients against the oracle's, and the argument
checks of Sampler.sample(..., solver=...).

Endpoints. The loops run over the package's own time steps (set_timesteps: uniform in t, so in lambda = log(alpha /
sigma) the first and last steps stay long at any step count). Their last step returns x0 = E[x0 | x_{t_1}] at the
last non-zero step t_1 for every solver; the reference endpoint is the exact probability-flow solution at t_1 pushed
through that same step (multistep_oracle.exact_endpoint), so the error measured is the solver's.
"""
import math

import pytest
import torch

import algebra_cases as ac
import multistep_oracle as mo
from mdm_b200 import config as mc
from mdm_b200 import samplers
from oracle import diffusion_ref as dref

SHAPE = (1, 3, 8, 8)


def _denoisers():
    g = torch.Generator().manual_seed(1)

    def u(lo, hi):
        return lo + (hi - lo) * torch.rand(SHAPE, generator=g)

    return {"gaussian": mo.Gaussian(u(-0.5, 0.5), u(0.3, 0.5)),
            "mixture": mo.Mixture(0.4, u(-0.6, -0.4), u(0.15, 0.25), u(0.3, 0.5), u(0.15, 0.25))}


DEN = _denoisers()
X_T = torch.randn(SHAPE, generator=torch.Generator().manual_seed(2)).double()


def _errors(den, schedule, ptype, num):
    tab = mo.table(schedule)
    ts = dref.set_timesteps(1000, num)
    exact = mo.exact_endpoint(den, X_T, tab, ts)
    return {s: mo.rms(mo.sample_loop(den, X_T, tab, ts, s, ptype), exact) for s in ("ddim", "dpmpp_2m")}


@pytest.mark.parametrize("schedule", ["DEEPFLOYD", "COSINE", "DDPM"])
@pytest.mark.parametrize("ptype", [dref.DDPM, dref.V_PREDICTION])
@pytest.mark.parametrize("threshold", ["NONE", "CLIP", "DYNAMIC_IF"])
def test_first_order_step_is_ddim_eta0(schedule, ptype, threshold):
    tab = mo.table(schedule)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 3, 5, 7, generator=g).double() * 1.5
    pred = torch.randn(2, 3, 5, 7, generator=g).double()
    for t, s in ((1000, 950), (500, 480), (40, 1), (1, 0), (300, 0)):
        gt, gs = torch.tensor(float(tab[t]), dtype=torch.float64), torch.tensor(float(tab[s]), dtype=torch.float64)
        A, B, Cc, S, _ = mo.coefficients("dpmpp_2m", tab[t], tab[s], s, None)
        x0, xs = mo.step(x, pred, gt, ptype, threshold, 2.0, (A, B, Cc, S))
        r0, rs = mo.ddim_step(x, pred, gt, gs, ptype, threshold, 2.0)
        assert torch.equal(x0, r0)
        torch.testing.assert_close(xs, rs, rtol=1e-12, atol=1e-12)


def test_fine_flow_matches_the_gaussian_flow():
    den = DEN["gaussian"]
    tab = mo.table("DEEPFLOYD")
    g_T, g_1 = float(tab[1000]), float(tab[20])
    assert float((mo.fine_flow(den, X_T, g_T, g_1) - den.flow(X_T, g_T, g_1)).abs().max()) < 1e-5


@pytest.mark.parametrize("den", sorted(DEN))
@pytest.mark.parametrize("schedule", ["DEEPFLOYD", "COSINE"])
def test_convergence_order(den, schedule):
    """Halving the step size from 200 to 400 steps: DDIM's error falls by 1.85-1.91x (first order), 2M's by
    2.32-3.93x (measured). 2M is second order in lambda (3.94x on a uniform lambda grid); with the time steps uniform in
    t it only approaches that in this range. Margins: DDIM 1.7-2.1x, 2M at least 2.2x and 1.2x DDIM's."""
    e200 = _errors(DEN[den], schedule, dref.V_PREDICTION, 200)
    e400 = _errors(DEN[den], schedule, dref.V_PREDICTION, 400)
    r_ddim, r_2m = e200["ddim"] / e400["ddim"], e200["dpmpp_2m"] / e400["dpmpp_2m"]
    assert 1.7 <= r_ddim <= 2.1, r_ddim
    assert r_2m >= 2.2 and r_2m >= 1.2 * r_ddim, (r_2m, r_ddim)


@pytest.mark.parametrize("den", sorted(DEN))
@pytest.mark.parametrize("schedule", ["DEEPFLOYD", "COSINE"])
@pytest.mark.parametrize("ptype", [dref.DDPM, dref.V_PREDICTION])
def test_2m_beats_ddim_at_20_steps(den, schedule, ptype):
    """At 20 steps 2M's endpoint is 2.8-11.7x closer than DDIM's (measured; 10-82x at 400 steps). Margin: 2.5x."""
    e = _errors(DEN[den], schedule, ptype, 20)
    assert e["dpmpp_2m"] * 2.5 <= e["ddim"], e


@pytest.mark.parametrize("solver", mo.SOLVERS)
@pytest.mark.parametrize("schedule,shift", [("DEEPFLOYD", 1), ("COSINE", 1), ("DEEPFLOYD", 4)])
def test_package_coefficients_match_oracle(solver, schedule, shift):
    tab = dref.shift_table(dref.gammas_f32(schedule, 1000), shift)
    ts = dref.set_timesteps(1000, 25)
    h_prev = h_ref = None
    for i, t in enumerate(ts[:-1]):
        s = int(ts[i + 1])
        *got, h_prev = samplers.multistep_coefficients(solver, tab, int(t), s, h_prev)
        *ref, h_ref = mo.coefficients(solver, tab[int(t)], tab[s], s, h_ref)
        for a, b in zip(got, ref):
            assert math.isclose(a, b, rel_tol=1e-12, abs_tol=1e-15), (t, s, got, ref)
    assert got == [0.0, 1.0, 0.0, 0.0]


def _sampler():
    cfg = ac.loss_config(ac._loss("", "V_PREDICTION", "V_PREDICTION"))
    return samplers.Sampler(mc.diffusion_config_from_dict(cfg, False).sampler_config)


@pytest.mark.parametrize("kw,msg", [(dict(solver="unipc"), "unknown solver"),
                                    (dict(solver="dpmpp_2m", ddim_eta=0.0), "ddim_eta"),
                                    (dict(solver="dpmpp_2m_sde", ddim_eta=1.0), "ddim_eta")])
def test_solver_argument_checks(kw, msg):
    smp = _sampler()
    x = torch.zeros(1, 3, 4, 4)
    with pytest.raises(ValueError, match=msg):
        smp.sample(None, x, None, None, {}, **kw)
    with pytest.raises(ValueError, match=msg):  # the generator form raises on its first step
        next(smp.sample(None, x, None, None, {}, yield_output=True, **kw))
