"""The oracle's diffusion algebra (oracle/diffusion_ref.py) with the stub denoiser against the reference's own outputs
(tests/golden/algebra.npz, tests/golden/make_golden_algebra.py) at every point of the option grids of
tests/algebra_cases.py, and the sensitivity of the GPU tests' bound: on the same inputs, the fp64 oracle with one
deliberate change (a gamma index off by one, the loss type swapped, eta ignored, a level weight dropped, image_div
ignored) must violate the bound that tests/test_algebra_gpu.py holds the kernels to."""
import os

import numpy as np
import pytest
import torch

import algebra_cases as ac
from oracle import diffusion_ref as dref

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "algebra.npz"))
Mag = ac.Mag
CASES = {c["name"]: c for c in ac.LOSS_GRID}


def close(got, key, tol=1e-6):
    ref = torch.from_numpy(GOLD[key]).double()
    got = got.detach().double()
    assert got.shape == ref.shape, key
    err = float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
    assert err <= tol, (key, err)


def loss_inputs(case):
    seed, nest = ac.case_seed(case["name"]), case["nest"]
    B, side = case.get("B", ac.LOSS_B), ac.loss_side(case)
    p = f"loss/{case['name']}/"
    eps = [torch.from_numpy(GOLD[p + f"eps{i}"]) for i in range(len(ac.scales_of(nest)))]
    lm, mask = ac.text(B, seed)
    stub = ac.NestedStub(nest, seed) if nest else ac.Stub(seed)
    return stub, ac.images(B, side, seed), eps, torch.from_numpy(GOLD[p + "time"]), lm, mask


def fp32_loss(case, stub, imgs, eps, time, lm, mask, **over):
    P = {n: getattr(stub, n).detach().clone().requires_grad_(True) for n in "wbkq"}
    o = dict(ptype=ac.PT[case["ptype"]], ltype=ac.PT[case["ltype"]], shifted=case.get("shifted", False),
             power=case.get("power", 1), gam=dref.gammas_f32(case["schedule"], 1000))
    mr = dref.mixed_ratio_fractions(case.get("mixed_ratio"))
    w = [float(v) for v in case["multi_res_weights"].split(":")] if case.get("multi_res_weights") else None
    loss, x_t, outs = dref.training_loss(ac.StubNet, P, imgs, eps, time, lm, mask, o["gam"], ac.scales_of(case["nest"]),
                                         o["ptype"], o["ltype"], o["shifted"], o["power"], weights=w,
                                         double_loss=case.get("double_loss", True), mixed_ratio=mr,
                                         rescale_signal=case.get("rescale_signal"))
    return P, loss, x_t, outs, o


@pytest.mark.parametrize("name", list(CASES))
def test_loss_matches_reference(name):
    case = CASES[name]
    stub, imgs, eps, time, lm, mask = loss_inputs(case)
    P, loss, x_t, outs, o = fp32_loss(case, stub, imgs, eps, time, lm, mask)
    p = f"loss/{name}/"
    assert torch.equal(x_t[0], torch.from_numpy(GOLD[p + "x_t"]))  # the same fp32 ops in the same order
    close(loss, p + "loss")
    g = o["gam"][time + 1]
    if case["nest"] and o["shifted"]:
        g = dref.shift_table(g, ac.scales_of(case["nest"])[0], o["power"])
    div = 1.0 if (not case["nest"] or o["shifted"]) else float(case["nest"][0])
    _, pred, tgt = dref.level_loss(outs[0], x_t[0], imgs / div if div != 1.0 else imgs, eps[0], g, o["ptype"], o["ltype"])
    close(tgt, p + "tgt")
    close(pred if case["nest"] else outs[0], p + "pred")
    if case.get("use_vdm_loss_weights"):
        assert torch.equal(dref.vdm_weights(o["gam"])[time + 1], torch.from_numpy(GOLD[p + "weights"]))
    loss.mean().backward()
    for k in "wbkq":
        close(P[k].grad, p + "grad_" + k, 1e-5)


@pytest.mark.parametrize("case", ac.STEP_GRID, ids=lambda c: c[0])
def test_reverse_step_matches_reference(case):
    name, pname, ptype, eta, thr, gs, t, s = case
    seed, nest = ac.case_seed(name), ac.PIPES[pname][0]
    stub = ac.NestedStub(nest, seed) if nest else ac.Stub(seed)
    xs, lm, mask = ac.step_inputs(pname, gs, seed)
    p = f"step/{name}/"
    noises = [torch.from_numpy(GOLD[p + f"noise{i}"]) if p + f"noise{i}" in GOLD else None for i in range(len(xs))]
    for i, (r0, rs) in enumerate(ac.oracle_step(stub, pname, ptype, eta, thr, gs, t, s, xs, lm, noises)):
        close(r0.v, p + f"x0_{i}", 4e-6)  # the fp64 oracle against the reference's fp32 step
        close(rs.v, p + f"xs_{i}", 4e-6)


@pytest.mark.parametrize("thr", ["NONE", "CLIP", "DYNAMIC", "DYNAMIC_IF"])
def test_clip_sample_matches_reference(thr):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(3, 3, 8, 8, generator=g) * torch.tensor([0.4, 1.3, 9.0]).view(3, 1, 1, 1)
    for sc in (1, 2, 4):
        assert torch.equal(dref.clip_sample(x, sc, False if thr == "NONE" else thr), torch.from_numpy(GOLD[f"clip/{thr}_{sc}"]))


@pytest.mark.parametrize("case", ac.LOOP_GRID, ids=lambda c: c[0])
def test_sample_loop_matches_reference(case):
    name, pname, ptype, eta, thr, gs, steps = case
    seed, (nest, shifted, power, rs, schedule, n) = ac.case_seed(name), ac.PIPES[pname]
    stub = ac.NestedStub(nest, seed) if nest else ac.Stub(seed)
    xs, lm, mask = ac.loop_inputs(pname, gs, seed)
    flat = torch.from_numpy(GOLD[f"loop/{name}/noise"]) if f"loop/{name}/noise" in GOLD else torch.zeros(0)
    nsteps = steps if steps is not None else n
    ts = dref.set_timesteps(n, nsteps)
    noises, k = [], 0
    for i, t in enumerate(ts[:-1]):
        need = (int(t) != 1) if nest else (int(ts[i + 1]) != 0)
        lv = []
        for x in xs:
            if ac.stochastic(need, eta):
                lv.append(flat[k:k + x.numel()].view(x.shape))
                k += x.numel()
            else:
                lv.append(None)
        noises.append(lv)
    assert k == flat.numel()
    P = {n_: getattr(stub, n_).detach() for n_ in "wbkq"}
    final = dref.sample_loop(ac.StubNet, P, xs, lm, mask, dref.gammas_f32(schedule, n), ac.scales_of(nest),
                             ac.PT[ptype], n, nsteps, eta, clip=False if thr == "NONE" else thr, shifted=shifted,
                             power=power, guidance_scale=gs, rescale_signal=rs, noises=noises)
    close(final[0], f"loop/{name}/final", 1e-5)


# ---------------------------------------------------------------- sensitivity of the GPU bounds
def _violates(bug, ref, c):
    return ac.excess(bug if isinstance(bug, torch.Tensor) else bug.v, ref, c) > 1.0


def _loss_bug(case, **change):
    """fp64 per-sample loss of level 0 with one change, against the correct one and the GPU test's loss bound."""
    stub, imgs, eps, time, lm, mask = loss_inputs(case)
    o = ac.oracle_loss(case, stub, imgs, eps, time, lm, mask)
    x_t, out = o["x_t"][0], o["out"][0]
    nest = case["nest"]
    gam = dref.gammas_f32(case["schedule"], 1000).double()
    sc = ac.scales_of(nest)
    shifted = case.get("shifted", False)
    g = gam[time + 1 + change.get("dt", 0)]
    if nest and shifted:
        g = dref.shift_table(g, sc[0], case.get("power", 1))
    div = 1.0 if (not nest or shifted or change.get("no_div")) else float(sc[0])
    lt = ac.PT[change.get("ltype", case["ltype"])]
    bug, _, _ = dref.level_loss(out.v, x_t.v, imgs.double() / div, eps[0].double(), g, ac.PT[case["ptype"]], lt)
    return bug, o


@pytest.mark.parametrize("name,change", [
    ("V_PREDICTION_DDPM", dict(dt=1)), ("V_PREDICTION_DDPM", dict(dt=-1)), ("DDPM_V_PREDICTION", dict(dt=1)),
    ("V_PREDICTION_DDPM", dict(ltype="V_PREDICTION")), ("DDPM_V_PREDICTION", dict(ltype="DDPM")),
    ("n2_unshift_DDPM_V", dict(no_div=True)),
])
def test_loss_bound_catches(name, change):
    case = CASES[name]
    bug, o = _loss_bug(case, **change)
    per = o["x_t"][0].v[0].numel()
    if len(o["out"]) == 1:
        assert _violates(bug, o["loss"], ac.loss_c(per) + 1)
    else:  # level 0 alone: the other levels' terms are unchanged
        ref0, _ = _loss_bug(case)
        assert float((bug - ref0).abs().max()) > (ac.loss_c(per) + 3) * ac.U * float(o["loss"].m.max())


@pytest.mark.parametrize("name", ["n3_p2_weights", "n3_mixed_weights"])
def test_loss_bound_catches_dropped_level_weight(name):
    case = dict(CASES[name], multi_res_weights=None)
    stub, imgs, eps, time, lm, mask = loss_inputs(CASES[name])
    good = ac.oracle_loss(CASES[name], stub, imgs, eps, time, lm, mask)["loss"]
    bug = ac.oracle_loss(case, stub, imgs, eps, time, lm, mask)["loss"]
    assert _violates(bug.v, good, ac.loss_c(imgs[0].numel()) + 3)


@pytest.mark.parametrize("case", [c for c in ac.STEP_GRID if c[0] in ("ddpm_clip", "ddim05_none", "ddim1_dyn_cfg",
                                                                      "eps_ddim05_clip_cfg", "n2u_ddpm_clip",
                                                                      "rs2_ddim05_clip")], ids=lambda c: c[0])
def test_step_bound_catches(case):
    name, pname, ptype, eta, thr, gs, t, s = case
    seed, nest = ac.case_seed(name), ac.PIPES[pname][0]
    stub = ac.NestedStub(nest, seed) if nest else ac.Stub(seed)
    xs, lm, mask = ac.step_inputs(pname, gs, seed)
    g = torch.Generator().manual_seed(seed)
    noises = [torch.randn(x.shape, generator=g) for x in xs]
    good = ac.oracle_step(stub, pname, ptype, eta, thr, gs, t, s, xs, lm, noises)
    bugs = [ac.oracle_step(stub, pname, ptype, eta, thr, gs, t + 1, s, xs, lm, noises),   # gamma index of t
            ac.oracle_step(stub, pname, ptype, eta, thr, gs, t, s + 1, xs, lm, noises)]   # gamma index of g_last
    if eta is not None and eta > 0:
        bugs.append(ac.oracle_step(stub, pname, ptype, 0.0, thr, gs, t, s, xs, lm, noises))  # eta ignored
    if PIPESCALE(pname) != 1.0:  # image scale of the clip ignored
        pipes = dict(ac.PIPES)
        ac.PIPES[pname + "_noscale"] = (pipes[pname][0], True if pipes[pname][0] else False, 1, None) + pipes[pname][4:]
        try:
            bugs.append(ac.oracle_step(stub, pname + "_noscale", ptype, eta, thr, gs, t, s, xs, lm, noises))
        finally:
            del ac.PIPES[pname + "_noscale"]
    for bug in bugs:
        assert any(_violates(b[1].v, r[1], ac.C_ELEM) or _violates(b[0].v, r[0], ac.C_ELEM) for b, r in zip(bug, good))


def PIPESCALE(pname):
    nest, shifted, power, rs = ac.PIPES[pname][:4]
    return (1.0 if shifted else float(nest[0])) if nest else (float(rs) if rs else 1.0)
