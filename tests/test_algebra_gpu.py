"""The diffusion algebra of csrc/diffusion.cu on the GPU against the fp64 oracle, with a stub denoiser in place of the
U-Net (tests/algebra_cases.py), so that each result is held to c * 2^-24 * mag, its fp32 forward error bound:

  pipeline level   get_loss (loss, x_t, pred, target, VDM weights, d loss / d model output, stub-parameter gradients),
                   get_xt_minus_1 (x0, x_s), clip_sample and sample (final / yield_output / output_inner) for every
                   point of the option grids, fed the package's own draws; one point per pipeline against the
                   reference's fixture tests/golden/algebra.npz
  kernel level     q-sample (fp32 and uint8), the loss forward / backward, the reverse step, CFG, avg_pool, clip /
                   scale through the package's entry points at the sizes where the kernels can go wrong: B = 1, odd
                   per-sample sizes, grid-stride wrap-around, the loss's 64-chunk cap, both ends of the gamma tables,
                   the pointer offsets of the mixed-ratio split
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import algebra_cases as ac
from mdm_b200 import config as mc
from mdm_b200 import samplers
from mdm_b200.diffusion import Diffusion, NestedDiffusion, _LossFn
from oracle import diffusion_ref as dref

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
Mag = ac.Mag


@pytest.fixture(scope="module")
def worst():
    """Largest |got - ref| / (u mag) per quantity over the module (printed at the end; pytest -s shows it)."""
    w = {}
    yield w
    print("\nworst |got - ref| / (u * mag):", {k: round(v, 2) for k, v in sorted(w.items())})


@pytest.fixture
def noise_log(monkeypatch):
    """Every torch.randn_like draw (the reverse step's noise), in order."""
    log, orig = [], torch.randn_like

    def rec(*a, **k):
        r = orig(*a, **k)
        log.append(r.clone())
        return r

    monkeypatch.setattr(torch, "randn_like", rec)
    return log


def make_pipe(nest, cfg, seed):
    stub = (ac.NestedStub(nest, seed) if nest else ac.Stub(seed)).cuda()
    dcfg = mc.diffusion_config_from_dict(cfg, bool(nest))
    return stub, (NestedDiffusion if nest else Diffusion)(stub, dcfg).to("cuda")


def check(got, ref, c, what, worst):
    ac.assert_bound(got, ref, c, what, worst)


# ---------------------------------------------------------------- pipeline level
def run_loss(case):
    seed = ac.case_seed(case["name"])
    nest, B, side = case["nest"], case.get("B", ac.LOSS_B), ac.loss_side(case)
    stub, pipe = make_pipe(nest, ac.loss_config(case), seed)
    imgs = ac.images(B, side, seed)
    lm, mask = ac.text(B, seed)
    pipe.train()
    torch.manual_seed(seed)
    loss, time, x_t, pred, tgt, w = pipe.get_loss({"images": imgs.cuda(), "lm_outputs": lm.cuda(), "lm_mask": mask.cuda()})
    loss.mean().backward()
    time_r, eps = ac.replay_loss_draws(B, ac.level_shapes(B, side, nest), 1000, seed, "cuda")
    assert torch.equal(time_r, time)
    return stub, imgs, eps, time, lm, mask, (loss, x_t, pred, tgt, w)


@pytest.mark.parametrize("case", ac.LOSS_GRID, ids=lambda c: c["name"])
def test_get_loss(case, worst):
    stub, imgs, eps, time, lm, mask, (loss, x_t, pred, tgt, w) = run_loss(case)
    o = ac.oracle_loss(case, stub, imgs, eps, time, lm, mask)
    B = imgs.shape[0]
    per = x_t[0].numel()
    check(x_t, o["x_t"][0], ac.C_XT, "x_t", worst)
    check(loss, o["loss"], ac.loss_c(per) + len(o["out"]), "loss", worst)
    check(tgt, o["t"][0], ac.C_ELEM, "target", worst)
    check(pred, o["p"][0] if case["nest"] else o["out"][0], ac.C_ELEM, "pred", worst)
    if case.get("use_vdm_loss_weights"):
        assert torch.equal(w.cpu(), dref.vdm_weights(dref.gammas_f32(case["schedule"], 1000))[time.cpu() + 1])
    else:
        assert w is None
    for l, out in enumerate(stub.outputs):
        n = out.shape[0]
        check(out.grad, Mag(o["gout"][l][:n], o["gmags"][l][:n]), ac.C_GRAD, f"d_model_out/level{l}", worst)
    for k in "wbkq":
        check(getattr(stub, k).grad, Mag(o["gpar"][k], o["gpar_mag"][k]), ac.C_PARAM, f"param_grad/{k}", worst)


@pytest.mark.parametrize("case", ac.STEP_GRID, ids=lambda c: c[0])
def test_reverse_step(case, worst, noise_log):
    name, pname, ptype, eta, thr, gs, t, s = case
    seed = ac.case_seed(name)
    nest = ac.PIPES[pname][0]
    stub, pipe = make_pipe(nest, ac.sampler_config(pname, ptype, thr), seed)
    pipe.eval()
    xs, lm, mask = ac.step_inputs(pname, gs, seed)
    xin = [x.cuda() for x in xs] if nest else xs[0].cuda()
    with torch.no_grad():
        x0, x_s, _ = pipe.sampler.get_xt_minus_1(pipe.get_model(), t, xin, lm.cuda(), mask.cuda(), {}, time_step_last=s,
                                                 guidance_scale=gs, ddim_eta=eta, return_details=True)
    x0, x_s = (x0, x_s) if nest else ([x0], [x_s])
    need = (t != 1) if nest else (s != 0)
    noises = list(noise_log) if ac.stochastic(need, eta) else [None] * len(xs)
    assert len(noises) == len(xs)
    ref = ac.oracle_step(stub, pname, ptype, eta, thr, gs, t, s, xs, lm, noises)
    for l, ((r0, rs), a, b) in enumerate(zip(ref, x0, x_s)):
        check(a, r0, ac.C_ELEM, f"step_x0/{name}/{l}", worst)
        check(b, rs, ac.C_ELEM, f"step_xs/{name}/{l}", worst)


@pytest.mark.parametrize("thr", ["NONE", "CLIP", "DYNAMIC", "DYNAMIC_IF"])
def test_clip_sample(thr, worst):
    stub, pipe = make_pipe(None, ac.sampler_config("plain", "V_PREDICTION", thr), 5)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(3, 3, 17, 23, generator=g) * torch.tensor([0.4, 1.3, 9.0]).view(3, 1, 1, 1)
    for scale in (1.0, 2.0, 4.0):
        got = pipe.sampler.clip_sample(x.cuda(), scale)
        ref = dref.clip_sample(Mag.of(x), scale, False if thr == "NONE" else thr)
        check(got, ref, ac.C_ELEM, "clip_sample", worst)


def _loop_oracle(stub, pname, ptype, eta, thr, gs, steps, init, lm, noise_log):
    nest, shifted, power, rs, schedule, n = ac.PIPES[pname]
    scales = ac.scales_of(nest)
    nsteps = steps if steps is not None else n
    ts = dref.set_timesteps(n, nsteps)
    noises, k = [], 0
    for i, t in enumerate(ts[:-1]):
        need = (int(t) != 1) if nest else (int(ts[i + 1]) != 0)
        if ac.stochastic(need, eta):
            noises.append([z.cpu() for z in noise_log[k:k + len(scales)]])
            k += len(scales)
        else:
            noises.append([None] * len(scales))
    assert k == len(noise_log)
    tabs = [Mag.of(tb) for tb in ac.gamma_tables(schedule, n, nest, shifted, power)]
    lm2 = lm.cpu()
    trace = []
    final = dref.sample_loop(ac.StubNet, ac.mag_params(stub), [Mag.of(x.cpu()) for x in init], lm2, None, None,
                             scales, ac.PT[ptype], n, nsteps, eta, clip=False if thr == "NONE" else thr, shifted=shifted,
                             guidance_scale=gs, rescale_signal=rs, noises=noises, tabs=tabs, trace=trace)
    return final, trace, len(ts) - 1


@pytest.mark.parametrize("case", ac.LOOP_GRID, ids=lambda c: c[0])
def test_sample_loop(case, worst, noise_log):
    name, pname, ptype, eta, thr, gs, steps = case
    seed = ac.case_seed(name)
    nest = ac.PIPES[pname][0]
    stub, pipe = make_pipe(nest, ac.sampler_config(pname, ptype, thr), seed)
    xs, lm, mask = ac.loop_inputs(pname, gs, seed)
    init = [x.cuda() for x in xs] if nest else xs[0].cuda()
    kw = dict(num_inference_steps=steps or 0, ddim_eta=eta, guidance_scale=gs, resample_steps=steps is not None)
    torch.manual_seed(seed)  # each of the three runs below draws the same noise
    out = pipe.sampler.sample(pipe.get_model(), init, lm.cuda(), mask.cuda(), {}, **kw)
    draws = list(noise_log)
    final, trace, nst = _loop_oracle(stub, pname, ptype, eta, thr, gs, steps, xs, lm, draws)
    c = ac.C_STEP_LOOP * nst
    check(out, final[0], c, f"sample/{name}", worst)
    # the generator forms: per step (x0, x_t) of level 0 scaled for display, the last frame clipped
    noise_log.clear()
    torch.manual_seed(seed)
    frames = list(pipe.sampler.sample(pipe.get_model(), init, lm.cuda(), mask.cuda(), {}, yield_output=True,
                                      yield_full=True, **kw))
    assert len(frames) == nst + 1
    nest_, shifted, power, rs, _, _ = ac.PIPES[pname]
    sc = (1.0 if shifted else float(ac.scales_of(nest)[0])) if nest else (float(rs) if rs else 1.0)
    for i, (f, (r0, rs_)) in enumerate(zip(frames[:-1], trace)):
        check(f[1], rs_[0] * sc, c, f"sample_yield/{name}", worst)
        check(f[0], r0[0] * sc, c, f"sample_yield_x0/{name}", worst)
    check(frames[-1][1], final[0], c, f"sample_yield/{name}", worst)
    if nest:
        noise_log.clear()
        torch.manual_seed(seed)
        inner = list(pipe.sampler.sample(pipe.get_model(), init, lm.cuda(), mask.cuda(), {}, yield_output=True,
                                         output_inner=True, **kw))[-1]
        H, W = out.shape[-2:]
        assert inner.shape == (out.shape[0], 3, H, W * len(xs))
        check(inner[..., -W:], final[0], c, f"sample_inner/{name}", worst)


@pytest.mark.parametrize("name", ["rescale2_DDPM_V", "n3_mixed_weights"])
def test_get_loss_matches_reference_fixture(name, monkeypatch):
    """One loss point per pipeline end to end against the reference's own outputs (algebra.npz), on its draws:
    get_eps_time returns the fixture's time and full-resolution noise, normal_ fills the lower levels from it."""
    gold = np.load(os.path.join(GOLD, "algebra.npz"))
    case = next(c for c in ac.LOSS_GRID if c["name"] == name)
    p = f"loss/{name}/"
    nlev = len(ac.scales_of(case["nest"]))
    eps = [torch.from_numpy(gold[p + f"eps{i}"]).cuda() for i in range(nlev)]
    time = torch.from_numpy(gold[p + "time"]).cuda()
    seed = ac.case_seed(name)
    stub, pipe = make_pipe(case["nest"], ac.loss_config(case), seed)
    monkeypatch.setattr(pipe.sampler, "get_eps_time", lambda images, time_=None: (eps[0], time, None))
    low = iter(eps[1:])
    monkeypatch.setattr(torch.Tensor, "normal_", lambda self, *a, **k: self.copy_(next(low)))
    B, side = case.get("B", ac.LOSS_B), ac.loss_side(case)
    lm, mask = ac.text(B, seed)
    pipe.train()
    loss, _, x_t, pred, tgt, _ = pipe.get_loss({"images": ac.images(B, side, seed).cuda(), "lm_outputs": lm.cuda(),
                                                "lm_mask": mask.cuda()})
    loss.mean().backward()
    for k, v in (("loss", loss), ("x_t", x_t), ("pred", pred), ("tgt", tgt)) + tuple(
            ("grad_" + n, getattr(stub, n).grad) for n in "wbkq"):
        ref = torch.from_numpy(gold[p + k]).double()
        assert float((v.detach().cpu().double() - ref).abs().max() / ref.abs().max()) <= 1e-5, (name, k)


# ---------------------------------------------------------------- kernel level
TS = torch.tensor([0, 1, 500, 998, 999])
SIZES = [(1, (3, 17, 23)), (5, (3, 17, 23)), (64, (3, 64, 64)), (1, (3, 1024, 1024))]


def _data(B, shp, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, *shp, generator=g) * 2 - 1)
    eps = torch.randn(B, *shp, generator=g)
    t = TS[torch.arange(B) % len(TS)]
    return x.cuda(), eps.cuda(), t.cuda()


def _sampler(ptype="V_PREDICTION", ltype="DDPM", thr="CLIP"):
    cfg = ac.loss_config(ac._loss("", ptype, ltype))
    cfg["sampler_config"]["threshold_function"] = thr
    return samplers.Sampler(mc.diffusion_config_from_dict(cfg, False).sampler_config).to("cuda")


@pytest.mark.parametrize("B,shp", SIZES, ids=lambda v: str(v))
def test_q_sample_sizes(B, shp, worst):
    smp = _sampler()
    x, eps, t = _data(B, shp, 1)
    gam = Mag.of(smp.gammas)
    for div in (1.0, 2.0):
        got = smp.q_sample(x, eps, t, image_div=div)
        ref = dref.q_sample(Mag.of(x) / div if div != 1.0 else Mag.of(x), Mag.of(eps), gam[t + 1])
        check(got, ref, ac.C_XT, "q_sample", worst)


@pytest.mark.parametrize("B,H,W", [(1, 5, 7), (3, 17, 23), (64, 64, 63)])
def test_q_sample_u8_odd_width(B, H, W, worst):
    smp = _sampler()
    g = torch.Generator().manual_seed(B)
    u8 = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8).cuda()
    eps = torch.randn(B, 3, H, W, generator=g).cuda()
    t = TS[torch.arange(B) % len(TS)].cuda()
    x, xt = smp.q_sample_u8(u8, eps, t, image_div=2.0)
    ref_x = (u8.permute(0, 3, 1, 2).double() - 127) / 128
    assert torch.equal(x.double(), ref_x)
    check(xt, dref.q_sample(Mag.of(ref_x) / 2.0, Mag.of(eps), Mag.of(smp.gammas)[t + 1]), ac.C_XT, "q_sample_u8", worst)


def _loss_ref(mo, xt, x, eps, g, ptype, ltype, div, weight):
    """fp64 per-sample loss, pred, target and the gradient magnitude pieces of one loss level, as Mags."""
    xi = Mag.of(x) / div if div != 1.0 else Mag.of(x)
    loss, p, t = dref.level_loss(Mag.of(mo), Mag.of(xt), xi, Mag.of(eps), g, ptype, ltype)
    return loss * weight, p, t


@pytest.mark.parametrize("B,shp", SIZES, ids=lambda v: str(v))
@pytest.mark.parametrize("types", [("V_PREDICTION", "DDPM"), ("DDPM", "V_PREDICTION"), ("DDIM", "DDPM"),
                                   ("V_PREDICTION", "V_PREDICTION")], ids=lambda v: "_".join(v))
def test_loss_kernels_sizes(B, shp, types, worst):
    if shp[1] == 1024 and types[1] == "V_PREDICTION" and types[0] != "DDPM":
        pytest.skip("one type pair at the 1024 size keeps the file short")
    smp = _sampler(*types)
    pt, lt = ac.PT[types[0]], ac.PT[types[1]]
    x, eps, t = _data(B, shp, 2)
    xt = smp.q_sample(x, eps, t)
    g = torch.Generator().manual_seed(3)
    mo = (torch.randn(B, *shp, generator=g)).cuda().requires_grad_(True)
    tab = smp.level_table(1.0, "cuda")
    gam = Mag.of(tab)[t + 1]
    per = x[0].numel()
    for valid, weight, div in ((B, 1.0, 1.0), (1, 2.5, 2.0), (B - 1, 0.75, 1.0)):
        if valid < 1:
            continue
        spec = dict(ptype=pt, ltype=lt, levels=[dict(table=tab, image_div=div, weight=weight, want_outputs=True,
                                                     valid=valid)])
        loss, p, tg = _LossFn.apply(spec, t, mo, xt, x, eps)
        (dmo,) = torch.autograd.grad(loss.sum(), mo)
        rl, rp, rt = _loss_ref(mo.detach(), xt, x, eps, gam, pt, lt, div, weight)
        keep = (torch.arange(B, device="cuda") < valid).double()
        check(loss, Mag(rl.v * keep, rl.m), ac.loss_c(per), "kernel_loss", worst)
        check(p, rp, ac.C_ELEM, "kernel_pred", worst)
        check(tg, rt, ac.C_ELEM, "kernel_target", worst)
        v = torch.ones(B, 1, 1, 1, dtype=torch.float64, device="cuda", requires_grad=True)
        dpdv = torch.autograd.grad(dref.pred_for_training(torch.zeros_like(v), v, gam.v, pt, lt).sum(), v)[0]
        kv = keep.view(-1, 1, 1, 1)
        gref = Mag(2 * weight * (rp.v - rt.v) * dpdv / per * kv, 2 * weight * (rp.m + rt.m) * dpdv.abs() / per)
        check(dmo, gref, ac.C_GRAD, "kernel_dloss", worst)
        if B > 1 and valid == B:  # the per-sample result does not depend on the batch around it (chunking, offsets)
            j = B // 2
            spec1 = dict(ptype=pt, ltype=lt, levels=[dict(table=tab, image_div=div, weight=weight, want_outputs=False)])
            l1 = _LossFn.apply(spec1, t[j:j + 1], mo[j:j + 1].detach().contiguous(), xt[j:j + 1], x[j:j + 1],
                               eps[j:j + 1])[0]
            check(l1, rl[j:j + 1], ac.loss_c(per), "kernel_loss_b1", worst)
            assert abs(float(l1[0]) - float(loss[j])) <= 2 * ac.loss_c(per) * ac.U * float(rl.m[j])


@pytest.mark.parametrize("B,shp", SIZES[:3], ids=lambda v: str(v))
@pytest.mark.parametrize("ptype,eta,thr", [("V_PREDICTION", 0.5, "DYNAMIC"), ("DDPM", None, "CLIP"),
                                           ("V_PREDICTION", 1.0, "NONE"), ("DDPM", 0.0, "DYNAMIC_IF")])
def test_step_and_cfg_kernels_sizes(B, shp, ptype, eta, thr, worst, noise_log):
    smp = _sampler(ptype, ptype, thr)
    g = torch.Generator().manual_seed(4)
    xt = (torch.randn(B, *shp, generator=g) * 2).cuda()
    u = torch.randn(B, *shp, generator=g).cuda()
    c = torch.randn(B, *shp, generator=g).cuda()
    pred = smp._cfg(u, c, 3.0)
    check(pred, Mag.of(u) + 3.0 * (Mag.of(c) - Mag.of(u)), ac.C_ELEM, "cfg", worst)
    tab = smp.level_table(1.0, "cuda")
    for t, s, scale in ((1000, 999, 1.0), (1000, 980, 2.0), (1, 0, 1.0), (2, 1, 4.0)):
        noise_log.clear()
        x0, xs = smp._step_level(xt, pred, t, s, 1.0, s != 0, eta, scale)
        nz = noise_log[0] if ac.stochastic(s != 0, eta) else None
        r0, rs = ac.mag_step(xt, pred, tab, t, s, ac.PT[ptype], thr, scale, eta, s != 0, nz)
        check(x0, r0, ac.C_ELEM, "kernel_step_x0", worst)
        check(xs, rs, ac.C_ELEM, "kernel_step_xs", worst)


@pytest.mark.parametrize("B,H,W,r", [(2, 48, 80, 4), (2, 48, 80, 16), (64, 64, 64, 2), (1, 1024, 1024, 4)])
def test_avg_pool_and_scale_clip(B, H, W, r, worst):
    g = torch.Generator().manual_seed(r)
    x = torch.randn(B, 3, H, W, generator=g).cuda()
    got = NestedDiffusion.avg_pool(x, r)
    ref = Mag(F.avg_pool2d(x.double(), r), F.avg_pool2d(x.double().abs(), r))
    check(got, ref, r * r + 2, "avg_pool", worst)
    for scale, clip in ((2.0, True), (0.5, False), (1.0, True)):
        y = samplers.Sampler._scale_clip(x, scale, clip)
        ref = Mag.of(x) * scale
        check(y, ref.clip(-1, 1) if clip else ref, 2, "scale_clip", worst)
