"""Pipelines on the GPU vs the oracle / reference goldens: q-sample (bit-exact), get_loss + gradients,
DDIM / DDPM / CFG reverse steps, 4-step DDIM sampling, for the tiny UNet and the 2-level nest."""
import copy
import os

import numpy as np
import pytest
import torch

import parity
import tiny_configs as tc
from mdm_b200 import config as mc
from mdm_b200.diffusion import Diffusion, NestedDiffusion
from oracle import diffusion_ref as dref

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def pipeline(kind):
    model, oracle, sd = parity.tiny_model(tc.TINY[kind])
    nested = kind == "nested"
    dcfg = mc.diffusion_config_from_dict(copy.deepcopy(tc.TINY_NESTED_DIFFUSION if nested else tc.TINY_DIFFUSION), nested)
    pipe = (NestedDiffusion if nested else Diffusion)(model, dcfg).to("cuda")
    gold = np.load(os.path.join(GOLD, f"tiny_{kind}.npz"))
    x, t, lm, mask = tc.seeded_inputs(3, 2, 32 if nested else 16, 6, nlevels=2 if nested else 1)
    return pipe, oracle, sd, gold, x, lm, mask, nested


def _calibrated_loss_check(pipe, oracle, sd, loss, P64, oloss, images, eps, time, lm, mask, scales, shifted, mixed_ratio=None):
    """loss and every parameter gradient of get_loss against the fp64 oracle, bounded by what the reference's own GPU
    arithmetic (the oracle in fp32 with TF32 on, same draws) scores on the same metric in the same run."""
    with parity.tf32():
        P32 = {k: v.float().cuda().requires_grad_(True) for k, v in sd.items()}
        gam = dref.gammas_f32("DEEPFLOYD", 1000).cuda()
        tl, _, _ = dref.training_loss(oracle, P32, images.float().cuda(), [e.float().cuda() for e in eps], time.cuda(),
                                      lm.float().cuda(), mask.float().cuda(), gam, scales, dref.V_PREDICTION, dref.DDPM,
                                      shifted=shifted, power=1, mixed_ratio=mixed_ratio)
        tl.mean().backward()
        torch.cuda.synchronize()
    ref_loss = oloss.detach()
    e_ours = parity.rel(loss.detach().cpu(), ref_loss)
    e_tf32 = parity.rel(tl.detach().cpu(), ref_loss)
    assert e_ours <= max(2e-3, 2.5 * e_tf32), (e_ours, e_tf32)  # per-sample loss: a mean over CHW of squared errors
    g64 = {k: v.grad for k, v in P64.items()}
    ours = parity.grad_errors({k: p.grad.cpu() for k, p in pipe.get_model().vision_model.named_parameters()}, g64)
    tf32 = parity.grad_errors({k: v.grad.cpu() for k, v in P32.items()}, g64)
    parity.assert_calibrated_grads({k: (v, tf32[k]) for k, v in ours.items()})


def test_q_sample_matches_to_one_ulp():
    """Not bit-exact by construction: torch's CPU sqrt kernel is not correctly rounded (differs from
    IEEE sqrt in ~0.6% of inputs), the device uses IEEE sqrt.rn; everything else is one rounding per op."""
    pipe, _, _, _, x, _, _, _ = pipeline("unet")
    g = torch.Generator().manual_seed(5)
    img = torch.rand(4, 3, 16, 16, generator=g) * 2 - 1
    eps = torch.randn(4, 3, 16, 16, generator=g)
    time = torch.tensor([0, 1, 500, 999])
    gam = dref.gammas_f32("DEEPFLOYD", 1000)
    ref = dref.q_sample(img, eps, gam[time + 1])
    got = pipe.sampler.q_sample(img.cuda(), eps.cuda(), time.cuda()).cpu()
    torch.testing.assert_close(got, ref, rtol=2.5e-7, atol=2.5e-7)


@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_get_loss_and_gradients(kind):
    pipe, oracle, sd, gold, x, lm, mask, nested = pipeline(kind)
    images = (x[0] if nested else x).clamp(-1, 1)
    # the product draws time/eps with torch's CUDA generator; parity is on identical noised inputs, so
    # the draws are replayed into the oracle
    torch.manual_seed(1234)
    pipe.train()
    loss, time, x_t, pred, tgt, w = pipe.get_loss({"images": images.cuda(), "lm_outputs": lm.cuda(), "lm_mask": mask.cuda()})
    loss.mean().backward()
    torch.manual_seed(1234)
    time_r = torch.randint(0, 1000, (2,), device="cuda")
    eps = [torch.randn_like(images.cuda())]
    if nested:
        eps.append(torch.empty(2, 3, 8, 8, device="cuda").normal_())
    assert torch.equal(time_r, time) and w is None
    scales = [4, 1] if nested else [1]
    P = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    gam = dref.gammas_f32("DEEPFLOYD", 1000)
    oloss, ox_t, _ = dref.training_loss(oracle, P, images.double(), [e.cpu().double() for e in eps], time.cpu(), lm.double(), mask.double(),
                                        gam, scales, dref.V_PREDICTION, dref.DDPM, shifted=nested, power=1)
    assert parity.rel(x_t.cpu().double(), ox_t[0]) <= 1e-6
    oloss.mean().backward()
    _calibrated_loss_check(pipe, oracle, sd, loss, P, oloss, images, [e.cpu() for e in eps], time.cpu(), lm, mask, scales,
                           shifted=nested)


@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_reverse_steps_vs_reference_golden(kind):
    pipe, _, _, gold, x, lm, mask, nested = pipeline(kind)
    pipe.eval()
    smp, m = pipe.sampler, pipe.get_model()
    xc = [xi.cuda() for xi in x] if nested else x.cuda()
    lmc, mc_ = lm.cuda(), mask.cuda()

    def clone(v):
        return [a.clone() for a in v] if nested else v.clone()

    with torch.no_grad():
        x0, xs, _ = smp.get_xt_minus_1(m, 500, clone(xc), lmc, mc_, {}, time_step_last=480, ddim_eta=0.0, return_details=True)
        for i, (a, b) in enumerate(zip(x0, xs) if nested else [(x0, xs)]):
            # one network evaluation (<= 2e-3 on v) pushed through x0 = a x_t - c v and the clip
            # (single-evaluation bound 2.5e-3, amplified by 1/sqrt(gamma) ~ 1.4-2 in x0 = a x_t - c v)
            assert parity.rel(a.cpu(), torch.from_numpy(gold[f"ddim_x0_{i}"])) <= 5e-3
            assert parity.rel(b.cpu(), torch.from_numpy(gold[f"ddim_xs_{i}"])) <= 5e-3
        lm2 = torch.cat([torch.zeros_like(lmc), lmc])
        xs = smp.get_xt_minus_1(m, 500, clone(xc), lm2, torch.cat([mc_, mc_]), {}, time_step_last=480, ddim_eta=0.0,
                                guidance_scale=3.0)
        for i, b in enumerate(xs if nested else [xs]):
            assert parity.rel(b.cpu(), torch.from_numpy(gold[f"cfg_xs_{i}"])) <= 5e-3
        # stochastic DDPM step: noise comes from the CUDA generator, so compare against the oracle's
        # deterministic part (posterior mean) by replaying the same noise
        torch.manual_seed(99)
        xs = smp.get_xt_minus_1(m, 500, clone(xc), lmc, mc_, {}, time_step_last=499, ddim_eta=None)
        torch.manual_seed(99)
        lv = xs if nested else [xs]
        noises = [torch.randn_like(a) for a in lv]
        gam = dref.gammas_f32("DEEPFLOYD", 1000)
        scales = [4, 1] if nested else [1]
        times = torch.full((2,), 499, dtype=torch.long, device="cuda")
        preds = m(xc, times, lmc, mc_, {})
        preds = list(preds) if nested else [preds[0]]
        for xi, p, s, nz, got in zip(x if nested else [x], preds, scales, noises, lv):
            tab = dref.shift_table(gam, s, 1) if nested else gam
            _, ref = dref.reverse_step(xi, p.cpu(), tab[500], tab[499], dref.V_PREDICTION, True, 1.0, None, True, noise=nz.cpu())
            assert parity.rel(got.cpu(), ref) <= 1e-5


@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_ddim_sampling_vs_reference_golden(kind):
    pipe, _, _, gold, x, lm, mask, nested = pipeline(kind)
    pipe.eval()
    smp, m = pipe.sampler, pipe.get_model()
    if nested:
        torch.manual_seed(7)
        low = torch.empty(2, 3, 8, 8).normal_()  # the golden's low-resolution start (CPU generator)
        init = [x[0].cuda(), low.cuda()]
    else:
        init = x.cuda()
    out = smp.sample(m, init, lm.cuda(), mask.cuda(), {}, num_inference_steps=4, ddim_eta=0.0, resample_steps=True)
    # four chained network evaluations, each within the single-evaluation bound of tests/test_net_gpu.py (2.5e-3)
    assert parity.rel(out.cpu(), torch.from_numpy(gold["sample4"])) <= 4 * 2.5e-3
    assert float(out.abs().max()) <= 1.0


def test_pipeline_sample_entry_point_shapes():
    pipe, _, _, _, x, lm, mask, _ = pipeline("nested")
    torch.manual_seed(0)
    out = pipe.sample(2, {"lm_outputs": lm.cuda(), "lm_mask": mask.cuda()}, 32, torch.device("cuda"),
                      num_inference_steps=3, ddim_eta=0.0, resample_steps=True)
    assert out.shape == (2, 3, 32, 32) and bool(torch.isfinite(out).all())
    gen = pipe.sample(2, {"lm_outputs": lm.cuda(), "lm_mask": mask.cuda()}, 32, torch.device("cuda"),
                      num_inference_steps=3, ddim_eta=1.0, resample_steps=True, yield_output=True, output_inner=True)
    frames = list(gen)
    assert len(frames) == 4 and frames[-1].shape == (2, 3, 32, 64)


def test_get_loss_mixed_ratio_batches():
    """NestedDiffusionConfig.mixed_ratio='2:1' (set by the shipped cc12m_256x256.yaml:108): the high-resolution level
    runs only the leading int(2/3 B) samples inside the engine (mdm_net_io.level_batch), predictions are zero-padded,
    the loss is rescaled and masked. Oracle: oracle.diffusion_ref.training_loss(mixed_ratio=...) -- itself pinned
    against the live reference in tests/test_oracle.py."""
    B = 3
    model, oracle, sd = parity.tiny_model(tc.TINY_NESTED)
    d = copy.deepcopy(tc.TINY_NESTED_DIFFUSION)
    d["mixed_ratio"] = "2:1"
    pipe = NestedDiffusion(model, mc.diffusion_config_from_dict(d, True)).to("cuda")
    assert pipe.mixed_ratio is not None and int(pipe.mixed_ratio[0] * B) == 2
    x, t, lm, mask = tc.seeded_inputs(3, B, 32, 6, nlevels=2)
    images = x[0].clamp(-1, 1)
    torch.manual_seed(1234)
    pipe.train()
    loss, time, x_t, pred, tgt, w = pipe.get_loss({"images": images.cuda(), "lm_outputs": lm.cuda(), "lm_mask": mask.cuda()})
    loss.mean().backward()
    assert x_t.shape[0] == pred.shape[0] == tgt.shape[0] == B
    torch.manual_seed(1234)
    time_r = torch.randint(0, 1000, (B,), device="cuda")
    eps = [torch.randn_like(images.cuda()), torch.empty(B, 3, 8, 8, device="cuda").normal_()]
    assert torch.equal(time_r, time)
    P = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    gam = dref.gammas_f32("DEEPFLOYD", 1000)
    mr = dref.mixed_ratio_fractions("2:1")
    oloss, ox_t, _ = dref.training_loss(oracle, P, images.double(), [e.cpu().double() for e in eps], time.cpu(), lm.double(),
                                        mask.double(), gam, [4, 1], dref.V_PREDICTION, dref.DDPM, shifted=True, power=1,
                                        mixed_ratio=mr)
    oloss.mean().backward()
    _calibrated_loss_check(pipe, oracle, sd, loss, P, oloss, images, [e.cpu() for e in eps], time.cpu(), lm, mask, [4, 1],
                           shifted=True, mixed_ratio=mr)


@pytest.mark.parametrize("mode,ratio,vmax", [("DYNAMIC", 0.995, 100.0), ("DYNAMIC_IF", 0.95, 1.5)])
@pytest.mark.parametrize("res", [16, 64, 256])
def test_dynamic_threshold_bound_is_torch_quantile_exactly(mode, ratio, vmax, res):
    """mdm_dynamic_threshold: exact order statistics by radix select + torch.quantile's fp32 rank / lerp arithmetic
    => the per-sample bound equals clamp(torch.quantile(|x0 s|, r), 1, max) bit for bit (samplers.py:461-498),
    including duplicated values (quantised inputs), saturated and tiny images."""
    import ctypes as C

    from mdm_b200 import _lib
    from mdm_b200.samplers import _ptr, _stream

    g = torch.Generator().manual_seed(res)
    B = 5
    amp = torch.tensor([0.3, 1.0, 2.5, 40.0, 400.0]).view(B, 1, 1, 1)
    x0 = torch.randn(B, 3, res, res, generator=g) * amp
    x0[1] = (x0[1] * 8).round() / 8           # many exact duplicates around the quantile
    x0 = x0.cuda()
    one = torch.ones(1, device="cuda")
    bound = torch.empty(B, device="cuda")
    for scale in (1.0, 4.0):
        _lib.check(_lib.lib().mdm_dynamic_threshold(_ptr(x0), _ptr(x0), _ptr(one), 0, 5, C.c_float(scale), C.c_float(ratio),
                                                    C.c_float(vmax), _ptr(bound), B, C.c_int64(x0.numel() // B), _stream()),
                   "mdm_dynamic_threshold")
        ref = torch.clamp(torch.quantile((x0 * scale).reshape(B, -1).abs(), ratio, dim=1), min=1, max=vmax)
        assert torch.equal(bound, ref), (bound.tolist(), ref.tolist())


@pytest.mark.parametrize("mode", ["DYNAMIC", "DYNAMIC_IF"])
def test_dynamic_threshold_reverse_step_and_sampling(mode):
    """Reverse step with threshold_function = DYNAMIC / DYNAMIC_IF (the web demo's default, generate_sample.py) vs the
    oracle (pinned bit-exactly to the reference's clip_sample), then a short sampling run through the entry point."""
    pipe, oracle, sd, gold, x, lm, mask, nested = pipeline("nested")
    pipe.eval()
    smp, m = pipe.sampler, pipe.get_model()
    smp._config.threshold_function = mode  # the CLIs assign the enum; plain names are accepted too
    xc = [(xi * 3).cuda() for xi in x]      # large x_t: the quantile bound is active (> 1)
    lmc, mc_ = lm.cuda(), mask.cuda()
    with torch.no_grad():
        times = torch.full((2,), 499, dtype=torch.long, device="cuda")
        preds = m(xc, times, lmc, mc_, {})   # ONE evaluation feeds both sides (two runs differ by fp32-atomic order)
        gam = dref.gammas_f32("DEEPFLOYD", 1000)
        for xi, p, s in zip(xc, preds, [4, 1]):
            a, b = smp._step_level(xi, p, 500, 480, s, True, 0.0, 1.0)
            tab = dref.shift_table(gam, s, 1)
            r0, rs = dref.reverse_step(xi.cpu(), p.cpu(), tab[500], tab[480], dref.V_PREDICTION, mode, 1.0, 0.0, True)
            assert float(r0.abs().max()) <= 1.0 + 1e-6
            assert parity.rel(a.cpu(), r0) <= 2e-6 and parity.rel(b.cpu(), rs) <= 2e-6
        x0, xs, _ = smp.get_xt_minus_1(m, 500, [a.clone() for a in xc], lmc, mc_, {}, time_step_last=480, ddim_eta=0.0,
                                       return_details=True)
        assert all(float(a.abs().max()) <= 1.0 + 1e-6 for a in x0)
    # clip_sample on a bare tensor (reference surface)
    t = (torch.randn(2, 3, 16, 16) * 2).cuda()
    assert parity.rel(smp.clip_sample(t, 2.0).cpu(), dref.clip_sample(t.cpu(), 2.0, mode)) <= 1e-6
    torch.manual_seed(0)
    out = pipe.sample(2, {"lm_outputs": lmc, "lm_mask": mc_}, 32, torch.device("cuda"), num_inference_steps=3,
                      ddim_eta=0.0, resample_steps=True)
    assert out.shape == (2, 3, 32, 32) and bool(torch.isfinite(out).all()) and float(out.abs().max()) <= 1.0


@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_get_loss_from_raw_reader_batch_uint8_and_unmasked_t5(kind):
    """Input side of the path (SURVEY.md 8f rank 3): get_loss fed the raw reader batch -- uint8 NHWC images and T5
    features not yet multiplied by their mask -- must equal get_loss fed what clis/train_parallel.py:193-199 and
    language_models/factory.py:101 prepare from it ((x - 127) / 128, permute, lm * mask) with the same draws."""
    pipe, _, _, _, x, lm, mask, nested = pipeline(kind)
    R = 32 if nested else 16
    g = torch.Generator().manual_seed(9)
    u8 = torch.randint(0, 256, (2, R, R, 3), generator=g, dtype=torch.uint8).cuda()
    mask = mask.clone()
    mask[0, 4:] = 0
    mask[1, 2:] = 0
    lm_raw, mask = lm.cuda(), mask.cuda()
    images = torch.permute((u8.float() - 127.0) / 128.0, (0, 3, 1, 2)).contiguous()   # train_parallel.py:194-195
    lm_masked = lm_raw * mask.unsqueeze(-1)                                           # factory.py:101
    pipe.train()
    vm = pipe.get_model().vision_model

    def run(sample):
        torch.manual_seed(77)
        loss, time, x_t, pred, tgt, _ = pipe.get_loss(sample)
        loss.mean().backward()
        grads = {k: p.grad.detach().clone() for k, p in vm.named_parameters()}
        vm.zero_grad(set_to_none=True)
        return loss.detach(), time, x_t, tgt, grads

    la, ta, xa, tga, ga = run({"images": images, "lm_outputs": lm_masked, "lm_mask": mask})
    lb, tb, xb, tgb, gb = run({"image": u8, "lm_outputs": lm_raw, "lm_mask": mask, "lm_mask_applied": False})
    assert torch.equal(ta, tb)
    assert torch.equal(xa, xb) and torch.equal(tga, tgb), "fused uint8 q-sample must be bit-identical"
    parity.assert_same_run([lb], [la], gb, ga)  # two engine runs differ by fp32-atomic order only
    assert vm.fuse_lm_mask is False
