"""GPU: general micro-conditioning (keys other than `scale`, per-level keys, orders and defaults) on the engine.
  - calibrated parity (DESIGN.md section 4) of outputs and every parameter gradient, cond_layers.* included, against the
    fp64 oracle with bounds set by the reference-TF32 arm of the same run: both tiny architectures with every micro
    set, a micros dict holding a key no level configures, the nest with mixed_ratio, and a full-width cc12m_256x256
    step with watermark_score added to both levels;
  - CUDA-graph replay against eager while the set of given keys changes between calls;
  - DDIM with guidance through forward_denoising, with one-row and 2B-row micros, against per-step forward;
  - NestedDiffusion.get_loss reading sample["watermark_score"]."""
import copy
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "ml-mdm_b200"))

import fullwidth_cases as fc  # noqa: E402
import micro_cases as mx  # noqa: E402
import tiny_configs as tc  # noqa: E402
from mdm_b200 import _lib  # noqa: E402
from mdm_b200 import config as mc  # noqa: E402
from mdm_b200.diffusion import NestedDiffusion, NestedModel  # noqa: E402
from mdm_b200.models import NestedUNet  # noqa: E402
from mdm_b200.samplers import NestedSampler  # noqa: E402

pytestmark = pytest.mark.gpu

RUN_OUT, RUN_GRAD = 3e-3, 2e-2  # two engine runs (fp32 atomics add in a varying order)


@pytest.mark.parametrize("which", mx.MICRO_SETS)
@pytest.mark.parametrize("arch", mx.ARCHS)
def test_calibrated_parity(arch, which):
    rep = mx.run_case(arch, mx.micro_set(arch, which))
    mx.assert_calibrated(rep)
    assert sum(1 for k in rep["grads"] if ".watermark_score." in "." + k) == 4 * (1 if arch == "unet" else 2)


def test_key_no_level_configures_is_ignored():
    micros = dict(mx.micro_set("nested_unet", "all"), aesthetic=torch.tensor([5.5, 2.0]))
    mx.assert_calibrated(mx.run_case("nested_unet", micros))


def test_nest_with_mixed_ratio():
    """The outer level runs the leading row only: it reads the leading row of every micro value."""
    rep = mx.run_case("nested_unet", mx.micro_set("nested_unet", "all", batch=3), batch=3, level_batch=(1, 3))
    mx.assert_calibrated(rep)


def test_full_width_cc12m_256_with_watermark_score():
    ucfg, _, _ = mc.load_yaml_configs(os.path.join(fc.CFG_DIR, "cc12m_256x256.yaml"))
    ucfg.micro_conditioning = ucfg.micro_conditioning + ",watermark_score:0"
    ucfg.inner_config.micro_conditioning = ucfg.inner_config.micro_conditioning + ",watermark_score:0"
    ocfg = copy.deepcopy(ucfg)
    torch.manual_seed(0)
    m = NestedUNet(3, 3, ucfg)
    with torch.no_grad():
        for p in m.parameters():
            if float(p.abs().max()) == 0:
                p.normal_(0, 0.02)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    xs, t, lm, mask, ws, _ = fc.inputs("cc12m_256x256", 2, 8)
    micros = {"scale": torch.tensor([48.0, 700.0]), "watermark_score": torch.tensor([0.2, 0.85])}
    o64, g64 = fc.run_oracle(ocfg, sd, xs, t, lm, mask, ws, micros, torch.float64, False)
    o32, g32 = fc.run_oracle(ocfg, sd, xs, t, lm, mask, ws, micros, torch.float32, True)
    oo, go = fc.run_ours(m, xs, t, lm, mask, ws, micros)
    # the bounds of tests/test_fullwidth_gpu.py
    for i, (a, b, r) in enumerate(zip(oo, o32, o64)):
        assert fc.rel(a, r) <= max(1e-3, 1.5 * fc.rel(b, r)), i
    assert not [k for k in g64 if k not in go]
    errs = {k: (fc.rel(go[k], r), fc.rel(g32[k], r)) for k, r in g64.items()}
    assert sum(1 for k in errs if ".watermark_score." in "." + k) == 8
    defined = {k: v for k, v in errs.items() if v[1] <= 0.5}
    typical = sorted(float(r.abs().max()) for r in g64.values())[len(g64) // 2]
    for k in errs:
        if k not in defined:
            lim = 3.0 * max(float(g32[k].abs().max()), 1e-3 * typical)
            assert float(go[k].abs().max()) <= lim, k
    o = sorted(v[0] for v in defined.values())
    r = sorted(v[1] for v in defined.values())
    n = len(o)
    assert o[n // 2] <= 1.25 * r[n // 2] and o[int(0.9 * n)] <= 1.25 * r[int(0.9 * n)]
    bad = {k: v for k, v in defined.items() if v[0] > 3.0 * max(v[1], r[n // 2])}
    assert not bad, bad


def _grads(m):
    return {k: (p.grad.detach().clone() if p.grad is not None else None) for k, p in m.named_parameters()}


def test_graph_replay_across_key_presence_changes():
    model, _, _ = mx.build("nested_unet")
    eager, graph = copy.deepcopy(model).cuda(), model.cuda()
    eager.native().set_graph_mode(False)
    graph.native().set_graph_mode(True)
    g0 = _lib.graph_launch_count()
    x, t, lm, mask = mx.tiny_inputs("nested_unet")
    xs = [xi.cuda() for xi in x]
    ws = [torch.randn(xi.shape, device="cuda") for xi in xs]
    gen = torch.Generator().manual_seed(21)
    presence = [("scale", "watermark_score"), ("watermark_score",), (), ("scale", "watermark_score")]
    for rnd in range(3):  # per signature: eager, capture, replay
        for keys in presence:
            vals = {"scale": 120 * torch.rand(2, generator=gen), "watermark_score": torch.rand(2, generator=gen)}
            micros = {k: vals[k].cuda() for k in keys}
            res = []
            for m in (graph, eager):
                outs = m(xs, t.cuda(), lm.cuda(), mask.cuda(), micros)
                sum((o * w).sum() for o, w in zip(outs, ws)).backward()
                gr = _grads(m)
                m.zero_grad(set_to_none=True)
                with torch.no_grad():
                    inf = m(xs, t.cuda(), lm.cuda(), mask.cuda(), micros)
                res.append(([o.detach() for o in outs] + list(inf), gr))
            (og, gg), (oe, ge) = res
            for a, b in zip(og, oe):
                assert mx.rel(a, b) <= RUN_OUT, (rnd, keys)
            mags = sorted(float(v.abs().max()) for v in ge.values() if v is not None)
            floor = 1e-2 * mags[len(mags) // 2]
            for k in ge:
                if ge[k] is not None:
                    assert float((gg[k] - ge[k]).abs().max()) / max(float(ge[k].abs().max()), floor) <= RUN_GRAD, (k, keys)
    assert _lib.graph_launch_count() - g0 >= 3 * 2 * 2  # replays of the forward and backward of >= 2 signatures


def _sample(sampler, model, x, lm, mask, micros, g, steps, per_step):
    if per_step:
        sampler._encode_text = lambda *a: None  # what a foreign model wrapper gets: model(...) at every step
    torch.manual_seed(5)
    try:
        return sampler.sample(model, x, lm, mask, micros, num_inference_steps=steps, ddim_eta=0.0, resample_steps=True,
                              guidance_scale=g)
    finally:
        if per_step:
            del sampler._encode_text


@pytest.mark.parametrize("B,rows", [(1, 1), (2, 4)], ids=["one_row", "doubled_rows"])
def test_ddim_with_guidance_through_forward_denoising(B, rows):
    """One-row micros broadcast over the guidance-doubled batch; 2B-row micros are generate_batch's doubled tensors."""
    vm, _, _ = mx.build("nested_unet")
    model = NestedModel(vm.cuda(), mc.NestedDiffusionConfig(no_use_residual=True)).eval()
    sampler = NestedSampler(mc.SamplerConfig(num_diffusion_steps=32)).cuda()
    _, _, lm, mask = mx.tiny_inputs("nested_unet", batch=2 * B)
    x = torch.randn(B, 3, 32, 32, generator=torch.Generator().manual_seed(9)).cuda()
    micros = {"scale": torch.tensor([30.0, 90.0, 30.0, 90.0][:rows]).cuda(),
              "watermark_score": torch.tensor([0.25, 0.75, 0.25, 0.75][:rows]).cuda()}
    a = _sample(sampler, model, x, lm.cuda(), mask.cuda(), micros, 3.0, 8, False)
    b = _sample(sampler, model, x, lm.cuda(), mask.cuda(), micros, 3.0, 8, True)
    b2 = _sample(sampler, model, x, lm.cuda(), mask.cuda(), micros, 3.0, 8, True)
    # guidance amplifies each evaluation's run-to-run difference by 2w - 1: the bound is the per-step loop's own spread
    assert mx.rel(a, b) <= max(RUN_OUT, 3.0 * mx.rel(b2, b)), (mx.rel(a, b), mx.rel(b2, b))
    c = _sample(sampler, model, x, lm.cuda(), mask.cuda(), {}, 3.0, 8, False)
    assert mx.rel(a, c) > 10 * RUN_OUT  # the values reach the samples


def test_nested_get_loss_reads_watermark_score():
    vm, _, _ = mx.build("nested_unet")
    dcfg = mc.NestedDiffusionConfig(**{k: v for k, v in tc.TINY_NESTED_DIFFUSION.items() if k != "sampler_config"})
    dcfg.sampler_config = mc.SamplerConfig(num_diffusion_steps=1000)
    pipe = NestedDiffusion(vm, dcfg).to("cuda")
    pipe.train()
    g = torch.Generator().manual_seed(17)
    B = 2
    sample = {"images": (torch.rand(B, 3, 32, 32, generator=g) * 2 - 1).cuda(),
              "lm_outputs": torch.randn(B, 6, tc.LM_DIM, generator=g).cuda(), "lm_mask": torch.ones(B, 6).cuda(),
              "watermark_score": torch.tensor([0.1, 0.95]).cuda()}
    loss, *_ = pipe.get_loss(sample)
    loss.mean().backward()
    assert bool(torch.isfinite(loss).all())
    for k, p in vm.named_parameters():
        if ".watermark_score." in "." + k:
            assert p.grad is not None and float(p.grad.abs().max()) > 0, k
