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
import parity  # noqa: E402
import tiny_configs as tc  # noqa: E402
from mdm_b200 import _lib  # noqa: E402
from mdm_b200 import config as mc  # noqa: E402
from mdm_b200.diffusion import NestedDiffusion, NestedModel  # noqa: E402
from mdm_b200.samplers import NestedSampler  # noqa: E402
from oracle import unet_ref  # noqa: E402

pytestmark = pytest.mark.gpu


def build(arch):
    return parity.tiny_model(mx.tiny_config(arch), seed=mx.PARAM_SEED)


def run_case(arch, micros, batch=mx.BATCH, level_batch=None):
    """parity.report of the engine, the fp64 oracle and the reference-TF32 arm, all on the GPU. level_batch: leading
    rows each level runs (mixed_ratio), outermost first."""
    model, oracle, sd = build(arch)
    x, t, lm, mask = mx.tiny_inputs(arch, batch)
    xs = [x] if arch == "unet" else list(x)
    if level_batch is not None:
        xs = [xi[:b] for xi, b in zip(xs, level_batch)]
    args = (sd, xs, t, lm, mask, micros, mx.loss_weights(xs))
    f64 = parity.oracle_arm(oracle.forward, *args, torch.float64, "cuda")
    tf32 = parity.oracle_arm(oracle.forward, *args, torch.float32, "cuda", tf32=True)
    return parity.report(parity.engine_arm(model, *args[1:]), f64, tf32)


@pytest.mark.parametrize("which", mx.MICRO_SETS)
@pytest.mark.parametrize("arch", mx.ARCHS)
def test_calibrated_parity(arch, which):
    rep = run_case(arch, mx.micro_set(arch, which))
    parity.assert_calibrated(rep)
    assert sum(1 for k in rep["grads"] if ".watermark_score." in "." + k) == 4 * (1 if arch == "unet" else 2)


def test_key_no_level_configures_is_ignored():
    micros = dict(mx.micro_set("nested_unet", "all"), aesthetic=torch.tensor([5.5, 2.0]))
    parity.assert_calibrated(run_case("nested_unet", micros))


def test_nest_with_mixed_ratio():
    """The outer level runs the leading row only: it reads the leading row of every micro value."""
    rep = run_case("nested_unet", mx.micro_set("nested_unet", "all", batch=3), batch=3, level_batch=(1, 3))
    parity.assert_calibrated(rep)


def test_full_width_cc12m_256_with_watermark_score():
    def add_watermark_score(c):
        c.micro_conditioning = c.micro_conditioning + ",watermark_score:0"
        c.inner_config.micro_conditioning = c.inner_config.micro_conditioning + ",watermark_score:0"

    m, ocfg = fc.build("cc12m_256x256", edit=add_watermark_score)
    micros = {"scale": torch.tensor([48.0, 700.0]), "watermark_score": torch.tensor([0.2, 0.85])}
    rep = fc.run_case("cc12m_256x256", m, unet_ref.OracleNet(ocfg, 2048), B=2, S=8, micros=micros)
    assert sum(1 for k in rep["grads"] if ".watermark_score." in "." + k) == 8
    parity.assert_calibrated_full_width(rep)


def _grads(m):
    return {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}


def test_graph_replay_across_key_presence_changes():
    model, _, _ = build("nested_unet")
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
            parity.assert_same_run(og, oe, gg, ge)
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
    vm, _, _ = build("nested_unet")
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
    assert parity.rel(a, b) <= max(parity.RUN_OUT, 3.0 * parity.rel(b2, b)), (parity.rel(a, b), parity.rel(b2, b))
    c = _sample(sampler, model, x, lm.cuda(), mask.cuda(), {}, 3.0, 8, False)
    assert parity.rel(a, c) > 10 * parity.RUN_OUT  # the values reach the samples


def test_nested_get_loss_reads_watermark_score():
    vm, _, _ = build("nested_unet")
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
