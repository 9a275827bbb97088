"""GPU: DiffusionConfig.model_output_scale on the engine. Model.forward returns s * tanh(out / s) (diffusion.py:83-85),
computed in the engine's output conversion, and its backward seeds the network with dout * (1 - (out / s)^2);
NestedModel and a U-Net called directly are never scaled, and the encoded-once sampling path scales as Model does.

Two evaluations of the engine on the same inputs differ by ~1e-3 (GroupNorm partial sums are combined by fp32
atomics, DESIGN.md section 4), so comparisons between two calls allow the spread the test measures between two
unscaled calls."""
import copy

import numpy as np
import pytest
import torch

import net_cases as nc
import test_rect_oracle as fx
from mdm_b200 import config as mc
from mdm_b200.diffusion import Diffusion, Model, NestedModel
from oracle import diffusion_ref as dref

pytestmark = pytest.mark.gpu


def _unet_inputs(hw=(24, 40), seed=3):
    x, t, lm, mask = fx.rect_inputs(seed, 2, hw, 6)
    return x.cuda(), t.cuda(), lm.cuda(), mask.cuda()


def _cfg(s, nested=False):
    d = copy.deepcopy(fx.tc.TINY_NESTED_DIFFUSION if nested else fx.tc.TINY_DIFFUSION)
    d["model_output_scale"] = s
    return mc.diffusion_config_from_dict(d, nested=nested)


@pytest.mark.parametrize("s", [0.1, 1.0, 4.0])
def test_forward_is_tanh_of_the_unscaled_output(s):
    vm, _, _ = nc.build("unet")
    vm = vm.cuda()
    inp = _unet_inputs()
    with torch.no_grad():
        o1 = vm(*inp, {})
        o2 = vm(*inp, {})
        y = Model(vm, _cfg(s))(*inp, {})[0]
    spread = float((o1 - o2).abs().max())
    assert spread <= 5e-3 * float(o1.abs().max())
    # d/do of s*tanh(o/s) is at most 1, so the run-to-run spread of o bounds its effect on y; the spread of one pair
    # of calls is itself a sample, hence the factor 2
    assert float((y - s * torch.tanh(o1 / s)).abs().max()) <= 1e-6 + 2 * spread


# at s = 0.1 the factor 1 - (y/s)^2 turns the outputs' run-to-run spread (~1e-3 of O(1) outputs) into ~1e-2 of the
# factor, so the gradients of two calls agree only to that
@pytest.mark.parametrize("s,med_tol,max_tol", [(0.1, 1e-2, 5e-2), (1.0, 3e-3, 2e-2), (4.0, 3e-3, 2e-2)])
def test_gradient_matches_autograd_through_tanh(s, med_tol, max_tol):
    vm, _, _ = nc.build("unet")
    vm = vm.cuda()
    inp = _unet_inputs()
    g = torch.Generator().manual_seed(17)
    w = torch.randn(2, 3, 24, 40, generator=g).cuda()
    grads = []
    for scaled in (False, True):
        if scaled:
            y = Model(vm, _cfg(s))(*inp, {})[0]
        else:
            o = vm(*inp, {})
            y = s * torch.tanh(o / s)
        (y * w).sum().backward()
        grads.append({k: p.grad.detach().clone() for k, p in vm.named_parameters()})
        vm.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    ref, got = grads
    mags = sorted(float(v.abs().max()) for v in ref.values())
    floor = 1e-2 * mags[len(mags) // 2]
    errs = sorted(float((got[k] - v).abs().max()) / max(float(v.abs().max()), floor) for k, v in ref.items())
    assert errs[len(errs) // 2] <= med_tol and errs[-1] <= max_tol, (errs[len(errs) // 2], errs[-1])


def test_get_loss_matches_reference_fixture():
    """The u24x40_s case of tests/golden/rect.npz: the reference's x_t and times through Model.forward with s = 0.1,
    then the per-sample loss of Diffusion.get_loss, against the reference's loss."""
    gold = np.load(fx.GOLD)
    tag, h, w, s = "u24x40_s", 24, 40, 0.1
    vm, _, _ = nc.build("unet")
    model = Model(vm.cuda(), _cfg(s))
    x, _, lm, mask = fx.rect_inputs(3, 2, (h, w), 6)
    images = x.clamp(-1, 1)
    torch.manual_seed(1234)
    time = torch.randint(0, 1000, (2,))
    eps = torch.randn_like(images)
    x_t = torch.from_numpy(gold[f"{tag}.loss_xt"])
    with torch.no_grad():
        out = model(x_t.cuda(), time.cuda(), lm.cuda(), mask.cuda(), {})[0].cpu()
    g = dref.gammas_f32("DEEPFLOYD", 1000)[time + 1]
    loss, _, _ = dref.level_loss(out.double(), x_t.double(), images.double(), eps.double(), g.double(),
                                 dref.V_PREDICTION, dref.DDPM)
    ref = torch.from_numpy(gold[f"{tag}.loss"]).double()
    assert float((loss - ref).abs().max() / ref.abs().max()) <= 2e-3


def test_ddim50_cfg_encoded_once_matches_per_step():
    class PerStep(Model):  # overrides forward: the sampler calls it in full at every step
        def forward(self, *a, **k):
            return super().forward(*a, **k)

    vm, _, _ = nc.build("unet")
    vm = vm.cuda()
    pipe = Diffusion(vm, _cfg(0.1)).to("cuda")
    _, _, lm, mask = _unet_inputs()
    lm2 = torch.cat([torch.zeros_like(lm), lm])
    mask2 = torch.cat([mask, mask])
    imgs = []
    for m in (pipe.model, PerStep(vm, _cfg(0.1)), pipe.model):
        torch.manual_seed(5)
        noise = torch.randn(2, 3, 24, 40).cuda()
        imgs.append(pipe.sampler.sample(m, noise, lm2, mask2, {}, num_inference_steps=50, resample_steps=True,
                                        ddim_eta=0.0, guidance_scale=3.0))
    torch.cuda.synchronize()
    assert nc.rel(imgs[0], imgs[1]) <= max(3e-3, 3.0 * nc.rel(imgs[2], imgs[0])), (nc.rel(imgs[0], imgs[1]),
                                                                                nc.rel(imgs[2], imgs[0]))


def _spy(native):
    seen = []
    orig = native._forward

    def fwd(*a, **k):
        seen.append(k.get("output_scale", 0.0))
        return orig(*a, **k)
    native._forward = fwd
    return seen


def test_nested_model_and_direct_unet_are_never_scaled():
    vm, _, _ = nc.build("nested")
    vm = vm.cuda()
    xs, t, lm, mask = fx.rect_inputs(3, 2, fx.NEST_HW, 6, nlevels=2)
    inp = ([x.cuda() for x in xs], t.cuda(), lm.cuda(), mask.cuda())
    seen = _spy(vm.native())
    with torch.no_grad():
        a = NestedModel(vm, _cfg(0.1, nested=True))(*inp, {})
        b = vm(*inp, {})
    # the engine runs the same unscaled code path (the scale reaches it as 0) for both calls
    assert seen == [0.0, 0.0]
    for p, q in zip(a, b):
        assert nc.rel(p, q) <= 3e-3
        assert float(p.abs().max()) > 0.15  # not squashed into (-0.1, 0.1)
    u, _, _ = nc.build("unet")
    u = u.cuda()
    seen = _spy(u.native())
    Model(u, _cfg(0.1))  # constructing the pipeline model changes nothing about direct calls
    x, t, lm, mask = _unet_inputs()
    with torch.no_grad():
        u(x, t, lm, mask, {})
        cemb, cond, cmask = u.forward_conditioning(lm, mask)
        u.forward_denoising(x, t, cemb, cond, cmask)
    assert seen == [0.0, 0.0]


def test_graph_replay_follows_the_scale():
    vm, _, _ = nc.build("unet")
    eager = copy.deepcopy(vm).cuda()
    graph = vm.cuda()
    eager.native().set_graph_mode(False)
    graph.native().set_graph_mode(True)
    for step, s in enumerate([0.1, 1.0, 0.1, 1.0, 0.1, 1.0, 0.0, 0.1]):
        inp = _unet_inputs(seed=300 + step)
        outs = []
        for m in (graph, eager):
            y = Model(m, _cfg(s))(*inp, {})[0]
            (y * y).sum().backward()
            outs.append((y.detach().clone(), m.conv_out.weight.grad.clone()))
            m.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        # absolute: with |y| <= s the relative metric inflates the unscaled outputs' ~1e-3 spread by 1/s, while a graph
        # replaying another s is off by up to |s - s'|
        assert float((outs[0][0] - outs[1][0]).abs().max()) <= 1e-2, (step, s)
        assert nc.rel(outs[0][1], outs[1][1]) <= 5e-2, (step, s)
        if s:
            assert float(outs[0][0].abs().max()) <= s * (1 + 1e-6)  # |s tanh| <= s, up to fp32 rounding of s
