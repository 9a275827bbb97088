"""CPU: the oracle on non-square images and with DiffusionConfig.model_output_scale, pinned against
tests/golden/rect.npz, which tests/golden/make_golden_rect.py generates from the unmodified reference.

The reference's U-Net is fully convolutional, so any (B, C, H, W) whose sides divide by the downsampling runs; its
Model.forward returns s * tanh(out / s) for s != 0 (diffusion.py:83-85) and NestedModel.forward never applies s.
The oracle has no notion of the scale, so `scaled` below adds that rule on the test side (as lm_head_oracle.py adds
the lm_head layers). The fixture layout is shared with the generator through the helpers of this module."""
import copy
import os
import types

import numpy as np
import pytest
import torch

import tiny_configs as tc
from oracle import diffusion_ref as dref
from oracle import unet_ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rect.npz")
PARAM_SEED = 7
# tiny UNet cases: (tag, H, W, model_output_scale). 18x30 runs an odd 9x15 inner resolution and W/2 = 15 on the
# folded 32-channel convs; 24x40 / 40x24 put partial 8x16 conv tiles on both axes
UNET_CASES = [("u24x40", 24, 40, 0.0), ("u40x24", 40, 24, 0.0), ("u18x30", 18, 30, 0.0), ("u24x40_s", 24, 40, 0.1)]
NEST_HW = (48, 80)      # tiny nest, outer level; the inner level runs 12x20
FULL = "cc12m_64x64"
FULL_HW = (64, 96)      # innermost 8x12
FULL_PARAM_SEED = 21
FULL_SAMPLES = 4096


def ns(d):
    if isinstance(d, dict):
        return types.SimpleNamespace(**{k: ns(v) for k, v in d.items()})
    return d


def rect_inputs(seed, batch, hw, tokens, lm_dim=tc.LM_DIM, nlevels=1, ratio=4):
    """tiny_configs.seeded_inputs for an (H, W) image: the same draws in the same order."""
    rng = np.random.default_rng(seed)
    xs = []
    h, w = hw
    for _ in range(nlevels):
        xs.append(torch.from_numpy(rng.standard_normal((batch, 3, h, w)).astype(np.float32)))
        h, w = h // ratio, w // ratio
    times = torch.from_numpy(rng.integers(0, 1000, size=(batch,)).astype(np.int64))
    lm = torch.from_numpy(rng.standard_normal((batch, tokens, lm_dim)).astype(np.float32))
    lens = rng.integers(1, tokens + 1, size=(batch,))
    mask = torch.zeros(batch, tokens)
    for i, n in enumerate(lens):
        mask[i, :n] = 1
    lm = lm * mask.unsqueeze(-1)
    return (xs if nlevels > 1 else xs[0]), times, lm, mask


def loss_weights(outs, seed=11):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(o.shape, generator=g) for o in outs]


def sample_index(n, salt, count):
    """A fixed sample of `count` flat positions of an n-element tensor."""
    return np.random.default_rng(1000 + salt).integers(0, n, size=min(count, n))


def full_inputs():
    return rect_inputs(5, 1, FULL_HW, 77, lm_dim=2048)


class scaled:
    """Model.forward's model_output_scale on top of an oracle net: s * tanh(out / s) (diffusion.py:83-85)."""

    def __init__(self, net, s):
        self.net, self.s = net, float(s)

    def forward(self, *a, **k):
        o = self.net.forward(*a, **k)
        return self.s * torch.tanh(o / self.s) if self.s != 0 else o


def tiny(kind):
    ucfg = copy.deepcopy(tc.TINY_NESTED if kind == "nested" else tc.TINY_UNET)
    if kind == "nested":
        ucfg["initialize_inner_with_pretrained"] = None
    return unet_ref.OracleNet(ns(ucfg), tc.LM_DIM)


def params(kind, requires_grad=False):
    from mdm_b200 import config as mc
    from mdm_b200.models import NestedUNet, UNet

    cfg = mc.unet_config_from_dict(copy.deepcopy(tc.TINY_NESTED if kind == "nested" else tc.TINY_UNET))
    cfg.conditioning_feature_dim = tc.LM_DIM
    m = (NestedUNet if kind == "nested" else UNet)(3, 3, cfg)
    sd = tc.seeded_state_dict(m.state_dict(), PARAM_SEED)
    return {k: v.clone().requires_grad_(requires_grad) for k, v in sd.items()}, [k for k, _ in m.named_parameters()]


def close(a, b, tol=1e-5):
    a = torch.as_tensor(a).double()
    b = torch.as_tensor(b).double()
    err = float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
    assert err <= tol, err


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.mark.parametrize("tag,h,w,s", UNET_CASES)
def test_unet_forward_loss_and_sample_match_reference(gold, tag, h, w, s):
    net = scaled(tiny("unet"), s)
    P, names = params("unet", requires_grad=True)
    x, t, lm, mask = rect_inputs(3, 2, (h, w), 6)
    with torch.no_grad():
        close(net.forward(P, x, t, lm, mask, {}), gold[f"{tag}.fwd"])
    # Diffusion.get_loss: the CPU generator's draws (time, then eps), as samplers.py:233-242 makes them
    images = x.clamp(-1, 1)
    torch.manual_seed(1234)
    time = torch.randint(0, 1000, (2,))
    eps = [torch.randn_like(images)]
    assert np.array_equal(time.numpy(), gold[f"{tag}.loss_time"])
    gam = dref.gammas_f32("DEEPFLOYD", 1000)
    loss, x_t, _ = dref.training_loss(net, P, images, eps, time, lm, mask, gam, [1], dref.V_PREDICTION, dref.DDPM,
                                      shifted=False, power=1)
    close(x_t[0], gold[f"{tag}.loss_xt"], 1e-6)
    close(loss, gold[f"{tag}.loss"])
    loss.mean().backward()
    norms = np.array([float(P[k].grad.norm()) for k in names])
    ref = gold[f"{tag}.grad_norms"]
    assert np.max(np.abs(norms - ref) / np.maximum(ref, 1e-3 * np.median(ref))) < 1e-3
    close(P["conv_out.weight"].grad, gold[f"{tag}.grad_conv_out"], 1e-4)
    # 2-step DDIM sample from seeded noise
    torch.manual_seed(7)
    noise = torch.randn(2, 3, h, w)
    final = dref.sample_loop(net, {k: v.detach() for k, v in P.items()}, [noise], lm, mask, gam, [1],
                             dref.V_PREDICTION, 1000, 2, 0.0)
    close(final[0], gold[f"{tag}.sample2"], 1e-5)


def test_nest_forward_and_backward_match_reference(gold):
    net = tiny("nested")
    P, names = params("nested", requires_grad=True)
    xs, t, lm, mask = rect_inputs(3, 2, NEST_HW, 6, nlevels=2)
    assert tuple(xs[1].shape[2:]) == (NEST_HW[0] // 4, NEST_HW[1] // 4)
    outs = list(net.forward(P, xs, t, lm, mask, {}))
    for i, o in enumerate(outs):
        close(o.detach(), gold[f"nest.fwd{i}"])
    sum((o * w).sum() for o, w in zip(outs, loss_weights(outs))).backward()
    norms = np.array([float(P[k].grad.norm()) for k in names])
    ref = gold["nest.grad_norms"]
    assert np.max(np.abs(norms - ref) / np.maximum(ref, 1e-3 * np.median(ref))) < 1e-3


def full_config():
    import yaml

    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    with open(os.path.join(root, "ml-mdm_b200", "mdm_b200", "configs", f"{FULL}.yaml")) as f:
        return yaml.safe_load(f)["unet_config"]


def test_fullwidth_64_forward_on_64x96_matches_reference(gold):
    net = unet_ref.OracleNet(ns(full_config()), 2048)
    shapes = {k: torch.empty(tuple(int(d) for d in s.split("x"))) for k, s in zip(gold[f"{FULL}.keys"],
                                                                                 gold[f"{FULL}.shapes"])}
    P = tc.seeded_state_dict(shapes, FULL_PARAM_SEED)
    x, t, lm, mask = full_inputs()
    with torch.no_grad():
        o = net.forward(P, x, t, lm, mask, {})
    assert tuple(o.shape) == tuple(gold[f"{FULL}.shape"])
    flat = o.reshape(-1).numpy()
    got = flat[sample_index(flat.size, 0, FULL_SAMPLES)]
    assert np.max(np.abs(got - gold[f"{FULL}.out"])) <= 1e-5 * float(gold[f"{FULL}.outmax"])
