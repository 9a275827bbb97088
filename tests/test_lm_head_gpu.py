"""lm_head (UNetConfig.num_lm_head_layers) on the GPU: the token self-attention operator against the fp64
restatement of SelfAttention1D.attention element by element (the bound of tests/attn_cases.py), and the native UNet /
NestedUNet with lm_head layers against the oracle, the reference fixtures and graph replay."""
import os
import sys

import pytest
import torch

import attn_cases as ac

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "ml-mdm_b200"))

pytestmark = pytest.mark.gpu


def check_token(name, spec):
    ratios = ac.run_token(spec)
    print(name, {k: round(v, 3) for k, v in ratios.items()})
    for k, v in ratios.items():
        assert v <= ac.C, (name, k, v)


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("T", [1, 6, 77, 128, 200])
@pytest.mark.parametrize("d", [8, 64, 128, 256])
def test_token_attention_op(d, T, masked):
    check_token(f"d{d}_t{T}", ac.token_grid_spec(d, T, masked))


@pytest.mark.parametrize("name", list(ac.TOKEN))
def test_token_attention_case(name):
    """Several key chunks with planted keys 127, 128 and T - 1, head widths 136 and 192 (a partly filled second
    128-column half), and a sample whose keys are all masked (zero outputs and gradients)."""
    check_token(name, ac.TOKEN[name])


# ------------------------------------------------------------------------------------------ the network
import copy  # noqa: E402

import numpy as np  # noqa: E402

import fullwidth_cases as fc  # noqa: E402
import lm_head_oracle  # noqa: E402
import net_cases as nc  # noqa: E402
import parity  # noqa: E402
import test_lm_head_host as host  # noqa: E402
import test_net_gpu as tng  # noqa: E402
import tiny_configs as tc  # noqa: E402

MASKS = [0, 1]
KINDS = ["unet", "nested"]


def tiny_build(kind, masked, seed=7):
    """parity.tiny_model of the tiny config with two lm_head layers at the given masked_cross_attention."""
    return parity.tiny_model(host.tiny_config("unet" if kind == "unet" else "nested_unet", masked),
                             lm_head_oracle.OracleNet, seed)


@pytest.mark.parametrize("masked", MASKS, ids=["m0", "m1"])
@pytest.mark.parametrize("kind", KINDS)
def test_lm_head_forward_backward_vs_oracle(kind, masked):
    r = nc.run_case(kind, tiny_build(kind, masked), verbose=False)
    assert any(".lm_head.1.attn.qkv.weight" in k or k.startswith("lm_head.1.") for k in r["grads"])
    parity.assert_calibrated(r)


@pytest.mark.parametrize("masked", MASKS, ids=["m0", "m1"])
@pytest.mark.parametrize("kind", KINDS)
def test_lm_head_forward_vs_reference_golden(kind, masked):
    """Parameters and inputs of tests/golden/lm_head.npz (the unmodified reference in fp32)."""
    arch = "unet" if kind == "unet" else "nested_unet"
    tag = f"{kind}_m{masked}"
    model, _, _ = tiny_build(kind, masked, seed=host.PARAM_SEED)
    gold = np.load(host.GOLD)
    x, t, lm, mask = host.tiny_inputs(arch)
    nested = kind == "nested"
    model = model.cuda()
    with torch.no_grad():
        out = model([xi.cuda() for xi in x] if nested else x.cuda(), t.cuda(), lm.cuda(), mask.cuda(), {})
    for i, o in enumerate(out if nested else [out]):
        # the bound of test_net_gpu.test_forward_vs_reference_golden
        assert host.sampled_error(o, gold, tag, i, host.OUT_SAMPLES) <= 2.5e-3


def test_lm_head_full_width_calibrated_against_reference_tf32():
    """cc12m_64x64 with two lm_head layers (D = 2048, head width 256) at 77 tokens, bounds of test_fullwidth_gpu."""
    m, ocfg = fc.build("cc12m_64x64", edit=lambda c: setattr(c, "num_lm_head_layers", 2))
    rep = fc.run_case("cc12m_64x64", m, lm_head_oracle.OracleNet(ocfg, 2048), B=2, S=77, micro=True)
    parity.assert_calibrated_full_width(rep)


@pytest.mark.parametrize("kind", KINDS)
def test_lm_head_graph_replay_matches_eager_across_token_counts(kind):
    from mdm_b200 import _lib

    model, _, _ = tiny_build(kind, 1)
    eager = copy.deepcopy(model).cuda()
    graph = model.cuda()
    eager.native().set_graph_mode(False)
    graph.native().set_graph_mode(True)
    nlev = 1 if kind == "unet" else 2
    g0 = _lib.graph_launch_count()

    def step(m, inp):
        xs, t, lm, mask = inp
        out = m(xs, t, lm, mask, {})
        outs = list(out) if isinstance(out, list) else [out]
        sum((o * o).sum() for o in outs).backward()
        grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
        m.zero_grad(set_to_none=True)
        return [o.detach().clone() for o in outs], grads

    for i, tokens in enumerate([6, 6, 6, 9, 9, 9, 6]):
        x, t, lm, mask = tc.seeded_inputs(200 + i, 2, 16 if nlev == 1 else 32, tokens, nlevels=nlev)
        inp = (x.cuda() if nlev == 1 else [xi.cuda() for xi in x], t.cuda(), lm.cuda(), mask.cuda())
        og, gg = step(graph, inp)
        oe, ge = step(eager, inp)
        torch.cuda.synchronize()
        parity.assert_same_run(og, oe, gg, ge)
    # per signature the first step runs eagerly and the next ones launch a forward and a backward graph: steps 1, 2,
    # 4 and 5 (and 6 when the first signature's graphs are still cached)
    assert _lib.graph_launch_count() - g0 >= 8


@pytest.mark.parametrize("kind", KINDS)
def test_lm_head_grad_ready_ranges_are_final(kind):
    tng.check_grad_ready_ranges(tiny_build(kind, 1)[0], kind)
