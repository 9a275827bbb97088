"""lm_head (UNetConfig.num_lm_head_layers) without a GPU: the oracle and the drop-in modules against the fixture of
the unmodified reference (tests/golden/lm_head.npz, written by tests/golden/make_golden_lm_head.py, which takes its
configurations, inputs and sample positions from here), and the ctypes mirror of mdm_net_cfg."""
import copy
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "ml-mdm_b200"))

import lm_head_oracle  # noqa: E402
import tiny_configs as tc  # noqa: E402
from mdm_b200 import _lib  # noqa: E402
from mdm_b200 import config as mc  # noqa: E402
from mdm_b200.models import NestedUNet, UNet  # noqa: E402

# ---- fixture layout
GOLD = os.path.join(HERE, "golden", "lm_head.npz")
LAYERS = 2
# (fixture tag, architecture, masked_cross_attention)
TINY = [("unet_m0", "unet", 0), ("unet_m1", "unet", 1), ("nested_m0", "nested_unet", 0),
        ("nested_m1", "nested_unet", 1)]
FULL = "cc12m_64x64"
PARAM_SEED, FULL_PARAM_SEED = 31, 14
OUT_SAMPLES, GRAD_SAMPLES, FULL_SAMPLES = 512, 16, 2048


def sample_index(n, salt, k):
    """Sorted positions of a fixed sample of at most k of n elements."""
    rng = np.random.default_rng(7000 + salt)
    return np.sort(rng.choice(n, size=min(n, k), replace=False)).astype(np.int64)


def tiny_config(arch, masked):
    ucfg = copy.deepcopy(tc.TINY_UNET if arch == "unet" else tc.TINY_NESTED)
    inner = ucfg if arch == "unet" else ucfg["inner_config"]  # NestedUNet conditions through its innermost UNet
    inner["num_lm_head_layers"] = LAYERS
    inner["masked_cross_attention"] = masked
    return ucfg


def tiny_inputs(arch):
    nested = arch != "unet"
    return tc.seeded_inputs(5, 2, 32 if nested else 16, 6, nlevels=2 if nested else 1)


def full_inputs():
    return tc.seeded_inputs(24, 1, 64, 77, lm_dim=2048)


def loss_weights(outs):
    g = torch.Generator().manual_seed(11)
    return [torch.randn(o.shape, generator=g) for o in outs]


# ---- tests
def ns(d):
    if isinstance(d, dict):
        return types.SimpleNamespace(**{k: ns(v) for k, v in d.items()})
    return d


def mirror(arch, masked):
    cfg = mc.unet_config_from_dict(tiny_config(arch, masked))
    cfg.conditioning_feature_dim = tc.LM_DIM
    return (UNet if arch == "unet" else NestedUNet)(3, 3, cfg)


def keys_and_shapes(gold, tag):
    return {k: torch.empty([int(s) for s in sh.split("x")] if sh else [], device="meta")
            for k, sh in zip(gold[f"{tag}.keys"], gold[f"{tag}.shapes"])}


def sampled_error(out, gold, key, i, k):
    """max |out - reference| over the fixture's sample positions, relative to max|reference output|."""
    flat = out.detach().reshape(-1).double().cpu()
    got = flat[torch.from_numpy(sample_index(flat.numel(), i, k))]
    ref = torch.from_numpy(gold[f"{key}.out{i}"]).double()
    return float((got - ref).abs().max()) / float(gold[f"{key}.outmax{i}"])


@pytest.mark.parametrize("tag,arch,masked", TINY, ids=[t[0] for t in TINY])
def test_oracle_matches_reference_lm_head(tag, arch, masked):
    gold = np.load(GOLD)
    net = lm_head_oracle.OracleNet(ns(tiny_config(arch, masked)), tc.LM_DIM)
    sd = tc.seeded_state_dict(keys_and_shapes(gold, tag), PARAM_SEED)
    P = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    x, t, lm, mask = tiny_inputs(arch)
    xs = [xi.double() for xi in x] if isinstance(x, list) else x.double()
    out = net.forward(P, xs, t, lm.double(), mask.double(), {})
    out = out if isinstance(out, (list, tuple)) else [out]
    sum((o * w.double()).sum() for o, w in zip(out, loss_weights(out))).backward()
    for i, o in enumerate(out):
        err = sampled_error(o, gold, tag, i, OUT_SAMPLES)
        assert err <= 1e-5, (tag, i, err)
    # Gradients that are mathematically zero (a bias in front of a GroupNorm) hold only round-off in the reference:
    # those must stay at round-off size, the rest match (as in test_oracle's mixed_ratio test)
    gmax = gold[f"{tag}.gmax"].astype(np.float64)
    gval = gold[f"{tag}.gval"]
    roundoff = 1e-4 * float(np.sort(gmax)[len(gmax) // 2])
    pos = 0
    for i, k in enumerate(gold[f"{tag}.keys"]):
        g = P[k].grad.reshape(-1)
        idx = sample_index(g.numel(), i, GRAD_SAMPLES)
        ref = torch.from_numpy(gval[pos:pos + idx.size]).double()
        pos += idx.size
        if gmax[i] <= roundoff:
            assert float(g.abs().max()) <= roundoff, (tag, k)
            continue
        assert float((g[torch.from_numpy(idx)] - ref).abs().max()) / gmax[i] <= 1e-5, (tag, k)
    assert pos == gval.size


def test_oracle_matches_reference_lm_head_full_width():
    """cc12m_64x64 with two lm_head layers (D = 2048, head width 256) at B = 1 and 77 tokens."""
    import yaml

    gold = np.load(GOLD)
    with open(os.path.join(ROOT, "ml-mdm_b200", "mdm_b200", "configs", f"{FULL}.yaml")) as f:
        y = yaml.safe_load(f)
    y["unet_config"]["num_lm_head_layers"] = LAYERS
    net = lm_head_oracle.OracleNet(ns(y["unet_config"]), 2048)
    P = tc.seeded_state_dict(keys_and_shapes(gold, FULL), FULL_PARAM_SEED)
    x, t, lm, mask = full_inputs()
    with torch.no_grad():
        out = net.forward(P, x, t, lm, mask, {})
    assert tuple(out.shape) == tuple(gold[f"{FULL}.shape0"])
    assert sampled_error(out, gold, FULL, 0, FULL_SAMPLES) <= 1e-5


@pytest.mark.parametrize("tag,arch,masked", TINY, ids=[t[0] for t in TINY])
def test_mirror_state_dict_matches_reference(tag, arch, masked):
    gold = np.load(GOLD)
    sd = mirror(arch, masked).state_dict()
    assert list(sd) == list(gold[f"{tag}.keys"])
    assert ["x".join(str(s) for s in v.shape) for v in sd.values()] == list(gold[f"{tag}.shapes"])


def test_mirror_lm_head_init():
    """Default torch initialisation with proj_out and the MLP's last Linear zeroed, as in the reference."""
    m = mirror("unet", 1)
    assert len(m.lm_head) == LAYERS
    for blk in m.lm_head:
        for p in (*blk.attn.proj_out.parameters(), *blk.mlp.main[3].parameters()):
            assert float(p.detach().abs().max()) == 0.0
        assert float(blk.attn.qkv.weight.detach().abs().max()) > 0.0
        assert float(blk.mlp.main[1].weight.detach().abs().max()) > 0.0


def test_temporal_mode_still_refused():
    ucfg = copy.deepcopy(tc.TINY_UNET)
    ucfg["temporal_mode"] = True
    cfg = mc.unet_config_from_dict(ucfg)
    cfg.conditioning_feature_dim = tc.LM_DIM
    with pytest.raises(NotImplementedError):
        UNet(3, 3, cfg)


def test_net_cfg_mirror_size():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libmdm_b200.so is not built")
    from mdm_b200.models import native

    lib = ctypes.CDLL(_lib.LIB_PATH)
    lib.mdm_abi_sizeof.restype = ctypes.c_longlong
    assert native.NetCfg._fields_[-1][0] == "num_lm_head_layers"
    assert lib.mdm_abi_sizeof(3) == ctypes.sizeof(native.NetCfg)
