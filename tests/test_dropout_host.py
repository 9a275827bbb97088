"""ResNet dropout (ResNetConfig.dropout) without a GPU: the dropout oracle, given the reference's own masks, against the
fixture of the unmodified reference in train mode (tests/golden/dropout.npz, written by
tests/golden/make_golden_dropout.py, which takes its configurations, inputs and sample positions from here), and the
Python side of the drop-in modules: construction, state_dict keys and the per-level p handed to the engine."""
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

import dropout_oracle  # noqa: E402
import tiny_configs as tc  # noqa: E402
from mdm_b200 import config as mc  # noqa: E402
from mdm_b200.models import NestedUNet, UNet  # noqa: E402
from mdm_b200.models import native  # noqa: E402

# ---- fixture layout
GOLD = os.path.join(HERE, "golden", "dropout.npz")
P_OUTER, P_INNER = 0.1, 0.25  # different per level, so that a mix-up of the levels' p shows
ARCHS = ["unet", "nested_unet"]
PARAM_SEED, TORCH_SEED = 41, 1234
OUT_SAMPLES, GRAD_SAMPLES = 512, 16


def sample_index(n, salt, k):
    """Sorted positions of a fixed sample of at most k of n elements."""
    rng = np.random.default_rng(9000 + salt)
    return np.sort(rng.choice(n, size=min(n, k), replace=False)).astype(np.int64)


def tiny_config(arch, p_outer=P_OUTER, p_inner=P_INNER):
    ucfg = copy.deepcopy(tc.TINY_UNET if arch == "unet" else tc.TINY_NESTED)
    ucfg["resnet_config"]["dropout"] = p_outer
    if arch != "unet":
        ucfg["inner_config"]["resnet_config"]["dropout"] = p_inner
    return ucfg


def tiny_inputs(arch):
    nested = arch != "unet"
    return tc.seeded_inputs(6, 2, 32 if nested else 16, 6, nlevels=2 if nested else 1)


def loss_weights(outs):
    g = torch.Generator().manual_seed(12)
    return [torch.randn(o.shape, generator=g) for o in outs]


def gold_masks(gold, arch):
    """{ResNet prefix: (N, C, H, W) keep mask as 0/1 float64} of the fixture."""
    out = {}
    for k in gold.files:
        if k.startswith(f"{arch}.mask.") and not k.endswith(".shape"):
            name = k[len(f"{arch}.mask."):]
            shape = tuple(int(s) for s in gold[k + ".shape"])
            bits = np.unpackbits(gold[k])[:int(np.prod(shape))]
            out[name] = torch.from_numpy(bits.reshape(shape).astype(np.float64))
    return out


# ---- tests
def ns(d):
    if isinstance(d, dict):
        return types.SimpleNamespace(**{k: ns(v) for k, v in d.items()})
    return d


def mirror(arch, **kw):
    cfg = mc.unet_config_from_dict(tiny_config(arch, **kw))
    cfg.conditioning_feature_dim = tc.LM_DIM
    return (UNet if arch == "unet" else NestedUNet)(3, 3, cfg)


def keys_and_shapes(gold, tag):
    return {k: torch.empty([int(s) for s in sh.split("x")] if sh else [], device="meta")
            for k, sh in zip(gold[f"{tag}.keys"], gold[f"{tag}.shapes"])}


@pytest.mark.parametrize("arch", ARCHS)
def test_oracle_with_reference_masks_matches_reference(arch):
    gold = np.load(GOLD)
    keep = gold_masks(gold, arch)
    p = {name: (P_INNER if name.startswith("inner_unet.") else P_OUTER) for name in keep}
    assert any(v == P_INNER for v in p.values()) == (arch != "unet")
    net = dropout_oracle.OracleNet(ns(tiny_config(arch)), tc.LM_DIM,
                                   lambda pre, shape: keep[pre].reshape(shape) / (1 - p[pre]))
    sd = tc.seeded_state_dict(keys_and_shapes(gold, arch), PARAM_SEED)
    P = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    x, t, lm, mask = tiny_inputs(arch)
    xs = [xi.double() for xi in x] if isinstance(x, list) else x.double()
    out = net.forward(P, xs, t, lm.double(), mask.double(), {})
    out = out if isinstance(out, (list, tuple)) else [out]
    sum((o * w.double()).sum() for o, w in zip(out, loss_weights(out))).backward()
    for i, o in enumerate(out):
        flat = o.detach().reshape(-1)
        got = flat[torch.from_numpy(sample_index(flat.numel(), i, OUT_SAMPLES))]
        ref = torch.from_numpy(gold[f"{arch}.out{i}"]).double()
        err = float((got - ref).abs().max()) / float(gold[f"{arch}.outmax{i}"])
        assert err <= 1e-5, (arch, i, err)
    # as in test_lm_head_host: mathematically zero gradients stay at round-off size, the rest match
    gmax = gold[f"{arch}.gmax"].astype(np.float64)
    gval = gold[f"{arch}.gval"]
    roundoff = 1e-4 * float(np.sort(gmax)[len(gmax) // 2])
    pos = 0
    for i, k in enumerate(gold[f"{arch}.keys"]):
        g = P[k].grad.reshape(-1)
        idx = sample_index(g.numel(), i, GRAD_SAMPLES)
        ref = torch.from_numpy(gval[pos:pos + idx.size]).double()
        pos += idx.size
        if gmax[i] <= roundoff:
            assert float(g.abs().max()) <= roundoff, (arch, k)
            continue
        assert float((g[torch.from_numpy(idx)] - ref).abs().max()) / gmax[i] <= 1e-5, (arch, k)
    assert pos == gval.size


@pytest.mark.parametrize("arch", ARCHS)
def test_reference_masks_drop_at_the_configured_rate(arch):
    """The fixture's masks are what nn.Dropout(p) drew: the kept fraction of each level lies near 1 - p."""
    gold = np.load(GOLD)
    for inner in ([False, True] if arch != "unet" else [False]):
        m = [v for k, v in gold_masks(gold, arch).items() if k.startswith("inner_unet.") == inner]
        n = sum(v.numel() for v in m)
        kept = sum(float(v.sum()) for v in m) / n
        p = P_INNER if inner else P_OUTER
        assert abs(kept - (1 - p)) <= 6 * np.sqrt(p * (1 - p) / n), (arch, inner, kept)


@pytest.mark.parametrize("p", [-0.1, 1.5])
def test_dropout_outside_unit_interval_is_refused(p):
    with pytest.raises(ValueError):
        mirror("unet", p_outer=p)
    with pytest.raises(ValueError):
        mirror("nested_unet", p_inner=p)


@pytest.mark.parametrize("name", ["cc12m_64x64", "cc12m_256x256", "cc12m_1024x1024"])
def test_state_dict_keys_unchanged_with_dropout(name):
    ucfg, _, nested = mc.load_yaml_configs(os.path.join(ROOT, "ml-mdm_b200", "mdm_b200", "configs", name + ".yaml"))
    c = ucfg
    while c is not None:
        c.resnet_config.dropout = 0.1
        c = getattr(c, "inner_config", None)
    with torch.device("meta"):
        m = (NestedUNet if nested else UNet)(3, 3, ucfg)
    want = [ln.split() for ln in open(os.path.join(HERE, "golden", f"keys_{name}.txt")).read().strip().split("\n")]
    assert [[k, "x".join(str(d) for d in v.shape)] for k, v in m.state_dict().items()] == want
    assert all(mod.training for mod in m.modules() if isinstance(mod, torch.nn.Dropout))


def test_net_cfg_carries_dropout_per_level():
    nc = native.build_net_cfg(mirror("nested_unet", p_outer=0.1, p_inner=0.25))
    assert nc.num_levels == 2
    assert nc.levels[0].dropout == pytest.approx(0.1)
    assert nc.levels[1].dropout == pytest.approx(0.25)
    assert native.build_net_cfg(mirror("unet", p_outer=0.0)).levels[0].dropout == 0.0
    assert native.LevelCfg._fields_[-1][0] == "dropout"
    assert native.NetIO._fields_[-2:] == [("dropout", ctypes.c_int32), ("dropout_seed", ctypes.c_uint64)]

