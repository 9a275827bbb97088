"""General micro-conditioning (UNetConfig.micro_conditioning with keys other than `scale`): the configurations, inputs
and micro sets shared by the fixture generator (tests/golden/make_golden_micro.py), the host tests
(tests/test_micro_host.py), the GPU tests (tests/test_micro_gpu.py) and tests/profile_micro.py, and the calibrated
parity run of the engine against the fp64 oracle.

Two tiny architectures:
  unet          TINY_UNET with "scale:16,watermark_score:0,aesthetic:5"
  nested_unet   TINY_NESTED with "scale:64,watermark_score:0" outside and "watermark_score:0,scale:16" inside (the
                same keys in a different order per level)
Three micro sets: every key given (scale values below and above each level's default), only watermark_score, none."""
import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.join(HERE, ".."), os.path.join(HERE, "..", "ml-mdm_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import tiny_configs as tc  # noqa: E402

GOLD = os.path.join(HERE, "golden", "micro.npz")
ARCHS = ["unet", "nested_unet"]
MICRO_SETS = ["all", "wm", "none"]
PARAM_SEED = 43
BATCH, TOKENS = 2, 6
OUT_SAMPLES, GRAD_SAMPLES = 512, 16


def tiny_config(arch):
    if arch == "unet":
        ucfg = copy.deepcopy(tc.TINY_UNET)
        ucfg["micro_conditioning"] = "scale:16,watermark_score:0,aesthetic:5"
    else:
        ucfg = copy.deepcopy(tc.TINY_NESTED)
        ucfg["micro_conditioning"] = "scale:64,watermark_score:0"
        ucfg["inner_config"]["micro_conditioning"] = "watermark_score:0,scale:16"
    return ucfg


def tiny_inputs(arch, batch=BATCH):
    nested = arch != "unet"
    return tc.seeded_inputs(8, batch, 32 if nested else 16, TOKENS, nlevels=2 if nested else 1)


def micro_set(arch, which, batch=BATCH):
    """fp32 (batch,) CPU tensors. `scale` straddles every level's default (16 / 64): 8 passes, 100 is clamped."""
    base = {"scale": [8.0, 100.0], "watermark_score": [0.3, 0.9], "aesthetic": [4.5, 6.25]}
    if which == "all":
        keys = ["scale", "watermark_score"] + (["aesthetic"] if arch == "unet" else [])
    elif which == "wm":
        keys = ["watermark_score"]
    else:
        keys = []
    return {k: torch.tensor((base[k] * batch)[:batch], dtype=torch.float32) for k in keys}


def loss_weights(outs):
    g = torch.Generator().manual_seed(13)
    return [torch.randn(o.shape, generator=g) for o in outs]


def sample_index(n, salt, k):
    """Sorted positions of a fixed sample of at most k of n elements."""
    rng = np.random.default_rng(9100 + salt)
    return np.sort(rng.choice(n, size=min(n, k), replace=False)).astype(np.int64)


# ---------------------------------------------------------------- GPU: the engine against the fp64 oracle
def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def build(arch, ucfg=None):
    """(drop-in model with seeded parameters, oracle config, state_dict)."""
    from mdm_b200 import config as mc
    from mdm_b200.models import NestedUNet, UNet

    cfg = mc.unet_config_from_dict(ucfg or tiny_config(arch))
    cfg.conditioning_feature_dim = tc.LM_DIM
    ocfg = copy.deepcopy(cfg)  # the model constructor mutates conditioning_feature_dim
    model = (UNet if arch == "unet" else NestedUNet)(3, 3, cfg)
    sd = tc.seeded_state_dict(model.state_dict(), PARAM_SEED)
    model.load_state_dict(sd)
    return model, ocfg, sd


def _oracle(ocfg, sd, xs, t, lm, mask, ws, micros, dtype, tf32):
    from oracle import unet_ref

    torch.backends.cuda.matmul.allow_tf32 = bool(tf32)
    torch.backends.cudnn.allow_tf32 = bool(tf32)
    try:
        net = unet_ref.OracleNet(ocfg, tc.LM_DIM)
        P = {k: v.cuda().to(dtype).requires_grad_(True) for k, v in sd.items()}
        xin = [x.cuda().to(dtype) for x in xs]
        mic = {k: v.cuda() for k, v in micros.items()}
        out = net.forward(P, xin if len(xs) > 1 else xin[0], t.cuda(), lm.cuda().to(dtype), mask.cuda().to(dtype), mic)
        outs = list(out) if len(xs) > 1 else [out]
        sum((o * w.cuda().to(dtype)).sum() for o, w in zip(outs, ws)).backward()
        torch.cuda.synchronize()
        return [o.detach().cpu() for o in outs], {k: P[k].grad.detach().cpu() for k in P if P[k].grad is not None}
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False


def run_case(arch, micros, ucfg=None, batch=BATCH, level_batch=None):
    """Forward + backward of loss = sum <out_l, w_l> on the engine, the fp64 oracle and the reference-TF32 arm.
    level_batch: leading rows each level runs (mixed_ratio), outermost first. Returns the errors of the engine and
    of the TF32 arm against fp64: {"out": [(ours, tf32)], "grads": {name: (ours, tf32)}, "absmax": ...}."""
    model, ocfg, sd = build(arch, ucfg)
    x, t, lm, mask = tiny_inputs(arch, batch)
    xs = [x] if arch == "unet" else list(x)
    if level_batch is not None:
        xs = [xi[:b] for xi, b in zip(xs, level_batch)]
    ws = loss_weights(xs)
    o64, g64 = _oracle(ocfg, sd, xs, t, lm, mask, ws, micros, torch.float64, False)
    o32, g32 = _oracle(ocfg, sd, xs, t, lm, mask, ws, micros, torch.float32, True)
    model = model.cuda()
    xin = [xi.cuda() for xi in xs]
    out = model(xin if len(xs) > 1 else xin[0], t.cuda(), lm.cuda(), mask.cuda(), {k: v.cuda() for k, v in micros.items()})
    outs = list(out) if len(xs) > 1 else [out]
    sum((o * w.cuda()).sum() for o, w in zip(outs, ws)).backward()
    torch.cuda.synchronize()
    go = {k: p.grad.detach().cpu() for k, p in model.named_parameters() if p.grad is not None}
    rep = {"out": [(rel(a.cpu(), r), rel(b, r)) for a, b, r in zip(outs, o32, o64)], "grads": {},
           "missing": sorted(k for k in g64 if k not in go)}
    mags = sorted(float(r.abs().max()) for r in g64.values())
    floor = 1e-2 * mags[len(mags) // 2]  # mathematically zero gradients are judged on the scale of real ones
    for k, r in g64.items():
        if k in go:
            d = max(float(r.abs().max()), floor)
            rep["grads"][k] = (float((go[k].double() - r).abs().max()) / d, float((g32[k].double() - r).abs().max()) / d)
    return rep


def assert_calibrated(rep):
    """The bounds of tests/net_cases.assert_calibrated (DESIGN.md section 4), against the reference-TF32 errors of
    the same run."""
    assert not rep["missing"], rep["missing"]
    for ours, tf32 in rep["out"]:
        assert ours <= max(1e-3, 1.75 * tf32), rep["out"]
    t = sorted(v[1] for v in rep["grads"].values())
    o = sorted(v[0] for v in rep["grads"].values())
    med = t[len(t) // 2]
    assert o[len(o) // 2] <= 1.5 * med, (o[len(o) // 2], med)
    bad = {k: v for k, v in rep["grads"].items() if not (v[0] <= 3.5 * max(v[1], med))}
    assert not bad, bad
