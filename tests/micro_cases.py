"""General micro-conditioning (UNetConfig.micro_conditioning with keys other than `scale`): the configurations, inputs
and micro sets shared by the fixture generator (tests/golden/make_golden_micro.py), the host tests
(tests/test_micro_host.py), the GPU tests (tests/test_micro_gpu.py) and tests/profile_micro.py.

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
