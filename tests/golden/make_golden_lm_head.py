"""Generate tests/golden/lm_head.npz, the fixture of the lm_head layers (UNetConfig.num_lm_head_layers), by running the
UNMODIFIED reference (the apple/ml-mdm checkout given by $ML_MDM_ROOT, imported through tests/refharness.py) on CPU
in fp32:

    ML_MDM_ROOT=<checkout> python tests/golden/make_golden_lm_head.py

Contents (layout and sample positions: tests/test_lm_head_host.py):
  <tag>.*        the tiny UNet and tiny nest with two lm_head layers at masked_cross_attention 0 and 1: state_dict key
                 order and shapes, each output at a fixed sample of positions with max|output|, and for the loss
                 sum(out * w) max|gradient| and a fixed sample of each parameter gradient
  cc12m_64x64.*  the shipped 64-px UNet at full width (D = 2048, head width 256) with two lm_head layers, B = 1, 77 tokens:
                 key order and shapes, output at a fixed sample of positions with max|output|
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

import refharness as rh  # noqa: E402
import test_lm_head_host as fx  # noqa: E402  (fixture layout shared with the tests)
import tiny_configs as tc  # noqa: E402


def main():
    torch.set_num_threads(16)
    rh.load()
    out = {}
    for tag, arch, masked in fx.TINY:
        model, _ = rh.build(fx.tiny_config(arch, masked), {}, arch, tc.LM_DIM)
        model.load_state_dict(tc.seeded_state_dict(model.state_dict(), fx.PARAM_SEED))
        x, t, lm, mask = fx.tiny_inputs(arch)
        o = model(x, t, lm, mask, {})
        o = o if isinstance(o, (list, tuple)) else [o]
        sum((oi * w).sum() for oi, w in zip(o, fx.loss_weights(o))).backward()
        sd = model.state_dict()
        names = [k for k, _ in model.named_parameters()]
        assert names == list(sd), "state_dict holds more than the parameters"
        out[f"{tag}.keys"] = np.array(names)
        out[f"{tag}.shapes"] = np.array(["x".join(str(s) for s in v.shape) for v in sd.values()])
        for i, oi in enumerate(o):
            flat = oi.detach().reshape(-1).numpy()
            out[f"{tag}.out{i}"] = flat[fx.sample_index(flat.size, i, fx.OUT_SAMPLES)]
            out[f"{tag}.outmax{i}"] = np.float32(np.abs(flat).max())
        gval, gmax = [], []
        for i, (_, p) in enumerate(model.named_parameters()):
            g = p.grad.reshape(-1).numpy()
            gval.append(g[fx.sample_index(g.size, i, fx.GRAD_SAMPLES)])
            gmax.append(np.abs(g).max())
        out[f"{tag}.gval"] = np.concatenate(gval).astype(np.float32)
        out[f"{tag}.gmax"] = np.array(gmax, dtype=np.float32)
        print(tag, [tuple(oi.shape) for oi in o], flush=True)

    cfg = fx.FULL
    y = rh.load_yaml(f"{cfg}.yaml")
    y["unet_config"]["num_lm_head_layers"] = fx.LAYERS
    model, _ = rh.build(y["unet_config"], y["diffusion_config"], "unet", 2048)
    sd = tc.seeded_state_dict(model.state_dict(), fx.FULL_PARAM_SEED)
    model.load_state_dict(sd)
    x, t, lm, mask = fx.full_inputs()
    with torch.no_grad():
        o = model(x, t, lm, mask, {})
    flat = o.reshape(-1).numpy()
    out[f"{cfg}.keys"] = np.array(list(sd))
    out[f"{cfg}.shapes"] = np.array(["x".join(str(s) for s in v.shape) for v in sd.values()])
    out[f"{cfg}.out0"] = flat[fx.sample_index(flat.size, 0, fx.FULL_SAMPLES)]
    out[f"{cfg}.outmax0"] = np.float32(np.abs(flat).max())
    out[f"{cfg}.shape0"] = np.array(o.shape)
    print(cfg, tuple(o.shape), flush=True)
    np.savez_compressed(fx.GOLD, **out)


if __name__ == "__main__":
    main()
