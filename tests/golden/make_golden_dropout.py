"""Generate tests/golden/dropout.npz, the fixture of the ResNet dropout (ResNetConfig.dropout), by running the UNMODIFIED
reference (the apple/ml-mdm checkout given by $ML_MDM_ROOT, imported through tests/refharness.py) on CPU in fp32, in
train mode:

    ML_MDM_ROOT=<checkout> python tests/golden/make_golden_dropout.py

Contents (layout, configurations and sample positions: tests/test_dropout_host.py), per architecture (the tiny UNet
with p = 0.1, the tiny nest with p = 0.1 outside and 0.25 inside):
  <arch>.keys / .shapes          state_dict key order and shapes
  <arch>.mask.<ResNet prefix>    the keep mask nn.Dropout drew in that ResNet (NCHW, bit-packed), and its .shape
  <arch>.out<i> / .outmax<i>     each output at a fixed sample of positions, and max|output|
  <arch>.gval / .gmax            for the loss sum(out * w): a fixed sample of each parameter gradient, and max|gradient|
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

import refharness as rh  # noqa: E402
import test_dropout_host as fx  # noqa: E402  (fixture layout shared with the tests)
import tiny_configs as tc  # noqa: E402


def main():
    torch.set_num_threads(16)
    rh.load()
    out = {}
    for arch in fx.ARCHS:
        model, _ = rh.build(fx.tiny_config(arch), {}, arch, tc.LM_DIM)
        model.load_state_dict(tc.seeded_state_dict(model.state_dict(), fx.PARAM_SEED))
        model.train()
        masks = {}

        def record(name):
            def hook(mod, inp, o):
                assert bool((inp[0] != 0).all())  # so that a zero output means a dropped element
                masks[name] = (o != 0).detach().numpy()
            return hook

        for name, mod in model.named_modules():
            if name.endswith(".dropout") and isinstance(mod, torch.nn.Dropout):
                mod.register_forward_hook(record(name[:-len(".dropout")]))
        x, t, lm, mask = fx.tiny_inputs(arch)
        torch.manual_seed(fx.TORCH_SEED)
        o = model(x, t, lm, mask, {})
        o = o if isinstance(o, (list, tuple)) else [o]
        sum((oi * w).sum() for oi, w in zip(o, fx.loss_weights(o))).backward()
        sd = model.state_dict()
        names = [k for k, _ in model.named_parameters()]
        assert names == list(sd), "state_dict holds more than the parameters"
        out[f"{arch}.keys"] = np.array(names)
        out[f"{arch}.shapes"] = np.array(["x".join(str(s) for s in v.shape) for v in sd.values()])
        for name, m in masks.items():
            out[f"{arch}.mask.{name}"] = np.packbits(m.reshape(-1))
            out[f"{arch}.mask.{name}.shape"] = np.array(m.shape)
        for i, oi in enumerate(o):
            flat = oi.detach().reshape(-1).numpy()
            out[f"{arch}.out{i}"] = flat[fx.sample_index(flat.size, i, fx.OUT_SAMPLES)]
            out[f"{arch}.outmax{i}"] = np.float32(np.abs(flat).max())
        gval, gmax = [], []
        for i, (_, p) in enumerate(model.named_parameters()):
            g = p.grad.reshape(-1).numpy()
            gval.append(g[fx.sample_index(g.size, i, fx.GRAD_SAMPLES)])
            gmax.append(np.abs(g).max())
        out[f"{arch}.gval"] = np.concatenate(gval).astype(np.float32)
        out[f"{arch}.gmax"] = np.array(gmax, dtype=np.float32)
        print(arch, [tuple(oi.shape) for oi in o], len(masks), "dropout masks", flush=True)
    np.savez_compressed(fx.GOLD, **out)


if __name__ == "__main__":
    main()
