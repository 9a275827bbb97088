"""Generate tests/golden/micro.npz, the fixture of general micro-conditioning (UNetConfig.micro_conditioning with keys
other than `scale`), by running the UNMODIFIED reference (the apple/ml-mdm checkout given by $ML_MDM_ROOT, imported
through tests/refharness.py) on CPU in fp32:

    ML_MDM_ROOT=<checkout> python tests/golden/make_golden_micro.py

Contents (configurations, inputs, micro sets and sample positions: tests/micro_cases.py), per architecture:
  <arch>.keys / .shapes                  state_dict key order and shapes
and per architecture and micro set (all / wm / none), for the loss sum(out * w):
  <arch>.<set>.out<i> / .outmax<i>       each output at a fixed sample of positions, and max|output|
  <arch>.<set>.gval / .gmax              a fixed sample of each parameter gradient, and max|gradient|
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

import micro_cases as mx  # noqa: E402
import refharness as rh  # noqa: E402
import tiny_configs as tc  # noqa: E402


def main():
    torch.set_num_threads(16)
    rh.load()
    out = {}
    for arch in mx.ARCHS:
        model, _ = rh.build(mx.tiny_config(arch), {}, arch, tc.LM_DIM)
        # every tensor redrawn, the zero-initialised cond_layers.<key>.1 included
        model.load_state_dict(tc.seeded_state_dict(model.state_dict(), mx.PARAM_SEED))
        model.eval()
        sd = model.state_dict()
        names = [k for k, _ in model.named_parameters()]
        assert names == list(sd), "state_dict holds more than the parameters"
        out[f"{arch}.keys"] = np.array(names)
        out[f"{arch}.shapes"] = np.array(["x".join(str(s) for s in v.shape) for v in sd.values()])
        x, t, lm, mask = mx.tiny_inputs(arch)
        for which in mx.MICRO_SETS:
            model.zero_grad(set_to_none=True)
            o = model(x, t, lm, mask, mx.micro_set(arch, which))
            o = o if isinstance(o, (list, tuple)) else [o]
            sum((oi * w).sum() for oi, w in zip(o, mx.loss_weights(o))).backward()
            tag = f"{arch}.{which}"
            for i, oi in enumerate(o):
                flat = oi.detach().reshape(-1).numpy()
                out[f"{tag}.out{i}"] = flat[mx.sample_index(flat.size, i, mx.OUT_SAMPLES)]
                out[f"{tag}.outmax{i}"] = np.float32(np.abs(flat).max())
            gval, gmax = [], []
            for i, (_, p) in enumerate(model.named_parameters()):
                g = p.grad.reshape(-1).numpy()
                gval.append(g[mx.sample_index(g.size, i, mx.GRAD_SAMPLES)])
                gmax.append(np.abs(g).max())
            out[f"{tag}.gval"] = np.concatenate(gval).astype(np.float32)
            out[f"{tag}.gmax"] = np.array(gmax, dtype=np.float32)
            print(tag, [tuple(oi.shape) for oi in o], flush=True)
    np.savez_compressed(mx.GOLD, **out)


if __name__ == "__main__":
    main()
