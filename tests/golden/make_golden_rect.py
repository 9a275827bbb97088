"""Generate tests/golden/rect.npz, the fixture of non-square images and of DiffusionConfig.model_output_scale, by
running the UNMODIFIED reference (the apple/ml-mdm checkout given by $ML_MDM_ROOT, imported through
tests/refharness.py) on CPU in fp32:

    ML_MDM_ROOT=<checkout> python tests/golden/make_golden_rect.py

Contents (layout, inputs and sample positions: tests/test_rect_oracle.py):
  u<H>x<W>[_s].*  the tiny UNet through its pipeline (Model.forward, so with model_output_scale when the tag ends in
                  _s): the forward output, Diffusion.get_loss (drawn times, x_t, per-sample loss, the gradient norm of
                  every parameter and conv_out's full gradient after loss.mean().backward()) and a 2-step DDIM sample
  nest.*          the tiny nest at an outer 48x80 (inner 12x20): both outputs and every parameter's gradient norm for the
                  loss sum(out * w)
  cc12m_64x64.*   the shipped 64-px UNet at full width on a 64x96 image: key order and shapes, the output at a fixed
                  sample of positions and max|output|
The reference's nested pipeline (NestedSampler.get_gammas) resizes its gamma maps to a square and cannot run
rectangles, so the nest is pinned at the network level.
"""
import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

import refharness as rh  # noqa: E402
import test_rect_oracle as fx  # noqa: E402  (fixture layout shared with the tests)
import tiny_configs as tc  # noqa: E402


def main():
    torch.set_num_threads(16)
    rh.load()
    out = {}
    for tag, h, w, s in fx.UNET_CASES:
        dcfg = copy.deepcopy(tc.TINY_DIFFUSION)
        dcfg["model_output_scale"] = s
        model, pipe = rh.build(copy.deepcopy(tc.TINY_UNET), dcfg, "unet", tc.LM_DIM)
        model.load_state_dict(tc.seeded_state_dict(model.state_dict(), fx.PARAM_SEED))
        x, t, lm, mask = fx.rect_inputs(3, 2, (h, w), 6)
        with torch.no_grad():
            out[f"{tag}.fwd"] = pipe.model(x, t, lm, mask, {})[0].numpy()
        torch.manual_seed(1234)
        loss, time, x_t, _, _, _ = pipe.get_loss({"images": x.clamp(-1, 1), "lm_outputs": lm, "lm_mask": mask})
        loss.mean().backward()
        out[f"{tag}.loss"] = loss.detach().numpy()
        out[f"{tag}.loss_time"] = time.numpy()
        out[f"{tag}.loss_xt"] = x_t.detach().numpy()
        out[f"{tag}.grad_norms"] = np.array([float(p.grad.norm()) for _, p in model.named_parameters()])
        out[f"{tag}.grad_conv_out"] = model.conv_out.weight.grad.numpy()
        model.zero_grad()
        torch.manual_seed(7)
        noise = torch.randn(2, 3, h, w)
        with torch.no_grad():
            smp = pipe.sampler.sample(pipe.model, noise, lm, mask, {}, num_inference_steps=2, resample_steps=True,
                                      ddim_eta=0.0)
        out[f"{tag}.sample2"] = smp.numpy()
        print(tag, tuple(x.shape), loss.detach().numpy(), flush=True)

    ucfg = copy.deepcopy(tc.TINY_NESTED)
    model, _ = rh.build(ucfg, copy.deepcopy(tc.TINY_NESTED_DIFFUSION), "nested_unet", tc.LM_DIM)
    model.load_state_dict(tc.seeded_state_dict(model.state_dict(), fx.PARAM_SEED))
    xs, t, lm, mask = fx.rect_inputs(3, 2, fx.NEST_HW, 6, nlevels=2)
    o = list(model(xs, t, lm, mask, {}))
    sum((oi * wi).sum() for oi, wi in zip(o, fx.loss_weights(o))).backward()
    for i, oi in enumerate(o):
        out[f"nest.fwd{i}"] = oi.detach().numpy()
    out["nest.grad_norms"] = np.array([float(p.grad.norm()) for _, p in model.named_parameters()])
    print("nest", [tuple(oi.shape) for oi in o], flush=True)

    y = rh.load_yaml(f"{fx.FULL}.yaml")
    model, _ = rh.build(y["unet_config"], y["diffusion_config"], "unet", 2048)
    sd = tc.seeded_state_dict(model.state_dict(), fx.FULL_PARAM_SEED)
    model.load_state_dict(sd)
    x, t, lm, mask = fx.full_inputs()
    with torch.no_grad():
        o = model(x, t, lm, mask, {})
    flat = o.reshape(-1).numpy()
    out[f"{fx.FULL}.keys"] = np.array(list(sd))
    out[f"{fx.FULL}.shapes"] = np.array(["x".join(str(d) for d in v.shape) for v in sd.values()])
    out[f"{fx.FULL}.out"] = flat[fx.sample_index(flat.size, 0, fx.FULL_SAMPLES)]
    out[f"{fx.FULL}.outmax"] = np.float32(np.abs(flat).max())
    out[f"{fx.FULL}.shape"] = np.array(o.shape)
    print(fx.FULL, tuple(o.shape), flush=True)
    np.savez_compressed(os.path.join(HERE, "rect.npz"), **out)


if __name__ == "__main__":
    main()
