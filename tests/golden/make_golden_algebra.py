"""Generate tests/golden/algebra.npz by running the UNMODIFIED reference (the apple/ml-mdm checkout given by
$ML_MDM_ROOT, imported through tests/refharness.py) on CPU in fp32 with the stub denoiser of tests/algebra_cases.py:

    ML_MDM_ROOT=<checkout> python tests/golden/make_golden_algebra.py

  loss/<case>/...   Diffusion / NestedDiffusion.get_loss for every point of algebra_cases.LOSS_GRID: the draws (time,
                    eps per level) and the six returned values (loss, x_t, the returned prediction, target, VDM weights
                    when on), plus the stub-parameter gradients of loss.mean()
  step/<case>/...   Sampler.get_xt_minus_1 (get_prediction_xt_last per level) for every point of STEP_GRID: the noise
                    drawn per level and x0, x_s per level
  clip/<mode>_<s>   Sampler.clip_sample for every threshold mode at image scales 1, 2 and 4
  loop/<case>/...   Sampler.sample for every point of LOOP_GRID: every noise drawn, in order, and the final image

Stub parameters, images, text and step inputs come from seeds (algebra_cases); only draws and outputs are stored.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

import algebra_cases as ac  # noqa: E402
import refharness as rh  # noqa: E402

ref = rh.load()


def pipeline(nest, cfg, seed):
    stub = ac.NestedStub(nest, seed) if nest else ac.Stub(seed)
    cls = ref.diffusion.NestedDiffusionConfig if nest else ref.diffusion.DiffusionConfig
    dcfg = rh.from_dict(cls, cfg)
    return stub, (ref.diffusion.NestedDiffusion if nest else ref.diffusion.Diffusion)(stub, dcfg)


class Recorder:
    """Records every torch.randn_like draw while active."""

    def __enter__(self):
        self.log, self.orig = [], torch.randn_like

        def rec(*a, **k):
            r = self.orig(*a, **k)
            self.log.append(r.clone())
            return r

        torch.randn_like = rec
        return self

    def __exit__(self, *a):
        torch.randn_like = self.orig


def f32(t):
    return t.detach().float().numpy()


def main():
    out = {}
    for case in ac.LOSS_GRID:
        name, nest = case["name"], case["nest"]
        seed = ac.case_seed(name)
        B, side = case.get("B", ac.LOSS_B), ac.loss_side(case)
        stub, pipe = pipeline(nest, ac.loss_config(case), seed)
        lm, mask = ac.text(B, seed)
        torch.manual_seed(seed)
        loss, time, x_t, pred, tgt, w = pipe.get_loss({"images": ac.images(B, side, seed), "lm_outputs": lm,
                                                       "lm_mask": mask})
        loss.mean().backward()
        time_r, eps = ac.replay_loss_draws(B, ac.level_shapes(B, side, nest), 1000, seed, "cpu")
        assert torch.equal(time_r, time)
        p = f"loss/{name}/"
        out[p + "time"] = time.numpy()
        for i, e in enumerate(eps):
            out[p + f"eps{i}"] = f32(e)
        for k, v in (("loss", loss), ("x_t", x_t), ("pred", pred), ("tgt", tgt)):
            out[p + k] = f32(v)
        if w is not None:
            out[p + "weights"] = f32(w)
        for k in "wbkq":
            out[p + "grad_" + k] = f32(getattr(stub, k).grad)
    for name, pname, ptype, eta, thr, gs, t, s in ac.STEP_GRID:
        seed = ac.case_seed(name)
        nest = ac.PIPES[pname][0]
        stub, pipe = pipeline(nest, ac.sampler_config(pname, ptype, thr), seed)
        xs, lm, mask = ac.step_inputs(pname, gs, seed)
        torch.manual_seed(seed)
        with torch.no_grad(), Recorder() as r:
            x0, x_s, _ = pipe.sampler.get_xt_minus_1(pipe.get_model(), torch.tensor(t), xs if nest else xs[0], lm, mask,
                                                     {}, time_step_last=torch.tensor(s), guidance_scale=gs,
                                                     ddim_eta=eta, return_details=True)
        x0, x_s = (x0, x_s) if nest else ([x0], [x_s])
        p = f"step/{name}/"
        for i, z in enumerate(r.log):
            out[p + f"noise{i}"] = f32(z)
        for i, (a, b) in enumerate(zip(x0, x_s)):
            out[p + f"x0_{i}"], out[p + f"xs_{i}"] = f32(a), f32(b)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(3, 3, 8, 8, generator=g) * torch.tensor([0.4, 1.3, 9.0]).view(3, 1, 1, 1)
    for thr in ("NONE", "CLIP", "DYNAMIC", "DYNAMIC_IF"):
        _, pipe = pipeline(None, ac.sampler_config("plain", "V_PREDICTION", thr), 5)
        for sc in (1, 2, 4):
            out[f"clip/{thr}_{sc}"] = f32(pipe.sampler.clip_sample(x, sc))
    for name, pname, ptype, eta, thr, gs, steps in ac.LOOP_GRID:
        seed = ac.case_seed(name)
        nest = ac.PIPES[pname][0]
        stub, pipe = pipeline(nest, ac.sampler_config(pname, ptype, thr), seed)
        xs, lm, mask = ac.loop_inputs(pname, gs, seed)
        torch.manual_seed(seed)
        with torch.no_grad(), Recorder() as r:
            final = pipe.sampler.sample(pipe.get_model(), xs[0], lm, mask, {},
                                        num_inference_steps=steps or 0, ddim_eta=eta, guidance_scale=gs,
                                        resample_steps=steps is not None)
        p = f"loop/{name}/"
        out[p + "final"] = f32(final)
        if r.log:
            out[p + "noise"] = np.concatenate([f32(z).reshape(-1) for z in r.log])
    path = os.path.join(HERE, "algebra.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
