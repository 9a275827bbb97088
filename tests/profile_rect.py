"""Cost of non-square images and of model_output_scale on the GPU, in one run:
  - the card and its power limit;
  - the cc12m_64x64 training step (get_loss + backward) at batch 64 on 64x64, 64x96 and 96x64 images: ms per step and
    ms per megapixel of the batch (64x96 has 1.5x the pixels of 64x64);
  - model_output_scale 0 against 0.1: the cc12m_64x64 training step at batch 64 and DDIM-50 at batch 16 (Model applies
    the scale), and the same on the 2-level 256 nest at batch 32 / 8 (NestedModel accepts the setting and ignores it,
    as the reference does, so the two settings run the same work);
each warmed up and timed by CUDA events, in blocks that alternate the settings (one model alive at a time).
Usage: python tests/profile_rect.py [--rounds N] [--steps K]"""
import argparse
import gc
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "ml-mdm_b200"))
import bench  # noqa: E402
import profile_dropout  # noqa: E402


def build(name, scale, dev):
    from mdm_b200 import config as mc
    from mdm_b200.diffusion import Diffusion, NestedDiffusion
    from mdm_b200.models import NestedUNet, UNet

    gc.collect()
    torch.cuda.empty_cache()
    ucfg, dcfg, nested = mc.load_yaml_configs(os.path.join(ROOT, "ml-mdm_b200", "mdm_b200", "configs", name + ".yaml"))
    dcfg.model_output_scale = scale
    torch.manual_seed(4321)
    model = (NestedUNet if nested else UNet)(3, 3, ucfg)
    with torch.no_grad():  # as bench.build_pipeline: no layer left at its zero initialisation
        for q in model.parameters():
            if float(q.detach().abs().max()) == 0:
                q.normal_(0, 0.02)
    return (NestedDiffusion if nested else Diffusion)(model, dcfg).to(dev)


def timed(fn, n):
    out = []
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def batch(name, B, hw, dev):
    host = bench.synthetic_host_batch(name, B, 1234)
    g = torch.Generator().manual_seed(9)
    return {"images": (torch.rand(B, 3, *hw, generator=g) * 2 - 1).to(dev),
            "lm_outputs": host["lm_outputs"].to(dev), "lm_mask": host["lm_mask"].to(dev)}


def measure(name, kind, B, settings, rounds, n, dev):
    """settings: list of (label, (H, W), model_output_scale)."""
    times = {lab: [] for lab, _, _ in settings}
    for _ in range(rounds):
        for lab, hw, scale in settings:
            pipe = build(name, scale, dev)
            sample = batch(name, B, hw, dev)
            if kind == "train":
                pipe.train()

                def fn():
                    loss, *_ = pipe.get_loss(sample)
                    loss.mean().backward()
                    pipe.get_model().vision_model.zero_grad(set_to_none=True)
            else:
                pipe.eval()

                def fn():
                    with torch.no_grad():
                        pipe.sample(B, sample, hw[0], dev, num_inference_steps=50, ddim_eta=0.0, resample_steps=True,
                                    guidance_scale=1.0)
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            times[lab] += timed(fn, n)
            del pipe, fn, sample
    res = {"batch": B, "rounds": rounds, "per_round": n}
    for lab, hw, _ in settings:
        v = sorted(times[lab])
        med = v[len(v) // 2]
        res[lab] = {"ms_median": round(med, 3), "ms_min": round(v[0], 3), "ms_max": round(v[-1], 3)}
        if kind == "train":
            res[lab]["ms_per_megapixel"] = round(med / (B * hw[0] * hw[1] / 1e6), 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=8)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": profile_dropout.card()}), flush=True)
    rect = [("64x64", (64, 64), 0.0), ("64x96", (64, 96), 0.0), ("96x64", (96, 64), 0.0)]
    print(json.dumps({"cc12m_64x64_train_b64": measure("cc12m_64x64", "train", 64, rect, a.rounds, a.steps, dev)}),
          flush=True)
    for name, sq, bt, bs in (("cc12m_64x64", 64, 64, 16), ("cc12m_256x256", 256, 32, 8)):
        sc = [("s=0", (sq, sq), 0.0), ("s=0.1", (sq, sq), 0.1)]
        print(json.dumps({f"{name}_train_b{bt}": measure(name, "train", bt, sc, a.rounds, a.steps, dev)}), flush=True)
        print(json.dumps({f"{name}_ddim50_b{bs}": measure(name, "sample", bs, sc, a.rounds, max(2, a.steps // 4), dev)}),
              flush=True)


if __name__ == "__main__":
    main()
