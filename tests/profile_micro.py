"""Cost of one extra micro-conditioning key on the GPU: cc12m_64x64 with "scale:64" against "scale:64,watermark_score:0",
in one run:
  - the card and its power limit;
  - the training step (get_loss + backward) at batch 64;
  - DDIM sampling, 50 steps, batch 16, guidance 1;
each warmed up and timed by CUDA events, in blocks that alternate the two settings (one model alive at a time).
Usage: python tests/profile_micro.py [--rounds N] [--steps K]"""
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

NAME = "cc12m_64x64"
SETTINGS = ("scale:64", "scale:64,watermark_score:0")


def build(micro, dev):
    from mdm_b200 import config as mc
    from mdm_b200.diffusion import Diffusion
    from mdm_b200.models import UNet

    gc.collect()
    torch.cuda.empty_cache()
    ucfg, dcfg, _ = mc.load_yaml_configs(os.path.join(ROOT, "ml-mdm_b200", "mdm_b200", "configs", NAME + ".yaml"))
    ucfg.micro_conditioning = micro
    torch.manual_seed(4321)
    model = UNet(3, 3, ucfg)
    with torch.no_grad():  # as bench.build_pipeline: no layer left at its zero initialisation
        for q in model.parameters():
            if float(q.detach().abs().max()) == 0:
                q.normal_(0, 0.02)
    return Diffusion(model, dcfg).to(dev)


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


def measure(kind, B, rounds, n, dev):
    host = bench.synthetic_host_batch(NAME, B, 1234)
    sample = {k: v.to(dev) for k, v in host.items()}
    g = torch.Generator().manual_seed(5)
    sample["scale"] = torch.full((B,), 64.0, device=dev)
    sample["watermark_score"] = torch.rand(B, generator=g).to(dev)
    times = {s: [] for s in SETTINGS}
    for _ in range(rounds):
        for s in SETTINGS:
            pipe = build(s, dev)
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
                        pipe.sample(B, sample, bench.RES[NAME][0], dev, num_inference_steps=50, ddim_eta=0.0,
                                    resample_steps=True, guidance_scale=1.0)
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            times[s] += timed(fn, n)
            del pipe, fn
    med = {s: sorted(v)[len(v) // 2] for s, v in times.items()}
    return {"batch": B, "rounds": rounds, "per_round": n,
            "ms_median": {s: round(v, 3) for s, v in med.items()},
            "ms_min": {s: round(min(v), 3) for s, v in times.items()},
            "overhead_pct": round(100 * (med[SETTINGS[1]] / med[SETTINGS[0]] - 1), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=8)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": profile_dropout.card()}), flush=True)
    print(json.dumps({f"{NAME}_train_step_b64": measure("train", 64, a.rounds, a.steps, dev)}), flush=True)
    print(json.dumps({f"{NAME}_ddim50_b16": measure("sample", 16, a.rounds, max(2, a.steps // 4), dev)}), flush=True)


if __name__ == "__main__":
    main()
