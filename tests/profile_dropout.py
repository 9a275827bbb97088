"""Cost of the ResNet dropout (ResNetConfig.dropout) on the GPU, p = 0 against p = 0.1, in one run:
  - the card and its power limit;
  - the training step (get_loss + backward) of cc12m_64x64 at batch 64 and of the cc12m_256x256 nest at batch 32,
    warmed up, timed by CUDA events in blocks that alternate the two settings (one model alive at a time);
  - the GroupNorm apply and backward kernels of the cc12m_64x64 step at batch 64: device time per step of each kernel
    family, from torch.profiler in separate eager steps (the kernels are internal: no C entry point to time them
    alone), also alternating the two settings.
Usage: python tests/profile_dropout.py [--rounds N] [--steps K]"""
import argparse
import gc
import json
import os
import re
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "ml-mdm_b200"))
import bench  # noqa: E402

CASES = [("cc12m_64x64", 64), ("cc12m_256x256", 32)]
PS = (0.0, 0.1)
GN = re.compile(r"(gn_apply_staged_kernel|gn_apply_kernel|gn_bwd_reduce_staged_kernel|gn_bwd_reduce_kernel|"
                r"gn_bwd_apply_staged_kernel|gn_bwd_apply_kernel|gn_stats_kernel|gn_bwd_finalize_kernel)")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def build(name, p, dev):
    from mdm_b200 import config as mc
    from mdm_b200.diffusion import Diffusion, NestedDiffusion
    from mdm_b200.models import NestedUNet, UNet

    gc.collect()
    torch.cuda.empty_cache()
    ucfg, dcfg, nested = mc.load_yaml_configs(os.path.join(ROOT, "ml-mdm_b200", "mdm_b200", "configs", name + ".yaml"))
    if nested:
        dcfg.mixed_ratio = None  # as bench.py's cc12m_256x256_train
    c = ucfg
    while c is not None:
        c.resnet_config.dropout = p
        c = getattr(c, "inner_config", None)
    torch.manual_seed(4321)
    model = (NestedUNet if nested else UNet)(3, 3, ucfg)
    with torch.no_grad():  # as bench.build_pipeline: no layer left at its zero initialisation
        for q in model.parameters():
            if float(q.detach().abs().max()) == 0:
                q.normal_(0, 0.02)
    pipe = (NestedDiffusion if nested else Diffusion)(model, dcfg).to(dev)
    pipe.train()
    return pipe


def stepper(pipe, sample):
    def step():
        loss, *_ = pipe.get_loss(sample)
        loss.mean().backward()
        pipe.get_model().vision_model.zero_grad(set_to_none=True)
    return step


def time_steps(name, B, rounds, steps, dev):
    sample = {k: v.to(dev) for k, v in bench.synthetic_host_batch(name, B, 1234).items()}
    times = {p: [] for p in PS}
    for _ in range(rounds):
        for p in PS:
            pipe = build(name, p, dev)
            step = stepper(pipe, sample)
            for _ in range(3):
                step()
            torch.cuda.synchronize()
            for _ in range(steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step()
                e1.record()
                torch.cuda.synchronize()
                times[p].append(e0.elapsed_time(e1))
            del pipe, step
    med = {p: sorted(v)[len(v) // 2] for p, v in times.items()}
    return {"batch": B, "rounds": rounds, "steps_per_round": steps,
            "step_ms_median": {f"p={p}": round(v, 2) for p, v in med.items()},
            "step_ms_min": {f"p={p}": round(min(v), 2) for p, v in times.items()},
            "overhead_pct": round(100 * (med[PS[1]] / med[PS[0]] - 1), 2)}


def gn_kernels(name, B, rounds, steps, dev):
    """Device ms per step of each GroupNorm kernel family (summed over its launches), per setting."""
    from torch.profiler import ProfilerActivity, profile

    sample = {k: v.to(dev) for k, v in bench.synthetic_host_batch(name, B, 1234).items()}
    acc = {p: {} for p in PS}
    for _ in range(rounds):
        for p in PS:
            pipe = build(name, p, dev)
            pipe.get_model().vision_model.native().set_graph_mode(False)  # separate kernel records
            step = stepper(pipe, sample)
            for _ in range(2):
                step()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(steps):
                    step()
                torch.cuda.synchronize()
            for ev in prof.key_averages():
                m = GN.search(ev.key)
                if m is None:
                    continue
                us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                d = acc[p].setdefault(m.group(1), [0.0, 0])
                d[0] += us / 1000.0 / (steps * rounds)
                d[1] += ev.count / (steps * rounds)
            del pipe, step
    out = {}
    for p in PS:
        out[f"p={p}"] = {k: {"ms_per_step": round(v[0], 3), "launches_per_step": round(v[1], 1)}
                         for k, v in sorted(acc[p].items())}
        out[f"p={p}"]["total_ms_per_step"] = round(sum(v[0] for v in acc[p].values()), 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=6)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    print(json.dumps({"gn_kernels_cc12m_64x64_b64": gn_kernels("cc12m_64x64", 64, 1, 2, dev)}), flush=True)
    for name, B in CASES:
        print(json.dumps({f"{name}_train_step": time_steps(name, B, a.rounds, a.steps, dev)}), flush=True)


if __name__ == "__main__":
    main()
