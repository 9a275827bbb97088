"""What running the weight products on the hi fp16 plane only (torch autocast, mdm_net_io.single_plane) changes, in one
run:
  - the card and its power limit;
  - cc12m_64x64 training (get_loss + backward) at batch 64, fp32 against torch.autocast(bf16);
  - the cc12m_1024x1024 nest at batch 4 through trainer.train_batch with FusedAdam, args.fp16 = 0 against 1;
  - DDIM-50 sampling of the cc12m_256x256 nest at batch 16, fp32 against torch.autocast(bf16);
each timed by CUDA events in blocks that alternate the two arms on one pipeline, after warm-up of both (pool sizes,
CUDA graphs of both signatures), and the largest relative difference between the two arms' outputs on the same draws
(the model's predictions for training, the images for sampling).
Usage: python tests/profile_autocast.py [--rounds N] [--steps K] [--only NAME]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from contextlib import nullcontext

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "ml-mdm_b200"))
import bench  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def autocast(on):
    return torch.autocast("cuda", dtype=torch.bfloat16) if on else nullcontext()


def rel(a, b):
    return float((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-30))


def alternate(arms, rounds, steps, per):
    """{arm: [ms per unit, one entry per block]}: blocks of `steps` calls, arms alternating, order flipped per round."""
    times = {a: [] for a in arms}
    order = list(arms)
    for r in range(rounds):
        for a in (order if r % 2 == 0 else order[::-1]):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(steps):
                arms[a]()
            e1.record()
            torch.cuda.synchronize()
            times[a].append(e0.elapsed_time(e1) / (steps * per))
    return times


def summary(times, diff, spread, unit):
    f, h = statistics.median(times["fp32"]), statistics.median(times["autocast"])
    return {f"{unit}_fp32": round(f, 3), f"{unit}_autocast": round(h, 3), "speedup": round(f / h, 4),
            "max_rel_output_diff": diff, "fp32_run_to_run": spread,
            "blocks": {k: [round(t, 3) for t in v] for k, v in times.items()}}


def outputs(pipe, sample, on):
    """The model's predictions of one get_loss on fixed draws."""
    torch.manual_seed(99)
    with torch.no_grad(), autocast(on):
        _, _, _, means, _, _ = pipe.get_loss(sample)
    return means if torch.is_tensor(means) else means[0]


def train_64(args, dev):
    pipe, _ = bench.build_pipeline("cc12m_64x64", dev)
    pipe.train()
    sample = {k: v.to(dev) for k, v in bench.synthetic_host_batch("cc12m_64x64", 64, 1234).items()}
    vm = pipe.get_model().vision_model

    def step(on):
        with autocast(on):
            loss, *_ = pipe.get_loss(sample)
        loss.mean().backward()
        vm.zero_grad(set_to_none=True)
    arms = {"fp32": lambda: step(False), "autocast": lambda: step(True)}
    for _ in range(3):
        for f in arms.values():
            f()
    ref = outputs(pipe, sample, False)
    diff, spread = rel(outputs(pipe, sample, True), ref), rel(outputs(pipe, sample, False), ref)
    return summary(alternate(arms, args.rounds, args.steps, 1), diff, spread, "ms_per_step") | {
        "workload": "cc12m_64x64 training get_loss + backward, batch 64"}


class _Sched:
    def get_last_lr(self):
        return [1e-5]

    def step(self):
        pass


def train_1024(args, dev):
    from mdm_b200 import optim, trainer

    pipe, _ = bench.build_pipeline("cc12m_1024x1024", dev)
    pipe.train()
    sample = {k: v.to(dev) for k, v in bench.synthetic_host_batch("cc12m_1024x1024", 4, 1234).items()}
    opt = optim.FusedAdam(pipe.get_model().vision_model, lr=1e-5)
    ref = outputs(pipe, sample, False)  # before any step moves the weights
    diff, spread = rel(outputs(pipe, sample, True), ref), rel(outputs(pipe, sample, False), ref)

    def step(fp16):
        a = argparse.Namespace(fp16=fp16, gradient_clip_norm=2.0)
        trainer.train_batch(pipe, sample, opt, _Sched(), None, a)
    arms = {"fp32": lambda: step(False), "autocast": lambda: step(True)}
    for _ in range(3):
        for f in arms.values():
            f()
    return summary(alternate(arms, args.rounds, args.steps, 1), diff, spread, "ms_per_step") | {
        "workload": "cc12m_1024x1024 trainer.train_batch (FusedAdam step included), batch 4; fp32 = args.fp16 0, "
                    "autocast = args.fp16 1"}


def ddim_256(args, dev):
    pipe, _ = bench.build_pipeline("cc12m_256x256", dev)
    pipe.eval()
    B, steps = 16, 50
    host = bench.synthetic_host_batch("cc12m_256x256", B, 4321)
    sample = {k: host[k].to(dev) for k in ("lm_outputs", "lm_mask")}
    kw = dict(num_inference_steps=steps, ddim_eta=0.0, resample_steps=True, guidance_scale=1.0)

    def run(on):
        torch.manual_seed(7)
        with autocast(on):
            return pipe.sample(B, sample, 256, dev, **kw)
    imgs = {on: [run(on), run(on)] for on in (False, True)}
    diff, spread = rel(imgs[True][1], imgs[False][1]), rel(imgs[False][0], imgs[False][1])
    arms = {"fp32": lambda: run(False), "autocast": lambda: run(True)}
    return summary(alternate(arms, args.rounds, 1, steps), diff, spread, "ms_per_denoiser_eval") | {
        "workload": f"cc12m_256x256 DDIM-{steps} sampling, batch {B}"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5, help="training steps per timed block")
    ap.add_argument("--only", default=None, choices=["train_64", "train_1024", "ddim_256"])
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    report = {"card": card()}
    for name, fn in (("train_64", train_64), ("train_1024", train_1024), ("ddim_256", ddim_256)):
        if args.only in (None, name):
            report[name] = fn(args, dev)
            print(json.dumps({name: report[name]}), flush=True)
    print(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
