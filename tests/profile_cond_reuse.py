"""What encoding the text once per sampling run saves, in one run:
  - the card and its power limit;
  - DDIM-50 sampling of the cc12m_256x256 nest at batch 16 (bench.py's cc12m_256x256_ddim50 workload), with
    num_lm_head_layers 0 and 2: the sampler as shipped (forward_conditioning once, then forward_denoising with the
    engine's K/V cache) against the same sampler calling the model's forward at every step, timed by CUDA events in
    runs that alternate the two arms;
  - the largest relative difference between the images the two arms produce.
Usage: python tests/profile_cond_reuse.py [--rounds N] [--batch B]"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "ml-mdm_b200"))
import bench  # noqa: E402

STEPS = 50


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def build(layers, dev):
    from mdm_b200 import config as mc
    from mdm_b200.diffusion import NestedDiffusion
    from mdm_b200.models import NestedUNet

    gc.collect()
    torch.cuda.empty_cache()
    ucfg, dcfg, _ = mc.load_yaml_configs(os.path.join(ROOT, "ml-mdm_b200", "mdm_b200", "configs", "cc12m_256x256.yaml"))
    c = ucfg
    while getattr(c, "inner_config", None) is not None:
        c = c.inner_config
    c.num_lm_head_layers = layers
    torch.manual_seed(4321)
    model = NestedUNet(3, 3, ucfg)
    with torch.no_grad():
        for p in model.parameters():
            if float(p.detach().abs().max()) == 0:
                p.normal_(0, 0.02)
    pipe = NestedDiffusion(model, dcfg).to(dev)
    pipe.eval()
    return pipe


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--layers", default="0,2", help="num_lm_head_layers settings to run")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    B, R = args.batch, 256
    host = bench.synthetic_host_batch("cc12m_256x256", B, 4321)
    sample = {k: host[k].to(dev) for k in ("lm_outputs", "lm_mask")}
    kw = dict(num_inference_steps=STEPS, ddim_eta=0.0, resample_steps=True, guidance_scale=1.0)
    report = {"card": card(), "workload": f"cc12m_256x256 DDIM-{STEPS}, batch {B}, {sample['lm_outputs'].shape[1]} tokens"}
    for layers in (int(v) for v in args.layers.split(",")):
        pipe = build(layers, dev)
        sampler = pipe.sampler

        def run(reuse):
            if not reuse:
                sampler._encode_text = lambda *a: None  # model(...) at every step, as before the split
            torch.manual_seed(7)
            try:
                return pipe.sample(B, sample, R, dev, **kw)
            finally:
                if not reuse:
                    del sampler._encode_text

        imgs = {}
        for reuse in (True, False):  # warm-up: pool sizes, sampler tables, CUDA graphs of every signature
            run(reuse)
            imgs[reuse] = run(reuse)
        times = {True: [], False: []}
        for r in range(args.rounds):
            for reuse in ((True, False) if r % 2 == 0 else (False, True)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                run(reuse)
                b.record()
                torch.cuda.synchronize()
                times[reuse].append(a.elapsed_time(b) / STEPS)
        diff = float((imgs[True] - imgs[False]).abs().max() / imgs[False].abs().max().clamp_min(1e-30))
        m_re, m_per = statistics.median(times[True]), statistics.median(times[False])
        report[f"lm_head_layers_{layers}"] = {
            "ms_per_eval_reuse": round(m_re, 3), "ms_per_eval_per_step": round(m_per, 3),
            "saving_pct": round(100 * (1 - m_re / m_per), 2), "image_max_rel_diff": diff,
            "runs": {"reuse": [round(t, 3) for t in times[True]], "per_step": [round(t, 3) for t in times[False]]}}
        print(json.dumps({layers: report[f"lm_head_layers_{layers}"]}), flush=True)
        del pipe, sampler
    print(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
