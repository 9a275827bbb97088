"""What DPM-Solver++ multistep sampling costs and buys, in one run:
  - the card and its power limit;
  - mdm_sampler_multistep (second-order SDE step: reads x_t, pred, x0_prev, noise; writes x0, x_s) against
    mdm_sampler_step (DDIM) per level size, CUDA events over many launches, and the multistep kernel's achieved
    bytes/s from its 4 reads + 2 writes of fp32;
  - wall time per sampling run of the cc12m_256x256 nest at batch 16, guidance 7.5: DDIM-250, DDIM-50, dpmpp_2m-25 and
    dpmpp_2m_sde-25, in rounds that alternate the arms (random weights: times only, no image quality);
  - the endpoint error against step count of DDIM and dpmpp_2m on the analytic two-component mixture at 256x256
    (fp64 oracle, tests/multistep_oracle.py), against the exact flow through the shared final step.
Usage: python tests/profile_multistep.py [--rounds N] [--batch B] [--out DIR]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE, os.path.join(ROOT, "ml-mdm_b200")):
    sys.path.insert(0, p)
import bench  # noqa: E402
import multistep_oracle as mo  # noqa: E402
from oracle import diffusion_ref as dref  # noqa: E402

ARMS = [("ddim_250", dict(num_inference_steps=250, ddim_eta=0.0)), ("ddim_50", dict(num_inference_steps=50, ddim_eta=0.0)),
        ("dpmpp_2m_25", dict(num_inference_steps=25, solver="dpmpp_2m")),
        ("dpmpp_2m_sde_25", dict(num_inference_steps=25, solver="dpmpp_2m_sde"))]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def kernel_times_pure(B, iters=200):
    """The two entry points alone (no tensor allocation, no randn): what the kernels take."""
    import ctypes as C

    from mdm_b200 import _lib
    from mdm_b200 import samplers

    p, st = samplers._ptr, samplers._stream
    tab = torch.tensor(dref.gammas_f32("DEEPFLOYD", 1000)).cuda()
    out = {}
    for side in (64, 256, 1024):
        x = torch.randn(B, 3, side, side, device="cuda")
        pred, x0p, z, x0, xs = (torch.randn_like(x) for _ in range(5))
        n = x.numel()

        def multistep():
            _lib.check(_lib.lib().mdm_sampler_multistep(p(x), p(pred), p(x0p), p(z), p(tab), 500, 5, 1, None,
                                                        C.c_float(1.0), C.c_float(0.9), C.c_float(0.1),
                                                        C.c_float(-0.05), C.c_float(0.2), p(x0), p(xs), B,
                                                        C.c_int64(n // B), st()))

        def step():
            _lib.check(_lib.lib().mdm_sampler_step(p(x), p(pred), None, p(tab), 500, 480, 5, 1, C.c_float(1.0), 1,
                                                   C.c_float(0.0), 0, p(x0), p(xs), C.c_int64(n), st()))

        res = {}
        for name, f in (("multistep", multistep), ("sampler_step", step)):
            for _ in range(10):
                f()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                f()
            b.record()
            torch.cuda.synchronize()
            res[name] = a.elapsed_time(b) / iters
        out[f"{B}x3x{side}x{side}"] = {
            "multistep_us": round(res["multistep"] * 1e3, 2), "sampler_step_us": round(res["sampler_step"] * 1e3, 2),
            "multistep_GBps_4R2W": round(6 * n * 4 / (res["multistep"] * 1e-3) / 1e9, 1),
            "sampler_step_GBps_2R2W": round(4 * n * 4 / (res["sampler_step"] * 1e-3) / 1e9, 1)}
    return out


def sampling_times(B, rounds):
    dev = torch.device("cuda:0")
    pipe, _ = bench.build_pipeline("cc12m_256x256", dev)
    pipe.eval()
    host = bench.synthetic_host_batch("cc12m_256x256", B, 4321)
    lm = host["lm_outputs"].to(dev)
    sample = {"lm_outputs": torch.cat([torch.zeros_like(lm), lm]),
              "lm_mask": torch.cat([host["lm_mask"]] * 2).to(dev)}

    def run(kw):
        torch.manual_seed(7)
        return pipe.sample(B, sample, 256, dev, resample_steps=True, guidance_scale=7.5, **kw)

    for _, kw in ARMS:  # warm-up: pool sizes, tables, the engine's buffers of every signature
        run(kw)
    times = {n: [] for n, _ in ARMS}
    for r in range(rounds):
        for name, kw in (ARMS if r % 2 == 0 else ARMS[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            run(kw)
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b))
    out = {}
    for name, kw in ARMS:
        m = statistics.median(times[name])
        out[name] = {"ms_per_run": round(m, 1), "evaluations": kw["num_inference_steps"],
                     "ms_per_evaluation": round(m / kw["num_inference_steps"], 2),
                     "runs_ms": [round(t, 1) for t in times[name]]}
    return out


def endpoint_errors(side=256, counts=(10, 15, 20, 25, 50, 100, 250)):
    den = mo.mixture_case((3, side, side), 3)
    x_T = torch.randn(1, 3, side, side, generator=torch.Generator().manual_seed(4)).double()
    tab = mo.table("DEEPFLOYD")
    out = {}
    for n in counts:
        ts = dref.set_timesteps(1000, n)
        exact = mo.exact_endpoint(den, x_T, tab, ts)
        out[n] = {s: mo.rms(mo.sample_loop(den, x_T, tab, ts, s, dref.V_PREDICTION), exact)
                  for s in ("ddim", "dpmpp_2m")}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--out", default=None, help="directory for profile_multistep.json")
    ap.add_argument("--skip-sampling", action="store_true")
    args = ap.parse_args()
    report = {"card": card(), "kernels": kernel_times_pure(args.batch)}
    print(json.dumps(report), flush=True)
    if not args.skip_sampling:
        report["sampling_cc12m_256x256_b%d_cfg7.5" % args.batch] = sampling_times(args.batch, args.rounds)
        print(json.dumps(report), flush=True)
    report["endpoint_rms_mixture_256_deepfloyd"] = endpoint_errors()
    print(json.dumps(report, indent=1), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "profile_multistep.json"), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
