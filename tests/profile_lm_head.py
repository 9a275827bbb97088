"""Cost of the lm_head layers (UNetConfig.num_lm_head_layers) on the GPU, in one run:
  - the card and its power limit;
  - the token self-attention operator alone (mdm_op_token_attention_fwd / _bwd) at B = 64, T = 128, D = 2048 (8 heads
    of 256), timed by CUDA events, with algorithmic TFLOP/s (QK^T and PV forward, five products backward);
  - the algorithmic FLOPs of one lm_head layer, from shapes;
  - the cc12m_64x64 training step (get_loss + backward) at batch 64 with num_lm_head_layers 0 and 2, warmed up, then
    timed in alternating blocks.
Usage: python tests/profile_lm_head.py [--rounds N] [--steps K]"""
import argparse
import ctypes as C
import gc
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "ml-mdm_b200"))
import bench  # noqa: E402
from mdm_b200 import _lib  # noqa: E402

B, T, D, HEADS = 64, 128, 2048, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def layer_flops(b, t, d):
    """Forward FLOPs of one SelfAttention1DBlock: qkv (3 D^2), proj_out (D^2), MLP (4 D^2 + 4 D^2) multiply-adds per
    token, plus QK^T and PV (2 T D per token)."""
    linear = 2 * b * t * 12 * d * d
    attention = 4 * b * t * t * d
    return linear, attention


def time_op(iters=50):
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = (torch.randn(B, T, 3 * D, device=dev, generator=g) * 0.7).half()
    dO = (torch.randn(B, T, D, device=dev, generator=g) * 0.5).half()
    o16 = torch.empty(B, T, D, device=dev, dtype=torch.float16)
    stats = torch.empty(B, HEADS, T, 2, device=dev)
    Dterm = torch.empty(B, HEADS, T, device=dev)
    dq32 = torch.empty(B, T, D, device=dev)
    dqkv = torch.empty(B, T, 3 * D, device=dev, dtype=torch.float16)
    lib = _lib.lib()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: C.c_void_p(t.data_ptr())

    def fwd():
        _lib.check(lib.mdm_op_token_attention_fwd(P(qkv), None, B, T, D, HEADS, P(o16), P(stats), st), "fwd")

    def bwd():
        _lib.check(lib.mdm_op_token_attention_bwd(P(qkv), None, P(dO), P(o16), P(stats), B, T, D, HEADS, P(Dterm),
                                                  P(dq32), P(dqkv), st), "bwd")

    out = {}
    flops = {"fwd": 4 * B * T * T * D, "bwd": 10 * B * T * T * D}
    for name, fn in (("fwd", fwd), ("bwd", bwd)):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        out[name] = {"ms": round(ms, 4), "algorithmic_tflops": round(flops[name] / ms / 1e9, 1)}
    return out


def build(layers, dev):
    from mdm_b200 import config as mc
    from mdm_b200.diffusion import Diffusion
    from mdm_b200.models import UNet

    ucfg, dcfg, _ = mc.load_yaml_configs(os.path.join(ROOT, "ml-mdm_b200", "mdm_b200", "configs", "cc12m_64x64.yaml"))
    ucfg.num_lm_head_layers = layers
    torch.manual_seed(4321)
    model = UNet(3, 3, ucfg)
    with torch.no_grad():  # as bench.build_pipeline: no layer left at its zero initialisation
        for p in model.parameters():
            if float(p.detach().abs().max()) == 0:
                p.normal_(0, 0.02)
    return Diffusion(model, dcfg).to(dev)


def time_steps(rounds, steps):
    """Blocks of `steps` timed training steps, 0 and 2 layers alternating, `rounds` blocks each. One model is alive at
    a time (two engines of this size do not fit in 80 GB beside each other); every block is warmed up first."""
    dev = torch.device("cuda", 0)
    sample = {k: v.to(dev) for k, v in bench.synthetic_host_batch("cc12m_64x64", B, 1234).items()}

    def step(pipe):
        pipe.train()
        loss, *_ = pipe.get_loss(sample)
        loss.mean().backward()
        pipe.get_model().vision_model.zero_grad(set_to_none=True)

    times = {0: [], 2: []}
    for _ in range(rounds):
        for n in (0, 2):
            gc.collect()
            torch.cuda.empty_cache()
            pipe = build(n, dev)
            for _ in range(3):
                step(pipe)
            torch.cuda.synchronize()
            for _ in range(steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step(pipe)
                e1.record()
                torch.cuda.synchronize()
                times[n].append(e0.elapsed_time(e1))
            del pipe
    med = {n: sorted(v)[len(v) // 2] for n, v in times.items()}
    return {"batch": B, "tokens": bench.TOKENS, "rounds": rounds, "steps_per_round": steps,
            "step_ms_median": {f"lm_head_{n}": round(v, 2) for n, v in med.items()},
            "step_ms_min": {f"lm_head_{n}": round(min(v), 2) for n, v in times.items()},
            "overhead_2_layers_pct": round(100 * (med[2] / med[0] - 1), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=8)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    print(json.dumps({"card": card()}), flush=True)
    lin, att = layer_flops(B, T, D)
    print(json.dumps({"layer_forward_flops": {"B": B, "T": T, "D": D, "linear_tflop": round(lin / 1e12, 4),
                                              "attention_tflop": round(att / 1e12, 4),
                                              "training_tflop_x3": round(3 * (lin + att) / 1e12, 4)}}), flush=True)
    print(json.dumps({"token_attention_op": {"B": B, "T": T, "D": D, "heads": HEADS, **time_op()}}), flush=True)
    print(json.dumps({"cc12m_64x64_train_step": time_steps(a.rounds, a.steps)}), flush=True)


if __name__ == "__main__":
    main()
