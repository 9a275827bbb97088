"""Parity of the native (nested) U-Net against the oracle on tiny configs: forward, intermediate
activations and every parameter gradient.  Used by tests/test_net_gpu.py; runnable as a script."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "ml-mdm_b200"))

import parity  # noqa: E402
import tiny_configs as tc  # noqa: E402
from parity import assert_calibrated  # noqa: E402,F401  (the bounds run_case's report is held to)


def run_case(kind, built=None, inputs=None, acts=True, verbose=True):
    """Forward + backward of loss = sum_l <out_l, w_l> on the engine, the fp64 oracle (CPU) and the reference-TF32 arm
    (the oracle in fp32 on the GPU with TF32 on): parity.report, and with acts the error of every residual-stream
    activation the fp64 oracle traces ("acts"). built: (model, oracle, state_dict), by default parity.tiny_model of
    the kind's tiny config; inputs: (x, t, lm, mask), by default tc.seeded_inputs(3, ...) at batch 2 and 6 tokens."""
    nlev = 1 if kind == "unet" else 2
    model, oracle, sd = built or parity.tiny_model(tc.TINY[kind])
    x, t, lm, mask = inputs or tc.seeded_inputs(3, 2, 16 if kind == "unet" else 32, 6, nlevels=nlev)
    xs = [x] if nlev == 1 else x
    g = torch.Generator().manual_seed(11)
    ws = [torch.randn(xi.shape, generator=g) for xi in xs]
    trace = {}
    f64 = parity.oracle_arm(oracle.forward, sd, xs, t, lm, mask, {}, ws, torch.float64, "cpu", trace=trace)
    ours = parity.engine_arm(model, xs, t, lm, mask, {}, ws)
    tf32 = parity.oracle_arm(oracle.forward, sd, xs, t, lm, mask, {}, ws, torch.float32, "cuda", tf32=True)
    report = parity.report(ours, f64, tf32)
    if acts:
        report["acts"] = {}
        for name, ref in trace.items():
            try:
                b, c, h, w = ref.shape
                got = model.native().debug_fetch(name, (b, h, w, c)).permute(0, 3, 1, 2)
                report["acts"][name] = parity.rel(got.cpu(), ref.detach())
            except Exception as e:  # intermediates are released in inference mode only; report and go on
                report["acts"][name] = str(e)
    if verbose:
        grads = report["grads"]
        print(f"== {kind}: out rel err (ours, reference-tf32) {report['out']}")
        og = sorted(v[0] for v in grads.values())
        tg = sorted(v[1] for v in grads.values())
        print(f"   grads: ours median {og[len(og) // 2]:.2e} max {og[-1]:.2e} | reference-tf32 median {tg[len(tg) // 2]:.2e} "
              f"max {tg[-1]:.2e}")
        bad_a = {k: v for k, v in report.get("acts", {}).items() if isinstance(v, str) or v > 2e-3}
        print(f"   activations checked: {len(report.get('acts', {}))}, above 2e-3: {bad_a}")
        worst = sorted(grads.items(), key=lambda kv: -(kv[1][0] if kv[1][0] == kv[1][0] else 1e9))[:12]
        print("   worst grads (ours, reference-tf32):", [(k, f"{a:.2e}", f"{b:.2e}") for k, (a, b) in worst])
        print(f"   grads above 5e-3: {sum(1 for v in og if not (v <= 5e-3))} / {len(og)}")
        print(f"   missing gradients: {report['missing']}")
        print("   pool bytes (reserved, high-water):", model.native().workspace_bytes())
    return report


if __name__ == "__main__":
    kinds = sys.argv[1:] or ["unet", "nested"]
    ok = True
    for k in kinds:
        r = run_case(k)
        try:
            assert_calibrated(r)
        except AssertionError as e:
            print("   NOT within the calibrated bounds:", str(e)[:300])
            ok = False
    print("RESULT", "PASS" if ok else "FAIL")
    sys.exit(0 if ok else 1)
