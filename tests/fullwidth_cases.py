"""Full-width parity of the shipped architectures (cc12m_64x64, cc12m_256x256, cc12m_1024x1024), forward AND
backward, on the GPU, with the reference's own GPU arithmetic measured beside it.

Three implementations of the same step (same parameters, same inputs, loss = sum_l <out_l, w_l>):
  ours   the native engine (fp16 operands, fp32 accumulation)
  f64    the oracle (oracle/unet_ref.py, plain functional torch) in float64 on the same GPU -- the arbiter
  tf32   the oracle in float32 on the GPU with torch.backends.{cuda.matmul,cudnn}.allow_tf32 = True, i.e. the
         arithmetic the reference itself trains with (clis/train_parallel.py:18-19); its distance from f64 is the
         calibration: what "matches the reference PyTorch path" can mean on this hardware
Errors are max|a - f64| / max|f64| per tensor (outputs per level, every parameter gradient).

Used by tests/test_fullwidth_gpu.py; runnable as a script:  python tests/fullwidth_cases.py [config ...]
writes gpurun_out/parity_fullwidth_<config>.txt"""
import copy
import os
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.join(HERE, ".."), os.path.join(HERE, "..", "ml-mdm_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import parity  # noqa: E402
from mdm_b200 import config as mc  # noqa: E402
from mdm_b200.models import NestedUNet, UNet  # noqa: E402
from oracle import unet_ref  # noqa: E402

RES = {"cc12m_64x64": [64], "cc12m_256x256": [256, 64], "cc12m_1024x1024": [1024, 256, 64]}
CFG_DIR = os.path.join(HERE, "..", "ml-mdm_b200", "mdm_b200", "configs")


def build(name, seed=0, edit=None):
    """(the model of configs/<name>.yaml, its config for the oracle). edit(config), when given, changes the loaded
    config before the model is built, e.g. to add lm_head layers or dropout."""
    ucfg, _, nested = mc.load_yaml_configs(os.path.join(CFG_DIR, name + ".yaml"))
    if edit is not None:
        edit(ucfg)
    ocfg = copy.deepcopy(ucfg)
    torch.manual_seed(seed)
    m = (NestedUNet if nested else UNet)(3, 3, ucfg)
    with torch.no_grad():  # the reference zero-initialises ~1/3 of its layers; a trained net has none at zero
        for p in m.parameters():
            if float(p.abs().max()) == 0:
                p.normal_(0, 0.02)
    return m, ocfg


def inputs(name, B, S, seed=1, ragged=True, micro=False):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(B, 3, r, r, generator=g) for r in RES[name]]
    t = torch.randint(0, 1000, (B,), generator=g)
    lm = torch.randn(B, S, 2048, generator=g)
    mask = torch.ones(B, S)
    if ragged and S > 2:  # padded captions: masked pooling (and masked cross-attention where configured)
        for b in range(B):
            n = max(1, S - 1 - (b % 3))
            mask[b, n:] = 0
        lm = lm * mask.unsqueeze(-1)  # language_models/factory.py:101
    ws = [torch.randn(x.shape, generator=g) for x in xs]
    micros = {}
    if micro:  # explicit micro-conditioning: some below the level default (passes through), some above (clamped)
        micros = {"scale": torch.tensor([48.0, 700.0, 2000.0, 64.0][:B] + [256.0] * max(0, B - 4))}
    return xs, t, lm, mask, ws, micros


def run_case(name, m, oracle, B=1, S=8, micro=False, micros=None, verbose=False):
    """The engine `m`, `oracle` in float64 and the oracle in float32 with TF32 on, all on the GPU, with inputs(name, B,
    S, micro=micro) (micros, when given, in place of its micro-conditioning values). Returns parity.report(...,
    floor=False) with "seconds" per arm and the extras of parity.assert_calibrated_full_width."""
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    xs, t, lm, mask, ws, mic = inputs(name, B, S, micro=micro)
    args = (sd, xs, t, lm, mask, mic if micros is None else micros, ws)
    tm = {}
    t0 = time.time()
    o64, g64 = parity.oracle_arm(oracle.forward, *args, torch.float64, "cuda")
    tm["f64"] = time.time() - t0
    t0 = time.time()
    o32, g32 = parity.oracle_arm(oracle.forward, *args, torch.float32, "cuda", tf32=True)
    tm["tf32"] = time.time() - t0
    t0 = time.time()
    oo, go = parity.engine_arm(m, xs, *args[2:])
    tm["ours"] = time.time() - t0
    rep = parity.report((oo, go), (o64, g64), (o32, g32), floor=False)
    rep["seconds"] = tm
    rep["grad_absmax"] = {k: float(go[k].abs().max()) for k in go}
    rep["grad_absmax_tf32"] = {k: float(g32[k].abs().max()) for k in g32}
    mags = sorted(float(r.abs().max()) for r in g64.values())
    rep["grad_typical"] = mags[len(mags) // 2]  # median over parameters of max|d loss / d parameter|
    if verbose:
        print(f"== {name} B={B} S={S} micro={micro}: seconds {tm}")
        for i, (a, b) in enumerate(rep["out"]):
            print(f"   out[{i}]  ours {a:.3e}   reference-tf32 {b:.3e}")
        defined = parity.defined_grads(rep["grads"])
        print(f"   numerically undefined gradients (reference-tf32 error > 0.5, mathematically zero): "
              f"{sorted(k for k in rep['grads'] if k not in defined)}")
        ge = sorted(defined.items(), key=lambda kv: -kv[1][0])
        ours = sorted(v[0] for v in defined.values())
        ref = sorted(v[1] for v in defined.values())
        n = len(ours)
        print(f"   {n} parameter gradients: ours median {ours[n // 2]:.3e} p90 {ours[int(.9 * n)]:.3e} max {ours[-1]:.3e} | "
              f"reference-tf32 median {ref[n // 2]:.3e} p90 {ref[int(.9 * n)]:.3e} max {ref[-1]:.3e}")
        print("   worst (ours, tf32):")
        for k, (a, b) in ge[:12]:
            print(f"      {a:.3e} {b:.3e}  {k}")
        over = [(k, a, b) for k, (a, b) in ge if a > 2.0 * max(b, 1e-3)]
        print(f"   gradients with ours > 2 x max(tf32, 1e-3): {len(over)}")
        for k, a, b in over[:20]:
            print(f"      {a:.3e} {b:.3e}  {k}")
        print(f"   missing gradients: {rep['missing']}")
    return rep


if __name__ == "__main__":
    names = [a for a in sys.argv[1:] if a in RES] or list(RES)
    os.makedirs(os.path.join(HERE, "..", "gpurun_out"), exist_ok=True)
    for nm in names:
        import contextlib
        import io

        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            m, ocfg = build(nm)
            run_case(nm, m, unet_ref.OracleNet(ocfg, 2048), B=2 if nm != "cc12m_1024x1024" else 1, S=8, micro=True,
                     verbose=True)
        print(buf.getvalue(), flush=True)
        with open(os.path.join(HERE, "..", "gpurun_out", f"parity_fullwidth_{nm}.txt"), "w") as f:
            f.write(buf.getvalue())
