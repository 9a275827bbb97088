"""The native denoiser under torch autocast (mdm_net_io.single_plane): a call that torch runs inside an active CUDA
autocast region multiplies the weights' hi fp16 plane only, and every other call runs as before.

- accuracy: engine under autocast against the fp64 oracle, bounded by the error of the reference's own autocast
  arithmetic (the oracle in fp32 under the same torch.autocast, same run, same metric), for bf16 and fp16;
- the path: the GEMM profile's planes column of an autocast forward and backward, and of an fp32 call;
- nothing else changed: a net that ran single-plane passes and then had its weights updated in place computes what a
  net that never saw autocast computes (the stale lo planes are refilled), eagerly and with graph replay;
- graphs alternating between the modes, the K/V cache across a mode change, DDIM sampling with the text encoded once,
  and train_batch with args.fp16.

Forward outputs are compared to 1e-6 relative (plus ten times the spread of two runs of the same call): GroupNorm
statistics are summed by fp32 atomics, so two runs of one forward can differ in the last bits, while a pass that read a
stale or missing lo plane is off by more than 1e-5 (asserted). Gradients: the run-to-run bound of tests/parity.py
(weight-gradient split-K and attention dQ accumulate with fp32 atomics)."""
import argparse
import copy
import csv
import ctypes as C
import os
import sys
import tempfile

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.join(HERE, ".."), os.path.join(HERE, "..", "ml-mdm_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import lm_head_oracle  # noqa: E402
import micro_cases as mcases  # noqa: E402
import parity  # noqa: E402
import tiny_configs as tc  # noqa: E402
from mdm_b200 import _lib, optim, trainer  # noqa: E402
from mdm_b200 import config as mc  # noqa: E402
from mdm_b200.diffusion import NestedDiffusion, NestedModel  # noqa: E402
from mdm_b200.samplers import NestedSampler  # noqa: E402

pytestmark = pytest.mark.gpu

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


def ucfg_of(kind):
    """The tiny UNet, or the tiny 2-level nest with two lm_head layers and micro-conditioning keys at both levels."""
    if kind == "unet":
        return copy.deepcopy(tc.TINY_UNET)
    u = mcases.tiny_config("nested_unet")
    u["inner_config"]["num_lm_head_layers"] = 2
    return u


def build(kind):
    return parity.tiny_model(ucfg_of(kind), lm_head_oracle.OracleNet)


def inputs(kind, batch=2):
    nested = kind != "unet"
    x, t, lm, mask = tc.seeded_inputs(3, batch, 32 if nested else 16, 6, nlevels=2 if nested else 1)
    xs = list(x) if nested else [x]
    micros = {} if kind == "unet" else mcases.micro_set("nested_unet", "all", batch)
    return xs, t, lm, mask, micros


def call(model, xs, t, lm, mask, micros):
    out = model(xs if len(xs) > 1 else xs[0], t, lm, mask, micros)
    return list(out) if len(xs) > 1 else [out]


def cuda_all(xs, t, lm, mask, micros):
    return [x.cuda() for x in xs], t.cuda(), lm.cuda(), mask.cuda(), {k: v.cuda() for k, v in micros.items()}


def weights(xs):
    g = torch.Generator().manual_seed(11)
    return [torch.randn(x.shape, generator=g).cuda() for x in xs]


def step(model, ins, ws, autocast=None):
    """Forward (under `autocast` when given) and backward outside it, as the reference's training step does;
    returns (outputs, {name: gradient}) and leaves the gradients cleared."""
    if autocast is None:
        outs = call(model, *ins)
    else:
        with torch.autocast("cuda", dtype=autocast):
            outs = call(model, *ins)
    sum((o * w).sum() for o, w in zip(outs, ws)).backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}
    model.zero_grad(set_to_none=True)
    return [o.detach().clone() for o in outs], grads


def close_out(a, b, spread):
    bound = 1e-6 + 10.0 * spread
    for x, y in zip(a, b):
        assert parity.rel(x, y) <= bound, (parity.rel(x, y), bound)


def profiled(fn):
    """Runs fn with the GEMM profile on; returns fn's result and the profile rows."""
    lib = _lib.lib()
    torch.cuda.synchronize()
    lib.mdm_profile_gemm(1)
    try:
        r = fn()
        torch.cuda.synchronize()
    finally:
        lib.mdm_profile_gemm(0)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "gemm.csv")
        assert lib.mdm_profile_dump(path.encode()) == 0
        tot, n = C.c_double(), C.c_longlong()
        lib.mdm_profile_read(C.byref(tot), C.byref(n))
        rows = list(csv.DictReader(open(path)))
    return r, rows


# ---------------------------------------------------------------- 1. calibrated accuracy
def accuracy_report(kind, dtype):
    """Errors against the fp64 oracle (CPU) of the engine under autocast and of the oracle in fp32 under the same
    autocast: parity.report."""
    model, oracle, sd = build(kind)
    xs, t, lm, mask, micros = inputs(kind)
    ws = [w.cpu() for w in weights(xs)]
    args = (sd, xs, t, lm, mask, micros, ws)
    return parity.report(parity.engine_arm(model, xs, t, lm, mask, micros, ws, autocast=DTYPES[dtype]),
                         parity.oracle_arm(oracle.forward, *args, torch.float64, "cpu"),
                         parity.oracle_arm(oracle.forward, *args, torch.float32, "cuda", autocast=DTYPES[dtype]))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_autocast_within_the_reference_autocast_error(kind, dtype):
    rep = accuracy_report(kind, dtype)
    # the bounds of the fp32 path (DESIGN.md section 4), with the reference's autocast error in place of its TF32 one
    parity.assert_calibrated(rep)


# ---------------------------------------------------------------- 2. the path really changed
def test_profile_shows_single_plane_under_autocast():
    model, _, _ = build("nested")
    model = model.cuda()
    ins = cuda_all(*inputs("nested"))
    ws = weights(ins[0])
    step(model, ins, ws)  # pack and size everything outside the profiled calls
    _, ac = profiled(lambda: step(model, ins, ws, torch.bfloat16))
    _, fp = profiled(lambda: step(model, ins, ws))
    assert ac and all(int(r["planes"]) == 0 for r in ac), sorted({r["planes"] for r in ac})
    # the same products, but the fp32 call multiplies the weights' lo planes (and the ResNet data gradients' A lo planes)
    shape = lambda r: (r["kind"], r["M"], r["N"], r["K"])  # noqa: E731
    assert sorted(map(shape, ac)) == sorted(map(shape, fp))
    assert sum(1 for r in fp if int(r["planes"]) & 1) >= len(fp) // 4
    assert any(int(r["planes"]) & 2 for r in fp)


# ---------------------------------------------------------------- 3. nothing else changed
@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graph"])
def test_fp32_after_autocast_and_weight_update_matches_a_fresh_net(graphs):
    model, _, _ = build("nested")
    a = model.cuda()
    ins = cuda_all(*inputs("nested"))
    ws = weights(ins[0])
    a.native().set_graph_mode(graphs)
    step(a, ins, ws)  # both planes packed
    g = torch.Generator(device="cuda").manual_seed(4)
    with torch.no_grad():
        for p in a.parameters():
            p.add_(1e-2 * torch.randn(p.shape, device="cuda", generator=g))  # in place: the engine repacks
    for _ in range(3):  # single-plane passes after the update: hi planes only, lo planes stale (captured in graph mode)
        step(a, ins, ws, torch.bfloat16)
    b = copy.deepcopy(a)  # a fresh engine on the updated weights
    b.native().set_graph_mode(graphs)
    for _ in range(3 if graphs else 1):  # eager, capture, replay
        oa, ga = step(a, ins, ws)
        ob, gb = step(b, ins, ws)
    ob2, _ = step(b, ins, ws)
    close_out(oa, ob, max(parity.rel(x, y) for x, y in zip(ob2, ob)))
    parity.assert_same_run([], [], ga, gb)
    # what the comparison guards: a single-plane result is far outside that bound
    ob_ac, _ = step(b, ins, ws, torch.bfloat16)
    assert min(parity.rel(x, y) for x, y in zip(ob_ac, ob)) > 1e-5


# ---------------------------------------------------------------- 4. graphs alternating between the modes
def test_graph_replay_alternating_modes_matches_eager():
    model, _, _ = build("nested")
    graph = model.cuda()
    eager = copy.deepcopy(graph)
    graph.native().set_graph_mode(True)
    eager.native().set_graph_mode(False)
    ins = cuda_all(*inputs("nested"))
    ws = weights(ins[0])
    g0 = _lib.graph_launch_count()
    for i in range(8):
        ac = torch.bfloat16 if i % 2 == 0 else None
        og, gg = step(graph, ins, ws, ac)
        oe, ge = step(eager, ins, ws, ac)
        oe2, _ = step(eager, ins, ws, ac)
        close_out(og, oe, max(parity.rel(x, y) for x, y in zip(oe2, oe)))
        parity.assert_same_run([], [], gg, ge)
        with torch.no_grad():  # the same in-place update on both
            for pg, pe in zip(graph.parameters(), eager.parameters()):
                d = 1e-3 * torch.sin(pg * (i + 1))
                pg.add_(d)
                pe.add_(d)
    assert _lib.graph_launch_count() - g0 >= 4  # both modes reached replay


# ---------------------------------------------------------------- 5. split forward and the K/V cache
def test_cond_cache_across_a_mode_change():
    model, _, _ = build("nested")
    model = model.cuda().eval()
    xs, t, lm, mask, micros = cuda_all(*inputs("nested"))
    nat = model.native()
    with torch.no_grad():
        enc = model.forward_conditioning(lm, mask)
        model.forward_denoising(xs, t, *enc, micros)  # fill, two-plane
        # the engine refuses a single-plane read of a two-plane fill, whatever the caller asks for
        real = nat._cache_mode
        nat._cache_mode = lambda *a: 2
        with pytest.raises(_lib.MdmError, match="two-plane forward"):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                model.forward_denoising(xs, t, *enc, micros)
        nat._cache_mode = real
        # NativeNet refills instead, and a refill in the new mode is then reused
        with torch.autocast("cuda", dtype=torch.bfloat16):
            assert nat._cache_mode(xs, enc[1], enc[2]) == 1
            o1 = model.forward_denoising(xs, t, *enc, micros)
            assert nat._cache_mode(xs, enc[1], enc[2]) == 2
            o2 = model.forward_denoising(xs, t, *enc, micros)
            ref = model(xs, t, lm, mask, micros)
        assert nat._cache_mode(xs, enc[1], enc[2]) == 1  # back outside autocast: the single-plane fill is not reused
    parity.assert_same_run(o1, ref)
    parity.assert_same_run(o2, ref)


def test_ddim_under_autocast_with_text_encoded_once_matches_per_step():
    vm, _, _ = build("nested")
    model = NestedModel(vm.cuda(), mc.NestedDiffusionConfig(no_use_residual=True)).eval()
    sampler = NestedSampler(mc.SamplerConfig(num_diffusion_steps=32)).cuda()
    _, _, lm, mask, micros = cuda_all(*inputs("nested"))
    x = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(9)).cuda()

    def run(per_step):
        if per_step:
            sampler._encode_text = lambda *a: None  # model(...) at every step
        torch.manual_seed(5)
        try:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return sampler.sample(model, x, lm, mask, micros, num_inference_steps=8, ddim_eta=0.0,
                                      resample_steps=True, guidance_scale=1.0)
        finally:
            if per_step:
                del sampler._encode_text

    _, rows = profiled(lambda: run(False))
    assert rows and all(int(r["planes"]) == 0 for r in rows)
    a = run(False)
    b = run(True)
    b2 = run(True)
    assert parity.rel(a, b) <= max(parity.RUN_OUT, 3.0 * parity.rel(b2, b)), (parity.rel(a, b), parity.rel(b2, b))


# ---------------------------------------------------------------- 6. train_batch with args.fp16
class _Sched:
    def get_last_lr(self):
        return [1e-3]

    def step(self):
        pass


def test_train_batch_fp16_runs_single_plane_and_matches_explicit_autocast():
    vm, _, _ = build("nested")
    dcfg = mc.diffusion_config_from_dict(copy.deepcopy(tc.TINY_NESTED_DIFFUSION), True)
    pipe = NestedDiffusion(vm, dcfg).to("cuda")
    xs, _, lm, mask, micros = cuda_all(*inputs("nested"))
    sample = {"images": xs[0], "lm_outputs": lm, "lm_mask": mask, **micros}
    args = argparse.Namespace(fp16=True, gradient_clip_norm=1.0)
    opt = optim.FusedAdam(vm, lr=1e-3)
    params = list(pipe.get_model().vision_model.parameters())

    def explicit():
        torch.manual_seed(21)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            losses, *_ = pipe.get_loss(sample)
            loss = losses.mean()
        loss.backward()
        g = [p.grad.detach().clone() for p in params]
        for p in params:
            p.grad = None
        return float(loss.detach()), g

    def batch():
        torch.manual_seed(21)
        # accumulate_gradient: the gradients stay in .grad (no optimizer step) to be compared
        r = trainer.train_batch(pipe, sample, opt, _Sched(), None, args, accumulate_gradient=True)
        g = [p.grad.detach().clone() for p in params]
        for p in params:
            p.grad = None
        return r[0], g

    explicit()  # pack and size outside the profiled call
    (loss_b, grads_b), rows = profiled(batch)
    assert rows and all(int(r["planes"]) == 0 for r in rows)
    loss_e, grads_e = explicit()
    assert abs(loss_b - loss_e) <= parity.RUN_OUT * abs(loss_e)
    names = [k for k, _ in pipe.get_model().vision_model.named_parameters()]
    parity.assert_same_run([], [], dict(zip(names, grads_b)), dict(zip(names, grads_e)))
