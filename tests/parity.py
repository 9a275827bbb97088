"""Calibrated parity (DESIGN.md section 4): the one definition of the metric, the arms and the bounds of the GPU tests.

The engine is measured against the fp64 oracle, and its error is bounded by multiples of the error that the
reference's own arithmetic makes in the same run: the oracle in fp32 with TF32 enabled (what the reference trains
with, clis/train_parallel.py:18-19), or the oracle under the same torch.autocast for the autocast tests. Errors are
max|a - ref| / max|ref| per tensor. Two runs of the engine differ by the order of its fp32 atomics, and are held to
RUN_OUT / RUN_GRAD."""
import contextlib
import copy

import torch

import tiny_configs as tc
from mdm_b200 import config as mc
from mdm_b200.models import NestedUNet, UNet
from oracle import unet_ref

RUN_OUT, RUN_GRAD = 3e-3, 2e-2  # two engine runs on the same inputs: outputs, gradients


def rel(a, b):
    """max|a - b| / max|b|, in float64."""
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


@contextlib.contextmanager
def tf32():
    """TF32 on for cuBLAS and cuDNN; the previous settings come back on exit."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


_tf32 = tf32  # oracle_arm's tf32 argument shadows the name


def grad_floor(ref):
    """1e-2 of the median over tensors of max|ref|. Gradients that are mathematically zero (a conv bias in front of a
    GroupNorm whose groups are single channels) come out as round-off on every side; below this floor they are judged
    on the scale of the real gradients."""
    mags = sorted(float(r.abs().max()) for r in ref.values())
    return 1e-2 * mags[len(mags) // 2]


def grad_errors(got, ref, floor=True):
    """{name: max|got - ref| / max(max|ref|, grad_floor(ref))} over the names of `ref` that `got` holds. The floor is
    taken over exactly the tensors of `ref`; floor=False divides by max|ref| alone."""
    f = grad_floor(ref) if floor else 0.0
    return {k: float((got[k].double() - r.double()).abs().max()) / max(float(r.abs().max()), f, 1e-300)
            for k, r in ref.items() if k in got}


def _loss_backward(outs, ws, dtype, device):
    sum((o.to(dtype) * w.to(device, dtype)).sum() for o, w in zip(outs, ws)).backward()


def oracle_arm(forward, sd, xs, t, lm, mask, micros, ws, dtype, device, tf32=False, autocast=None, leaves=None,
               **kw):
    """Forward and backward of loss = sum_l <out_l, w_l> through `forward` (an oracle's OracleNet.forward, or a function
    of the same arguments) with the parameters `sd`, everything in `dtype` on `device`: with TF32 on when tf32, the
    forward under torch.autocast(dtype=autocast) when given. xs and ws hold one tensor per level. leaves: further inputs
    {name: tensor}, passed to `forward` as keywords, whose gradients come back as "<name>"; kw: further keywords of
    `forward` (trace=). Returns ([out_l], {name: gradient}) on the CPU in float64."""
    P = {k: v.to(device, dtype).requires_grad_(True) for k, v in sd.items()}
    L = {k: v.to(device, dtype).requires_grad_(True) for k, v in (leaves or {}).items()}
    xin = [x.to(device, dtype) for x in xs]
    args = (P, xin if len(xs) > 1 else xin[0], t.to(device), lm.to(device, dtype), mask.to(device, dtype),
            {k: v.to(device) for k, v in micros.items()})
    with _tf32() if tf32 else contextlib.nullcontext():
        with torch.autocast("cuda", dtype=autocast, enabled=autocast is not None):
            out = forward(*args, **L, **kw)
        outs = list(out) if len(xs) > 1 else [out]
        _loss_backward(outs, ws, dtype, device)
    grads = {k: p.grad for k, p in P.items() if p.grad is not None}
    grads.update({f"<{k}>": v.grad for k, v in L.items()})
    res = [o.detach().cpu().double() for o in outs], {k: g.detach().cpu().double() for k, g in grads.items()}
    del P, L, out, outs, grads
    torch.cuda.empty_cache()
    return res


def engine_arm(model, xs, t, lm, mask, micros, ws, autocast=None, leaves=None, forward=None):
    """oracle_arm for the engine on the GPU: `model` (or `forward`, a function of the model's call arguments and the
    leaves as keywords) called in its own arithmetic, under torch.autocast(dtype=autocast) when given. Gradients are
    those of the model's parameters that have one, and of the leaves. The model stays on the GPU."""
    model = model.cuda()
    L = {k: v.cuda().requires_grad_(True) for k, v in (leaves or {}).items()}
    xin = [x.cuda() for x in xs]
    with torch.autocast("cuda", dtype=autocast, enabled=autocast is not None):
        out = (forward or model)(xin if len(xs) > 1 else xin[0], t.cuda(), lm.cuda(), mask.cuda(),
                                 {k: v.cuda() for k, v in micros.items()}, **L)
    outs = list(out) if len(xs) > 1 else [out]
    _loss_backward(outs, ws, torch.float32, "cuda")
    torch.cuda.synchronize()
    grads = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    grads.update({f"<{k}>": v.grad for k, v in L.items()})
    return [o.detach().cpu().double() for o in outs], {k: g.detach().cpu().double() for k, g in grads.items()}


def report(engine, f64, reference, floor=True):
    """Errors against the fp64 arm of the engine arm and of the reference arm, each an (outs, grads) pair:
    {"out": [(ours, reference)], "grads": {name: (ours, reference)}, "missing": [names the engine left without a
    gradient]}. floor: grad_errors' floor over the fp64 arm's gradients."""
    (oo, go), (o64, g64), (orf, grf) = engine, f64, reference
    ours, ref = grad_errors(go, g64, floor), grad_errors(grf, g64, floor)
    return {"out": [(rel(a, r), rel(b, r)) for a, b, r in zip(oo, orf, o64)],
            "grads": {k: (v, ref[k]) for k, v in ours.items()},
            "missing": sorted(k for k in g64 if k not in go)}


def _median(v):
    v = sorted(v)
    return v[len(v) // 2]


def assert_calibrated(rep):
    """Tiny nets: every output <= max(1e-3, 1.75 x its reference error), every traced activation (rep["acts"], when
    present) <= max(2e-3, 2 x the largest reference output error), the gradient median <= 1.5 x the reference's, and
    every gradient <= 3.5 x max(its reference error, the reference median). No gradient may be missing."""
    assert not rep["missing"], rep["missing"]
    for ours, ref in rep["out"]:
        assert ours <= max(1e-3, 1.75 * ref), rep["out"]
    act_lim = max(2e-3, 2.0 * max(ref for _, ref in rep["out"]))
    bad = {k: v for k, v in rep.get("acts", {}).items() if isinstance(v, str) or not v <= act_lim}
    assert not bad, (bad, act_lim)
    assert_calibrated_grads(rep["grads"])


def assert_calibrated_grads(grads):
    """The gradient bounds of assert_calibrated on {name: (ours, reference)}."""
    med = _median(v[1] for v in grads.values())
    ours_med = _median(v[0] for v in grads.values())
    assert ours_med <= 1.5 * med, (ours_med, med)
    bad = {k: v for k, v in grads.items() if not v[0] <= 3.5 * max(v[1], med)}
    assert not bad, bad


def defined_grads(grads):
    """The gradients of {name: (ours, reference)} that the reference defines at full width: reference error <= 0.5.
    The others are mathematically zero (a conv bias in front of single-channel GroupNorm groups) and round-off on every
    implementation."""
    return {k: v for k, v in grads.items() if v[1] <= 0.5}


def assert_calibrated_full_width(rep):
    """The shipped architectures (tests/test_fullwidth_gpu.py): every output <= max(1e-3, 1.5 x its reference error);
    gradient median and 90th percentile <= 1.25 x the reference's and each gradient <= 3 x max(its reference error, the
    reference median), over the gradients the reference defines (reference error <= 0.5). The others are mathematically
    zero, at most 5 % of all: their max|gradient| <= 3 x max(the reference's, 1e-3 x the typical max|gradient|).
    rep: report(..., floor=False) with "grad_absmax", "grad_absmax_tf32" ({name: max|gradient|} of the engine and of
    the reference) and "grad_typical" (the median over parameters of the fp64 max|gradient|)."""
    assert not rep["missing"], rep["missing"]
    assert_outputs_full_width(rep["out"])
    defined = defined_grads(rep["grads"])
    undefined = [k for k in rep["grads"] if k not in defined]
    assert len(undefined) <= 0.05 * len(rep["grads"]), sorted(undefined)[:10]
    for k in undefined:
        lim = 3.0 * max(rep["grad_absmax_tf32"][k], 1e-3 * rep["grad_typical"])
        assert rep["grad_absmax"][k] <= lim, (k, rep["grad_absmax"][k], rep["grad_absmax_tf32"][k], rep["grad_typical"])
    o = sorted(v[0] for v in defined.values())
    r = sorted(v[1] for v in defined.values())
    n = len(o)
    assert o[n // 2] <= 1.25 * r[n // 2], (o[n // 2], r[n // 2])
    assert o[int(0.9 * n)] <= 1.25 * r[int(0.9 * n)], (o[int(0.9 * n)], r[int(0.9 * n)])
    bad = {k: v for k, v in defined.items() if not v[0] <= 3.0 * max(v[1], r[n // 2])}
    assert not bad, bad


def assert_outputs_full_width(out):
    """The output bound of assert_calibrated_full_width on [(ours, reference)]."""
    for i, (ours, ref) in enumerate(out):
        assert ours <= max(1e-3, 1.5 * ref), (i, ours, ref)


def assert_same_run(outs, ref_outs, grads=None, ref_grads=None):
    """Two engine runs on the same inputs: every output within RUN_OUT of its counterpart, and, when given, the same
    gradient names with every gradient within RUN_GRAD (grad_errors, floor over ref_grads)."""
    for i, (a, b) in enumerate(zip(outs, ref_outs)):
        assert rel(a, b) <= RUN_OUT, (i, rel(a, b))
    if ref_grads is not None:
        assert grads.keys() == ref_grads.keys(), sorted(grads.keys() ^ ref_grads.keys())
        bad = {k: e for k, e in grad_errors(grads, ref_grads).items() if not e <= RUN_GRAD}
        assert not bad, bad


def tiny_model(ucfg, oracle_cls=unet_ref.OracleNet, seed=7, **oracle_kw):
    """(UNet or NestedUNet of the tiny config dict `ucfg` with tc.seeded_state_dict(seed) loaded, its oracle
    oracle_cls(config, tc.LM_DIM, **oracle_kw), the state_dict)."""
    cfg = mc.unet_config_from_dict(copy.deepcopy(ucfg))
    cfg.conditioning_feature_dim = tc.LM_DIM
    ocfg = copy.deepcopy(cfg)  # the model constructor mutates conditioning_feature_dim
    model = (NestedUNet if "inner_config" in ucfg else UNet)(3, 3, cfg)
    sd = tc.seeded_state_dict(model.state_dict(), seed)
    model.load_state_dict(sd)
    return model, oracle_cls(ocfg, tc.LM_DIM, **oracle_kw), sd
