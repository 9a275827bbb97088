"""GPU: the fused clip + Adam/AdamW + EMA + zero-grad sweep (mdm_grad_norm, mdm_adam_ema_sweep through the C ABI)
against the golden fixture of torch's Adam/AdamW + clip_grad_norm_ + the reference ModelEma, and
mdm_b200.optim.FusedAdam / trainer.train_batch against the reference's separate calls on a tiny U-Net.

Tolerance: fp32 formulas restated op for op, differing only in fused-multiply-add contraction and the reduction
order of the norm: |delta| <= 2e-6 * |ref| + 1e-7 per element (a few ulps), norm 1e-6 relative."""
import ctypes as C
import copy
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "ml-mdm_b200"))
sys.path.insert(0, HERE)
from mdm_b200 import _lib, optim  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(HERE, "golden", "optim_steps.npz"))
VARIANTS = {"adam": (False, 0.0), "adamw": (True, 0.01), "adam_l2": (False, 0.01)}
NT = 4
RTOL, ATOL = 2e-6, 1e-7


def close(a, b):
    return bool(((a.double().cpu() - b.double()).abs() <= RTOL * b.double().abs() + ATOL).all())


def gold_list(tag, key):
    return [torch.from_numpy(GOLD[f"{tag}/{key}/{i}"].copy()) for i in range(NT)]


@pytest.mark.parametrize("tag", list(VARIANTS))
def test_sweep_kernels_vs_torch_golden(tag):
    adamw, wd = VARIANTS[tag]
    dev = "cuda"
    lib = _lib.lib()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ps = [p.to(dev) for p in gold_list(tag, "p0")]
    emas = [p.clone() for p in ps]
    pad = lambda n: (n + 63) // 64 * 64
    offs, total = [], 0
    for p in ps:
        offs.append(total)
        total += pad(p.numel())
    arena = torch.zeros(total, device=dev)
    m = torch.zeros(total, device=dev)
    v = torch.zeros(total, device=dev)
    rows = []
    for p, e, off in zip(ps, emas, offs):
        rows += optim.chunk_rows(p.data_ptr(), arena.data_ptr() + 4 * off, m.data_ptr() + 4 * off,
                                 v.data_ptr() + 4 * off, e.data_ptr(), p.numel(), chunk=300)  # several chunks, odd tails
    table = torch.tensor(rows, dtype=torch.int64).reshape(-1, 6).to(dev)
    scratch = torch.zeros(optim.GRAD_NORM_SCRATCH, device=dev, dtype=torch.float64)
    norm = torch.zeros(1, device=dev)
    for step in range(3):
        for g, p, off in zip(gold_list(tag, f"g{step}"), ps, offs):
            arena[off:off + p.numel()] = g.to(dev).flatten()
        _lib.check(lib.mdm_grad_norm(C.c_void_p(arena.data_ptr()), C.c_int64(total), C.c_float(1.0),
                                     C.c_void_p(scratch.data_ptr()), C.c_int32(optim.GRAD_NORM_SCRATCH),
                                     C.c_void_p(norm.data_ptr()), st), "mdm_grad_norm")
        cfg = optim.AdamCfg()
        cfg.lr, cfg.beta1, cfg.beta2, cfg.eps, cfg.weight_decay = 3e-3, 0.9, 0.999, 1e-8, wd
        cfg.adamw, cfg.step, cfg.grad_scale, cfg.max_norm, cfg.zero_grad = int(adamw), step + 1, 1.0, 2.0, 1
        cfg.ema_decay = float(step >= 1) * 0.9
        _lib.check(lib.mdm_adam_ema_sweep(C.c_void_p(table.data_ptr()), C.c_int32(table.shape[0]), C.byref(cfg),
                                          C.c_void_p(norm.data_ptr()), st), "mdm_adam_ema_sweep")
        torch.cuda.synchronize()
        ref_norm = float(GOLD[f"{tag}/norm{step}"])
        assert abs(float(norm) - ref_norm) <= 1e-6 * ref_norm
        assert float(arena.abs().max()) == 0.0, "gradients must be left zeroed"
        ms = [m[off:off + p.numel()].view_as(p) for p, off in zip(ps, offs)]
        vs = [v[off:off + p.numel()].view_as(p) for p, off in zip(ps, offs)]
        for name, mine in (("p", ps), ("ema", emas), ("m", ms), ("v", vs)):
            for i, (a, b) in enumerate(zip(mine, gold_list(tag, f"{name}{step + 1}"))):
                assert close(a, b), f"{tag} step {step} {name}[{i}]: max diff {float((a.cpu() - b).abs().max()):.3e}"


class _Ema:  # the attributes of ml_mdm.models.model_ema.ModelEma that the sweep uses
    def __init__(self, model, decay, warmup_steps):
        self.module = copy.deepcopy(model)
        self.decay, self.warmup_steps, self.counter = decay, warmup_steps, 0

    def update(self, model):  # model_ema.py:25-34
        decay = (self.counter >= self.warmup_steps) * self.decay
        self.counter += 1
        with torch.no_grad():
            msd = model.state_dict()
            for k, ema_v in self.module.state_dict().items():
                ema_v.mul_(decay).add_(msd[k].detach(), alpha=1.0 - decay)


def test_fused_adam_on_tiny_unet_matches_separate_calls():
    """Two optimisation steps of a tiny U-Net: FusedAdam.step(clip, ema) on the engine's gradient arena vs
    clip_grad_norm_ + torch Adam + ModelEma.update on a copy that is handed the very same gradients (Adam divides
    by sqrt(v): feeding both sides one set of gradients keeps round-off-sized gradients from deciding signs)."""
    import parity
    import tiny_configs as tc
    model_a, _, _ = parity.tiny_model(tc.TINY_UNET)
    model_a = model_a.cuda()
    model_b = copy.deepcopy(model_a)
    x, t, lm, mask = tc.seeded_inputs(3, 2, 16, 6, nlevels=1)
    x, t, lm, mask = x.cuda(), t.cuda(), lm.cuda(), mask.cuda()
    opt_a = optim.FusedAdam(model_a, lr=2e-3)
    opt_b = torch.optim.Adam(model_b.parameters(), lr=2e-3, eps=1e-8)
    ema_a, ema_b = _Ema(model_a, 0.9, 1), _Ema(model_b, 0.9, 1)
    for step in range(2):
        out = model_a(x, t, lm, mask, {})
        ((out - 0.3 * x) ** 2).mean().backward()
        for pa, pb in zip(model_a.parameters(), model_b.parameters()):
            pb.grad = pa.grad.detach().clone()
        total_b = torch.nn.utils.clip_grad_norm_(model_b.parameters(), 0.05)
        opt_b.step()
        ema_b.update(model_b)
        opt_b.zero_grad()
        opt_a.step(max_grad_norm=0.05, ema_model=ema_a)
        assert all(float(p.grad.abs().max()) == 0.0 for p in model_a.parameters()), "arena must be left zeroed"
        opt_a.zero_grad()
        torch.cuda.synchronize()
        assert abs(float(opt_a.last_grad_norm) - float(total_b)) <= 2e-6 * float(total_b)
    sa, sb = model_a.state_dict(), model_b.state_dict()
    for k in sb:
        assert close(sa[k], sb[k].cpu()), f"{k}: {float((sa[k] - sb[k]).abs().max()):.3e}"
    for (k, ea), (_, eb) in zip(ema_a.module.state_dict().items(), ema_b.module.state_dict().items()):
        assert close(ea, eb.cpu()), f"ema {k}: {float((ea - eb).abs().max()):.3e}"
    assert ema_a.counter == ema_b.counter == 2
    st = opt_a.state_dict()["state"]
    assert len(st) == len(list(model_a.parameters())) and float(st[0]["step"]) == 2.0
    # and the engine picks the updated weights up: a third forward differs from the first
    out3 = model_a(x, t, lm, mask, {})
    assert float((out3 - out).abs().max()) > 0


def _tiny(kind="unet"):
    import parity
    import tiny_configs as tc
    nlev = 1 if kind == "unet" else 2
    model, _, _ = parity.tiny_model(tc.TINY[kind])
    model = model.cuda()
    x, t, lm, mask = tc.seeded_inputs(3, 2, 16 if nlev == 1 else 32, 6, nlevels=nlev)
    xs = x.cuda() if nlev == 1 else [xi.cuda() for xi in x]
    return model, xs, t.cuda(), lm.cuda(), mask.cuda()


def _loss(model, xs, t, lm, mask):
    out = model(xs, t, lm, mask, {})
    outs = list(out) if isinstance(out, (list, tuple)) else [out]
    return sum((o ** 2).mean() for o in outs)


def test_frozen_inner_unet_gradients_stay_out_of_norm_and_sweep():
    """freeze_inner_unet (nested_unet.py:147-150) sets requires_grad=False on the inner U-Net: the engine must not
    accumulate those gradients (they would never be zeroed by the sweep, inflate the global norm step after step and
    drive the clip coefficient to 0), and the norm must equal clip_grad_norm_'s over the trainable parameters."""
    model, xs, t, lm, mask = _tiny("nested")
    for p in model.inner_unet.parameters():
        p.requires_grad_(False)
    frozen = {k: v.detach().clone() for k, v in model.inner_unet.state_dict().items()}
    opt = optim.FusedAdam(model, lr=1e-3)
    norms = []
    for step in range(3):
        _loss(model, xs, t, lm, mask).backward()
        assert all(p.grad is None for p in model.inner_unet.parameters())
        ref = torch.nn.utils.clip_grad_norm_([p for p in model.parameters() if p.requires_grad], 1e9)
        native = model.native()
        assert float(native.grad_arena.abs().max()) > 0
        opt.step(max_grad_norm=1e9)
        torch.cuda.synchronize()
        assert abs(float(opt.last_grad_norm) - float(ref)) <= 1e-5 * float(ref)
        assert float(native.grad_arena.abs().max()) == 0.0, "arena (frozen slots included) must be zero after the sweep"
        norms.append(float(ref))
        opt.zero_grad()
    for k, v in model.inner_unet.state_dict().items():
        assert torch.equal(v, frozen[k]), f"frozen parameter {k} moved"
    assert norms[2] < 10 * norms[0]


def test_ema_engine_sees_fused_updates():
    """The sweep writes EMA parameters through raw pointers; an engine already built for the EMA module has to repack
    its fp16 operand copies (ModelEma consumers sample from ema.module between updates)."""
    model, xs, t, lm, mask = _tiny("unet")
    ema = _Ema(model, 0.5, 0)
    opt = optim.FusedAdam(model, lr=5e-2)
    with torch.no_grad():
        e0 = ema.module(xs, t, lm, mask, {}).clone()     # builds + caches the EMA module's engine
    for _ in range(2):
        _loss(model, xs, t, lm, mask).backward()
        opt.step(max_grad_norm=1.0, ema_model=ema)
        opt.zero_grad()
    with torch.no_grad():
        e1 = ema.module(xs, t, lm, mask, {})
        fresh = copy.deepcopy(ema.module)               # no cached engine: packs from the current fp32 values
        e2 = fresh(xs, t, lm, mask, {})
    assert float((e1 - e0).abs().max()) > 0, "EMA forward still uses the weights packed before the updates"
    # not bit-identical run to run: GroupNorm partial sums are combined by fp32 atomics
    assert float((e1 - e2).abs().max()) <= 1e-3 * float(e2.abs().max())


def test_fused_adam_state_dict_round_trip_matches_torch_adam():
    """save -> load -> step: bias corrections continue from the loaded step and the loaded moments are the ones used
    (torch.optim.Adam on a copy, fed the same gradients, is the reference)."""
    model_a, xs, t, lm, mask = _tiny("unet")
    model_b = copy.deepcopy(model_a)
    opt_a = optim.FusedAdam(model_a, lr=2e-3)
    opt_b = torch.optim.Adam(model_b.parameters(), lr=2e-3, eps=1e-8)

    def both_step(oa):
        _loss(model_a, xs, t, lm, mask).backward()
        for pa, pb in zip(model_a.parameters(), model_b.parameters()):
            pb.grad = pa.grad.detach().clone()
        opt_b.step()
        opt_b.zero_grad()
        oa.step()
        oa.zero_grad()

    for _ in range(3):
        both_step(opt_a)
    sd = copy.deepcopy(opt_a.state_dict())
    # (a) a brand-new optimizer that loads the state; (b) the same optimizer re-loading after having stepped
    opt_new = optim.FusedAdam(model_a, lr=2e-3)
    opt_new.load_state_dict(sd)
    assert opt_new.steps == 3
    both_step(opt_new)
    torch.cuda.synchronize()
    for (k, a), (_, b) in zip(model_a.state_dict().items(), model_b.state_dict().items()):
        assert close(a, b.cpu()), f"{k}: {float((a - b).abs().max()):.3e}"
    assert float(opt_new.state_dict()["state"][0]["step"]) == 4.0
    sb = opt_b.state_dict()["state"]
    for i, st in opt_new.state_dict()["state"].items():
        assert close(st["exp_avg"], sb[i]["exp_avg"].cpu()) and close(st["exp_avg_sq"], sb[i]["exp_avg_sq"].cpu())
    sd4 = copy.deepcopy(opt_new.state_dict())
    both_step(opt_new)                 # moves on to step 5 ...
    opt_new.load_state_dict(sd4)       # ... and is rolled back to the state after step 4
    assert opt_new.steps == 4
    m0 = opt_new.state_dict()["state"][0]["exp_avg"].clone()
    _loss(model_a, xs, t, lm, mask).backward()
    g0 = next(iter(model_a.parameters())).grad.detach().clone()
    opt_new.step()
    torch.cuda.synchronize()
    m1 = opt_new.state_dict()["state"][0]["exp_avg"]
    assert close(m1, (0.9 * m0 + 0.1 * g0).cpu()), "loaded exp_avg was not the one the kernel used"
