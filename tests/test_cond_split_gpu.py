"""forward_conditioning / forward_denoising on the GPU: each stage against the oracle (fp64, with bounds calibrated by
the reference-TF32 error of the same run as in DESIGN §4), the split path against `forward`, and the engine's reuse of
the text encoding across denoising steps (the K/V cache of the cross-attention blocks)."""
import copy
import ctypes as C
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "ml-mdm_b200"))

import fullwidth_cases as fc  # noqa: E402
import lm_head_oracle  # noqa: E402
import parity  # noqa: E402
import tiny_configs as tc  # noqa: E402
from mdm_b200 import _lib  # noqa: E402
from mdm_b200 import config as mc  # noqa: E402
from mdm_b200.diffusion import NestedDiffusion, NestedModel  # noqa: E402
from mdm_b200.models import NestedUNet  # noqa: E402
from mdm_b200.samplers import NestedSampler  # noqa: E402
from oracle import unet_ref  # noqa: E402

pytestmark = pytest.mark.gpu


def build(kind, masked=1, layers=0, seed=7, dropout=0.0):
    ucfg = copy.deepcopy(tc.TINY_UNET if kind == "unet" else tc.TINY_NESTED)
    inner = ucfg if kind == "unet" else ucfg["inner_config"]
    inner["num_lm_head_layers"] = layers
    inner["masked_cross_attention"] = masked
    c = ucfg
    while c is not None:
        c["resnet_config"]["dropout"] = dropout
        c = c.get("inner_config")
    return parity.tiny_model(ucfg, lm_head_oracle.OracleNet, seed)


def inputs(kind, seed=3, batch=2, tokens=6):
    nested = kind != "unet"
    return tc.seeded_inputs(seed, batch, 32 if nested else 16, tokens, nlevels=2 if nested else 1)


def text_param(name):
    return any(s in name for s in ("lm_proj.", "lm_head.", "cond_emb."))


# ---------------------------------------------------------------- 1. forward_conditioning against the oracle
@pytest.mark.parametrize("layers", [0, 2])
@pytest.mark.parametrize("masked", [0, 1], ids=["m0", "m1"])
@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_forward_conditioning_vs_oracle(kind, masked, layers):
    model, oracle, sd = build(kind, masked, layers)
    _, _, lm, mask = inputs(kind)
    ipre, iplan, _ = oracle.levels[-1]

    def ora(dev, dt):
        P = {k: v.to(dev, dt) for k, v in sd.items()}
        return lm_head_oracle.forward_conditioning(P, ipre, iplan, lm.to(dev, dt), mask.to(dev, dt))

    ref = ora("cpu", torch.float64)
    with parity.tf32():
        t32 = ora("cuda", torch.float32)
    model = model.cuda()
    with torch.no_grad():
        emb, cond, cm = model.forward_conditioning(lm.cuda(), mask.cuda())
    assert (cm is None) == (masked == 0)
    for ours, r, t in ((emb, ref[0], t32[0]), (cond, ref[1], t32[1])):
        e, et = parity.rel(ours.cpu(), r), parity.rel(t.cpu(), r)
        assert e <= max(2e-3, 2.0 * et), (e, et)


def test_forward_conditioning_fused_lm_mask():
    """fuse_lm_mask: the raw encoder output goes in and is multiplied by the mask on the way, as forward does."""
    model, oracle, sd = build("unet", 1, 2)
    _, _, lm, mask = inputs("unet")
    raw = lm + (1 - mask).unsqueeze(-1) * torch.randn(lm.shape, generator=torch.Generator().manual_seed(2))
    ipre, iplan, _ = oracle.levels[-1]
    P = {k: v.double() for k, v in sd.items()}
    ref = lm_head_oracle.forward_conditioning(P, ipre, iplan, lm.double(), mask.double())
    model = model.cuda()
    model.fuse_lm_mask = True
    with torch.no_grad():
        emb, cond, _ = model.forward_conditioning(raw.cuda(), mask.cuda())
    assert parity.rel(cond.cpu(), ref[1]) <= 2e-3
    assert parity.rel(emb.cpu(), ref[0]) <= 2e-3


# ---------------------------------------------------------------- 2. forward_denoising on arbitrary inputs
@pytest.mark.parametrize("masked", [0, 1], ids=["m0", "m1"])
@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_forward_denoising_random_inputs_vs_oracle(kind, masked):
    model, oracle, sd = build(kind, masked)
    x, t, _, _ = inputs(kind)
    xs = [x] if kind == "unet" else list(x)
    ipre, iplan, _ = oracle.levels[-1]
    td, cd = sd[ipre + "cond_emb.weight"].shape
    g = torch.Generator().manual_seed(17)
    B, S = xs[0].shape[0], 5
    cond = torch.randn(B, S, cd, generator=g)
    cemb = torch.randn(B, td, generator=g) * 0.5
    cmask = torch.ones(B, S)
    cmask[1, 3:] = 0
    ws = [torch.randn(xi.shape, generator=g) for xi in xs]
    # the conditioning tokens and embedding are leaves whose gradients are compared too; the tokens also fill the
    # arms' text argument, which forward_denoising does not read
    leaves = {"conditioning": cond, "cond_emb": cemb}

    def ora(P, x, t, lm, mask, micros, conditioning, cond_emb):
        if not oracle.nested:
            return unet_ref.unet_denoise(P, "", iplan, x, t, cond_emb, conditioning, mask, {})
        return oracle._nested(0, P, x, None, t, cond_emb, conditioning, mask, {}, None)

    args = (sd, xs, t, cond, cmask, {}, ws)
    f64 = parity.oracle_arm(ora, *args, torch.float64, "cpu", leaves=leaves)
    t32 = parity.oracle_arm(ora, *args, torch.float32, "cuda", tf32=True, leaves=leaves)
    ours = parity.engine_arm(model, xs, t, cond, cmask, {}, ws, leaves=leaves, forward=lambda x, t, lm, mask, micros,
                             conditioning, cond_emb: model.forward_denoising(x, t, cond_emb, conditioning, mask))
    assert all(text_param(k) for k, _ in model.named_parameters() if k not in ours[1])
    parity.assert_calibrated(parity.report(ours, f64, t32))


# ---------------------------------------------------------------- 3. split path against forward
def _grads(m):
    return {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("case", ["unet_l2", "nested", "nested_dropout", "nested_frozen_inner"])
def test_split_matches_forward(case):
    kind = "unet" if case.startswith("unet") else "nested"
    model, _, _ = build(kind, 1, 2 if case == "unet_l2" else 0, dropout=0.1 if "dropout" in case else 0.0)
    if "frozen" in case:
        for p in model.inner_unet.parameters():
            p.requires_grad = False
    a, b = copy.deepcopy(model).cuda(), model.cuda()
    x, t, lm, mask = inputs(kind)
    xs = [x.cuda()] if kind == "unet" else [xi.cuda() for xi in x]
    ws = [torch.randn(xi.shape, device="cuda") for xi in xs]
    arg = xs[0] if kind == "unet" else xs
    for m in (a, b):
        m.train("dropout" in case)
    torch.manual_seed(123)
    oa = a(arg, t.cuda(), lm.cuda(), mask.cuda(), {})
    torch.manual_seed(123)
    emb, cond, cm = b.forward_conditioning(lm.cuda(), mask.cuda())
    ob = b.forward_denoising(arg, t.cuda(), emb, cond, cm)
    oa, ob = ([oa], [ob]) if kind == "unet" else (oa, ob)
    la = sum((o * w).sum() for o, w in zip(oa, ws))
    lb = sum((o * w).sum() for o, w in zip(ob, ws))
    la.backward()
    lb.backward()
    torch.cuda.synchronize()
    # the loss on the scale of its terms (it is a sum of terms of both signs)
    scale = float(sum((o.detach() * w).abs().sum() for o, w in zip(oa, ws)))
    assert abs(float(la.detach()) - float(lb.detach())) <= parity.RUN_OUT * scale
    ga, gb = _grads(a), _grads(b)
    parity.assert_same_run([v.detach() for v in ob], [u.detach() for u in oa], gb, ga)
    if "frozen" in case:
        assert not any(k.startswith("inner_unet.") for k in gb)
    else:
        assert any(text_param(k) for k in gb)


# ---------------------------------------------------------------- 4. the K/V cache
def _fetch_kv(native):
    buf = torch.empty(1 << 22, device="cuda")
    n = native.lib.mdm_net_debug_fetch(native.handle, b"cond_kv", C.c_void_p(buf.data_ptr()), C.c_int64(buf.numel()),
                                       C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert n > 0
    return buf[:n].clone().view(torch.int32)


def _modes(native):
    """Record the cache mode of every forward_denoising call."""
    seen = []
    real = native._cache_mode

    def spy(*a):
        m = real(*a)
        seen.append(m)
        return m
    native._cache_mode = spy
    return seen


def test_cache_reads_back_what_a_fresh_fill_computes():
    model, _, _ = build("nested", 1)
    model = model.cuda().eval()
    x, t, lm, mask = inputs("nested")
    xs = [xi.cuda() for xi in x]
    nat = model.native()
    modes = _modes(nat)
    with torch.no_grad():
        enc = model.forward_conditioning(lm.cuda(), mask.cuda())
        o1 = model.forward_denoising(xs, t.cuda(), *enc)
        k1 = _fetch_kv(nat)
        o2 = model.forward_denoising(xs, t.cuda(), *enc)
        k2 = _fetch_kv(nat)
        nat._kv = None  # forget the key: the next call fills the cache again
        model.forward_denoising(xs, t.cuda(), *enc)
        k3 = _fetch_kv(nat)
        ref = model(xs, t.cuda(), lm.cuda(), mask.cuda(), {})
    assert modes == [1, 2, 1]
    assert torch.equal(k1, k2) and torch.equal(k1, k3)
    parity.assert_same_run(o1, ref)
    parity.assert_same_run(o2, ref)


def test_cache_invalidation():
    model, _, _ = build("unet", 1)
    model = model.cuda().eval()
    x, t, lm, mask = inputs("unet")
    x, t = x.cuda(), t.cuda()
    nat = model.native()
    modes = _modes(nat)
    with torch.no_grad():
        emb, cond, cm = model.forward_conditioning(lm.cuda(), mask.cuda())
        model.forward_denoising(x, t, emb, cond, cm)                    # fill
        model.forward_denoising(x, t, emb, cond, cm)                    # reuse
        w = next(p for k, p in model.named_parameters() if k.endswith("kv_cond.weight"))
        w.mul_(1.5)                                                     # in-place weight update
        o = model.forward_denoising(x, t, emb, cond, cm)
        ref = model.forward_denoising(x, t, emb, cond.clone(), cm)      # a different tensor
        parity.assert_same_run([o], [ref])
        cond.mul_(0.5)                                                  # in-place write to the tokens
        o = model.forward_denoising(x, t, emb, cond, cm)
        ref = model.forward_denoising(x, t, emb, cond.clone(), cm)
        parity.assert_same_run([o], [ref])
        model.forward_denoising(x, t, emb, cond, cm)
    assert modes == [1, 2, 1, 1, 1, 1, 1]
    # the engine itself refuses a stale or mismatched cache, whatever the caller asks for
    with torch.no_grad():
        nat._cache_mode = lambda *a: 2
        nat.lib.mdm_net_weights_changed(nat.handle)
        with pytest.raises(_lib.MdmError, match="holds nothing valid"):
            model.forward_denoising(x, t, emb, cond, cm)
        nat._cache_mode = lambda *a: 1
        model.forward_denoising(x, t, emb, cond, cm)
        nat._cache_mode = lambda *a: 2
        with pytest.raises(_lib.MdmError, match="filled for batch"):
            model.forward_denoising(x[:1], t[:1], emb[:1], cond[:1], cm[:1])
        with pytest.raises(_lib.MdmError, match="filled for batch"):
            model.forward_denoising(x, t, emb, cond[:, :4].contiguous(), cm[:, :4].contiguous())
        out = model.forward_denoising(x, t, emb, cond, cm)  # the net is still usable
    assert torch.isfinite(out).all()


def test_graph_replay_of_stage2_matches_eager():
    model, _, _ = build("nested", 1)
    eager, graph = copy.deepcopy(model).cuda(), model.cuda()
    eager.native().set_graph_mode(False)
    graph.native().set_graph_mode(True)
    g0 = _lib.graph_launch_count()
    x, t, lm, mask = inputs("nested")
    xs = [xi.cuda() for xi in x]
    ws = [torch.randn(xi.shape, device="cuda") for xi in xs]
    for step in range(4):
        res = []
        for m in (graph, eager):
            emb, cond, cm = m.forward_conditioning(lm.cuda(), mask.cuda())
            outs = m.forward_denoising(xs, t.cuda(), emb, cond, cm)
            sum((o * w).sum() for o, w in zip(outs, ws)).backward()
            gr = _grads(m)
            m.zero_grad(set_to_none=True)
            with torch.no_grad():
                inf = m.forward_denoising(xs, t.cuda(), emb, cond, cm)
            res.append(([o.detach() for o in outs], gr, inf))
        (og, gg, ig), (oe, ge, ie) = res
        parity.assert_same_run(og + ig, oe + ie, gg, ge)
    assert _lib.graph_launch_count() - g0 >= 4


def _sample(pipe_or_sampler, model, x, lm, mask, g, steps, per_step):
    s = pipe_or_sampler
    if per_step:
        s._encode_text = lambda *a: None  # what a foreign model wrapper gets: model(...) at every step
    torch.manual_seed(5)
    try:
        return s.sample(model, x, lm, mask, {}, num_inference_steps=steps, ddim_eta=0.0, resample_steps=True,
                        guidance_scale=g)
    finally:
        if per_step:
            del s._encode_text


@pytest.mark.parametrize("guidance", [1.0, 3.0])
def test_ddim_with_reuse_matches_per_step_forward_tiny_nest(guidance):
    vm, _, _ = build("nested", 1)
    model = NestedModel(vm.cuda(), mc.NestedDiffusionConfig(no_use_residual=True)).eval()
    sampler = NestedSampler(mc.SamplerConfig(num_diffusion_steps=32)).cuda()
    B = 2
    _, _, lm, mask = inputs("nested", batch=2 * B if guidance != 1 else B)
    x = torch.randn(B, 3, 32, 32, generator=torch.Generator().manual_seed(9)).cuda()
    modes = _modes(vm.native())
    a = _sample(sampler, model, x, lm.cuda(), mask.cuda(), guidance, 8, False)
    assert modes == [1] + [2] * 7
    b = _sample(sampler, model, x, lm.cuda(), mask.cuda(), guidance, 8, True)
    # guidance amplifies the run-to-run differences of each evaluation (fp32 atomics) by 2w - 1 per step: the bound
    # is the spread of two runs of the per-step loop itself
    b2 = _sample(sampler, model, x, lm.cuda(), mask.cuda(), guidance, 8, True)
    assert parity.rel(a, b) <= max(parity.RUN_OUT, 3.0 * parity.rel(b2, b)), (parity.rel(a, b), parity.rel(b2, b))


@pytest.mark.parametrize("guidance", [1.0, 3.0])
def test_ddim_with_reuse_matches_per_step_forward_cc12m_256(guidance):
    _, dcfg, _ = mc.load_yaml_configs(os.path.join(fc.CFG_DIR, "cc12m_256x256.yaml"))
    vm, _ = fc.build("cc12m_256x256", seed=4321)
    pipe = NestedDiffusion(vm, dcfg).to("cuda")
    pipe.eval()
    B = 2
    n = 2 * B if guidance != 1 else B
    g = torch.Generator().manual_seed(3)
    lm = torch.randn(n, 16, 2048, generator=g).cuda()
    mask = torch.ones(n, 16)
    mask[0, 10:] = 0
    mask = mask.cuda()
    x = torch.randn(B, 3, 256, 256, generator=g).cuda()
    a = _sample(pipe.sampler, pipe.get_model(), x, lm, mask * 1, guidance, 6, False)
    b = _sample(pipe.sampler, pipe.get_model(), x, lm, mask * 1, guidance, 6, True)
    parity.assert_same_run([a], [b])


def test_launches_drop_by_the_skipped_text_path():
    """Per evaluation, reuse skips exactly: the input cast, lm_proj, the token LayerNorm, one kv_cond GEMM per
    cross-attention block, the masked mean and cond_emb (cc12m_256x256 has no lm_head layers)."""
    ucfg, _, _ = mc.load_yaml_configs(os.path.join(fc.CFG_DIR, "cc12m_256x256.yaml"))
    torch.manual_seed(0)
    vm = NestedUNet(3, 3, ucfg).cuda().eval()
    nat = vm.native()
    nat.set_graph_mode(False)
    n_kv = sum(1 for k in vm.state_dict() if k.endswith("kv_cond.weight"))
    assert n_kv == 31
    g = torch.Generator().manual_seed(3)
    B, S = 2, 16
    lm = torch.randn(B, S, 2048, generator=g).cuda()
    mask = torch.ones(B, S).cuda()
    xs = [torch.randn(B, 3, r, r, generator=g).cuda() for r in (256, 64)]
    t = torch.tensor([10, 500]).cuda()
    with torch.no_grad():
        vm(xs, t, lm, mask, {})
        k0 = _lib.launch_count()
        vm(xs, t, lm, mask, {})
        full = _lib.launch_count() - k0
        enc = vm.forward_conditioning(lm, mask)
        vm.forward_denoising(xs, t, *enc)  # fills the cache
        k0 = _lib.launch_count()
        vm.forward_denoising(xs, t, *enc)
        reuse = _lib.launch_count() - k0
    torch.cuda.synchronize()
    assert full - reuse == n_kv + 5, (full, reuse)
