"""ResNet dropout (ResNetConfig.dropout) on the GPU: the mask operator's statistics, and the native UNet / NestedUNet in
train mode against the dropout oracle fed with the engine's own masks (rebuilt by mdm_op_dropout_mask from the seed the
model draws from torch's CPU generator), eval mode, no_grad, p = 1, CUDA-graph replay and a full-width nested step."""
import copy
import ctypes as C
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", "ml-mdm_b200"))

import dropout_oracle  # noqa: E402
import net_cases as nc  # noqa: E402
import test_dropout_host as host  # noqa: E402
import tiny_configs as tc  # noqa: E402
from mdm_b200 import _lib  # noqa: E402
from mdm_b200 import config as mc  # noqa: E402
from mdm_b200.models import NestedUNet, UNet  # noqa: E402

pytestmark = pytest.mark.gpu

DROP_SEED = 2024  # torch.manual_seed before the forward whose masks are rebuilt


def engine_mask(seed, stream, n, p):
    """The factors (0 or 1/(1-p)) the engine applies to the n elements of a ResNet with this stream id, fp32 cuda."""
    out = torch.empty(n, device="cuda", dtype=torch.float32)
    _lib.check(_lib.lib().mdm_op_dropout_mask(C.c_uint64(seed), C.c_uint32(stream), C.c_int64(n), C.c_float(p),
                                              C.c_void_p(out.data_ptr()),
                                              C.c_void_p(torch.cuda.current_stream().cuda_stream)), "dropout mask")
    return out


def seed_after(torch_seed):
    """The dropout seed NativeNet draws right after torch.manual_seed(torch_seed)."""
    return int(torch.randint(2**63 - 1, (), generator=torch.Generator().manual_seed(torch_seed)))


def mask_fn(model, seed, ps):
    """dropout_oracle masks of the engine: ps[level] is p of the level with that many "inner_unet." prefixes."""
    names = model.native().names
    cache = {}

    def masks(pre, shape):
        if pre not in cache:
            n, c, h, w = shape
            m = engine_mask(seed, names.index(pre + ".conv2.weight"), n * h * w * c, ps[pre.count("inner_unet.")])
            cache[pre] = m.view(n, h, w, c).permute(0, 3, 1, 2).cpu()  # the fp32 factors the engine multiplies by
        return cache[pre]
    return masks


# ------------------------------------------------------------------------------------------ the operator
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_mask_operator_statistics(p):
    n = (1 << 24) + 3  # >= 16 M elements, and a partial last group of four
    a = engine_mask(123456789, 7, n, p)
    scale = torch.tensor(1.0 / (1.0 - p), dtype=torch.float32).item()
    kept = a != 0
    assert bool(((a == 0) | (a == scale)).all())  # exactly {0, 1/(1-p)} in fp32
    frac = float(kept.double().mean())
    sigma = (p * (1 - p) / n) ** 0.5
    assert abs(frac - (1 - p)) <= 6 * sigma, (frac, 1 - p, sigma)
    assert torch.equal(a, engine_mask(123456789, 7, n, p))  # a pure function of (seed, stream, index)
    agree_ind = (1 - p) ** 2 + p ** 2
    s_agree = (agree_ind * (1 - agree_ind) / n) ** 0.5
    for other in (engine_mask(123456790, 7, n, p), engine_mask(123456789, 8, n, p)):
        agree = float((kept == (other != 0)).double().mean())
        assert abs(agree - agree_ind) <= 6 * s_agree, (agree, agree_ind)
    z = engine_mask(5, 1, 1000, 1.0)
    assert not bool(z.any())


# ------------------------------------------------------------------------------------------ the network
def tiny_build(masked, p_outer=host.P_OUTER, p_inner=host.P_INNER):
    """net_cases.build for the tiny configs with dropout, whose oracle applies the engine's masks of the forward that
    follows (run_case runs the native model once, right after build)."""
    def build(kind, seed=7):
        ucfg = host.tiny_config("unet" if kind == "unet" else "nested_unet", p_outer, p_inner)
        (ucfg if kind == "unet" else ucfg["inner_config"])["masked_cross_attention"] = masked
        cfg = mc.unet_config_from_dict(ucfg)
        cfg.conditioning_feature_dim = tc.LM_DIM
        ocfg = copy.deepcopy(cfg)
        model = (UNet if kind == "unet" else NestedUNet)(3, 3, cfg)
        sd = tc.seeded_state_dict(model.state_dict(), seed)
        model.load_state_dict(sd)
        oracle = dropout_oracle.OracleNet(ocfg, tc.LM_DIM, mask_fn(model, seed_after(DROP_SEED), [p_outer, p_inner]))
        torch.manual_seed(DROP_SEED)
        return model, oracle, sd
    return build


@pytest.mark.parametrize("masked", [0, 1], ids=["m0", "m1"])
@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_dropout_forward_backward_vs_oracle(kind, masked, monkeypatch):
    monkeypatch.setattr(nc, "build", tiny_build(masked))
    nc.assert_calibrated(nc.run_case(kind, verbose=False))


def test_dropout_mixed_ratio_nest_vs_oracle(monkeypatch):
    """The outer level runs the first sample only (level_batch 1 of 2): its masks index a (1, H, W, C) tensor."""
    monkeypatch.setattr(nc, "build", tiny_build(1))
    real = tc.seeded_inputs

    def narrow_outer(*a, **k):
        xs, t, lm, mask = real(*a, **k)
        return [xs[0][:1]] + xs[1:], t, lm, mask

    monkeypatch.setattr(nc.tc, "seeded_inputs", narrow_outer)
    nc.assert_calibrated(nc.run_case("nested", verbose=False))


def test_dropout_p1_gives_reference_zeros():
    """p = 1: every ResNet's conv2 sees zeros (nn.Dropout(p=1)), so the gradients inside the ResNets are exactly zero,
    not NaN, and the rest of the step matches the oracle with all-zero masks."""
    model, oracle, sd = tiny_build(1, 1.0, 1.0)("nested")
    x, t, lm, mask = _inputs("nested")
    P = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    ref = oracle.forward(P, [xi.cpu().double() for xi in x], t.cpu(), lm.cpu().double(), mask.cpu().double(), {})
    sum((o * o).sum() for o in ref).backward()
    model = model.cuda()
    out = model(x, t, lm, mask, {})
    sum((o * o).sum() for o in out).backward()
    for o, r in zip(out, ref):
        assert nc.rel(o.detach().cpu().double(), r.detach()) <= 2.5e-3
    mags = sorted(float(P[k].grad.abs().max()) for k in P if float(P[k].grad.abs().max()) > 0)
    floor = 1e-2 * mags[len(mags) // 2]
    inside = (".norm1.", ".conv1.", ".time_layer.", ".norm2.", ".conv2.weight")
    for k, p in model.named_parameters():
        g = p.grad.detach().cpu().double()
        assert bool(torch.isfinite(g).all()), k
        if ".resnets." in k and any(s in k for s in inside):
            assert float(g.abs().max()) == 0.0, k
        elif float(P[k].grad.abs().max()) < floor:  # mathematically zero (a bias in front of norm_out): round-off
            assert float(g.abs().max()) <= floor, k
        else:
            assert float((g - P[k].grad).abs().max()) / float(P[k].grad.abs().max()) <= 5e-2, k


def _model(kind, p_outer, p_inner, seed=7):
    return tiny_build(1, p_outer, p_inner)(kind, seed)[0].cuda()


def _inputs(kind, seed=3):
    nlev = 1 if kind == "unet" else 2
    x, t, lm, mask = tc.seeded_inputs(seed, 2, 16 if nlev == 1 else 32, 6, nlevels=nlev)
    return (x.cuda() if nlev == 1 else [xi.cuda() for xi in x]), t.cuda(), lm.cuda(), mask.cuda()


def _outs(o):
    return [t.detach().clone() for t in (o if isinstance(o, list) else [o])]


@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_eval_mode_runs_as_p0(kind):
    """Eval mode with p > 0 takes the p = 0 kernels. The forward is not bit-reproducible from run to run (fp32 atomics
    in the GroupNorm statistics and split-K products add in a varying order), so the outputs are held to that level,
    which lies far below what dropout changes (test_no_grad_forward_in_train_mode_drops)."""
    a, b = _model(kind, 0.1, 0.25).eval(), _model(kind, 0.0, 0.0).eval()
    inp = _inputs(kind)
    with torch.no_grad():
        for x, y in zip(_outs(a(*inp, {})), _outs(b(*inp, {}))):
            assert nc.rel(x, y) <= 3e-3, nc.rel(x, y)


@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_no_grad_forward_in_train_mode_drops(kind):
    m = _model(kind, 0.1, 0.25)
    inp = _inputs(kind)
    with torch.no_grad():
        train = _outs(m(*inp, {}))
        ev = _outs(m.eval()(*inp, {}))
    assert all(nc.rel(x, y) > 1e-2 for x, y in zip(train, ev)), [nc.rel(x, y) for x, y in zip(train, ev)]


def test_nested_dropout_modules_disagreeing_with_the_model_are_refused():
    m = _model("nested", 0.1, 0.25)
    m.inner_unet.eval()  # the top module stays in training mode
    with pytest.raises(_lib.MdmError):
        m(*_inputs("nested"), {})


@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_rng_state_untouched_without_dropout(kind):
    m = _model(kind, 0.0, 0.0)
    inp = _inputs(kind)
    before = torch.get_rng_state()
    m(*inp, {})
    assert torch.equal(before, torch.get_rng_state())
    m2 = _model(kind, 0.1, 0.25)
    before = torch.get_rng_state()
    m2(*inp, {})
    assert not torch.equal(before, torch.get_rng_state())  # with dropout the seed is drawn from it


def _step(m, inp):
    out = m(*inp, {})
    outs = out if isinstance(out, list) else [out]
    sum((o * o).sum() for o in outs).backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    return [o.detach().clone() for o in outs], grads


@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_graph_steps_match_eager_steps_under_one_seed(kind):
    """Four training steps (eager, capture, replay, replay in graph mode) against the same steps without graphs under
    the same torch seed: the same masks, so the outputs and gradients agree to the fp32-atomics run-to-run level of
    test_lm_head_gpu's graph test (the GroupNorm statistics and split-K products add in a varying order, so two runs
    are not bit-identical whatever the masks). A step under a different seed is far outside that level."""
    eager, graph = _model(kind, 0.1, 0.25), _model(kind, 0.1, 0.25)
    eager.native().set_graph_mode(False)
    graph.native().set_graph_mode(True)
    inp = _inputs(kind)
    g0 = _lib.graph_launch_count()
    torch.manual_seed(77)
    gsteps = [_step(graph, inp) for _ in range(4)]
    assert _lib.graph_launch_count() - g0 >= 4  # steps 2-4 replayed forward and backward graphs
    torch.manual_seed(77)
    esteps = [_step(eager, inp) for _ in range(4)]
    for i, ((og, gg), (oe, ge)) in enumerate(zip(gsteps, esteps)):
        for a, b in zip(og, oe):
            assert nc.rel(a, b) <= 3e-3, (i, nc.rel(a, b))
        mags = sorted(float(v.abs().max()) for v in ge.values())
        floor = 1e-2 * mags[len(mags) // 2]
        for k in ge:
            e = float((gg[k] - ge[k]).abs().max() / max(float(ge[k].abs().max()), floor))
            assert e <= 2e-2, (i, k, e)
    # consecutive steps draw fresh masks, replays included: identical inputs, different outputs
    for i in range(1, 4):
        assert all(nc.rel(a, b) > 1e-2 for a, b in zip(gsteps[i][0], gsteps[i - 1][0])), i


def test_full_width_nested_step_with_dropout(monkeypatch):
    """One cc12m_256x256 training step with p = 0.1 on both levels, bounds of test_fullwidth_gpu."""
    import fullwidth_cases as fc
    import test_fullwidth_gpu as tfw

    real_build = fc.build
    state = {}

    def build(name, seed=0):
        ucfg, _, nested = mc.load_yaml_configs(os.path.join(fc.CFG_DIR, name + ".yaml"))
        c = ucfg
        while c is not None:
            c.resnet_config.dropout = 0.1
            c = getattr(c, "inner_config", None)
        ocfg = copy.deepcopy(ucfg)
        m, _, _ = real_build(name, seed)
        dm = (NestedUNet if nested else UNet)(3, 3, ucfg)
        dm.load_state_dict(m.state_dict())
        state["masks"] = mask_fn(dm, seed_after(DROP_SEED), [0.1, 0.1])
        torch.manual_seed(DROP_SEED)
        return dm, ocfg, nested

    oracle_mod = type(sys)("dropout_unet_ref")
    oracle_mod.OracleNet = lambda cfg, lm_dim: dropout_oracle.OracleNet(cfg, lm_dim, state["masks"])
    monkeypatch.setattr(fc, "build", build)
    monkeypatch.setattr(fc, "unet_ref", oracle_mod)
    tfw.test_forward_backward_full_width_calibrated_against_reference_tf32("cc12m_256x256", 2)
