"""GPU: non-square images through the engine. The tiny UNet and nest against the fp64 oracle within the calibrated
bounds of DESIGN.md section 4 at shapes whose conv tiles are partial on both axes (and their transposes), the shipped
configurations at rectangular sizes, graph replay across signatures that differ only in orientation, the K/V-cache
sampling path of a rectangular nest, and the conv GEMM forms called directly at edge shapes."""
import copy

import pytest
import torch

import gemm_cases as gc
import net_cases as nc
import test_rect_oracle as fx
from mdm_b200 import _lib
from mdm_b200 import config as mc
from mdm_b200.diffusion import NestedDiffusion, NestedModel
from mdm_b200.models import NestedUNet, UNet
from oracle import unet_ref

pytestmark = pytest.mark.gpu

ROOT_CFG = fx.os.path.join(fx.os.path.dirname(fx.os.path.abspath(__file__)), "..", "ml-mdm_b200", "mdm_b200", "configs")


def run_rect_case(kind, hw, batch=2, tokens=6, dtype=torch.float64):
    """net_cases.run_case on an (H, W) image: engine, fp64 oracle and TF32 oracle, same parameters and loss."""
    nlev = 1 if kind == "unet" else 2
    model, oracle, sd = nc.build(kind)
    x, t, lm, mask = fx.rect_inputs(3, batch, hw, tokens, nlevels=nlev)
    xs = [x] if nlev == 1 else x
    ws = fx.loss_weights(xs)
    P = {k: v.to(dtype).requires_grad_(True) for k, v in sd.items()}
    o_out = oracle.forward(P, [xi.to(dtype) for xi in xs] if nlev > 1 else xs[0].to(dtype), t, lm.to(dtype),
                           mask.to(dtype), {})
    o_outs = [o_out] if nlev == 1 else list(o_out)
    sum((o * w.to(dtype)).sum() for o, w in zip(o_outs, ws)).backward()
    model = model.cuda()
    xs_c = [xi.cuda() for xi in xs]
    out = model(xs_c if nlev > 1 else xs_c[0], t.cuda(), lm.cuda(), mask.cuda(), {})
    outs = [out] if nlev == 1 else list(out)
    sum((o * w.cuda()).sum() for o, w in zip(outs, ws)).backward()
    torch.cuda.synchronize()
    r = {"out": [nc.rel(o.detach().cpu().to(dtype), q.detach()) for o, q in zip(outs, o_outs)], "acts": {}}
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    try:
        Pt = {k: v.float().cuda().requires_grad_(True) for k, v in sd.items()}
        t_out = oracle.forward(Pt, [xi.cuda() for xi in xs] if nlev > 1 else xs[0].cuda(), t.cuda(), lm.cuda(),
                               mask.cuda(), {})
        t_outs = [t_out] if nlev == 1 else list(t_out)
        sum((o * w.cuda()).sum() for o, w in zip(t_outs, ws)).backward()
        torch.cuda.synchronize()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
    r["tf32_out"] = [nc.rel(o.detach().cpu().to(dtype), q.detach()) for o, q in zip(t_outs, o_outs)]
    mags = sorted(float(P[k].grad.abs().max()) for k, _ in model.named_parameters())
    floor = 1e-2 * mags[len(mags) // 2]
    r["grads"], r["tf32_grads"] = {}, {}
    for k, p in model.named_parameters():
        ref = P[k].grad
        den = max(float(ref.abs().max()), floor)
        r["grads"][k] = float((p.grad.detach().cpu().to(dtype) - ref).abs().max() / den)
        r["tf32_grads"][k] = float((Pt[k].grad.detach().cpu().to(dtype) - ref).abs().max() / den)
    return r


TINY_SHAPES = [("unet", (24, 40)), ("unet", (40, 24)), ("unet", (18, 30)), ("unet", (30, 18)),
               ("nested", fx.NEST_HW), ("nested", fx.NEST_HW[::-1])]


@pytest.mark.parametrize("kind,hw", TINY_SHAPES, ids=[f"{k}-{h}x{w}" for k, (h, w) in TINY_SHAPES])
def test_tiny_rect_within_calibrated_bounds(kind, hw):
    nc.assert_calibrated(run_rect_case(kind, hw))


def test_inner_level_shape_is_checked_before_anything_runs():
    model, _, _ = nc.build("nested")
    model = model.cuda()
    xs, t, lm, mask = fx.rect_inputs(3, 2, fx.NEST_HW, 6, nlevels=2)
    bad = [xs[0].cuda(), xs[1].transpose(2, 3).contiguous().cuda()]  # 20x12 under a 48x80 outer level
    k0 = _lib.launch_count()
    with pytest.raises(_lib.MdmError, match="level 1 input"):
        model(bad, t.cuda(), lm.cuda(), mask.cuda(), {})
    assert _lib.launch_count() == k0


def test_graph_replay_follows_orientation():
    """32x48, 48x32 and 32x32 have equal byte counts pairwise; replay must pick the graph of the right shape."""
    model, _, _ = nc.build("unet")
    eager = copy.deepcopy(model).cuda()
    graph = model.cuda()
    eager.native().set_graph_mode(False)
    graph.native().set_graph_mode(True)
    g0 = _lib.graph_launch_count()
    shapes = [(32, 48), (48, 32), (32, 32)] * 4
    for step, hw in enumerate(shapes):
        x, t, lm, mask = fx.rect_inputs(200 + step, 2, hw, 6)
        inp = (x.cuda(), t.cuda(), lm.cuda(), mask.cuda())
        res = []
        for m in (graph, eager):
            out = m(*inp, {})
            (out * out).sum().backward()
            grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
            m.zero_grad(set_to_none=True)
            res.append((out.detach().clone(), grads))
        torch.cuda.synchronize()
        assert res[0][0].shape == (2, 3) + hw
        assert nc.rel(res[0][0], res[1][0]) <= 3e-3, (step, hw)
        mags = sorted(float(v.abs().max()) for v in res[1][1].values())
        floor = 1e-2 * mags[len(mags) // 2]
        worst = max(float((res[0][1][k] - v).abs().max()) / max(float(v.abs().max()), floor)
                    for k, v in res[1][1].items())
        assert worst <= 2e-2, (step, hw, worst)
    assert _lib.graph_launch_count() > g0  # the later rounds replayed


def _full_model(name, nested):
    ucfg, dcfg, _ = mc.load_yaml_configs(fx.os.path.join(ROOT_CFG, name + ".yaml"))
    m = (NestedUNet if nested else UNet)(3, 3, copy.deepcopy(ucfg))
    m.load_state_dict(fx.tc.seeded_state_dict(m.state_dict(), fx.FULL_PARAM_SEED))
    return m, ucfg, dcfg


def test_cc12m_64_training_step_on_64x96_batch8():
    m, ucfg, _ = _full_model("cc12m_64x64", False)
    x, t, lm, mask = fx.rect_inputs(9, 8, fx.FULL_HW, 77, lm_dim=2048)
    oracle = unet_ref.OracleNet(ucfg, 2048)
    P = {k: v.double().cuda() for k, v in m.state_dict().items()}
    with torch.no_grad():
        ref = oracle.forward(P, x.double().cuda(), t.cuda(), lm.double().cuda(), mask.double().cuda(), {})
        torch.backends.cuda.matmul.allow_tf32 = True
        torch.backends.cudnn.allow_tf32 = True
        try:
            Pt = {k: v.float() for k, v in P.items()}
            tf = oracle.forward(Pt, x.cuda(), t.cuda(), lm.cuda(), mask.cuda(), {})
        finally:
            torch.backends.cuda.matmul.allow_tf32 = False
            torch.backends.cudnn.allow_tf32 = False
    del P, Pt
    m = m.cuda()
    out = m(x.cuda(), t.cuda(), lm.cuda(), mask.cuda(), {})
    assert out.shape == (8, 3) + fx.FULL_HW
    (out * out).sum().backward()
    torch.cuda.synchronize()
    tf32_err = nc.rel(tf.double(), ref)
    assert nc.rel(out.detach().double(), ref) <= max(1e-3, 1.5 * tf32_err)
    assert all(torch.isfinite(p.grad).all() for p in m.parameters() if p.grad is not None)


@pytest.mark.parametrize("mixed", [False, True])
def test_cc12m_256_nest_get_loss_on_256x192(mixed):
    m, _, dcfg = _full_model("cc12m_256x256", True)
    dcfg = copy.deepcopy(dcfg)
    if not mixed:
        dcfg.mixed_ratio = None
    else:
        dcfg.mixed_ratio = "2:1"
    pipe = NestedDiffusion(m, dcfg).to("cuda")
    B = 4
    g = torch.Generator().manual_seed(3)
    images = (torch.rand(B, 3, 256, 192, generator=g) * 2 - 1).cuda()
    lm = torch.randn(B, 77, 2048, generator=g).cuda()
    mask = torch.ones(B, 77).cuda()
    loss = pipe.get_loss({"images": images, "lm_outputs": lm, "lm_mask": mask})[0]
    loss.mean().backward()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    assert all(torch.isfinite(p.grad).all() for p in m.parameters() if p.grad is not None)


class _PerStep(NestedModel):
    """A NestedModel subclass that overrides forward: the sampler calls it in full at every step."""

    def forward(self, *a, **k):
        return super().forward(*a, **k)


def test_kv_cache_sampling_matches_per_step_on_rect_nest():
    model, _, _ = nc.build("nested")
    cfg = mc.diffusion_config_from_dict(copy.deepcopy(fx.tc.TINY_NESTED_DIFFUSION), nested=True)
    pipe = NestedDiffusion(model, cfg).to("cuda")
    model = pipe.get_model().vision_model
    _, _, lm, mask = fx.rect_inputs(4, 2, fx.NEST_HW, 6, nlevels=2)
    lm2 = torch.cat([torch.zeros_like(lm), lm]).cuda()
    mask2 = torch.cat([mask, mask]).cuda()
    imgs = []
    for m in (pipe.model, _PerStep(model, cfg), pipe.model):
        torch.manual_seed(5)
        noise = torch.randn(2, 3, *fx.NEST_HW).cuda()
        imgs.append(pipe.sampler.sample(m, noise, lm2, mask2, {}, num_inference_steps=8, resample_steps=True,
                                        ddim_eta=0.0, guidance_scale=3.0))
    torch.cuda.synchronize()
    assert imgs[0].shape == (2, 3) + fx.NEST_HW
    # guidance amplifies each evaluation's run-to-run differences (fp32 atomics) step after step: the bound is measured
    # by a second run of the cached path, as test_cond_split_gpu does for square nests
    assert nc.rel(imgs[0], imgs[1]) <= max(3e-3, 3.0 * nc.rel(imgs[2], imgs[0])), (nc.rel(imgs[0], imgs[1]),
                                                                                nc.rel(imgs[2], imgs[0]))


# conv GEMM forms at edges no square power-of-two size reaches: W mod 16 not in {0, 8}, H mod 8 != 0, odd sides
CONV_EDGES = [
    ("fwd_18x30", lambda: gc.run_conv_fwd(2, 18, 30, 64, 64, 64)),
    ("fwd_9x15", lambda: gc.run_conv_fwd(2, 9, 15, 128, 128, 128)),
    ("fwd_12x20_res", lambda: gc.run_conv_fwd(3, 12, 20, 64, 192, 192, residual=True)),
    ("fwd_paired_6x10", lambda: gc.run_conv_fwd(2, 6, 10, 768, 768, 256)),
    ("fwd_w15", lambda: gc.run_conv_fwd(2, 18, 15, 64, 64, 64)),
    ("dgrad_18x30", lambda: gc.run_conv_dgrad(2, 18, 30, 64, 64, 64)),
    ("dgrad_9x15", lambda: gc.run_conv_dgrad(2, 9, 15, 128, 128, 128)),
    ("dgrad_paired_6x10", lambda: gc.run_conv_dgrad(2, 6, 10, 768, 768, 256)),
    ("wgrad_18x30", lambda: gc.run_conv_wgrad(2, 18, 30, 64, 128, 128, nsplit=2)),
    ("wgrad_9x15", lambda: gc.run_conv_wgrad(3, 9, 15, 128, 128, 128)),
    ("wgrad_256px_20x36_c32", lambda: gc.run_conv_wgrad(2, 20, 36, 32, 32, 32, nsplit=2, kfactor=4)),
    ("wgrad_256px_24x40_c64", lambda: gc.run_conv_wgrad(2, 24, 40, 64, 64, 64, kfactor=4)),
]


@pytest.mark.parametrize("name,fn", CONV_EDGES, ids=[c[0] for c in CONV_EDGES])
def test_conv_forms_at_edge_shapes(name, fn):
    errs = fn()
    for k, v in errs.items():
        assert v <= gc.TOL[k], (name, k, v)
