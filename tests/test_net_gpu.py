"""Native denoiser parity on the GPU against the fp64 oracle (tiny UNet and 2-level NestedUNet):
outputs, every intermediate residual-stream activation, and every parameter gradient.

Bounds are stated against the reference's own GPU arithmetic, measured in the same run with the same metric
(max|delta| / max|ref| against the fp64 oracle): the oracle in fp32 on the same GPU with TF32 enabled, which is what the
reference trains with (clis/train_parallel.py:18-19). Measured: outputs 1.1-1.5e-3
vs 1.0-1.3e-3 for reference-TF32, gradient median 2.5-2.7e-3 vs 1.9-2.0e-3, worst single gradient 2.3x its
reference-TF32 error. Asserted: outputs and activations <= max(1e-3, 1.75 x reference-TF32), gradient median <= 1.5 x,
every gradient <= 3.5 x max(its reference-TF32 error, the reference-TF32 median)."""
import os

import numpy as np
import pytest
import torch

import fullwidth_cases as fc
import net_cases as nc
import parity
import tiny_configs as tc

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_forward_backward_vs_oracle(kind):
    parity.assert_calibrated(nc.run_case(kind, verbose=False))


@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_forward_vs_reference_golden(kind):
    """Same inputs/parameters as tests/golden (generated from the unmodified reference in fp32)."""
    model, _, _ = parity.tiny_model(tc.TINY[kind])
    nested = kind == "nested"
    x, t, lm, mask = tc.seeded_inputs(3, 2, 32 if nested else 16, 6, nlevels=2 if nested else 1)
    gold = np.load(os.path.join(GOLD, f"tiny_{kind}.npz"))
    model = model.cuda()
    with torch.no_grad():
        out = model([xi.cuda() for xi in x] if nested else x.cuda(), t.cuda(), lm.cuda(), mask.cuda(), {})
    for i, o in enumerate(out if nested else [out]):
        ref = torch.from_numpy(gold[f"fwd_out{i}"])
        assert parity.rel(o.cpu(), ref) <= 2.5e-3  # ~1.75 x the reference-TF32 error of these outputs (1.0-1.3e-3)


def test_fresh_model_outputs_exact_zero():
    """Size-independent property: conv_out is zero-initialised, so an untrained model predicts 0
    (bias included) for any input -- checked on the full cc12m_64x64 width."""
    from mdm_b200 import config as mc
    from mdm_b200.models import UNet

    cfgp = os.path.join(os.path.dirname(GOLD), "..", "ml-mdm_b200", "mdm_b200", "configs", "cc12m_64x64.yaml")
    ucfg, _, _ = mc.load_yaml_configs(cfgp)
    torch.manual_seed(0)
    m = UNet(3, 3, ucfg).cuda()
    with torch.no_grad():
        out = m(torch.randn(2, 3, 64, 64, device="cuda"), torch.tensor([3, 900], device="cuda"),
                torch.randn(2, 32, 2048, device="cuda"), torch.ones(2, 32, device="cuda"), {})
    assert float(out.abs().max()) == 0.0


def test_batch_independence_full_width():
    """Every op is per-sample (no BatchNorm): sample i's output must not depend on its batch mates."""
    m, _ = fc.build("cc12m_64x64")
    m = m.cuda()
    x = torch.randn(3, 3, 64, 64, device="cuda")
    t = torch.tensor([10, 500, 990], device="cuda")
    lm = torch.randn(3, 16, 2048, device="cuda")
    mask = torch.ones(3, 16, device="cuda")
    with torch.no_grad():
        full = m(x, t, lm, mask, {})
        one = m(x[1:2], t[1:2], lm[1:2], mask[1:2], {})
    # Not bit-identical: the GroupNorm partial sums are combined by fp32 atomics whose order depends on
    # the grid, and a 1e-7 change upstream flips fp16 roundings (2^-11 each) downstream -- the same
    # noise floor as two runs of one batch, far below any cross-sample leak (which would be O(1)).
    assert parity.rel(one, full[1:2]) <= parity.RUN_OUT


# (full-width forward AND backward parity of the three shipped configs: tests/test_fullwidth_gpu.py)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["unet", "nested"])
def test_grad_ready_ranges_are_final(kind):
    """mdm_net_set_grad_ready (include/mdm_b200.h): every address range reported during backward must
    already hold its final values in stream order (this is what lets the data-parallel all-reduce start
    before backward has finished, parallel.GradientOverlap). A snapshot enqueued inside the callback is
    compared bit-for-bit with the arena after backward."""
    check_grad_ready_ranges(parity.tiny_model(tc.TINY[kind])[0], kind)


def check_grad_ready_ranges(model, kind):
    nlev = 1 if kind == "unet" else 2
    res = 16 if kind == "unet" else 32
    model = model.cuda()
    x, t, lm, mask = tc.seeded_inputs(3, 2, res, 6, nlevels=nlev)
    xs = [x.cuda()] if nlev == 1 else [xi.cuda() for xi in x]
    native = model.native()
    snaps = []

    def on_ready(lo, hi):
        arena = native.active_arena
        a = (lo - arena.data_ptr()) // 4
        b = (hi - arena.data_ptr()) // 4
        assert 0 <= a < b <= arena.numel()
        snaps.append((a, b, arena[a:b].clone()))  # enqueued at this point of the backward stream

    def step():
        out = model(xs if nlev > 1 else xs[0], t.cuda(), lm.cuda(), mask.cuda(), {})
        outs = [out] if nlev == 1 else list(out)
        sum((o * o).sum() for o in outs).backward()
        torch.cuda.synchronize()

    native_bytes_hint = 0  # report every newly final byte
    step()                       # the engine learns which closure touches which parameter
    model.zero_grad(set_to_none=True)
    assert native.optimize_arena_layout()   # arena re-sorted by gradient finalisation order
    native.set_grad_ready(on_ready, native_bytes_hint)
    arena = None
    # second backward: recorded as one CUDA graph per reported range (graph mode) or run eagerly (MDM_NO_GRAPH);
    # third and fourth: replayed segment by segment with the callback between the launches
    for rnd in range(3):
        snaps.clear()
        model.zero_grad(set_to_none=True)
        step()
        assert len(snaps) >= 3, "no gradient range was reported during backward %d" % (rnd + 2)
        arena = native.grad_arena
        covered = 0
        prev_lo = max(off + p.numel() for p, off in zip(native.params, native.offsets))  # end of the last gradient
        top = prev_lo
        for a, b, snap in snaps:
            assert b == prev_lo, "ranges must tile the arena from the top down without gaps or overlap"
            prev_lo = a
            covered += b - a
            assert torch.equal(snap, arena[a:b]), f"gradient range [{a},{b}) changed after it was reported final"
        assert prev_lo == 0 and covered == top
    native.set_grad_ready(None)
    # gradients handed to autograd alias the arena (adopted, not cloned)
    lo_b, hi_b = arena.data_ptr(), arena.data_ptr() + 4 * arena.numel()
    assert all(lo_b <= p.grad.data_ptr() < hi_b for p in model.parameters())
    # and the step still produced non-trivial gradients
    assert float(arena.abs().max()) > 0
