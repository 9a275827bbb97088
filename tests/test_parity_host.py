"""The calibrated-parity policy of tests/parity.py pinned on the CPU: every bound passes exactly at its edge and fails 1 %
beyond it, a missing gradient or a NaN error fails, the gradient floor follows its rule, and the oracle arm runs the
tiny UNet in float64 and float32 into a report."""
import math

import pytest
import torch

import parity
import tiny_configs as tc

OVER = 1.01  # 1 % beyond a bound


def tiny_rep(out=((1e-3, 1e-3),), grads=None, acts=None, missing=()):
    rep = {"out": list(out), "grads": grads or {f"g{i}": (1e-3, 1e-3) for i in range(5)}, "missing": list(missing)}
    if acts is not None:
        rep["acts"] = acts
    return rep


def passes(check, rep):
    try:
        check(rep)
    except AssertionError:
        return False
    return True


# ---------------------------------------------------------------- tiny nets
@pytest.mark.parametrize("ref", [2e-3, 1e-4])
def test_tiny_output_bound(ref):
    edge = max(1e-3, 1.75 * ref)
    assert passes(parity.assert_calibrated, tiny_rep(out=[(edge, ref)]))
    assert not passes(parity.assert_calibrated, tiny_rep(out=[(edge * OVER, ref)]))


@pytest.mark.parametrize("ref", [2e-3, 1e-4])
def test_tiny_activation_bound(ref):
    edge = max(2e-3, 2.0 * ref)
    out = [(min(ref, 1e-3), ref)]
    assert passes(parity.assert_calibrated, tiny_rep(out=out, acts={"a": 1e-4, "b": edge}))
    assert not passes(parity.assert_calibrated, tiny_rep(out=out, acts={"a": 1e-4, "b": edge * OVER}))
    assert not passes(parity.assert_calibrated, tiny_rep(out=out, acts={"a": "released"}))


def test_tiny_gradient_median_bound():
    grads = {f"g{i}": (1.5 * 1e-3, 1e-3) for i in range(5)}
    assert passes(parity.assert_calibrated, tiny_rep(grads=grads))
    grads = {f"g{i}": (1.5 * 1e-3 * OVER, 1e-3) for i in range(5)}
    assert not passes(parity.assert_calibrated, tiny_rep(grads=grads))


@pytest.mark.parametrize("own", [1e-4, 2e-3])  # below the reference median, and above it
def test_tiny_per_tensor_bound(own):
    grads = {f"g{i}": (1e-3, 1e-3) for i in range(5)}
    edge = 3.5 * max(own, 1e-3)
    assert passes(parity.assert_calibrated, tiny_rep(grads=dict(grads, x=(edge, own))))
    assert not passes(parity.assert_calibrated, tiny_rep(grads=dict(grads, x=(edge * OVER, own))))


def test_tiny_missing_and_nan_fail():
    assert passes(parity.assert_calibrated, tiny_rep())
    assert not passes(parity.assert_calibrated, tiny_rep(missing=["conv_out.bias"]))
    assert not passes(parity.assert_calibrated, tiny_rep(grads={f"g{i}": (1e-3, 1e-3) for i in range(5)} | {"x": (math.nan, 1e-3)}))
    assert not passes(parity.assert_calibrated, tiny_rep(out=[(math.nan, 1e-3)]))


# ---------------------------------------------------------------- full width
def full_rep(out=((1e-3, 1e-3),), grads=None, undefined=None, absmax=1.0, missing=()):
    """100 defined gradients at (1e-3, 1e-3) unless given; `undefined` {name: (max|ours|, max|reference|)}."""
    grads = dict(grads or {f"g{i}": (1e-3, 1e-3) for i in range(100)})
    rep = {"out": list(out), "missing": list(missing), "grad_typical": 1.0,
           "grad_absmax": {k: absmax for k in grads}, "grad_absmax_tf32": {k: absmax for k in grads}}
    for k, (ours, ref) in (undefined or {}).items():
        grads[k] = (1.0, 0.9)
        rep["grad_absmax"][k], rep["grad_absmax_tf32"][k] = ours, ref
    rep["grads"] = grads
    return rep


@pytest.mark.parametrize("ref", [2e-3, 1e-4])
def test_full_width_output_bound(ref):
    edge = max(1e-3, 1.5 * ref)
    assert passes(parity.assert_calibrated_full_width, full_rep(out=[(edge, ref)]))
    assert not passes(parity.assert_calibrated_full_width, full_rep(out=[(edge * OVER, ref)]))


def test_full_width_median_and_p90_bounds():
    # the median (index 50) and the 90th percentile (index 90) of 100 sorted errors, each at 1.25 x
    for idx in (50, 90):
        ours = [1e-3] * 100
        ours[idx:] = [1.25 * 1e-3] * (100 - idx)
        grads = {f"g{i}": (o, 1e-3) for i, o in enumerate(ours)}
        assert passes(parity.assert_calibrated_full_width, full_rep(grads=grads))
        ours[idx] = 1.25 * 1e-3 * OVER
        ours[idx + 1:] = [1.25 * 1e-3 * OVER] * (99 - idx)
        grads = {f"g{i}": (o, 1e-3) for i, o in enumerate(ours)}
        assert not passes(parity.assert_calibrated_full_width, full_rep(grads=grads))


@pytest.mark.parametrize("own", [1e-4, 2e-3])
def test_full_width_per_tensor_bound(own):
    grads = {f"g{i}": (1e-3, 1e-3) for i in range(100)}
    edge = 3.0 * max(own, 1e-3)
    assert passes(parity.assert_calibrated_full_width, full_rep(grads=dict(grads, x=(edge, own))))
    assert not passes(parity.assert_calibrated_full_width, full_rep(grads=dict(grads, x=(edge * OVER, own))))


def test_full_width_defined_threshold():
    grads = {f"g{i}": (1e-3, 1e-3) for i in range(100)}
    # reference error exactly 0.5: defined, so held to 3 x its reference error
    assert not passes(parity.assert_calibrated_full_width, full_rep(grads=dict(grads, x=(3.0 * 0.5 * OVER, 0.5))))
    # 1 % above: undefined, judged by magnitude only
    assert passes(parity.assert_calibrated_full_width, full_rep(grads=dict(grads, x=(3.0 * 0.5 * OVER, 0.5 * OVER))))


def test_full_width_undefined_share():
    grads = {f"g{i}": (1e-3, 1e-3) for i in range(95)}
    assert passes(parity.assert_calibrated_full_width, full_rep(grads=grads, undefined={f"u{i}": (0.0, 0.0) for i in range(5)}))
    # 6 of 100: more than 5 %
    grads = {f"g{i}": (1e-3, 1e-3) for i in range(94)}
    assert not passes(parity.assert_calibrated_full_width, full_rep(grads=grads, undefined={f"u{i}": (0.0, 0.0) for i in range(6)}))


@pytest.mark.parametrize("ref_absmax", [1e-2, 1e-4])  # the reference's own magnitude, and 1e-3 x the typical one
def test_full_width_undefined_magnitude(ref_absmax):
    grads = {f"g{i}": (1e-3, 1e-3) for i in range(99)}
    edge = 3.0 * max(ref_absmax, 1e-3 * 1.0)
    assert passes(parity.assert_calibrated_full_width, full_rep(grads=grads, undefined={"u": (edge, ref_absmax)}))
    assert not passes(parity.assert_calibrated_full_width, full_rep(grads=grads, undefined={"u": (edge * OVER, ref_absmax)}))


def test_full_width_missing_and_nan_fail():
    assert passes(parity.assert_calibrated_full_width, full_rep())
    assert not passes(parity.assert_calibrated_full_width, full_rep(missing=["conv_out.bias"]))
    grads = {f"g{i}": (1e-3, 1e-3) for i in range(100)}
    assert not passes(parity.assert_calibrated_full_width, full_rep(grads=dict(grads, x=(math.nan, 1e-3))))
    assert not passes(parity.assert_calibrated_full_width, full_rep(out=[(math.nan, 1e-3)]))


# ---------------------------------------------------------------- two engine runs
def _pair(delta):
    """(a, b) with max|b| = 1 and max|a - b| = delta exactly."""
    b = torch.tensor([0.0, 1.0, -0.5], dtype=torch.float64)
    return b + torch.tensor([delta, 0.0, 0.0], dtype=torch.float64), b


def test_same_run_output_bound():
    assert passes(lambda r: parity.assert_same_run(*r), ([_pair(parity.RUN_OUT)[0]], [_pair(parity.RUN_OUT)[1]]))
    a, b = _pair(parity.RUN_OUT * OVER)
    assert not passes(lambda r: parity.assert_same_run(*r), ([a], [b]))
    assert parity.RUN_OUT == 3e-3


def test_same_run_gradient_bound():
    def run(delta, extra=None):
        a, b = _pair(delta)
        grads, ref = {"w": a, "v": b.clone()}, {"w": b, "v": b.clone()}
        grads.update(extra or {})
        return passes(lambda _: parity.assert_same_run([], [], grads, ref), None)

    assert parity.RUN_GRAD == 2e-2
    assert run(parity.RUN_GRAD)
    assert not run(parity.RUN_GRAD * OVER)
    assert not run(0.0, {"u": torch.zeros(1)})  # a gradient only one run has
    assert not run(math.nan)


# ---------------------------------------------------------------- the metric and the floor
def test_rel_is_float64():
    a = torch.tensor([1.0 + 2 ** -20], dtype=torch.float32)
    b = torch.tensor([1.0], dtype=torch.float32)
    assert parity.rel(a, b) == 2 ** -20


def test_grad_floor_rule():
    ref = {"a": torch.tensor([1.0, -0.5]), "b": torch.tensor([2.0]), "c": torch.tensor([1e-4]), "d": torch.tensor([-4.0])}
    assert parity.grad_floor(ref) == pytest.approx(2e-2)  # 1e-2 x the upper median of (1e-4, 1, 2, 4)
    got = {"a": torch.tensor([1.5, -0.5]), "b": torch.tensor([2.0]), "c": torch.tensor([0.0]), "e": torch.tensor([9.0])}
    err = parity.grad_errors(got, ref)
    assert err.keys() == {"a", "b", "c"}  # ref's names that got holds
    assert err["a"] == pytest.approx(0.5) and err["b"] == 0.0
    assert err["c"] == pytest.approx(1e-4 / 2e-2)  # below the floor: judged on its scale
    del ref["d"]  # three tensors: the median is 1
    assert parity.grad_errors(got, ref)["c"] == pytest.approx(1e-4 / 1e-2)
    assert parity.grad_errors(got, ref, floor=False)["c"] == pytest.approx(1.0)


# ---------------------------------------------------------------- the oracle arm on the CPU
def test_oracle_arm_tiny_unet_fp64_and_fp32():
    _, oracle, sd = parity.tiny_model(tc.TINY_UNET)
    x, t, lm, mask = tc.seeded_inputs(3, 2, 16, 6)
    ws = [torch.randn(x.shape, generator=torch.Generator().manual_seed(11))]
    args = (sd, [x], t, lm, mask, {}, ws)
    f64 = parity.oracle_arm(oracle.forward, *args, torch.float64, "cpu")
    f32 = parity.oracle_arm(oracle.forward, *args, torch.float32, "cpu")
    for outs, grads in (f64, f32):
        assert len(outs) == 1 and outs[0].shape == x.shape and outs[0].dtype == torch.float64
        assert grads.keys() == sd.keys() and all(g.dtype == torch.float64 for g in grads.values())
    rep = parity.report(f32, f64, f32)
    assert rep["missing"] == [] and rep["grads"].keys() == sd.keys()
    (ours, ref), = rep["out"]
    assert ours == ref and 0 < ours < 1e-5  # fp32 round-off against fp64
    assert all(a == b and a < 1e-3 for a, b in rep["grads"].values())
    parity.assert_calibrated(rep)
    without = parity.report((f32[0], {k: v for k, v in f32[1].items() if k != "conv_out.bias"}), f64, f32)
    assert without["missing"] == ["conv_out.bias"]
    assert not passes(parity.assert_calibrated, without)
