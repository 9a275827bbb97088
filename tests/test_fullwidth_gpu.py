"""GPU: forward AND backward parity of the three shipped architectures at full width (cc12m_64x64: 461 M parameters,
cc12m_256x256: 2-level nest, cc12m_1024x1024: 3-level nest with per-sample std input normalisation on its middle
level, 1- and 3-channel GroupNorm groups at C = 32 / 96, K = 13824 weight gradients), explicit micro-conditioning
values on both sides of the clamp, ragged caption masks.

Arbiter: the oracle in float64 on the same GPU. Calibration: the oracle in float32 with TF32 enabled -- the arithmetic
the reference itself trains with (clis/train_parallel.py:18-19). The north star's "1e-3 relative" is what that path
scores on the OUTPUTS (0.6e-3 .. 1.5e-3 measured) and it scores ~3e-3 (median) to
~7e-3 (max) on parameter gradients; the bounds below are stated against those measured reference errors, tensor by
tensor, not as free constants:
  outputs     ours <= max(1e-3, 1.5 x reference-TF32 error of the same output)   (measured ratios 1.06 .. 1.42; both
              sides move by ~10 % run to run with the order of their fp32 atomics)
  gradients   median and 90th percentile over all parameters within 1.25 x of the reference-TF32's, and every single
              tensor within 3 x max(its reference-TF32 error, the median reference-TF32 error)
Gradients that are mathematically zero (a conv bias in front of a GroupNorm whose groups are single channels, C = 32)
are round-off on every implementation (reference-TF32 relative error > 0.5): their magnitude is checked against the
magnitude the reference-TF32 path leaves in the same tensor (or 1e-3 of the typical gradient, whichever is larger)."""
import pytest

import fullwidth_cases as fc
import parity
from oracle import unet_ref

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,batch", [("cc12m_64x64", 2), ("cc12m_256x256", 2), ("cc12m_1024x1024", 1)])
def test_forward_backward_full_width_calibrated_against_reference_tf32(name, batch):
    m, ocfg = fc.build(name)
    parity.assert_calibrated_full_width(fc.run_case(name, m, unet_ref.OracleNet(ocfg, 2048), B=batch, S=8, micro=True))
