"""Fused attention operator (wgmma flash-style forward + backward) against the fp64 restatement of
SelfAttention.attention (reference models/unet.py:276-307) on the same fp16 operands, element by element:
|got - ref| <= C 2^-11 mag for h, the self-branch output and dQ, dK, dV, dK_c, dV_c (tests/attn_cases.py). Every
output and scratch buffer starts as NaN; a sample whose keys are all masked gets exactly the self branch and zero
dK_c, dV_c."""
import pytest

import attn_cases as ac

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(ac.SPATIAL))
def test_attention_case(name):
    ratios = ac.run_spatial(name)
    print(name, {k: round(v, 3) for k, v in ratios.items()})
    for k, v in ratios.items():
        assert v <= ac.C, (name, k, v)
