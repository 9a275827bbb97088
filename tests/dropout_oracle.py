"""Oracle of the ResNet dropout (ResNetConfig.dropout; test infrastructure only). Extends oracle/unet_ref.OracleNet so
that every ResNet multiplies SiLU(norm2(h) * (1 + ta) + tb) by a given mask before conv2 (reference models/unet.py:208,
233-235), in the same plain functional torch (fp32 or fp64). torch's dropout generator cannot be reproduced by another
implementation, so the masks are inputs: the reference's own (tests/golden/dropout.npz, written by
tests/golden/make_golden_dropout.py) or the engine's, rebuilt with mdm_op_dropout_mask."""
import os
import sys

import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import unet_ref  # noqa: E402


def resnet(P, pre, x, temb, cin, cout, groups, mask):
    """ResNet.forward (unet.py:223-238) with h = dropout(h) as h * mask; mask: (N, cout, H, W) factors 0 or 1/(1-p)."""
    h = F.conv2d(F.silu(unet_ref._gn(x, P, pre + ".norm1", groups)), P[pre + ".conv1.weight"],
                 P[pre + ".conv1.bias"], padding=1)
    t = F.linear(F.silu(temb), P[pre + ".time_layer.weight"], P[pre + ".time_layer.bias"])
    ta, tb = t[:, :cout, None, None], t[:, cout:, None, None]
    h = F.silu(unet_ref._gn(h, P, pre + ".norm2", groups) * (1 + ta) + tb)
    h = h * mask.to(device=h.device, dtype=h.dtype)
    h = F.conv2d(h, P[pre + ".conv2.weight"], P[pre + ".conv2.bias"], padding=1)
    if cin != cout:
        x = F.conv2d(x, P[pre + ".conv3.weight"], P[pre + ".conv3.bias"])
    return h + x


class OracleNet(unet_ref.OracleNet):
    """unet_ref.OracleNet whose ResNets apply dropout masks. masks(prefix, shape) returns the mask of the ResNet with
    that state_dict prefix (e.g. "inner_unet.down_blocks.0.resnets.1") for its (N, C, H, W) activation."""

    def __init__(self, cfg, lm_dim, masks):
        super().__init__(cfg, lm_dim)
        self.masks = masks

    def forward(self, *args, **kwargs):
        plain = unet_ref.resnet

        def with_mask(P, pre, x, temb, cin, cout, groups):
            n, _, hh, ww = x.shape
            return resnet(P, pre, x, temb, cin, cout, groups, self.masks(pre, (n, cout, hh, ww)))

        unet_ref.resnet = with_mask  # res_block looks the ResNet up in its module at call time
        try:
            return super().forward(*args, **kwargs)
        finally:
            unet_ref.resnet = plain
