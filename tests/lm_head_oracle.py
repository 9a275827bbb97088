"""Oracle of the lm_head layers (UNetConfig.num_lm_head_layers; test infrastructure only). Extends
oracle/unet_ref.OracleNet with the SelfAttention1DBlocks that UNet.forward_conditioning runs on the projected tokens
(reference models/unet.py:316-446, 847-865), in the same plain functional torch (fp32 or fp64). Pinned against
tests/golden/lm_head.npz, generated from the unmodified reference by tests/golden/make_golden_lm_head.py."""
import os
import sys

import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import unet_ref  # noqa: E402


def lm_head_layer(P, pre, x, mask, heads=8):
    """SelfAttention1DBlock.forward: SelfAttention1D (no FFN) then MLP, on tokens x (B,S,D)."""
    dim = x.shape[-1]
    h = F.layer_norm(x, (dim,), P[pre + ".attn.norm.weight"], P[pre + ".attn.norm.bias"], eps=1e-5)
    qkv = F.linear(h, P[pre + ".attn.qkv.weight"], P[pre + ".attn.qkv.bias"])
    q, k, v = (t.transpose(1, 2) for t in qkv.chunk(3, dim=-1))  # (B,D,S): channels head-major as in _attend
    a = unet_ref._attend(q, k, v, heads, mask).transpose(1, 2)
    x = x + F.linear(a, P[pre + ".attn.proj_out.weight"], P[pre + ".attn.proj_out.bias"])
    h = F.layer_norm(x, (dim,), P[pre + ".mlp.main.0.weight"], P[pre + ".mlp.main.0.bias"], eps=1e-5)
    h = F.gelu(F.linear(h, P[pre + ".mlp.main.1.weight"], P[pre + ".mlp.main.1.bias"]))
    return x + F.linear(h, P[pre + ".mlp.main.3.weight"], P[pre + ".mlp.main.3.bias"])


def num_lm_head_layers(plan):
    """The layers exist only beside cond_emb (unet.py:760-771)."""
    return (unet_ref._get(plan.cfg, "num_lm_head_layers", 0) or 0) if plan.has_cond_emb else 0


def forward_conditioning(P, pre, plan, lm, mask):
    """UNet.forward_conditioning with lm_head: the layers get the mask only with masked_cross_attention, and with
    lm_head present and masked_cross_attention == 0 the pooled y is the plain mean over all tokens."""
    nl = num_lm_head_layers(plan)
    cond = lm
    if plan.has_lm_proj:
        cond = F.linear(cond, P[pre + "lm_proj.weight"], P[pre + "lm_proj.bias"])
    for i in range(nl):
        cond = lm_head_layer(P, f"{pre}lm_head.{i}", cond, mask if plan.masked_cross_attention else None)
    if mask is None or (not plan.masked_cross_attention and nl > 0):
        y = cond.mean(dim=1)
    else:
        y = (mask.unsqueeze(-1) * cond).sum(dim=1) / mask.sum(dim=1, keepdim=True)
    if not plan.masked_cross_attention:
        mask = None
    return F.linear(y, P[pre + "cond_emb.weight"]), cond, mask


class OracleNet(unet_ref.OracleNet):
    """unet_ref.OracleNet whose text conditioning runs the lm_head layers."""

    def forward(self, P, x_t, times, lm, lm_mask, micros=None, trace=None):
        ipre, iplan, _ = self.levels[-1]
        cond_emb, cond, cmask = None, lm, lm_mask
        if iplan.cond_dim > 0:
            cond_emb, cond, cmask = forward_conditioning(P, ipre, iplan, lm, lm_mask)
        if not self.nested:
            return unet_ref.unet_denoise(P, "", iplan, x_t, times, cond_emb, cond, cmask, micros, trace)
        return self._nested(0, P, x_t, None, times, cond_emb, cond, cmask, micros, trace)
