"""Generate tests/golden/attention.npz by running the UNMODIFIED reference's SelfAttention.attention (spatial self and
cross branch) and SelfAttention1D.attention (lm_head tokens) in float64 on CPU, through tests/refharness.py:

    ML_MDM_ROOT=<checkout> python tests/golden/make_golden_attention.py

  spatial.{q,k,v,kc,vc,mask,heads}  inputs, (B,T,C) / (B,S,C); sample 1's keys are all masked, sample 2's mask holds
                                    the values 0.5 and 2
  spatial.{self,cross}              the reference's two branch outputs, (B,T,C); cross is NaN for sample 1
  token.{qkv,mask,heads,out}        the same for the token attention; sample 1's keys are all masked (out NaN)

The file is written with fixed zip timestamps, so that running this again reproduces it byte for byte.
"""
import io
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))

import refharness as rh  # noqa: E402


def spatial(ref, out):
    B, T, S, heads, d = 3, 20, 9, 2, 32
    Cc = heads * d
    g = torch.Generator().manual_seed(11)
    q, k, v = (torch.randn(B, T, Cc, generator=g, dtype=torch.float64) * 0.7 for _ in range(3))
    kc, vc = (torch.randn(B, S, Cc, generator=g, dtype=torch.float64) * 0.7 for _ in range(2))
    mask = torch.ones(B, S, dtype=torch.float64)
    mask[0, 6:] = 0
    mask[1] = 0
    mask[2] = torch.tensor([0.5, 0, 2, 2, 0, 0.5, 1, 0, 2], dtype=torch.float64)
    attn = ref.unet.SelfAttention(Cc, num_heads=heads).double()
    cf = lambda x: x.transpose(1, 2).contiguous()  # noqa: E731 -- the reference's (B, C, length) layout
    with torch.no_grad():
        h_self = attn.attention(cf(q), cf(k), cf(v)).transpose(1, 2)
        h_cross = attn.attention(cf(q), cf(kc), cf(vc), mask).transpose(1, 2)
    for n, t in (("q", q), ("k", k), ("v", v), ("kc", kc), ("vc", vc), ("mask", mask), ("self", h_self),
                 ("cross", h_cross)):
        out["spatial." + n] = t.contiguous().numpy()
    out["spatial.heads"] = np.array(heads)


def token(ref, out):
    B, T, heads, d = 3, 12, 2, 16
    D = heads * d
    g = torch.Generator().manual_seed(12)
    qkv = torch.randn(B, T, 3 * D, generator=g, dtype=torch.float64) * 0.7
    mask = torch.ones(B, T, dtype=torch.float64)
    mask[0, 9:] = 0
    mask[1] = 0
    mask[2, ::3] = 0
    attn = ref.unet.SelfAttention1D(D, num_heads=heads).double()
    q, k, v = qkv.chunk(3, dim=2)
    with torch.no_grad():
        o = attn.attention(q, k, v, mask)
    out["token.qkv"], out["token.mask"], out["token.out"] = qkv.numpy(), mask.numpy(), o.contiguous().numpy()
    out["token.heads"] = np.array(heads)


def save(path, arrays):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    torch.set_num_threads(1)
    ref = rh.load()
    out = {}
    spatial(ref, out)
    token(ref, out)
    path = os.path.join(HERE, "attention.npz")
    save(path, out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
