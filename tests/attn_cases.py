"""The fused attention operators (mdm_op_attention_fwd / _bwd: the spatial self + cross attention of
SelfAttention.attention, reference models/unet.py:276-307; mdm_op_token_attention_fwd / _bwd: the masked token
attention of SelfAttention1D.attention, unet.py:354-377) against an fp64 restatement, element by element.

Bound: |got - ref| <= C * 2^-11 * mag for every element of every output tensor, where `mag` is the same fp64
expression with |.| on every operand plus a term for each point where the kernels round to fp16:
  forward   mag_out[t,j] = sum_branch sum_s (P_ts + 2^-13) |v_sj|   (fp16 P; 2^-13 covers its underflow)
  dS        magdS_ts = alpha (P_ts + 2^-13) (sum_j |dO_tj||v_sj| + sum_j |dO_tj| (|h_tj| + |oself_tj|))
            (D comes from the fp16 outputs; the token kernel has one output, |o_tj|)
  gradients mag_dV = sum_t (P_ts + 2^-13) |dO_tj|,  mag_dK = sum_t magdS_ts |q_tj|,
            mag_dQ = sum_branch sum_s magdS_ts |k_sj|
Masked keys contribute nothing to `mag`: the kernels set their P to exactly 0. A sample whose keys are all masked has
no softmax; the oracle gives it a zero branch (zero output, zero dK / dV), which is what both kernels document.

The same restatement runs as (a) the fp64 oracle, (b) a float32 emulation of the kernels' rounding points
(tests/test_attention_oracle.py: the bound holds with margin) and (c) with one deliberate change (`bug`: the bound is
sharp enough to reject it). Inputs: `flat` (q, k, v ~ 0.7 N(0, 1): scores of std ~0.5, a nearly uniform softmax, the
production statistics), `planted` (chosen keys carry >= 0.9 of the softmax of a few query rows and a large distinct
v, so that a kernel that loses one key fails) and `large` (scores of std ~6)."""
import ctypes as C_
import json
import math
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "ml-mdm_b200"))

U16 = 2.0 ** -11  # unit roundoff of fp16
P_FLOOR = 2.0 ** -13  # absolute error of an fp16 P that underflows
C = 3.5  # one constant for every output tensor of both kernels: 2x the worst ratio measured on an H100 (1.73,
# DESIGN.md section 3.1b)
TILE = 128  # key chunk / key tile of both kernels
PLANT_SCORE = 20.0  # alpha q . k of a planted (query row, key) pair

SPATIAL_OUT = ("out", "oself", "dq", "dk", "dv", "dkc", "dvc")
TOKEN_OUT = ("out", "dq", "dk", "dv")


# ------------------------------------------------------------------------------------------ the restatement
def _split(x, heads):  # (B, N, heads * d) -> (B, heads, N, d)
    B, N, Cc = x.shape
    return x.reshape(B, N, heads, Cc // heads).permute(0, 2, 1, 3)


def _merge(x):  # (B, heads, N, d) -> (B, N, heads * d)
    B, H, N, d = x.shape
    return x.permute(0, 2, 1, 3).reshape(B, N, H * d)


def oracle(q, branches, dO, heads, token=False, emu=False, bug=None, backward=True):
    """q (B,T,C); branches: [(k, v, mask)] with k, v (B,S,C) and mask (B,S) or None -- [self, cross] for the spatial
    operator, [self] for the token one; dO (B,T,C) or None. Returns (values, mags, P): dicts of (B,N,C) tensors named
    as SPATIAL_OUT / TOKEN_OUT, and the softmax of each branch (B,heads,T,S).

    emu=False: fp64. emu=True: float32 with the kernels' fp16 roundings (P before P V -- unnormalised where the kernel
    divides by the row sum afterwards --, the outputs, D from the fp16 outputs, P and dS before the gradient products,
    the gradients). `bug`: one deliberate change (test_attention_oracle.MUTANTS)."""
    dt = torch.float32 if emu else torch.float64
    r16 = (lambda x: x.half().to(dt)) if emu else (lambda x: x)
    B, T, Cc = q.shape
    d = Cc // heads
    alpha = 1.0 / math.sqrt(d)

    def sp(x):
        x = _split(x.to(dt), heads)
        if bug == "head_neighbour":  # the last head reads the columns of the one before it
            x = x.clone()
            x[:, -1] = x[:, -2]
        return x

    Q = sp(q)
    branches = list(branches)
    if bug == "swap_kv_c":
        k, v, m = branches[1]
        branches[1] = (v, k, m)
    fw = []
    for bi, (k, v, mask) in enumerate(branches):
        cross = bi == 1
        K, V = sp(k), sp(v)
        S = K.shape[2]
        if (bug == "cross_nomask" and cross) or (bug == "nomask" and token):
            mask = None
        keep = torch.ones(B, S, dtype=torch.bool, device=q.device) if mask is None else (mask != 0)
        if bug == "mask_next_sample" and mask is not None:
            keep = keep.roll(-1, 0)
        if bug == "mask_shift" and mask is not None:
            keep = keep.roll(1, 1)
        if bug == "drop_last":
            keep = keep.clone()
            keep[:, S - 1] = False
        if bug == "drop_128" and S > TILE:
            keep = keep.clone()
            keep[:, TILE] = False
        kp = keep[:, None, None, :]
        s = (Q @ K.transpose(-1, -2)) * alpha
        s = s.masked_fill(~kp, float("-inf"))
        m = s.amax(-1, keepdim=True)
        m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
        e = torch.exp(s - m)  # 0 for masked keys
        if bug == "mask_queries" and token and mask is not None:
            e = e * keep[:, None, :, None]
        l = e.sum(-1, keepdim=True)
        il = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
        if bug == "cross_self_l" and cross:
            il = fw[0]["il"]
        P = e * il
        deferred = not cross and T > TILE  # the kernels divide O by l after P V
        O = (r16(e) @ V) * il if (emu and deferred) else r16(P) @ V
        fw.append(dict(K=K, V=V, keep=kp, P=P, O=O, il=il))

    vals, mags = {}, {}
    if token:
        h = r16(fw[0]["O"])
        vals["out"] = h
        Dsrc = [h]
        magD_src = [h.abs()]
    else:
        oself = r16(fw[0]["O"])
        h = r16(fw[0]["O"] + fw[1]["O"]) if len(fw) > 1 else oself
        vals["out"], vals["oself"] = h, oself
        Dsrc = [oself, h - oself]
        magD_src = [h.abs() + oself.abs()] * 2
    mags["out"] = sum((f["P"] + P_FLOOR * f["keep"]) @ f["V"].abs() for f in fw)
    if not token:
        mags["oself"] = (fw[0]["P"] + P_FLOOR * fw[0]["keep"]) @ fw[0]["V"].abs()
    Pm = [f["P"] for f in fw]
    if not backward:
        return ({k: _merge(v) for k, v in vals.items()}, {k: _merge(v) for k, v in mags.items()}, Pm)

    G = sp(dO)
    dQ = torch.zeros_like(Q)
    mdQ = torch.zeros_like(Q)
    Ds = [(G * Dsrc[i]).sum(-1, keepdim=True) for i in range(len(fw))]
    if bug == "cross_D_self" and len(fw) > 1:
        Ds[1] = Ds[0]
    names = [("dk", "dv"), ("dkc", "dvc")]
    for bi, f in enumerate(fw):
        P, K, V, kp = f["P"], f["K"], f["V"], f["keep"]
        dP = G @ V.transpose(-1, -2)
        dS = P * (dP - Ds[bi]) * alpha
        dV = r16(r16(P).transpose(-1, -2) @ G)
        dK = r16(r16(dS).transpose(-1, -2) @ Q)
        if not (bug == "dq_no_cross" and bi == 1):
            dQ = dQ + r16(dS) @ K
        Pf = P + P_FLOOR * kp
        magD = (G.abs() * magD_src[bi]).sum(-1, keepdim=True)
        mdS = alpha * Pf * (G.abs() @ V.abs().transpose(-1, -2) + magD)
        S = K.shape[2]
        if bug == "last_tile_unwritten":
            k0 = (S - 1) // TILE * TILE
            dK, dV = dK.clone(), dV.clone()
            dK[:, :, k0:] = 0
            dV[:, :, k0:] = 0
        nk, nv = names[bi]
        vals[nk], vals[nv] = dK, dV
        mags[nk] = mdS.transpose(-1, -2) @ Q.abs()
        mags[nv] = Pf.transpose(-1, -2) @ G.abs()
        mdQ = mdQ + mdS @ K.abs()
    vals["dq"], mags["dq"] = r16(dQ), mdQ
    return ({k: _merge(v) for k, v in vals.items()}, {k: _merge(v) for k, v in mags.items()}, Pm)


def ref_attention(qkv, kv, mask, heads):
    """fp64 SelfAttention.attention of both branches: qkv (B,T,3C), kv (B,S,2C) or None, mask (B,S) or None ->
    (out, oself), each (B,T,C). A cross branch whose keys are all masked is zero (the reference gives NaN)."""
    q, k, v = qkv.double().chunk(3, dim=2)
    br = [(k, v, None)]
    if kv is not None:
        kc, vc = kv.double().chunk(2, dim=2)
        br.append((kc, vc, mask))
    vals, _, _ = oracle(q, br, None, heads, backward=False)
    return vals["out"], vals["oself"]


def ref_token_attention(qkv, mask, heads):
    """fp64 SelfAttention1D.attention: qkv (B,T,3D), mask (B,T) or None -> (B,T,D); zero for a sample whose keys are
    all masked (the reference gives NaN)."""
    q, k, v = qkv.double().chunk(3, dim=2)
    vals, _, _ = oracle(q, [(k, v, mask)], None, heads, token=True, backward=False)
    return vals["out"]


def ratio(got, ref, mag):
    """max |got - ref| / (2^-11 mag): the smallest C under which `got` passes (inf for a non-finite element, 0/0 = 0)."""
    got = got.to(ref.device).double()
    diff = (got - ref.double()).abs()
    r = diff / (U16 * mag.double())
    r = torch.where(diff == 0, torch.zeros_like(r), r)
    r = torch.where(torch.isfinite(got), r, torch.full_like(r, float("inf")))
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------ inputs
def prefix(S, n):
    m = torch.zeros(S)
    m[:n] = 1
    return m


def scattered(S, seed, p=0.7, keep=()):
    """A random key mask that keeps about p of the keys, at least one, and every key of `keep`."""
    g = torch.Generator().manual_seed(seed)
    m = (torch.rand(S, generator=g) < p).float()
    m[int(torch.randint(S, (1,), generator=g))] = 1
    for s in keep:
        m[s] = 1
    return m


def _plant(q, k, v, b, s, h, d, i, rows):
    """Makes key s of head h in sample b carry >= 0.9 of the softmax of query rows `rows` (alpha q . k = PLANT_SCORE
    with a key three times the typical length, so the other keys stay far below) and gives it a large distinct v."""
    cols = slice(h * d, (h + 1) * d)
    ks = k[b, s, cols]
    ks = ks / ks.norm() * (2.1 * math.sqrt(d))
    k[b, s, cols] = ks
    for t in rows:
        q[b, t, cols] = ks * (PLANT_SCORE * math.sqrt(d) / float(ks.norm()) ** 2)
    g = torch.Generator().manual_seed(1000 + i)
    v[b, s, cols] = (2.0 + 0.5 * (i % 4)) * torch.sign(torch.randn(d, generator=g) + 1e-3)


def plant_rows(i, T):
    return sorted({(5 + 37 * i) % T, (23 + 37 * i) % T})


def make_spatial(spec):
    """CPU fp16 inputs of one spatial case: dict(qkv (B,T,3C), kv (B,S,2C) or None, mask (B,S) or None, dO (B,T,C),
    plants [(branch, b, head, key, rows)])."""
    B, T, S, d, heads = spec["B"], spec["T"], spec["S"], spec["d"], spec.get("heads", 8)
    Cc = d * heads
    g = torch.Generator().manual_seed(spec.get("seed", 0))
    sig = math.sqrt(6.0) if spec.get("mode") == "large" else 0.7  # large: alpha q . k has std 6
    q = torch.randn(B, T, Cc, generator=g) * sig
    k = torch.randn(B, T, Cc, generator=g) * sig
    v = torch.randn(B, T, Cc, generator=g) * 0.7
    kc = torch.randn(B, S, Cc, generator=g) * sig
    vc = torch.randn(B, S, Cc, generator=g) * 0.7
    dO = torch.randn(B, T, Cc, generator=g) * 0.5
    mask = torch.stack([m if m is not None else torch.ones(S) for m in spec["masks"]]) if spec.get("masks") else None
    plants = []
    for i, (br, b, s) in enumerate(spec.get("plants", ())):
        h = i % heads
        rows = plant_rows(i, T)
        if br == 0:
            _plant(q, k, v, b, s, h, d, i, rows)
        else:
            assert mask is None or mask[b, s] != 0
            _plant(q, kc, vc, b, s, h, d, i, rows)
        plants.append((br, b, h, s, rows))
    return dict(qkv=torch.cat([q, k, v], 2).half(), kv=torch.cat([kc, vc], 2).half() if S > 0 else None,
                mask=mask, dO=dO.half(), plants=plants, heads=heads)


def make_token(spec):
    """CPU fp16 inputs of one token case: dict(qkv (B,T,3D), mask (B,T) or None, dO (B,T,D), plants)."""
    B, T, d, heads = spec["B"], spec["T"], spec["d"], spec.get("heads", 8)
    D = d * heads
    g = torch.Generator().manual_seed(spec.get("seed", 0))
    q, k, v = (torch.randn(B, T, D, generator=g) * 0.7 for _ in range(3))
    dO = torch.randn(B, T, D, generator=g) * 0.5
    mask = torch.stack([m if m is not None else torch.ones(T) for m in spec["masks"]]) if spec.get("masks") else None
    plants = []
    for i, (b, s) in enumerate(spec.get("plants", ())):
        assert mask is None or mask[b, s] != 0
        h = i % heads
        rows = plant_rows(i, T)
        _plant(q, k, v, b, s, h, d, i, rows)
        plants.append((0, b, h, s, rows))
    return dict(qkv=torch.cat([q, k, v], 2).half(), mask=mask, dO=dO.half(), plants=plants, heads=heads)


def spatial_oracle(x, device="cpu", **kw):
    q, k, v = x["qkv"].to(device).double().chunk(3, dim=2)
    br = [(k, v, None)]
    if x["kv"] is not None:
        kc, vc = x["kv"].to(device).double().chunk(2, dim=2)
        br.append((kc, vc, x["mask"].to(device) if x["mask"] is not None else None))
    return oracle(q, br, x["dO"].to(device).double(), x["heads"], **kw)


def token_oracle(x, device="cpu", **kw):
    q, k, v = x["qkv"].to(device).double().chunk(3, dim=2)
    m = x["mask"].to(device) if x["mask"] is not None else None
    return oracle(q, [(k, v, m)], x["dO"].to(device).double(), x["heads"], token=True, **kw)


def planted_mass(P, plants):
    """The smallest softmax share a planted key holds in its query rows."""
    return min((float(P[br][b, h, t, s]) for br, b, h, s, rows in plants for t in rows), default=1.0)


def _old_mask(B, S):  # the masks of the first version of these tests: sample i keeps keys < S / 2 + i
    return [prefix(S, S // 2 + i) for i in range(B)]


# The spatial cases. Production level 1 is cc12m_64x64 (64x64 pixels, 512 channels at 32x32); level 2 its 16x16
# inner level at 768 channels. T <= 128 with S > 128 runs one self chunk and several cross chunks (pass 0 rescales the
# cross row sum online); "keys >= 130" masks a whole cross chunk.
SPATIAL = {
    "l1_cc12m_64x64": dict(B=2, T=1024, S=128, d=64, masks=[prefix(128, 128), prefix(128, 77)],
                           plants=[(0, 0, 0), (0, 1, 1023), (0, 0, 127), (0, 1, 128),
                                   (1, 0, 0), (1, 0, 127), (1, 1, 76)]),
    "l2_three_masks": dict(B=3, T=256, S=128, d=96, masks=[prefix(128, 128), prefix(128, 1), prefix(128, 100)],
                           plants=[(0, 0, 0), (0, 1, 255), (0, 2, 127), (0, 0, 128),
                                   (1, 1, 0), (1, 0, 127), (1, 2, 99)]),
    "bench_like": dict(B=2, T=256, S=128, d=96),
    "nonsquare_12x20": dict(B=2, T=240, S=77, d=64, masks=[prefix(77, 77), prefix(77, 23)]),
    "t1_s1_d8": dict(B=2, T=1, S=1, d=8),
    "self1_cross2": dict(B=2, T=64, S=129, d=96, masks=[prefix(129, 129), scattered(129, 11)],
                         plants=[(1, 0, 128), (1, 0, 127), (0, 1, 63), (0, 0, 0)]),
    "cross_chunk0_masked": dict(B=2, T=65, S=300, d=40,
                                masks=[scattered(300, 12, keep=(128,)), torch.arange(300).ge(130).float()],
                                plants=[(1, 1, 130), (1, 1, 299), (1, 0, 128), (0, 0, 64)]),
    "nocross_t129": dict(B=2, T=129, S=0, d=72, plants=[(0, 0, 128), (0, 1, 127), (0, 1, 0)]),
    "t127_s128_d104": dict(B=2, T=127, S=128, d=104, masks=[scattered(128, 13), scattered(128, 14)]),
    "t128_s257_d128": dict(B=2, T=128, S=257, d=128, masks=[scattered(257, 15, keep=(128, 256)), scattered(257, 16)],
                           plants=[(1, 0, 256), (1, 0, 128), (0, 1, 127)]),
    "t257_s1_d24": dict(B=3, T=257, S=1, d=24),
    "t384_s130_d80": dict(B=1, T=384, S=130, d=80),
    "fully_masked": dict(B=3, T=256, S=128, d=64, masks=[prefix(128, 128), prefix(128, 0), prefix(128, 50)]),
    "fully_masked_chunks": dict(B=2, T=130, S=260, d=64, masks=[prefix(260, 0), prefix(260, 200)]),
    "mask_values": dict(B=2, T=128, S=77, d=64,
                        masks=[scattered(77, 17) * torch.tensor([0.5, 2.0]).repeat(39)[:77],
                               scattered(77, 18) * 2.0]),
    "large_logits": dict(B=2, T=1024, S=128, d=64, mode="large", masks=[prefix(128, 128), prefix(128, 60)]),
    "heads4": dict(B=2, T=256, S=77, d=64, heads=4, masks=[scattered(77, 19), prefix(77, 77)]),
    # the first version's cases
    "t256_d96_s128": dict(B=2, T=256, S=128, d=96),
    "t1024_d64_s128": dict(B=1, T=1024, S=128, d=64),
    "t16_d8_s6_masked": dict(B=2, T=16, S=6, d=8, masks=_old_mask(2, 6)),
    "t200_d32_s77_masked": dict(B=2, T=200, S=77, d=32, masks=_old_mask(2, 77)),
    "t256_d64_nocross": dict(B=2, T=256, S=0, d=64),
    "t384_d96_s130": dict(B=1, T=384, S=130, d=96),
}
for _i, _s in enumerate(SPATIAL.values()):
    _s.setdefault("seed", _i)


def token_grid_spec(d, T, masked):
    """The (d, T, masked) grid of the first token tests: sample i keeps keys < max(1, T / 2 + i)."""
    B = 4 if d * T <= 64 * 128 else 2
    masks = [prefix(T, max(1, T // 2 + i)) for i in range(B)] if masked else None
    return dict(B=B, T=T, d=d, masks=masks, seed=d * 1000 + T)


# Token cases beyond the grid: several key chunks with planted keys at the chunk boundary and the end, head widths
# whose second 128-column half is partly filled, and a sample whose keys are all masked.
TOKEN = {}
for _T in (129, 257):
    for _d in (64, 256):
        TOKEN[f"planted_t{_T}_d{_d}"] = dict(B=2, T=_T, d=_d, masks=[prefix(_T, _T), prefix(_T, _T - 20)],
                                             plants=[(0, 127), (0, 128), (0, _T - 1), (1, _T - 21), (1, 0)],
                                             seed=_T + _d)
for _d in (136, 192):
    for _T in (77, 200):
        TOKEN[f"half_t{_T}_d{_d}"] = dict(B=2, T=_T, d=_d, masks=[scattered(_T, _d + _T), None], seed=_d * 7 + _T)
for _d, _T in ((64, 77), (256, 77), (64, 200), (256, 200)):
    TOKEN[f"fully_masked_t{_T}_d{_d}"] = dict(B=3, T=_T, d=_d, masks=[prefix(_T, _T), prefix(_T, 0), prefix(_T, 30)],
                                              seed=_d + 3 * _T)


def fully_masked_samples(mask):
    return [] if mask is None else [b for b in range(mask.shape[0]) if not bool((mask[b] != 0).any())]


# ------------------------------------------------------------------------------------------ the kernels
def _ptr(t):
    return C_.c_void_p(t.data_ptr()) if t is not None else None


def run_spatial(name_or_spec):
    """Runs mdm_op_attention_fwd / _bwd on NaN-filled outputs, checks what the kernels own against the fp64 oracle
    (evaluated on the GPU) and returns the ratio of each output tensor (see `ratio`)."""
    from mdm_b200 import _lib

    spec = SPATIAL[name_or_spec] if isinstance(name_or_spec, str) else name_or_spec
    x = make_spatial(spec)
    B, T, S, heads = spec["B"], spec["T"], spec["S"], x["heads"]
    Cc = spec["d"] * heads
    dev = "cuda"
    nan = float("nan")
    qc, dOc = x["qkv"].to(dev), x["dO"].to(dev)
    kc = x["kv"].to(dev) if x["kv"] is not None else None
    mc = x["mask"].to(dev) if x["mask"] is not None else None
    h16 = torch.full((B, T, Cc), nan, device=dev, dtype=torch.float16)
    os16 = torch.full_like(h16, nan)
    stats = torch.full((B, heads, 2, T, 2), nan, device=dev)
    Dterm = torch.full((B, heads, 2, T), nan, device=dev)
    dq32 = torch.full((B, T, Cc), nan, device=dev)
    dqkv = torch.full((B, T, 3 * Cc), nan, device=dev, dtype=torch.float16)
    dkv = torch.full((B, max(S, 1), 2 * Cc), nan, device=dev, dtype=torch.float16)
    lib = _lib.lib()
    st = C_.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.mdm_op_attention_fwd(_ptr(qc), _ptr(kc), _ptr(mc), B, T, S, Cc, heads, _ptr(h16), _ptr(os16),
                                        _ptr(stats), st), "attn fwd")
    _lib.check(lib.mdm_op_attention_bwd(_ptr(qc), _ptr(kc), _ptr(mc), _ptr(dOc), _ptr(h16), _ptr(os16), _ptr(stats),
                                        B, T, S, Cc, heads, _ptr(Dterm), _ptr(dq32), _ptr(dqkv),
                                        _ptr(dkv) if S > 0 else None, st), "attn bwd")
    torch.cuda.synchronize()

    vals, mags, P = spatial_oracle(x, dev)
    assert planted_mass(P, x["plants"]) >= 0.9, planted_mass(P, x["plants"])
    got = {"out": h16, "oself": os16, "dq": dqkv[..., :Cc], "dk": dqkv[..., Cc:2 * Cc], "dv": dqkv[..., 2 * Cc:]}
    if S > 0:
        got["dkc"], got["dvc"] = dkv[..., :Cc], dkv[..., Cc:]
    for k in (k for k in got if k in vals):
        assert bool(torch.isfinite(got[k]).all()), (k, "non-finite or unwritten elements")
    # the statistics and D of every row are written; m of a row whose keys are all masked is -inf
    full = fully_masked_samples(x["mask"])
    branches = 2 if S > 0 else 1
    st_ = stats[:, :, :branches]
    assert not bool(torch.isnan(st_).any()) and not bool(torch.isnan(Dterm[:, :, :branches]).any())
    fin = torch.isfinite(st_)
    for b in full:
        fin[b, :, 1, :, 0] = True
    assert bool(fin.all()), "infinite row statistics"
    for b in full:  # documented: a zero cross branch and zero dK_c, dV_c
        assert torch.equal(h16[b].view(torch.int16), os16[b].view(torch.int16)), b
        assert bool((dkv[b] == 0).all()), b
    return {k: ratio(got[k], vals[k], mags[k]) for k in got if k in vals}


def run_token(spec):
    """Runs mdm_op_token_attention_fwd / _bwd on NaN-filled outputs against the fp64 oracle; ratios per tensor."""
    from mdm_b200 import _lib

    x = make_token(spec)
    B, T, heads = spec["B"], spec["T"], x["heads"]
    D = spec["d"] * heads
    dev = "cuda"
    nan = float("nan")
    qc, dOc = x["qkv"].to(dev), x["dO"].to(dev)
    mc = x["mask"].to(dev) if x["mask"] is not None else None
    o16 = torch.full((B, T, D), nan, device=dev, dtype=torch.float16)
    stats = torch.full((B, heads, T, 2), nan, device=dev)
    Dterm = torch.full((B, heads, T), nan, device=dev)
    dq32 = torch.full((B, T, D), nan, device=dev)
    dqkv = torch.full((B, T, 3 * D), nan, device=dev, dtype=torch.float16)
    lib = _lib.lib()
    st = C_.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.mdm_op_token_attention_fwd(_ptr(qc), _ptr(mc), B, T, D, heads, _ptr(o16), _ptr(stats), st),
               "token attn fwd")
    _lib.check(lib.mdm_op_token_attention_bwd(_ptr(qc), _ptr(mc), _ptr(dOc), _ptr(o16), _ptr(stats), B, T, D, heads,
                                              _ptr(Dterm), _ptr(dq32), _ptr(dqkv), st), "token attn bwd")
    torch.cuda.synchronize()

    vals, mags, P = token_oracle(x, dev)
    assert planted_mass(P, x["plants"]) >= 0.9, planted_mass(P, x["plants"])
    got = {"out": o16, "dq": dqkv[..., :D], "dk": dqkv[..., D:2 * D], "dv": dqkv[..., 2 * D:]}
    for k in got:
        assert bool(torch.isfinite(got[k]).all()), (k, "non-finite or unwritten elements")
    full = fully_masked_samples(x["mask"])
    assert not bool(torch.isnan(stats).any()) and not bool(torch.isnan(Dterm).any())
    fin = torch.isfinite(stats)
    for b in full:
        fin[b, :, :, 0] = True
    assert bool(fin.all()), "infinite row statistics"
    for b in full:  # documented: zero outputs and gradients
        assert bool((o16[b] == 0).all()) and bool((dqkv[b] == 0).all()), b
    return {k: ratio(got[k], vals[k], mags[k]) for k in got}


def worst(results):
    """{case: {tensor: ratio}} -> {tensor: (worst ratio, case)}."""
    w = {}
    for name, r in results.items():
        for k, v in r.items():
            if k not in w or v > w[k][0]:
                w[k] = (v, name)
    return w


if __name__ == "__main__":
    # python tests/attn_cases.py [out.json]: every case of both kernels, the ratio per output tensor and the worst
    import time

    res = {"spatial": {}, "token": {}}
    t0 = time.time()
    for name in SPATIAL:
        res["spatial"][name] = run_spatial(name)
        print("spatial", name, {k: round(v, 3) for k, v in res["spatial"][name].items()}, flush=True)
    grid = {f"grid_d{d}_t{T}_{'m' if m else 'u'}": token_grid_spec(d, T, m)
            for d in (8, 64, 128, 256) for T in (1, 6, 77, 128, 200) for m in (False, True)}
    for name, spec in {**grid, **TOKEN}.items():
        res["token"][name] = run_token(spec)
        print("token", name, {k: round(v, 3) for k, v in res["token"][name].items()}, flush=True)
    res["worst"] = {kind: worst(res[kind]) for kind in ("spatial", "token")}
    print("worst", json.dumps(res["worst"]), f"{time.time() - t0:.1f} s", flush=True)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)
    bad = [(kind, k, v) for kind in ("spatial", "token") for k, (v, _) in res["worst"][kind].items() if v > C]
    print("C =", C, "failures:", bad)
    sys.exit(1 if bad else 0)
