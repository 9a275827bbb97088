"""The attention oracle of tests/attn_cases.py without a GPU: pinned to the reference's own outputs
(tests/golden/attention.npz, tests/golden/make_golden_attention.py), the bound of the GPU tests shown to be loose
enough (a float32 emulation of the kernels' fp16 rounding points passes it with 2x margin) and sharp (the fp64 oracle
with one deliberate change violates it)."""
import os

import numpy as np
import pytest
import torch

import attn_cases as ac

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "attention.npz"))

# the cases small enough for the CPU (T <= 257)
SMALL = [n for n, s in ac.SPATIAL.items() if s["T"] <= 257 and s["T"] * max(s["S"], 1) * s["B"] <= 2 ** 17]
TOKEN_SMALL = [n for n in ac.TOKEN if "d256" not in n and "d192" not in n]


@pytest.fixture(scope="module", autouse=True)
def _threads():
    n = torch.get_num_threads()
    torch.set_num_threads(min(n, 8))
    yield
    torch.set_num_threads(n)


_cache = {}


def spatial(name):
    if name not in _cache:
        x = ac.make_spatial(ac.SPATIAL[name])
        _cache[name] = (x,) + ac.spatial_oracle(x)
    return _cache[name]


def token(name):
    if name not in _cache:
        x = ac.make_token(ac.TOKEN[name])
        _cache[name] = (x,) + ac.token_oracle(x)
    return _cache[name]


# ------------------------------------------------------------------------------------------ pinned to the reference
def test_spatial_oracle_matches_reference():
    q, k, v, kc, vc = (torch.from_numpy(GOLD["spatial." + n]) for n in ("q", "k", "v", "kc", "vc"))
    mask = torch.from_numpy(GOLD["spatial.mask"])
    heads = int(GOLD["spatial.heads"])
    out, oself = ac.ref_attention(torch.cat([q, k, v], 2), torch.cat([kc, vc], 2), mask, heads)
    ref_self, ref_cross = (torch.from_numpy(GOLD["spatial." + n]) for n in ("self", "cross"))
    # the reference computes its softmax in float32 (`weight.float()`), also when run in float64
    tol = 1e-6
    assert float((oself - ref_self).abs().max() / ref_self.abs().max()) <= tol
    full = ac.fully_masked_samples(mask)
    assert full == [1]
    kept = [b for b in range(mask.shape[0]) if b not in full]
    ref_out = (ref_self + ref_cross)[kept]
    assert float((out[kept] - ref_out).abs().max() / ref_out.abs().max()) <= tol
    # where every key is masked the reference's cross branch is NaN; the oracle (and the kernel) give zero
    assert bool(torch.isnan(ref_cross[full]).all())
    assert torch.equal(out[full], oself[full])


def test_token_oracle_matches_reference():
    qkv = torch.from_numpy(GOLD["token.qkv"])
    mask = torch.from_numpy(GOLD["token.mask"])
    out = ac.ref_token_attention(qkv, mask, int(GOLD["token.heads"]))
    ref = torch.from_numpy(GOLD["token.out"])
    full = ac.fully_masked_samples(mask)
    assert full == [1]
    kept = [0, 2]
    assert float((out[kept] - ref[kept]).abs().max() / ref[kept].abs().max()) <= 1e-6
    assert bool(torch.isnan(ref[full]).all())
    assert bool((out[full] == 0).all())


# ------------------------------------------------------------------------------------------ not too tight
@pytest.mark.parametrize("name", SMALL)
def test_emulated_kernel_passes_with_margin(name):
    x, vals, mags, P = spatial(name)
    emu, _, _ = ac.spatial_oracle(x, emu=True)
    for k in vals:
        assert ac.ratio(emu[k], vals[k], mags[k]) <= ac.C / 2, (name, k)
    assert ac.planted_mass(P, x["plants"]) >= 0.9


@pytest.mark.parametrize("name", TOKEN_SMALL)
def test_emulated_token_kernel_passes_with_margin(name):
    x, vals, mags, P = token(name)
    emu, _, _ = ac.token_oracle(x, emu=True)
    for k in vals:
        assert ac.ratio(emu[k], vals[k], mags[k]) <= ac.C / 2, (name, k)
    assert ac.planted_mass(P, x["plants"]) >= 0.9


# ------------------------------------------------------------------------------------------ sharp
SPATIAL_MUTANTS = {
    "drop_last": "the last key of each branch is ignored",
    "drop_128": "key 128 is ignored",
    "mask_next_sample": "sample b reads the mask of sample b + 1",
    "mask_shift": "the mask is shifted by one key",
    "cross_nomask": "the cross branch ignores the mask",
    "cross_self_l": "the cross branch is normalised by the self branch's row sum",
    "swap_kv_c": "K_c and V_c are swapped",
    "head_neighbour": "the last head reads its neighbour's columns",
    "cross_D_self": "the cross branch's D is the self branch's",
    "dq_no_cross": "dQ lacks the cross contribution",
    "last_tile_unwritten": "dK and dV of the last key tile stay 0",
}
TOKEN_MUTANTS = {
    "drop_last": "the last key is ignored",
    "drop_128": "key 128 is ignored",
    "mask_next_sample": "sample b reads the mask of sample b + 1",
    "mask_shift": "the mask is shifted by one key",
    "nomask": "the mask is ignored",
    "head_neighbour": "the last head reads its neighbour's columns",
    "last_tile_unwritten": "dK and dV of the last key tile stay 0",
    "mask_queries": "the mask is also applied to queries",
}
# the cases each mutant is tried on: planted keys at the branch ends and at 127 / 128, masks with boundaries inside a
# chunk and a masked first chunk
MUTANT_CASES = ["self1_cross2", "cross_chunk0_masked", "nocross_t129", "t128_s257_d128"]
TOKEN_MUTANT_CASES = ["planted_t129_d64", "planted_t257_d64"]


def _violations(vals, mags, bad):
    return {k: r for k in vals if (r := ac.ratio(bad[k], vals[k], mags[k])) > ac.C}


@pytest.mark.parametrize("bug", list(SPATIAL_MUTANTS))
def test_bound_rejects_spatial_mutant(bug):
    hits = {}
    for name in MUTANT_CASES:
        x, vals, mags, _ = spatial(name)
        if bug in ("swap_kv_c", "cross_nomask", "cross_self_l", "cross_D_self", "dq_no_cross") and x["kv"] is None:
            continue
        bad, _, _ = ac.spatial_oracle(x, bug=bug)
        if v := _violations(vals, mags, bad):
            hits[name] = v
    assert hits, (bug, SPATIAL_MUTANTS[bug])


@pytest.mark.parametrize("bug", list(TOKEN_MUTANTS))
def test_bound_rejects_token_mutant(bug):
    hits = {}
    for name in TOKEN_MUTANT_CASES:
        x, vals, mags, _ = token(name)
        bad, _, _ = ac.token_oracle(x, bug=bug)
        if v := _violations(vals, mags, bad):
            hits[name] = v
    assert hits, (bug, TOKEN_MUTANTS[bug])
