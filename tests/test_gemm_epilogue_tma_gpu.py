"""TMA epilogue of the persistent weight-product GEMM (p.epi_tma = 1): the residual or GELU' source is loaded by TMA into
the staging tile, the consumers fold their accumulators into it, and the outputs leave by TMA stores. The launcher
chooses it for plain products with a GELU or GELU' epilogue or at most 8 k blocks, when tensor maps can describe every
epilogue buffer (16 B-aligned bases, ldc and batch strides multiples of 16 B, a tile width that is a multiple of 32
columns up to 128, fp32 or fp16 epilogue buffers but not both); the cases
below sit on both sides of that rule, and each checks which path it ran (the profile record's majors bits 3 and 4) as
well as its results against fp64 torch, including that nothing is written outside the output. tools/gemm_bitwise.py
also dumps these cases to compare two builds bit for bit."""
import csv
import ctypes as C
import os
import tempfile

import pytest

from mdm_b200 import _lib
from test_gemm_epilogue_gpu import TOL, run_conv, run_plain

STAGED, TMA = 8, 16

CASES = [
    # (name, expected path, case)
    ("tma_res_bias", "tma", lambda: run_plain(1000, 384, 512, 128, bias=True, residual=True)),
    ("tma_alpha", "tma", lambda: run_plain(300, 256, 192, 128, bias=True, residual=True, alpha=0.3)),
    ("tma_alpha_dev", "tma", lambda: run_plain(256, 128, 320, 128, alpha=0.75, alpha_dev=0.37, bias=True,
                                               residual=True)),
    ("tma_inplace", "tma", lambda: run_plain(384, 256, 512, 128, residual=True, inplace=True)),
    ("tma_ragged_mn", "tma", lambda: run_plain(200, 200, 128, 128, bias=True, residual=True)),
    ("tma_ragged_n_bn96", "tma", lambda: run_plain(333, 164, 256, 96, bias=True, residual=True)),
    ("tma_ldc_gt_n", "tma", lambda: run_plain(260, 250, 128, 128, ldc=264, bias=True, residual=True)),
    ("tma_f32_only", "tma", lambda: run_plain(515, 64, 256, 64, b_mn=True)),
    ("tma_f16", "tma", lambda: run_plain(777, 384, 256, 128, bias=True, f16=True, f32=False)),
    ("tma_f16_bn32", "tma", lambda: run_plain(333, 32, 128, 32, b_mn=True, f16=True, f32=False)),
    ("tma_gelu", "tma", lambda: run_plain(777, 512, 256, 128, bias=True, f16=True, act=True, f32=False)),
    ("tma_gelu_alpha", "tma", lambda: run_plain(300, 256, 192, 128, bias=True, f16=True, act=True, f32=False,
                                                alpha=0.3)),
    ("tma_gelu_act_only", "tma", lambda: run_plain(300, 200, 192, 128, bias=True, act=True, f32=False)),
    ("tma_ggrad", "tma", lambda: run_plain(513, 384, 256, 128, b_mn=True, ggrad=True, f16=True, f32=False)),
    ("tma_ggrad_ragged", "tma", lambda: run_plain(200, 96, 128, 96, b_mn=True, ggrad=True, f16=True, f32=False)),
    ("tma_batched", "tma", lambda: run_plain(130, 96, 128, 96, nz1=3, nz2=2, zpad=4, bias=True, residual=True)),
    ("tma_batched_f16", "tma", lambda: run_plain(100, 64, 64, 64, nz1=2, nz2=2, zpad=8, f16=True, f32=False)),
    ("tma_many_tiles", "tma", lambda: run_plain(128 * 70 + 9, 640, 128, 128, residual=True)),
    # the ordinary staged epilogue: 3x3 convs
    ("staged_conv_fwd_edges", "staged", lambda: run_conv(3, 24, 40, 64, 192, 128, bias=True, residual=True)),
    ("staged_conv_fwd_ldc", "staged", lambda: run_conv(2, 16, 24, 64, 64, 64, ldc=72, off=4, residual=True)),
    ("staged_conv_fwd_inplace", "staged", lambda: run_conv(2, 16, 16, 128, 128, 128, residual=True, inplace=True)),
    ("staged_conv_dgrad_edges", "staged", lambda: run_conv(3, 20, 12, 128, 128, 128, dgrad=True)),
    ("staged_conv_dgrad_two_planes_n64", "staged", lambda: run_conv(2, 16, 24, 64, 128, 64, dgrad=True, a_lo=True)),
    # the ordinary staged epilogue: 3x3 convs (above), long contractions without GELU, misaligned base or ldc, odd N, a
    # tile width not a multiple of 32, fp32 and fp16 buffers together
    ("staged_long_k", "staged", lambda: run_plain(300, 256, 768, 128, bias=True, residual=True)),
    ("tma_gelu_long_k", "tma", lambda: run_plain(300, 256, 1024, 128, bias=True, f16=True, act=True, f32=False)),
    ("fallback_misaligned_base", "staged", lambda: run_plain(200, 256, 128, 128, off=1, bias=True, residual=True)),
    ("fallback_misaligned_ldc", "staged", lambda: run_plain(150, 96, 64, 96, ldc=98, residual=True)),
    ("fallback_odd_n", "staged", lambda: run_plain(200, 77, 128, 80, bias=True, residual=True)),
    ("fallback_bn48", "staged", lambda: run_plain(100, 48, 64, 48, residual=True)),
    ("fallback_f32_and_f16", "staged", lambda: run_plain(300, 256, 192, 128, bias=True, residual=True, f16=True)),
    ("fallback_batch_stride", "staged", lambda: run_plain(100, 64, 64, 64, nz1=2, nz2=2, zpad=3, residual=True)),
    # the in-register epilogue: GELU' on a misaligned output, the two-plane 3x3 data gradient at 128 columns
    ("fallback_ggrad_misaligned", "register",
     lambda: run_plain(200, 96, 128, 96, b_mn=True, ggrad=True, off=1, f16=True, f32=False)),
    ("fallback_conv_dgrad_two_planes", "register",
     lambda: run_conv(2, 24, 40, 256, 256, 128, dgrad=True, a_lo=True)),
]


def _run_profiled(fn):
    """Runs one case with the GEMM profile on; returns its errors and the majors bits of every launch."""
    lib = _lib.lib()
    lib.mdm_profile_gemm(1)
    try:
        errs = fn()
    finally:
        lib.mdm_profile_gemm(0)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "gemm.csv")
        assert lib.mdm_profile_dump(path.encode()) == 0
        tot, n = C.c_double(), C.c_longlong()
        lib.mdm_profile_read(C.byref(tot), C.byref(n))
        majors = [int(r["majors"]) for r in csv.DictReader(open(path))]
    return errs, majors


@pytest.mark.gpu
@pytest.mark.parametrize("name,path,fn", CASES, ids=[n for n, _, _ in CASES])
def test_epilogue_tma(name, path, fn):
    errs, majors = _run_profiled(fn)
    assert all(v <= TOL[k] for k, v in errs.items()), errs
    assert len(majors) == 1, majors
    m = majors[0]
    got = "tma" if m & TMA else ("staged" if m & STAGED else "register")
    assert got == path, (got, m)
