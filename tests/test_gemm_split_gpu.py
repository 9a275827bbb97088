"""wgmma GEMM engine with the split operand planes of the weight products (DESIGN §2), through the C ABI
(mdm_gemm_raw_split): every weight GEMM also multiplies the lo plane of B, and the ResNet data-gradient convs the lo
plane of their K-major A. Checked against A (B_hi + B_lo) + A_lo B_hi in fp64 on the same fp16 planes, within the
fp32-output tolerance of test_gemm_gpu.py. The lo planes hold values ~1e-3 of the hi planes, so a product that left
one out would miss by far more than that tolerance."""
import pytest
import torch

import gemm_cases as gc
from mdm_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _planes(shape, g, scale, lo):
    hi = (torch.randn(*shape, generator=g) * scale).to(torch.float16).to(DEV)
    if not lo:
        return hi, None
    return hi, (torch.randn(*shape, generator=g) * scale * 1e-3).to(torch.float16).to(DEV)


def _launch(sa, sb, a_mn, b_mn, p, b_lo, a_lo):
    _lib.gemm_raw_split(sa, sb, a_mn, b_mn, p, b_lo.data_ptr() if b_lo is not None else 0,
                        a_lo.data_ptr() if a_lo is not None else 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def run_plain(M, N, K, b_mn, bn, b_lo=True, a_lo=False, nz1=1, nz2=1, seed=0):
    """C[z2, z1] = A (M x K, K-major) @ (B + B_lo)^T + A_lo @ B^T; B stored K-major (N x K) or MN-major (K x N)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    nb = nz1 * nz2
    A, Alo = _planes((nb, M, K), g, 0.5, a_lo)
    B, Blo = _planes((nb, N, K), g, 0.5, b_lo)
    B_st = B.transpose(1, 2).contiguous() if b_mn else B
    Blo_st = Blo.transpose(1, 2).contiguous() if (b_mn and Blo is not None) else Blo
    sa = _lib.tmap(A.data_ptr(), (K, M, nz1, nz2), (1, K, K * M, K * M * nz1), (64, 128, 1, 1))
    if b_mn:
        sb = _lib.tmap(B_st.data_ptr(), (N, K, nz1, nz2), (1, N, K * N, K * N * nz1), (64, 64, 1, 1))
    else:
        sb = _lib.tmap(B_st.data_ptr(), (K, N, nz1, nz2), (1, K, K * N, K * N * nz1), (64, bn, 1, 1))
    p = _lib.GemmParams()
    p.kind = 0
    p.M, p.N, p.K = M, N, K
    p.block_n = bn
    p.nz1, p.nz2, p.nsplit = nz1, nz2, 1
    p.a_use_z = p.b_use_z = 1
    p.num_kblocks = (K + 63) // 64
    p.alpha = 1.0
    p.ldc = N
    p.c_z1_stride = M * N
    p.c_z2_stride = M * N * nz1
    out = torch.zeros(nb, M, N, device=DEV)
    p.out_f32 = out.data_ptr()
    _launch(sa, sb, 0, b_mn, p, Blo_st, Alo)
    Bd = B.double()
    ref = torch.matmul(A.double(), (Bd if Blo is None else Bd + Blo.double()).transpose(1, 2))
    if Alo is not None:
        ref = ref + torch.matmul(Alo.double(), Bd.transpose(1, 2))
    return out, ref


def _oihw(wp):
    co, _, ci = wp.shape
    return wp.double().reshape(co, 3, 3, ci).permute(0, 3, 1, 2)


def run_conv(nimg, H, W, Cin, Cout, bn, dgrad=False, b_lo=True, a_lo=False, seed=0):
    """3x3 conv forward (x: NHWC Cin -> Cout, K-major weights) or data gradient (dy: NHWC Cout -> Cin, the packed
    [Cout][tap][Cin] weights read MN-major)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    cx, cy = (Cout, Cin) if dgrad else (Cin, Cout)
    X, Xlo = _planes((nimg, H, W, cx), g, 0.5, a_lo)
    Wp, Wlo = _planes((Cout, 9, Cin), g, 0.1, b_lo)
    PW = 16 if W >= 16 else 8
    PH = 128 // PW
    sa = _lib.tmap(X.data_ptr(), (cx, W, H, nimg), (1, cx, W * cx, H * W * cx), (64, PW, PH, 1))
    sb = _lib.tmap(Wp.data_ptr(), (Cin, Cout, 9, 1), (1, 9 * Cin, Cin, 9 * Cin * Cout),
                   (64, 64 if dgrad else bn, 1, 1))
    p = _lib.GemmParams()
    p.kind = 1
    p.N, p.K = cy, cx
    p.block_n = bn
    p.H, p.W, p.PW, p.PH = H, W, PW, PH
    p.tiles_w, p.tiles_h, p.nimg = (W + PW - 1) // PW, (H + PH - 1) // PH, nimg
    p.taps = 9
    p.flip = 1 if dgrad else 0
    p.kblocks_c = (cx + 63) // 64
    p.num_kblocks = 9 * p.kblocks_c
    p.alpha = 1.0
    p.ldc = cy
    out = torch.zeros(nimg, H, W, cy, device=DEV)
    p.out_f32 = out.data_ptr()
    _launch(sa, sb, 0, 1 if dgrad else 0, p, Wlo, Xlo)

    def conv(x, w):
        xx = x.double().permute(0, 3, 1, 2)
        if dgrad:
            r = torch.nn.grad.conv2d_input((nimg, Cin, H, W), _oihw(w), xx, padding=1)
        else:
            r = torch.nn.functional.conv2d(xx, _oihw(w), padding=1)
        return r.permute(0, 2, 3, 1)

    ref = conv(X, Wp if Wlo is None else Wp.double() + Wlo.double())
    if Xlo is not None:
        ref = ref + conv(Xlo, Wp)
    return out, ref


CASES = [
    # linear forward (K-major weights) and data gradient (MN-major weights)
    ("kk_blo", lambda: run_plain(128 * 4, 256, 320, 0, 256)),
    ("kk_blo_ragged", lambda: run_plain(128 * 3 + 37, 384, 200, 0, 192)),
    ("kk_blo_bn16", lambda: run_plain(300, 16, 128, 0, 16)),
    ("kk_blo_bn96_alo", lambda: run_plain(128 * 2 + 5, 96, 256, 0, 96, a_lo=True)),
    ("kk_alo_only", lambda: run_plain(256, 128, 192, 0, 128, b_lo=False, a_lo=True)),
    ("kk_blo_batched", lambda: run_plain(200, 128, 128, 0, 128, nz1=3, nz2=2)),
    ("kmn_blo", lambda: run_plain(128 * 3, 256, 320, 1, 256)),
    ("kmn_blo_bn192_alo", lambda: run_plain(128 * 2 + 9, 192, 256, 1, 192, a_lo=True)),
    ("kmn_blo_bn32", lambda: run_plain(200, 32, 192, 1, 32)),
    ("kmn_blo_batched", lambda: run_plain(130, 96, 128, 1, 96, nz1=2, nz2=2)),
    # 3x3 conv forward and data gradient (the ResNet data gradient also carries the lo plane of its fp16 dy)
    ("conv_fwd_blo", lambda: run_conv(2, 32, 32, 256, 256, 256)),
    ("conv_fwd_blo_ragged", lambda: run_conv(3, 24, 40, 64, 128, 128)),
    ("conv_fwd_blo_w8_alo", lambda: run_conv(3, 8, 8, 128, 64, 64, a_lo=True)),
    ("conv_dgrad_blo_alo", lambda: run_conv(2, 16, 16, 192, 256, 192, dgrad=True, a_lo=True)),
    ("conv_dgrad_blo_bn64", lambda: run_conv(2, 24, 24, 64, 128, 64, dgrad=True)),
]


@pytest.mark.parametrize("name,fn", CASES, ids=[c[0] for c in CASES])
def test_gemm_split_planes(name, fn):
    out, ref = fn()
    err = float((out.double() - ref).abs().max() / ref.abs().max())
    assert err <= gc.TOL["f32"], (name, err)
