"""Epilogue of the persistent weight-product GEMM (gemm_persistent_kernel) through mdm_gemm_raw_split, with the
weights' lo plane as the engine launches it: every epilogue field (alpha and alpha_dev, bias, fp32 residual, in-place
accumulate, GELU' source, fp32 / fp16 / GELU outputs) on ragged and odd shapes, padded (ldc > N), batched and
misaligned outputs and conv edge tiles. Tile widths up to 128 columns run the staged epilogue (a shared-memory tile
drained by warps of their own) unless the staging tile would leave fewer than three pipeline stages, as with the
two-plane 3x3 data gradients at 128 columns, or the epilogue evaluates GELU or GELU'; those and wider tiles keep the
epilogue in the consumers' registers. Cases on both sides of that rule are here. Checked against fp64 torch on the
same fp16 planes, at the tolerances of test_gemm_gpu.py. tools/gemm_bitwise.py also dumps these cases to compare two builds bit for bit."""
import pytest
import torch

from mdm_b200 import _lib

DEV = "cuda"
TOL = {"f32": 2e-5, "f16": 1.5e-3, "act": 1.5e-3}


def _rel(x, ref):
    return float((x.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def _gelu_grad(x):
    return 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5


def _planes(shape, g, scale, lo):
    hi = (torch.randn(*shape, generator=g) * scale).to(torch.float16).to(DEV)
    if not lo:
        return hi, None
    return hi, (torch.randn(*shape, generator=g) * scale * 1e-3).to(torch.float16).to(DEV)


def _outputs(p, g, nb, rows, N, ldc, zpad, off, ref, bias, residual, inplace, ggrad, f32, f16, act):
    """Epilogue operands and output buffers of nb row blocks of `rows` x N in a padded layout: row stride ldc, block
    stride rows * ldc + zpad, base `off` elements into each buffer. Returns the operand tensors (kept alive until the
    launch has run) and a function that checks the outputs: errors per output, nothing stored outside them."""
    zs = rows * ldc + zpad
    size = off + nb * zs

    def view(buf):
        return buf.as_strided((nb, rows, N), (zs, ldc, 1), off)

    if bias:
        b = torch.randn(N, generator=g).to(DEV)
        p.bias = b.data_ptr()
        ref = ref + b.double()
    keep = []
    out32 = torch.zeros(size, device=DEV)
    if residual:
        res = torch.randn(size, generator=g).to(DEV)
        if inplace:  # out_f32 += result: the residual is the output buffer itself
            out32.copy_(res)
            res = out32
        p.residual = view(res).data_ptr()
        ref = ref + view(res).double().clone()
        keep.append(res)
    if ggrad:
        src = (torch.randn(size, generator=g) * 1.5).to(torch.float16).to(DEV)
        p.gelu_grad_src = view(src).data_ptr()
        ref = ref * _gelu_grad(view(src).double())
        keep.append(src)
    outs = {}
    if f32:
        p.out_f32 = view(out32).data_ptr()
        outs["f32"] = out32
    if f16:
        o = torch.zeros(size, device=DEV, dtype=torch.float16)
        p.out_f16 = view(o).data_ptr()
        outs["f16"] = o
    if act:
        o = torch.zeros(size, device=DEV, dtype=torch.float16)
        p.out_act_f16 = view(o).data_ptr()
        p.act = 1
        outs["act"] = o
    p.ldc = ldc
    p.c_z1_stride = zs
    p.c_z2_stride = zs * (p.nz1 if p.nz1 > 0 else 1)

    def check():
        errs = {}
        for k, buf in outs.items():
            r = torch.nn.functional.gelu(ref) if k == "act" else ref
            errs[k] = _rel(view(buf), r)
            if not (inplace and k == "f32"):  # nothing outside the N columns of each written row
                mask = torch.ones(size, dtype=torch.bool, device=DEV)
                view(mask).fill_(False)
                assert not buf[mask].any(), f"{k}: stores outside the output"
        return errs

    return keep, check


def run_plain(M, N, K, bn, b_mn=False, nz1=1, nz2=1, ldc=None, zpad=0, off=0, alpha=1.0, alpha_dev=None, bias=False,
              residual=False, inplace=False, ggrad=False, f32=True, f16=False, act=False, seed=0):
    """C[z2, z1] = epilogue(alpha A (B + B_lo)^T); A M x K K-major, B N x K (K-major) or K x N (MN-major)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    nb = nz1 * nz2
    A, _ = _planes((nb, M, K), g, 0.5, False)
    B, Blo = _planes((nb, N, K), g, 0.5, True)
    B_st = B.transpose(1, 2).contiguous() if b_mn else B
    Blo_st = Blo.transpose(1, 2).contiguous() if b_mn else Blo
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
    p.alpha = alpha
    scale = alpha
    ad = None
    if alpha_dev is not None:
        ad = torch.tensor([alpha_dev], device=DEV)
        p.alpha_dev = ad.data_ptr()
        scale = alpha * alpha_dev
    ref = scale * torch.matmul(A.double(), (B.double() + Blo.double()).transpose(1, 2))
    keep, check = _outputs(p, g, nb, M, N, ldc or N, zpad, off, ref, bias, residual, inplace, ggrad, f32, f16, act)
    _lib.gemm_raw_split(sa, sb, 0, int(b_mn), p, Blo_st.data_ptr(), 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    del keep, ad
    return check()


def run_conv(nimg, H, W, Cin, Cout, bn, dgrad=False, a_lo=False, ldc=None, off=0, bias=False, residual=False,
             inplace=False, f16=False, seed=0):
    """3x3 conv forward (x: NHWC Cin -> Cout) or data gradient (dy: NHWC Cout -> Cin) with the weights' lo plane and,
    for the ResNet data gradients, the lo plane of dy; output NHWC with row (pixel) stride ldc."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    cx, cy = (Cout, Cin) if dgrad else (Cin, Cout)
    X, Xlo = _planes((nimg, H, W, cx), g, 0.5, a_lo)
    Wp, Wlo = _planes((Cout, 9, Cin), g, 0.1, True)
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
    p.tiles_w, p.tiles_h, p.nimg = -(-W // PW), -(-H // PH), nimg
    p.taps = 9
    p.flip = 1 if dgrad else 0
    p.kblocks_c = (cx + 63) // 64
    p.num_kblocks = 9 * p.kblocks_c
    p.alpha = 1.0
    w = Wp.double() + Wlo.double()
    oihw = w.reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2)
    xs = [X] + ([Xlo] if a_lo else [])
    ref = 0
    for i, x in enumerate(xs):
        wi = oihw if i == 0 else Wp.double().reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2)
        xc = x.double().permute(0, 3, 1, 2)
        if dgrad:
            r = torch.nn.grad.conv2d_input((nimg, Cin, H, W), wi, xc, padding=1)
        else:
            r = torch.nn.functional.conv2d(xc, wi, padding=1)
        ref = ref + r.permute(0, 2, 3, 1)
    ref = ref.reshape(1, nimg * H * W, cy)
    p.nz1 = p.nz2 = 1
    keep, check = _outputs(p, g, 1, nimg * H * W, cy, ldc or cy, 0, off, ref, bias, residual, inplace, False, True,
                           f16, False)
    _lib.gemm_raw_split(sa, sb, 0, int(dgrad), p, Wlo.data_ptr(), Xlo.data_ptr() if a_lo else 0,
                        torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    del keep
    return check()


CASES = [
    # staged: tile widths up to 128 columns with room for three stages
    ("proj_res_bias", lambda: run_plain(1000, 384, 768, 128, bias=True, residual=True)),
    ("all_outputs_alpha", lambda: run_plain(300, 256, 192, 128, bias=True, residual=True, f16=True, alpha=0.3)),
    ("alpha_dev", lambda: run_plain(256, 128, 320, 128, alpha=0.75, alpha_dev=0.37, bias=True, residual=True)),
    ("inplace_accumulate", lambda: run_plain(384, 256, 512, 128, residual=True, inplace=True)),
    ("odd_n", lambda: run_plain(200, 77, 128, 80, bias=True, residual=True, f16=True)),
    ("odd_n_wide", lambda: run_plain(130, 301, 192, 128, bias=True, residual=True, f16=True)),
    ("ldc_gt_n", lambda: run_plain(260, 250, 128, 128, ldc=264, bias=True, residual=True, f16=True)),
    ("misaligned", lambda: run_plain(200, 256, 128, 128, off=1, bias=True, residual=True, f16=True)),
    ("misaligned_ldc", lambda: run_plain(150, 96, 64, 96, ldc=98, off=2, residual=True, f16=True)),
    ("batched", lambda: run_plain(130, 96, 128, 96, nz1=3, nz2=2, zpad=4, bias=True, residual=True, f16=True)),
    ("batched_odd_stride", lambda: run_plain(100, 48, 64, 48, nz1=2, nz2=2, zpad=3, residual=True)),
    ("narrow_16", lambda: run_plain(515, 16, 256, 16, bias=True, residual=True, f16=True)),
    ("narrow_32_mn", lambda: run_plain(333, 32, 128, 32, b_mn=True, f16=True)),
    ("bn64_mn", lambda: run_plain(1024, 64, 640, 64, b_mn=True, bias=True, f16=True, f32=False)),
    ("one_kblock", lambda: run_plain(384, 384, 64, 128, bias=True, residual=True)),
    ("many_tiles", lambda: run_plain(128 * 70 + 9, 640, 128, 128, residual=True, f16=True)),
    ("conv_fwd_edges", lambda: run_conv(3, 24, 40, 64, 192, 128, bias=True, residual=True)),
    ("conv_fwd_small", lambda: run_conv(2, 8, 12, 64, 96, 96, bias=True, f16=True)),
    ("conv_fwd_ldc", lambda: run_conv(2, 16, 24, 64, 64, 64, ldc=72, off=4, residual=True)),
    ("conv_dgrad_edges", lambda: run_conv(3, 24, 40, 128, 128, 128, dgrad=True)),
    ("conv_dgrad_two_planes_n64", lambda: run_conv(2, 16, 24, 64, 128, 64, dgrad=True, a_lo=True)),
    ("conv_fwd_inplace", lambda: run_conv(2, 16, 16, 128, 128, 128, residual=True, inplace=True)),
    # in-register: GELU / GELU' epilogues, the two-plane 3x3 data gradient at 128 columns (two stages left), and tiles
    # wider than 128 columns
    ("ffn_up_gelu", lambda: run_plain(777, 512, 256, 128, bias=True, f16=True, act=True, f32=False)),
    ("gelu_all_outputs", lambda: run_plain(300, 256, 192, 128, bias=True, residual=True, f16=True, act=True,
                                           alpha=0.3)),
    ("ggrad_mn", lambda: run_plain(513, 384, 256, 128, b_mn=True, ggrad=True, f16=True)),
    ("ggrad_misaligned", lambda: run_plain(200, 96, 128, 96, b_mn=True, ggrad=True, off=1, f16=True)),
    ("conv_dgrad_two_planes", lambda: run_conv(2, 24, 40, 256, 256, 128, dgrad=True, a_lo=True)),
    ("wide_tile", lambda: run_plain(300, 176, 256, 176, bias=True, residual=True, f16=True)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,fn", CASES, ids=[n for n, _ in CASES])
def test_epilogue(name, fn):
    errs = fn()
    assert all(v <= TOL[k] for k, v in errs.items()), errs
