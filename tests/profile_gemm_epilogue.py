"""Per-tile cost of the persistent weight-product GEMM's epilogue (development aid, needs a GPU).

  python tests/profile_gemm_epilogue.py [--root TREE] [--quick]

Times gemm_persistent_kernel through mdm_gemm_raw_split with the weights' lo plane, as the engine launches it, on the
shapes of the cc12m_64x64 training step at batch 64 (the 16x16 attention level: M = 16384 rows at 768 channels; the
32x32 level: M = 65536 at 512; 3x3 convs of the 64x64 level). Per case:
  * the time at the real K, with algorithmic TFLOP/s (2 M N K) and issued TFLOP/s (every plane's wgmma counted);
  * a K sweep at the same M, N and epilogue, fitted as time per tile = fixed + slope x k blocks. The intercept is the
    fixed per-tile cost (epilogue plus tile switch) that the mainloop does not amortise.
CUDA events around blocks of launches after a warm-up; the median of the blocks is reported. --root loads the library
built in another tree, so two builds can be alternated on the same card."""
import argparse
import os
import statistics
import subprocess
import sys

import numpy as np

NUM_SMS = 132


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return q


def block_n(n):
    return (n + 15) // 16 * 16 if n < 192 else 128


class Case:
    """One persistent-kernel launch: operands, lo planes and epilogue buffers, built once and relaunched."""

    def __init__(self, torch, lib, kind, M, N, K, b_mn=False, epi="f16", a_lo=False, conv=None):
        self.torch, self.lib = torch, lib
        dev = "cuda"
        g = torch.Generator(device="cpu").manual_seed(1)
        h = torch.float16
        p = lib.GemmParams()
        p.alpha = 1.0
        bn = block_n(N)
        p.block_n = bn
        keep = []
        planes = 2 if not a_lo else 3
        if kind == "plain":
            A = torch.randn(M, K, generator=g).to(h).to(dev)
            Alo = (torch.randn(M, K, generator=g) * 1e-3).to(h).to(dev) if a_lo else None
            Bsh = (K, N) if b_mn else (N, K)
            B = (torch.randn(*Bsh, generator=g) * 0.05).to(h).to(dev)
            Blo = (torch.randn(*Bsh, generator=g) * 5e-5).to(h).to(dev)
            self.sa = lib.tmap(A.data_ptr(), (K, M, 1, 1), (1, K, K * M, K * M), (64, 128, 1, 1))
            if b_mn:
                self.sb = lib.tmap(B.data_ptr(), (N, K, 1, 1), (1, N, N * K, N * K), (64, 64, 1, 1))
            else:
                self.sb = lib.tmap(B.data_ptr(), (K, N, 1, 1), (1, K, K * N, K * N), (64, bn, 1, 1))
            p.kind = 0
            p.M, p.N, p.K = M, N, K
            p.nz1 = p.nz2 = p.nsplit = 1
            p.num_kblocks = (K + 63) // 64
            rows = M
            self.tiles = -(-M // 128) * -(-N // bn)
            self.flop = 2.0 * M * N * K
        else:  # 3x3 conv forward (B K-major) or data gradient (B MN-major), NHWC activations
            nimg, H, W = conv
            A = torch.randn(nimg, H, W, K, generator=g).to(h).to(dev)
            Alo = (torch.randn(nimg, H, W, K, generator=g) * 1e-3).to(h).to(dev) if a_lo else None
            cin, cout = (N, K) if b_mn else (K, N)
            B = (torch.randn(cout, 9, cin, generator=g) * 0.05).to(h).to(dev)
            Blo = (torch.randn(cout, 9, cin, generator=g) * 5e-5).to(h).to(dev)
            PW = 16 if W >= 16 else 8
            PH = 128 // PW
            self.sa = lib.tmap(A.data_ptr(), (K, W, H, nimg), (1, K, W * K, H * W * K), (64, PW, PH, 1))
            self.sb = lib.tmap(B.data_ptr(), (cin, cout, 9, 1), (1, 9 * cin, cin, 9 * cin * cout),
                               (64, 64 if b_mn else bn, 1, 1))
            p.kind = 1
            p.N, p.K = N, K
            p.H, p.W, p.PW, p.PH = H, W, PW, PH
            p.tiles_w, p.tiles_h, p.nimg = -(-W // PW), -(-H // PH), nimg
            p.taps = 9
            p.flip = 1 if b_mn else 0
            p.kblocks_c = (K + 63) // 64
            p.num_kblocks = 9 * p.kblocks_c
            rows = nimg * H * W
            self.tiles = nimg * p.tiles_w * p.tiles_h * -(-N // bn)
            self.flop = 2.0 * rows * N * 9 * K
        self.issued = self.flop * planes
        p.ldc = N
        if epi in ("res", "f32"):
            out = torch.zeros(rows, N, device=dev)
            p.out_f32 = out.data_ptr()
            keep.append(out)
        if epi == "res":
            bias = torch.randn(N, generator=g).to(dev)
            res = torch.randn(rows, N, generator=g).to(dev)
            p.bias, p.residual = bias.data_ptr(), res.data_ptr()
            keep += [bias, res]
        if epi in ("f16", "gelu", "ggrad"):
            out = torch.zeros(rows, N, device=dev, dtype=h)
            p.out_f16 = out.data_ptr()
            keep.append(out)
        if epi == "gelu":
            bias = torch.randn(N, generator=g).to(dev)
            act = torch.zeros(rows, N, device=dev, dtype=h)
            p.bias, p.out_act_f16, p.act = bias.data_ptr(), act.data_ptr(), 1
            keep += [bias, act]
        if epi == "ggrad":
            src = torch.randn(rows, N, generator=g).to(h).to(dev)
            p.gelu_grad_src = src.data_ptr()
            keep.append(src)
        self.p, self.b_mn = p, int(b_mn)
        self.keep = [A, Alo, B, Blo] + keep
        self.blo, self.alo = Blo.data_ptr(), (Alo.data_ptr() if Alo is not None else 0)
        self.kblocks = p.num_kblocks
        self.tiles_per_cta = self.tiles / min(self.tiles, NUM_SMS)

    def launch(self):
        self.lib.gemm_raw_split(self.sa, self.sb, 0, self.b_mn, self.p, self.blo, self.alo,
                                self.torch.cuda.current_stream().cuda_stream)

    def time_ms(self, iters, blocks):
        torch = self.torch
        for _ in range(3):
            self.launch()
        torch.cuda.synchronize()
        ms = []
        for _ in range(blocks):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                self.launch()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / iters)
        return statistics.median(ms)


# (name, kind, M, N, K, b_mn, epilogue, a_lo, conv geometry); M of a conv is its pixel count
CASES = [
    ("attn16.qkv", "plain", 16384, 2304, 768, False, "f16", False, None),
    ("attn16.proj_out", "plain", 16384, 768, 768, False, "res", False, None),
    ("attn16.ffn_up", "plain", 16384, 3072, 768, False, "gelu", False, None),
    ("attn16.ffn_down", "plain", 16384, 768, 3072, False, "res", False, None),
    ("attn16.ffn_down.dgrad", "plain", 16384, 3072, 768, True, "ggrad", False, None),
    ("attn16.ffn_up.dgrad", "plain", 16384, 768, 3072, True, "f32", False, None),
    ("attn16.qkv.dgrad", "plain", 16384, 768, 2304, True, "f32", False, None),
    ("attn32.qkv", "plain", 65536, 1536, 512, False, "f16", False, None),
    ("attn32.proj_out", "plain", 65536, 512, 512, False, "res", False, None),
    ("attn32.ffn_up", "plain", 65536, 2048, 512, False, "gelu", False, None),
    ("attn32.ffn_down", "plain", 65536, 512, 2048, False, "res", False, None),
    ("attn32.ffn_down.dgrad", "plain", 65536, 2048, 512, True, "ggrad", False, None),
    ("conv64.fwd", "conv", 262144, 256, 256, False, "res", False, (64, 64, 64)),
    ("conv64.dgrad", "conv", 262144, 256, 256, True, "f32", True, (64, 64, 64)),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    ap.add_argument("--quick", action="store_true", help="real K only, no sweep")
    ap.add_argument("--only", default="", help="comma-separated case name prefixes")
    args = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.abspath(args.root), "ml-mdm_b200"))
    import torch

    from mdm_b200 import _lib

    assert torch.cuda.is_available(), "needs a GPU"
    print(f"card: {card()}  library: {_lib.__file__}", flush=True)
    sel = [c for c in CASES if not args.only or any(c[0].startswith(s) for s in args.only.split(","))]
    for name, kind, M, N, K, b_mn, epi, a_lo, conv in sel:
        c = Case(torch, _lib, kind, M, N, K, b_mn, epi, a_lo, conv)
        ms = c.time_ms(10, 7)
        line = (f"CASE {name:24s} M={M} N={N} K={K} b_mn={int(b_mn)} epi={epi:5s} tiles={c.tiles}: {ms * 1e3:8.1f} us "
                f"{c.flop / ms / 1e9:5.0f} alg TFLOP/s {c.issued / ms / 1e9:5.0f} issued TFLOP/s "
                f"{ms * 1e3 / c.tiles_per_cta:6.2f} us/tile")
        del c
        if not args.quick:
            ks = [256, 512, 768, 1536, 3072] if kind == "plain" else [64, 128, 256, 512]
            xs, ys = [], []
            for k in ks:
                s = Case(torch, _lib, kind, M, N, k, b_mn, epi, a_lo, conv)
                t = s.time_ms(10, 5)
                xs.append(s.kblocks)
                ys.append(t * 1e3 / s.tiles_per_cta)
                del s
            slope, icpt = np.polyfit(xs, ys, 1)
            at_k = icpt + slope * (9 * ((K + 63) // 64) if kind == "conv" else (K + 63) // 64)
            line += (f" | sweep {' '.join(f'{x}:{y:.2f}' for x, y in zip(xs, ys))} -> fixed {icpt:5.2f} us/tile + "
                     f"{slope * 1e3:5.1f} ns/kblock ({100 * icpt / at_k:4.1f} % of a tile at K={K})")
        print(line, flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
