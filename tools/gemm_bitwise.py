"""Bitwise comparison of the wgmma GEMM engine's outputs between two builds (development aid, needs a GPU).

  python tools/gemm_bitwise.py dump OUT.npz [--root TREE]   run every non-atomic case of tests/gemm_cases.py,
                                                            tests/test_gemm_split_gpu.py and
                                                            tests/test_gemm_epilogue_gpu.py and
                                                            tests/test_gemm_epilogue_tma_gpu.py with the library built in
                                                            TREE (default: this repository) and store the outputs
  python tools/gemm_bitwise.py compare A.npz B.npz          exit 1 unless every stored output is bit-identical

A schedule change that keeps each output element's sum of products in the same order must give the same bits; split-K
cases (fp32 atomics) are left out because their order is not fixed from run to run."""
import argparse
import inspect
import os
import re
import sys

import numpy as np


class _RecordingTorch:
    """Stands in for `torch` inside a case module: records every tensor made by torch.zeros (the output buffers)."""

    def __init__(self, torch):
        self._torch = torch
        self.made = []

    def zeros(self, *a, **kw):
        t = self._torch.zeros(*a, **kw)
        self.made.append(t)
        return t

    def __getattr__(self, name):
        return getattr(self._torch, name)


def dump(out, root):
    sys.path[:0] = [os.path.join(root, "ml-mdm_b200"), os.path.join(root, "tests")]
    import torch

    import gemm_cases
    import test_gemm_epilogue_gpu
    import test_gemm_epilogue_tma_gpu
    import test_gemm_split_gpu

    def split_k(fn):  # the case asks for nsplit > 1
        m = re.search(r"nsplit=(\d+)", inspect.getsource(fn))
        return m is not None and int(m.group(1)) > 1

    cases = [(f"gemm_cases.{n}", gemm_cases, fn) for n, fn in gemm_cases.CASES if not split_k(fn)]
    cases += [(f"split_planes.{n}", test_gemm_split_gpu, fn) for n, fn in test_gemm_split_gpu.CASES]
    cases += [(f"epilogue.{n}", test_gemm_epilogue_gpu, fn) for n, fn in test_gemm_epilogue_gpu.CASES]
    # run_plain / run_conv of test_gemm_epilogue_gpu make these cases' buffers
    cases += [(f"epilogue_tma.{n}", test_gemm_epilogue_gpu, fn) for n, _, fn in test_gemm_epilogue_tma_gpu.CASES]
    arrays = {}
    for name, mod, fn in cases:
        rec = _RecordingTorch(torch)
        mod.torch = rec
        try:
            fn()
        finally:
            mod.torch = torch
        torch.cuda.synchronize()
        for i, t in enumerate(rec.made):
            arrays[f"{name}.{i}"] = t.cpu().numpy()
    np.savez(out, **arrays)
    print(f"{len(cases)} cases, {len(arrays)} output buffers -> {out}")


def compare(a, b):
    x, y = np.load(a), np.load(b)
    bad = sorted(set(x.files) ^ set(y.files))
    for k in sorted(set(x.files) & set(y.files)):
        u, v = x[k], y[k]
        if u.shape != v.shape or u.dtype != v.dtype or u.tobytes() != v.tobytes():
            diff = np.abs(u.astype(np.float64) - v.astype(np.float64)).max() if u.shape == v.shape else float("nan")
            print(f"DIFFER {k}: max abs diff {diff:g}")
            bad.append(k)
    print(f"{len(x.files)} vs {len(y.files)} buffers, {len(bad)} differ")
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    d = sub.add_parser("dump")
    d.add_argument("out")
    d.add_argument("--root", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    c = sub.add_parser("compare")
    c.add_argument("a")
    c.add_argument("b")
    args = ap.parse_args()
    if args.cmd == "dump":
        dump(args.out, os.path.abspath(args.root))
        return 0
    return compare(args.a, args.b)


if __name__ == "__main__":
    sys.exit(main())
