"""CPU side of the autocast (single-plane) mode: the ctypes mirror of mdm_net_io.single_plane, the planes column of the
GEMM profile, and the trainer's fp16 branch running get_loss inside bf16 autocast as the reference does
(ml_mdm/trainer.py:29-30), while the fp32 branch never enters it. GPU behaviour: tests/test_autocast_gpu.py."""
import argparse
import contextlib
import csv
import ctypes
import os
import sys

import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.join(HERE, ".."), os.path.join(HERE, "..", "ml-mdm_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from mdm_b200 import _lib, trainer  # noqa: E402
from mdm_b200.models import native  # noqa: E402


def test_net_io_mirror_carries_single_plane():
    names = [f[0] for f in native.NetIO._fields_]
    i = names.index("single_plane")
    assert native.NetIO._fields_[i][1] is ctypes.c_int32
    assert names[i - 1:] == ["output_scale", "single_plane", "dropout", "dropout_seed"]
    lib = ctypes.CDLL(_lib.LIB_PATH)
    lib.mdm_abi_sizeof.restype = ctypes.c_longlong
    assert lib.mdm_abi_sizeof(4) == ctypes.sizeof(native.NetIO)
    assert native.NetIO().single_plane == 0  # a zeroed struct is the two-plane path every existing caller gets


def test_profile_dump_has_a_planes_column(tmp_path):
    lib = ctypes.CDLL(_lib.LIB_PATH)
    path = tmp_path / "gemm.csv"
    assert lib.mdm_profile_dump(str(path).encode()) == 0
    header = next(csv.reader(open(path)))
    assert header[-1] == "planes" and header[:-1][-1] == "ms"


class _Vision(nn.Module):
    def __init__(self):
        super().__init__()
        self.a = nn.Linear(4, 4)


class _Pipe(nn.Module):
    """What train_batch touches of a pipeline; get_loss records the autocast state it was called in."""

    def __init__(self, log):
        super().__init__()
        self.model = nn.Module()
        self.model.vision_model = _Vision()
        self.log = log

    def get_loss(self, sample):
        self.log.append(("get_loss", autocast_state[-1]))
        x = sample["x"]
        losses = (self.model.vision_model.a(x) ** 2).mean(dim=1)
        return losses, torch.zeros(2), x, x, x, None


autocast_state = [None]


class _RecordingAutocast(contextlib.ContextDecorator):
    """Stands in for torch.autocast: records the device type and dtype while the region is open."""

    def __init__(self, device_type, dtype=None, **kw):
        self.state = (device_type, dtype)

    def __enter__(self):
        autocast_state.append(self.state)
        return self

    def __exit__(self, *exc):
        autocast_state.pop()
        return False


class _Sched:
    def get_last_lr(self):
        return [1e-3]

    def step(self):
        pass


def _run(fp16, monkeypatch):
    log = []
    pipe = _Pipe(log)
    monkeypatch.setattr(torch, "autocast", _RecordingAutocast)
    orig = torch.Tensor.backward

    def backward(self, *a, **k):
        log.append(("backward", autocast_state[-1]))
        return orig(self, *a, **k)
    monkeypatch.setattr(torch.Tensor, "backward", backward)
    opt = torch.optim.SGD(pipe.model.vision_model.parameters(), lr=0.1)
    args = argparse.Namespace(fp16=fp16, gradient_clip_norm=1.0)
    trainer.train_batch(pipe, {"x": torch.ones(2, 4)}, opt, _Sched(), None, args)
    return log


def test_fp16_branch_computes_the_loss_under_bf16_autocast(monkeypatch):
    log = _run(True, monkeypatch)
    assert log == [("get_loss", ("cuda", torch.bfloat16)), ("backward", None)]


def test_fp32_branch_never_enters_autocast(monkeypatch):
    log = _run(False, monkeypatch)
    assert log == [("get_loss", None), ("backward", None)]
