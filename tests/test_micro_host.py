"""General micro-conditioning without a GPU: the drop-in's parameter tree and the oracle against the fixture of the
unmodified reference (tests/golden/micro.npz, written by tests/golden/make_golden_micro.py), the ctypes mirrors of the
new C structs, the micro table handed to the engine, and the inputs refused before the engine is entered."""
import ctypes
import os
import re
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "ml-mdm_b200"))

import micro_cases as mx  # noqa: E402
import tiny_configs as tc  # noqa: E402
from mdm_b200 import _lib  # noqa: E402
from mdm_b200 import config as mc  # noqa: E402
from mdm_b200.models import NestedUNet, UNet  # noqa: E402
from mdm_b200.models import native  # noqa: E402
from oracle import unet_ref  # noqa: E402

HEADER = os.path.join(ROOT, "include", "mdm_b200.h")


def mirror(arch, ucfg=None):
    cfg = mc.unet_config_from_dict(ucfg or mx.tiny_config(arch))
    cfg.conditioning_feature_dim = tc.LM_DIM
    return (UNet if arch == "unet" else NestedUNet)(3, 3, cfg)


def keys_and_shapes(gold, arch):
    return [(k, sh) for k, sh in zip(gold[f"{arch}.keys"], gold[f"{arch}.shapes"])]


@pytest.mark.parametrize("arch", mx.ARCHS)
def test_state_dict_matches_reference(arch):
    gold = np.load(mx.GOLD)
    m = mirror(arch)
    got = [(k, "x".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()]
    assert got == [(str(k), str(s)) for k, s in keys_and_shapes(gold, arch)]
    assert any(".cond_layers.watermark_score.1.weight" in "." + k for k, _ in got)


@pytest.mark.parametrize("arch", mx.ARCHS)
@pytest.mark.parametrize("which", mx.MICRO_SETS)
def test_oracle_matches_reference(arch, which):
    gold = np.load(mx.GOLD)
    sd = tc.seeded_state_dict({k: torch.empty([int(s) for s in sh.split("x")] if sh else [], device="meta")
                               for k, sh in keys_and_shapes(gold, arch)}, mx.PARAM_SEED)
    net = unet_ref.OracleNet(_ns(mx.tiny_config(arch)), tc.LM_DIM)
    # fp32, the reference's arithmetic: a key other than "scale" is multiplied by 1000 before the sinusoid, and the
    # fp32 rounding of such arguments (~1e3 rad) is part of the reference's result
    P = {k: v.requires_grad_(True) for k, v in sd.items()}
    x, t, lm, mask = mx.tiny_inputs(arch)
    out = net.forward(P, x, t, lm, mask, mx.micro_set(arch, which))
    out = out if isinstance(out, (list, tuple)) else [out]
    sum((o * w).sum() for o, w in zip(out, mx.loss_weights(out))).backward()
    tag = f"{arch}.{which}"
    for i, o in enumerate(out):
        flat = o.detach().reshape(-1)
        got = flat[torch.from_numpy(mx.sample_index(flat.numel(), i, mx.OUT_SAMPLES))]
        ref = torch.from_numpy(gold[f"{tag}.out{i}"])
        assert float((got - ref).abs().max()) / float(gold[f"{tag}.outmax{i}"]) <= 1e-5, (tag, i)
    gmax = gold[f"{tag}.gmax"].astype(np.float64)
    gval = gold[f"{tag}.gval"]
    roundoff = 1e-4 * float(np.sort(gmax)[len(gmax) // 2])
    pos = 0
    for i, k in enumerate(gold[f"{arch}.keys"]):
        g = P[k].grad.reshape(-1)
        idx = mx.sample_index(g.numel(), i, mx.GRAD_SAMPLES)
        ref = torch.from_numpy(gval[pos:pos + idx.size])
        pos += idx.size
        if gmax[i] <= roundoff:
            assert float(g.abs().max()) <= roundoff, (tag, k)
            continue
        assert float((g[torch.from_numpy(idx)] - ref).abs().max()) / gmax[i] <= 1e-5, (tag, k)
    assert pos == gval.size


def _ns(d):
    if isinstance(d, dict):
        return types.SimpleNamespace(**{k: _ns(v) for k, v in d.items()})
    return d


def test_micro_terms_reach_the_reference_outputs():
    """The fixture's three micro sets give different outputs (the keys are live, not silently defaulted)."""
    gold = np.load(mx.GOLD)
    for arch in mx.ARCHS:
        a, b, c = (gold[f"{arch}.{w}.out0"] for w in mx.MICRO_SETS)
        assert not np.allclose(a, b) and not np.allclose(b, c), arch


def _header_struct(name):
    src = open(HEADER).read()
    body = re.search(r"typedef struct " + name + r" \{(.*?)\} " + name + ";", src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return [re.match(r"\s*(?:const\s+)?\w+\*?\s*\**\s*(\w+)", d).group(1) for d in body.split(";") if d.strip()]


def test_ctypes_mirrors_match_header():
    src = open(HEADER).read()
    assert f"#define MDM_MAX_MICRO {native.MAX_MICRO} " in src
    assert f"#define MDM_MICRO_NAME_LEN {native.MICRO_NAME_LEN} " in src
    assert _header_struct("mdm_micro_cfg") == [f[0] for f in native.MicroCfg._fields_]
    assert _header_struct("mdm_net_micro_io") == [f[0] for f in native.MicroIO._fields_]
    assert ("int mdm_net_create_micro(const mdm_net_cfg* cfg, const mdm_micro_cfg* micro, mdm_net** out);") in src
    assert ("int mdm_net_forward_micro(mdm_net* net, const mdm_net_io* io, const mdm_net_stage_io* stage,\n"
            "                          const mdm_net_micro_io* micro, mdm_stream_t stream);") in src
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert hasattr(lib, "mdm_net_create_micro") and hasattr(lib, "mdm_net_forward_micro")
    # the existing structs keep their layout
    lib.mdm_abi_sizeof.restype = ctypes.c_longlong
    mirrors = [_lib.TmapSpec, _lib.GemmParams, native.LevelCfg, native.NetCfg, native.NetIO, native.NetGradIO]
    for which, cls in enumerate(mirrors):
        assert lib.mdm_abi_sizeof(which) == ctypes.sizeof(cls), cls.__name__
    assert lib.mdm_abi_sizeof(8) == -1
    assert native.LevelCfg._fields_[-1][0] == "dropout"
    assert native.NetCfg._fields_[-1][0] == "num_lm_head_layers"
    assert [f[0] for f in native.NetIO._fields_[-2:]] == ["dropout", "dropout_seed"]


def test_micro_table_of_the_nest():
    mcfg = native.build_micro_cfg(mirror("nested_unet"))
    names = [mcfg.names[k].value.decode() for k in range(mcfg.num_keys)]
    assert names == ["scale", "watermark_score"]  # first appearance, outermost level first
    assert list(mcfg.level_num_keys) == [2, 2, 0, 0]
    assert list(mcfg.level_keys[0])[:2] == [0, 1] and list(mcfg.level_keys[1])[:2] == [1, 0]
    assert list(mcfg.level_defaults[0])[:2] == [64.0, 0.0] and list(mcfg.level_defaults[1])[:2] == [0.0, 16.0]
    nc = native.build_net_cfg(mirror("nested_unet"))
    assert nc.levels[0].has_micro_scale == 0 and nc.levels[1].has_micro_scale == 0  # the table carries it
    mcfg = native.build_micro_cfg(mirror("unet"))
    assert [mcfg.names[k].value.decode() for k in range(mcfg.num_keys)] == ["scale", "watermark_score", "aesthetic"]
    assert list(mcfg.level_defaults[0])[:3] == [16.0, 0.0, 5.0]


@pytest.mark.parametrize("name,defaults", [("cc12m_64x64", [64.0]), ("cc12m_256x256", [256.0, 64.0]),
                                           ("cc12m_1024x1024", [1024.0, 256.0, 64.0])])
def test_build_net_cfg_of_shipped_configs_unchanged(name, defaults):
    ucfg, _, nested = mc.load_yaml_configs(os.path.join(ROOT, "ml-mdm_b200", "mdm_b200", "configs", name + ".yaml"))
    with torch.device("meta"):
        m = (NestedUNet if nested else UNet)(3, 3, ucfg)
    nc = native.build_net_cfg(m)
    assert nc.num_levels == len(defaults)
    for li, d in enumerate(defaults):
        assert nc.levels[li].has_micro_scale == 1 and nc.levels[li].micro_scale_default == d
    mcfg = native.build_micro_cfg(m)
    assert mcfg.num_keys == 1 and mcfg.names[0].value == b"scale"


def _with_micro(arch, outer, inner=None):
    ucfg = mx.tiny_config(arch)
    ucfg["micro_conditioning"] = outer
    if inner is not None:
        ucfg["inner_config"]["micro_conditioning"] = inner
    return ucfg


def test_zero_scale_default_is_refused():
    with pytest.raises(ValueError, match="'scale'"):
        mirror("unet", _with_micro("unet", "scale:0,watermark_score:0"))
    with pytest.raises(ValueError, match="'scale'"):
        mirror("nested_unet", _with_micro("nested_unet", "scale:64", "scale:0"))
    mirror("unet", _with_micro("unet", "scale:-4,watermark_score:0"))  # a negative default is the reference's arithmetic


def test_too_many_keys_are_refused():
    nine = ",".join(f"k{i}:0" for i in range(native.MAX_MICRO + 1))
    with pytest.raises(ValueError, match="at most"):
        mirror("unet", _with_micro("unet", nine))
    # eight per level, but more than eight distinct keys in the nest
    outer = ",".join(f"a{i}:0" for i in range(5))
    inner = ",".join(f"b{i}:0" for i in range(5))
    with pytest.raises(_lib.MdmError, match="distinct keys"):
        native.build_micro_cfg(mirror("nested_unet", _with_micro("nested_unet", outer, inner)))


def test_too_long_key_name_is_refused():
    long = "k" * native.MICRO_NAME_LEN
    with pytest.raises(ValueError, match="longer than"):
        mirror("unet", _with_micro("unet", f"scale:16,{long}:0"))
    mirror("unet", _with_micro("unet", "scale:16," + "k" * (native.MICRO_NAME_LEN - 1) + ":0"))


def _enter_only(arch):
    """A NativeNet shell with the micro table of the model, enough for _enter (no engine handle)."""
    n = native.NativeNet.__new__(native.NativeNet)
    n.module = mirror(arch)
    mcfg = native.build_micro_cfg(n.module)
    n.micro_keys = [mcfg.names[k].value.decode() for k in range(mcfg.num_keys)]
    n.max_dropout = 0.0
    return n


def test_micro_values_are_checked_before_the_engine():
    n = _enter_only("unet")
    with pytest.raises(_lib.MdmError, match="CUDA tensor"):
        n._enter({"watermark_score": torch.zeros(2)}, 2)
    with pytest.raises(_lib.MdmError, match="CUDA tensor"):
        n._enter({"watermark_score": 0.5}, 2)
    with pytest.raises(_lib.MdmError, match="3 elements"):
        n._enter({"scale": torch.zeros(3)}, 2)
    with pytest.raises(_lib.MdmError, match="2 elements"):
        n._enter({"scale": torch.zeros(2)}, 4)
    assert n._enter({}, 2) == [None, None, None]
    assert n._enter({"unknown": torch.zeros(3)}, 2) == [None, None, None]  # keys no level configures are ignored
