"""forward_conditioning / forward_denoising without a GPU: the reference's signatures (written out here: tests never
import the reference), the ctypes mirrors of mdm_net_stage_io and the appended mdm_net_grad_io fields against the header, and
the errors and fall-backs that are decided before the engine is entered."""
import copy
import ctypes
import inspect
import os
import re
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "ml-mdm_b200"))

import tiny_configs as tc  # noqa: E402
from mdm_b200 import _lib  # noqa: E402
from mdm_b200 import config as mc  # noqa: E402
from mdm_b200 import samplers  # noqa: E402
from mdm_b200.models import NestedUNet, UNet, native  # noqa: E402

# the reference's parameter lists (ml_mdm/models/unet.py:847,935-937; nested_unet.py:165,168-170), defaults as written
COND = [("conditioning", inspect.Parameter.empty), ("cond_mask", inspect.Parameter.empty)]
DENOISE = [("x_t", inspect.Parameter.empty), ("times", inspect.Parameter.empty), ("cond_emb", None),
           ("conditioning", None), ("cond_mask", None), ("micros", {})]


def _params(fn):
    ps = list(inspect.signature(fn).parameters.values())
    assert ps[0].name == "self"
    return [(p.name, p.default) for p in ps[1:]]


@pytest.mark.parametrize("cls", [UNet, NestedUNet])
def test_signatures_match_reference(cls):
    assert _params(cls.forward_denoising) == DENOISE
    assert _params(cls.forward_conditioning) == COND


def _header_fields(cname):
    hdr = open(os.path.join(ROOT, "include", "mdm_b200.h")).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (cname, cname), hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            names += [re.sub(r"\[.*\]", "", p.strip().split()[-1].lstrip("*")) for p in decl.split(",")]
    return names


def test_stage_fields_match_header():
    stage = ["stage", "cond_out", "cond_emb_out", "cond", "cond_emb", "cross_mask", "cond_cache"]
    grad_new = ["stage", "dcond", "dcond_emb", "dcond_in", "dcond_emb_in"]
    assert [f[0] for f in native.StageIO._fields_] == stage
    assert _header_fields("mdm_net_stage_io") == stage
    assert [f[0] for f in native.NetGradIO._fields_] == ["dout"] + grad_new
    assert _header_fields("mdm_net_grad_io") == [f[0] for f in native.NetGradIO._fields_]
    assert _header_fields("mdm_net_io") == [f[0] for f in native.NetIO._fields_]
    # appended after every existing field: a zero-initialised mdm_net_grad_io is the stage-0 backward
    assert native.NetGradIO.stage.offset == ctypes.sizeof(ctypes.c_void_p) * 4
    lib = ctypes.CDLL(_lib.LIB_PATH)
    lib.mdm_abi_sizeof.restype = ctypes.c_longlong
    assert lib.mdm_abi_sizeof(4) == ctypes.sizeof(native.NetIO)
    assert lib.mdm_abi_sizeof(5) == ctypes.sizeof(native.NetGradIO)
    assert hasattr(lib, "mdm_net_forward_stage")
    hdr = open(os.path.join(ROOT, "include", "mdm_b200.h")).read()
    assert ("int mdm_net_forward_stage(mdm_net* net, const mdm_net_io* io, const mdm_net_stage_io* stage, "
            "mdm_stream_t stream);") in hdr


def test_build_net_cfg_unchanged_by_split():
    cfg = mc.unet_config_from_dict(copy.deepcopy(tc.TINY_NESTED))
    cfg.conditioning_feature_dim = tc.LM_DIM
    m = NestedUNet(3, 3, cfg)
    nc = native.build_net_cfg(m)
    assert nc.num_levels == 2 and nc.cond_dim > 0 and nc.has_cond_emb == 1


def test_nested_inner_net_refuses_split_calls():
    cfg = mc.unet_config_from_dict(copy.deepcopy(tc.TINY_NESTED))
    cfg.conditioning_feature_dim = tc.LM_DIM
    m = NestedUNet(3, 3, cfg)
    x = torch.zeros(1, 3, 8, 8)
    with pytest.raises(_lib.MdmError, match="nesting=True"):
        m.inner_unet.forward_denoising(x, torch.zeros(1, dtype=torch.long))
    with pytest.raises(_lib.MdmError, match="nesting=True"):
        m.inner_unet.forward_conditioning(torch.zeros(1, 2, tc.LM_DIM), None)


def test_sampler_calls_foreign_models_every_step():
    """A model that is not this package's Model / NestedModel gets no text encoding: it is called as it is."""
    s = samplers.Sampler.__new__(samplers.Sampler)
    calls = []

    def wrapper(*args):
        calls.append(args)
        return "out"

    assert s._encode_text(wrapper, torch.zeros(1, 2, 3), None) is None
    s._text = None
    assert s._model(wrapper, 1, 2, 3, 4, {}) == "out" and len(calls) == 1
