"""CPU: DiffusionConfig.model_output_scale is accepted. The reference's own tests/test_models.py::test_initialize_unet
builds a Model with model_output_scale=0.1 through the registries that plugin.register() fills, then a ModelEma of
its vision model; this runs that scenario on a stand-in config module (the tests do not import the reference)."""
import copy
import types

import pytest

from mdm_b200 import config as mc
from mdm_b200 import plugin
from mdm_b200.diffusion import Model, NestedModel


def _registries():
    fake = types.SimpleNamespace(MODEL_REGISTRY={}, PIPELINE_REGISTRY={}, MODEL_CONFIG_REGISTRY={},
                                 PIPELINE_CONFIG_REGISTRY={})
    plugin.register(fake)
    return fake


def test_initialize_unet_scenario_with_model_output_scale():
    reg = _registries()
    denoising_model = reg.MODEL_REGISTRY["unet"](input_channels=3, output_channels=3, config=mc.UNetConfig())
    diffusion_config = mc.DiffusionConfig(use_vdm_loss_weights=True, model_output_scale=0.1)
    diffusion_model = reg.PIPELINE_REGISTRY["unet"](denoising_model, diffusion_config)
    assert isinstance(diffusion_model.model, Model)
    assert diffusion_model.model._output_scale == pytest.approx(0.1)
    ema = copy.deepcopy(diffusion_model.model.vision_model).eval()  # what ModelEma.__init__ does
    assert ema is not None
    assert getattr(ema, "output_scale", 0.0) == 0.0  # a copied vision model called directly is never scaled


def test_nested_model_accepts_model_output_scale():
    reg = _registries()
    cfg = mc.unet_config_from_dict(copy.deepcopy(__import__("tiny_configs").TINY_NESTED))
    net = reg.MODEL_REGISTRY["nested_unet"](3, 3, cfg)
    pipe = reg.PIPELINE_REGISTRY["nested_unet"](net, mc.NestedDiffusionConfig(model_output_scale=0.1, no_use_residual=True))
    assert isinstance(pipe.model, NestedModel)
