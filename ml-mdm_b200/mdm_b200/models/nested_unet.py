"""Drop-in `NestedUNet` for ml_mdm.models.nested_unet.NestedUNet (reference nested_unet.py:96-230).

An outer U-Net whose middle is a whole inner (Nested)UNet, joined by `in_adapter` / `out_adapter`
3x3 convolutions; inputs and outputs are lists ordered high -> low resolution.  The whole nest is
one native network: `forward` enters the engine once.
"""
import numpy as np
import torch.nn as nn

from .unet import UNet, zero_module


class NestedUNet(UNet):
    def __init__(self, input_channels, output_channels, config):
        super().__init__(input_channels, output_channels=output_channels, config=config)
        config.inner_config.conditioning_feature_dim = config.conditioning_feature_dim
        if getattr(config.inner_config, "inner_config", None) is None:
            self.inner_unet = UNet(input_channels, output_channels, config.inner_config)
        else:
            self.inner_unet = NestedUNet(input_channels, output_channels, config.inner_config)
        if getattr(config, "skip_inner_unet_input", False) or getattr(config, "interp_conditioning", False):
            raise NotImplementedError("skip_inner_unet_input / interp_conditioning are off in all shipped configs")
        co = config.resolution_channels[-1]
        ci = config.inner_config.resolution_channels[0]
        self.in_adapter = zero_module(nn.Conv2d(co, ci, 3, padding=1))
        self.out_adapter = zero_module(nn.Conv2d(ci, co, 3, padding=1))
        self.is_temporal = [False] + list(getattr(self.inner_unet, "is_temporal", []))
        nest_ratio = int(2 ** (len(config.resolution_channels) - 1))
        if self.inner_unet.config.nesting and self.inner_unet.model_type == "nested_unet":
            self.nest_ratio = [nest_ratio * self.inner_unet.nest_ratio[0]] + self.inner_unet.nest_ratio
        else:
            self.nest_ratio = [nest_ratio]
        if getattr(config, "initialize_inner_with_pretrained", None) is not None:
            try:
                self.inner_unet.load(config.initialize_inner_with_pretrained.replace("/", "_"))
            except Exception as e:  # same tolerance as the reference (nested_unet.py:147-152)
                print("<-- load pretrained checkpoint error -->")
                print(f"{e}")
        if getattr(config, "freeze_inner_unet", False):
            for p in self.inner_unet.parameters():
                p.requires_grad = False

    @property
    def model_type(self):
        return "nested_unet"

    def forward_conditioning(self, conditioning, cond_mask):
        """NestedUNet.forward_conditioning (nested_unet.py:165-166) hands the text to its innermost U-Net. The engine
        runs the whole nest as one network, and its conditioning pass is the innermost level's text path."""
        return super().forward_conditioning(conditioning, cond_mask)

    def _level_configs(self):
        return [self._config] + self.inner_unet._level_configs()

    def _levels(self):
        return [self] + self.inner_unet._levels()

    def print_size(self, target_image_size=256):
        pass
