"""Drop-in for the reference's models/dymn/model.py: DyMN + get_model().

Same factory signature, module tree / state_dict keys, `forward(x, return_fmaps=False)` and
`update_params(epoch)` as reference models/dymn/model.py:36-361; compute runs in
efficientat_b200.engine_dymn (fused sm_90a kernels).
"""
import urllib.parse
from functools import partial
from typing import Any, Callable, List, Optional, Sequence, Tuple

import torch
from torch import Tensor, nn
from torch.hub import load_state_dict_from_url

from ..common import check_head, check_setting, mlp_head, reference_init_, v3_large_rows
from ..mn.block_types import ConvNormActivation, InvertedResidual
from .dy_block import DY_Block, DynamicConv, DynamicInvertedResidualConfig

model_url = "https://github.com/fschmid56/EfficientAT/releases/download/v0.0.1/"
model_dir = "resources"
_release_files = {
    "dymn04_im": "dymn04_im.pt", "dymn10_im": "dymn10_im.pt", "dymn20_im": "dymn20_im.pt",
    "dymn04_as": "dymn04_as.pt", "dymn10_as": "dymn10_as.pt", "dymn20_as": "dymn20_as_mAP_493.pt",
    "dymn20_as(2)": "dymn20_as_mAP_493.pt", "dymn20_as(3)": "dymn20_as_mAP_490.pt",
    "dymn04_replace_se_as": "dymn04_replace_se_as.pt", "dymn10_replace_se_as": "dymn10_replace_se_as.pt",
}
pretrained_models = {k: urllib.parse.urljoin(model_url, v) for k, v in _release_files.items()}


class DyMN(nn.Module):
    """in_c (stem) -> layers[15] (DY_Block | InvertedResidual) -> out_c (1x1) -> classifier; parameter container."""

    def __init__(self, inverted_residual_setting: List[DynamicInvertedResidualConfig], last_channel: int,
                 num_classes: int = 527, head_type: str = "mlp", block: Optional[Callable[..., nn.Module]] = None,
                 norm_layer: Optional[Callable[..., nn.Module]] = None, dropout: float = 0.2,
                 in_conv_kernel: int = 3, in_conv_stride: int = 2, in_channels: int = 1, context_ratio: int = 4,
                 max_context_size: int = 128, min_context_size: int = 32, dyrelu_k=2, dyconv_k=4,
                 no_dyrelu: bool = False, no_dyconv: bool = False, no_ca: bool = False,
                 temp_schedule: tuple = (30, 1, 1, 0.05), **kwargs: Any) -> None:
        super().__init__()
        check_setting(inverted_residual_setting, DynamicInvertedResidualConfig)
        check_head(head_type)
        if in_conv_kernel != 3 or in_channels != 1:
            raise NotImplementedError("the fused stem kernel implements a 3x3 convolution on 1 input channel")
        make_block = DY_Block if block is None else block
        bn = partial(nn.BatchNorm2d, eps=0.001, momentum=0.01) if norm_layer is None else norm_layer
        dy_kwargs = dict(context_ratio=context_ratio, max_context_size=max_context_size,
                         min_context_size=min_context_size, dyrelu_k=dyrelu_k, dyconv_k=dyconv_k, no_dyrelu=no_dyrelu,
                         no_dyconv=no_dyconv, no_ca=no_ca, temp_schedule=temp_schedule)
        first, last = inverted_residual_setting[0], inverted_residual_setting[-1]
        self.layers = nn.ModuleList()
        self.in_c = ConvNormActivation(in_channels, first.input_channels, kernel_size=in_conv_kernel,
                                       stride=in_conv_stride, norm_layer=bn, activation_layer=nn.Hardswish)
        for cnf in inverted_residual_setting:
            self.layers.append(make_block(cnf, **dy_kwargs) if cnf.use_dy_block else
                               InvertedResidual(cnf, None, bn, partial(nn.BatchNorm2d, eps=0.001, momentum=0.01)))
        self.out_c = ConvNormActivation(last.out_channels, 6 * last.out_channels, kernel_size=1, norm_layer=bn,
                                        activation_layer=nn.Hardswish)
        self.head_type = head_type
        self.classifier = mlp_head(6 * last.out_channels, last_channel, num_classes, dropout)
        reference_init_(self)
        self._engine = None
        self.precision = kwargs.get("precision", "fp32")

    def engine(self):
        if self._engine is None:
            from ...engine_dymn import DyMNEngine
            object.__setattr__(self, "_engine", DyMNEngine(self))
        return self._engine

    def _forward_impl(self, x: Tensor, return_fmaps: bool = False, lengths=None):
        """lengths (eval only): each clip's frame count, as MN._forward_impl"""
        logits, embed, fmaps = self.engine().forward(x, return_fmaps=return_fmaps, lengths=lengths)
        return (logits, fmaps) if return_fmaps else (logits, embed)

    def forward(self, x: Tensor, return_fmaps: bool = False, lengths=None):
        return self._forward_impl(x, return_fmaps, lengths)

    def update_params(self, epoch):
        """per-epoch DynamicConv temperature update (ex_audioset.py:132-133)"""
        for module in self.modules():
            if isinstance(module, DynamicConv):
                module.update_params(epoch)


_REPLACE_SE = (3, 4, 5, 10, 11, 12, 13, 14)       # rows that carry squeeze-excitation in MobileNetV3


def _dymn_conf(width_mult: float = 1.0, reduced_tail: bool = False, dilated: bool = False,
               strides: Tuple[int, ...] = (2, 2, 2, 2), use_dy_blocks: str = "all", **kwargs: Any):
    """15 block configs + classifier width (reference models/dymn/model.py:209-254)."""
    rows, last = v3_large_rows(strides, reduced_tail, dilated)
    if use_dy_blocks == "all":
        dynamic = [True] * len(rows)
    elif use_dy_blocks == "replace_se":
        dynamic = [i in _REPLACE_SE for i in range(len(rows))]
    else:
        raise NotImplementedError(f"Config use_dy_blocks={use_dy_blocks} not implemented.")
    setting = [DynamicInvertedResidualConfig(cin, k, cexp, cout, dynamic[i], act, stride, dil, width_mult)
               for i, (cin, k, cexp, cout, _se, act, stride, dil) in enumerate(rows)]
    return setting, DynamicInvertedResidualConfig.adjust_channels(last, width_mult)


def _dymn(inverted_residual_setting, last_channel, pretrained_name, **kwargs):
    model = DyMN(inverted_residual_setting, last_channel, **kwargs)
    if pretrained_name:                                                            # dymn/model.py:264-280
        url = pretrained_models.get(pretrained_name)
        state_dict = load_state_dict_from_url(url, model_dir=model_dir, map_location="cpu")
        cls_in_state_dict = state_dict["classifier.5.weight"].shape[0]
        cls_in_current_model = model.classifier[5].out_features
        if cls_in_state_dict != cls_in_current_model:
            print(f"The number of classes in the loaded state dict (={cls_in_state_dict}) and "
                  f"the current model (={cls_in_current_model}) is not the same. Dropping final fully-connected "
                  f"layer and loading weights in non-strict mode!")
            del state_dict["classifier.5.weight"]
            del state_dict["classifier.5.bias"]
            model.load_state_dict(state_dict, strict=False)
        else:
            model.load_state_dict(state_dict)
    return model


def dymn(pretrained_name: str = None, **kwargs: Any):
    setting, last_channel = _dymn_conf(**kwargs)
    return _dymn(setting, last_channel, pretrained_name, **kwargs)


def get_model(num_classes: int = 527, pretrained_name: str = None, width_mult: float = 1.0,
              strides: Tuple[int, int, int, int] = (2, 2, 2, 2), context_ratio: int = 4,
              max_context_size: int = 128, min_context_size: int = 32, dyrelu_k: int = 2, no_dyrelu: bool = False,
              dyconv_k: int = 4, no_dyconv: bool = False, T_max: float = 30.0, T0_slope: float = 1.0,
              T1_slope: float = 0.02, T_min: float = 1, pretrain_final_temp: float = 1.0, no_ca: bool = False,
              use_dy_blocks="all", precision: str = "fp32", verbose: bool = True):
    """Reference signature (dymn/model.py:289-310) + `precision`, `verbose` (see mn.model.get_model)."""
    if pretrained_name:
        T_max = pretrain_final_temp            # dymn/model.py:336-340
    temp_schedule = (T_max, T_min, T0_slope, T1_slope)
    m = dymn(num_classes=num_classes, pretrained_name=pretrained_name, block=DY_Block, width_mult=width_mult,
             strides=strides, context_ratio=context_ratio, max_context_size=max_context_size,
             min_context_size=min_context_size, dyrelu_k=dyrelu_k, dyconv_k=dyconv_k, no_dyrelu=no_dyrelu,
             no_dyconv=no_dyconv, no_ca=no_ca, temp_schedule=temp_schedule, use_dy_blocks=use_dy_blocks,
             precision=precision)
    if verbose:
        print(m)
    return m
