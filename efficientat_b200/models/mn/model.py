"""Drop-in for the reference's models/mn/model.py: MN (MobileNetV3 for audio tagging) + get_model().

Same factory signature, module tree / state_dict keys, `(logits, features)` return and B == 1
behaviour as reference models/mn/model.py:73-367.  The forward and backward passes run as fused
sm_90a kernels through efficientat_b200.engine; parameters stay ordinary fp32 nn.Parameters so
optimisers, `state_dict()` and `load_state_dict()` behave as in the reference.
"""
import urllib.parse
from functools import partial
from typing import Any, Callable, List, Optional, Sequence, Tuple

import torch
from torch import Tensor, nn
from torch.hub import load_state_dict_from_url

from ..common import check_head, check_setting, mlp_head, reference_init_, v3_large_rows
from ..mn.attention_pooling import MultiHeadAttentionPooling
from ..mn.block_types import ConvNormActivation, InvertedResidual, InvertedResidualConfig
from ..mn.utils import cnn_out_size

# release assets of the reference (models/mn/model.py:18-70); only the names are needed here
model_url = "https://github.com/fschmid56/EfficientAT/releases/download/v0.0.1/"
model_dir = "resources"
_release_files = {
    "mn10_im_pytorch": "mn10_im_pytorch.pt",
    **{f"mn{w}_im": f"mn{w}_im.pt" for w in ("01", "02", "04", "05", "10", "20", "30", "40")},
    "mn01_as": "mn01_as_mAP_298.pt", "mn02_as": "mn02_as_mAP_378.pt", "mn04_as": "mn04_as_mAP_432.pt",
    "mn05_as": "mn05_as_mAP_443.pt", "mn10_as": "mn10_as_mAP_471.pt", "mn20_as": "mn20_as_mAP_478.pt",
    "mn30_as": "mn30_as_mAP_482.pt", "mn40_as": "mn40_as_mAP_484.pt", "mn40_as(2)": "mn40_as_mAP_483.pt",
    "mn40_as(3)": "mn40_as_mAP_483(2).pt", "mn40_as_no_im_pre": "mn40_as_no_im_pre_mAP_483.pt",
    "mn40_as_no_im_pre(2)": "mn40_as_no_im_pre_mAP_483(2).pt", "mn40_as_no_im_pre(3)": "mn40_as_no_im_pre_mAP_482.pt",
    "mn40_as_ext": "mn40_as_ext_mAP_487.pt", "mn40_as_ext(2)": "mn40_as_ext_mAP_486.pt",
    "mn40_as_ext(3)": "mn40_as_ext_mAP_485.pt", "mn10_as_hop_5": "mn10_as_hop_5_mAP_475.pt",
    "mn10_as_hop_15": "mn10_as_hop_15_mAP_463.pt", "mn10_as_hop_20": "mn10_as_hop_20_mAP_456.pt",
    "mn10_as_hop_25": "mn10_as_hop_25_mAP_447.pt", "mn10_as_mels_40": "mn10_as_mels_40_mAP_453.pt",
    "mn10_as_mels_64": "mn10_as_mels_64_mAP_461.pt", "mn10_as_mels_256": "mn10_as_mels_256_mAP_474.pt",
    "mn10_as_fc": "mn10_as_fc_mAP_465.pt", "mn10_as_fc_s2221": "mn10_as_fc_s2221_mAP_466.pt",
    "mn10_as_fc_s2211": "mn10_as_fc_s2211_mAP_466.pt",
}
pretrained_models = {k: urllib.parse.urljoin(model_url, v) for k, v in _release_files.items()}


class MN(nn.Module):
    """features[0] stem -> features[1..15] InvertedResidual -> features[16] 1x1 conv -> classifier; parameter container."""

    def __init__(self, inverted_residual_setting: List[InvertedResidualConfig], last_channel: int,
                 num_classes: int = 1000, block: Optional[Callable[..., nn.Module]] = None,
                 norm_layer: Optional[Callable[..., nn.Module]] = None, dropout: float = 0.2,
                 in_conv_kernel: int = 3, in_conv_stride: int = 2, in_channels: int = 1, **kwargs: Any) -> None:
        super().__init__()
        check_setting(inverted_residual_setting, InvertedResidualConfig)
        self.head_type = kwargs.get("head_type", False)
        check_head(self.head_type, supported=("mlp", "multihead_attention_pooling"))
        if in_conv_kernel != 3 or in_channels != 1:
            raise NotImplementedError("the fused stem kernel implements a 3x3 convolution on 1 input channel")
        make_block = InvertedResidual if block is None else block
        bn = partial(nn.BatchNorm2d, eps=0.001, momentum=0.01) if norm_layer is None else norm_layer   # mn/model.py:114-115
        se_cnf = kwargs.get("se_conf", None)
        first, last = inverted_residual_setting[0], inverted_residual_setting[-1]
        # spatial sizes are tracked only because squeeze-excitation over f / t would need them (mn/model.py:138-151)
        f_dim, t_dim = (cnn_out_size(d, 1, 1, 3, 2) for d in kwargs.get("input_dims", (128, 1000)))
        layers: List[nn.Module] = [ConvNormActivation(in_channels, first.input_channels, kernel_size=in_conv_kernel,
                                                      stride=in_conv_stride, norm_layer=bn,
                                                      activation_layer=nn.Hardswish)]
        for cnf in inverted_residual_setting:
            f_dim, t_dim = cnf.out_size(f_dim), cnf.out_size(t_dim)
            cnf.f_dim, cnf.t_dim = f_dim, t_dim
            layers.append(make_block(cnf, se_cnf, bn, bn))
        layers.append(ConvNormActivation(last.out_channels, 6 * last.out_channels, kernel_size=1, norm_layer=bn,
                                         activation_layer=nn.Hardswish))
        self.features = nn.Sequential(*layers)
        if self.head_type == "multihead_attention_pooling":                          # mn/model.py:170-172
            self.classifier = MultiHeadAttentionPooling(6 * last.out_channels, num_classes,
                                                        num_heads=kwargs.get("multihead_attention_heads"))
        else:
            self.classifier = mlp_head(6 * last.out_channels, last_channel, num_classes, dropout)
        reference_init_(self)
        self._engine = None
        # 'fp32' keeps activations in fp32 (tensor-core bf16x3 / exact fp32 CUDA-core math, logits within 1e-3 of
        # the reference); 'bf16' stores activations in bf16.  See DESIGN.md section 3.
        self.precision = kwargs.get("precision", "fp32")

    def engine(self):
        if self._engine is None:
            from ...engine import MNEngine
            object.__setattr__(self, "_engine", MNEngine(self))
        return self._engine

    def _forward_impl(self, x: Tensor, return_fmaps: bool = False, lengths=None):
        """lengths (eval only): each clip's frame count, a sequence of ints or a CPU integer tensor of length B.  Row b
        of the result then equals the model on x[b:b+1, :, :, :lengths[b]] alone; x past a clip's length is never used."""
        logits, features, fmaps = self.engine().forward(x, return_fmaps=return_fmaps, lengths=lengths)
        return (logits, fmaps) if return_fmaps else (logits, features)

    def forward(self, x: Tensor, lengths=None):
        return self._forward_impl(x, lengths=lengths)


def _mobilenet_v3_conf(width_mult: float = 1.0, reduced_tail: bool = False, dilated: bool = False,
                       strides: Tuple[int, ...] = (2, 2, 2, 2), **kwargs: Any):
    """15 block configs + classifier width (reference models/mn/model.py:237-271)."""
    rows, last = v3_large_rows(strides, reduced_tail, dilated)
    setting = [InvertedResidualConfig(*row, width_mult=width_mult) for row in rows]
    return setting, InvertedResidualConfig.adjust_channels(last, width_mult)


def _mobilenet_v3(inverted_residual_setting, last_channel, pretrained_name, **kwargs):
    model = MN(inverted_residual_setting, last_channel, **kwargs)
    if pretrained_name in pretrained_models:                                        # mn/model.py:282-310
        url = pretrained_models.get(pretrained_name)
        state_dict = load_state_dict_from_url(url, model_dir=model_dir, map_location="cpu")
        # the released checkpoints have the 'mlp' head; for any other head the reference looks up the keys of the
        # 'fully_convolutional' one and raises KeyError (mn/model.py:287-302), and so does this branch
        if kwargs["head_type"] == "mlp":
            num_classes = state_dict["classifier.5.bias"].size(0)
        else:
            print("Loading weights for classifier only implemented for head types 'mlp' and 'fully_convolutional'")
            num_classes = -1
        if kwargs["num_classes"] != num_classes:
            pretrain_logits = state_dict["classifier.5.bias"].size(0) if kwargs["head_type"] == "mlp" \
                else state_dict["classifier.1.bias"].size(0)
            print(f"Number of classes defined: {kwargs['num_classes']}, "
                  f"but try to load pre-trained layer with logits: {pretrain_logits}\nDropping last layer.")
            if kwargs["head_type"] == "mlp":
                del state_dict["classifier.5.weight"]
                del state_dict["classifier.5.bias"]
            else:
                state_dict = {k: v for k, v in state_dict.items() if not k.startswith("classifier")}
        try:
            model.load_state_dict(state_dict)
        except RuntimeError as e:
            print(str(e))
            print("Loading weights pre-trained weights in a non-strict manner.")
            model.load_state_dict(state_dict, strict=False)
    elif pretrained_name:
        raise NotImplementedError(f"Model name '{pretrained_name}' unknown.")
    return model


def mobilenet_v3(pretrained_name: str = None, **kwargs: Any) -> MN:
    setting, last_channel = _mobilenet_v3_conf(**kwargs)
    return _mobilenet_v3(setting, last_channel, pretrained_name, **kwargs)


def get_model(num_classes: int = 527, pretrained_name: str = None, width_mult: float = 1.0,
              reduced_tail: bool = False, dilated: bool = False, strides: Tuple[int, int, int, int] = (2, 2, 2, 2),
              head_type: str = "mlp", multihead_attention_heads: int = 4, input_dim_f: int = 128,
              input_dim_t: int = 1000, se_dims: str = "c", se_agg: str = "max", se_r: int = 4,
              precision: str = "fp32", verbose: bool = True):
    """Reference signature (mn/model.py:326-329) plus two keyword-only extensions:
    `precision` ('fp32' | 'bf16' activation storage) and `verbose` (print the module tree, as the reference does)."""
    dim_map = {"c": 1, "f": 2, "t": 3}
    assert len(se_dims) <= 3 and all(s in dim_map for s in se_dims) or se_dims == "none"
    se_dims_l = None if se_dims == "none" else [dim_map[s] for s in se_dims]
    se_conf = dict(se_dims=se_dims_l, se_agg=se_agg, se_r=se_r)
    m = mobilenet_v3(pretrained_name=pretrained_name, num_classes=num_classes, width_mult=width_mult,
                     reduced_tail=reduced_tail, dilated=dilated, strides=strides, head_type=head_type,
                     multihead_attention_heads=multihead_attention_heads, input_dims=(input_dim_f, input_dim_t),
                     se_conf=se_conf, precision=precision)
    if verbose:
        print(m)
    return m
