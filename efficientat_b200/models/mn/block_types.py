"""Parameter containers mirroring reference models/mn/block_types.py (state_dict keys, repr).

The modules below hold nn.Parameters/buffers under exactly the reference's names
(`block.{j}.0.weight`, `block.{j}.1.running_mean`, `conc_se_layers.0.fc1.weight`, ...) so that
reference checkpoints load unchanged; they do not compute.  The whole network is executed by
efficientat_b200.engine (fused CUDA kernels); calling a container's forward directly raises --
there is deliberately no PyTorch-op fallback.
"""
from typing import Callable, Dict, List

import torch.nn as nn

from .utils import cnn_out_size, make_divisible


class FusedOnly(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError(f"{type(self).__name__} is a parameter container; it is executed by the fused CUDA "
                           "engine through the top-level model's forward (no per-module PyTorch fallback)")


class ConvNormActivation(nn.Sequential, FusedOnly):
    """conv(bias=False, padding=(k-1)//2*dilation) -> norm -> activation  (torchvision.ops.misc
    semantics as used at models/mn/block_types.py:140-170)."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, groups=1, norm_layer=None,
                 activation_layer=None, dilation=1):
        padding = (kernel_size - 1) // 2 * dilation
        layers: List[nn.Module] = [nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding,
                                             dilation=dilation, groups=groups, bias=norm_layer is None)]
        if norm_layer is not None:
            layers.append(norm_layer(out_channels))
        if activation_layer is not None:
            layers.append(activation_layer(inplace=True))
        nn.Sequential.__init__(self, *layers)
        self.out_channels = out_channels

    forward = FusedOnly.forward


class SqueezeExcitation(FusedOnly):
    """fc1 -> ReLU -> fc2 -> Sigmoid gate over the mean of the non-squeezed dims (block_types.py:45-83)."""

    def __init__(self, input_dim, squeeze_dim, se_dim):
        super().__init__()
        self.fc1 = nn.Linear(input_dim, squeeze_dim)
        self.fc2 = nn.Linear(squeeze_dim, input_dim)
        assert se_dim in [1, 2, 3]
        self.se_dim = [d for d in (1, 2, 3) if d != se_dim]
        self.activation = nn.ReLU()
        self.scale_activation = nn.Sigmoid()


class ConcurrentSEBlock(FusedOnly):
    def __init__(self, c_dim, f_dim, t_dim, se_cnf: Dict):
        super().__init__()
        dims = [c_dim, f_dim, t_dim]
        if se_cnf["se_agg"] not in ("max", "avg", "add", "min"):
            raise NotImplementedError(f"SE aggregation operation '{se_cnf['se_agg']}' not implemented")
        if list(se_cnf["se_dims"]) != [1]:
            raise NotImplementedError("the fused engine implements channel squeeze-excitation (se_dims='c') only; "
                                      f"got se_dims={se_cnf['se_dims']}")
        self.conc_se_layers = nn.ModuleList()
        for d in se_cnf["se_dims"]:
            input_dim = dims[d - 1]
            squeeze_dim = make_divisible(input_dim // se_cnf["se_r"], 8)
            self.conc_se_layers.append(SqueezeExcitation(input_dim, squeeze_dim, d))


class InvertedResidualConfig:
    """One row of the MobileNetV3 table scaled by width_mult (block_types.py:86-117)."""

    def __init__(self, input_channels, kernel, expanded_channels, out_channels, use_se, activation, stride,
                 dilation, width_mult):
        self.input_channels = self.adjust_channels(input_channels, width_mult)
        self.kernel = kernel
        self.expanded_channels = self.adjust_channels(expanded_channels, width_mult)
        self.out_channels = self.adjust_channels(out_channels, width_mult)
        self.use_se = use_se
        self.use_hs = activation == "HS"
        self.stride = stride
        self.dilation = dilation
        self.f_dim = None
        self.t_dim = None

    @staticmethod
    def adjust_channels(channels, width_mult):
        return make_divisible(channels * width_mult, 8)

    def out_size(self, in_size):
        padding = (self.kernel - 1) // 2 * self.dilation
        return cnn_out_size(in_size, padding, self.dilation, self.kernel, self.stride)


class InvertedResidual(FusedOnly):
    """[expand 1x1] -> depthwise -> [SE] -> project 1x1 (+ input)  (block_types.py:120-181)."""

    def __init__(self, cnf: InvertedResidualConfig, se_cnf: Dict, norm_layer: Callable[..., nn.Module],
                 depthwise_norm_layer: Callable[..., nn.Module]):
        super().__init__()
        if not (1 <= cnf.stride <= 2):
            raise ValueError("illegal stride value")
        if cnf.dilation not in (1, 2):
            raise NotImplementedError("the fused engine implements depthwise dilation 1 and 2 only")
        self.use_res_connect = cnf.stride == 1 and cnf.input_channels == cnf.out_channels
        layers: List[nn.Module] = []
        activation_layer = nn.Hardswish if cnf.use_hs else nn.ReLU
        if cnf.expanded_channels != cnf.input_channels:
            layers.append(ConvNormActivation(cnf.input_channels, cnf.expanded_channels, kernel_size=1,
                                             norm_layer=norm_layer, activation_layer=activation_layer))
        layers.append(ConvNormActivation(cnf.expanded_channels, cnf.expanded_channels, kernel_size=cnf.kernel,
                                         stride=1 if cnf.dilation > 1 else cnf.stride, dilation=cnf.dilation,
                                         groups=cnf.expanded_channels,
                                         norm_layer=depthwise_norm_layer, activation_layer=activation_layer))
        if cnf.use_se and se_cnf is not None and se_cnf["se_dims"] is not None:
            layers.append(ConcurrentSEBlock(cnf.expanded_channels, cnf.f_dim, cnf.t_dim, se_cnf))
        layers.append(ConvNormActivation(cnf.expanded_channels, cnf.out_channels, kernel_size=1,
                                         norm_layer=norm_layer, activation_layer=None))
        self.block = nn.Sequential(*layers)
        self.out_channels = cnf.out_channels
        self._is_cn = cnf.stride > 1
        self.cnf = cnf
