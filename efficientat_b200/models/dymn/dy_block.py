"""Parameter containers mirroring reference models/dymn/dy_block.py (state_dict keys, repr,
temperature schedule).  Compute is done by efficientat_b200.engine_dymn; see mn/block_types.py
for the container convention (forward of a container raises: no PyTorch fallback)."""
from functools import partial
from typing import Any

import numpy as np
import torch
import torch.nn as nn

from ..mn.block_types import FusedOnly
from .utils import cnn_out_size, make_divisible


class DynamicInvertedResidualConfig:
    """dy_block.py:11-41"""

    def __init__(self, input_channels, kernel, expanded_channels, out_channels, use_dy_block, activation, stride,
                 dilation, width_mult):
        self.input_channels = self.adjust_channels(input_channels, width_mult)
        self.kernel = kernel
        self.expanded_channels = self.adjust_channels(expanded_channels, width_mult)
        self.out_channels = self.adjust_channels(out_channels, width_mult)
        self.use_dy_block = use_dy_block
        self.use_hs = activation == "HS"
        self.use_se = False
        self.stride = stride
        self.dilation = dilation
        self.width_mult = width_mult

    @staticmethod
    def adjust_channels(channels, width_mult):
        return make_divisible(channels * width_mult, 8)

    def out_size(self, in_size):
        padding = (self.kernel - 1) // 2 * self.dilation
        return cnn_out_size(in_size, padding, self.dilation, self.kernel, self.stride)


class DynamicConv(FusedOnly):
    """K kernel banks [1, 1, K, Cout*Cin/g*ks*ks] mixed per sample by softmax(Linear(h_c)/T)
    (dy_block.py:44-139)."""

    def __init__(self, in_channels, out_channels, context_dim, kernel_size, stride=1, dilation=1, padding=0,
                 groups=1, att_groups=1, bias=False, k=4, temp_schedule=(30, 1, 1, 0.05)):
        super().__init__()
        assert in_channels % groups == 0
        if att_groups != 1 or bias:
            raise NotImplementedError("DynamicConv: att_groups > 1 and bias are not implemented by the fused engine")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding, self.dilation = kernel_size, stride, padding, dilation
        self.groups, self.k, self.att_groups = groups, k, att_groups
        self.T_max, self.T_min, self.T0_slope, self.T1_slope = temp_schedule
        self.temperature = self.T_max
        self.residuals = nn.Sequential(nn.Linear(context_dim, k * att_groups))
        weight = torch.randn(k, out_channels, in_channels // groups, kernel_size, kernel_size)
        for i in range(k):
            nn.init.kaiming_normal_(weight[i], mode="fan_out")
        self.weight = nn.Parameter(weight.view(1, 1, k, -1).clone(), requires_grad=True)
        self.bias = None

    def extra_repr(self):
        return (f"{self.in_channels}, {self.out_channels}, kernel_size={self.kernel_size}, stride={self.stride}, "
                f"groups={self.groups}, k={self.k}")

    def update_params(self, epoch):
        """temperature schedule, dy_block.py:133-139 (prints like the reference)"""
        t0 = self.T_max - self.T0_slope * epoch
        t1 = 1 + self.T1_slope * (self.T_max - 1) / self.T0_slope - self.T1_slope * epoch
        self.temperature = max(t0, t1, self.T_min)
        print(f"Setting temperature for attention over kernels to {self.temperature}")


class DyReLU(FusedOnly):
    def __init__(self, channels, context_dim, M=2):
        super().__init__()
        self.channels = channels
        self.M = M
        self.coef_net = nn.Sequential(nn.Linear(context_dim, 2 * M))
        self.sigmoid = nn.Sigmoid()
        self.register_buffer("lambdas", torch.Tensor([1.] * M + [0.5] * M).float())
        self.register_buffer("init_v", torch.Tensor([1.] + [0.] * (2 * M - 1)).float())


class DyReLUB(DyReLU):
    """max_m (a_m x + b_m) over M linear pieces with per-(sample, channel) coefficients (dy_block.py:165-188).
    M = dyrelu_k in 1..4: the kernels hold the 2M coefficients of a channel in registers, and four pieces is where
    that budget ends.  On a tie the gradient goes to the lowest piece index (for M = 2 the reference's torch.maximum
    splits it in half; for M != 2 its torch.max also picks one piece)."""

    MAX_PIECES = 4

    def __init__(self, channels, context_dim, M=2):
        if not 1 <= M <= self.MAX_PIECES:
            raise NotImplementedError(f"DyReLUB: dyrelu_k (the number of linear pieces M) must be in "
                                      f"1..{self.MAX_PIECES} for the fused engine, got {M}")
        super().__init__(channels, context_dim, M)
        self.coef_net[-1] = nn.Linear(context_dim, 2 * M * self.channels)


class CoordAtt(FusedOnly):
    """x * sigmoid(g_f) * sigmoid(g_t)  (dy_block.py:191-201); parameter-free."""


class DynamicWrapper(FusedOnly):
    def __init__(self, module):
        super().__init__()
        self.module = module


class ContextGen(FusedOnly):
    """dy_block.py:214-254"""

    def __init__(self, context_dim, in_ch, exp_ch, norm_layer, stride: int = 1):
        super().__init__()
        self.joint_conv = nn.Conv2d(in_ch, context_dim, kernel_size=(1, 1), stride=(1, 1), padding=0, bias=False)
        self.joint_norm = norm_layer(context_dim)
        self.joint_act = nn.Hardswish(inplace=True)
        self.conv_f = nn.Conv2d(context_dim, exp_ch, kernel_size=(1, 1), stride=(1, 1), padding=0)
        self.conv_t = nn.Conv2d(context_dim, exp_ch, kernel_size=(1, 1), stride=(1, 1), padding=0)
        if stride > 1:
            self.pool_f = nn.AvgPool2d(kernel_size=(3, 1), stride=(stride, 1), padding=(1, 0))
            self.pool_t = nn.AvgPool2d(kernel_size=(1, 3), stride=(1, stride), padding=(0, 1))
        else:
            self.pool_f = nn.Sequential()
            self.pool_t = nn.Sequential()
        self.stride = stride


class DY_Block(FusedOnly):
    """dy_block.py:257-409"""

    def __init__(self, cnf: DynamicInvertedResidualConfig, context_ratio: int = 4, max_context_size: int = 128,
                 min_context_size: int = 32, temp_schedule: tuple = (30, 1, 1, 0.05), dyrelu_k: int = 2,
                 dyconv_k: int = 4, no_dyrelu: bool = False, no_dyconv: bool = False, no_ca: bool = False,
                 **kwargs: Any):
        super().__init__()
        if not (1 <= cnf.stride <= 2):
            raise ValueError("illegal stride value")
        if no_dyrelu or no_dyconv or no_ca:
            raise NotImplementedError("the ablation switches no_dyrelu / no_dyconv / no_ca are not implemented "
                                      "by the fused engine")
        if cnf.dilation != 1:
            raise NotImplementedError("dilated depthwise convolutions are not implemented by the fused engine")
        self.use_res_connect = cnf.stride == 1 and cnf.input_channels == cnf.out_channels
        self.context_dim = int(np.clip(make_divisible(cnf.expanded_channels // context_ratio, 8),
                                       make_divisible(min_context_size * cnf.width_mult, 8),
                                       make_divisible(max_context_size * cnf.width_mult, 8)))
        activation_layer = nn.Hardswish if cnf.use_hs else nn.ReLU
        norm_layer = partial(nn.BatchNorm2d, eps=0.001, momentum=0.01)
        if cnf.expanded_channels != cnf.input_channels:
            self.exp_conv = DynamicConv(cnf.input_channels, cnf.expanded_channels, self.context_dim, kernel_size=1,
                                        k=dyconv_k, temp_schedule=temp_schedule, stride=1, dilation=1, padding=0)
            self.exp_norm = norm_layer(cnf.expanded_channels)
            self.exp_act = DynamicWrapper(activation_layer(inplace=True))
        else:
            self.exp_conv = DynamicWrapper(nn.Identity())
            self.exp_norm = nn.Identity()
            self.exp_act = DynamicWrapper(nn.Identity())
        stride = cnf.stride
        padding = (cnf.kernel - 1) // 2 * cnf.dilation
        self.depth_conv = DynamicConv(cnf.expanded_channels, cnf.expanded_channels, self.context_dim,
                                      kernel_size=cnf.kernel, k=dyconv_k, temp_schedule=temp_schedule,
                                      groups=cnf.expanded_channels, stride=stride, dilation=cnf.dilation,
                                      padding=padding)
        self.depth_norm = norm_layer(cnf.expanded_channels)
        self.depth_act = DyReLUB(cnf.expanded_channels, self.context_dim, M=dyrelu_k)
        self.ca = CoordAtt()
        self.proj_conv = DynamicConv(cnf.expanded_channels, cnf.out_channels, self.context_dim, kernel_size=1,
                                     k=dyconv_k, temp_schedule=temp_schedule, stride=1, dilation=1, padding=0)
        self.proj_norm = norm_layer(cnf.out_channels)
        self.context_gen = ContextGen(self.context_dim, cnf.input_channels, cnf.expanded_channels,
                                      norm_layer=norm_layer, stride=stride)
        self.cnf = cnf
