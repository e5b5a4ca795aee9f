"""Pieces shared by the MN and DyMN builders: the MobileNetV3-large row table, the 'mlp' classifier head and the
reference's weight initialisation.  (Reference: models/mn/model.py:186-210,252-268 and the identical code in
models/dymn/model.py:122-152,233-251.)"""
from torch import nn

# columns: input channels, kernel, expanded channels, output channels, squeeze-excitation, activation, stride slot
# (stride slot i means strides[i]; None means stride 1); channel numbers are for width_mult == 1.
_V3_LARGE = (
    (16, 3, 16, 16, False, "RE", None),
    (16, 3, 64, 24, False, "RE", 0),
    (24, 3, 72, 24, False, "RE", None),
    (24, 5, 72, 40, True, "RE", 1),
    (40, 5, 120, 40, True, "RE", None),
    (40, 5, 120, 40, True, "RE", None),
    (40, 3, 240, 80, False, "HS", 2),
    (80, 3, 200, 80, False, "HS", None),
    (80, 3, 184, 80, False, "HS", None),
    (80, 3, 184, 80, False, "HS", None),
    (80, 3, 480, 112, True, "HS", None),
    (112, 3, 672, 112, True, "HS", None),
    (112, 5, 672, 160, True, "HS", 3),
    (160, 5, 960, 160, True, "HS", None),
    (160, 5, 960, 160, True, "HS", None),
)
N_TAIL = 3      # the last three rows shrink with reduced_tail and dilate with dilated


def v3_large_rows(strides=(2, 2, 2, 2), reduced_tail=False, dilated=False):
    """-> list of (cin, kernel, cexp, cout, use_se, act, stride, dilation) for width_mult == 1."""
    div = 2 if reduced_tail else 1
    rows = []
    first_tail = len(_V3_LARGE) - N_TAIL
    for i, (cin, k, cexp, cout, se, act, slot) in enumerate(_V3_LARGE):
        tail = i >= first_tail
        if tail:
            cout //= div
            if i > first_tail:
                cin //= div
                cexp //= div
        rows.append((cin, k, cexp, cout, se, act, 1 if slot is None else strides[slot], 2 if (tail and dilated) else 1))
    return rows, 1280 // div


def mlp_head(in_features, hidden, num_classes, dropout):
    """AdaptiveAvgPool -> Flatten -> Linear -> Hardswish -> Dropout -> Linear, with the reference's child indices
    (classifier.2 / classifier.5 are the Linear layers; released checkpoints rely on those names)."""
    return nn.Sequential(nn.AdaptiveAvgPool2d(1), nn.Flatten(start_dim=1), nn.Linear(in_features, hidden),
                         nn.Hardswish(inplace=True), nn.Dropout(p=dropout, inplace=True), nn.Linear(hidden, num_classes))


def reference_init_(model):
    """kaiming-normal(fan_out) convs, unit BatchNorm, N(0, 0.01) Linear layers -- what the reference constructors do."""
    norm_types = (nn.BatchNorm2d, nn.GroupNorm, nn.LayerNorm, nn.InstanceNorm2d)
    for m in model.modules():
        if isinstance(m, nn.Conv2d):
            nn.init.kaiming_normal_(m.weight, mode="fan_out")
        elif isinstance(m, norm_types) and m.weight is not None:
            nn.init.ones_(m.weight)
        elif isinstance(m, nn.Linear):
            nn.init.normal_(m.weight, 0, 0.01)
        if isinstance(m, (nn.Conv2d, nn.Linear) + norm_types) and getattr(m, "bias", None) is not None:
            nn.init.zeros_(m.bias)


def head_dropout(model):
    """dropout rate of the classifier: the 'mlp' head's nn.Dropout (classifier.4); heads without dropout give 0"""
    return float(model.classifier[4].p) if isinstance(model.classifier, nn.Sequential) else 0.0


def check_head(head_type, supported=("mlp",)):
    """supported: the heads the calling model implements (MN adds 'multihead_attention_pooling'; DyMN, like the reference
    (dymn/model.py:140-142), has only 'mlp' and 'fully_convolutional')"""
    if head_type in supported:
        return
    if head_type in ("mlp", "fully_convolutional", "multihead_attention_pooling"):
        raise NotImplementedError(f"head_type '{head_type}' is not implemented by the fused engine "
                                  "(every released *_as checkpoint used by the benchmarks has the 'mlp' head)")
    raise NotImplementedError(f"Head '{head_type}' unknown. Must be one of: 'mlp', 'fully_convolutional', "
                              f"'multihead_attention_pooling'")


def check_setting(setting, cfg_type):
    if not setting:
        raise ValueError("The inverted_residual_setting should not be empty")
    if not (isinstance(setting, (list, tuple)) and all(isinstance(s, cfg_type) for s in setting)):
        raise TypeError(f"The inverted_residual_setting should be List[{cfg_type.__name__}]")
