"""Parameter container mirroring reference models/mn/attention_pooling.py:9-56 (MN head_type='multihead_attention_pooling').

Same attribute names, construction order and initialisation as the reference (`subspace_proj` Linear first, then
`head_weight` = 1/num_heads), so state_dict keys, `named_parameters()` order and the RNG draws of model construction
match.  The head is executed by efficientat_b200.engine (frequency mean, projection GEMM, attention pooling kernels)."""
import torch
import torch.nn as nn

from .block_types import FusedOnly


class MultiHeadAttentionPooling(FusedOnly):
    """Multi-head attention pooling as in PSLA (https://arxiv.org/pdf/2102.01243.pdf): per head, a sigmoid attention over
    time (clamped to [epsilon, 1 - epsilon] and normalised) weighs an identity-activated value; heads are mixed by
    `head_weight`."""

    def __init__(self, in_dim, out_dim, att_activation: str = "sigmoid", clf_activation: str = "ident",
                 num_heads: int = 4, epsilon: float = 1e-7):
        super().__init__()
        if att_activation != "sigmoid" or clf_activation != "ident":
            raise NotImplementedError("the fused engine implements att_activation='sigmoid', clf_activation='ident' "
                                      "(what MN builds, mn/model.py:170-172)")
        self.in_dim = in_dim
        self.out_dim = out_dim
        self.num_heads = num_heads
        self.epsilon = epsilon
        self.att_activation = att_activation
        self.clf_activation = clf_activation
        self.subspace_proj = nn.Linear(self.in_dim, self.out_dim * 2 * self.num_heads)
        self.head_weight = nn.Parameter(torch.tensor([1.0 / self.num_heads] * self.num_heads).view(1, -1, 1))
