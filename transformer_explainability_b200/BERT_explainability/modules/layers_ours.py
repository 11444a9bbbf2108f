"""Drop-in for ``BERT_explainability/modules/layers_ours.py``: the ViT rule library plus ``MatMul``, ``Mul``,
``Tanh`` (``:77-91`` of the reference)."""
import torch
import torch.nn as nn

from transformer_explainability_b200.modules.layers_ours import *            # noqa: F401,F403
from transformer_explainability_b200.modules.layers_ours import RelProp, RelPropSimple, _c, _mix
from transformer_explainability_b200.modules import layers_ours as _base
from transformer_explainability_b200 import ops

__all__ = list(_base.__all__) + ["MatMul", "Mul", "Tanh"]

Tanh = _mix("Tanh", nn.Tanh, RelProp)           # identity relprop


class MatMul(RelPropSimple):
    """``torch.matmul(*inputs)`` with the attention matmul rules: inputs [q, k^T] or [probs, v]."""

    def forward(self, inputs):
        return torch.matmul(*inputs)

    def relprop(self, R, alpha):
        a, b = self.X
        if a.shape[-1] == a.shape[-2] == b.shape[-2] and R.shape == torch.Size(list(a.shape[:-1]) + [b.shape[-1]]) \
                and a.shape[-1] != b.shape[-1]:
            return list(ops.matmul_av_relprop(_c(a), _c(b), _c(R)))                 # [probs, v]
        # [q, k^T]: the rule is stated for (q, k); return the k relevance transposed like the stored operand
        rq, rk = ops.matmul_qk_relprop(_c(a), _c(b.transpose(-1, -2)), _c(R))
        return [rq, rk.transpose(-1, -2)]


class Mul(RelPropSimple):
    def forward(self, inputs):
        return torch.mul(*inputs)
