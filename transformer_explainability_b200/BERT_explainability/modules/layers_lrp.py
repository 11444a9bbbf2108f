"""Drop-in for ``BERT_explainability/modules/layers_lrp.py``: the ViT ``layers_lrp`` rule library plus ``MatMul``, ``Mul``,
``Tanh``, whose rules are the same in both libraries (``RelPropSimple`` / identity)."""
from transformer_explainability_b200.modules.layers_lrp import *             # noqa: F401,F403
from transformer_explainability_b200.modules import layers_lrp as _base
from .layers_ours import MatMul, Mul, Tanh                                    # noqa: F401

__all__ = list(_base.__all__) + ["MatMul", "Mul", "Tanh"]
