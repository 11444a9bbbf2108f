"""Drop-in for ``modules/layers_lrp.py``: the rule library of the "LRP" baselines.  Identical to ``layers_ours`` except
``Linear.relprop`` (each half divided by its OWN denominator, ``layers_lrp.py:199-200``) and ``Add.relprop`` (plain
``RelPropSimple``, no ratio normalisation, ``:98-100``); every ``relprop`` is one C-ABI call."""
from transformer_explainability_b200 import ops
from .layers_ours import *                                            # noqa: F401,F403
from .layers_ours import RelPropSimple, RelProp, _c, nn, torch

__all__ = ['forward_hook', 'Clone', 'Add', 'Cat', 'ReLU', 'GELU', 'Dropout', 'BatchNorm2d', 'Linear', 'MaxPool2d',
           'AdaptiveAvgPool2d', 'AvgPool2d', 'Conv2d', 'Sequential', 'safe_divide', 'einsum', 'Softmax', 'IndexSelect',
           'LayerNorm', 'AddEye']


class Add(RelPropSimple):
    def forward(self, inputs):
        return torch.add(*inputs)

    def relprop(self, R, alpha):
        a, b = self.X
        if b.shape != a.shape:
            raise NotImplementedError("broadcast Add.relprop is not on the ViT_orig_LRP path")
        return list(ops.add_relprop(_c(a), _c(b), _c(R), variant="lrp"))


class Linear(nn.Linear, RelProp):
    def relprop(self, R, alpha):
        return ops.linear_relprop(_c(self.X), _c(self.weight), _c(R), variant="lrp", alpha=alpha)
