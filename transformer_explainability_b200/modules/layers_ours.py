"""Drop-in for the reference's ``modules/layers_ours.py``: same names, same ``relprop(R, alpha)``
protocol, but every rule runs as an sm_90a CUDA kernel through the C ABI (``ops``) instead of a
re-forward + ``torch.autograd.grad``.

``Linear.relprop(R, alpha)`` applies the LRP-alpha-beta rule with beta = alpha - 1 (``layers_ours.py:207-230``); every
other rule does not depend on alpha and ignores it, as in the reference.  Layers whose
relprop is the identity in the reference (Softmax, LayerNorm, GELU, Dropout, ReLU —
``layers_ours.py:45-46,67-80``) stay the identity.  Layers that are not on the
transformer-attribution path (Conv2d, BatchNorm2d, pools, Cat, AddEye) keep their forward and raise
in ``relprop`` — they are out of scope (SURVEY.md §8f-3).
"""
import torch
import torch.nn as nn

from transformer_explainability_b200 import ops

__all__ = ['forward_hook', 'Clone', 'Add', 'Cat', 'ReLU', 'GELU', 'Dropout', 'BatchNorm2d', 'Linear', 'MaxPool2d',
           'AdaptiveAvgPool2d', 'AvgPool2d', 'Conv2d', 'Sequential', 'safe_divide', 'einsum', 'Softmax', 'IndexSelect',
           'LayerNorm', 'AddEye']


def safe_divide(a, b):
    """``layers_ours.py:10-13`` (plain tensor arithmetic; the fused kernels inline the same formula)."""
    den = b.clamp(min=1e-9) + b.clamp(max=1e-9)
    den = den + den.eq(0).type(den.type()) * 1e-9
    return a / den * b.ne(0).type(b.type())


def forward_hook(self, input, output):
    """``layers_ours.py:16-27``: keep the layer input(s) for relprop (detached; no autograd graph is needed)."""
    if type(input[0]) in (list, tuple):
        self.X = [i.detach() for i in input[0]]
    else:
        self.X = input[0].detach()
    self.Y = output


def _c(t):
    return t.detach().to(torch.float32).contiguous()


class RelProp(nn.Module):
    def __init__(self):
        super(RelProp, self).__init__()
        self.register_forward_hook(forward_hook)

    def relprop(self, R, alpha):
        return R


class RelPropSimple(RelProp):
    def relprop(self, R, alpha):
        raise NotImplementedError("%s.relprop is not on the transformer-attribution path" % type(self).__name__)


def _mix(name, base, rule):
    """``class <name>(<base>, <rule>): pass`` — torch forward + the given relprop rule."""
    return type(name, (base, rule), {"__module__": __name__})


# identity relprop in the reference (layers_ours.py:67-80)
ReLU = _mix("ReLU", nn.ReLU, RelProp)
GELU = _mix("GELU", nn.GELU, RelProp)
Softmax = _mix("Softmax", nn.Softmax, RelProp)
LayerNorm = _mix("LayerNorm", nn.LayerNorm, RelProp)
Dropout = _mix("Dropout", nn.Dropout, RelProp)
# not on the attribution path
MaxPool2d = _mix("MaxPool2d", nn.MaxPool2d, RelPropSimple)
AdaptiveAvgPool2d = _mix("AdaptiveAvgPool2d", nn.AdaptiveAvgPool2d, RelPropSimple)
AvgPool2d = _mix("AvgPool2d", nn.AvgPool2d, RelPropSimple)


class AddEye(RelPropSimple):
    def forward(self, input):
        return input + torch.eye(input.shape[2]).expand_as(input).to(input.device)


class Add(RelPropSimple):
    def forward(self, inputs):
        return torch.add(*inputs)

    def relprop(self, R, alpha):
        a, b = self.X
        if b.shape != a.shape:
            raise NotImplementedError("broadcast Add.relprop is handled inside the BERT engine")
        ra, rb = ops.add_relprop(_c(a), _c(b), _c(R))
        return [ra, rb]


class einsum(RelPropSimple):
    def __init__(self, equation):
        super().__init__()
        self.equation = equation

    def forward(self, *operands):
        return torch.einsum(self.equation, *operands)

    def relprop(self, R, alpha):
        a, b = self.X
        if self.equation == 'bhij,bhjd->bhid':
            return list(ops.matmul_av_relprop(_c(a), _c(b), _c(R)))
        if self.equation == 'bhid,bhjd->bhij':
            return list(ops.matmul_qk_relprop(_c(a), _c(b), _c(R)))
        raise NotImplementedError("einsum.relprop: only the two attention equations are implemented")


class IndexSelect(RelProp):
    def forward(self, inputs, dim, indices):
        self.__setattr__('dim', dim)
        self.__setattr__('indices', indices)
        return torch.index_select(inputs, dim, indices)

    def relprop(self, R, alpha):
        if self.dim != 1 or int(self.indices) != 0:
            raise NotImplementedError("IndexSelect.relprop: only dim=1, index 0 (the CLS pool) is implemented")
        return ops.index_select_relprop(_c(self.X), _c(R))


class Clone(RelProp):
    def forward(self, input, num):
        self.__setattr__('num', num)
        return [input for _ in range(num)]

    def relprop(self, R, alpha):
        return ops.clone_relprop(_c(self.X), [_c(r) for r in R])


class Cat(RelProp):
    def forward(self, inputs, dim):
        self.__setattr__('dim', dim)
        return torch.cat(inputs, dim)

    def relprop(self, R, alpha):
        raise NotImplementedError("Cat.relprop is not on the transformer-attribution path")


class Sequential(nn.Sequential):
    def relprop(self, R, alpha):
        for m in reversed(self._modules.values()):
            R = m.relprop(R, alpha)
        return R


class BatchNorm2d(nn.BatchNorm2d, RelProp):
    def relprop(self, R, alpha):
        raise NotImplementedError("BatchNorm2d.relprop is not on the transformer-attribution path")


class Linear(nn.Linear, RelProp):
    def relprop(self, R, alpha):
        return ops.linear_relprop(_c(self.X), _c(self.weight), _c(R), alpha=alpha)


class Conv2d(nn.Conv2d, RelProp):
    def relprop(self, R, alpha):
        """``layers_ours.py:242-259``, 3-channel (z^B) branch, for the patch-embedding geometry the reference uses it
        with (kernel == stride, no padding, ``ViT_LRP.py:228``): R [B,D,H/P,W/P] -> [B,3,H,W]."""
        x = self.X
        k, st = self.kernel_size, self.stride
        if x.shape[1] != 3 or k != st or k[0] != k[1] or tuple(self.padding) != (0, 0) or x.shape[2] != x.shape[3]:
            raise NotImplementedError("Conv2d.relprop: only the 3-channel z^B rule of a square kernel == stride, "
                                      "unpadded (patch-embedding) convolution is on the attribution path")
        r = R.flatten(2).transpose(1, 2)                       # [B, np, D], the layout PatchEmbed.relprop receives
        return ops.patch_embed_relprop(_c(x), _c(self.weight), _c(r), per_channel=True)
