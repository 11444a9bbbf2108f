"""Drop-in for the reference's ``baselines/ViT/ViT_new.py`` — the hook-free ViT that ``Baselines``
(``ViT_explanation_generator.py:45-83``) explains.  Same constructor arguments, ``state_dict`` keys and factories;
``forward(x, register_hook=False)`` runs on the CUDA engine and ``blk.attn.get_attention_map()`` /
``get_attn_gradients()`` read the engine workspace.  (The forward pass is the one of ``ViT_LRP``; only the final
LayerNorm epsilon differs: this file's factories pass ``eps=1e-6`` to every norm, ``ViT_new.py:226-254``.)"""
from functools import partial

import torch.nn as nn

from transformer_explainability_b200.baselines.ViT import ViT_LRP as _lrp

__all__ = ["VisionTransformer", "vit_base_patch16_224", "vit_large_patch16_224", "deit_base_patch16_224"]


class VisionTransformer(_lrp.VisionTransformer):
    def __init__(self, img_size=224, patch_size=16, in_chans=3, num_classes=1000, embed_dim=768, depth=12,
                 num_heads=12, mlp_ratio=4., qkv_bias=False, drop_rate=0., attn_drop_rate=0., norm_layer=nn.LayerNorm):
        if drop_rate or attn_drop_rate:
            raise NotImplementedError("dropout is inactive on the (eval-mode) explanation path")
        eps = norm_layer(4).eps
        super().__init__(img_size=img_size, patch_size=patch_size, in_chans=in_chans, num_classes=num_classes,
                         embed_dim=embed_dim, depth=depth, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias,
                         norm_eps=eps)

    def forward(self, x, register_hook=False):
        return super().forward(x)


def vit_base_patch16_224(pretrained=False, **kwargs):
    _lrp._no_pretrained(pretrained)
    return VisionTransformer(patch_size=16, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def vit_large_patch16_224(pretrained=False, **kwargs):
    _lrp._no_pretrained(pretrained)
    return VisionTransformer(patch_size=16, embed_dim=1024, depth=24, num_heads=16, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def deit_base_patch16_224(pretrained=False, **kwargs):
    _lrp._no_pretrained(pretrained)
    return VisionTransformer(patch_size=16, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)
