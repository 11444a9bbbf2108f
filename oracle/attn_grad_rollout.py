"""Gradient-weighted attention rollout oracle (TEST INFRASTRUCTURE, CPU, any float dtype).

The LRP-free method of Chefer, Gur, Wolf, *Generic Attention-model Explainability for Interpreting Bi-Modal and
Encoder-Decoder Transformers* (ICCV 2021), self-attention rule, for one sample with L blocks, H heads, N tokens:

    A_l = attention probabilities of block l (``get_attn()``), G_l = d y_c / d A_l (``get_attn_gradients()``)
    Abar_l = mean_h max(G_l * A_l, 0)                                          [N, N]
    R = I ; for l = start_layer .. L-1:  R <- R + Abar_l @ R

ViT / DeiT maps are ``R[0, prefix:]``; BERT maps are ``R[0, :]`` with element 0 set to 0 (as the reference BERT
comparison generators do).  The rule is not in the reference repository; ``oracle/make_golden_attn_grad_rollout.py``
pins it on the reference's own attention maps and gradients.  Every map is computed one sample at a time, in the op
order ``cam = (grad * attn).clamp(min=0).mean(dim=0)``, ``R = R + cam @ R``, so the fixture's maps are reproduced
bit for bit from its stored taps.
"""
import torch

from . import bert as obert
from . import vit as ovit


def rollout(attns, grads, start_layer=0):
    """attns, grads: per block [B,H,N,N] -> R [B,N,N], each sample on its own."""
    B, _, N, _ = attns[0].shape
    out = []
    for b in range(B):
        R = torch.eye(N, dtype=attns[0].dtype)
        for l in range(start_layer, len(attns)):
            cam = (grads[l][b] * attns[l][b]).clamp(min=0).mean(dim=0)
            R = R + cam @ R
        out.append(R)
    return torch.stack(out)


def vit_map(attns, grads, start_layer=0, prefix=1):
    return rollout(attns, grads, start_layer)[:, 0, prefix:]


def bert_map(attns, grads, start_layer=0):
    m = rollout(attns, grads, start_layer)[:, 0].clone()
    m[:, 0] = 0
    return m


def _seed(logits, index):
    if index is None:
        index = logits.argmax(dim=-1)
    index = torch.as_tensor(index).reshape(-1).long()
    if index.numel() == 1 and logits.shape[0] > 1:
        index = index.expand(logits.shape[0])
    seed = torch.zeros_like(logits)
    seed[torch.arange(logits.shape[0]), index] = 1
    return seed, index


def vit_taps(params, x, num_heads, index=None, norm_eps=None):
    """(attns, grads, index) of the oracle's own ViT forward (``oracle/vit.py``); for DeiT-distilled the logits are the
    average of the two heads, so each head's share of the one-hot seed is one half.  ``norm_eps``: one epsilon for every
    LayerNorm (the ``ViT_new`` models)."""
    with torch.enable_grad():
        logits, cache = ovit.forward(params, x, num_heads, need_grad=True, norm_eps=norm_eps)
        seed, index = _seed(logits, index)
        grads = ovit.attention_gradients(cache, seed)
    return [c["attn"].detach() for c in cache["blocks"]], [g.detach() for g in grads], index


def bert_taps(params, input_ids, attention_mask, num_heads, index=None):
    with torch.enable_grad():
        logits, cache = obert.forward(params, input_ids, attention_mask, num_heads, need_grad=True)
        seed, index = _seed(logits, index)
        grads = obert.attention_gradients(cache, seed)
    return [c["probs"].detach() for c in cache["layers"]], [g.detach() for g in grads], index


def explain_vit(params, x, num_heads, index=None, start_layer=0, norm_eps=None):
    """-> (maps [B, N - prefix], index [B])."""
    attns, grads, index = vit_taps(params, x, num_heads, index, norm_eps)
    prefix = 2 if "dist_token" in params else 1
    with torch.no_grad():
        return vit_map(attns, grads, start_layer, prefix), index


def explain_bert(params, input_ids, attention_mask, num_heads, index=None, start_layer=0):
    """-> (maps [B, S], index [B]); padded positions are exactly 0."""
    attns, grads, index = bert_taps(params, input_ids, attention_mask, num_heads, index)
    with torch.no_grad():
        return bert_map(attns, grads, start_layer), index
