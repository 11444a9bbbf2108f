"""BERT oracle for sentence pairs (TEST INFRASTRUCTURE, CPU, any float dtype): ``oracle/bert.py`` with ``token_type_ids``.

``BertEmbeddings.forward`` (``BERT.py:61-85``) adds ``token_type_embeddings(token_type_ids)`` before the embedding
LayerNorm, in the order ``(token_type + position) + word``; ``oracle.bert.forward`` restates it for ``token_type_ids = 0``
only.  ``forward`` below restates the embedding with any token types and runs the layers, pooler and classifier through
``oracle.bert``'s own ``layer_forward``; ``token_type_ids = None`` is segment 0, the same operations on the same operands
as ``oracle.bert.forward``, so the results are bit for bit those of ``oracle.bert``.

``explain`` / ``generate`` (and ``attn_grad_rollout.explain_bert``) run ``oracle.bert``'s unchanged generator code inside
``segments(token_type_ids)``, which binds the module's ``forward`` to this one for the duration of the call, the way
``oracle/make_golden_bert_pairs.py`` binds the reference model's ``forward`` with ``functools.partial``.
"""
import contextlib
import functools

import torch
import torch.nn.functional as F

from . import attn_grad_rollout as agr
from . import bert as obert


def forward(params, input_ids, attention_mask, num_heads, need_grad=False, token_type_ids=None):
    """``oracle.bert.forward`` with ``token_type_ids`` [B,S] (None: every token in segment 0) -> (logits, cache)."""
    p = params
    dm = obert.BertDims(params, num_heads)
    dtype = p["classifier.weight"].dtype
    B, S = input_ids.shape
    E = "bert.embeddings."
    types = torch.zeros_like(input_ids) if token_type_ids is None else torch.as_tensor(token_type_ids).long()
    word = p[E + "word_embeddings.weight"][input_ids]
    pos = p[E + "position_embeddings.weight"][:S].unsqueeze(0).expand(B, -1, -1)
    tt = p[E + "token_type_embeddings.weight"][types]
    emb = (tt + pos) + word                                           # add1([tt, pos]) ; add2([., word])  :80-81
    h = F.layer_norm(emb, (dm.dim,), p[E + "LayerNorm.weight"], p[E + "LayerNorm.bias"], dm.eps)
    if need_grad:
        h = h.detach().requires_grad_(True)
    ext_mask = (1.0 - attention_mask[:, None, None, :].to(dtype)) * -10000.0       # transformers 3.5.1
    cache = {"dims": dm, "layers": [], "ext_mask": ext_mask}
    for i in range(dm.depth):
        h, c = obert.layer_forward(p, dm, i, h, ext_mask)
        cache["layers"].append(c)
    cache["h_last"] = h
    pooled = torch.tanh(F.linear(h[:, 0], p["bert.pooler.dense.weight"], p["bert.pooler.dense.bias"]))
    cache["pooled"] = pooled
    logits = F.linear(pooled, p["classifier.weight"], p["classifier.bias"])
    cache["logits"] = logits
    return logits, cache


@contextlib.contextmanager
def segments(token_type_ids):
    """Within the block, every ``oracle.bert.forward`` call embeds with ``token_type_ids``."""
    orig = obert.forward
    obert.forward = functools.partial(forward, token_type_ids=token_type_ids)
    try:
        yield
    finally:
        obert.forward = orig


def explain(params, input_ids, attention_mask, num_heads, index=None, start_layer=11, return_taps=False,
            token_type_ids=None):
    """``oracle.bert.explain`` (``Generator.generate_LRP``) of sentence pairs -> ([B,S] maps, [B] index)."""
    with segments(token_type_ids):
        return obert.explain(params, input_ids, attention_mask, num_heads, index=index, start_layer=start_layer,
                             return_taps=return_taps)


def generate(params, input_ids, attention_mask, num_heads, which, index=None, start_layer=0, token_type_ids=None):
    """``oracle.bert.generate`` (the comparison generators of ``Generator``) of sentence pairs -> [B,S]."""
    with segments(token_type_ids):
        return obert.generate(params, input_ids, attention_mask, num_heads, which, index=index, start_layer=start_layer)


def explain_attn_grad_rollout(params, input_ids, attention_mask, num_heads, index=None, start_layer=0,
                              token_type_ids=None):
    """``attn_grad_rollout.explain_bert`` of sentence pairs -> ([B,S] maps, [B] index)."""
    with segments(token_type_ids):
        return agr.explain_bert(params, input_ids, attention_mask, num_heads, index=index, start_layer=start_layer)
