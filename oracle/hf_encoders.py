"""RoBERTa / XLM-RoBERTa and DistilBERT sequence-classifier oracle (TEST INFRASTRUCTURE, CPU, any float dtype).

The three families share BERT's post-LN encoder layer; only the embedding and the head differ (``transformers``
``RobertaEmbeddings`` / ``RobertaClassificationHead``, DistilBERT ``Embeddings`` / ``pre_classifier``):

* RoBERTa     position ids ``pad + cumsum(ids != pad)`` for non-pad tokens, ``pad`` for pad tokens
              (``create_position_ids_from_input_ids``); ``(word + type) + position``; ``out_proj(tanh(dense(h0)))``.
* DistilBERT  position ids ``arange(S)``; ``word + position``; ``classifier(relu(pre_classifier(h0)))``; eps 1e-12.

``to_bert_keys`` renames a family's ``state_dict`` to ``oracle.bert``'s key names (the head's dense takes the pooler's
name, its output layer the classifier's), and ``forward`` restates the family's embedding and head around
``oracle.bert.layer_forward``.  ``explain`` / ``generate`` / ``explain_attn_grad_rollout`` run ``oracle.bert``'s (and
``oracle.attn_grad_rollout``'s) unchanged generator code inside ``family(...)``, which binds ``oracle.bert.forward`` to
this ``forward`` for the duration of the call, the way ``oracle/bert_pairs.py`` binds its forward.  The relevance rules
are the BERT graph's: tanh and ReLU are identities for both rule libraries, so the relprop starts from the cached head
activation exactly as for BERT.  Any code that calls ``oracle.bert.forward`` (the layers_lrp oracle of the tests
included) runs a family's model inside ``family(...)``.

The mask is BERT's additive ``(1 - mask) * -10000``; ``transformers`` masks these families with the dtype minimum.
Padded keys get probability 0 either way (exp underflows), so the two agree up to rounding.
"""
import contextlib
import functools

import torch
import torch.nn.functional as F

from . import attn_grad_rollout as agr
from . import bert as obert

BERT, ROBERTA, DISTILBERT = 0, 1, 2              # TE_BERT_ARCH_*
DISTILBERT_EPS = 1e-12

_DISTIL_LAYER = {"attention.q_lin": "attention.self.query", "attention.k_lin": "attention.self.key",
                 "attention.v_lin": "attention.self.value", "attention.out_lin": "attention.output.dense",
                 "sa_layer_norm": "attention.output.LayerNorm", "ffn.lin1": "intermediate.dense",
                 "ffn.lin2": "output.dense", "output_layer_norm": "output.LayerNorm"}


def to_bert_keys(state_dict, arch):
    """A RoBERTa / XLM-R / DistilBERT classifier's ``state_dict`` under ``oracle.bert``'s key names."""
    out = {}
    for k, v in state_dict.items():
        if k.endswith("position_ids") or k.endswith("embeddings.token_type_ids"):
            continue
        if arch == ROBERTA:
            k = k.replace("roberta.", "bert.", 1)
            k = k.replace("classifier.dense.", "bert.pooler.dense.").replace("classifier.out_proj.", "classifier.")
        elif arch == DISTILBERT:
            k = k.replace("distilbert.", "bert.", 1).replace("bert.transformer.layer.", "bert.encoder.layer.")
            k = k.replace("pre_classifier.", "bert.pooler.dense.")
            if k.startswith("bert.encoder.layer."):
                head, rest = k.split(".", 4)[:4], k.split(".", 4)[4]
                mod, leaf = rest.rsplit(".", 1)
                k = ".".join(head) + "." + _DISTIL_LAYER[mod] + "." + leaf
        out[k] = v
    return out


def position_ids(input_ids, arch, pad):
    """The position of every token: RoBERTa's ``create_position_ids_from_input_ids``, else ``arange(S)``."""
    if arch == ROBERTA:
        m = input_ids.ne(pad).long()
        return torch.cumsum(m, dim=1) * m + pad
    return torch.arange(input_ids.shape[1]).unsqueeze(0).expand_as(input_ids)


def forward(params, input_ids, attention_mask, num_heads, need_grad=False, arch=ROBERTA, pad=1, eps=1e-5,
            token_type_ids=None):
    """The family's classifier on ``to_bert_keys`` parameters -> (logits, cache) as ``oracle.bert.forward``."""
    p = params
    dm = obert.BertDims(params, num_heads)
    dm.eps = eps
    dtype = p["classifier.weight"].dtype
    E = "bert.embeddings."
    word = p[E + "word_embeddings.weight"][input_ids]
    pos = p[E + "position_embeddings.weight"][position_ids(input_ids, arch, pad)]
    if arch == DISTILBERT:
        if token_type_ids is not None:
            raise ValueError("DistilBERT has no token-type table")
        emb = word + pos
    else:
        types = torch.zeros_like(input_ids) if token_type_ids is None else torch.as_tensor(token_type_ids).long()
        emb = (word + p[E + "token_type_embeddings.weight"][types]) + pos
    h = F.layer_norm(emb, (dm.dim,), p[E + "LayerNorm.weight"], p[E + "LayerNorm.bias"], dm.eps)
    if need_grad:
        h = h.detach().requires_grad_(True)
    ext_mask = (1.0 - attention_mask[:, None, None, :].to(dtype)) * -10000.0
    cache = {"dims": dm, "layers": [], "ext_mask": ext_mask}
    for i in range(dm.depth):
        h, c = obert.layer_forward(p, dm, i, h, ext_mask)
        cache["layers"].append(c)
    cache["h_last"] = h
    pre = F.linear(h[:, 0], p["bert.pooler.dense.weight"], p["bert.pooler.dense.bias"])
    pooled = torch.relu(pre) if arch == DISTILBERT else torch.tanh(pre)
    cache["pooled"] = pooled
    logits = F.linear(pooled, p["classifier.weight"], p["classifier.bias"])
    cache["logits"] = logits
    return logits, cache


@contextlib.contextmanager
def family(arch, pad=1, eps=1e-5, token_type_ids=None):
    """Within the block, every ``oracle.bert.forward`` call runs the family's embedding and head."""
    orig = obert.forward
    obert.forward = functools.partial(forward, arch=arch, pad=pad, eps=eps, token_type_ids=token_type_ids)
    try:
        yield
    finally:
        obert.forward = orig


def explain(params, input_ids, attention_mask, num_heads, arch, pad=1, eps=1e-5, index=None, start_layer=11,
            token_type_ids=None):
    """``Generator.generate_LRP`` (layers_ours rules) -> ([B,S] maps, [B] index)."""
    with family(arch, pad, eps, token_type_ids):
        return obert.explain(params, input_ids, attention_mask, num_heads, index=index, start_layer=start_layer)


def generate(params, input_ids, attention_mask, num_heads, which, arch, pad=1, eps=1e-5, index=None, start_layer=0,
             token_type_ids=None):
    """The comparison generators of ``Generator`` (``oracle.bert.GENERATORS``) -> [B,S]."""
    with family(arch, pad, eps, token_type_ids):
        return obert.generate(params, input_ids, attention_mask, num_heads, which, index=index, start_layer=start_layer)


def explain_attn_grad_rollout(params, input_ids, attention_mask, num_heads, arch, pad=1, eps=1e-5, index=None,
                              start_layer=0, token_type_ids=None):
    """``Generator.generate_attn_grad_rollout`` -> ([B,S] maps, [B] index)."""
    with family(arch, pad, eps, token_type_ids):
        return agr.explain_bert(params, input_ids, attention_mask, num_heads, index=index, start_layer=start_layer)


def init_params(arch, seed=0, vocab=100, max_pos=32, types=2, dim=64, depth=3, inter=128, labels=2):
    """The family's ``transformers`` ``state_dict`` (its key names), random: N(0, 0.02) weights, LayerNorm scales
    1 + 0.2 N(0, 1), biases 0.05 N(0, 1), every value an fp32 number (returned in fp64)."""
    p, _ = obert.init_params(seed=seed, vocab=vocab, max_pos=max_pos, types=max(types, 1), dim=dim, depth=depth,
                             inter=inter, labels=labels, rand_affine=True)
    return {_from_bert_key(k, arch): v.double() for k, v in p.items()
            if not (arch == DISTILBERT and k.endswith("token_type_embeddings.weight"))}


def _from_bert_key(k, arch):
    if arch == ROBERTA:
        if k.startswith("bert.pooler.dense."):
            return k.replace("bert.pooler.dense.", "classifier.dense.")
        if k.startswith("classifier."):
            return k.replace("classifier.", "classifier.out_proj.")
        return k.replace("bert.", "roberta.", 1)
    if k.startswith("bert.pooler.dense."):
        return k.replace("bert.pooler.dense.", "pre_classifier.")
    if k.startswith("classifier."):
        return k
    if k.startswith("bert.encoder.layer."):
        parts = k.split(".")
        i, rest = parts[3], ".".join(parts[4:])
        mod, leaf = rest.rsplit(".", 1)
        back = {v: m for m, v in _DISTIL_LAYER.items()}
        return "distilbert.transformer.layer.%s.%s.%s" % (i, back[mod], leaf)
    return k.replace("bert.", "distilbert.", 1)
