"""Generate ``tests/golden/hf_encoders.npz`` (TEST INFRASTRUCTURE, CPU).

    python -m oracle.make_golden_hf_encoders      # from the repo root

Tiny random RoBERTa (pad 1, ``type_vocab_size`` 2 so that a pair reaches the table) and DistilBERT sequence classifiers
at the widths of ``bert_pairs`` (hidden 64, 3 layers, 4 heads, intermediate 128, vocabulary 100, 32 positions), built
with the ``transformers`` classes in fp64 with eager attention from ``oracle.hf_encoders.init_params`` (regenerated
from the seed, not stored).  The batch (S = 24) holds a full row, a right-padded row, a left-padded row and a sentence
pair (segment 1 from token 11 for RoBERTa; DistilBERT has no segments).  ``transformers`` gives the forward and the
gradients; the relevance maps are the fp64 oracle's (``oracle/hf_encoders.py``; the layers_lrp rules of
``tests/bert_lrp_oracle.py``).

Keys (``{f}`` = ``roberta`` / ``distilbert``):

``{f}.ids`` / ``{f}.mask`` [4, 24] int64, ``roberta.token_type_ids`` [4, 24] int64
``{f}.hf.logits`` [4, 2]; ``{f}.hf.attn.{l}`` / ``{f}.hf.grad.{l}`` [4, H, S, S]: attention probabilities and
                                 d logit_c / d attention (c = arg-max, ``retain_grad``)
``{f}.ours.LRP.sl{0|1}``, ``{f}.ours.{which}`` (``oracle.bert.GENERATORS``), ``{f}.ours.attn_grad_rollout`` [4, S]
``{f}.lrp.LRP.sl{0|1}``, ``{f}.lrp.LRP_last_layer``, ``{f}.lrp.full_lrp`` [4, S]
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import bert as obert               # noqa: E402
from oracle import hf_encoders as ohf          # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "hf_encoders.npz")
SEED = 23
S = 24
HEADS = 4
WIDTHS = dict(vocab=100, max_pos=32, dim=64, depth=3, inter=128, labels=2)
FAMILIES = {"roberta": dict(arch=ohf.ROBERTA, pad=1, eps=1e-5), "distilbert": dict(arch=ohf.DISTILBERT, pad=0, eps=1e-12)}


def hf_config(name):
    import transformers
    w = WIDTHS
    if name == "roberta":
        return transformers.RobertaConfig(vocab_size=w["vocab"], max_position_embeddings=w["max_pos"], type_vocab_size=2,
                                          hidden_size=w["dim"], num_hidden_layers=w["depth"], num_attention_heads=HEADS,
                                          intermediate_size=w["inter"], num_labels=w["labels"], pad_token_id=1,
                                          bos_token_id=0, eos_token_id=2, layer_norm_eps=1e-5,
                                          attn_implementation="eager")
    return transformers.DistilBertConfig(vocab_size=w["vocab"], max_position_embeddings=w["max_pos"], dim=w["dim"],
                                         n_layers=w["depth"], n_heads=HEADS, hidden_dim=w["inter"],
                                         num_labels=w["labels"], pad_token_id=0, attn_implementation="eager")


def params(name):
    f = FAMILIES[name]
    return ohf.init_params(f["arch"], seed=SEED + f["arch"], types=2 if name == "roberta" else 0, **WIDTHS)


def inputs(name):
    """Row 0 full; row 1 right-padded from token 17; row 2 left-padded (its first 6 tokens); row 3 a pair: a separator
    pair at tokens 10 / 11, segment 1 from token 11 (RoBERTa)."""
    pad = FAMILIES[name]["pad"]
    g = torch.Generator().manual_seed(SEED)
    ids = torch.randint(5, WIDTHS["vocab"], (4, S), generator=g)
    ids[:, 0] = 3                                    # a class token
    mask = torch.ones(4, S, dtype=torch.long)
    mask[1, 17:] = 0
    ids[1, 17:] = pad
    mask[2, :6] = 0
    ids[2, :6] = pad
    ids[3, 10:12] = 4                                # separators
    tt = torch.zeros(4, S, dtype=torch.long)
    tt[3, 11:] = 1
    return ids, mask, (tt if name == "roberta" else None)


def hf_model(name):
    import transformers
    cls = (transformers.RobertaForSequenceClassification if name == "roberta"
           else transformers.DistilBertForSequenceClassification)
    m = cls(hf_config(name)).double().eval()
    res = m.load_state_dict(params(name), strict=False)
    assert not res.unexpected_keys and all("position_ids" in k or "token_type_ids" in k for k in res.missing_keys)
    return m


def hf_taps(name):
    """``transformers``' logits, attention probabilities and d logit_c / d attention (c = arg-max) in fp64."""
    m = hf_model(name)
    ids, mask, tt = inputs(name)
    kw = {"token_type_ids": tt} if tt is not None else {}
    with torch.enable_grad():
        out = m(input_ids=ids, attention_mask=mask, output_attentions=True, return_dict=True, **kw)
        for a in out.attentions:
            a.retain_grad()
        logits = out.logits
        seed = torch.zeros_like(logits)
        seed[torch.arange(4), logits.argmax(dim=-1)] = 1
        (logits * seed).sum().backward()
    return logits.detach(), [a.detach() for a in out.attentions], [a.grad.detach() for a in out.attentions]


def oracle_maps(name):
    import bert_lrp_oracle as olrp
    f = FAMILIES[name]
    p = ohf.to_bert_keys(params(name), f["arch"])
    ids, mask, tt = inputs(name)
    kw = dict(arch=f["arch"], pad=f["pad"], eps=f["eps"], token_type_ids=tt)
    out = {}
    for sl in (0, 1):
        out["ours.LRP.sl%d" % sl] = ohf.explain(p, ids, mask, HEADS, start_layer=sl, **kw)[0]
        with ohf.family(**{k: kw[k] for k in ("arch", "pad", "eps", "token_type_ids")}):
            out["lrp.LRP.sl%d" % sl] = olrp.explain(p, ids, mask, HEADS, start_layer=sl)[0]
    for which in obert.GENERATORS:
        out["ours." + which] = ohf.generate(p, ids, mask, HEADS, which, **kw)
    out["ours.attn_grad_rollout"] = ohf.explain_attn_grad_rollout(p, ids, mask, HEADS, **kw)[0]
    with ohf.family(**kw):
        for which in olrp.GENERATORS:
            out["lrp." + which] = olrp.generate(p, ids, mask, HEADS, which)
    return out


def golden():
    out = {}
    for name in FAMILIES:
        ids, mask, tt = inputs(name)
        out[name + ".ids"], out[name + ".mask"] = ids.numpy(), mask.numpy()
        if tt is not None:
            out[name + ".token_type_ids"] = tt.numpy()
        logits, attns, grads = hf_taps(name)
        out[name + ".hf.logits"] = logits.numpy()
        for l, (a, g) in enumerate(zip(attns, grads)):
            out["%s.hf.attn.%d" % (name, l)] = a.numpy()
            out["%s.hf.grad.%d" % (name, l)] = g.numpy()
        for k, v in oracle_maps(name).items():
            out["%s.%s" % (name, k)] = v.numpy()
    np.savez_compressed(OUT, **out)
    print(os.path.basename(OUT), len(out), "arrays")


if __name__ == "__main__":
    golden()
