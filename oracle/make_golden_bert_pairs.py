"""Generate ``tests/golden/bert_pairs.npz`` (TEST INFRASTRUCTURE, authoring container).

    python -m oracle.make_golden_bert_pairs      # from the repo root, needs /root/reference

Sentence-pair inputs of the tiny BERT classifier (3 layers, hidden 64, 4 heads, S = 24, ``type_vocab_size = 2``; the
parameters are regenerated from their seed, the inputs are stored): a padded batch whose rows switch from segment 0 to
segment 1 at different positions, and one row entirely in segment 1.  The UNMODIFIED reference models run through
``oracle/ref_harness.py`` one sample at a time (the reference is only correct at B = 1).  The reference ``Generator``
calls ``model(input_ids=..., attention_mask=...)``; to give the model the pair's segments, its ``forward`` is bound to the
sample's ``token_type_ids`` with ``functools.partial`` and the ``Generator`` is called unchanged.

Keys (``{lib}`` = ``ours`` for ``BertForSequenceClassification``, ``lrp`` for ``BERT_cls_lrp``; ``{dt}`` = f32 / f64):

``ids`` / ``mask`` / ``token_type_ids``       [3, 24] int64
``{lib}.{dt}.s{k}.logits``                    [1, 2] the reference's logits
``ours.{dt}.s{k}.attn.{l}`` / ``.grad.{l}``  [1, H, S, S] get_attn() / get_attn_gradients() after generate_LRP
``{lib}.{dt}.s{k}.LRP.sl{0|1}``               [1, S] generate_LRP(start_layer)
``{lib}.{dt}.s{k}.{which}.{tag}``             [1, S] the comparison generators (``oracle.bert.GENERATORS``; tag argmax /
                                              index0 / index1, rollout sl0 / sl1)
``oracle.s{k}.LRP.sl{0|1}``, ``oracle.s{k}.{which}.{tag}``, ``oracle.s{k}.attn_grad_rollout.sl{0|1}``
                                              [1, S] the fp64 oracle of sentence pairs (``oracle/bert_pairs.py`` on
                                              ``oracle/bert.py`` and ``oracle/attn_grad_rollout.py``) of the ``ours``
                                              library
"""
import functools
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import bert as obert               # noqa: E402
from oracle import bert_pairs as opairs        # noqa: E402
from oracle import ref_harness as rh           # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "bert_pairs.npz")
PARAM_SEED = 11
PARAMS = dict(seed=PARAM_SEED, vocab=100, max_pos=32, types=2, dim=64, depth=3, heads=4, inter=128, rand_affine=True)
CFG = dict(hidden_size=64, num_hidden_layers=3, num_attention_heads=4, intermediate_size=128, vocab_size=100,
           max_position_embeddings=32, type_vocab_size=2)
S = 24


def _np(t):
    return t.detach().cpu().numpy()


def pair_inputs():
    """Row 0: segment 1 from token 9, no padding; row 1: segment 1 from token 5, padded from token 19 (padding in
    segment 0, as a tokenizer pads); row 2: every token in segment 1."""
    g = torch.Generator().manual_seed(13)
    ids = torch.randint(5, 100, (3, S), generator=g)
    mask = torch.ones(3, S, dtype=torch.long)
    mask[1, 19:] = 0
    tt = torch.zeros(3, S, dtype=torch.long)
    tt[0, 9:] = 1
    tt[1, 5:19] = 1
    tt[2, :] = 1
    return ids, mask, tt


def variants(which):
    if which == "rollout":
        return [("sl0", dict(start_layer=0)), ("sl1", dict(start_layer=1))]
    return [("argmax", dict()), ("index0", dict(index=0)), ("index1", dict(index=1))]


def _build(lib, params, dt):
    if lib == "ours":
        model = rh.build_bert(seed=PARAM_SEED, dtype=dt, **CFG)
        res = model.load_state_dict({k: v.to(dt) for k, v in params.items()}, strict=False)
        assert not res.unexpected_keys and all("position_ids" in k for k in res.missing_keys)
        return model
    rh._prepare_bert_imports()
    from transformers import BertConfig
    with rh._ref_imports():
        from BERT_explainability.modules.BERT.BERT_cls_lrp import BertForSequenceClassification
        torch.manual_seed(PARAM_SEED)
        model = BertForSequenceClassification(BertConfig(num_labels=2, return_dict=False, **CFG))
        res = model.load_state_dict({k: v.to(dt) for k, v in params.items()}, strict=False)
        assert not res.unexpected_keys and all("position_ids" in k for k in res.missing_keys)
    return model.to(dt).eval()


def golden():
    params, heads = obert.init_params(**PARAMS)
    ids, mask, tt = pair_inputs()
    out = {"ids": _np(ids), "mask": _np(mask), "token_type_ids": _np(tt), "heads": np.int64(heads),
           "param_seed": np.int64(PARAM_SEED)}
    for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        torch.set_default_dtype(dt)
        try:
            for lib in ("ours", "lrp"):
                model = _build(lib, params, dt)
                forward = model.forward
                for s in range(ids.shape[0]):
                    x, m = ids[s:s + 1], mask[s:s + 1]
                    model.forward = functools.partial(forward, token_type_ids=tt[s:s + 1])
                    key = "%s.%s.s%d" % (lib, tag, s)
                    out[key + ".logits"] = _np(rh.bert_logits(model, x, m))
                    for sl in (0, 1):
                        r = rh.bert_generate_lrp(model, x, m, start_layer=sl, taps=(sl == 0))
                        out["%s.LRP.sl%d" % (key, sl)] = _np(r["map"])
                        if sl == 0 and lib == "ours":          # the forward and its gradients do not depend on the rules
                            for l in range(CFG["num_hidden_layers"]):
                                out["%s.attn.%d" % (key, l)] = _np(r["attn"][l])
                                out["%s.grad.%d" % (key, l)] = _np(r["grads"][l])
                    for which in obert.GENERATORS:
                        for vt, kw in variants(which):
                            out["%s.%s.%s" % (key, which, vt)] = _np(rh.bert_generate(model, x, m, which, **kw))
                model.forward = forward
        finally:
            torch.set_default_dtype(torch.float32)
    p64 = {k: v.double() for k, v in params.items()}
    for s in range(ids.shape[0]):
        x, m, t = ids[s:s + 1], mask[s:s + 1], tt[s:s + 1]
        key = "oracle.s%d" % s
        for sl in (0, 1):
            out["%s.LRP.sl%d" % (key, sl)] = _np(opairs.explain(p64, x, m, heads, start_layer=sl, token_type_ids=t)[0])
            out["%s.attn_grad_rollout.sl%d" % (key, sl)] = _np(
                opairs.explain_attn_grad_rollout(p64, x, m, heads, start_layer=sl, token_type_ids=t)[0])
        for which in obert.GENERATORS:
            for vt, kw in variants(which):
                out["%s.%s.%s" % (key, which, vt)] = _np(opairs.generate(p64, x, m, heads, which, token_type_ids=t, **kw))
    np.savez_compressed(OUT, **out)
    print(os.path.basename(OUT), len(out), "arrays; NaN maps:",
          [k for k, v in out.items() if isinstance(v, np.ndarray) and v.dtype.kind == "f" and np.isnan(v).any()])


if __name__ == "__main__":
    golden()
