"""BERT oracle of the ``layers_lrp`` classifier (TEST INFRASTRUCTURE, CPU, any float dtype), and the generator of its
fixture ``tests/golden/bert_cls_lrp.npz``.

``BERT_explainability/modules/BERT/BERT_cls_lrp.py`` is ``BertForSequenceClassification.py`` on ``BERT_orig_lrp.py``,
which is ``BERT.py`` on the rule library of ``modules/layers_lrp.py``.  Only two rules differ from ``layers_ours``:
Linear divides its two halves by their own denominators (``oracle.rules.linear_relprop_lrp``) and Add is a plain
``RelPropSimple`` (``oracle.rules.add_relprop_simple``), which for the attention-mask Add (``BERT.py:386-388``) keeps
``scores * sd(cam, scores + mask)``.  The forward and the attention gradients are those of ``oracle.bert``; the relprop
below restates ``oracle.bert.relprop`` with the two rules swapped, so its wiring cites the same reference lines.

    python tests/bert_lrp_oracle.py        # from the repo root, with the reference checkout: writes the fixture
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import bert as obert          # noqa: E402
from oracle import rules                  # noqa: E402

_heads, _merge = obert._heads, obert._merge


def relprop(params, cache, seed, lowest=0, to_input=False):
    """``oracle.bert.relprop`` on the ``layers_lrp`` rules: per-layer attn_cam [B,H,S,S] (None below ``lowest``);
    ``to_input``: ``(cams, r)`` with r [B,S,D] what ``model.relprop`` returns."""
    p = params
    dm = cache["dims"]
    lin, add = rules.linear_relprop_lrp, rules.add_relprop_simple
    r = lin(cache["pooled"], p["classifier.weight"], seed)                         # classifier ; dropout id
    r = lin(cache["h_last"][:, 0], p["bert.pooler.dense.weight"], r)               # Tanh id ; pooler.dense
    r = rules.index_select_relprop(cache["h_last"], r.unsqueeze(1), 0)
    cams = [None] * dm.depth
    for i in reversed(range(lowest, dm.depth)):
        L = "bert.encoder.layer.%d." % i
        c = cache["layers"][i]
        r_d2, r_ao2 = add(c["d2"], c["ao"], r)                                      # BertOutput
        r_g = lin(c["g"], p[L + "output.dense.weight"], r_d2)
        r_ao1 = lin(c["ao"], p[L + "intermediate.dense.weight"], r_g)              # BertIntermediate ; GELU id
        r = rules.clone_relprop(c["ao"], (r_ao1, r_ao2))                            # BertLayer.clone
        r_d1, r_h2 = add(c["d1"], c["h"], r)                                        # BertSelfOutput
        r_ctx = lin(c["ctx"], p[L + "attention.output.dense.weight"], r_d1)
        r_ctx = _heads(r_ctx, dm.heads)                                             # BertSelfAttention
        cam1, cam_v = rules.matmul_av_relprop(c["probs"], c["v"], r_ctx)
        cam1, cam_v = cam1 / 2, cam_v / 2
        cams[i] = cam1
        if i == lowest and not to_input:
            break
        cam1 = add(c["scores"], cache["ext_mask"], cam1)[0]                        # mask Add: first operand only
        cam_q, cam_k = rules.matmul_qk_relprop(c["q"], c["k"], cam1)
        cam_q, cam_k = cam_q / 2, cam_k / 2
        r_q = lin(c["h"], p[L + "attention.self.query.weight"], _merge(cam_q))
        r_k = lin(c["h"], p[L + "attention.self.key.weight"], _merge(cam_k))
        r_v = lin(c["h"], p[L + "attention.self.value.weight"], _merge(cam_v))
        r_a = rules.clone_relprop(c["h"], (r_q, r_k, r_v))                          # self.clone (3-way)
        r = rules.clone_relprop(c["h"], (r_a, r_h2))                                # attention.clone
    if to_input:
        return cams, r
    return cams


def _passes(params, input_ids, attention_mask, num_heads, index):
    with torch.enable_grad():
        logits, cache = obert.forward(params, input_ids, attention_mask, num_heads, need_grad=True)
        if index is None:
            index = logits.argmax(dim=-1)
        index = torch.as_tensor(index).reshape(-1).long()
        seed = torch.zeros_like(logits)
        seed[torch.arange(logits.shape[0]), index] = 1
        grads = obert.attention_gradients(cache, seed)
    cd = {"dims": cache["dims"], "ext_mask": cache["ext_mask"], "h_last": cache["h_last"].detach(),
          "pooled": cache["pooled"].detach(), "layers": [{k: v.detach() for k, v in c.items()} for c in cache["layers"]]}
    return logits.detach(), index, seed, grads, cd


GENERATORS = ("LRP_last_layer", "full_lrp")


def generate(params, input_ids, attention_mask, num_heads, which, index=None):
    """``Generator.generate_LRP_last_layer`` / ``generate_full_lrp`` (``ExplanationGenerator.py:61-105``) of the
    ``layers_lrp`` classifier, batch = independent sequences -> [B,S].  The other generators of ``Generator`` read only
    the forward and the gradients, which are those of ``oracle.bert.generate``."""
    _, _, seed, _, cd = _passes(params, input_ids, attention_mask, num_heads, index)
    with torch.no_grad():
        if which == "LRP_last_layer":
            cam = relprop(params, cd, seed, lowest=cd["dims"].depth - 1)[-1].clamp(min=0).mean(dim=1)
            cam[:, 0, 0] = 0
            return cam[:, 0]
        if which == "full_lrp":
            _, r = relprop(params, cd, seed, lowest=0, to_input=True)
            cam = r.sum(dim=2)
            cam[:, 0] = 0
            return cam
    raise ValueError("unknown generator %r" % (which,))


def model_relprop(params, input_ids, attention_mask, num_heads, index=None):
    """``model.relprop(one_hot)``: relevance at the encoder input [B,S,D]."""
    _, _, seed, _, cd = _passes(params, input_ids, attention_mask, num_heads, index)
    with torch.no_grad():
        return relprop(params, cd, seed, lowest=0, to_input=True)[1]


def explain(params, input_ids, attention_mask, num_heads, index=None, start_layer=11, return_taps=False):
    """``Generator.generate_LRP`` (``ExplanationGenerator.py:28-59``) of the ``layers_lrp`` classifier -> ([B,S], [B])."""
    logits, index, seed, grads, cd = _passes(params, input_ids, attention_mask, num_heads, index)
    with torch.no_grad():
        cams = relprop(params, cd, seed, lowest=start_layer)
        mats = [rules.aggregate(g, c) if c is not None else torch.zeros_like(g[:, 0]) for g, c in zip(grads, cams)]
        joint = rules.rollout(mats, start_layer=start_layer, normalize=True)
        row = joint[:, 0].clone()
        row[:, 0] = row.min(dim=1).values
    if return_taps:
        return row, index, {"logits": logits, "grads": grads, "cams": cams}
    return row, index


# ---- fixture: the unmodified reference BERT_cls_lrp ----------------------------------------------------------------------
# the tiny model and inputs of tests/golden/bert_generators.npz (oracle/make_golden.py: golden_bert_generators)
TINY = dict(seed=4, vocab=100, max_pos=32, dim=64, depth=3, heads=4, inter=128)
TINY_CFG = dict(hidden_size=64, num_hidden_layers=3, num_attention_heads=4, intermediate_size=128, vocab_size=100,
                max_position_embeddings=32)


def tiny_inputs():
    g = torch.Generator().manual_seed(7)
    S = 24
    ids = torch.randint(5, 100, (2, S), generator=g)
    mask = torch.ones(2, S, dtype=torch.long)
    mask[1, 18:] = 0
    return ids, mask


def _build_ref_cls_lrp(params, dtype):
    from oracle import ref_harness as rh
    rh._prepare_bert_imports()
    from transformers import BertConfig
    with rh._ref_imports():
        from BERT_explainability.modules.BERT.BERT_cls_lrp import BertForSequenceClassification
        cfg = BertConfig(num_labels=2, return_dict=False, **TINY_CFG)
        torch.manual_seed(TINY["seed"])
        model = BertForSequenceClassification(cfg)
        res = model.load_state_dict(params, strict=False)
        assert not res.unexpected_keys and all("position_ids" in k for k in res.missing_keys)
        return model.to(dtype).eval()


def make_golden():
    import numpy as np
    from oracle import ref_harness as rh

    def _np(t):
        return t.detach().cpu().numpy()

    params, heads = obert.init_params(rand_affine=True, **TINY)
    ids, mask = tiny_inputs()
    out = {"ids": _np(ids), "mask": _np(mask), "heads": np.int64(heads), "param_seed": np.int64(TINY["seed"])}
    for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        torch.set_default_dtype(dt)
        try:
            model = _build_ref_cls_lrp({k: v.to(dt) for k, v in params.items()}, dt)
            for s in range(2):
                x, m = ids[s:s + 1], mask[s:s + 1]
                for which in GENERATORS:
                    for name, kw in (("argmax", {}), ("index0", dict(index=0)), ("index1", dict(index=1))):
                        out["%s.s%d.%s.%s" % (tag, s, which, name)] = _np(rh.bert_generate(model, x, m, which, **kw))
                for sl in (0, 1):
                    r = rh.bert_generate_lrp(model, x, m, start_layer=sl, taps=(sl == 0))
                    out["%s.s%d.LRP.sl%d" % (tag, s, sl)] = _np(r["map"])
                    if sl == 0:
                        for l in range(TINY["depth"]):
                            out["%s.s%d.cam.%d" % (tag, s, l)] = _np(r["cams"][l])
        finally:
            torch.set_default_dtype(torch.float32)
    path = os.path.join(ROOT, "tests", "golden", "bert_cls_lrp.npz")
    np.savez_compressed(path, **out)
    print(path, len(out), "arrays; NaN maps:",
          [k for k, v in out.items() if isinstance(v, np.ndarray) and v.dtype.kind == "f" and np.isnan(v).any()])


if __name__ == "__main__":
    make_golden()
