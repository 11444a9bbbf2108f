"""The LRP-alpha-beta rule of the reference's ``Linear.relprop(R, alpha)`` (TEST INFRASTRUCTURE, CPU, any float dtype).

``modules/layers_ours.py:207-230`` and ``modules/layers_lrp.py:187-210`` (and the BERT copies of both) compute, with
beta = alpha - 1,

    activator = f(W+, W-),  inhibitor = f(W-, W+),  R_in = alpha * activator - beta * inhibitor

where ``f(w1, w2)`` is the z+ rule of the library on the weight parts ``w1`` (paired with x+) and ``w2`` (paired with
x-).  The generators always pass alpha = 1; a user's own ``model.relprop(cam, alpha=...)`` may pass another value.
Only the Linear rule reads alpha.

The ViT / BERT wiring is the one of ``oracle.vit`` / ``oracle.bert`` (pinned to the reference at alpha = 1 by the other
fixtures): ``alpha_rules`` binds alpha into the Linear rules of ``oracle.rules`` while that wiring runs.  The functions
here state the rule in the reference's order of operations (``f`` for each half, then ``alpha * act - beta * inh``), so
that ``tests/golden/alphabeta.npz`` (``oracle/make_golden_alphabeta.py``) pins them bit-exactly; at alpha = 1 they are
``oracle.rules``' z+ rules unchanged.
"""
import contextlib

import torch

from oracle import bert as obert
from oracle import rules
from oracle import vit as ovit

_LINEAR = rules.linear_relprop
_LINEAR_LRP = rules.linear_relprop_lrp


def _parts(x, w):
    return x.clamp(min=0), x.clamp(max=0), w.clamp(min=0), w.clamp(max=0)


def linear_relprop(x, w, r, alpha=1):
    """``layers_ours`` Linear.relprop(r, alpha): f(w1, w2) = x+ * (S w1) + x- * (S w2), S = sd(R, x+ w1^T + x- w2^T)."""
    if alpha == 1:
        return _LINEAR(x, w, r)
    px, nx, pw, nw = _parts(x, w)

    def f(w1, w2):
        s = rules.safe_divide(r, px @ w1.t() + nx @ w2.t())
        return px * (s @ w1) + nx * (s @ w2)

    beta = alpha - 1
    return alpha * f(pw, nw) - beta * f(nw, pw)


def linear_relprop_lrp(x, w, r, alpha=1):
    """``layers_lrp`` Linear.relprop(r, alpha): each product over its own denominator,
    f(w1, w2) = x+ * (sd(R, x+ w1^T) w1) + x- * (sd(R, x- w2^T) w2)."""
    if alpha == 1:
        return _LINEAR_LRP(x, w, r)
    px, nx, pw, nw = _parts(x, w)

    def f(w1, w2):
        s1 = rules.safe_divide(r, px @ w1.t())
        s2 = rules.safe_divide(r, nx @ w2.t())
        return px * (s1 @ w1) + nx * (s2 @ w2)

    beta = alpha - 1
    return alpha * f(pw, nw) - beta * f(nw, pw)


@contextlib.contextmanager
def alpha_rules(alpha, add_rule=None):
    """Inside the block, ``rules.linear_relprop`` / ``rules.linear_relprop_lrp`` are the alpha-beta rules above (and
    ``rules.add_relprop`` is ``add_rule`` when given), so the wiring of ``oracle.vit`` / ``oracle.bert`` runs
    ``model.relprop(cam, alpha=alpha)``."""
    saved = rules.linear_relprop, rules.linear_relprop_lrp, rules.add_relprop
    rules.linear_relprop = lambda x, w, r: linear_relprop(x, w, r, alpha)
    rules.linear_relprop_lrp = lambda x, w, r: linear_relprop_lrp(x, w, r, alpha)
    if add_rule is not None:
        rules.add_relprop = add_rule
    try:
        yield
    finally:
        rules.linear_relprop, rules.linear_relprop_lrp, rules.add_relprop = saved


def vit_explain_method(params, x, num_heads, method, alpha, **kw):
    """``model(x)`` then ``model.relprop(one_hot, method=method, alpha=alpha, ...)`` (``ViT_LRP.py:324-398``, with
    ``variant="lrp"`` ``ViT_orig_LRP.py``): ``oracle.vit.explain_method`` with the alpha-beta Linear rule."""
    with alpha_rules(alpha):
        return ovit.explain_method(params, x, num_heads, method, **kw)


def vit_explain(params, x, num_heads, alpha, **kw):
    """``oracle.vit.explain`` (transformer_attribution, with taps) with the alpha-beta Linear rule."""
    with alpha_rules(alpha):
        return ovit.explain(params, x, num_heads, **kw)


def bert_model_relprop(params, input_ids, attention_mask, num_heads, alpha, variant="ours", index=None):
    """``model(ids, mask)`` then ``model.relprop(one_hot, alpha=alpha)`` (``BertForSequenceClassification.py:83-88``) of the
    ``layers_ours`` classifier, or with ``variant="lrp"`` of ``BERT_cls_lrp.py`` (its Linear with separate denominators and
    its Add = ``RelPropSimple``, also for the attention-mask Add), batch = independent sequences.
    Returns (cams, r): attn_cam of every layer [B,H,S,S] and the relevance at the encoder input [B,S,D]."""
    with torch.enable_grad():
        logits, cache = obert.forward(params, input_ids, attention_mask, num_heads)
    if index is None:
        index = logits.argmax(dim=-1)
    index = torch.as_tensor(index).reshape(-1).long()
    seed = torch.zeros_like(logits)
    seed[torch.arange(logits.shape[0]), index] = 1
    lrp = variant == "lrp"
    with torch.no_grad(), alpha_rules(alpha, add_rule=rules.add_relprop_simple if lrp else None):
        cd = {"dims": cache["dims"], "ext_mask": cache["ext_mask"], "h_last": cache["h_last"].detach(),
              "pooled": cache["pooled"].detach(), "layers": [{k: v.detach() for k, v in c.items()} for c in cache["layers"]]}
        if lrp:                       # the library's Linear rule in the slot oracle.bert calls
            rules.linear_relprop = rules.linear_relprop_lrp
        return obert.relprop(params, cd, seed.detach(), lowest=0, to_input=True)


# ---- the unmodified reference with alpha != 1 (authoring container) ------------------------------------------------------
def ref_vit_relprop(model, x, method, alpha, is_ablation=False, start_layer=0):
    """``model(x)`` then ``model.relprop(one_hot(argmax), method=..., alpha=alpha)`` of a reference ViT (``ViT_LRP`` or
    ``ViT_orig_LRP``), B=1, CPU, the one-hot in the model's dtype (as ``ref_harness._generate_lrp_any_dtype``)."""
    import numpy as np
    from oracle import ref_harness as rh
    with rh._cpu_cuda_shim():
        output = model(x)
        one_hot = np.zeros((1, output.size()[-1]), dtype=np.float64)
        one_hot[0, int(output.argmax())] = 1
        oh = torch.from_numpy(one_hot).to(x.dtype)
        model.zero_grad()
        torch.sum(oh * output).backward(retain_graph=True)
        return model.relprop(oh.clone(), method=method, is_ablation=is_ablation, start_layer=start_layer,
                             alpha=alpha).detach()


def ref_bert_relprop(model, input_ids, attention_mask, alpha):
    """``model(ids, mask)`` then ``model.relprop(one_hot(argmax), alpha=alpha)`` of a reference BERT classifier, B=1, CPU:
    returns (relevance at the encoder input [1,S,D], attn_cam of every layer)."""
    import numpy as np
    from oracle import ref_harness as rh
    rh._prepare_bert_imports()
    assert input_ids.shape[0] == 1
    with rh._ref_imports():
        output = model(input_ids=input_ids, attention_mask=attention_mask)[0]
        one_hot = np.zeros((1, output.size()[-1]), dtype=np.float64)
        one_hot[0, int(output.argmax())] = 1
        r = model.relprop(torch.from_numpy(one_hot).to(output.dtype), alpha=alpha)
    cams = [l.attention.self.get_attn_cam().detach() for l in model.bert.encoder.layer]
    return r.detach(), cams
